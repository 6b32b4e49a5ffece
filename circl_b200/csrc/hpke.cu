// HPKE's DHKEMs (RFC 9180 section 4.1) as the reference's kem/schemes registers them, batched on the device:
//   hpke/xkem.go:55-71              DeriveKeyPair                  -> hpke_derive_kernel + the X25519 / X448 KeyGen
//   hpke/kembase.go:120-241         Encap / Decap / AuthEncap / AuthDecap
//                                   dh = Shared(...)               -> x25519_kernel / x448_kernel (hybrid.cu)
//                                   ss = ExtractAndExpand(dh, ctx) -> hpke_ss_kernel
//   ids 0x20 DHKEM(X25519, HKDF-SHA256) and 0x21 DHKEM(X448, HKDF-SHA512) (hpke/algs.go:248-277)
// The curve kernels are hybrid.cu's, reached through hybrid::x25519_rows / x448_rows; this file adds the KDF kernels
// (sha2.cuh, thread per op, profiling class KID_HPKE) and the flows around them.
#include <cstring>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "sha2.cuh"

namespace cb200 {
namespace hpke {

// N: Nsk = Npk = Nenc = seed = encapsulation seed (xkem.go:20-24); the shared secret is one digest (Nh)
template <int ID>
struct Kem;
template <>
struct Kem<CB200_HPKE_X25519_HKDF_SHA256> {
  using S = sha2::Sha256;
  static constexpr int kN = 32;
};
template <>
struct Kem<CB200_HPKE_X448_HKDF_SHA512> {
  using S = sha2::Sha512;
  static constexpr int kN = 56;
};

// the first `bytes` bytes of a digest to a 4-byte-aligned row
template <class S>
__device__ __forceinline__ void store_digest(uint8_t* row, const typename S::W (&h)[8], int bytes, uint32_t mask) {
#pragma unroll
  for (int q = 0; q < bytes / 4; q++) {
    uint32_t v = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) v |= (uint32_t)sha2::digest_byte<S>(h, 4 * q + b) << (8 * b);
    reinterpret_cast<uint32_t*>(row)[q] = v & mask;
  }
}

// sk[i] = LabeledExpand(LabeledExtract("", "dkp_prk", seed[i]), "sk", "", Nsk): DeriveKeyPair's private key, stored
// unclamped (xkem.go:55-71); KeyGen clamps it
template <int ID>
__global__ void __launch_bounds__(128) hpke_derive_kernel(const uint8_t* __restrict__ seeds, size_t s_stride,
                                                          uint8_t* __restrict__ sk, size_t sk_stride, size_t n) {
  using K = Kem<ID>;
  using S = typename K::S;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  typename S::W prk[8], t[8];
  sha2::labeled_extract<S>(prk, sha2::Labeled{0, 0, ID, "dkp_prk", 7, seeds + i * s_stride, nullptr, nullptr, K::kN, 0, 0});
  sha2::labeled_expand<S>(t, prk, sha2::Labeled{1, K::kN, ID, "sk", 2, nullptr, nullptr, nullptr, 0, 0, 0});
  store_digest<S>(sk + i * sk_stride, t, K::kN, 0xffffffffu);
}

// ss[i] = LabeledExpand(LabeledExtract("", "eae_prk", dh[i]), "shared_secret", kem_context[i], Nh) (kembase.go:94-118)
// with dh = ND rows of Npk bytes (d0 [|| d1]) and kem_context = NC rows of Npk bytes (c0 || c1 [|| c2]), each read at
// its own stride.  An op whose status bit 0 is set (a DH with a low-order point) gets an all-zero ss.
template <int ID, int ND, int NC>
__global__ void __launch_bounds__(128) hpke_ss_kernel(const uint8_t* __restrict__ d0, size_t d0s,
                                                      const uint8_t* __restrict__ d1, size_t d1s,
                                                      const uint8_t* __restrict__ c0, size_t c0s,
                                                      const uint8_t* __restrict__ c1, size_t c1s,
                                                      const uint8_t* __restrict__ c2, size_t c2s,
                                                      const uint8_t* __restrict__ status, uint8_t* __restrict__ ss,
                                                      size_t n) {
  using K = Kem<ID>;
  using S = typename K::S;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  typename S::W prk[8], t[8];
  sha2::labeled_extract<S>(prk, sha2::Labeled{0, 0, ID, "eae_prk", 7, d0 + i * d0s, ND == 2 ? d1 + i * d1s : nullptr,
                                               nullptr, K::kN, ND == 2 ? K::kN : 0, 0});
  sha2::labeled_expand<S>(t, prk, sha2::Labeled{1, S::kDigest, ID, "shared_secret", 13, c0 + i * c0s, c1 + i * c1s,
                                                NC == 3 ? c2 + i * c2s : nullptr, K::kN, K::kN, NC == 3 ? K::kN : 0});
  const uint32_t mask = (uint32_t)(status[i] & 1) - 1u;
  store_digest<S>(ss + (size_t)S::kDigest * i, t, S::kDigest, mask);
}

// ------------------------------------------------------------------ host side
static inline unsigned blocks(size_t units, size_t per) { return (unsigned)((units + per - 1) / per); }

struct Id {
  int id;
  size_t N;   // key, encapsulation and seed bytes
  size_t ss;  // shared secret bytes (Nh)
};
static bool id_of(int id, Id* k) {
  switch (id) {
    case CB200_HPKE_X25519_HKDF_SHA256: *k = {id, 32, 32}; return true;
    case CB200_HPKE_X448_HKDF_SHA512: *k = {id, 56, 64}; return true;
  }
  return false;
}
// per-op intermediates: skE (N) | dh (2N) | the recomputed public key (N); a shared key's public key sits in row 0
static size_t work_unit(const Id& k) { return 4 * k.N; }

static int derive(const Id& k, const uint8_t* seeds, size_t ss_, uint8_t* sk, size_t sks, size_t n, cudaStream_t st) {
  {
    KernelScope ks(KID_HPKE, st);
    if (k.id == CB200_HPKE_X25519_HKDF_SHA256)
      hpke_derive_kernel<CB200_HPKE_X25519_HKDF_SHA256><<<blocks(n, 128), 128, 0, st>>>(seeds, ss_, sk, sks, n);
    else
      hpke_derive_kernel<CB200_HPKE_X448_HKDF_SHA512><<<blocks(n, 128), 128, 0, st>>>(seeds, ss_, sk, sks, n);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}
// KeyGen (p null) or Shared on rows
static void dh(const Id& k, const uint8_t* sk, size_t sks, const uint8_t* p, size_t ps, uint8_t* out, size_t os,
               uint8_t* status, size_t n, cudaStream_t st) {
  if (k.N == 32)
    hybrid::x25519_rows(sk, sks, p, ps, out, os, status, n, st);
  else
    hybrid::x448_rows(sk, sks, p, ps, out, os, status, n, st);
}
template <int ND, int NC>
static void ss_launch(int id, const uint8_t* d0, size_t d0s, const uint8_t* d1, size_t d1s, const uint8_t* c0, size_t c0s, const uint8_t* c1, size_t c1s,
                      const uint8_t* c2, size_t c2s, const uint8_t* status, uint8_t* ss, size_t n, cudaStream_t st) {
  KernelScope ks(KID_HPKE, st);
  if (id == CB200_HPKE_X25519_HKDF_SHA256)
    hpke_ss_kernel<CB200_HPKE_X25519_HKDF_SHA256, ND, NC>
        <<<blocks(n, 128), 128, 0, st>>>(d0, d0s, d1, d1s, c0, c0s, c1, c1s, c2, c2s, status, ss, n);
  else
    hpke_ss_kernel<CB200_HPKE_X448_HKDF_SHA512, ND, NC>
        <<<blocks(n, 128), 128, 0, st>>>(d0, d0s, d1, d1s, c0, c0s, c1, c1s, c2, c2s, status, ss, n);
}

// The work rows of a call: the staged kScratch rows on the host path, the level-1 work area on the device path.
static int work_rows(const Id& k, const Row& r, size_t n, int slot, uint8_t** w) {
  if (r.p) {
    *w = r.p;
    return 0;
  }
  Arena A;
  int rc = arena(slot, n * work_unit(k), &A);
  if (rc) return rc;
  *w = A.take(n * work_unit(k));
  return 0;
}

// The four flows.  W = work rows of U bytes: skE at 0, dh at N (Shared(.,.) || Shared(.,.) for auth), the public key
// recomputed from skR / skS at 3N (row 0 only when that key is shared by the batch).  A DH of two keys that are both
// shared by the batch is also computed once, into row 0.
static int encaps_dev(const Id& k, const uint8_t* pkR, size_t pkRs, const uint8_t* skS, size_t skSs, const uint8_t* seeds,
                      uint8_t* enc, uint8_t* ss, uint8_t* status, uint8_t* W, size_t n, cudaStream_t st) {
  const size_t N = k.N, U = work_unit(k);
  CB200_CUDA(cudaMemsetAsync(status, 0, n, st));
  int rc = derive(k, seeds, N, W, U, n, st);  // skE (kembase.go:128)
  if (rc) return rc;
  dh(k, W, U, nullptr, 0, enc, N, nullptr, n, st);              // enc = pkE
  dh(k, W, U, pkR, pkRs, W + N, U, status, n, st);              // Shared(skE, pkR)
  if (!skS) {
    ss_launch<1, 2>(k.id, W + N, U, nullptr, 0, enc, N, pkR, pkRs, nullptr, 0, status, ss, n, st);
  } else {
    // Shared(skS, pkR): once when both keys are shared.  It fails only for a low-order pkR, and then so does
    // Shared(skE, pkR) above for every op, so the status of row 0 alone is enough.
    const bool once = !pkRs && !skSs;
    dh(k, skS, skSs, pkR, pkRs, W + 2 * N, U, status, once ? 1 : n, st);
    dh(k, skS, skSs, nullptr, 0, W + 3 * N, U, nullptr, skSs ? n : 1, st);  // pkS = KeyGen(skS), once for a shared skS
    ss_launch<2, 3>(k.id, W + N, U, W + 2 * N, once ? 0 : U, enc, N, pkR, pkRs, W + 3 * N, skSs ? U : 0, status, ss, n,
                    st);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}
static int decaps_dev(const Id& k, const uint8_t* skR, size_t skRs, const uint8_t* enc, const uint8_t* pkS, size_t pkSs,
                      uint8_t* ss, uint8_t* status, uint8_t* W, size_t n, cudaStream_t st) {
  const size_t N = k.N, U = work_unit(k);
  CB200_CUDA(cudaMemsetAsync(status, 0, n, st));
  dh(k, skR, skRs, nullptr, 0, W + 3 * N, U, nullptr, skRs ? n : 1, st);  // pkR = KeyGen(skR), once for a shared skR
  dh(k, skR, skRs, enc, N, W + N, U, status, n, st);                       // Shared(skR, enc)
  if (!pkS) {
    ss_launch<1, 2>(k.id, W + N, U, nullptr, 0, enc, N, W + 3 * N, skRs ? U : 0, nullptr, 0, status, ss, n, st);
  } else {
    dh(k, skR, skRs, pkS, pkSs, W + 2 * N, U, status, n, st);  // Shared(skR, pkS)
    ss_launch<2, 3>(k.id, W + N, U, W + 2 * N, U, enc, N, W + 3 * N, skRs ? U : 0, pkS, pkSs, status, ss, n, st);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// Host-pointer calls: failed operations are reported after the whole batch ran (hpke.ErrInvalidKEMSharedSecret)
static int status_result(size_t bad, size_t n, const char* fn) {
  if (!bad) return 0;
  set_error("%s: %zu of %zu operations hit a low-order public key or encapsulation (hpke: invalid KEM shared secret)", fn,
            bad, n);
  return CB200_ERR_PUBKEY;
}
// Device-pointer calls read and write their rows in 32-bit units; the X25519 entry points ask for 16-byte alignment
// like cb200_x25519, the X448 ones for 8 like cb200_x448.
static size_t align_of(const Id& k) { return k.N == 32 ? 16 : 8; }
static const char* align_text(const Id& k) {
  return k.N == 32 ? "%s: device buffers and strides must be 16-byte aligned"
                   : "%s: device buffers and strides must be 8-byte aligned";
}
static const char* kNeedStatus = "%s: device-pointer calls need a status array (it marks the failed operations)";
static bool bad_stride(size_t s, const Id& k) { return s != 0 && s < k.N; }

// encaps and auth encaps (skS null for the former)
static int encaps_entry(const char* fn, int id, const uint8_t* pkR, size_t pkRs, const uint8_t* skS, size_t skSs,
                        const uint8_t* seeds, uint8_t* enc, uint8_t* ss, uint8_t* status, size_t n, bool auth) {
  int rc = require_ready();
  if (rc) return rc;
  Id k;
  if (!id_of(id, &k) || !pkR || !seeds || !enc || !ss || (auth && !skS) || bad_stride(pkRs, k) ||
      (auth && bad_stride(skSs, k))) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const size_t N = k.N;
  Batch b{fn, n, enc, 1u << 16, 1u << 13,
          {{pkR, N, pkRs, kIn}, {seeds, N, N, kIn}, {enc, N, N, kOut}, {ss, k.ss, k.ss, kOut}, {status, 1, 1, kStatus},
           {nullptr, work_unit(k), work_unit(k), kScratch}, {skS, N, skSs, kIn}},
          {{!status, kNeedStatus},
           {!aligned({pkR, seeds, enc, ss, skS}, {pkRs, skSs}, align_of(k)), align_text(k)}}};
  Counts c;
  rc = run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    uint8_t* W;
    int e = work_rows(k, r[5], cnt, slot, &W);
    if (e) return e;
    return encaps_dev(k, r[0].p, r[0].stride, r[6].p, r[6].stride, r[1].p, r[2].p, r[3].p, r[4].p, W, cnt, st);
  }, &c);
  if (rc) return rc;
  return status_result(c.bit0, n, fn);
}

// decaps and auth decaps (pkS null for the former)
static int decaps_entry(const char* fn, int id, const uint8_t* skR, size_t skRs, const uint8_t* enc, const uint8_t* pkS,
                        size_t pkSs, uint8_t* ss, uint8_t* status, size_t n, bool auth) {
  int rc = require_ready();
  if (rc) return rc;
  Id k;
  if (!id_of(id, &k) || !skR || !enc || !ss || (auth && !pkS) || bad_stride(skRs, k) || (auth && bad_stride(pkSs, k))) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const size_t N = k.N;
  Batch b{fn, n, ss, 1u << 16, 1u << 13,
          {{skR, N, skRs, kIn}, {enc, N, N, kIn}, {ss, k.ss, k.ss, kOut}, {status, 1, 1, kStatus},
           {nullptr, work_unit(k), work_unit(k), kScratch}, {pkS, N, pkSs, kIn}},
          {{!status, kNeedStatus},
           {!aligned({skR, enc, ss, pkS}, {skRs, pkSs}, align_of(k)), align_text(k)}}};
  Counts c;
  rc = run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    uint8_t* W;
    int e = work_rows(k, r[4], cnt, slot, &W);
    if (e) return e;
    return decaps_dev(k, r[0].p, r[0].stride, r[1].p, r[5].p, r[5].stride, r[2].p, r[3].p, W, cnt, st);
  }, &c);
  if (rc) return rc;
  return status_result(c.bit0, n, fn);
}

}  // namespace hpke
}  // namespace cb200

using namespace cb200;
using namespace cb200::hpke;

extern "C" {

size_t cb200_hpke_public_key_size(int id) {
  Id k;
  return id_of(id, &k) ? k.N : 0;
}
size_t cb200_hpke_private_key_size(int id) {
  Id k;
  return id_of(id, &k) ? k.N : 0;
}
size_t cb200_hpke_ciphertext_size(int id) {
  Id k;
  return id_of(id, &k) ? k.N : 0;
}
size_t cb200_hpke_shared_key_size(int id) {
  Id k;
  return id_of(id, &k) ? k.ss : 0;
}
size_t cb200_hpke_seed_size(int id) {
  Id k;
  return id_of(id, &k) ? k.N : 0;
}
size_t cb200_hpke_encapsulation_seed_size(int id) {
  Id k;
  return id_of(id, &k) ? k.N : 0;
}

int cb200_hpke_keygen(int id, const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  Id k;
  if (!id_of(id, &k) || !seeds || !pk || !sk) {
    set_error("cb200_hpke_keygen: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const size_t N = k.N;
  Batch b{"cb200_hpke_keygen", n, pk, 1u << 16, 1u << 13, {{seeds, N, N, kIn}, {pk, N, N, kOut}, {sk, N, N, kOut}},
          {{!aligned({seeds, pk, sk}, {}, align_of(k)), align_text(k)}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) -> int {
    int e = derive(k, r[0].p, N, r[2].p, N, cnt, st);
    if (e) return e;
    dh(k, r[2].p, N, nullptr, 0, r[1].p, N, nullptr, cnt, st);
    CB200_CUDA(cudaGetLastError());
    return 0;
  });
}

int cb200_hpke_encaps(int id, const uint8_t* pkR, size_t pkR_stride, const uint8_t* seeds, uint8_t* enc, uint8_t* ss,
                      uint8_t* status, size_t n) {
  return encaps_entry("cb200_hpke_encaps", id, pkR, pkR_stride, nullptr, 0, seeds, enc, ss, status, n, false);
}

int cb200_hpke_decaps(int id, const uint8_t* skR, size_t skR_stride, const uint8_t* enc, uint8_t* ss, uint8_t* status,
                      size_t n) {
  return decaps_entry("cb200_hpke_decaps", id, skR, skR_stride, enc, nullptr, 0, ss, status, n, false);
}

int cb200_hpke_auth_encaps(int id, const uint8_t* pkR, size_t pkR_stride, const uint8_t* skS, size_t skS_stride,
                           const uint8_t* seeds, uint8_t* enc, uint8_t* ss, uint8_t* status, size_t n) {
  return encaps_entry("cb200_hpke_auth_encaps", id, pkR, pkR_stride, skS, skS_stride, seeds, enc, ss, status, n, true);
}

int cb200_hpke_auth_decaps(int id, const uint8_t* skR, size_t skR_stride, const uint8_t* enc, const uint8_t* pkS,
                           size_t pkS_stride, uint8_t* ss, uint8_t* status, size_t n) {
  return decaps_entry("cb200_hpke_auth_decaps", id, skR, skR_stride, enc, pkS, pkS_stride, ss, status, n, true);
}

}  // extern "C"
