// HPKE's DHKEMs (RFC 9180 section 4.1) as the reference's kem/schemes registers them, batched on the device:
//   hpke/xkem.go:55-71              DeriveKeyPair                  -> hpke_derive_kernel + the X25519 / X448 KeyGen
//   hpke/shortkem.go:63-90          DeriveKeyPair (candidate loop) -> hpke_derive_kernel<0x10 / 0x11 / 0x12> + the
//                                                                     P-256 / P-384 / P-521 KeyGen
//   hpke/kembase.go:120-241         Encap / Decap / AuthEncap / AuthDecap
//                                   dh = Shared(...)               -> x25519_kernel / x448_kernel (hybrid.cu),
//                                                                     p256_kernel / p384_kernel / p521_kernel (p256.cu)
//                                   ss = ExtractAndExpand(dh, ctx) -> hpke_ss_kernel
//   ids 0x20 DHKEM(X25519, HKDF-SHA256) and 0x21 DHKEM(X448, HKDF-SHA512) (hpke/algs.go:248-277), and the NIST ones
//   0x10 DHKEM(P-256, HKDF-SHA256), 0x11 DHKEM(P-384, HKDF-SHA384) and 0x12 DHKEM(P-521, HKDF-SHA512) (:248-262),
//   which have entry points of their own (cb200_hpke_p256_* / p384_* / p521_*)
// The curve kernels are reached through hybrid::x25519_rows / x448_rows / p256_rows / p384_rows / p521_rows; this file
// adds the KDF kernels (sha2.cuh, thread per op, profiling class KID_HPKE) and the flows around them.
#include <cstring>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "p384.cuh"
#include "p521.cuh"
#include "sha2.cuh"

namespace cb200 {
namespace hpke {

// kSk = Nsk = seed = encapsulation seed, kPk = Npk = Nenc, kDh = Ndh (xkem.go:20-24, shortkem.go:31-45); the shared
// secret is one digest (Nh).  kFail: the status bits that zero an op's ss.  kAligned: rows are 4-byte aligned (the
// 65-, 97- and 133-byte rows of the NIST curves are not, so theirs are written byte by byte).  Curve and kMask0: the
// curve type of P-384 and P-521 and DeriveKeyPair's bitmask on a candidate's first byte.
template <int ID>
struct Kem;
template <>
struct Kem<CB200_HPKE_X25519_HKDF_SHA256> {
  using S = sha2::Sha256;
  static constexpr int kSk = 32, kPk = 32, kDh = 32, kFail = 1;
  static constexpr bool kAligned = true;
};
template <>
struct Kem<CB200_HPKE_X448_HKDF_SHA512> {
  using S = sha2::Sha512;
  static constexpr int kSk = 56, kPk = 56, kDh = 56, kFail = 1;
  static constexpr bool kAligned = true;
};
template <>
struct Kem<CB200_HPKE_P256_HKDF_SHA256> {
  using S = sha2::Sha256;
  static constexpr int kSk = 32, kPk = 65, kDh = 32, kFail = 3;
  static constexpr bool kAligned = false;
};
template <>
struct Kem<CB200_HPKE_P384_HKDF_SHA384> {
  using S = sha2::Sha384;
  using Curve = nistp::P384;
  static constexpr int kSk = 48, kPk = 97, kDh = 48, kFail = 3;
  static constexpr bool kAligned = false;
  static constexpr uint8_t kMask0 = 0xff;
};
template <>
struct Kem<CB200_HPKE_P521_HKDF_SHA512> {
  using S = sha2::Sha512;
  using Curve = nistp::P521;
  static constexpr int kSk = 66, kPk = 133, kDh = 66, kFail = 3;
  static constexpr bool kAligned = false;
  static constexpr uint8_t kMask0 = 0x01;
};

// the first `bytes` bytes of a digest to a row (4-byte aligned unless !ALIGNED)
template <class S, bool ALIGNED = true>
__device__ __forceinline__ void store_digest(uint8_t* row, const typename S::W (&h)[8], int bytes, uint32_t mask) {
  if constexpr (!ALIGNED) {
#pragma unroll
    for (int j = 0; j < bytes; j++) row[j] = sha2::digest_byte<S>(h, j) & (uint8_t)mask;
  } else {
#pragma unroll
    for (int q = 0; q < bytes / 4; q++) {
      uint32_t v = 0;
#pragma unroll
      for (int b = 0; b < 4; b++) v |= (uint32_t)sha2::digest_byte<S>(h, 4 * q + b) << (8 * b);
      reinterpret_cast<uint32_t*>(row)[q] = v & mask;
    }
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
  sha2::labeled_extract<S>(prk, sha2::Labeled{0, 0, ID, "dkp_prk", 7, seeds + i * s_stride, nullptr, nullptr, K::kSk, 0, 0});
  sha2::labeled_expand<S>(t, prk, sha2::Labeled{1, K::kSk, ID, "sk", 2, nullptr, nullptr, nullptr, 0, 0, 0});
  store_digest<S>(sk + i * sk_stride, t, K::kSk, 0xffffffffu);
}

// LabeledExpand's message with a one-byte info held in a register (the candidate counter)
struct CandidateMsg {
  sha2::Labeled m;  // "candidate" with an info row of one byte that is never read through its pointer
  uint8_t ctr;
  CB200_XHD int len() const { return m.len(); }
  CB200_XHD uint8_t operator()(int j) const { return j == len() - 2 ? ctr : m(j); }
};

// P-256 (shortkem.go:63-90): prk = LabeledExtract("", "dkp_prk", seed); for ctr = 0..255 the candidate
// LabeledExpand(prk, "candidate", I2OSP(ctr, 1), 32) is the key if 0 < candidate < n (the bitmask is 0xff).  The
// loop stops at the first key, as the reference's does; the range test is branch-free.  Not finding one in 256
// candidates (probability about 2^-8192) leaves an all-zero sk, which KeyGen reports as an invalid private key.
template <>
__global__ void __launch_bounds__(128) hpke_derive_kernel<CB200_HPKE_P256_HKDF_SHA256>(const uint8_t* __restrict__ seeds,
                                                                                        size_t s_stride,
                                                                                        uint8_t* __restrict__ sk,
                                                                                        size_t sk_stride, size_t n) {
  constexpr int ID = CB200_HPKE_P256_HKDF_SHA256;
  using S = sha2::Sha256;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t prk[8], ki[8], ko[8], t[8];
  sha2::labeled_extract<S>(prk, sha2::Labeled{0, 0, ID, "dkp_prk", 7, seeds + i * s_stride, nullptr, nullptr, 32, 0, 0});
  sha2::hmac_key<S>(ki, ko, prk);
  // n in big-endian words, the order of the digest's words
  const uint32_t kN[8] = {0xffffffffu, 0x00000000u, 0xffffffffu, 0xffffffffu,
                          0xbce6faadu, 0xa7179e84u, 0xf3b9cac2u, 0xfc632551u};
  uint32_t ok = 0;
#pragma unroll 1
  for (int ctr = 0; ctr < 256; ctr++) {
    const CandidateMsg m{sha2::Labeled{1, 32, ID, "candidate", 9, nullptr, nullptr, nullptr, 1, 0, 0}, (uint8_t)ctr};
    sha2::hmac<S>(t, ki, ko, m.len(), m);
    uint32_t borrow = 0, nz = 0;
#pragma unroll
    for (int q = 7; q >= 0; q--) {
      borrow = (uint32_t)((((uint64_t)t[q] - kN[q] - borrow) >> 32) & 1u);
      nz |= t[q];
    }
    ok = borrow & (uint32_t)(nz != 0);
    if (ok) break;
  }
  store_digest<S, false>(sk + i * sk_stride, t, 32, 0u - ok);
}

// P-384 and P-521 (shortkem.go:63-90): P-256's loop above on candidates of Nsk bytes whose first byte is ANDed with
// kMask0, range-tested by nistp::candidate.  P-521's 66-byte candidate is T(1) || the first two bytes of T(2), where
// T(2) = HMAC(prk, T(1) || info || 0x02) with T(1) read from registers.
template <int ID>
__device__ __forceinline__ void nist_derive(const uint8_t* __restrict__ seed, uint8_t* __restrict__ sk) {
  using K = Kem<ID>;
  using S = typename K::S;
  using C = typename K::Curve;
  typename S::W prk[8], ki[8], ko[8], t1[8], t2[8];
  sha2::labeled_extract<S>(prk, sha2::Labeled{0, 0, ID, "dkp_prk", 7, seed, nullptr, nullptr, K::kSk, 0, 0});
  sha2::hmac_key<S>(ki, ko, prk);
  uint32_t k[C::kW];
  uint32_t ok = 0;
#pragma unroll 1
  for (int ctr = 0; ctr < 256; ctr++) {
    const CandidateMsg m{sha2::Labeled{1, K::kSk, ID, "candidate", 9, nullptr, nullptr, nullptr, 1, 0, 0}, (uint8_t)ctr};
    sha2::hmac<S>(t1, ki, ko, m.len(), m);
    if constexpr (K::kSk > S::kDigest) {
      const sha2::ExpandNext<S, CandidateMsg> m2{t1, m};
      sha2::hmac<S>(t2, ki, ko, m2.len(), m2);
    }
    ok = nistp::candidate<C>(k, [&](int j) {
      return j < S::kDigest ? sha2::digest_byte<S>(t1, j) : sha2::digest_byte<S>(t2, j - S::kDigest);
    }, K::kMask0);
    if (ok) break;
  }
  nistp::words_to_be<C>(sk, k, ok);
}
template <>
__global__ void __launch_bounds__(128) hpke_derive_kernel<CB200_HPKE_P384_HKDF_SHA384>(const uint8_t* __restrict__ seeds,
                                                                                        size_t s_stride,
                                                                                        uint8_t* __restrict__ sk,
                                                                                        size_t sk_stride, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  nist_derive<CB200_HPKE_P384_HKDF_SHA384>(seeds + i * s_stride, sk + i * sk_stride);
}
template <>
__global__ void __launch_bounds__(128) hpke_derive_kernel<CB200_HPKE_P521_HKDF_SHA512>(const uint8_t* __restrict__ seeds,
                                                                                        size_t s_stride,
                                                                                        uint8_t* __restrict__ sk,
                                                                                        size_t sk_stride, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  nist_derive<CB200_HPKE_P521_HKDF_SHA512>(seeds + i * s_stride, sk + i * sk_stride);
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
                                               nullptr, K::kDh, ND == 2 ? K::kDh : 0, 0});
  sha2::labeled_expand<S>(t, prk, sha2::Labeled{1, S::kDigest, ID, "shared_secret", 13, c0 + i * c0s, c1 + i * c1s,
                                                NC == 3 ? c2 + i * c2s : nullptr, K::kPk, K::kPk, NC == 3 ? K::kPk : 0});
  const uint32_t mask = K::kFail == 1 ? (uint32_t)(status[i] & 1) - 1u : (uint32_t)((status[i] & K::kFail) != 0) - 1u;
  store_digest<S, K::kAligned>(ss + (size_t)S::kDigest * i, t, S::kDigest, mask);
}

// status[i] |= status[0]: the failure of a DH computed once for the batch (from two shared keys) reaches every op
__global__ void __launch_bounds__(256) hpke_status_bcast_kernel(uint8_t* __restrict__ status, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > 0 && i < n) status[i] |= status[0];
}

// ------------------------------------------------------------------ host side
static inline unsigned blocks(size_t units, size_t per) { return (unsigned)((units + per - 1) / per); }

struct Id {
  int id;
  size_t sk;  // private key and seed bytes (Nsk)
  size_t pk;  // public key and encapsulation bytes (Npk = Nenc)
  size_t dh;  // bytes of one DH result (Ndh)
  size_t ss;  // shared secret bytes (Nh)
};
// the ids of cb200_hpke_*; the NIST curves are reached only through cb200_hpke_p256_* / p384_* / p521_*, which use
// kP256 / kP384 / kP521
static bool id_of(int id, Id* k) {
  switch (id) {
    case CB200_HPKE_X25519_HKDF_SHA256: *k = {id, 32, 32, 32, 32}; return true;
    case CB200_HPKE_X448_HKDF_SHA512: *k = {id, 56, 56, 56, 64}; return true;
  }
  return false;
}
static const Id kP256 = {CB200_HPKE_P256_HKDF_SHA256, 32, 65, 32, 32};
static const Id kP384 = {CB200_HPKE_P384_HKDF_SHA384, 48, 97, 48, 48};
static const Id kP521 = {CB200_HPKE_P521_HKDF_SHA512, 66, 133, 66, 64};
// the NIST curve of a NIST id, else null
static const char* nist_curve(int id) {
  switch (id) {
    case CB200_HPKE_P256_HKDF_SHA256: return "P-256";
    case CB200_HPKE_P384_HKDF_SHA384: return "P-384";
    case CB200_HPKE_P521_HKDF_SHA512: return "P-521";
  }
  return nullptr;
}
// per-op intermediates: skE (Nsk) | dh (2 Ndh) | the recomputed public key (Npk); a shared key's public key sits in
// row 0
static size_t work_unit(const Id& k) { return k.sk + 2 * k.dh + k.pk; }

static int derive(const Id& k, const uint8_t* seeds, size_t ss_, uint8_t* sk, size_t sks, size_t n, cudaStream_t st) {
  {
    KernelScope ks(KID_HPKE, st);
    if (k.id == CB200_HPKE_X25519_HKDF_SHA256)
      hpke_derive_kernel<CB200_HPKE_X25519_HKDF_SHA256><<<blocks(n, 128), 128, 0, st>>>(seeds, ss_, sk, sks, n);
    else if (k.id == CB200_HPKE_X448_HKDF_SHA512)
      hpke_derive_kernel<CB200_HPKE_X448_HKDF_SHA512><<<blocks(n, 128), 128, 0, st>>>(seeds, ss_, sk, sks, n);
    else if (k.id == CB200_HPKE_P384_HKDF_SHA384)
      hpke_derive_kernel<CB200_HPKE_P384_HKDF_SHA384><<<blocks(n, 128), 128, 0, st>>>(seeds, ss_, sk, sks, n);
    else if (k.id == CB200_HPKE_P521_HKDF_SHA512)
      hpke_derive_kernel<CB200_HPKE_P521_HKDF_SHA512><<<blocks(n, 128), 128, 0, st>>>(seeds, ss_, sk, sks, n);
    else
      hpke_derive_kernel<CB200_HPKE_P256_HKDF_SHA256><<<blocks(n, 128), 128, 0, st>>>(seeds, ss_, sk, sks, n);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}
// KeyGen (p null) or Shared on rows
static void dh(const Id& k, const uint8_t* sk, size_t sks, const uint8_t* p, size_t ps, uint8_t* out, size_t os,
               uint8_t* status, size_t n, cudaStream_t st) {
  if (k.id == CB200_HPKE_X25519_HKDF_SHA256)
    hybrid::x25519_rows(sk, sks, p, ps, out, os, status, n, st);
  else if (k.id == CB200_HPKE_X448_HKDF_SHA512)
    hybrid::x448_rows(sk, sks, p, ps, out, os, status, n, st);
  else if (k.id == CB200_HPKE_P384_HKDF_SHA384)
    hybrid::p384_rows(sk, sks, p, ps, out, os, status, n, st);
  else if (k.id == CB200_HPKE_P521_HKDF_SHA512)
    hybrid::p521_rows(sk, sks, p, ps, out, os, status, n, st);
  else
    hybrid::p256_rows(sk, sks, p, ps, out, os, status, n, st);
}
template <int ND, int NC>
static void ss_launch(int id, const uint8_t* d0, size_t d0s, const uint8_t* d1, size_t d1s, const uint8_t* c0, size_t c0s, const uint8_t* c1, size_t c1s,
                      const uint8_t* c2, size_t c2s, const uint8_t* status, uint8_t* ss, size_t n, cudaStream_t st) {
  KernelScope ks(KID_HPKE, st);
  if (id == CB200_HPKE_X25519_HKDF_SHA256)
    hpke_ss_kernel<CB200_HPKE_X25519_HKDF_SHA256, ND, NC>
        <<<blocks(n, 128), 128, 0, st>>>(d0, d0s, d1, d1s, c0, c0s, c1, c1s, c2, c2s, status, ss, n);
  else if (id == CB200_HPKE_X448_HKDF_SHA512)
    hpke_ss_kernel<CB200_HPKE_X448_HKDF_SHA512, ND, NC>
        <<<blocks(n, 128), 128, 0, st>>>(d0, d0s, d1, d1s, c0, c0s, c1, c1s, c2, c2s, status, ss, n);
  else if (id == CB200_HPKE_P384_HKDF_SHA384)
    hpke_ss_kernel<CB200_HPKE_P384_HKDF_SHA384, ND, NC>
        <<<blocks(n, 128), 128, 0, st>>>(d0, d0s, d1, d1s, c0, c0s, c1, c1s, c2, c2s, status, ss, n);
  else if (id == CB200_HPKE_P521_HKDF_SHA512)
    hpke_ss_kernel<CB200_HPKE_P521_HKDF_SHA512, ND, NC>
        <<<blocks(n, 128), 128, 0, st>>>(d0, d0s, d1, d1s, c0, c0s, c1, c1s, c2, c2s, status, ss, n);
  else
    hpke_ss_kernel<CB200_HPKE_P256_HKDF_SHA256, ND, NC>
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

// The four flows.  W = work rows of U bytes: skE at 0, dh at D = Nsk (Shared(.,.) || Shared(.,.) for auth), the public
// key recomputed from skR / skS at Q = Nsk + 2 Ndh (row 0 only when that key is shared by the batch).  A DH of two keys
// that are both shared by the batch is also computed once, into row 0.
static int encaps_dev(const Id& k, const uint8_t* pkR, size_t pkRs, const uint8_t* skS, size_t skSs, const uint8_t* seeds,
                      uint8_t* enc, uint8_t* ss, uint8_t* status, uint8_t* W, size_t n, cudaStream_t st) {
  const size_t U = work_unit(k), D = k.sk, Q = k.sk + 2 * k.dh, P = k.pk;
  CB200_CUDA(cudaMemsetAsync(status, 0, n, st));
  int rc = derive(k, seeds, k.sk, W, U, n, st);  // skE (kembase.go:128)
  if (rc) return rc;
  dh(k, W, U, nullptr, 0, enc, P, nullptr, n, st);              // enc = pkE
  dh(k, W, U, pkR, pkRs, W + D, U, status, n, st);              // Shared(skE, pkR)
  if (!skS) {
    ss_launch<1, 2>(k.id, W + D, U, nullptr, 0, enc, P, pkR, pkRs, nullptr, 0, status, ss, n, st);
  } else {
    // Shared(skS, pkR): once when both keys are shared.  A bad pkR also fails Shared(skE, pkR) above for every op, but
    // an invalid skS (P-256) is seen only here, so the status of row 0 is passed on to every op.
    const bool once = !pkRs && !skSs;
    dh(k, skS, skSs, pkR, pkRs, W + D + k.dh, U, status, once ? 1 : n, st);
    if (once && n > 1) {
      KernelScope ks(KID_HPKE, st);
      hpke_status_bcast_kernel<<<blocks(n, 256), 256, 0, st>>>(status, n);
    }
    dh(k, skS, skSs, nullptr, 0, W + Q, U, nullptr, skSs ? n : 1, st);  // pkS = KeyGen(skS), once for a shared skS
    ss_launch<2, 3>(k.id, W + D, U, W + D + k.dh, once ? 0 : U, enc, P, pkR, pkRs, W + Q, skSs ? U : 0, status, ss, n,
                    st);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}
static int decaps_dev(const Id& k, const uint8_t* skR, size_t skRs, const uint8_t* enc, const uint8_t* pkS, size_t pkSs,
                      uint8_t* ss, uint8_t* status, uint8_t* W, size_t n, cudaStream_t st) {
  const size_t U = work_unit(k), D = k.sk, Q = k.sk + 2 * k.dh, P = k.pk;
  CB200_CUDA(cudaMemsetAsync(status, 0, n, st));
  dh(k, skR, skRs, nullptr, 0, W + Q, U, nullptr, skRs ? n : 1, st);  // pkR = KeyGen(skR), once for a shared skR
  dh(k, skR, skRs, enc, P, W + D, U, status, n, st);                   // Shared(skR, enc)
  if (!pkS) {
    ss_launch<1, 2>(k.id, W + D, U, nullptr, 0, enc, P, W + Q, skRs ? U : 0, nullptr, 0, status, ss, n, st);
  } else {
    dh(k, skR, skRs, pkS, pkSs, W + D + k.dh, U, status, n, st);  // Shared(skR, pkS)
    ss_launch<2, 3>(k.id, W + D, U, W + D + k.dh, U, enc, P, W + Q, skRs ? U : 0, pkS, pkSs, status, ss, n, st);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// Host-pointer calls: failed operations are reported after the whole batch ran.  X25519 / X448: a low-order point
// (hpke.ErrInvalidKEMSharedSecret).  NIST curves: bit 1 = an invalid skR / skS (hpke.ErrInvalidKEMPrivateKey) before
// bit 0 = an invalid pkR, enc or pkS (hpke.ErrInvalidKEMPublicKey).
static int status_result(const Id& k, const Counts& c, size_t n, const char* fn) {
  if (const char* curve = nist_curve(k.id)) {
    if (c.bit1) {
      set_error("%s: %zu of %zu operations have a private key outside [1, n - 1] (hpke: invalid KEM private key)", fn,
                c.bit1, n);
      return CB200_ERR_PRIVKEY;
    }
    if (c.bit0) {
      set_error("%s: %zu of %zu operations have a public key or encapsulation that is not a %s point "
                "(hpke: invalid KEM public key)", fn, c.bit0, n, curve);
      return CB200_ERR_PUBKEY;
    }
    return 0;
  }
  if (!c.bit0) return 0;
  set_error("%s: %zu of %zu operations hit a low-order public key or encapsulation (hpke: invalid KEM shared secret)", fn,
            c.bit0, n);
  return CB200_ERR_PUBKEY;
}
// Device-pointer calls read and write their rows in 32-bit units; the X25519 entry points ask for 16-byte alignment
// like cb200_x25519, the X448 ones for 8 like cb200_x448.  NIST curve rows are read and written byte by byte.
static size_t align_of(const Id& k) { return k.pk == 32 ? 16 : k.pk == 56 ? 8 : 1; }
static const char* align_text(const Id& k) {
  return k.pk == 32 ? "%s: device buffers and strides must be 16-byte aligned"
                    : "%s: device buffers and strides must be 8-byte aligned";
}
static const char* kNeedStatus = "%s: device-pointer calls need a status array (it marks the failed operations)";
static bool bad_stride(size_t s, size_t row) { return s != 0 && s < row; }

// encaps and auth encaps (skS null for the former); k null = an unknown id
static int encaps_entry(const char* fn, const Id* kp, const uint8_t* pkR, size_t pkRs, const uint8_t* skS, size_t skSs,
                        const uint8_t* seeds, uint8_t* enc, uint8_t* ss, uint8_t* status, size_t n, bool auth) {
  int rc = require_ready();
  if (rc) return rc;
  if (!kp || !pkR || !seeds || !enc || !ss || (auth && !skS) || bad_stride(pkRs, kp->pk) ||
      (auth && bad_stride(skSs, kp->sk))) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const Id k = *kp;
  Batch b{fn, n, enc, 1u << 16, 1u << 13,
          {{pkR, k.pk, pkRs, kIn}, {seeds, k.sk, k.sk, kIn}, {enc, k.pk, k.pk, kOut}, {ss, k.ss, k.ss, kOut},
           {status, 1, 1, kStatus}, {nullptr, work_unit(k), work_unit(k), kScratch}, {skS, k.sk, skSs, kIn}},
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
  return status_result(k, c, n, fn);
}

// decaps and auth decaps (pkS null for the former); k null = an unknown id
static int decaps_entry(const char* fn, const Id* kp, const uint8_t* skR, size_t skRs, const uint8_t* enc,
                        const uint8_t* pkS, size_t pkSs, uint8_t* ss, uint8_t* status, size_t n, bool auth) {
  int rc = require_ready();
  if (rc) return rc;
  if (!kp || !skR || !enc || !ss || (auth && !pkS) || bad_stride(skRs, kp->sk) || (auth && bad_stride(pkSs, kp->pk))) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const Id k = *kp;
  Batch b{fn, n, ss, 1u << 16, 1u << 13,
          {{skR, k.sk, skRs, kIn}, {enc, k.pk, k.pk, kIn}, {ss, k.ss, k.ss, kOut}, {status, 1, 1, kStatus},
           {nullptr, work_unit(k), work_unit(k), kScratch}, {pkS, k.pk, pkSs, kIn}},
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
  return status_result(k, c, n, fn);
}

// DeriveKeyPair; k null = an unknown id
static int keygen_entry(const char* fn, const Id* kp, const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!kp || !seeds || !pk || !sk) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const Id k = *kp;
  Batch b{fn, n, pk, 1u << 16, 1u << 13, {{seeds, k.sk, k.sk, kIn}, {pk, k.pk, k.pk, kOut}, {sk, k.sk, k.sk, kOut}},
          {{!aligned({seeds, pk, sk}, {}, align_of(k)), align_text(k)}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) -> int {
    int e = derive(k, r[0].p, k.sk, r[2].p, k.sk, cnt, st);
    if (e) return e;
    dh(k, r[2].p, k.sk, nullptr, 0, r[1].p, k.pk, nullptr, cnt, st);
    CB200_CUDA(cudaGetLastError());
    return 0;
  });
}

static const Id* known(int id, Id* k) { return id_of(id, k) ? k : nullptr; }

}  // namespace hpke
}  // namespace cb200

using namespace cb200;
using namespace cb200::hpke;

extern "C" {

size_t cb200_hpke_public_key_size(int id) {
  Id k;
  return id_of(id, &k) ? k.pk : 0;
}
size_t cb200_hpke_private_key_size(int id) {
  Id k;
  return id_of(id, &k) ? k.sk : 0;
}
size_t cb200_hpke_ciphertext_size(int id) {
  Id k;
  return id_of(id, &k) ? k.pk : 0;
}
size_t cb200_hpke_shared_key_size(int id) {
  Id k;
  return id_of(id, &k) ? k.ss : 0;
}
size_t cb200_hpke_seed_size(int id) {
  Id k;
  return id_of(id, &k) ? k.sk : 0;
}
size_t cb200_hpke_encapsulation_seed_size(int id) {
  Id k;
  return id_of(id, &k) ? k.sk : 0;
}

int cb200_hpke_keygen(int id, const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  Id k;
  return keygen_entry("cb200_hpke_keygen", known(id, &k), seeds, pk, sk, n);
}

int cb200_hpke_encaps(int id, const uint8_t* pkR, size_t pkR_stride, const uint8_t* seeds, uint8_t* enc, uint8_t* ss,
                      uint8_t* status, size_t n) {
  Id k;
  return encaps_entry("cb200_hpke_encaps", known(id, &k), pkR, pkR_stride, nullptr, 0, seeds, enc, ss, status, n, false);
}

int cb200_hpke_decaps(int id, const uint8_t* skR, size_t skR_stride, const uint8_t* enc, uint8_t* ss, uint8_t* status,
                      size_t n) {
  Id k;
  return decaps_entry("cb200_hpke_decaps", known(id, &k), skR, skR_stride, enc, nullptr, 0, ss, status, n, false);
}

int cb200_hpke_auth_encaps(int id, const uint8_t* pkR, size_t pkR_stride, const uint8_t* skS, size_t skS_stride,
                           const uint8_t* seeds, uint8_t* enc, uint8_t* ss, uint8_t* status, size_t n) {
  Id k;
  return encaps_entry("cb200_hpke_auth_encaps", known(id, &k), pkR, pkR_stride, skS, skS_stride, seeds, enc, ss, status,
                      n, true);
}

int cb200_hpke_auth_decaps(int id, const uint8_t* skR, size_t skR_stride, const uint8_t* enc, const uint8_t* pkS,
                           size_t pkS_stride, uint8_t* ss, uint8_t* status, size_t n) {
  Id k;
  return decaps_entry("cb200_hpke_auth_decaps", known(id, &k), skR, skR_stride, enc, pkS, pkS_stride, ss, status, n,
                      true);
}

// DHKEM(P-256, HKDF-SHA256), DHKEM(P-384, HKDF-SHA384) and DHKEM(P-521, HKDF-SHA512)
#define CB200_HPKE_NIST_ENTRIES(c, K)                                                                                  \
  size_t cb200_hpke_##c##_public_key_size(void) { return K.pk; }                                                       \
  size_t cb200_hpke_##c##_private_key_size(void) { return K.sk; }                                                      \
  size_t cb200_hpke_##c##_ciphertext_size(void) { return K.pk; }                                                       \
  size_t cb200_hpke_##c##_shared_key_size(void) { return K.ss; }                                                       \
  size_t cb200_hpke_##c##_seed_size(void) { return K.sk; }                                                             \
  size_t cb200_hpke_##c##_encapsulation_seed_size(void) { return K.sk; }                                               \
  int cb200_hpke_##c##_keygen(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {                              \
    return keygen_entry("cb200_hpke_" #c "_keygen", &K, seeds, pk, sk, n);                                             \
  }                                                                                                                    \
  int cb200_hpke_##c##_encaps(const uint8_t* pkR, size_t pkR_stride, const uint8_t* seeds, uint8_t* enc, uint8_t* ss,  \
                              uint8_t* status, size_t n) {                                                             \
    return encaps_entry("cb200_hpke_" #c "_encaps", &K, pkR, pkR_stride, nullptr, 0, seeds, enc, ss, status, n,        \
                        false);                                                                                        \
  }                                                                                                                    \
  int cb200_hpke_##c##_decaps(const uint8_t* skR, size_t skR_stride, const uint8_t* enc, uint8_t* ss, uint8_t* status, \
                              size_t n) {                                                                              \
    return decaps_entry("cb200_hpke_" #c "_decaps", &K, skR, skR_stride, enc, nullptr, 0, ss, status, n, false);       \
  }                                                                                                                    \
  int cb200_hpke_##c##_auth_encaps(const uint8_t* pkR, size_t pkR_stride, const uint8_t* skS, size_t skS_stride,       \
                                   const uint8_t* seeds, uint8_t* enc, uint8_t* ss, uint8_t* status, size_t n) {       \
    return encaps_entry("cb200_hpke_" #c "_auth_encaps", &K, pkR, pkR_stride, skS, skS_stride, seeds, enc, ss, status, \
                        n, true);                                                                                      \
  }                                                                                                                    \
  int cb200_hpke_##c##_auth_decaps(const uint8_t* skR, size_t skR_stride, const uint8_t* enc, const uint8_t* pkS,      \
                                   size_t pkS_stride, uint8_t* ss, uint8_t* status, size_t n) {                        \
    return decaps_entry("cb200_hpke_" #c "_auth_decaps", &K, skR, skR_stride, enc, pkS, pkS_stride, ss, status, n,     \
                        true);                                                                                         \
  }
CB200_HPKE_NIST_ENTRIES(p256, kP256)
CB200_HPKE_NIST_ENTRIES(p384, kP384)
CB200_HPKE_NIST_ENTRIES(p521, kP521)
#undef CB200_HPKE_NIST_ENTRIES

}  // extern "C"
