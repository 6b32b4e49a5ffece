// sign/ed25519 and sign/eddilithium2, batched on the device:
//   sign/ed25519/ed25519.go:206-223,290-294,329-368   NewKeyFromSeed / Sign / Verify   -> ed25519_*_kernel (thread per op)
//   sign/eddilithium2/eddilithium.go:59-115           Ed25519-Dilithium2               -> the round-3 Dilithium2 flows of
//                                                                                         mldsa.cu (mldsa_internal.h) + the
//                                                                                         Ed25519 kernels
// The curve code is ed25519.cuh; [k]B uses the fixed-base table that cb200_init builds for X25519 KeyGen.
#include <cstring>
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "ed25519.cuh"
#include "flow_internal.h"
#include "mldsa_internal.h"

namespace cb200 {
namespace eddsa {

template <int N>
__device__ __forceinline__ void ldw(uint32_t (&w)[N], const uint8_t* p) {
#pragma unroll
  for (int i = 0; i < N; i++) w[i] = reinterpret_cast<const uint32_t*>(p)[i];
}
template <int N>
__device__ __forceinline__ void stw(uint8_t* p, const uint32_t (&w)[N]) {
#pragma unroll
  for (int i = 0; i < N; i++) reinterpret_cast<uint32_t*>(p)[i] = w[i];
}

// pk[i] = A, and sk[i] = seed || A when sk is not null.  Rows are 4-byte aligned.
__global__ void __launch_bounds__(128) ed25519_keygen_kernel(const uint8_t* __restrict__ seeds, size_t s_stride,
                                                             uint8_t* __restrict__ pk, size_t pk_stride,
                                                             uint8_t* __restrict__ sk, const int32_t* __restrict__ table,
                                                             size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t seed[8], A[8];
  ldw(seed, seeds + i * s_stride);
  ed25519::public_from_seed(A, seed, table);
  stw(pk + i * pk_stride, A);
  if (sk) {
    stw(sk + 64 * i, seed);
    stw(sk + 64 * i + 32, A);
  }
}

// sig[i] = Sign(sk[i], msg i).  sk rows hold seed || A (ed25519.PrivateKey); with derive_a they hold the seed only
// and A is recomputed from it (eddilithium2's PrivateKey.Unpack).  sk_stride 0: one key for the batch.
__global__ void __launch_bounds__(128) ed25519_sign_kernel(const uint8_t* __restrict__ sk, size_t sk_stride, int derive_a,
                                                           const uint8_t* __restrict__ msgs,
                                                           const uint64_t* __restrict__ msg_off, uint8_t* __restrict__ sig,
                                                           size_t sig_stride, const int32_t* __restrict__ table, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* row = sk + i * sk_stride;
  uint32_t seed[8], A[8], R[8], S[8];
  ldw(seed, row);
  if (derive_a)
    ed25519::public_from_seed(A, seed, table);
  else
    ldw(A, row + 32);
  const uint64_t m0 = msg_off[i], m1 = msg_off[i + 1];
  ed25519::sign(R, S, seed, A, msgs + m0, m1 - m0, table);
  stw(sig + i * sig_stride, R);
  stw(sig + i * sig_stride + 32, S);
}

// ok[i] = Verify(pk[i], msg i, sig[i]); with and_ok the result is ANDed into ok[i] (the composite's other half)
__global__ void __launch_bounds__(128) ed25519_verify_kernel(const uint8_t* __restrict__ pk, size_t pk_stride,
                                                             const uint8_t* __restrict__ msgs,
                                                             const uint64_t* __restrict__ msg_off,
                                                             const uint8_t* __restrict__ sig, size_t sig_stride,
                                                             uint8_t* __restrict__ ok, int and_ok,
                                                             const int32_t* __restrict__ table, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t A[8], R[8], S[8];
  ldw(A, pk + i * pk_stride);
  ldw(R, sig + i * sig_stride);
  ldw(S, sig + i * sig_stride + 32);
  const uint64_t m0 = msg_off[i], m1 = msg_off[i + 1];
  const bool good = ed25519::verify(A, msgs + m0, m1 - m0, R, S, table);
  if (and_ok)
    ok[i] = (ok[i] && good) ? 1 : 0;
  else
    ok[i] = good ? 1 : 0;
}

// ------------------------------------------------------------------ host side
static inline unsigned blocks(size_t units, size_t per) { return (unsigned)((units + per - 1) / per); }
static const int32_t* base_table() { return (const int32_t*)ctx().x25519_table; }

static int ed_keygen_dev(const uint8_t* seeds, size_t s_stride, uint8_t* pk, size_t pk_stride, uint8_t* sk, size_t n,
                         cudaStream_t st) {
  {
    KernelScope ks(KID_ED25519, st);
    ed25519_keygen_kernel<<<blocks(n, 128), 128, 0, st>>>(seeds, s_stride, pk, pk_stride, sk, base_table(), n);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}
static int ed_sign_dev(const uint8_t* sk, size_t sk_stride, int derive_a, const uint8_t* msgs, const uint64_t* msg_off,
                       uint8_t* sig, size_t sig_stride, size_t n, cudaStream_t st) {
  {
    KernelScope ks(KID_ED25519, st);
    ed25519_sign_kernel<<<blocks(n, 128), 128, 0, st>>>(sk, sk_stride, derive_a, msgs, msg_off, sig, sig_stride, base_table(),
                                                        n);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}
static int ed_verify_dev(const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                         const uint8_t* sig, size_t sig_stride, uint8_t* ok, int and_ok, size_t n, cudaStream_t st) {
  {
    KernelScope ks(KID_ED25519, st);
    ed25519_verify_kernel<<<blocks(n, 128), 128, 0, st>>>(pk, pk_stride, msgs, msg_off, sig, sig_stride, ok, and_ok,
                                                          base_table(), n);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// ---- Ed25519-Dilithium2 (eddilithium.go): pk = Dilithium2 pk (1312) || A (32), sk = Dilithium2 sk (2528) || Ed25519
// seed (32), sig = Dilithium2 sig (2420) || Ed25519 sig (64).  The Dilithium2 flows read and write contiguous rows,
// so the parts that do not sit at a row start with the flows' own stride go through aligned scratch in the level-1
// work area (level 0 belongs to those flows) and are moved with 2D copies on the call's stream.
constexpr size_t kDPk = 1312, kDSk = 2528, kDSig = 2420;
constexpr size_t kEdPk = kDPk + 32, kEdSk = kDSk + 32, kEdSig = kDSig + 64;

// NewKeyFromSeed (eddilithium.go:59-78): SHAKE256(seed) -> Dilithium2 seed (32) || Ed25519 seed (32)
static int edd2_keygen_dev(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n, cudaStream_t st, int slot) {
  Arena A;
  int rc = arena(slot, n * (64 + 32 + kDPk + kDSk) + 4096, &A);
  if (rc) return rc;
  uint8_t *ex = A.take(n * 64), *dseed = A.take(n * 32), *dpk = A.take(n * kDPk), *dsk = A.take(n * kDSk);
  hybrid::shake256_rows(seeds, 32, 32, ex, 64, 64, n, st);
  if ((rc = copy2d(dseed, 32, ex, 64, 32, n, st))) return rc;
  if ((rc = copy2d(sk + kDSk, kEdSk, ex + 32, 64, 32, n, st))) return rc;
  rc = mldsa::dev_keygen(2, dseed, dpk, dsk, n, st, slot);
  if (rc) return rc;
  if ((rc = copy2d(pk, kEdPk, dpk, kDPk, kDPk, n, st))) return rc;
  if ((rc = copy2d(sk, kEdSk, dsk, kDSk, kDSk, n, st))) return rc;
  return ed_keygen_dev(ex + 32, 64, pk + kDPk, kEdPk, nullptr, n, st);
}
// SignTo (eddilithium.go:82-93): the Dilithium2 half reads the key rows in place (their stride is a multiple of 16)
static int edd2_sign_dev(const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off, uint8_t* sig,
                         uint8_t* status, size_t n, cudaStream_t st, int slot) {
  Arena A;
  int rc = arena(slot, n * (kDSig + 1) + 4096, &A);
  if (rc) return rc;
  uint8_t* dsig = A.take(n * kDSig);
  if (!status) status = A.take(n);  // the flow always writes per-op status bytes
  rc = mldsa::dev_sign(2, sk, sk_stride, msgs, msg_off, dsig, status, n, st, slot, (volatile uint32_t*)wset(slot).pin);
  if (rc) return rc;
  if ((rc = copy2d(sig, kEdSig, dsig, kDSig, kDSig, n, st))) return rc;
  return ed_sign_dev(sk + kDSk, sk_stride, 1, msgs, msg_off, sig + kDSig, kEdSig, n, st);
}
// Verify (eddilithium.go:96-115): both halves must hold
static int edd2_verify_dev(const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                           const uint8_t* sig, uint8_t* ok, size_t n, cudaStream_t st, int slot) {
  Arena A;
  int rc = arena(slot, n * kDSig + 4096, &A);
  if (rc) return rc;
  uint8_t* dsig = A.take(n * kDSig);
  if ((rc = copy2d(dsig, kDSig, sig, kEdSig, kDSig, n, st))) return rc;
  rc = mldsa::dev_verify(2, pk, pk_stride, msgs, msg_off, dsig, ok, n, st, slot);
  if (rc) return rc;
  return ed_verify_dev(pk + kDPk, pk_stride, msgs, msg_off, sig + kDSig, kEdSig, ok, 1, n, st);
}

}  // namespace eddsa
}  // namespace cb200

using namespace cb200;
using namespace cb200::eddsa;

extern "C" {

size_t cb200_ed25519_public_key_size(void) { return 32; }
size_t cb200_ed25519_private_key_size(void) { return 64; }
size_t cb200_ed25519_signature_size(void) { return 64; }
size_t cb200_ed25519_seed_size(void) { return 32; }
size_t cb200_eddilithium2_public_key_size(void) { return kEdPk; }
size_t cb200_eddilithium2_private_key_size(void) { return kEdSk; }
size_t cb200_eddilithium2_signature_size(void) { return kEdSig; }
size_t cb200_eddilithium2_seed_size(void) { return 32; }

int cb200_ed25519_keygen(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!seeds || !pk) {
    set_error("cb200_ed25519_keygen: null pointer");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_ed25519_keygen", n, pk, 1u << 16, 1u << 13, {{seeds, 32, 32, kIn}, {pk, 32, 32, kOut}, {sk, 64, 64, kOut}},
          {{!aligned({seeds, pk, sk}, {}, 4), "%s: device buffers must be 4-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return ed_keygen_dev(r[0].p, 32, r[1].p, 32, r[2].p, cnt, st);
  });
}

int cb200_ed25519_sign(const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off, uint8_t* sig,
                       size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!sk || !msgs || !msg_off || !sig || (sk_stride != 0 && sk_stride < 64)) {
    set_error("cb200_ed25519_sign: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_ed25519_sign", n, sig, 1u << 15, 1u << 12, {{sk, 64, sk_stride, kIn}, {sig, 64, 64, kOut}},
          {{!aligned({sk, sig}, {sk_stride}, 4) || !aligned({msg_off}, {}, 8),
            "%s: device sk, sk_stride and sig must be 4-byte aligned, msg_off 8-byte aligned"}},
          msgs, msg_off};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return ed_sign_dev(r[0].p, r[0].stride, 0, r.msgs, r.msg_off, r[1].p, 64, cnt, st);
  });
}

int cb200_ed25519_verify(const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                         const uint8_t* sig, uint8_t* ok, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!pk || !msgs || !msg_off || !sig || !ok || (pk_stride != 0 && pk_stride < 32)) {
    set_error("cb200_ed25519_verify: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_ed25519_verify", n, ok, 1u << 15, 1u << 12,
          {{pk, 32, pk_stride, kIn}, {sig, 64, 64, kIn}, {ok, 1, 1, kOut}},
          {{!aligned({pk, sig}, {pk_stride}, 4) || !aligned({msg_off}, {}, 8),
            "%s: device pk, pk_stride and sig must be 4-byte aligned, msg_off 8-byte aligned"}},
          msgs, msg_off};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return ed_verify_dev(r[0].p, r[0].stride, r.msgs, r.msg_off, r[1].p, 64, r[2].p, 0, cnt, st);
  });
}

int cb200_eddilithium2_keygen(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!seeds || !pk || !sk) {
    set_error("cb200_eddilithium2_keygen: null pointer");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_eddilithium2_keygen", n, pk, 1u << 14, 1u << 12,
          {{seeds, 32, 32, kIn}, {pk, kEdPk, kEdPk, kOut}, {sk, kEdSk, kEdSk, kOut}},
          {{!aligned({seeds, pk, sk}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return edd2_keygen_dev(r[0].p, r[1].p, r[2].p, cnt, st, slot);
  });
}

int cb200_eddilithium2_sign(const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off, uint8_t* sig,
                            uint8_t* status, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!sk || !msgs || !msg_off || !sig || (sk_stride != 0 && sk_stride < kEdSk)) {
    set_error("cb200_eddilithium2_sign: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_eddilithium2_sign", n, sig, 1u << 15, 1u << 12,
          {{sk, kEdSk, sk_stride, kIn}, {sig, kEdSig, kEdSig, kOut}, {status, 1, 1, kStatus}},
          {{!aligned({sk, msg_off}, {sk_stride}, 16) || !aligned({sig}, {}, 4),
            "%s: device sk, sk_stride and msg_off must be 16-byte aligned, sig 4-byte aligned"},
           // the limit of the Dilithium2 signing flow
           {n >= (1u << 24), "%s: a device-pointer batch is limited to 2^24 - 1 signatures per call (got %zu)"}},
          msgs, msg_off};
  Counts c;
  rc = run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return edd2_sign_dev(r[0].p, r[0].stride, r.msgs, r.msg_off, r[1].p, r[2].p, cnt, st, slot);
  }, &c);
  if (rc) return rc;
  return sign_attempts_result("cb200_eddilithium2_sign", c.nonzero, n);
}

int cb200_eddilithium2_verify(const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                              const uint8_t* sig, uint8_t* ok, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!pk || !msgs || !msg_off || !sig || !ok || (pk_stride != 0 && pk_stride < kEdPk)) {
    set_error("cb200_eddilithium2_verify: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_eddilithium2_verify", n, ok, 1u << 15, 1u << 12,
          {{pk, kEdPk, pk_stride, kIn}, {sig, kEdSig, kEdSig, kIn}, {ok, 1, 1, kOut}},
          {{!aligned({pk, msg_off}, {pk_stride}, 16) || !aligned({sig}, {}, 4),
            "%s: device pk, pk_stride and msg_off must be 16-byte aligned, sig 4-byte aligned"}},
          msgs, msg_off};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return edd2_verify_dev(r[0].p, r[0].stride, r.msgs, r.msg_off, r[1].p, r[2].p, cnt, st, slot);
  });
}

}  // extern "C"
