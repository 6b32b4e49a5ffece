// sign/ed448 and sign/eddilithium3, batched on the device:
//   sign/ed448/ed448.go:191-205,207-271,294-339   newKeyFromSeed / signAll / verify   -> ed448_*_kernel (thread per op)
//   sign/eddilithium3/eddilithium.go:59-110       Ed448-Dilithium3                    -> the round-3 Dilithium3 flows of
//                                                                                       mldsa.cu (mldsa_internal.h) + the
//                                                                                       Ed448 kernels
// The curve code is ed448.cuh; [s]G and [r]G use the fixed-base table that cb200_init builds here (init_ed448_table).
#include <cstring>
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "ed448.cuh"
#include "flow_internal.h"
#include "mldsa_internal.h"

namespace cb200 {

int init_ed448_table(Dev& c) {  // device c.device is current
  std::vector<int32_t> t(ed448::kTableWords);
  ed448::build_base_table(t.data());
  if (c.ed448_table) cudaFree(c.ed448_table);
  CB200_CUDA(cudaMalloc(&c.ed448_table, t.size() * sizeof(int32_t)));
  CB200_CUDA(cudaMemcpy(c.ed448_table, t.data(), t.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
  return 0;
}

namespace ed448k {

// Rows of 57 and 114 bytes sit at any byte offset (every row size of Ed448-Dilithium3 is odd): all row accesses are
// byte loads and stores.
__device__ __forceinline__ void ld57(uint8_t (&b)[57], const uint8_t* p) {
#pragma unroll
  for (int i = 0; i < 57; i++) b[i] = p[i];
}
__device__ __forceinline__ void st57(uint8_t* p, const uint32_t (&w)[ed448::kW], uint32_t top) {
#pragma unroll
  for (int i = 0; i < 56; i++) p[i] = ed448::byte_of(w, i);
  p[56] = (uint8_t)top;
}

// pk[i] = A, and sk[i] = seed || A (114-byte rows) when sk is not null
__global__ void __launch_bounds__(128) ed448_keygen_kernel(const uint8_t* __restrict__ seeds, size_t s_stride,
                                                           uint8_t* __restrict__ pk, size_t pk_stride,
                                                           uint8_t* __restrict__ sk, const int32_t* __restrict__ table,
                                                           size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t seed[57];
  ld57(seed, seeds + i * s_stride);
  uint32_t A[ed448::kW], top;
  ed448::public_from_seed(A, top, seed, table);
  st57(pk + i * pk_stride, A, top);
  if (sk) {
    uint8_t* row = sk + 114 * i;
#pragma unroll
    for (int b = 0; b < 57; b++) row[b] = seed[b];
    st57(row + 57, A, top);
  }
}

// sig[i] = Sign(sk[i], msg i, ctx).  sk rows hold seed || A (ed448.PrivateKey); with derive_a they hold the seed only
// and A is recomputed from it (eddilithium3's PrivateKey.Unpack).  sk_stride 0: one key for the batch.
__global__ void __launch_bounds__(128) ed448_sign_kernel(const uint8_t* __restrict__ sk, size_t sk_stride, int derive_a,
                                                         const uint8_t* __restrict__ ctx, int ctxlen,
                                                         const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ msg_off,
                                                         uint8_t* __restrict__ sig, size_t sig_stride,
                                                         const int32_t* __restrict__ table, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* row = sk + i * sk_stride;
  uint8_t seed[57], A[57];
  ld57(seed, row);
  if (derive_a) {
    uint32_t w[ed448::kW], top;
    ed448::public_from_seed(w, top, seed, table);
#pragma unroll
    for (int b = 0; b < 56; b++) A[b] = ed448::byte_of(w, b);
    A[56] = (uint8_t)top;
  } else {
    ld57(A, row + 57);
  }
  const uint64_t m0 = msg_off[i], m1 = msg_off[i + 1];
  ed448::sign(sig + i * sig_stride, seed, A, ctx, ctxlen, msgs + m0, m1 - m0, table);
}

// ok[i] = Verify(pk[i], msg i, sig[i], ctx); with and_ok the result is ANDed into ok[i] (the composite's other half)
__global__ void __launch_bounds__(128) ed448_verify_kernel(const uint8_t* __restrict__ pk, size_t pk_stride,
                                                           const uint8_t* __restrict__ ctx, int ctxlen,
                                                           const uint8_t* __restrict__ msgs,
                                                           const uint64_t* __restrict__ msg_off,
                                                           const uint8_t* __restrict__ sig, size_t sig_stride,
                                                           uint8_t* __restrict__ ok, int and_ok,
                                                           const int32_t* __restrict__ table, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t m0 = msg_off[i], m1 = msg_off[i + 1];
  const bool good = ed448::verify(pk + i * pk_stride, ctx, ctxlen, msgs + m0, m1 - m0, sig + i * sig_stride, table);
  if (and_ok)
    ok[i] = (ok[i] && good) ? 1 : 0;
  else
    ok[i] = good ? 1 : 0;
}

// Ed448-Dilithium3 NewKeyFromSeed (eddilithium.go:59-78): SHAKE256(seed, 89) -> Dilithium3 seed (32) || Ed448 seed
// (57).  The Ed448 seed goes to its scratch row and to the end of the private key row.
__global__ void __launch_bounds__(128) edd3_split_kernel(const uint8_t* __restrict__ seeds, uint8_t* __restrict__ dseed,
                                                         uint8_t* __restrict__ eseed, uint8_t* __restrict__ sk_tail,
                                                         size_t sk_stride, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t seed[57];
  ld57(seed, seeds + 57 * i);
  uint64_t a[25];
  uint32_t h[30];
  ed448::shake256(a, nullptr, -1, seed, 57, nullptr, 0);
  ed448::lanes_to_words(h, a);
#pragma unroll
  for (int b = 0; b < 8; b++) reinterpret_cast<uint32_t*>(dseed + 32 * i)[b] = h[b];
#pragma unroll
  for (int b = 0; b < 57; b++) {
    const uint8_t v = ed448::byte_of(h, 32 + b);
    eseed[57 * i + b] = v;
    sk_tail[sk_stride * i + b] = v;
  }
}

// ------------------------------------------------------------------ host side
static inline unsigned blocks(size_t units, size_t per) { return (unsigned)((units + per - 1) / per); }
static const int32_t* base_table() { return (const int32_t*)ctx().ed448_table; }

static int keygen_dev(const uint8_t* seeds, size_t s_stride, uint8_t* pk, size_t pk_stride, uint8_t* sk, size_t n,
                      cudaStream_t st) {
  {
    KernelScope ks(KID_ED448, st);
    ed448_keygen_kernel<<<blocks(n, 128), 128, 0, st>>>(seeds, s_stride, pk, pk_stride, sk, base_table(), n);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}
static int sign_dev(const uint8_t* sk, size_t sk_stride, int derive_a, const uint8_t* dctx, int ctxlen, const uint8_t* msgs,
                    const uint64_t* msg_off, uint8_t* sig, size_t sig_stride, size_t n, cudaStream_t st) {
  {
    KernelScope ks(KID_ED448, st);
    ed448_sign_kernel<<<blocks(n, 128), 128, 0, st>>>(sk, sk_stride, derive_a, dctx, ctxlen, msgs, msg_off, sig, sig_stride,
                                                      base_table(), n);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}
static int verify_dev(const uint8_t* pk, size_t pk_stride, const uint8_t* dctx, int ctxlen, const uint8_t* msgs,
                      const uint64_t* msg_off, const uint8_t* sig, size_t sig_stride, uint8_t* ok, int and_ok, size_t n,
                      cudaStream_t st) {
  {
    KernelScope ks(KID_ED448, st);
    ed448_verify_kernel<<<blocks(n, 128), 128, 0, st>>>(pk, pk_stride, dctx, ctxlen, msgs, msg_off, sig, sig_stride, ok,
                                                        and_ok, base_table(), n);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// ---- Ed448-Dilithium3 (eddilithium.go): pk = Dilithium3 pk (1952) || A (57), sk = Dilithium3 sk (4000) || Ed448 seed
// (57), sig = Dilithium3 sig (3293) || Ed448 sig (114).  Every row size is odd, so the Dilithium3 halves never sit at a
// 16-byte boundary with the flows' own stride: each is staged through aligned scratch in the level-1 work area
// (level 0 belongs to those flows) and moved with 2D copies on the call's stream.  The Ed448 kernels read and write
// their parts in place.
constexpr size_t kDPk = 1952, kDSk = 4000, kDSig = 3293;
constexpr size_t kEdPk = kDPk + 57, kEdSk = kDSk + 57, kEdSig = kDSig + 114;

static int edd3_keygen_dev(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n, cudaStream_t st, int slot) {
  Arena A;
  int rc = arena(slot, n * (32 + 57 + kDPk + kDSk) + 4096, &A);
  if (rc) return rc;
  uint8_t *dseed = A.take(n * 32), *eseed = A.take(n * 57), *dpk = A.take(n * kDPk), *dsk = A.take(n * kDSk);
  {
    KernelScope ks(KID_ED448, st);
    edd3_split_kernel<<<blocks(n, 128), 128, 0, st>>>(seeds, dseed, eseed, sk + kDSk, kEdSk, n);
  }
  CB200_CUDA(cudaGetLastError());
  if ((rc = mldsa::dev_keygen(3, dseed, dpk, dsk, n, st, slot))) return rc;
  if ((rc = copy2d(pk, kEdPk, dpk, kDPk, kDPk, n, st))) return rc;
  if ((rc = copy2d(sk, kEdSk, dsk, kDSk, kDSk, n, st))) return rc;
  return keygen_dev(eseed, 57, pk + kDPk, kEdPk, nullptr, n, st);
}
// SignTo (eddilithium.go:82-93): round-3 Dilithium3, then Ed448 with an empty context and A re-derived from the seed
static int edd3_sign_dev(const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off, uint8_t* sig,
                         uint8_t* status, size_t n, cudaStream_t st, int slot) {
  const size_t nk = sk_stride ? n : 1;
  Arena A;
  int rc = arena(slot, nk * kDSk + n * (kDSig + 1) + 4096, &A);
  if (rc) return rc;
  uint8_t *dsk = A.take(nk * kDSk), *dsig = A.take(n * kDSig);
  if (!status) status = A.take(n);  // the flow always writes per-op status bytes
  if ((rc = copy2d(dsk, kDSk, sk, sk_stride ? sk_stride : kEdSk, kDSk, nk, st))) return rc;
  rc = mldsa::dev_sign(3, dsk, sk_stride ? kDSk : 0, msgs, msg_off, dsig, status, n, st, slot,
                       (volatile uint32_t*)wset(slot).pin);
  if (rc) return rc;
  if ((rc = copy2d(sig, kEdSig, dsig, kDSig, kDSig, n, st))) return rc;
  return sign_dev(sk + kDSk, sk_stride, 1, nullptr, 0, msgs, msg_off, sig + kDSig, kEdSig, n, st);
}
// Verify (eddilithium.go:96-110): both halves must hold
static int edd3_verify_dev(const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                           const uint8_t* sig, uint8_t* ok, size_t n, cudaStream_t st, int slot) {
  const size_t nk = pk_stride ? n : 1;
  Arena A;
  int rc = arena(slot, nk * kDPk + n * kDSig + 4096, &A);
  if (rc) return rc;
  uint8_t *dpk = A.take(nk * kDPk), *dsig = A.take(n * kDSig);
  if ((rc = copy2d(dpk, kDPk, pk, pk_stride ? pk_stride : kEdPk, kDPk, nk, st))) return rc;
  if ((rc = copy2d(dsig, kDSig, sig, kEdSig, kDSig, n, st))) return rc;
  rc = mldsa::dev_verify(3, dpk, pk_stride ? kDPk : 0, msgs, msg_off, dsig, ok, n, st, slot);
  if (rc) return rc;
  return verify_dev(pk + kDPk, pk_stride, nullptr, 0, msgs, msg_off, sig + kDSig, kEdSig, ok, 1, n, st);
}

}  // namespace ed448k
}  // namespace cb200

using namespace cb200;
using namespace cb200::ed448k;

extern "C" {

size_t cb200_ed448_public_key_size(void) { return 57; }
size_t cb200_ed448_private_key_size(void) { return 114; }
size_t cb200_ed448_signature_size(void) { return 114; }
size_t cb200_ed448_seed_size(void) { return 57; }
size_t cb200_eddilithium3_public_key_size(void) { return kEdPk; }
size_t cb200_eddilithium3_private_key_size(void) { return kEdSk; }
size_t cb200_eddilithium3_signature_size(void) { return kEdSig; }
size_t cb200_eddilithium3_seed_size(void) { return 57; }

int cb200_ed448_keygen(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!seeds || !pk) {
    set_error("cb200_ed448_keygen: null pointer");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_ed448_keygen", n, pk, 1u << 16, 1u << 13, {{seeds, 57, 57, kIn}, {pk, 57, 57, kOut}, {sk, 114, 114, kOut}}, {}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return keygen_dev(r[0].p, 57, r[1].p, 57, r[2].p, cnt, st);
  });
}

int cb200_ed448_sign(const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* context,
                     size_t ctxlen, uint8_t* sig, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!sk || !msgs || !msg_off || !sig || (sk_stride != 0 && sk_stride < 114) || (ctxlen && !context)) {
    set_error("cb200_ed448_sign: bad argument");
    return CB200_ERR_ARG;
  }
  if (ctxlen > ed448::kMaxContext) {  // signAll panics
    set_error("cb200_ed448_sign: context longer than 255 bytes (%zu)", ctxlen);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_ed448_sign", n, sig, 1u << 15, 1u << 12, {{sk, 114, sk_stride, kIn}, {sig, 114, 114, kOut}},
          {{!aligned({msg_off}, {}, 8), "%s: device msg_off must be 8-byte aligned"}}, msgs, msg_off, context, ctxlen};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return sign_dev(r[0].p, r[0].stride, 0, r.ctx, (int)ctxlen, r.msgs, r.msg_off, r[1].p, 114, cnt, st);
  });
}

int cb200_ed448_verify(const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                       const uint8_t* context, size_t ctxlen, const uint8_t* sig, uint8_t* ok, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!pk || !msgs || !msg_off || !sig || !ok || (pk_stride != 0 && pk_stride < 57) || (ctxlen && !context)) {
    set_error("cb200_ed448_verify: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const bool long_ctx = ctxlen > ed448::kMaxContext;  // verify returns false
  Batch b{"cb200_ed448_verify", n, ok, 1u << 15, 1u << 12, {{pk, 57, pk_stride, kIn}, {sig, 114, 114, kIn}, {ok, 1, 1, kOut}},
          {{!aligned({msg_off}, {}, 8), "%s: device msg_off must be 8-byte aligned"}}, msgs, msg_off, context,
          long_ctx ? 0 : ctxlen};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) -> int {
    if (long_ctx) {
      CB200_CUDA(cudaMemsetAsync(r[2].p, 0, cnt, st));
      return 0;
    }
    return verify_dev(r[0].p, r[0].stride, r.ctx, (int)ctxlen, r.msgs, r.msg_off, r[1].p, 114, r[2].p, 0, cnt, st);
  });
}

int cb200_eddilithium3_keygen(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!seeds || !pk || !sk) {
    set_error("cb200_eddilithium3_keygen: null pointer");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_eddilithium3_keygen", n, pk, 1u << 14, 1u << 12,
          {{seeds, 57, 57, kIn}, {pk, kEdPk, kEdPk, kOut}, {sk, kEdSk, kEdSk, kOut}}, {}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return edd3_keygen_dev(r[0].p, r[1].p, r[2].p, cnt, st, slot);
  });
}

int cb200_eddilithium3_sign(const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off, uint8_t* sig,
                            uint8_t* status, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!sk || !msgs || !msg_off || !sig || (sk_stride != 0 && sk_stride < kEdSk)) {
    set_error("cb200_eddilithium3_sign: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_eddilithium3_sign", n, sig, 1u << 15, 1u << 12,
          {{sk, kEdSk, sk_stride, kIn}, {sig, kEdSig, kEdSig, kOut}, {status, 1, 1, kStatus}},
          {{!aligned({msg_off}, {}, 16), "%s: device msg_off must be 16-byte aligned"},
           // the limit of the Dilithium3 signing flow
           {n >= (1u << 24), "%s: a device-pointer batch is limited to 2^24 - 1 signatures per call (got %zu)"}},
          msgs, msg_off};
  Counts c;
  rc = run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return edd3_sign_dev(r[0].p, r[0].stride, r.msgs, r.msg_off, r[1].p, r[2].p, cnt, st, slot);
  }, &c);
  if (rc) return rc;
  return sign_attempts_result("cb200_eddilithium3_sign", c.nonzero, n);
}

int cb200_eddilithium3_verify(const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                              const uint8_t* sig, uint8_t* ok, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!pk || !msgs || !msg_off || !sig || !ok || (pk_stride != 0 && pk_stride < kEdPk)) {
    set_error("cb200_eddilithium3_verify: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_eddilithium3_verify", n, ok, 1u << 15, 1u << 12,
          {{pk, kEdPk, pk_stride, kIn}, {sig, kEdSig, kEdSig, kIn}, {ok, 1, 1, kOut}},
          {{!aligned({msg_off}, {}, 16), "%s: device msg_off must be 16-byte aligned"}}, msgs, msg_off};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return edd3_verify_dev(r[0].p, r[0].stride, r.msgs, r.msg_off, r[1].p, r[2].p, cnt, st, slot);
  });
}

}  // extern "C"
