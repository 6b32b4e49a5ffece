// RFC 9497 OPRF servers over P-256, P-384 and P-521 (the reference's oprf package, suites P256-SHA256, P384-SHA384
// and P521-SHA512), modes 0x00 (Server), 0x01 (VerifiableServer) and 0x02 (PartialObliviousServer), batched on the
// device.  The arithmetic is oprf.cuh; each kernel holds one call site of the variable-base multiplication:
//   DeriveKey      oprf_derive_kernel      thread per op: HashToScalar loop, [sk]G
//   Evaluate       oprf_eval_kernel        thread per blinded element: decode, [k]B or [t^-1]B
//                  oprf_composite_kernel   thread per request (modes 1, 2): Y = [k]G, M = sum d_j B_j
//                  oprf_proof_kernel       thread per request: status, Z = [k]M, t3 = [r]M, t2 = [r]G, c, s; zeroes
//                                          the rows of a failed request
//   FullEvaluate   oprf_full_kernel        thread per op: HashToGroup, [k]P or [t^-1]P, the Finalize hash
// Timed under the curve's profiling class (p256 / p384 / p521).
#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "oprf.cuh"

namespace cb200 {
namespace oprfk {

using nistp::Fe;
using nistp::Pt;
using oprf::Sc;

template <class C>
__global__ void __launch_bounds__(128) oprf_derive_kernel(const uint8_t* __restrict__ seeds, const uint8_t* info,
                                                          int info_len, int mode, uint8_t* __restrict__ sk,
                                                          uint8_t* __restrict__ pk, const uint32_t* __restrict__ table,
                                                          size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t ctx[24];
  const int clen = oprf::context<C>(ctx, mode);
  oprf::derive_key<C>(sk + i * C::kBytes, pk + i * oprf::kNe<C>, seeds + 32 * i, info, info_len, table, ctx, clen);
}

template <class C>
__global__ void __launch_bounds__(128) oprf_eval_kernel(const uint8_t* __restrict__ sk, size_t sk_stride,
                                                        const uint8_t* __restrict__ blinded, size_t m, int mode,
                                                        Sc<C> m_info, uint8_t* __restrict__ evaluated,
                                                        uint8_t* __restrict__ estat, size_t ne) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  uint32_t kp[C::kW], ke[C::kW];
  oprf::op_keys<C>(kp, ke, sk + (e / m) * sk_stride, mode, m_info);
  estat[e] = (uint8_t)oprf::eval_element<C>(evaluated + e * oprf::kNe<C>, blinded + e * oprf::kNe<C>, ke);
}

template <class C>
__global__ void __launch_bounds__(128) oprf_composite_kernel(const uint8_t* __restrict__ sk, size_t sk_stride,
                                                             const uint8_t* __restrict__ blinded,
                                                             const uint8_t* __restrict__ evaluated, size_t m, int mode,
                                                             Sc<C> m_info, uint8_t* __restrict__ ybuf,
                                                             uint8_t* __restrict__ mbuf,
                                                             const uint32_t* __restrict__ table, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  constexpr int Ne = oprf::kNe<C>;
  uint8_t ctx[24];
  const int clen = oprf::context<C>(ctx, mode);
  uint32_t kp[C::kW], ke[C::kW];
  oprf::op_keys<C>(kp, ke, sk + i * sk_stride, mode, m_info);
  uint8_t* Y = ybuf + i * Ne;
  Pt<C> P;
  oprf::mul_base(P, kp, table);
  oprf::encode(Y, P, ~0u);
  // mode 1 proves D = [k]B; mode 2 proves B = [t]D (server.go:50-72)
  const uint8_t *b = blinded + i * m * Ne, *d = evaluated + i * m * Ne;
  uint32_t st;
  oprf::composite<C>(P, st, Y, mode == 2 ? d : b, Ne, mode == 2 ? b : d, Ne, (int)m, ctx, clen);
  Fe<C> x, y;
  oprf::to_affine(x, y, P);
  nistp::words_to_be<C>(mbuf + i * 2 * C::kBytes, x.v, ~0u);
  nistp::words_to_be<C>(mbuf + i * 2 * C::kBytes + C::kBytes, y.v, ~0u);
}

template <class C>
__global__ void __launch_bounds__(128) oprf_proof_kernel(const uint8_t* __restrict__ sk, size_t sk_stride,
                                                         const uint8_t* __restrict__ rnd, size_t m, int mode,
                                                         Sc<C> m_info, const uint8_t* __restrict__ ybuf,
                                                         const uint8_t* __restrict__ mbuf,
                                                         const uint8_t* __restrict__ estat, uint8_t* __restrict__ evaluated,
                                                         uint8_t* __restrict__ proof, uint8_t* __restrict__ status,
                                                         const uint32_t* __restrict__ table, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  constexpr int Ne = oprf::kNe<C>;
  uint32_t kp[C::kW], ke[C::kW];
  uint32_t st = oprf::op_keys<C>(kp, ke, sk + i * sk_stride, mode, m_info);
  for (size_t j = 0; j < m; j++) st |= estat[i * m + j];
  if (mode != 0) {
    uint8_t ctx[24];
    const int clen = oprf::context<C>(ctx, mode);
    uint8_t* out = proof + i * 2 * C::kBytes;
    const uint32_t rok = oprf::prove<C>(out, kp, ybuf + i * Ne, mbuf + i * 2 * C::kBytes, rnd + i * C::kBytes, table,
                                        ctx, clen, ~0u);
    st |= rok ? 0u : 4u;
    if (st)
      for (int j = 0; j < 2 * C::kBytes; j++) out[j] = 0;
  }
  if (st)
    for (size_t j = 0; j < m * Ne; j++) evaluated[i * m * Ne + j] = 0;
  status[i] = (uint8_t)st;
}

template <class C>
__global__ void __launch_bounds__(128) oprf_full_kernel(const uint8_t* __restrict__ sk, size_t sk_stride, int mode,
                                                        Sc<C> m_info, const uint8_t* __restrict__ msgs,
                                                        const uint64_t* __restrict__ msg_off, const uint8_t* info,
                                                        int info_len, uint8_t* __restrict__ out,
                                                        uint8_t* __restrict__ status, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t ctx[24];
  const int clen = oprf::context<C>(ctx, mode);
  uint32_t kp[C::kW], ke[C::kW];
  const uint64_t m0 = msg_off[i], m1 = msg_off[i + 1];
  // an input over 65535 bytes (only a device-pointer call can pass one) fails its op rather than being hashed with a
  // truncated length prefix
  const uint32_t st = oprf::op_keys<C>(kp, ke, sk + i * sk_stride, mode, m_info) | (m1 - m0 > 65535 ? 16u : 0u);
  oprf::full_evaluate<C>(out + i * oprf::kNh<C>, ke, msgs + m0, (int)(st ? 0 : m1 - m0), info, info_len, mode, ctx, clen,
                         st ? 0u : ~0u);
  status[i] = (uint8_t)st;
}

static inline unsigned blocks(size_t units, size_t per) { return (unsigned)((units + per - 1) / per); }

// ---------------------------------------------------------------- host side
template <class C>
struct Curve;
template <>
struct Curve<nistp::P256> {
  static constexpr int kid = KID_P256;
  static const uint32_t* table() { return (const uint32_t*)ctx().p256_table; }
};
template <>
struct Curve<nistp::P384> {
  static constexpr int kid = KID_P384;
  static const uint32_t* table() { return (const uint32_t*)ctx().p384_table; }
};
template <>
struct Curve<nistp::P521> {
  static constexpr int kid = KID_P521;
  static const uint32_t* table() { return (const uint32_t*)ctx().p521_table; }
};

// HashToScalar("Info" || I2OSP(len(info), 2) || info, "HashToScalar-" || contextString) of mode 2, once per call on the
// host (scalarFromInfo, oprf.go:156-170)
template <class C>
static Sc<C> info_scalar(const uint8_t* info, size_t len) {
  uint8_t ctx[24], dst[13 + 24];
  const int clen = oprf::context<C>(ctx, 2);
  for (int i = 0; i < 13; i++) dst[i] = (uint8_t)"HashToScalar-"[i];
  for (int i = 0; i < clen; i++) dst[13 + i] = ctx[i];
  const oprf::Len2 l((int)len);
  Sc<C> s;
  oprf::hash_to_scalar<C>(s, oprf::Cat<3>{{{(const uint8_t*)"Info", 4}, {l.b, 2}, {info, (int)len}}}, dst, 13 + clen);
  return s;
}

// the shared info string, copied into the call's level-1 work area (null when empty)
static int stage_info(int slot, const uint8_t* info, size_t len, size_t extra, Arena* A, const uint8_t** dinfo,
                      cudaStream_t st) {
  int rc = arena(slot, len + extra + 4096, A);
  if (rc) return rc;
  *dinfo = nullptr;
  if (len) {
    uint8_t* d = A->take(len);
    CB200_CUDA(cudaMemcpyAsync(d, info, len, cudaMemcpyHostToDevice, st));
    *dinfo = d;
  }
  return 0;
}

template <class C>
static int derive(const char* fn, int mode, const uint8_t* seeds, const uint8_t* info, size_t info_len, uint8_t* sk,
                  uint8_t* pk, size_t n) {
  constexpr size_t Ns = C::kBytes, Ne = oprf::kNe<C>;
  Batch b{fn, n, sk, 1u << 15, 1u << 12, {{seeds, 32, 32, kIn}, {sk, Ns, Ns, kOut}, {pk, Ne, Ne, kOut}}, {}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    Arena A;
    const uint8_t* dinfo;
    int rc = stage_info(slot, info, info_len, 0, &A, &dinfo, st);
    if (rc) return rc;
    {
      KernelScope ks(Curve<C>::kid, st);
      oprf_derive_kernel<C><<<blocks(cnt, 128), 128, 0, st>>>(r[0].p, dinfo, (int)info_len, mode, r[1].p, r[2].p,
                                                              Curve<C>::table(), cnt);
    }
    CB200_CUDA(cudaGetLastError());
    return 0;
  });
}

template <class C>
static int evaluate(const char* fn, int mode, const uint8_t* sk, size_t sk_stride, const uint8_t* blinded, size_t m,
                    const uint8_t* rnd, const uint8_t* info, size_t info_len, uint8_t* evaluated, uint8_t* proof,
                    uint8_t* status, size_t n) {
  constexpr size_t Ns = C::kBytes, Ne = oprf::kNe<C>;
  const Sc<C> mi = mode == 2 ? info_scalar<C>(info, info_len) : Sc<C>{};
  const size_t chunk = std::max<size_t>(1, (1u << 15) / m);
  const size_t pw = mode ? 2 * Ns : 0;
  Batch b{fn, n, evaluated, chunk, std::max<size_t>(1, (1u << 12) / m),
          {{sk, Ns, sk_stride, kIn}, {blinded, m * Ne, m * Ne, kIn}, {mode ? rnd : nullptr, Ns, Ns, kIn},
           {evaluated, m * Ne, m * Ne, kOut}, {mode ? proof : nullptr, pw, pw, kOut}, {status, 1, 1, kStatus}},
          {}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    Arena A;
    int rc = arena(slot, cnt * (m + Ne + 2 * Ns) + 4096, &A);
    if (rc) return rc;
    uint8_t *estat = A.take(cnt * m), *ybuf = A.take(cnt * Ne), *mbuf = A.take(cnt * 2 * Ns);
    KernelScope ks(Curve<C>::kid, st);
    oprf_eval_kernel<C><<<blocks(cnt * m, 128), 128, 0, st>>>(r[0].p, r[0].stride, r[1].p, m, mode, mi, r[3].p, estat,
                                                             cnt * m);
    if (mode)
      oprf_composite_kernel<C><<<blocks(cnt, 128), 128, 0, st>>>(r[0].p, r[0].stride, r[1].p, r[3].p, m, mode, mi,
                                                                 ybuf, mbuf, Curve<C>::table(), cnt);
    oprf_proof_kernel<C><<<blocks(cnt, 128), 128, 0, st>>>(r[0].p, r[0].stride, r[2].p, m, mode, mi, ybuf, mbuf, estat,
                                                          r[3].p, r[4].p, r[5].p, Curve<C>::table(), cnt);
    CB200_CUDA(cudaGetLastError());
    return 0;
  });
}

template <class C>
static int full(const char* fn, int mode, const uint8_t* sk, size_t sk_stride, const uint8_t* msgs,
                const uint64_t* msg_off, const uint8_t* info, size_t info_len, uint8_t* out, uint8_t* status,
                size_t n) {
  constexpr size_t Ns = C::kBytes, Nh = oprf::kNh<C>;
  const Sc<C> mi = mode == 2 ? info_scalar<C>(info, info_len) : Sc<C>{};
  Batch b{fn, n, out, 1u << 15, 1u << 12, {{sk, Ns, sk_stride, kIn}, {out, Nh, Nh, kOut}, {status, 1, 1, kStatus}},
          {{!aligned({msg_off}, {}, 8), "%s: device msg_off must be 8-byte aligned"}}, msgs, msg_off};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    Arena A;
    const uint8_t* dinfo;
    int rc = stage_info(slot, info, info_len, 0, &A, &dinfo, st);
    if (rc) return rc;
    {
      KernelScope ks(Curve<C>::kid, st);
      oprf_full_kernel<C><<<blocks(cnt, 128), 128, 0, st>>>(r[0].p, r[0].stride, mode, mi, r.msgs, r.msg_off, dinfo,
                                                            (int)info_len, r[1].p, r[2].p, cnt);
    }
    CB200_CUDA(cudaGetLastError());
    return 0;
  });
}

static size_t scalar_bytes(int suite) {
  return suite == CB200_OPRF_P256_SHA256 ? 32 : suite == CB200_OPRF_P384_SHA384 ? 48 : suite == CB200_OPRF_P521_SHA512 ? 66 : 0;
}
// the argument rules every entry point shares: a known suite and mode, a null-free call, info of at most 65535 bytes
static int check(const char* fn, int suite, int mode, const void* a, const void* b, const uint8_t* info, size_t info_len) {
  int rc = require_ready();
  if (rc) return rc;
  if (!scalar_bytes(suite) || mode < 0 || mode > 2 || !a || !b || (info_len && !info) || info_len > 65535) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  return 0;
}

}  // namespace oprfk
}  // namespace cb200

using namespace cb200;
using namespace cb200::oprfk;

extern "C" {

size_t cb200_oprf_element_size(int suite) { return scalar_bytes(suite) ? 1 + scalar_bytes(suite) : 0; }
size_t cb200_oprf_scalar_size(int suite) { return scalar_bytes(suite); }
size_t cb200_oprf_output_size(int suite) { return scalar_bytes(suite) == 66 ? 64 : scalar_bytes(suite); }
size_t cb200_oprf_proof_size(int suite) { return 2 * scalar_bytes(suite); }

int cb200_oprf_derive_key(int suite, int mode, const uint8_t* seeds, const uint8_t* info, size_t info_len, uint8_t* sk,
                          uint8_t* pk, size_t n) {
  const char* fn = "cb200_oprf_derive_key";
  int rc = check(fn, suite, mode, seeds, sk, info, info_len);
  if (rc) return rc;
  if (!pk) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
#define CALL(C) derive<C>(fn, mode, seeds, info, info_len, sk, pk, n)
  switch (suite) {
    case CB200_OPRF_P256_SHA256: return CALL(nistp::P256);
    case CB200_OPRF_P384_SHA384: return CALL(nistp::P384);
    default: return CALL(nistp::P521);
  }
#undef CALL
}

int cb200_oprf_evaluate(int suite, int mode, const uint8_t* sk, size_t sk_stride, const uint8_t* blinded, size_t m,
                        const uint8_t* rnd, const uint8_t* info, size_t info_len, uint8_t* evaluated, uint8_t* proof,
                        uint8_t* status, size_t n) {
  const char* fn = "cb200_oprf_evaluate";
  int rc = check(fn, suite, mode, sk, blinded, info, info_len);
  if (rc) return rc;
  if (!evaluated || !status || m < 1 || m > 65535 || (mode && (!rnd || !proof)) ||
      (sk_stride && sk_stride < scalar_bytes(suite))) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
#define CALL(C) evaluate<C>(fn, mode, sk, sk_stride, blinded, m, rnd, info, info_len, evaluated, proof, status, n)
  switch (suite) {
    case CB200_OPRF_P256_SHA256: return CALL(nistp::P256);
    case CB200_OPRF_P384_SHA384: return CALL(nistp::P384);
    default: return CALL(nistp::P521);
  }
#undef CALL
}

int cb200_oprf_full_evaluate(int suite, int mode, const uint8_t* sk, size_t sk_stride, const uint8_t* msgs,
                             const uint64_t* msg_off, const uint8_t* info, size_t info_len, uint8_t* out,
                             uint8_t* status, size_t n) {
  const char* fn = "cb200_oprf_full_evaluate";
  int rc = check(fn, suite, mode, sk, out, info, info_len);
  if (rc) return rc;
  if (!msgs || !msg_off || !status || (sk_stride && sk_stride < scalar_bytes(suite))) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  if (!is_device_ptr(msg_off)) {  // inputs of at most 65535 bytes (RFC 9497 section 3.3; the reference truncates)
    for (size_t i = 0; i < n; i++)
      if (msg_off[i + 1] < msg_off[i] || msg_off[i + 1] - msg_off[i] > 65535) {
        set_error("%s: input %zu is longer than 65535 bytes", fn, i);
        return CB200_ERR_ARG;
      }
  }
#define CALL(C) full<C>(fn, mode, sk, sk_stride, msgs, msg_off, info, info_len, out, status, n)
  switch (suite) {
    case CB200_OPRF_P256_SHA256: return CALL(nistp::P256);
    case CB200_OPRF_P384_SHA384: return CALL(nistp::P384);
    default: return CALL(nistp::P521);
  }
#undef CALL
}

}  // extern "C"
