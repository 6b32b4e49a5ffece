// circl_b200/csrc/dil_kernels.cu -- batched q=8380417 kernels (sm_90a), launchers and C ABI.
//
// cb200_dil_ntt      <- (*Poly).NTT / InvNTT   sign/internal/dilithium/generic.go:11,15 (stubs_amd64.go:8-14)
// cb200_dil_mulhat   <- (*Poly).MulHat         generic.go:19 (poly.go:88)
// cb200_dil_dot      <- PolyDotHat             sign/mldsa/mldsa65/internal/mat.go:52-59
// cb200_dil_poly_op  <- Add/Sub/ReduceLe2Q/Normalize/NormalizeAssumingLe2Q/MulBy2toD   generic.go:23-89
// cb200_dil_exceeds  <- (*Poly).Exceeds        generic.go (poly.go:51-71; stubs_amd64.go:32 exceedsAVX2)
#include "../../include/circl_b200.h"
#include "context.h"
#include "dilithium.cuh"
#include "flow_internal.h"

namespace cb200 {
namespace dil {

constexpr int kThreads = 128;
constexpr int kOctetsPerCta = kThreads / 8;

// In-place NTT / InvNTT: 1 KiB read + 1 KiB written per polynomial.  Twiddle pairs of the C-layout pass come from a
// staged shared-memory copy (dilithium.cuh: stage_pairs), those of the S-layout pass are immediates.
template <bool INV>
__global__ void __launch_bounds__(kThreads, 6) ntt_kernel(uint32_t* __restrict__ polys, size_t n,
                                                          const uint32_t* __restrict__ zetas /* dil_fill_twiddles */) {
  __shared__ __align__(16) uint32_t tiles[kOctetsPerCta * kPolyWords];
  __shared__ __align__(8) uint2 pairs[256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, oct = lane >> 3, v = lane & 7;
  uint32_t* tile = tiles + (warp * 4 + oct) * kPolyWords;
  stage_pairs<INV>(pairs, zetas);
  __syncthreads();
  const volatile uint2* zs = pairs;
  const size_t stride = (size_t)gridDim.x * kOctetsPerCta;
  for (size_t base = ((size_t)blockIdx.x * 4 + warp) * 4; base < n; base += stride) {
    const size_t p = base + oct;
    const bool active = p < n;
    uint32_t* poly = polys + (active ? p : n - 1) * N;
    uint32_t r[32];
    // The C-layout side of either transform goes to / comes from memory in the interleaved "I" layout (dilithium.cuh):
    // an octet then moves 128 contiguous bytes per instruction instead of eight 16-byte pieces 128 bytes apart (one
    // L1 wavefront per lane: ncu showed the kernel waiting on the memory pipeline, mio / lg throttle, with both integer
    // pipes under 35 %); the change of layout is one more pass through the octet's tile.
    if (!INV) {
      gload_S(poly, v, r);
      ntt_octet_smem(r, tile, v, zs);
      gstore_C_via_tile(poly, tile, v, r, active);
    } else {
      uint4 w[8];
      gload_I(poly, v, w);
#pragma unroll
      for (int c = 0; c < 8; c++) {
        r[4 * c] = w[c].x;
        r[4 * c + 1] = w[c].y;
        r[4 * c + 2] = w[c].z;
        r[4 * c + 3] = w[c].w;
      }
      i_to_c(r, tile, v);
      invntt_octet_smem(r, tile, v, zs);
      if (active) gstore_S(poly, v, r);
    }
  }
}

// out[i] = sum_{j<k} MulHat(a[i*k+j], b[i*k+j]); one thread per 4 coefficients
__global__ void __launch_bounds__(256) dot_kernel(uint4* __restrict__ out, const uint4* __restrict__ a,
                                                  const uint4* __restrict__ b, int k, size_t n) {
  const size_t nvec = n * (N / 4);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    const size_t p = i / (N / 4), c = i % (N / 4);
    uint4 acc = make_uint4(0, 0, 0, 0);
    for (int j = 0; j < k; j++) {
      const uint4 x = a[(p * k + j) * (N / 4) + c], y = b[(p * k + j) * (N / 4) + c];
      acc.x += mont_mul(x.x, y.x);
      acc.y += mont_mul(x.y, y.y);
      acc.z += mont_mul(x.z, y.z);
      acc.w += mont_mul(x.w, y.w);
    }
    out[i] = acc;
  }
}

enum { OP_ADD = 0, OP_SUB, OP_REDUCE_LE2Q, OP_NORMALIZE, OP_NORMALIZE_LE2Q, OP_MUL_2D };
template <int OP>
__device__ __forceinline__ uint32_t ew(uint32_t x, uint32_t y) {
  if (OP == OP_ADD) return x + y;
  if (OP == OP_SUB) return x + (2 * Q - y);  // poly.go:41-45
  if (OP == OP_REDUCE_LE2Q) return reduce_le2q(x);
  if (OP == OP_NORMALIZE) return modq(x);
  if (OP == OP_NORMALIZE_LE2Q) return le2q_modq(x);
  return x << 13;  // mulBy2toD, poly.go:97
}
template <int OP>
__global__ void __launch_bounds__(256) ew_kernel(uint4* __restrict__ out, const uint4* __restrict__ a,
                                                 const uint4* __restrict__ b, size_t nvec) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 x = a[i];
    uint4 y = make_uint4(0, 0, 0, 0);
    if (OP == OP_ADD || OP == OP_SUB) y = b[i];
    out[i] = make_uint4(ew<OP>(x.x, y.x), ew<OP>(x.y, y.y), ew<OP>(x.z, y.z), ew<OP>(x.w, y.w));
  }
}

// flags[p] = Exceeds(poly p, bound): one warp per polynomial
__global__ void __launch_bounds__(256) exceeds_kernel(const uint4* __restrict__ a, uint32_t bound, size_t n,
                                                      uint8_t* __restrict__ flags) {
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= n) return;
  bool ex = false;
#pragma unroll
  for (int c = 0; c < 2; c++) {
    const uint4 x = a[warp * (N / 4) + c * 32 + lane];
    ex |= exceeds1(x.x, bound) | exceeds1(x.y, bound) | exceeds1(x.z, bound) | exceeds1(x.w, bound);
  }
  ex = __any_sync(0xffffffffu, ex);
  if (lane == 0) flags[warp] = ex ? 1 : 0;
}

// (*Poly).Power2Round (poly.go:77-84, field.go:35-49): a = a1 2^13 + a0 with -2^12 < a0 <= 2^12; returns Q + a0 and a1
__device__ __forceinline__ void power2round1(uint32_t a, uint32_t& a0q, uint32_t& a1) {
  uint32_t a0 = a & 0x1fff;
  a0 -= (1u << 12) + 1;
  a0 += (uint32_t)((int32_t)a0 >> 31) & (1u << 13);
  a0 -= (1u << 12) - 1;
  a0q = Q + a0;
  a1 = (a - a0) >> 13;
}
__global__ void __launch_bounds__(256) power2round_kernel(uint4* __restrict__ a0q, uint4* __restrict__ a1,
                                                          const uint4* __restrict__ a, size_t nvec) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 x = a[i];
    uint4 lo, hi;
    power2round1(x.x, lo.x, hi.x);
    power2round1(x.y, lo.y, hi.y);
    power2round1(x.z, lo.z, hi.z);
    power2round1(x.w, lo.w, hi.w);
    a0q[i] = lo;
    a1[i] = hi;
  }
}
// (*Poly).PackLe16 (pack.go:102-108): thread per 8 coefficients -> 4 bytes
__global__ void __launch_bounds__(256) pack_le16_kernel(uint32_t* __restrict__ out, const uint4* __restrict__ a, size_t nwords) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 x = a[2 * i], y = a[2 * i + 1];
    const uint32_t c[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
    uint32_t w = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) w |= (uint32_t)(uint8_t)(c[2 * k] | (c[2 * k + 1] << 4)) << (8 * k);
    out[i] = w;
  }
}

static int grid_for(size_t units, int per_cta, int ctas_per_sm) {
  size_t want = (units + per_cta - 1) / per_cta;
  size_t cap = (size_t)ctx().sm_count * ctas_per_sm;
  return (int)(want < cap ? (want ? want : 1) : cap);
}

}  // namespace dil

int launch_dil_ntt(uint32_t* d_polys, size_t n, int inverse, const void* tw, cudaStream_t st) {
  using namespace dil;
  if (n == 0) return 0;
  const int grid = grid_for(n, kOctetsPerCta, 6);
  KernelScope ks(inverse ? KID_DIL_INVNTT : KID_DIL_NTT, st);
  if (inverse)
    ntt_kernel<true><<<grid, kThreads, 0, st>>>(d_polys, n, (const uint32_t*)tw);
  else
    ntt_kernel<false><<<grid, kThreads, 0, st>>>(d_polys, n, (const uint32_t*)tw);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

int launch_dil_dot(uint32_t* out, const uint32_t* a, const uint32_t* b, int k, size_t n, cudaStream_t st) {
  using namespace dil;
  if (n == 0) return 0;
  KernelScope ks(KID_DIL_DOT, st);
  dot_kernel<<<grid_for(n * (N / 4), 256, 8), 256, 0, st>>>((uint4*)out, (const uint4*)a, (const uint4*)b, k, n);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

int launch_dil_poly_op(int op, uint32_t* out, const uint32_t* a, const uint32_t* b, size_t n, cudaStream_t st) {
  using namespace dil;
  if (n == 0) return 0;
  const size_t nvec = n * (N / 4);
  const int grid = grid_for(nvec, 256, 8);
  uint4* o = (uint4*)out;
  const uint4 *x = (const uint4*)a, *y = (const uint4*)b;
  KernelScope ks(KID_DIL_EW, st);
  switch (op) {
    case OP_ADD: ew_kernel<OP_ADD><<<grid, 256, 0, st>>>(o, x, y, nvec); break;
    case OP_SUB: ew_kernel<OP_SUB><<<grid, 256, 0, st>>>(o, x, y, nvec); break;
    case OP_REDUCE_LE2Q: ew_kernel<OP_REDUCE_LE2Q><<<grid, 256, 0, st>>>(o, x, y, nvec); break;
    case OP_NORMALIZE: ew_kernel<OP_NORMALIZE><<<grid, 256, 0, st>>>(o, x, y, nvec); break;
    case OP_NORMALIZE_LE2Q: ew_kernel<OP_NORMALIZE_LE2Q><<<grid, 256, 0, st>>>(o, x, y, nvec); break;
    case OP_MUL_2D: ew_kernel<OP_MUL_2D><<<grid, 256, 0, st>>>(o, x, y, nvec); break;
    default: set_error("cb200_dil_poly_op: unknown op %d", op); return CB200_ERR_ARG;
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

int launch_dil_exceeds(const uint32_t* a, uint32_t bound, size_t n, uint8_t* flags, cudaStream_t st) {
  using namespace dil;
  if (n == 0) return 0;
  KernelScope ks(KID_DIL_EW, st);
  exceeds_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>((const uint4*)a, bound, n, flags);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

int launch_dil_power2round(uint32_t* a0q, uint32_t* a1, const uint32_t* a, size_t n, cudaStream_t st) {
  using namespace dil;
  if (n == 0) return 0;
  KernelScope ks(KID_DIL_EW, st);
  const size_t nvec = n * (N / 4);
  power2round_kernel<<<grid_for(nvec, 256, 8), 256, 0, st>>>((uint4*)a0q, (uint4*)a1, (const uint4*)a, nvec);
  CB200_CUDA(cudaGetLastError());
  return 0;
}
int launch_dil_pack_le16(uint8_t* out, const uint32_t* a, size_t n, cudaStream_t st) {
  using namespace dil;
  if (n == 0) return 0;
  KernelScope ks(KID_DIL_EW, st);
  const size_t nwords = n * (N / 8);
  pack_le16_kernel<<<grid_for(nwords, 256, 8), 256, 0, st>>>((uint32_t*)out, (const uint4*)a, nwords);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

void dil_fill_twiddles(uint32_t* out /* dil::kTwWords: Zetas | InvZetas | forward pairs | inverse pairs */) {
  for (int i = 0; i < 256; i++) {
    const uint32_t z = dil::zeta_of(i), iz = dil::inv_zeta_of(i);
    out[i] = z;
    out[256 + i] = iz;
    out[dil::kTwFwdPairs + 2 * i] = dil::shoup_p(z);
    out[dil::kTwFwdPairs + 2 * i + 1] = dil::shoup_k(z);
    out[dil::kTwInvPairs + 2 * i] = dil::shoup_p(iz);
    out[dil::kTwInvPairs + 2 * i + 1] = dil::shoup_k(iz);
  }
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_dil_ntt(uint32_t* polys, size_t n, int inverse) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!polys) {
    set_error("cb200_dil_ntt: null pointer");
    return CB200_ERR_ARG;
  }
  Batch b{"cb200_dil_ntt", n, polys, 1u << 16, 1u << 14, {{polys, 1024, 1024, kInOut}},
          {{!aligned({polys}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch_dil_ntt((uint32_t*)r[0].p, cnt, inverse, ctx().dil_tw, st);
  });
}

int cb200_dil_dot(uint32_t* out, const uint32_t* a, const uint32_t* b, int k, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!out || !a || !b || k < 1 || k > 8) {
    set_error("cb200_dil_dot: bad argument");
    return CB200_ERR_ARG;
  }
  const size_t ku = 1024 * (size_t)k;
  Batch bt{"cb200_dil_dot", n, out, (1u << 16) / k, (1u << 14) / k,
           {{out, 1024, 1024, kOut}, {a, ku, ku, kIn}, {b, ku, ku, kIn}},
           {{!aligned({out, a, b}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(bt, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch_dil_dot((uint32_t*)r[0].p, (const uint32_t*)r[1].p, (const uint32_t*)r[2].p, k, cnt, st);
  });
}

int cb200_dil_mulhat(uint32_t* out, const uint32_t* a, const uint32_t* b, size_t n) {
  return cb200_dil_dot(out, a, b, 1, n);
}

int cb200_dil_poly_op(int op, uint32_t* out, const uint32_t* a, const uint32_t* b, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  const bool binary = (op == CB200_DIL_OP_ADD || op == CB200_DIL_OP_SUB);
  if (!out || !a || (binary && !b) || op < 0 || op > CB200_DIL_OP_MUL_2D) {
    set_error("cb200_dil_poly_op: bad argument");
    return CB200_ERR_ARG;
  }
  if (!binary) b = nullptr;
  Batch bt{"cb200_dil_poly_op", n, out, 1u << 16, 1u << 14,
           {{out, 1024, 1024, kOut}, {a, 1024, 1024, kIn}, {b, 1024, 1024, kIn}},
           {{!aligned({out, a, b}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(bt, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch_dil_poly_op(op, (uint32_t*)r[0].p, (const uint32_t*)r[1].p, (const uint32_t*)r[2].p, cnt, st);
  });
}

int cb200_dil_exceeds(const uint32_t* polys, uint32_t bound, uint8_t* flags, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!polys || !flags) {
    set_error("cb200_dil_exceeds: null pointer");
    return CB200_ERR_ARG;
  }
  Batch b{"cb200_dil_exceeds", n, polys, 1u << 16, 1u << 14, {{polys, 1024, 1024, kIn}, {flags, 1, 1, kOut}},
          {{!aligned({polys}, {}, 16), "%s: device polynomials must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch_dil_exceeds((const uint32_t*)r[0].p, bound, cnt, r[1].p, st);
  });
}

int cb200_dil_power2round(uint32_t* a0plusq, uint32_t* a1, const uint32_t* a, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!a0plusq || !a1 || !a) {
    set_error("cb200_dil_power2round: null pointer");
    return CB200_ERR_ARG;
  }
  Batch b{"cb200_dil_power2round", n, a, 1u << 16, 1u << 14,
          {{a, 1024, 1024, kIn}, {a0plusq, 1024, 1024, kOut}, {a1, 1024, 1024, kOut}},
          {{!aligned({a0plusq, a1, a}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch_dil_power2round((uint32_t*)r[1].p, (uint32_t*)r[2].p, (const uint32_t*)r[0].p, cnt, st);
  });
}

int cb200_dil_pack_le16(uint8_t* out, const uint32_t* polys, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!out || !polys) {
    set_error("cb200_dil_pack_le16: null pointer");
    return CB200_ERR_ARG;
  }
  Batch b{"cb200_dil_pack_le16", n, out, 1u << 16, 1u << 14, {{polys, 1024, 1024, kIn}, {out, 128, 128, kOut}},
          {{!aligned({out}, {}, 4) || !aligned({polys}, {}, 16),
            "%s: device buffers must be aligned (polynomials 16, output 4 bytes)"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch_dil_pack_le16(r[1].p, (const uint32_t*)r[0].p, cnt, st);
  });
}

}  // extern "C"
