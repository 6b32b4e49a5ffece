// circl_b200/csrc/kyber_kernels.cu -- batched q=3329 kernels (sm_90a) and their launchers.
//
// cb200_kyber_ntt      <- (*Poly).NTT / InvNTT      pke/kyber/internal/common/generic.go:24,36 (stubs_amd64.go:8-14)
// cb200_kyber_mulhat   <- (*Poly).MulHat            generic.go:49 (stubs_amd64.go:17)
// cb200_kyber_dot      <- PolyDotHat                pke/kyber/kyber768/internal/vec.go:30-37
// cb200_kyber_poly_op  <- Add/Sub/BarrettReduce/Normalize/ToMont  generic.go:7-77, poly.go:48
#include "context.h"
#include "kyber.cuh"
#include "launch.h"

namespace cb200 {
namespace kyber {

constexpr int kThreads = 128;               // 4 warps = 16 octets = 16 polynomials in flight per CTA
constexpr int kOctetsPerCta = kThreads / 8;

// out[i] = sum_{j<k} MulHat(a[i*k+j], b[i*k+j])   (k = 1: plain MulHat)
__global__ void __launch_bounds__(kThreads) dot_kernel(uint32_t* __restrict__ out, const uint32_t* __restrict__ a,
                                                       const uint32_t* __restrict__ b, int k, size_t n,
                                                       const TwPair* __restrict__ tw) {
  const int v = threadIdx.x & 7;
  LaneTw t;
  load_lane_tw(t, tw, v);
  const size_t stride = (size_t)gridDim.x * kOctetsPerCta;
  for (size_t p = (size_t)blockIdx.x * kOctetsPerCta + (threadIdx.x >> 3); p < n; p += stride) {
    int32_t acc[32];
#pragma unroll
    for (int i = 0; i < 32; i++) acc[i] = 0;
    for (int j = 0; j < k; j++) {
      int32_t x[32], y[32];
      gload_C(a + (p * k + j) * (N / 2), v, x);
      gload_C(b + (p * k + j) * (N / 2), v, y);
      mulhat_acc_C(acc, x, y, t);
    }
    gstore_C(out + p * (N / 2), v, acc);
  }
}

// element-wise family; one thread handles 8 coefficients (one 128-bit access)
enum PolyOp { OP_ADD = 0, OP_SUB = 1, OP_BARRETT = 2, OP_NORMALIZE = 3, OP_TOMONT = 4 };
template <int OP>
__device__ __forceinline__ int32_t ew(int32_t x, int32_t y) {
  if (OP == OP_ADD) return x + y;
  if (OP == OP_SUB) return x - y;
  if (OP == OP_BARRETT) return barrett_hi(x);
  if (OP == OP_NORMALIZE) return csubq_hi(barrett_hi(x));
  return mont_mul_hi(x >> 16, 1353, (int32_t)(((1353u * QINV) & 0xffffu) << 16));  // toMont, field.go:35-39
}
template <int OP>
__global__ void __launch_bounds__(256) ew_kernel(uint4* __restrict__ out, const uint4* __restrict__ a,
                                                 const uint4* __restrict__ b, size_t nvec) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    uint4 x = ldg_stream128(a + i), y = make_uint4(0, 0, 0, 0);
    if (OP == OP_ADD || OP == OP_SUB) y = ldg_stream128(b + i);
    uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w}, o[4];
#pragma unroll
    for (int w = 0; w < 4; w++) {
      int32_t xl, xh, yl, yh;
      unpack2(xs[w], xl, xh);
      unpack2(ys[w], yl, yh);
      o[w] = pack2(ew<OP>(xl, yl), ew<OP>(xh, yh));
    }
    stg_stream128(out + i, make_uint4(o[0], o[1], o[2], o[3]));
  }
}

// ---------------------------------------------------------------- fast-path kernels (see kyber.cuh, "low" format)
__device__ __forceinline__ void gstore_C_lo(uint32_t* __restrict__ poly, int v, const int32_t (&r)[32]) {
#pragma unroll
  for (int c = 0; c < 4; c++)
    stg_stream128(poly + 16 * v + 4 * c,
                  make_uint4(pack2_lo(r[8 * c], r[8 * c + 1]), pack2_lo(r[8 * c + 2], r[8 * c + 3]),
                             pack2_lo(r[8 * c + 4], r[8 * c + 5]), pack2_lo(r[8 * c + 6], r[8 * c + 7])));
}
__device__ __forceinline__ void gstore_S_lo(uint32_t* __restrict__ poly, int v, const int32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++) poly[8 * s + v] = pack2_lo(r[2 * s], r[2 * s + 1]);
}

constexpr int kSlotWords = 136;  // 512 B of coefficients + 32 B: consecutive octets start 8 banks apart
constexpr int kFwdCtasPerSm = 5, kInvCtasPerSm = 6;

// Forward NTT, in place.  HBM traffic: 512 B read + 512 B written per polynomial (the algorithmic minimum).
//   * Input: every octet owns a 544-byte slot; lane 0 of the octet has the TMA engine copy the octet's next polynomial
//     into it (UBLKCP, 512 B, one mbarrier per octet) as soon as the current one is in registers, so the copy has a
//     whole iteration to land.  Slots are 136 words apart: the raw S-layout reads (word 8s + v) of the four octets of a
//     warp fall on 32 different banks.
//   * In-contract polynomials (words_in_range, warp-uniform vote) run the low-format fast path of kyber.cuh: 5-instruction
//     butterflies, 128-bit transposition through the octet's own tile, per-lane twiddle pairs in registers.  Any other
//     input runs the general high-half code (int16 wrap-around exact) on the same words.
// 5 CTAs per SM: the kernel is bound by the two integer pipes.  Tried and dropped: the pairs read from shared memory at
// 6 / 7 CTAs per SM, two slots per octet, the whole shared-memory carve-out, and output / input of the C-layout side in
// 128-byte-contiguous order through the tile (what the Dilithium kernels do: their lanes are 128 bytes apart and they wait
// on the memory pipeline), which costs these pipe-bound kernels eight more shared-memory instructions per polynomial.
__global__ void __launch_bounds__(kThreads, kFwdCtasPerSm) ntt_fwd_kernel(uint32_t* __restrict__ polys, size_t n,
                                                                          const TwPair* __restrict__ tw) {
  extern __shared__ __align__(16) unsigned char dsm[];
  TwPair* tws = reinterpret_cast<TwPair*>(dsm);               // 128 x {zeta, zetaq}, then 128 x {zp, kk} (tw_slot order)
  uint32_t* slots = reinterpret_cast<uint32_t*>(dsm + 2048);  // [16 octets][kSlotWords]
  unsigned char* tiles = dsm + 2048 + kOctetsPerCta * kSlotWords * 4;
  uint64_t* bars = reinterpret_cast<uint64_t*>(tiles + kOctetsPerCta * kWideTileBytes);  // one per octet, then the table's
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int oct = lane >> 3, v = lane & 7, ob = warp * 4 + oct;
  unsigned char* tile = tiles + ob * kWideTileBytes;
  uint32_t* slot = slots + ob * kSlotWords;
  uint64_t* obar = bars + ob;
  uint64_t* tbar = bars + kOctetsPerCta;
  if (threadIdx.x == 0) mbar_init(tbar, 1);
  if (v == 0) mbar_init(obar, 1);
  fence_barrier_init();
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(tbar, 2048);
    bulk_g2s(tws, tw, 2048, tbar);
  }
  // Every octet walks its own polynomials p = first + oct + it * stride < n; the warp loops until its first octet (the
  // one with the most) is done, and an octet that has run out neither issues nor waits nor stores.
  const size_t stride = (size_t)gridDim.x * kOctetsPerCta, first = ((size_t)blockIdx.x * 4 + warp) * 4;
  const uint32_t n_it = first < n ? (uint32_t)((n - first + stride - 1) / stride) : 0;               // of the warp
  const uint32_t my_it = first + oct < n ? (uint32_t)((n - first - oct + stride - 1) / stride) : 0;  // of this octet
  const size_t step_words = stride * (N / 2);
  uint32_t* gp = polys + (first + oct) * (N / 2);  // the polynomial this octet transforms in iteration `it`
  const uint32_t* nxt = gp;                         // the next polynomial to request
  uint32_t issued = 0;
  auto issue = [&]() {  // lane 0 of the octet
    mbar_expect_tx(obar, N * 2);
    bulk_g2s(slot, nxt, N * 2, obar);
    nxt += step_words;
    issued++;
  };
  if (v == 0 && my_it > 0) issue();
  mbar_wait(tbar, 0);
  LaneTwLow t;
  load_lane_tw_lo(t, reinterpret_cast<const TwLow*>(tws + 128), v);
  for (uint32_t it = 0; it < n_it; it++, gp += step_words) {
    const bool active = it < my_it;
    uint32_t w[16];
    if (active) {
      mbar_wait(obar, it & 1);
#pragma unroll
      for (int s = 0; s < 16; s++) w[s] = slot[8 * s + v];
    } else {
#pragma unroll
      for (int s = 0; s < 16; s++) w[s] = 0;
    }
    // warp-uniform choice; the vote also orders every lane's slot reads before the refill below
    const bool fast = __all_sync(0xffffffffu, words_in_range(w, kFwdBound));
    if (v == 0 && issued < my_it) {
      fence_proxy_async();
      issue();
    }
    int32_t r[32];
    if (fast) {
#pragma unroll
      for (int s = 0; s < 16; s++) unpack2_lo(w[s], r[2 * s], r[2 * s + 1]);
      fwd_pass_S_lo(r);
      wide_store_S(tile, v, r);
      __syncwarp();
      wide_load_C(tile, v, r);
      fwd_pass_C_lo(r, t);
      if (active) gstore_C_lo(gp, v, r);
    } else {
#pragma unroll
      for (int s = 0; s < 16; s++) unpack2_ct(w[s], r[2 * s], r[2 * s + 1]);
      fwd_pass_S(r);
      store_S(reinterpret_cast<uint32_t*>(tile), v, r);
      __syncwarp();
      load_C_ct(reinterpret_cast<const uint32_t*>(tile), v, r);
      fwd_pass_C_smem(r, tws, v);
      if (active) gstore_C(gp, v, r);
    }
    __syncwarp();  // the tile is free again
  }
}
constexpr int kFwdSmem = 2048 + kOctetsPerCta * kSlotWords * 4 + kOctetsPerCta * kWideTileBytes + (kOctetsPerCta + 1) * 8;

// Inverse NTT, in place: C-layout input as four 128-bit loads per lane, the next polynomial's words requested before
// the current one is transformed; the same fast / general split (bound kInvBound); S-layout output as sixteen 32-bit
// stores per lane (one full sector per octet and instruction).
__global__ void __launch_bounds__(kThreads, kInvCtasPerSm) ntt_inv_kernel(uint32_t* __restrict__ polys, size_t n,
                                                                          const TwPair* __restrict__ tw) {
  __shared__ __align__(16) unsigned char tiles[kOctetsPerCta * kWideTileBytes];
  __shared__ __align__(16) TwPair tws[256];
  __shared__ __align__(8) uint64_t bar;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int oct = lane >> 3, v = lane & 7;
  unsigned char* tile = tiles + (warp * 4 + oct) * kWideTileBytes;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar, sizeof(tws));
    bulk_g2s(tws, tw, sizeof(tws), &bar);
  }
  const size_t stride = (size_t)gridDim.x * kOctetsPerCta;
  auto poly_at = [&](size_t base) {
    const size_t p = base + oct;
    return polys + (p < n ? p : n - 1) * (N / 2);  // idle octets recompute the last polynomial, never store
  };
  auto fetch = [&](const uint32_t* poly, uint32_t (&w)[16]) {
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const uint4 q4 = ldg_stream128(poly + 16 * v + 4 * c);
      w[4 * c] = q4.x;
      w[4 * c + 1] = q4.y;
      w[4 * c + 2] = q4.z;
      w[4 * c + 3] = q4.w;
    }
  };
  size_t base = ((size_t)blockIdx.x * 4 + warp) * 4;
  uint32_t wn[16];
  if (base < n) fetch(poly_at(base), wn);
  mbar_wait(&bar, 0);
  const volatile TwPair* tab = tws;
  const volatile TwLow* tabl = reinterpret_cast<const volatile TwLow*>(tws + 128);
  for (; base < n; base += stride) {
    const bool active = base + oct < n;
    uint32_t* poly = poly_at(base);
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = wn[i];
    if (base + stride < n) fetch(poly_at(base + stride), wn);
    const bool fast = __all_sync(0xffffffffu, words_in_range(w, kInvBound));
    int32_t r[32];
    if (fast) {
#pragma unroll
      for (int j = 0; j < 16; j++) unpack2_lo(w[j], r[2 * j], r[2 * j + 1]);
      inv_pass_C_lo(r, tabl, v);
      wide_store_C(tile, v, r);
      __syncwarp();
      wide_load_S(tile, v, r);
      inv_pass_S_lo(r, v);
      if (active) gstore_S_lo(poly, v, r);
    } else {
#pragma unroll
      for (int j = 0; j < 16; j++) unpack2(w[j], r[2 * j], r[2 * j + 1]);
      inv_pass_C_smem(r, tab, v);
      store_C(reinterpret_cast<uint32_t*>(tile), v, r);
      __syncwarp();
      load_S(reinterpret_cast<const uint32_t*>(tile), v, r);
      inv_pass_S(r, v);
      if (active) gstore_S(poly, v, r);
    }
    __syncwarp();
  }
}

static int grid_for(size_t units, int per_cta, int ctas_per_sm) {
  size_t want = (units + per_cta - 1) / per_cta;
  size_t cap = (size_t)ctx().sm_count * ctas_per_sm;
  return (int)(want < cap ? (want ? want : 1) : cap);
}

}  // namespace kyber

// ---------------------------------------------------------------- launchers (device pointers)
int launch_kyber_ntt(int16_t* d_polys, size_t n, int inverse, const void* tw, cudaStream_t st) {
  using namespace kyber;
  if (n == 0) return 0;
  KernelScope ks(inverse ? KID_KYBER_INVNTT : KID_KYBER_NTT, st);
  if (inverse)
    ntt_inv_kernel<<<grid_for(n, kOctetsPerCta, kInvCtasPerSm), kThreads, 0, st>>>((uint32_t*)d_polys, n, (const TwPair*)tw);
  else
    ntt_fwd_kernel<<<grid_for(n, kOctetsPerCta, kFwdCtasPerSm), kThreads, kFwdSmem, st>>>((uint32_t*)d_polys, n,
                                                                                         (const TwPair*)tw);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

int launch_kyber_dot(int16_t* d_out, const int16_t* d_a, const int16_t* d_b, int k, size_t n, const void* tw,
                     cudaStream_t st) {
  using namespace kyber;
  if (n == 0) return 0;
  int grid = grid_for(n, kOctetsPerCta, 8);
  KernelScope ks(KID_KYBER_DOT, st);
  dot_kernel<<<grid, kThreads, 0, st>>>((uint32_t*)d_out, (const uint32_t*)d_a, (const uint32_t*)d_b, k, n,
                                        (const TwPair*)tw);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

int launch_kyber_poly_op(int op, int16_t* d_out, const int16_t* d_a, const int16_t* d_b, size_t n, cudaStream_t st) {
  using namespace kyber;
  if (n == 0) return 0;
  size_t nvec = n * (N / 8);
  int grid = grid_for(nvec, 256, 8);
  uint4* o = (uint4*)d_out;
  const uint4 *a = (const uint4*)d_a, *b = (const uint4*)d_b;
  KernelScope ks(KID_KYBER_EW, st);
  switch (op) {
    case OP_ADD: ew_kernel<OP_ADD><<<grid, 256, 0, st>>>(o, a, b, nvec); break;
    case OP_SUB: ew_kernel<OP_SUB><<<grid, 256, 0, st>>>(o, a, b, nvec); break;
    case OP_BARRETT: ew_kernel<OP_BARRETT><<<grid, 256, 0, st>>>(o, a, b, nvec); break;
    case OP_NORMALIZE: ew_kernel<OP_NORMALIZE><<<grid, 256, 0, st>>>(o, a, b, nvec); break;
    case OP_TOMONT: ew_kernel<OP_TOMONT><<<grid, 256, 0, st>>>(o, a, b, nvec); break;
    default: set_error("cb200_kyber_poly_op: unknown op %d", op); return -1;
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// host-side twiddle table: {Zetas[k], (Zetas[k]*q^-1 mod 2^16) << 16}
void kyber_fill_twiddles(int32_t* out /* 128 x {zeta, zetaq}, then 128 x {zp, kk} in tw_slot order */) {
  for (int i = 0; i < 128; i++) {
    out[2 * i] = kyber::zeta_of(i);
    out[2 * i + 1] = kyber::zetaq_of(i);
    out[256 + 2 * kyber::tw_slot(i)] = kyber::zp_of(i);  // lane-transposed, see kyber.cuh
    out[256 + 2 * kyber::tw_slot(i) + 1] = kyber::kk_of(i);
  }
}

}  // namespace cb200
