// Round-2 pipe microbenchmarks (sm_90a): where can ALU-pipe work of the ML-KEM step move to?
//   1. Keccak-f[1600] with H of its 58 32-bit half-rotations per round computed on the FMA pipe
//      (IMAD.WIDE by 2^r from the constant bank + IMAD) instead of SHF on the ALU pipe.
//   2. The q = 3329 butterfly in exact fp32 integer arithmetic (FMUL/FFMA/FADD) against the int32 Montgomery one.
//   3. Both kinds of warps resident together (do the pipes overlap?).
// nvcc -O3 -std=c++17 --expt-relaxed-constexpr -gencode arch=compute_90a,code=sm_90a -I circl_b200/csrc scripts/ubench_r02.cu -o ubench_r02
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "keccak.cuh"

// multiprocessors of device 0: the grids below put the same number of CTAs on every SM
static int sms() {
  static int n = 0;
  if (!n) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0);
  return n;
}

using namespace cb200;

__constant__ uint32_t kPow2[32];

// (keep << R) | (in >> (32 - R)) on the FMA pipe: 1 IMAD.WIDE + 1 IMAD
template <int R>
__device__ __forceinline__ uint32_t half_rot_fma(uint32_t keep, uint32_t in) {
  uint64_t t;
  asm("mul.wide.u32 %0, %1, %2;" : "=l"(t) : "r"(in), "r"(kPow2[R]));
  uint32_t r;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(keep), "r"(kPow2[R]), "r"((uint32_t)(t >> 32)));
  return r;
}
template <int R>
__device__ __forceinline__ uint32_t half_rot_alu(uint32_t keep, uint32_t in) {
  return __funnelshift_l(in, keep, R);
}

// 64-bit rotate left by R; FH / FL: compute the high / low output word on the FMA pipe
template <int R, bool FH, bool FL>
__device__ __forceinline__ uint64_t rotl_mix(uint64_t v) {
  if constexpr (R == 0) {
    return v;
  } else {
    uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
    constexpr int S = R & 31;
    if constexpr (R >= 32) {
      uint32_t t = lo;
      lo = hi;
      hi = t;
    }
    uint32_t nhi, nlo;
    if constexpr (S == 0) {
      nhi = hi;
      nlo = lo;
    } else {
      nhi = FH ? half_rot_fma<S>(hi, lo) : half_rot_alu<S>(hi, lo);
      nlo = FL ? half_rot_fma<S>(lo, hi) : half_rot_alu<S>(lo, hi);
    }
    return ((uint64_t)nhi << 32) | nlo;
  }
}

// Offload policy: H half-rotations per round go to the FMA pipe.  Order: first one half of each of the 24 rho lanes
// (hybrid), then the theta rot-1 halves, then the second halves.
template <int H>
struct Policy {
  static constexpr bool rho_hi(int lane_rank) { return lane_rank < H; }                 // ranks 0..23
  static constexpr bool theta_hi(int x) { return 24 + x < H; }                           // 24..28
  static constexpr bool theta_lo(int x) { return 29 + x < H; }                           // 29..33
  static constexpr bool rho_lo(int lane_rank) { return 34 + lane_rank < H; }            // 34..57
};

template <int H, int I>
__device__ __forceinline__ void rho_pi_mix(const uint64_t (&a)[25], const uint64_t (&c)[5], const uint64_t (&r1)[5],
                                           uint64_t (&b)[25]) {
  if constexpr (I < 25) {
    constexpr int rank = I - 1;  // lane 0 has rotation 0
    constexpr bool fh = I > 0 && Policy<H>::rho_hi(rank), fl = I > 0 && Policy<H>::rho_lo(rank);
    b[keccak::pi_of(I)] =
        rotl_mix<keccak::rho_of(I), fh, fl>(keccak::xor3(a[I], c[(I % 5 + 4) % 5], r1[(I % 5 + 1) % 5]));
    rho_pi_mix<H, I + 1>(a, c, r1, b);
  }
}
template <int H, int X>
__device__ __forceinline__ void theta_rot(const uint64_t (&c)[5], uint64_t (&r1)[5]) {
  if constexpr (X < 5) {
    r1[X] = rotl_mix<1, Policy<H>::theta_hi(X), Policy<H>::theta_lo(X)>(c[X]);
    theta_rot<H, X + 1>(c, r1);
  }
}

template <int H>
__device__ __forceinline__ void f1600_mix(uint64_t (&a)[25]) {
#pragma unroll 1
  for (int r = 0; r < 24; r++) {
    uint64_t c[5], r1[5], b[25];
#pragma unroll
    for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
    theta_rot<H, 0>(c, r1);
    rho_pi_mix<H, 0>(a, c, r1, b);
#pragma unroll
    for (int y = 0; y < 25; y += 5)
#pragma unroll
      for (int x = 0; x < 5; x++) a[y + x] = b[y + x] ^ (~b[y + (x + 1) % 5] & b[y + (x + 2) % 5]);
    a[0] ^= keccak::kRC.v[r];
  }
}

template <int H>
__global__ void __launch_bounds__(128) keccak_kernel(uint64_t* out, int perms, uint64_t seed) {
  uint64_t a[25];
#pragma unroll
  for (int i = 0; i < 25; i++) a[i] = seed * (i + 1) + blockIdx.x * blockDim.x + threadIdx.x;
  for (int p = 0; p < perms; p++) {
    if (H < 0)
      keccak::f1600(a);
    else
      f1600_mix<(H < 0 ? 0 : H)>(a);
  }
  uint64_t s = 0;
#pragma unroll
  for (int i = 0; i < 25; i++) s ^= a[i];
  out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// ---------------------------------------------------------------- butterflies
// int32 high-half Montgomery butterfly of kyber.cuh (3 IMAD + 2 SHF + 2 IADD)
__device__ __forceinline__ void bfly_int(int32_t& a, int32_t& b, int32_t z, int32_t zq) {
  int32_t c = b >> 16;
  int32_t p = c * z;
  int32_t m = (c * zq) >> 16;
  int32_t t = p - m * 3329;
  b = a - t;
  a = a + t;
}
// exact fp32: |b| < 2^12ish, |z| <= 1664 -> p exact; r = rint(p/q) by the magic-number trick; t = p - q r in [-1668, 1668]
__device__ __forceinline__ void bfly_f32(float& a, float& b, float z) {
  const float p = b * z;
  float r = fmaf(p, 1.0f / 3329.0f, 12582912.0f);
  r -= 12582912.0f;
  const float t = fmaf(r, -3329.0f, p);
  b = a - t;
  a = a + t;
}

template <int MODE>
__global__ void __launch_bounds__(128) bfly_kernel(float* out, int iters, float seedf, int seedi) {
  if (MODE == 0) {
    int32_t a[16];
#pragma unroll
    for (int i = 0; i < 16; i++) a[i] = (seedi + threadIdx.x * 16 + i) << 16;
    const int32_t z = seedi | 1, zq = (seedi * 62209) << 16;
#pragma unroll 1
    for (int it = 0; it < iters; it++) {
#pragma unroll
      for (int i = 0; i < 8; i++) bfly_int(a[i], a[i + 8], z + i, zq);
#pragma unroll
      for (int i = 0; i < 16; i += 2) bfly_int(a[i], a[i + 1], z, zq + i);
    }
    int32_t s = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) s ^= a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = (float)s;
  } else {
    float a[16];
#pragma unroll
    for (int i = 0; i < 16; i++) a[i] = seedf + threadIdx.x + i;
    const float z = seedf * 3.0f;
#pragma unroll 1
    for (int it = 0; it < iters; it++) {
#pragma unroll
      for (int i = 0; i < 8; i++) bfly_f32(a[i], a[i + 8], z + (float)i);
#pragma unroll
      for (int i = 0; i < 16; i += 2) bfly_f32(a[i], a[i + 1], z - (float)i);
    }
    float s = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  }
}

// co-residency: even warps permute, odd warps run butterflies (MODE 0 int, 1 fp32)
template <int H, int MODE>
__global__ void __launch_bounds__(128) mixed_kernel(uint64_t* out, int perms, int iters, uint64_t seed, float seedf) {
  const int warp = threadIdx.x >> 5;
  if (warp & 1) {
    if (MODE == 0) {
      int32_t a[16];
#pragma unroll
      for (int i = 0; i < 16; i++) a[i] = ((int)seed + threadIdx.x * 16 + i) << 16;
      const int32_t z = (int)seed | 1, zq = ((int)seed * 62209) << 16;
#pragma unroll 1
      for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 8; i++) bfly_int(a[i], a[i + 8], z + i, zq);
#pragma unroll
        for (int i = 0; i < 16; i += 2) bfly_int(a[i], a[i + 1], z, zq + i);
      }
      int32_t s = 0;
#pragma unroll
      for (int i = 0; i < 16; i++) s ^= a[i];
      out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = (uint64_t)s;
    } else {
      float a[16];
#pragma unroll
      for (int i = 0; i < 16; i++) a[i] = seedf + threadIdx.x + i;
      const float z = seedf * 3.0f;
#pragma unroll 1
      for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 8; i++) bfly_f32(a[i], a[i + 8], z + (float)i);
#pragma unroll
        for (int i = 0; i < 16; i += 2) bfly_f32(a[i], a[i + 1], z - (float)i);
      }
      float s = 0;
#pragma unroll
      for (int i = 0; i < 16; i++) s += a[i];
      out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = (uint64_t)s;
    }
  } else {
    uint64_t a[25];
#pragma unroll
    for (int i = 0; i < 25; i++) a[i] = seed * (i + 1) + blockIdx.x * blockDim.x + threadIdx.x;
    for (int p = 0; p < perms; p++) f1600_mix<H>(a);
    uint64_t s = 0;
#pragma unroll
    for (int i = 0; i < 25; i++) s ^= a[i];
    out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
  }
}

static float time_ms(void (*launch)(void)) {
  launch();
  cudaDeviceSynchronize();
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  float best = 1e30f;
  for (int rep = 0; rep < 3; rep++) {
    cudaEventRecord(a);
    launch();
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    best = ms < best ? ms : best;
  }
  return best;
}

static uint64_t* g_out;
static int g_ctas = 0;  // set in main
constexpr int kPerms = 512, kIters = 4096;

template <int H>
static void launch_keccak() { keccak_kernel<H><<<g_ctas, 128>>>(g_out, kPerms, 0x9E3779B97F4A7C15ull); }
template <int M>
static void launch_bfly() { bfly_kernel<M><<<g_ctas, 128>>>((float*)g_out, kIters, 1.25f, 12345); }
template <int H, int M>
static void launch_mixed() { mixed_kernel<H, M><<<g_ctas, 128>>>(g_out, kPerms, kIters, 0x9E3779B97F4A7C15ull, 1.25f); }

template <int H>
static void report_keccak(const char* tag) {
  for (int per_sm : {3, 4, 6}) {
    g_ctas = sms() * per_sm;
    const float ms = time_ms(launch_keccak<H>);
    const double perms = (double)g_ctas * 128 * kPerms;
    printf("keccak %-10s H=%3d  ctas/SM=%d  %.3f ms  %.3e keccak-f/s\n", tag, H, per_sm, ms, perms / (ms * 1e-3));
  }
}

// bit-exactness of the FMA-rotating permutation against the plain one
template <int H>
__global__ void check_kernel(int* bad) {
  uint64_t a[25], b[25];
  for (int i = 0; i < 25; i++) a[i] = b[i] = 0x0123456789abcdefull * (i + 3) + threadIdx.x;
  keccak::f1600(a);
  f1600_mix<H>(b);
  for (int i = 0; i < 25; i++)
    if (a[i] != b[i]) atomicAdd(bad, 1);
}
template <int H>
static void check() {
  int* d;
  cudaMalloc(&d, 4);
  cudaMemset(d, 0, 4);
  check_kernel<H><<<1, 64>>>(d);
  int h = -1;
  cudaMemcpy(&h, d, 4, cudaMemcpyDeviceToHost);
  printf("check H=%d mismatches=%d\n", H, h);
  cudaFree(d);
}

int main() {
  uint32_t p2[32];
  for (int i = 0; i < 32; i++) p2[i] = 1u << i;
  cudaMemcpyToSymbol(kPow2, p2, sizeof p2);
  cudaMalloc(&g_out, (size_t)sms() * 8 * 128 * 8);
  check<12>();
  check<29>();
  check<58>();
  report_keccak<-1>("repo");
  report_keccak<0>("mix");
  report_keccak<8>("mix");
  report_keccak<16>("mix");
  report_keccak<24>("mix");
  report_keccak<29>("mix");
  report_keccak<34>("mix");
  report_keccak<40>("mix");
  report_keccak<46>("mix");
  report_keccak<58>("mix");
  for (int per_sm : {4, 6, 8}) {
    g_ctas = sms() * per_sm;
    float ms = time_ms(launch_bfly<0>);
    double nb = (double)g_ctas * 128 * kIters * 16;
    printf("bfly int32  ctas/SM=%d %.3f ms  %.3e bfly/s\n", per_sm, ms, nb / (ms * 1e-3));
    ms = time_ms(launch_bfly<1>);
    printf("bfly fp32   ctas/SM=%d %.3f ms  %.3e bfly/s\n", per_sm, ms, nb / (ms * 1e-3));
  }
  for (int per_sm : {4, 6}) {
    g_ctas = sms() * per_sm;
    printf("mixed (half the warps each; perms=%d iters=%d) ctas/SM=%d: keccak H=0 + int %.3f ms, H=0 + fp32 %.3f ms, "
           "H=29 + fp32 %.3f ms, H=29 + int %.3f ms\n",
           kPerms, kIters, per_sm, time_ms(launch_mixed<0, 0>), time_ms(launch_mixed<0, 1>), time_ms(launch_mixed<29, 1>),
           time_ms(launch_mixed<29, 0>));
  }
  cudaError_t e = cudaGetLastError();
  printf("last error: %s\n", cudaGetErrorString(e));
  return 0;
}
