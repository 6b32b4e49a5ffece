// circl_b200/csrc/dilithium.cuh -- q = 8380417 ring arithmetic for sm_90a.
//
// Replaces (bit-exactly, *generic* semantics; the reference's AVX2 path equals generic here):
//   sign/internal/dilithium/field.go:5-32     ReduceLe2Q / le2qModQ / montReduceLe2Q
//   sign/internal/dilithium/ntt.go:111-184    nttGeneric      (asm: amd64.s:9    nttAVX2)
//   sign/internal/dilithium/ntt.go:191-217    invNttGeneric   (asm: amd64.s:2796 invNttAVX2)
//   sign/internal/dilithium/poly.go:10-100    mulHat / add / sub / reduce / normalize / exceeds
//
// Same "octet" decomposition as kyber.cuh: 8 lanes own one polynomial, 32 uint32
// coefficients per lane, two register-local passes of 4 layers each
//   S layout  r[2s+b] = coefficient 16s + 2v + b   -> l = 128, 64, 32, 16 (twiddles are immediates)
//   C layout  r[i]    = coefficient 32v + i        -> l = 8, 4, 2, 1      (per-lane twiddles)
// joined by one transposition through padded shared memory.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace cb200 {
namespace dil {

constexpr int N = 256;
constexpr uint32_t Q = 8380417u;
constexpr uint32_t QINV = 4236238847u;  // -(q^-1) mod 2^32, params.go
constexpr uint32_t ROVER256 = 41978u;   // (256)^-1 R^2 mod q

// ---------------------------------------------------------------- twiddles (regenerated, ntt.go:3-18)
__host__ __device__ constexpr uint32_t brv8(uint32_t x) {
  uint32_t r = 0;
  for (int i = 0; i < 8; i++) r |= ((x >> i) & 1u) << (7 - i);
  return r;
}
__host__ __device__ constexpr uint32_t powmod(uint32_t b, uint32_t e) {
  uint64_t r = 1, x = b;
  while (e) {
    if (e & 1) r = r * x % Q;
    x = x * x % Q;
    e >>= 1;
  }
  return (uint32_t)r;
}
__host__ __device__ constexpr uint32_t zeta_of(int i) {  // Zetas[i] = 1753^brv8(i) * 2^32 mod q
  return (uint32_t)((uint64_t)powmod(1753, brv8((uint32_t)i)) * ((1ull << 32) % Q) % Q);
}
__host__ __device__ constexpr uint32_t inv_zeta_of(int i) {  // InvZetas[i] = 1753^-(256 - brv8(255-i)) * 2^32 mod q
  return (uint32_t)((uint64_t)powmod(powmod(1753, Q - 2), 256 - brv8((uint32_t)(255 - i))) * ((1ull << 32) % Q) % Q);
}
template <int I>
struct Zeta {
  static constexpr uint32_t z = zeta_of(I);
  static constexpr uint32_t iz = inv_zeta_of(I);
};
// Shoup form of a Montgomery multiplication by a CONSTANT c (a twiddle or ROver256): with cp = c * 2^-32 mod q and
// ck = (cp * 2^32 - c) / q,
//     montReduceLe2Q(c * b) = cp * b - q * hi32(ck * b)        (mod 2^32; the value is below 2q)
// for every uint32 b: ck * q = -c (mod 2^32) makes ck * b the reference's m = c b (-q^-1) mod 2^32 (field.go:20-24), so
// (c b + m q) / 2^32 = cp b - q (ck b - m) / 2^32 = cp b - q floor(ck b / 2^32).  One wide multiplication and two
// 32-bit ones instead of two wide ones and a 32-bit one (IMAD.WIDE issues at half the rate of IMAD).
__host__ __device__ constexpr uint32_t shoup_p(uint32_t c) {  // c * 2^-32 mod q
  return (uint32_t)((uint64_t)c * powmod((uint32_t)((1ull << 32) % Q), Q - 2) % Q);
}
__host__ __device__ constexpr uint32_t shoup_k(uint32_t c) { return (uint32_t)((((uint64_t)shoup_p(c) << 32) - c) / Q); }
template <uint32_t C>
struct Shoup {
  static constexpr uint32_t p = shoup_p(C), k = shoup_k(C);
  static_assert(((uint64_t)p << 32) - C == (uint64_t)k * Q, "exact quotient");
};

template <int B, int E, class F>
__host__ __device__ __forceinline__ void static_for(F&& f) {
  if constexpr (B < E) {
    f(std::integral_constant<int, B>{});
    static_for<B + 1, E>(f);
  }
}

// ---------------------------------------------------------------- field ops
__device__ __forceinline__ uint32_t mont_le2q(uint64_t x) {  // field.go:20-24
  const uint32_t m = (uint32_t)x * QINV;
  return (uint32_t)((x + (uint64_t)m * Q) >> 32);
}
__device__ __forceinline__ uint32_t mont_mul(uint32_t a, uint32_t b) { return mont_le2q((uint64_t)a * b); }
// hi32(k * b).  Written as a wide multiplication on purpose (IMAD.WIDE.U32; scripts/ubench_pipes.cu measures its issue
// rate against IMAD.HI.U32): the compiler turns the plain C expression into the latter.
__host__ __device__ __forceinline__ uint32_t mulhi_wide(uint32_t k, uint32_t b) {
#ifdef __CUDA_ARCH__
  uint32_t hi;
  asm("{ .reg .b64 t; mul.wide.u32 t, %1, %2; mov.b64 {_, %0}, t; }" : "=r"(hi) : "r"(k), "r"(b));
  return hi;
#else
  return (uint32_t)(((uint64_t)k * b) >> 32);
#endif
}
__host__ __device__ __forceinline__ uint32_t mont_mul_shoup(uint32_t b, uint32_t p, uint32_t k) {
  return p * b - mulhi_wide(k, b) * Q;
}
template <uint32_t C>
__host__ __device__ __forceinline__ uint32_t mont_mul_const(uint32_t b) {  // == mont_mul(C, b), see Shoup above
  return mont_mul_shoup(b, Shoup<C>::p, Shoup<C>::k);
}
__device__ __forceinline__ uint32_t reduce_le2q(uint32_t x) {  // field.go:5-13
  const uint32_t x1 = x >> 23, x2 = x & 0x7FFFFF;
  return x2 + (x1 << 13) - x1;
}
__device__ __forceinline__ uint32_t le2q_modq(uint32_t x) {  // field.go:27-32
  x -= Q;
  return x + ((uint32_t)((int32_t)x >> 31) & Q);
}
__device__ __forceinline__ uint32_t modq(uint32_t x) { return le2q_modq(reduce_le2q(x)); }
// exceedsGeneric on one coefficient (poly.go:51-71)
__device__ __forceinline__ bool exceeds1(uint32_t c, uint32_t bound) {
  int32_t x = (int32_t)((Q - 1) / 2) - (int32_t)c;
  x ^= (x >> 31);
  x = (int32_t)((Q - 1) / 2) - x;
  return (uint32_t)x >= bound;
}

// ---------------------------------------------------------------- butterflies
// A run-time twiddle is its Shoup pair {p, k} (see struct Shoup).
__host__ __device__ __forceinline__ void ct_bfly(uint32_t& a, uint32_t& b, uint2 z) {  // ntt.go:177-180
  const uint32_t t = mont_mul_shoup(b, z.x, z.y);
  b = a + (2 * Q - t);
  a = a + t;
}
__host__ __device__ __forceinline__ void gs_bfly(uint32_t& a, uint32_t& b, uint2 z) {  // ntt.go:202-208
  uint32_t t = a;
  a = t + b;
  t += 256 * Q - b;
  b = mont_mul_shoup(t, z.x, z.y);
}
template <uint32_t Z>
__host__ __device__ __forceinline__ void ct_bfly_const(uint32_t& a, uint32_t& b) {  // ntt.go:177-180, immediate twiddle
  const uint32_t t = mont_mul_const<Z>(b);
  b = a + (2 * Q - t);
  a = a + t;
}
template <uint32_t Z>
__host__ __device__ __forceinline__ void gs_bfly_const(uint32_t& a, uint32_t& b) {  // ntt.go:202-208, immediate twiddle
  uint32_t t = a;
  a = t + b;
  t += 256 * Q - b;
  b = mont_mul_const<Z>(t);
}

// Twiddle table in global memory (dil_fill_twiddles): words [0, 256) Zetas, [256, 512) InvZetas, then 256 forward and 256
// inverse Shoup pairs {p, k}.
constexpr int kTwWords = 512 + 2 * 512, kTwFwdPairs = 512, kTwInvPairs = 1024;
// Per-lane twiddles of the C-layout pass as pairs: l = 8, 4, 2 in registers (28); the sixteen of l = 1, each used for one
// butterfly, are read through the read-only path where they are used.
struct LaneTw {
  uint2 l8[2], l4[4], l2[8];
  const uint2* l1;
};
// read-only load of a pair that stays where it is written (volatile asm: not hoisted out of the polynomial loop, which
// would turn the sixteen l = 1 pairs back into 32 live registers)
__device__ __forceinline__ uint2 ldg_pair_here(const uint2* p) {
  uint2 z;
  asm volatile("ld.global.nc.v2.u32 {%0, %1}, [%2];" : "=r"(z.x), "=r"(z.y) : "l"(p));
  return z;
}
// forward: Zetas[16+2v+i], [32+4v+i], [64+8v+i], [128+16v+i]
__device__ __forceinline__ void load_lane_tw_fwd(LaneTw& t, const uint32_t* __restrict__ tab, int v) {
  const uint2* z = reinterpret_cast<const uint2*>(tab + kTwFwdPairs);
#pragma unroll
  for (int i = 0; i < 2; i++) t.l8[i] = __ldg(z + 16 + 2 * v + i);
#pragma unroll
  for (int i = 0; i < 4; i++) t.l4[i] = __ldg(z + 32 + 4 * v + i);
#pragma unroll
  for (int i = 0; i < 8; i++) t.l2[i] = __ldg(z + 64 + 8 * v + i);
  t.l1 = z + 128 + 16 * v;
}
// inverse (k counts up, ntt.go:191-217): l=1: InvZetas[16v+i], l=2: [128+8v+i], l=4: [192+4v+i], l=8: [224+2v+i]
__device__ __forceinline__ void load_lane_tw_inv(LaneTw& t, const uint32_t* __restrict__ tab, int v) {
  const uint2* iz = reinterpret_cast<const uint2*>(tab + kTwInvPairs);
  t.l1 = iz + 16 * v;
#pragma unroll
  for (int i = 0; i < 8; i++) t.l2[i] = __ldg(iz + 128 + 8 * v + i);
#pragma unroll
  for (int i = 0; i < 4; i++) t.l4[i] = __ldg(iz + 192 + 4 * v + i);
#pragma unroll
  for (int i = 0; i < 2; i++) t.l8[i] = __ldg(iz + 224 + 2 * v + i);
}

// forward pass 1, S layout: l = 128 (k=1), 64 (k=2+h), 32 (k=4+h), 16 (k=8+h)
__host__ __device__ __forceinline__ void fwd_pass_S(uint32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 16; i++) ct_bfly_const<Zeta<1>::z>(r[i], r[i + 16]);
  static_for<0, 2>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 8; i++) ct_bfly_const<Zeta<2 + h>::z>(r[16 * h + i], r[16 * h + i + 8]);
  });
  static_for<0, 4>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 4; i++) ct_bfly_const<Zeta<4 + h>::z>(r[8 * h + i], r[8 * h + i + 4]);
  });
  static_for<0, 8>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 2; i++) ct_bfly_const<Zeta<8 + h>::z>(r[4 * h + i], r[4 * h + i + 2]);
  });
}
// forward pass 2, C layout: l = 8, 4, 2, 1
__device__ __forceinline__ void fwd_pass_C(uint32_t (&r)[32], const LaneTw& t) {
#pragma unroll
  for (int blk = 0; blk < 2; blk++)
#pragma unroll
    for (int j = 0; j < 8; j++) ct_bfly(r[16 * blk + j], r[16 * blk + j + 8], t.l8[blk]);
#pragma unroll
  for (int blk = 0; blk < 4; blk++)
#pragma unroll
    for (int j = 0; j < 4; j++) ct_bfly(r[8 * blk + j], r[8 * blk + j + 4], t.l4[blk]);
#pragma unroll
  for (int blk = 0; blk < 8; blk++)
#pragma unroll
    for (int j = 0; j < 2; j++) ct_bfly(r[4 * blk + j], r[4 * blk + j + 2], t.l2[blk]);
#pragma unroll
  for (int blk = 0; blk < 16; blk++) ct_bfly(r[2 * blk], r[2 * blk + 1], ldg_pair_here(t.l1 + blk));
}
// inverse pass A, C layout: l = 1, 2, 4, 8
__device__ __forceinline__ void inv_pass_C(uint32_t (&r)[32], const LaneTw& t) {
#pragma unroll
  for (int blk = 0; blk < 16; blk++) gs_bfly(r[2 * blk], r[2 * blk + 1], ldg_pair_here(t.l1 + blk));
#pragma unroll
  for (int blk = 0; blk < 8; blk++)
#pragma unroll
    for (int j = 0; j < 2; j++) gs_bfly(r[4 * blk + j], r[4 * blk + j + 2], t.l2[blk]);
#pragma unroll
  for (int blk = 0; blk < 4; blk++)
#pragma unroll
    for (int j = 0; j < 4; j++) gs_bfly(r[8 * blk + j], r[8 * blk + j + 4], t.l4[blk]);
#pragma unroll
  for (int blk = 0; blk < 2; blk++)
#pragma unroll
    for (int j = 0; j < 8; j++) gs_bfly(r[16 * blk + j], r[16 * blk + j + 8], t.l8[blk]);
}
// The C-layout passes with the twiddle pairs read from a shared-memory copy at the point of use (30 registers less
// than LaneTw).  The copy is lane-transposed: a pass reads "entry i of lane v" of a layer, which in table order sits at
// base + c v + i (c = 16, 8, 4, 2 entries per lane for l = 1, 2, 4, 8) -- eight lanes 2c words apart, i.e. on one or two
// banks; stage_pairs stores it at base + 8 i + v instead, so that the eight lanes of an octet read eight consecutive
// pairs (the four octets of a warp read the same ones: a broadcast).
__host__ __device__ __forceinline__ uint2 pair_at(const volatile uint2* tab, int i) {
  uint2 z;
  z.x = tab[i].x;
  z.y = tab[i].y;
  return z;
}
template <bool INV>
__host__ __device__ __forceinline__ int staged_index(int p) {  // table index of a pair -> its place in the staged copy
  int b, c;
  if (!INV) {
    if (p >= 128) b = 128, c = 16;
    else if (p >= 64) b = 64, c = 8;
    else if (p >= 32) b = 32, c = 4;
    else if (p >= 16) b = 16, c = 2;
    else return p;
  } else {
    if (p < 128) b = 0, c = 16;
    else if (p < 192) b = 128, c = 8;
    else if (p < 224) b = 192, c = 4;
    else if (p < 240) b = 224, c = 2;
    else return p;
  }
  const int v = (p - b) / c, i = (p - b) % c;
  return b + 8 * i + v;
}
// fills the 2 KB staged copy of the forward or inverse pairs (all threads of the CTA; the caller synchronises)
template <bool INV>
__device__ __forceinline__ void stage_pairs(volatile uint2* dst, const uint32_t* __restrict__ tab) {
  const uint2* src = reinterpret_cast<const uint2*>(tab + (INV ? kTwInvPairs : kTwFwdPairs));
  for (int q = threadIdx.x; q < 256; q += blockDim.x) {
    const uint2 z = __ldg(src + q);
    const int d = staged_index<INV>(q);
    dst[d].x = z.x;
    dst[d].y = z.y;
  }
}
__host__ __device__ __forceinline__ void fwd_pass_C_smem(uint32_t (&r)[32], const volatile uint2* zs, int v) {
#pragma unroll
  for (int blk = 0; blk < 2; blk++) {
    const uint2 z = pair_at(zs, 16 + 8 * blk + v);
#pragma unroll
    for (int j = 0; j < 8; j++) ct_bfly(r[16 * blk + j], r[16 * blk + j + 8], z);
  }
#pragma unroll
  for (int blk = 0; blk < 4; blk++) {
    const uint2 z = pair_at(zs, 32 + 8 * blk + v);
#pragma unroll
    for (int j = 0; j < 4; j++) ct_bfly(r[8 * blk + j], r[8 * blk + j + 4], z);
  }
#pragma unroll
  for (int blk = 0; blk < 8; blk++) {
    const uint2 z = pair_at(zs, 64 + 8 * blk + v);
#pragma unroll
    for (int j = 0; j < 2; j++) ct_bfly(r[4 * blk + j], r[4 * blk + j + 2], z);
  }
#pragma unroll
  for (int blk = 0; blk < 16; blk++) ct_bfly(r[2 * blk], r[2 * blk + 1], pair_at(zs, 128 + 8 * blk + v));
}
__host__ __device__ __forceinline__ void inv_pass_C_smem(uint32_t (&r)[32], const volatile uint2* iz, int v) {
#pragma unroll
  for (int blk = 0; blk < 16; blk++) gs_bfly(r[2 * blk], r[2 * blk + 1], pair_at(iz, 8 * blk + v));
#pragma unroll
  for (int blk = 0; blk < 8; blk++) {
    const uint2 z = pair_at(iz, 128 + 8 * blk + v);
#pragma unroll
    for (int j = 0; j < 2; j++) gs_bfly(r[4 * blk + j], r[4 * blk + j + 2], z);
  }
#pragma unroll
  for (int blk = 0; blk < 4; blk++) {
    const uint2 z = pair_at(iz, 192 + 8 * blk + v);
#pragma unroll
    for (int j = 0; j < 4; j++) gs_bfly(r[8 * blk + j], r[8 * blk + j + 4], z);
  }
#pragma unroll
  for (int blk = 0; blk < 2; blk++) {
    const uint2 z = pair_at(iz, 224 + 8 * blk + v);
#pragma unroll
    for (int j = 0; j < 8; j++) gs_bfly(r[16 * blk + j], r[16 * blk + j + 8], z);
  }
}
// fills a 2 KB shared-memory copy of the inverse pairs for inv_pass_C_smem
__device__ __forceinline__ void stage_inv_pairs(volatile uint2* dst, const uint32_t* __restrict__ tab) {
  stage_pairs<true>(dst, tab);
}

// inverse pass B, S layout: l = 16 (k=240+h), 32 (248+h), 64 (252+h), 128 (254), then * ROver256
__host__ __device__ __forceinline__ void inv_pass_S(uint32_t (&r)[32]) {
  static_for<0, 8>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 2; i++) gs_bfly_const<Zeta<240 + h>::iz>(r[4 * h + i], r[4 * h + i + 2]);
  });
  static_for<0, 4>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 4; i++) gs_bfly_const<Zeta<248 + h>::iz>(r[8 * h + i], r[8 * h + i + 4]);
  });
  static_for<0, 2>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 8; i++) gs_bfly_const<Zeta<252 + h>::iz>(r[16 * h + i], r[16 * h + i + 8]);
  });
#pragma unroll
  for (int i = 0; i < 16; i++) gs_bfly_const<Zeta<254>::iz>(r[i], r[i + 16]);
#pragma unroll
  for (int i = 0; i < 32; i++) r[i] = mont_mul_const<ROVER256>(r[i]);
}

// ---------------------------------------------------------------- shared-memory tile (S <-> C)
// 256 words + 4 pad words after every 32; octet stride 304 words (== 16 mod 32).
constexpr int kPolyWords = 304;
__host__ __device__ __forceinline__ void store_S(uint32_t* tile, int v, const uint32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++)
    *reinterpret_cast<uint2*>(tile + 16 * s + 2 * v + 4 * (s >> 1)) = make_uint2(r[2 * s], r[2 * s + 1]);
}
__host__ __device__ __forceinline__ void load_S(const uint32_t* tile, int v, uint32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++) {
    const uint2 w = *reinterpret_cast<const uint2*>(tile + 16 * s + 2 * v + 4 * (s >> 1));
    r[2 * s] = w.x;
    r[2 * s + 1] = w.y;
  }
}
__host__ __device__ __forceinline__ void store_C(uint32_t* tile, int v, const uint32_t (&r)[32]) {
  uint4* p = reinterpret_cast<uint4*>(tile + 36 * v);
#pragma unroll
  for (int c = 0; c < 8; c++) p[c] = make_uint4(r[4 * c], r[4 * c + 1], r[4 * c + 2], r[4 * c + 3]);
}
__host__ __device__ __forceinline__ void load_C(const uint32_t* tile, int v, uint32_t (&r)[32]) {
  const uint4* p = reinterpret_cast<const uint4*>(tile + 36 * v);
#pragma unroll
  for (int c = 0; c < 8; c++) {
    const uint4 w = p[c];
    r[4 * c] = w.x;
    r[4 * c + 1] = w.y;
    r[4 * c + 2] = w.z;
    r[4 * c + 3] = w.w;
  }
}

// ---------------------------------------------------------------- global <-> registers
__device__ __forceinline__ void gload_S(const uint32_t* __restrict__ poly, int v, uint32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++) {
    const uint2 w = *reinterpret_cast<const uint2*>(poly + 16 * s + 2 * v);
    r[2 * s] = w.x;
    r[2 * s + 1] = w.y;
  }
}
__device__ __forceinline__ void gstore_S(uint32_t* __restrict__ poly, int v, const uint32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++) *reinterpret_cast<uint2*>(poly + 16 * s + 2 * v) = make_uint2(r[2 * s], r[2 * s + 1]);
}
__device__ __forceinline__ void gload_C(const uint32_t* __restrict__ poly, int v, uint32_t (&r)[32]) {
  const uint4* p = reinterpret_cast<const uint4*>(poly + 32 * v);
#pragma unroll
  for (int c = 0; c < 8; c++) {
    const uint4 w = p[c];
    r[4 * c] = w.x;
    r[4 * c + 1] = w.y;
    r[4 * c + 2] = w.z;
    r[4 * c + 3] = w.w;
  }
}
__device__ __forceinline__ void gstore_C(uint32_t* __restrict__ poly, int v, const uint32_t (&r)[32]) {
  uint4* p = reinterpret_cast<uint4*>(poly + 32 * v);
#pragma unroll
  for (int c = 0; c < 8; c++) p[c] = make_uint4(r[4 * c], r[4 * c + 1], r[4 * c + 2], r[4 * c + 3]);
}

// C-layout registers -> global memory in the interleaved order of gload_I through the octet's (free) tile: an octet
// writes 128 contiguous bytes per instruction instead of eight 16-byte pieces 128 bytes apart.  Every lane of the warp
// calls it; only active octets store.
__device__ __forceinline__ void gstore_C_via_tile(uint32_t* __restrict__ poly, uint32_t* tile, int v,
                                                  const uint32_t (&r)[32], bool active) {
  store_C(tile, v, r);
  __syncwarp();
  uint4 w[8];
#pragma unroll
  for (int c = 0; c < 8; c++) w[c] = *reinterpret_cast<const uint4*>(tile + 36 * c + 4 * v);
  __syncwarp();
  if (active) {
    uint4* dst = reinterpret_cast<uint4*>(poly) + v;
#pragma unroll
    for (int c = 0; c < 8; c++) dst[8 * c] = w[c];
  }
}

// Whole transforms on an octet.  fwd: in S layout -> out C layout; inv: in C layout -> out S layout.
__device__ __forceinline__ void ntt_octet(uint32_t (&r)[32], uint32_t* tile, int v, const LaneTw& t) {
  fwd_pass_S(r);
  store_S(tile, v, r);
  __syncwarp();
  load_C(tile, v, r);
  __syncwarp();
  fwd_pass_C(r, t);
}
__device__ __forceinline__ void invntt_octet(uint32_t (&r)[32], uint32_t* tile, int v, const LaneTw& t) {
  inv_pass_C(r, t);
  store_C(tile, v, r);
  __syncwarp();
  load_S(tile, v, r);
  __syncwarp();
  inv_pass_S(r);
}
__device__ __forceinline__ void ntt_octet_smem(uint32_t (&r)[32], uint32_t* tile, int v, const volatile uint2* zs) {
  fwd_pass_S(r);
  store_S(tile, v, r);
  __syncwarp();
  load_C(tile, v, r);
  __syncwarp();
  fwd_pass_C_smem(r, zs, v);
}
__device__ __forceinline__ void invntt_octet_smem(uint32_t (&r)[32], uint32_t* tile, int v, const volatile uint2* iz) {
  inv_pass_C_smem(r, iz, v);
  store_C(tile, v, r);
  __syncwarp();
  load_S(tile, v, r);
  __syncwarp();
  inv_pass_S(r);
}
// "I" (interleaved) layout for coefficient-wise work straight from global memory:
//   r[4c+e] = coefficient 32c + 4v + e, i.e. per instruction an octet reads 8 x 16 = 128 contiguous bytes.
// Pointwise products do not care about the layout as long as both operands share it; i_to_c brings the
// result into the C layout the inverse transform starts from.
__device__ __forceinline__ void gload_I(const uint32_t* __restrict__ poly, int v, uint4 (&w)[8]) {
  const uint4* p = reinterpret_cast<const uint4*>(poly) + v;
#pragma unroll
  for (int c = 0; c < 8; c++) w[c] = p[8 * c];
}
__device__ __forceinline__ void gload_I_ro(const uint32_t* __restrict__ poly, int v, uint4 (&w)[8]) {
  const uint4* p = reinterpret_cast<const uint4*>(poly) + v;
#pragma unroll
  for (int c = 0; c < 8; c++) w[c] = __ldg(p + 8 * c);
}
__device__ __forceinline__ void i_to_c(uint32_t (&r)[32], uint32_t* tile, int v) {
#pragma unroll
  for (int c = 0; c < 8; c++)
    *reinterpret_cast<uint4*>(tile + 36 * c + 4 * v) = make_uint4(r[4 * c], r[4 * c + 1], r[4 * c + 2], r[4 * c + 3]);
  __syncwarp();
  load_C(tile, v, r);
  __syncwarp();
}
// layout changes without arithmetic
__device__ __forceinline__ void s_to_c(uint32_t (&r)[32], uint32_t* tile, int v) {
  store_S(tile, v, r);
  __syncwarp();
  load_C(tile, v, r);
  __syncwarp();
}
__device__ __forceinline__ void c_to_s(uint32_t (&r)[32], uint32_t* tile, int v) {
  store_C(tile, v, r);
  __syncwarp();
  load_S(tile, v, r);
  __syncwarp();
}

}  // namespace dil
}  // namespace cb200
