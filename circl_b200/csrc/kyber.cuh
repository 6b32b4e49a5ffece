// circl_b200/csrc/kyber.cuh -- q = 3329 ring arithmetic for sm_90a.
//
// Replaces (bit-exactly, standard coefficient order, *generic* semantics):
//   pke/kyber/internal/common/field.go:4-74       montReduce / barrettReduce / csubq / toMont
//   pke/kyber/internal/common/ntt.go:60-135       nttGeneric        (asm: amd64.s:153  nttAVX2)
//   pke/kyber/internal/common/ntt.go:145-193      invNTTGeneric     (asm: amd64.s:737  invNttAVX2)
//   pke/kyber/internal/common/poly.go:63-100      mulHatGeneric     (asm: amd64.s:1443 mulHatAVX2)
//
// Work decomposition ("octet"): 8 lanes own one 256-coefficient polynomial, so a
// warp carries 4 polynomials.  Each lane keeps 32 coefficients in registers in
// one of two layouts:
//   S ("strided")     r[2s+b] = coefficient 16s + 2v + b   (s = 0..15, b = 0,1)
//                     -> layers l = 128,64,32,16 are register-local, twiddles are immediates
//   C ("contiguous")  r[i]    = coefficient 32v + i        (i = 0..31)
//                     -> layers l = 8,4,2 are register-local, twiddles are per-lane registers
// One transposition S<->C through (padded, conflict-free) shared memory joins
// the two passes; there is no cross-lane butterfly and no shuffle.
//
// Register format ("high-half"): a coefficient c lives in bits 31..16 of a
// 32-bit register; bits 15..0 are zero.  int16 wrap-around of the reference is
// then exactly the wrap-around of 32-bit adds, and
//   montReduce(zeta*c) << 16  ==  c*zeta - m*q   with  m = int16(c*zeta*q^-1)
// needs no final shift.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace cb200 {
namespace kyber {

constexpr int N = 256;
constexpr int Q = 3329;
constexpr uint32_t QINV = 62209;  // q^-1 mod 2^16, field.go:12

// ---------------------------------------------------------------- twiddles
// Zetas[i] = 17^brv7(i) * 2^16 mod q (ntt.go:5-15), regenerated at compile time.
__host__ __device__ constexpr uint32_t brv7(uint32_t x) {
  uint32_t r = 0;
  for (int i = 0; i < 7; i++) r |= ((x >> i) & 1u) << (6 - i);
  return r;
}
__host__ __device__ constexpr int32_t zeta_of(int i) {
  uint32_t z = 65536u % Q, e = brv7((uint32_t)i);
  for (uint32_t j = 0; j < e; j++) z = z * 17u % Q;
  return (int32_t)z;
}
// (zeta * q^-1 mod 2^16) << 16 : multiplying the sign-extended coefficient by this
// yields m << 16 directly.
__host__ __device__ constexpr int32_t zetaq_of(int i) {
  return (int32_t)((((uint32_t)zeta_of(i) * QINV) & 0xffffu) << 16);
}
// compile-time loop: f(std::integral_constant<int, I>) for I in [B, E)
template <int B, int E, class F>
__host__ __device__ __forceinline__ void static_for(F&& f) {
  if constexpr (B < E) {
    f(std::integral_constant<int, B>{});
    static_for<B + 1, E>(f);
  }
}

template <int I>
struct Zeta {
  static constexpr int32_t z = zeta_of(I);
  static constexpr int32_t zq = zetaq_of(I);
};

// Per-lane twiddles of the C-layout pass (index = Zetas position k), packed as
// {zeta, zetaq} pairs in global memory by the host at init.
struct TwPair {
  int32_t z, zq;
};

// ---------------------------------------------------------------- field ops
// c: sign-extended coefficient;  returns montReduce(z*c) << 16  (low half zero)
__device__ __forceinline__ int32_t mont_mul_hi(int32_t c, int32_t z, int32_t zq) {
  int32_t p = c * z;
  int32_t m = (c * zq) >> 16;  // == int16(c*z*62209), field.go:12
  return p - m * Q;            // == montReduce(p) << 16, field.go:31
}
// general product of two sign-extended values: montReduce(a*b) << 16
__device__ __forceinline__ int32_t mont_prod_hi(int32_t a, int32_t b) {
  int32_t p = a * b;
  int32_t m = (int32_t)((uint32_t)p * (QINV << 16)) >> 16;
  return p - m * Q;
}
// barrettReduce on a high-half register (field.go:45-64)
__device__ __forceinline__ int32_t barrett_hi(int32_t x) {
  int32_t c = x >> 16;
  int32_t t = (c * 20159) >> 26;
  return x - t * (Q << 16);
}
// csubq on a high-half register (field.go:67-74)
__device__ __forceinline__ int32_t csubq_hi(int32_t x) {
  x -= (Q << 16);
  x += (x >> 31) & (Q << 16);
  return x;
}

// ---------------------------------------------------------------- pack / unpack
// word = two consecutive int16 coefficients (little endian)
__device__ __forceinline__ void unpack2(uint32_t w, int32_t& lo, int32_t& hi) {
  lo = (int32_t)(w << 16);
  hi = (int32_t)(w & 0xffff0000u);
}
// The same for values that only go through Cooley-Tukey butterflies, Barrett steps and pack2: there the low half of a
// register is never read (b >> 16), and a +- t with a clean t neither carries into nor borrows from the high half,
// so the upper coefficient may keep the lower one as garbage in its low half -- one LOP3 less per word.
__device__ __forceinline__ void unpack2_ct(uint32_t w, int32_t& lo, int32_t& hi) {
  lo = (int32_t)(w << 16);
  hi = (int32_t)w;
}
__device__ __forceinline__ uint32_t pack2(int32_t lo, int32_t hi) {
  return __byte_perm((uint32_t)lo, (uint32_t)hi, 0x7632);
}

// ---------------------------------------------------------------- shared-memory tile
// One polynomial = 128 words, stored with 4 pad words after every 32 so that
// both access patterns below are bank-conflict free; octet stride 152 words
// (== 24 mod 32) separates the four octets of a warp.
constexpr int kPolyWords = 152;

// ---------------------------------------------------------------- butterflies
// Cooley-Tukey, ntt.go:129-131
__device__ __forceinline__ void ct_bfly(int32_t& a, int32_t& b, int32_t z, int32_t zq) {
  int32_t t = mont_mul_hi(b >> 16, z, zq);
  b = a - t;
  a = a + t;
}
// Gentleman-Sande, ntt.go:165-168
__device__ __forceinline__ void gs_bfly(int32_t& a, int32_t& b, int32_t z, int32_t zq) {
  int32_t t = b - a;
  a = a + b;
  b = mont_mul_hi(t >> 16, z, zq);
}

// Forward pass 1 on S layout: layers l = 128, 64, 32, 16.  All twiddles are
// template constants, i.e. IMAD immediates in SASS.
__device__ __forceinline__ void fwd_pass_S(int32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 16; i++) ct_bfly(r[i], r[i + 16], Zeta<1>::z, Zeta<1>::zq);  // l=128, k=1
  static_for<0, 2>([&](auto hc) {  // l=64, k = 2 + (s>>3)
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 8; i++) ct_bfly(r[16 * h + i], r[16 * h + i + 8], Zeta<2 + h>::z, Zeta<2 + h>::zq);
  });
  static_for<0, 4>([&](auto hc) {  // l=32, k = 4 + (s>>2)
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 4; i++) ct_bfly(r[8 * h + i], r[8 * h + i + 4], Zeta<4 + h>::z, Zeta<4 + h>::zq);
  });
  static_for<0, 8>([&](auto hc) {  // l=16, k = 8 + (s>>1)
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 2; i++) ct_bfly(r[4 * h + i], r[4 * h + i + 2], Zeta<8 + h>::z, Zeta<8 + h>::zq);
  });
}

// Per-lane twiddle registers for the C-layout passes: lane v needs Zetas[16+2v+{0,1}],
// Zetas[32+4v+{0..3}], Zetas[64+8v+{0..7}]  (forward) -- and the same entries,
// walked downwards, for the inverse (ntt.go:152-160).
struct LaneTw {
  TwPair l8[2], l4[4], l2[8];
};
__device__ __forceinline__ void load_lane_tw(LaneTw& t, const TwPair* __restrict__ tab, int v) {
#pragma unroll
  for (int i = 0; i < 2; i++) t.l8[i] = tab[16 + 2 * v + i];
#pragma unroll
  for (int i = 0; i < 4; i++) t.l4[i] = tab[32 + 4 * v + i];
#pragma unroll
  for (int i = 0; i < 8; i++) t.l2[i] = tab[64 + 8 * v + i];
}

// Forward pass 2 on C layout (layers l = 8, 4, 2) with the twiddles read from a shared-memory copy of the table at the
// point of use (28 registers less than holding them).  `tab` must be volatile-qualified by the caller's cast so the
// loads stay inside the polynomial loop.
__device__ __forceinline__ TwPair tw_at(const volatile TwPair* tab, int k) {
  const volatile int2* p = reinterpret_cast<const volatile int2*>(tab + k);
  TwPair t;
  t.z = p->x;
  t.zq = p->y;
  return t;
}
__device__ __forceinline__ void fwd_pass_C_smem(int32_t (&r)[32], const volatile TwPair* tab, int v) {
#pragma unroll
  for (int blk = 0; blk < 2; blk++) {
    const TwPair t = tw_at(tab, 16 + 2 * v + blk);
#pragma unroll
    for (int j = 0; j < 8; j++) ct_bfly(r[16 * blk + j], r[16 * blk + j + 8], t.z, t.zq);
  }
#pragma unroll
  for (int blk = 0; blk < 4; blk++) {
    const TwPair t = tw_at(tab, 32 + 4 * v + blk);
#pragma unroll
    for (int j = 0; j < 4; j++) ct_bfly(r[8 * blk + j], r[8 * blk + j + 4], t.z, t.zq);
  }
#pragma unroll
  for (int blk = 0; blk < 8; blk++) {
    const TwPair t = tw_at(tab, 64 + 8 * v + blk);
#pragma unroll
    for (int j = 0; j < 2; j++) ct_bfly(r[4 * blk + j], r[4 * blk + j + 2], t.z, t.zq);
  }
}
__device__ __forceinline__ void inv_pass_C_smem(int32_t (&r)[32], const volatile TwPair* tab, int v) {
#pragma unroll
  for (int blk = 0; blk < 8; blk++) {
    const TwPair t = tw_at(tab, 127 - 8 * v - blk);
#pragma unroll
    for (int j = 0; j < 2; j++) gs_bfly(r[4 * blk + j], r[4 * blk + j + 2], t.z, t.zq);
  }
#pragma unroll
  for (int blk = 0; blk < 4; blk++) {
    const TwPair t = tw_at(tab, 63 - 4 * v - blk);
#pragma unroll
    for (int j = 0; j < 4; j++) gs_bfly(r[8 * blk + j], r[8 * blk + j + 4], t.z, t.zq);
  }
#pragma unroll
  for (int blk = 0; blk < 2; blk++) {
    const TwPair t = tw_at(tab, 31 - 2 * v - blk);
#pragma unroll
    for (int j = 0; j < 8; j++) gs_bfly(r[16 * blk + j], r[16 * blk + j + 8], t.z, t.zq);
  }
  r[16] = barrett_hi(r[16]);
  r[17] = barrett_hi(r[17]);
}

// Inverse pass B on S layout: layers l = 16, 32, 64, 128 with the lazy Barrett
// schedule of ntt.go:44-49 and the final multiplication by 1441 (ntt.go:187-192).
// S layout: r[2s+b] = coefficient 16s + 2v + b.
// SCALE = false leaves the last step out (for callers that folded the constant into an operand): the outputs are
// then the int16-range values the reference holds right before it (|x| < 2^15), to be Barrett-reduced by the caller.
template <bool SCALE = true>
__device__ __forceinline__ void inv_pass_S(int32_t (&r)[32], int v) {
  static_for<0, 8>([&](auto hc) {  // l=16: pairs (s, s+1), k = 15 - (s>>1)
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 2; i++) gs_bfly(r[4 * h + i], r[4 * h + i + 2], Zeta<15 - h>::z, Zeta<15 - h>::zq);
  });
  // after layer 4: idx mod 64 in {0,1} -> (s&3)==0, v==0 ; {32..35} -> (s&3)==2, v<=1
#pragma unroll
  for (int s = 0; s < 16; s += 4)
#pragma unroll
    for (int b = 0; b < 2; b++) {
      if (v == 0) r[2 * s + b] = barrett_hi(r[2 * s + b]);
      if (v <= 1) r[2 * (s + 2) + b] = barrett_hi(r[2 * (s + 2) + b]);
    }
  static_for<0, 4>([&](auto hc) {  // l=32: pairs (s, s+2), k = 7 - (s>>2)
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 4; i++) gs_bfly(r[8 * h + i], r[8 * h + i + 4], Zeta<7 - h>::z, Zeta<7 - h>::zq);
  });
  // after layer 5: idx mod 128 in {2,3} -> (s&7)==0, v==1 ; {66..71} -> (s&7)==4, v in 1..3
#pragma unroll
  for (int s = 0; s < 16; s += 8)
#pragma unroll
    for (int b = 0; b < 2; b++) {
      if (v == 1) r[2 * s + b] = barrett_hi(r[2 * s + b]);
      if (v >= 1 && v <= 3) r[2 * (s + 4) + b] = barrett_hi(r[2 * (s + 4) + b]);
    }
  static_for<0, 2>([&](auto hc) {  // l=64: pairs (s, s+4), k = 3 - (s>>3)
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 8; i++) gs_bfly(r[16 * h + i], r[16 * h + i + 8], Zeta<3 - h>::z, Zeta<3 - h>::zq);
  });
  // after layer 6: idx in {4..7} -> s==0, v in {2,3} ; {132..143} -> s==8, v in 2..7
#pragma unroll
  for (int b = 0; b < 2; b++) {
    if (v == 2 || v == 3) r[b] = barrett_hi(r[b]);
    if (v >= 2) r[16 + b] = barrett_hi(r[16 + b]);
  }
#pragma unroll
  for (int i = 0; i < 16; i++) gs_bfly(r[i], r[i + 16], Zeta<1>::z, Zeta<1>::zq);  // l=128, k=1
  // p[j] = montReduce(1441 * p[j])
  if constexpr (SCALE) {
#pragma unroll
    for (int i = 0; i < 32; i++) r[i] = mont_mul_hi(r[i] >> 16, 1441, (int32_t)(((1441u * QINV) & 0xffffu) << 16));
  }
}

// ---------------------------------------------------------------- S <-> C transposition
// `tile` points at this octet's kPolyWords-word shared-memory tile.
__device__ __forceinline__ void store_S(uint32_t* tile, int v, const int32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++) tile[8 * s + v + 4 * (s >> 2)] = pack2(r[2 * s], r[2 * s + 1]);
}
__device__ __forceinline__ void load_S(const uint32_t* tile, int v, int32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++) unpack2(tile[8 * s + v + 4 * (s >> 2)], r[2 * s], r[2 * s + 1]);
}
__device__ __forceinline__ void store_C(uint32_t* tile, int v, const int32_t (&r)[32]) {
  uint4* p = reinterpret_cast<uint4*>(tile + 16 * v + 4 * (v >> 1));
#pragma unroll
  for (int c = 0; c < 4; c++)
    p[c] = make_uint4(pack2(r[8 * c], r[8 * c + 1]), pack2(r[8 * c + 2], r[8 * c + 3]), pack2(r[8 * c + 4], r[8 * c + 5]),
                      pack2(r[8 * c + 6], r[8 * c + 7]));
}
// load_C for the forward transform (see unpack2_ct)
__device__ __forceinline__ void load_C_ct(const uint32_t* tile, int v, int32_t (&r)[32]) {
  const uint4* p = reinterpret_cast<const uint4*>(tile + 16 * v + 4 * (v >> 1));
#pragma unroll
  for (int c = 0; c < 4; c++) {
    uint4 w = p[c];
    unpack2_ct(w.x, r[8 * c], r[8 * c + 1]);
    unpack2_ct(w.y, r[8 * c + 2], r[8 * c + 3]);
    unpack2_ct(w.z, r[8 * c + 4], r[8 * c + 5]);
    unpack2_ct(w.w, r[8 * c + 6], r[8 * c + 7]);
  }
}

// ---------------------------------------------------------------- global <-> registers
// S layout: 16 x 32-bit per lane, each octet moves one full 32-byte sector per instruction
__device__ __forceinline__ void gstore_S(uint32_t* __restrict__ poly, int v, const int32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++) poly[8 * s + v] = pack2(r[2 * s], r[2 * s + 1]);
}
// C layout: 4 x 128-bit per lane, 64 contiguous bytes per lane
__device__ __forceinline__ void gload_C(const uint32_t* __restrict__ poly, int v, int32_t (&r)[32]) {
  uint4 w[4];
#pragma unroll
  for (int c = 0; c < 4; c++) w[c] = ldg_stream128(poly + 16 * v + 4 * c);
#pragma unroll
  for (int c = 0; c < 4; c++) {
    unpack2(w[c].x, r[8 * c], r[8 * c + 1]);
    unpack2(w[c].y, r[8 * c + 2], r[8 * c + 3]);
    unpack2(w[c].z, r[8 * c + 4], r[8 * c + 5]);
    unpack2(w[c].w, r[8 * c + 6], r[8 * c + 7]);
  }
}
__device__ __forceinline__ void gstore_C(uint32_t* __restrict__ poly, int v, const int32_t (&r)[32]) {
#pragma unroll
  for (int c = 0; c < 4; c++)
    stg_stream128(poly + 16 * v + 4 * c,
                  make_uint4(pack2(r[8 * c], r[8 * c + 1]), pack2(r[8 * c + 2], r[8 * c + 3]),
                             pack2(r[8 * c + 4], r[8 * c + 5]), pack2(r[8 * c + 6], r[8 * c + 7])));
}

// ---------------------------------------------------------------- "low" format fast path
// A second register format for inputs inside the reference's contract.  A coefficient is a plain sign-extended
// int32 ("low" format) and montReduce(zeta*b) (field.go:4-32) is evaluated in its Shoup form
//     t = zp*b - q*n,   n = (kk*b + 32767) >> 16,
// where zp = zeta * 2^-16 mod q (centred) and kk = (zp*2^16 - zeta) / q.  This is the same integer as the reference's
// (zeta*b - m*q) / 2^16 with m = int16(zeta*b*q^-1) for EVERY int16 b: kk*q = -zeta (mod 2^16) gives kk*b = -m
// (mod 2^16), hence kk*b + m = 2^16 n with n = floor((kk*b + 32767) / 2^16) because -32768 <= m <= 32767.
// It costs 3 IMAD + 1 SHF instead of 3 IMAD + 2 SHF (no b >> 16: the operand already is sign-extended), i.e. a
// 6-instruction butterfly -- but 32-bit adds no longer wrap where the reference's int16 adds would.  The kernels
// therefore take this path only for polynomials whose coefficients are small enough that no intermediate value of
// the reference can leave int16 (interval analysis of ntt.go:60-193 with |montReduce(zeta*b)| <= |b|*3328/2^16 +
// 1665: |c| <= 13561 forward, |c| <= 3679 inverse; the reference's own contract is |c| <= q), checked on the packed
// input words with one VIADDMNMX.U16x2 each; any other input runs through the high-half code above.  Both paths
// return the reference's representatives bit for bit.
constexpr int kFwdBound = 13561, kInvBound = 3679;

__host__ __device__ constexpr int32_t zp_of(int i) {  // 17^brv7(i) mod q, centred
  uint32_t z = 1, e = brv7((uint32_t)i);
  for (uint32_t j = 0; j < e; j++) z = z * 17u % Q;
  return (int32_t)z > Q / 2 ? (int32_t)z - Q : (int32_t)z;
}
__host__ __device__ constexpr int32_t kk_of(int i) { return (zp_of(i) * 65536 - zeta_of(i)) / Q; }
template <int I>
struct ZetaL {
  static constexpr int32_t zp = zp_of(I);
  static constexpr int32_t kk = kk_of(I);
  static_assert(zp_of(I) * 65536 - zeta_of(I) == kk_of(I) * Q, "kk is an exact quotient");
};
// montReduce(1441 * x) (ntt.go:187-192): 1441 = 2^32/128 mod q, so zp = 2^16/128 = 512
constexpr int32_t kScaleZp = 512, kScaleKk = (512 * 65536 - 1441) / Q;
static_assert(512 * 65536 - 1441 == kScaleKk * Q, "scale constant");
struct TwLow {
  int32_t zp, kk;
};

__host__ __device__ __forceinline__ int32_t mont_mul_lo(int32_t b, int32_t zp, int32_t kk) {
  const int32_t n = (kk * b + 32767) >> 16;
  return zp * b - n * Q;
}
__host__ __device__ __forceinline__ int32_t barrett_lo(int32_t x) { return x - ((x * 20159) >> 26) * Q; }  // field.go:45-64
// Cooley-Tukey butterfly (ntt.go:129-131) in five instructions: a + t = (zp*b + a) - q*n is two multiply-adds, and
// a - t = 2a - (a + t) one three-input add
__host__ __device__ __forceinline__ void ct_lo(int32_t& a, int32_t& b, int32_t zp, int32_t kk) {
  const int32_t n = (kk * b + 32767) >> 16;
  const int32_t ap = (zp * b + a) - n * Q;
  b = 2 * a - ap;
  a = ap;
}
__host__ __device__ __forceinline__ void gs_lo(int32_t& a, int32_t& b, int32_t zp, int32_t kk) {
  const int32_t t = b - a;
  a = a + b;
  b = mont_mul_lo(t, zp, kk);
}
__host__ __device__ __forceinline__ void unpack2_lo(uint32_t w, int32_t& lo, int32_t& hi) {
  lo = (int32_t)(int16_t)(w & 0xffffu);
  hi = (int32_t)w >> 16;
}
__host__ __device__ __forceinline__ uint32_t pack2_lo(int32_t lo, int32_t hi) {
#ifdef __CUDA_ARCH__
  return __byte_perm((uint32_t)lo, (uint32_t)hi, 0x5410);
#else
  return ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16);
#endif
}
// max over both halves of all 16 words of (coefficient + bound) as unsigned 16-bit numbers: <= 2*bound iff every
// coefficient is in [-bound, bound]
__host__ __device__ __forceinline__ bool words_in_range(const uint32_t (&w)[16], uint32_t bound) {
#ifdef __CUDA_ARCH__
  uint32_t acc = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) acc = __viaddmax_u16x2(w[i], bound * 0x10001u, acc);
  return __vmaxu2(acc, 2 * bound * 0x10001u) == 2 * bound * 0x10001u;
#else  // the same predicate spelled out (host-side check of the fast path, tests/cpp/test_kyber_low.cu)
  uint32_t mx = 0;
  for (int i = 0; i < 16; i++)
    for (int h = 0; h < 2; h++) {
      const uint32_t u = ((w[i] >> (16 * h)) + bound) & 0xffffu;
      mx = u > mx ? u : mx;
    }
  return mx <= 2 * bound;
#endif
}

// ---------------------------------------------------------------- noise on the S layout
// prmt.b32 with the full selector: bit 3 of a nibble replicates the sign of the selected byte (__byte_perm masks it off)
__host__ __device__ __forceinline__ uint32_t prmt_sx(uint32_t a, uint32_t b, uint32_t sel) {
#ifdef __CUDA_ARCH__
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
#else
  const uint64_t x = ((uint64_t)b << 32) | a;
  uint32_t d = 0;
  for (int i = 0; i < 4; i++) {
    const uint32_t s = (sel >> (4 * i)) & 0xf, byte = (uint32_t)(x >> (8 * (s & 7))) & 0xff;
    d |= ((s & 8) ? ((byte & 0x80) ? 0xffu : 0u) : byte) << (8 * i);
  }
  return d;
#endif
}
// CBD_2 (sample.go:80-93) of four PRF bytes: w[q] = the pair (coefficient of the low nibble, of the high nibble) of byte
// q of t, packed as two int16.  d = (t & 0x55..) + ((t >> 1) & 0x55..) holds, per nibble j, a_j in its low and b_j in its
// high two bits, and coefficient j = a_j - b_j.  Bytewise: even coefficients sit in the low nibbles of the four bytes, odd
// ones in the high nibbles; (0x80 | a) - b never borrows across bytes and ^ 0x80 turns it into the signed byte a - b; one
// PRMT per output word then widens a byte pair to two int16 (selector bit 3 replicates the sign).  19 instructions per
// eight coefficients instead of ~55 for the field-by-field form.
__host__ __device__ __forceinline__ void cbd2_words(uint32_t t, uint32_t (&w)[4]) {
  const uint32_t d = (t & 0x55555555u) + ((t >> 1) & 0x55555555u);
  const uint32_t ae = d & 0x03030303u, be = (d >> 2) & 0x03030303u;
  const uint32_t ao = (d >> 4) & 0x03030303u, bo = (d >> 6) & 0x03030303u;
  const uint32_t ce = ((ae | 0x80808080u) - be) ^ 0x80808080u;  // signed bytes: coefficients 0, 2, 4, 6
  const uint32_t co = ((ao | 0x80808080u) - bo) ^ 0x80808080u;  // coefficients 1, 3, 5, 7
  w[0] = prmt_sx(ce, co, 0xc480);
  w[1] = prmt_sx(ce, co, 0xd591);
  w[2] = prmt_sx(ce, co, 0xe6a2);
  w[3] = prmt_sx(ce, co, 0xf7b3);
}

// CBD_eta (sample.go:31-95) of a PRF output B of 64 eta bytes, lane by lane: coefficient c is nibble c of B (eta = 2)
// or bits [6 c, 6 c + 6) (eta = 3), so for its S-layout coefficients 16 s + 2 v + b lane v needs, for s = 0..15, byte
// 8 s + v of B (eta = 2) or the 12 bits at bit 96 s + 12 v (eta = 3).  noise_select gathers them from the 32 / 48
// little-endian words of B into kNoiseWords words: byte s & 3 of word s >> 2 (eta = 2), the field of s at bit 16 (s & 1)
// of word s >> 1 (eta = 3).  noise_pairs turns the words of s = 4 k .. 4 k + 3 into the four packed pairs of
// coefficients 16 s + 2 v + {0, 1}.
template <int ETA>
constexpr int kNoiseWords = ETA == 2 ? 4 : 8;
template <int ETA>
__host__ __device__ __forceinline__ void noise_select(const uint32_t* w, int v, uint32_t (&x)[kNoiseWords<ETA>]) {
  if constexpr (ETA == 2) {
    const int h = v >> 2;
    const uint32_t sel = (uint32_t)(v & 3) | ((uint32_t)(4 + (v & 3)) << 4);  // byte v & 3 of two words
#pragma unroll
    for (int k = 0; k < 4; k++) {  // s = 4 k + q lies in word 2 s + h
      const uint32_t t01 = prmt_sx(w[8 * k + h], w[8 * k + 2 + h], sel);
      const uint32_t t23 = prmt_sx(w[8 * k + 4 + h], w[8 * k + 6 + h], sel);
      x[k] = prmt_sx(t01, t23, 0x5410);
    }
  } else {
    const int wo = (12 * v) >> 5, sh = (12 * v) & 31;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      uint32_t f[2];
#pragma unroll
      for (int b = 0; b < 2; b++) {
        const int s = 2 * i + b;
        const uint64_t lo = w[3 * s + wo], hi = sh > 20 ? w[3 * s + wo + 1] : 0u;  // lanes 2 and 5 straddle two words
        f[b] = (uint32_t)(((hi << 32) | lo) >> sh) & 0xfffu;
      }
      x[i] = f[0] | (f[1] << 16);
    }
  }
}
template <int ETA>
__host__ __device__ __forceinline__ void noise_pairs(const uint32_t (&x)[kNoiseWords<ETA>], int k, uint32_t (&p)[4]) {
  if constexpr (ETA == 2) {
    cbd2_words(x[k], p);
  } else {  // per 6-bit half of a field: (sum of its low three bits) - (sum of its high three bits)
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const uint32_t t = x[2 * k + i], m = 0x02490249u;
      const uint32_t d = (t & m) + ((t >> 1) & m) + ((t >> 2) & m);
#pragma unroll
      for (int b = 0; b < 2; b++) {
        const uint32_t e = d >> (16 * b);
        p[2 * i + b] = pack2_lo((int32_t)(e & 7) - (int32_t)((e >> 3) & 7), (int32_t)((e >> 6) & 7) - (int32_t)((e >> 9) & 7));
      }
    }
  }
}
// all 32 coefficients of the lane, S layout
template <int ETA>
__host__ __device__ __forceinline__ void noise_cbd(const uint32_t (&x)[kNoiseWords<ETA>], int32_t (&r)[32]) {
#pragma unroll
  for (int k = 0; k < 4; k++) {
    uint32_t p[4];
    noise_pairs<ETA>(x, k, p);
#pragma unroll
    for (int q = 0; q < 4; q++) unpack2_lo(p[q], r[8 * k + 2 * q], r[8 * k + 2 * q + 1]);
  }
}

// The low-format pairs of the C-layout passes are kept lane-transposed (in the device table and therefore in its
// shared-memory copy): "entry i of lane v" of a layer, Zetas position base + c v + i (c = 2, 4, 8 entries per lane for
// l = 8, 4, 2), is stored at base + 8 i + v, so the eight lanes of an octet read eight consecutive pairs instead of
// pairs 2c words apart (a 4-way bank conflict per read in table order).
__host__ __device__ constexpr int tw_slot(int k) {
  if (k < 16) return k;
  const int b = k >= 64 ? 64 : (k >= 32 ? 32 : 16), c = b / 8;
  return b + 8 * ((k - b) % c) + (k - b) / c;
}
struct LaneTwLow {
  TwLow l8[2], l4[4], l2[8];
};
__host__ __device__ __forceinline__ void load_lane_tw_lo(LaneTwLow& t, const TwLow* tab, int v) {
#pragma unroll
  for (int i = 0; i < 2; i++) t.l8[i] = tab[16 + 8 * i + v];
#pragma unroll
  for (int i = 0; i < 4; i++) t.l4[i] = tab[32 + 8 * i + v];
#pragma unroll
  for (int i = 0; i < 8; i++) t.l2[i] = tab[64 + 8 * i + v];
}
__host__ __device__ __forceinline__ TwLow twl_at(const volatile TwLow* tab, int k) {
  const volatile int2* p = reinterpret_cast<const volatile int2*>(tab + k);
  TwLow t;
  t.zp = p->x;
  t.kk = p->y;
  return t;
}

__host__ __device__ __forceinline__ void fwd_pass_S_lo(int32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 16; i++) ct_lo(r[i], r[i + 16], ZetaL<1>::zp, ZetaL<1>::kk);
  static_for<0, 2>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 8; i++) ct_lo(r[16 * h + i], r[16 * h + i + 8], ZetaL<2 + h>::zp, ZetaL<2 + h>::kk);
  });
  static_for<0, 4>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 4; i++) ct_lo(r[8 * h + i], r[8 * h + i + 4], ZetaL<4 + h>::zp, ZetaL<4 + h>::kk);
  });
  static_for<0, 8>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 2; i++) ct_lo(r[4 * h + i], r[4 * h + i + 2], ZetaL<8 + h>::zp, ZetaL<8 + h>::kk);
  });
}
__host__ __device__ __forceinline__ void fwd_pass_C_lo(int32_t (&r)[32], const LaneTwLow& t) {
#pragma unroll
  for (int blk = 0; blk < 2; blk++)
#pragma unroll
    for (int j = 0; j < 8; j++) ct_lo(r[16 * blk + j], r[16 * blk + j + 8], t.l8[blk].zp, t.l8[blk].kk);
#pragma unroll
  for (int blk = 0; blk < 4; blk++)
#pragma unroll
    for (int j = 0; j < 4; j++) ct_lo(r[8 * blk + j], r[8 * blk + j + 4], t.l4[blk].zp, t.l4[blk].kk);
#pragma unroll
  for (int blk = 0; blk < 8; blk++)
#pragma unroll
    for (int j = 0; j < 2; j++) ct_lo(r[4 * blk + j], r[4 * blk + j + 2], t.l2[blk].zp, t.l2[blk].kk);
}
// forward pass 2 with the pairs read from the shared-memory copy where they are used
__host__ __device__ __forceinline__ void fwd_pass_C_lo_smem(int32_t (&r)[32], const volatile TwLow* tab, int v) {
#pragma unroll
  for (int blk = 0; blk < 2; blk++) {
    const TwLow t = twl_at(tab, 16 + 8 * blk + v);
#pragma unroll
    for (int j = 0; j < 8; j++) ct_lo(r[16 * blk + j], r[16 * blk + j + 8], t.zp, t.kk);
  }
#pragma unroll
  for (int blk = 0; blk < 4; blk++) {
    const TwLow t = twl_at(tab, 32 + 8 * blk + v);
#pragma unroll
    for (int j = 0; j < 4; j++) ct_lo(r[8 * blk + j], r[8 * blk + j + 4], t.zp, t.kk);
  }
#pragma unroll
  for (int blk = 0; blk < 8; blk++) {
    const TwLow t = twl_at(tab, 64 + 8 * blk + v);
#pragma unroll
    for (int j = 0; j < 2; j++) ct_lo(r[4 * blk + j], r[4 * blk + j + 2], t.zp, t.kk);
  }
}
// inverse pass A: Zetas positions 127 - 8v - blk, 63 - 4v - blk, 31 - 2v - blk (ntt.go:152-160), i.e. entry 7 - blk
// (3 - blk, 1 - blk) of lane 7 - v in the transposed table
__host__ __device__ __forceinline__ void inv_pass_C_lo(int32_t (&r)[32], const volatile TwLow* tab, int v) {
#pragma unroll
  for (int blk = 0; blk < 8; blk++) {
    const TwLow t = twl_at(tab, 64 + 8 * (7 - blk) + (7 - v));
#pragma unroll
    for (int j = 0; j < 2; j++) gs_lo(r[4 * blk + j], r[4 * blk + j + 2], t.zp, t.kk);
  }
#pragma unroll
  for (int blk = 0; blk < 4; blk++) {
    const TwLow t = twl_at(tab, 32 + 8 * (3 - blk) + (7 - v));
#pragma unroll
    for (int j = 0; j < 4; j++) gs_lo(r[8 * blk + j], r[8 * blk + j + 4], t.zp, t.kk);
  }
#pragma unroll
  for (int blk = 0; blk < 2; blk++) {
    const TwLow t = twl_at(tab, 16 + 8 * (1 - blk) + (7 - v));
#pragma unroll
    for (int j = 0; j < 8; j++) gs_lo(r[16 * blk + j], r[16 * blk + j + 8], t.zp, t.kk);
  }
  r[16] = barrett_lo(r[16]);
  r[17] = barrett_lo(r[17]);
}
// the lazy Barrett schedule of inv_pass_S, on low-format registers.  The per-lane conditions of the schedule are folded
// into the Barrett multiplier (20159 where the reference reduces, 0 elsewhere: x - ((x * 0) >> 26) q = x), so every
// lane runs the same three instructions and the warp never diverges.
__host__ __device__ __forceinline__ int32_t barrett_if(int32_t x, int32_t mul) { return x - ((x * mul) >> 26) * Q; }
// SCALE = false leaves the multiplication by 1441 out (callers that folded the constant into an operand)
template <bool SCALE = true>
__host__ __device__ __forceinline__ void inv_pass_S_lo(int32_t (&r)[32], int v) {
  constexpr int32_t B = 20159;
  const int32_t m_v0 = v == 0 ? B : 0, m_v01 = v <= 1 ? B : 0, m_v1 = v == 1 ? B : 0, m_v13 = (v >= 1 && v <= 3) ? B : 0,
                m_v23 = (v == 2 || v == 3) ? B : 0, m_v27 = v >= 2 ? B : 0;
  static_for<0, 8>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 2; i++) gs_lo(r[4 * h + i], r[4 * h + i + 2], ZetaL<15 - h>::zp, ZetaL<15 - h>::kk);
  });
  // after layer 4: idx mod 64 in {0,1} -> (s&3)==0, v==0 ; {32..35} -> (s&3)==2, v<=1
#pragma unroll
  for (int s = 0; s < 16; s += 4)
#pragma unroll
    for (int b = 0; b < 2; b++) {
      r[2 * s + b] = barrett_if(r[2 * s + b], m_v0);
      r[2 * (s + 2) + b] = barrett_if(r[2 * (s + 2) + b], m_v01);
    }
  static_for<0, 4>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 4; i++) gs_lo(r[8 * h + i], r[8 * h + i + 4], ZetaL<7 - h>::zp, ZetaL<7 - h>::kk);
  });
  // after layer 5: idx mod 128 in {2,3} -> (s&7)==0, v==1 ; {66..71} -> (s&7)==4, v in 1..3
#pragma unroll
  for (int s = 0; s < 16; s += 8)
#pragma unroll
    for (int b = 0; b < 2; b++) {
      r[2 * s + b] = barrett_if(r[2 * s + b], m_v1);
      r[2 * (s + 4) + b] = barrett_if(r[2 * (s + 4) + b], m_v13);
    }
  static_for<0, 2>([&](auto hc) {
    constexpr int h = decltype(hc)::value;
#pragma unroll
    for (int i = 0; i < 8; i++) gs_lo(r[16 * h + i], r[16 * h + i + 8], ZetaL<3 - h>::zp, ZetaL<3 - h>::kk);
  });
  // after layer 6: idx in {4..7} -> s==0, v in {2,3} ; {132..143} -> s==8, v in 2..7
#pragma unroll
  for (int b = 0; b < 2; b++) {
    r[b] = barrett_if(r[b], m_v23);
    r[16 + b] = barrett_if(r[16 + b], m_v27);
  }
#pragma unroll
  for (int i = 0; i < 16; i++) gs_lo(r[i], r[i + 16], ZetaL<1>::zp, ZetaL<1>::kk);
  if constexpr (SCALE) {
#pragma unroll
    for (int i = 0; i < 32; i++) r[i] = mont_mul_lo(r[i], kScaleZp, kScaleKk);
  }
}

// Packed S <-> C transposition of low-format registers through the 608-byte tile of store_S / load_C (kernels whose
// shared memory has no room for the wide tile below)
__device__ __forceinline__ void store_S_lo(uint32_t* tile, int v, const int32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++) tile[8 * s + v + 4 * (s >> 2)] = pack2_lo(r[2 * s], r[2 * s + 1]);
}
__device__ __forceinline__ void load_S_lo(const uint32_t* tile, int v, int32_t (&r)[32]) {
#pragma unroll
  for (int s = 0; s < 16; s++) unpack2_lo(tile[8 * s + v + 4 * (s >> 2)], r[2 * s], r[2 * s + 1]);
}
__device__ __forceinline__ void store_C_lo(uint32_t* tile, int v, const int32_t (&r)[32]) {
  uint4* p = reinterpret_cast<uint4*>(tile + 16 * v + 4 * (v >> 1));
#pragma unroll
  for (int c = 0; c < 4; c++)
    p[c] = make_uint4(pack2_lo(r[8 * c], r[8 * c + 1]), pack2_lo(r[8 * c + 2], r[8 * c + 3]),
                      pack2_lo(r[8 * c + 4], r[8 * c + 5]), pack2_lo(r[8 * c + 6], r[8 * c + 7]));
}
__device__ __forceinline__ void load_C_lo(const uint32_t* tile, int v, int32_t (&r)[32]) {
  const uint4* p = reinterpret_cast<const uint4*>(tile + 16 * v + 4 * (v >> 1));
#pragma unroll
  for (int c = 0; c < 4; c++) {
    const uint4 w = p[c];
    unpack2_lo(w.x, r[8 * c], r[8 * c + 1]);
    unpack2_lo(w.y, r[8 * c + 2], r[8 * c + 3]);
    unpack2_lo(w.z, r[8 * c + 4], r[8 * c + 5]);
    unpack2_lo(w.w, r[8 * c + 6], r[8 * c + 7]);
  }
}

// Unpacked S <-> C transposition for the fast path: registers travel as 128-bit groups of four, one group per
// (writer lane, reader lane) pair, in a tile of 8 rows x 9 groups (144-byte rows): the eight lanes of an octet -- one
// quarter-warp, i.e. one shared-memory transaction of a 128-bit access -- hit eight different 16-byte bank groups both
// when they write (row = own lane, group = reader) and when they read (row = writer, group = own lane).
// 8 STS.128 + 8 LDS.128 per lane replace 16 PRMT + 16 STS.32 + 4 LDS.128 + 32 unpacking instructions.
constexpr int kWideTileBytes = 8 * 144;
__host__ __device__ __forceinline__ void wide_store_S(unsigned char* tile, int v, const int32_t (&r)[32]) {
  // S layout r[2s+b] = coefficient 16s + 2v + b: group u = r[4u..4u+3] = coefficients 32u + {2v, 2v+1, 16+2v, 17+2v}
  int4* wr = reinterpret_cast<int4*>(tile + v * 144);
#pragma unroll
  for (int u = 0; u < 8; u++) wr[u] = make_int4(r[4 * u], r[4 * u + 1], r[4 * u + 2], r[4 * u + 3]);
}
__host__ __device__ __forceinline__ void wide_load_C(const unsigned char* tile, int v, int32_t (&r)[32]) {
  const int4* rd = reinterpret_cast<const int4*>(tile + v * 16);
#pragma unroll
  for (int w = 0; w < 8; w++) {  // from writer lane w: C registers 2w, 2w+1, 16+2w, 17+2w
    const int4 g = rd[9 * w];
    r[2 * w] = g.x;
    r[2 * w + 1] = g.y;
    r[16 + 2 * w] = g.z;
    r[17 + 2 * w] = g.w;
  }
}
__host__ __device__ __forceinline__ void wide_store_C(unsigned char* tile, int v, const int32_t (&r)[32]) {
  // C layout r[i] = coefficient 32v + i: group u (for reader lane u) = r[2u], r[2u+1], r[16+2u], r[17+2u]
  int4* wr = reinterpret_cast<int4*>(tile + v * 144);
#pragma unroll
  for (int u = 0; u < 8; u++) wr[u] = make_int4(r[2 * u], r[2 * u + 1], r[16 + 2 * u], r[17 + 2 * u]);
}
__host__ __device__ __forceinline__ void wide_load_S(const unsigned char* tile, int v, int32_t (&r)[32]) {
  const int4* rd = reinterpret_cast<const int4*>(tile + v * 16);
#pragma unroll
  for (int w = 0; w < 8; w++) {  // from writer lane w: coefficients 32w + {2v, 2v+1, 16+2v, 17+2v} = S registers 4w..4w+3
    const int4 g = rd[9 * w];
    r[4 * w] = g.x;
    r[4 * w + 1] = g.y;
    r[4 * w + 2] = g.z;
    r[4 * w + 3] = g.w;
  }
}

// ---------------------------------------------------------------- MulHat on C layout
// poly.go:63-100.  p = a (*) b in Z_q[x]/(x^2 -+ zeta); quads (4j..4j+3) of lane v
// use Zetas[64 + 8v + j] == t.l2[j].z.  acc += result (PolyDotHat, vec.go:30-37).
__device__ __forceinline__ void mulhat_acc_C(int32_t (&acc)[32], const int32_t (&a)[32], const int32_t (&b)[32],
                                             const LaneTw& t) {
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int32_t a0 = a[4 * j] >> 16, a1 = a[4 * j + 1] >> 16, a2 = a[4 * j + 2] >> 16, a3 = a[4 * j + 3] >> 16;
    const int32_t b0 = b[4 * j] >> 16, b1 = b[4 * j + 1] >> 16, b2 = b[4 * j + 2] >> 16, b3 = b[4 * j + 3] >> 16;
    const int32_t z = t.l2[j].z, zq = t.l2[j].zq;
    int32_t p0 = mont_prod_hi(a1, b1);
    p0 = mont_mul_hi(p0 >> 16, z, zq);
    p0 += mont_prod_hi(a0, b0);
    int32_t p1 = mont_prod_hi(a0, b1) + mont_prod_hi(a1, b0);
    int32_t p2 = mont_prod_hi(a3, b3);
    p2 = -mont_mul_hi(p2 >> 16, z, zq);
    p2 += mont_prod_hi(a2, b2);
    int32_t p3 = mont_prod_hi(a2, b3) + mont_prod_hi(a3, b2);
    acc[4 * j] += p0;
    acc[4 * j + 1] += p1;
    acc[4 * j + 2] += p2;
    acc[4 * j + 3] += p3;
  }
}

}  // namespace kyber
}  // namespace cb200
