// X448 on one thread: GF(2^448 - 2^224 - 1) arithmetic and the Montgomery ladder (RFC 7748 section 5).
//
// Mirrors what dh/x448/key.go:33-46 computes: KeyGen = u([clamp(k)] G) with u(G) = 5 and Shared = u([clamp(k)] P),
// both in canonical little-endian form; the reference reaches the same values with a Joye ladder over a precomputed
// table (curve.go:9-48) and a Montgomery ladder over 64-bit limbs (curve.go:50-68, math/fp448).
//
// Representation: sixteen signed limbs of 28 bits (value = sum v[i] 2^(28 i)), carried into the balanced range
// |v[i]| <= 2^27 (limbs 1 and 9 take the small spill of the wrap-around carry), products accumulated in 64 bits --
// one IMAD.WIDE each.  With this radix 2^224 is limb 8, so the reduction 2^448 = 2^224 + 1 folds whole columns.
// A sum or difference of two carried values (|v| <= 2^28 + 2^8) may enter a multiplication: a folded column adds at
// most 38 products (column 8: 9 + 15 + 2 * 7), 38 * (2^28 + 2^8)^2 < 2^62, so the accumulators never overflow and
// the ladder needs no carry between its additions and multiplications.
#pragma once
#include <cstdint>

// Plain integer C++, like x25519.cuh: it compiles for the device (kernels), for the host inside the library and for
// the host-only limb test of the CPU suite.
#if defined(__CUDACC__)
#define CB200_XHD __host__ __device__ __forceinline__
#define CB200_XHD_NOINLINE static __host__ __device__ __noinline__
#else
#define CB200_XHD inline
#define CB200_XHD_NOINLINE inline
#endif

namespace cb200 {
namespace x448 {

constexpr int kWords = 14;  // 56 bytes

struct Fe {
  int32_t v[16];
};

CB200_XHD void fe_set(Fe& h, int32_t x) {
  h.v[0] = x;
#pragma unroll
  for (int i = 1; i < 16; i++) h.v[i] = 0;
}
CB200_XHD void fe_add(Fe& h, const Fe& f, const Fe& g) {
#pragma unroll
  for (int i = 0; i < 16; i++) h.v[i] = f.v[i] + g.v[i];
}
CB200_XHD void fe_sub(Fe& h, const Fe& f, const Fe& g) {
#pragma unroll
  for (int i = 0; i < 16; i++) h.v[i] = f.v[i] - g.v[i];
}
CB200_XHD void fe_cswap(Fe& f, Fe& g, uint32_t bit) {
  const int32_t m = -(int32_t)bit;
#pragma unroll
  for (int i = 0; i < 16; i++) {
    const int32_t x = m & (f.v[i] ^ g.v[i]);
    f.v[i] ^= x;
    g.v[i] ^= x;
  }
}

// Rounding carries bring every limb back to |v| <= 2^27; the carry out of limb 15 re-enters at limbs 0 and 8
// (2^448 = 2^224 + 1), whose carries then leave a small spill in limbs 1 and 9.
CB200_XHD void fe_carry(Fe& h, int64_t (&t)[16]) {
#pragma unroll
  for (int i = 0; i < 15; i++) {
    const int64_t c = (t[i] + ((int64_t)1 << 27)) >> 28;
    t[i + 1] += c;
    t[i] -= c << 28;
  }
  {
    const int64_t c = (t[15] + ((int64_t)1 << 27)) >> 28;
    t[15] -= c << 28;
    t[0] += c;
    t[8] += c;
  }
#pragma unroll
  for (int i = 0; i < 9; i += 8) {
    const int64_t c = (t[i] + ((int64_t)1 << 27)) >> 28;
    t[i + 1] += c;
    t[i] -= c << 28;
  }
#pragma unroll
  for (int i = 0; i < 16; i++) h.v[i] = (int32_t)t[i];
}

// Columns 16..30 of a double-width product folded onto 0..15: a column k >= 16 adds to k - 16 and k - 8, and a
// column k - 8 >= 16 folds again, so a column k >= 24 ends up twice in k - 16 and once in k - 24.
CB200_XHD void fe_fold(Fe& h, const int64_t (&t)[31]) {
  int64_t r[16];
#pragma unroll
  for (int c = 0; c < 8; c++) r[c] = t[c] + t[c + 16] + (c + 24 <= 30 ? t[c + 24] : 0);
#pragma unroll
  for (int c = 8; c < 16; c++) r[c] = t[c] + t[c + 8] + (c + 16 <= 30 ? 2 * t[c + 16] : 0);
  fe_carry(h, r);
}
// h = f * g (schoolbook, 256 wide multiplications)
CB200_XHD void fe_mul(Fe& h, const Fe& f, const Fe& g) {
  int64_t t[31];
#pragma unroll
  for (int k = 0; k < 31; k++) {
    int64_t acc = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const int j = k - i;
      if (j < 0 || j > 15) continue;
      acc += (int64_t)f.v[i] * g.v[j];
    }
    t[k] = acc;
  }
  fe_fold(h, t);
}
// h = f^2: every unordered pair of limbs once (136 wide multiplications)
CB200_XHD void fe_sq(Fe& h, const Fe& f) {
  int32_t f2[16];
#pragma unroll
  for (int i = 0; i < 16; i++) f2[i] = 2 * f.v[i];
  int64_t t[31];
#pragma unroll
  for (int k = 0; k < 31; k++) {
    int64_t acc = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const int j = k - i;
      if (j < i || j > 15) continue;
      acc += (int64_t)(i == j ? f.v[i] : f2[i]) * f.v[j];
    }
    t[k] = acc;
  }
  fe_fold(h, t);
}
CB200_XHD void fe_mul_small(Fe& h, const Fe& f, int32_t s) {
  int64_t t[16];
#pragma unroll
  for (int i = 0; i < 16; i++) t[i] = (int64_t)f.v[i] * s;
  fe_carry(h, t);
}

// z^(p - 2), p - 2 = [223 ones] 0 [222 ones] 0 1, by a 2^k - 1 addition chain (447 squarings, 13 multiplications)
CB200_XHD_NOINLINE void fe_invert(Fe& out, const Fe& z) {
  Fe t, z2, z3, z6, z12, z24, z30, z48, z96, z192, z222, z223;
  auto pow2k = [](Fe& h, const Fe& f, int k) {
    fe_sq(h, f);
#pragma unroll 1
    for (int i = 1; i < k; i++) fe_sq(h, h);
  };
  pow2k(t, z, 1);
  fe_mul(z2, t, z);  // 2^2 - 1
  pow2k(t, z2, 1);
  fe_mul(z3, t, z);  // 2^3 - 1
  pow2k(t, z3, 3);
  fe_mul(z6, t, z3);
  pow2k(t, z6, 6);
  fe_mul(z12, t, z6);
  pow2k(t, z12, 12);
  fe_mul(z24, t, z12);
  pow2k(t, z24, 6);
  fe_mul(z30, t, z6);
  pow2k(t, z24, 24);
  fe_mul(z48, t, z24);
  pow2k(t, z48, 48);
  fe_mul(z96, t, z48);
  pow2k(t, z96, 96);
  fe_mul(z192, t, z96);
  pow2k(t, z192, 30);
  fe_mul(z222, t, z30);
  pow2k(t, z222, 1);
  fe_mul(z223, t, z);
  pow2k(t, z223, 223);
  fe_mul(t, t, z222);  // [223 ones] 0 [222 ones]
  pow2k(t, t, 2);
  fe_mul(out, t, z);   // ... 0 1
}

// 56 little-endian bytes (as 14 words) -> carried limbs; all 448 bits are taken (no bit is masked, unlike X25519)
CB200_XHD void fe_frombytes(Fe& h, const uint32_t (&w)[kWords]) {
  int64_t t[16];
#pragma unroll
  for (int i = 0; i < 16; i++) {
    const int off = 28 * i, wi = off >> 5, sh = off & 31;
    uint32_t x = w[wi] >> sh;
    if (sh + 28 > 32) x |= w[wi + 1] << (32 - sh);
    t[i] = (int64_t)(x & ((1u << 28) - 1));
  }
  fe_carry(h, t);
}
// canonical encoding (math/fp448 ToBytes): limbs to [0, 2^28) with floor carries -- three passes settle the
// wrap-around carry of a value in (-2^448, 2^448) -- then subtract p exactly when the value is >= p
CB200_XHD void fe_tobytes(uint32_t (&w)[kWords], const Fe& f) {
  const int64_t M = ((int64_t)1 << 28) - 1;
  int64_t l[16];
#pragma unroll
  for (int i = 0; i < 16; i++) l[i] = f.v[i];
#pragma unroll
  for (int pass = 0; pass < 3; pass++) {
#pragma unroll
    for (int i = 0; i < 15; i++) {
      l[i + 1] += l[i] >> 28;
      l[i] &= M;
    }
    const int64_t c = l[15] >> 28;
    l[15] &= M;
    l[0] += c;
    l[8] += c;
  }
  // v >= p  <=>  v + 2^224 + 1 >= 2^448
  int64_t s[16];
#pragma unroll
  for (int i = 0; i < 16; i++) s[i] = l[i] + (i == 0 || i == 8 ? 1 : 0);
#pragma unroll
  for (int i = 0; i < 15; i++) {
    s[i + 1] += s[i] >> 28;
    s[i] &= M;
  }
  const int64_t ge = -(s[15] >> 28);  // all ones when v >= p
  s[15] &= M;
#pragma unroll
  for (int i = 0; i < 16; i++) l[i] = (s[i] & ge) | (l[i] & ~ge);
#pragma unroll
  for (int i = 0; i < kWords; i++) w[i] = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) {
    const int off = 28 * i, wi = off >> 5, sh = off & 31;
    const uint64_t x = (uint64_t)l[i] << sh;
    w[wi] |= (uint32_t)x;
    if (wi + 1 < kWords) w[wi + 1] |= (uint32_t)(x >> 32);
  }
}

// the three low-order values 0, 1 and p - 1 of curve.go:76-104, canonical form; key.go:22-30 rejects them after
// reduction mod p
CB200_XHD bool is_low_order(const uint32_t (&c)[kWords]) {
  uint32_t rest = 0, dm = (c[0] ^ 0xfffffffeu) | (c[7] ^ 0xfffffffeu);
#pragma unroll
  for (int i = 1; i < kWords; i++) {
    rest |= c[i];
    if (i != 7) dm |= ~c[i];
  }
  return (rest == 0 && c[0] <= 1) || dm == 0;
}

// out = u([clamp(k)] P) as 14 words; returns false when P is of low order (the result is then all zero).
// The scalar's 14 words are read where they lie, one per ladder step: a register copy selected by the bit index
// becomes a local-memory array once it has 14 words.
CB200_XHD bool scalarmult(uint32_t (&out)[kWords], const uint32_t* kin, const uint32_t (&pin)[kWords]) {
  Fe x1, x2, z2, x3, z3;
  fe_frombytes(x1, pin);
  uint32_t canon[kWords];
  fe_tobytes(canon, x1);
  const bool ok = !is_low_order(canon);
  fe_set(x2, 1);
  fe_set(z2, 0);
  x3 = x1;
  fe_set(z3, 1);
  uint32_t swap = 0;
#pragma unroll 1
  for (int s = 447; s >= 0; s--) {
    uint32_t word = kin[s >> 5];
    if (s < 32) word &= 0xfffffffcu;      // clamp (key.go:15-20): k[0] &= 252,
    if (s >= 416) word |= 0x80000000u;   // k[55] |= 128
    const uint32_t bit = (word >> (s & 31)) & 1;
    swap ^= bit;
    fe_cswap(x2, x3, swap);
    fe_cswap(z2, z3, swap);
    swap = bit;
    // the products that end the life of c and d come first, then those of a and b: fewer field elements live at once
    Fe a, b, c, d, aa, bb, e, da, cb, t;
    fe_add(a, x2, z2);
    fe_sub(b, x2, z2);
    fe_add(c, x3, z3);
    fe_sub(d, x3, z3);
    fe_mul(da, d, a);
    fe_mul(cb, c, b);
    fe_sq(aa, a);
    fe_sq(bb, b);
    fe_sub(e, aa, bb);
    fe_add(t, da, cb);
    fe_sq(x3, t);
    fe_sub(t, da, cb);
    fe_sq(t, t);
    fe_mul(z3, x1, t);
    fe_mul(x2, aa, bb);
    fe_mul_small(t, e, 39082);  // (A + 2) / 4, curve_generic.go:58-100: z2 = E (BB + a24 E)
    fe_add(t, t, bb);
    fe_mul(z2, e, t);
  }
  fe_cswap(x2, x3, swap);
  fe_cswap(z2, z3, swap);
  fe_invert(z2, z2);
  fe_mul(x2, x2, z2);
  fe_tobytes(out, x2);
  return ok;
}

}  // namespace x448
}  // namespace cb200
