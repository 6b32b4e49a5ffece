// X25519 on one thread: GF(2^255 - 19) arithmetic and the Montgomery ladder (RFC 7748 section 5).
//
// Mirrors what dh/x25519/key.go:44-56 computes: KeyGen = u([clamp(k)] G) and Shared = u([clamp(k)] P), both in
// canonical little-endian form; the reference reaches the same values with a Joye ladder over a precomputed table
// (curve.go:7-37) and a Montgomery ladder over 64-bit limbs (curve.go:40-75, math/fp25519).
//
// Representation: ten signed limbs of alternately 26 and 25 bits (value = sum v[i] 2^ceil(25.5 i)), products
// accumulated in 64 bits -- on sm_90a each product-accumulate is one IMAD.WIDE.  With ten independent accumulators
// per multiplication the wide-multiply latency is covered inside a single thread, so the kernel runs one scalar
// multiplication per thread and needs no shared memory.
#pragma once
#include <cstdint>

// The field and group code is plain integer C++: it compiles for the device (kernels), for the host inside the
// library (the fixed-base table is computed once at cb200_init) and for the host-only limb test of the CPU suite.
#if defined(__CUDACC__)
#define CB200_XHD __host__ __device__ __forceinline__
#define CB200_XHD_NOINLINE static __host__ __device__ __noinline__
#else
#define CB200_XHD inline
#define CB200_XHD_NOINLINE inline
#endif

namespace cb200 {
namespace x25519 {

struct Fe {
  int32_t v[10];
};

CB200_XHD void fe_set(Fe& h, int32_t x) {
  h.v[0] = x;
#pragma unroll
  for (int i = 1; i < 10; i++) h.v[i] = 0;
}
CB200_XHD void fe_add(Fe& h, const Fe& f, const Fe& g) {
#pragma unroll
  for (int i = 0; i < 10; i++) h.v[i] = f.v[i] + g.v[i];
}
CB200_XHD void fe_sub(Fe& h, const Fe& f, const Fe& g) {
#pragma unroll
  for (int i = 0; i < 10; i++) h.v[i] = f.v[i] - g.v[i];
}
CB200_XHD void fe_cswap(Fe& f, Fe& g, uint32_t bit) {
  const int32_t m = -(int32_t)bit;
#pragma unroll
  for (int i = 0; i < 10; i++) {
    const int32_t x = m & (f.v[i] ^ g.v[i]);
    f.v[i] ^= x;
    g.v[i] ^= x;
  }
}

// Rounding carries bring every limb back to |v[2i]| <= 2^25, |v[2i+1]| <= 2^24 (plus the small spill of the final step).
CB200_XHD void fe_carry(Fe& h, int64_t (&t)[10]) {
#pragma unroll
  for (int i = 0; i < 9; i++) {
    const int w = (i & 1) ? 25 : 26;
    const int64_t c = (t[i] + ((int64_t)1 << (w - 1))) >> w;
    t[i + 1] += c;
    t[i] -= c << w;
  }
  {
    const int64_t c = (t[9] + ((int64_t)1 << 24)) >> 25;
    t[0] += 19 * c;
    t[9] -= c << 25;
  }
  {
    const int64_t c = (t[0] + ((int64_t)1 << 25)) >> 26;
    t[1] += c;
    t[0] -= c << 26;
  }
#pragma unroll
  for (int i = 0; i < 10; i++) h.v[i] = (int32_t)t[i];
}

// h = f * g.  Inputs may be one addition or subtraction away from a carried value (|v| < 2^27).
// 2^ceil(25.5 i) * 2^ceil(25.5 j) = 2^ceil(25.5 (i + j)) * (2 if i and j are both odd), and 2^255 = 19.
CB200_XHD void fe_mul(Fe& h, const Fe& f, const Fe& g) {
  int32_t g19[10], f2[10];
#pragma unroll
  for (int i = 0; i < 10; i++) {
    g19[i] = 19 * g.v[i];
    f2[i] = (i & 1) ? 2 * f.v[i] : f.v[i];
  }
  int64_t t[10];
#pragma unroll
  for (int k = 0; k < 10; k++) {
    int64_t acc = 0;
#pragma unroll
    for (int i = 0; i < 10; i++) {
      const int j = (k - i + 10) % 10;
      const bool wrap = i > k;
      const int32_t a = (j & 1) ? f2[i] : f.v[i];  // doubled only when both indices are odd
      const int32_t b = wrap ? g19[j] : g.v[j];
      acc += (int64_t)a * b;
    }
    t[k] = acc;
  }
  fe_carry(h, t);
}
// h = f^2: every unordered pair of limbs once (55 wide multiplications instead of 100)
CB200_XHD void fe_sq(Fe& h, const Fe& f) {
  int32_t f19[10], fx2[10], fx4[10];
#pragma unroll
  for (int i = 0; i < 10; i++) {
    f19[i] = 19 * f.v[i];
    fx2[i] = 2 * f.v[i];
    fx4[i] = 4 * f.v[i];
  }
  int64_t t[10];
#pragma unroll
  for (int k = 0; k < 10; k++) {
    int64_t acc = 0;
#pragma unroll
    for (int i = 0; i < 10; i++) {
      const int j = (k - i + 10) % 10;
      if (i > j) continue;
      const bool wrap = i + j >= 10, both_odd = (i & 1) && (j & 1);
      const int coef = (i == j ? 1 : 2) * (both_odd ? 2 : 1);
      const int32_t a = coef == 1 ? f.v[i] : coef == 2 ? fx2[i] : fx4[i];
      const int32_t b = wrap ? f19[j] : f.v[j];
      acc += (int64_t)a * b;
    }
    t[k] = acc;
  }
  fe_carry(h, t);
}
CB200_XHD void fe_mul_small(Fe& h, const Fe& f, int32_t s) {
  int64_t t[10];
#pragma unroll
  for (int i = 0; i < 10; i++) t[i] = (int64_t)f.v[i] * s;
  fe_carry(h, t);
}

// z^(p - 2) by the usual 2^k - 1 addition chain (254 squarings, 11 multiplications)
CB200_XHD_NOINLINE void fe_invert(Fe& out, const Fe& z) {
  Fe z2, z9, z11, z5, z10, z20, z50, z100, t;
  auto pow2k = [](Fe& h, const Fe& f, int k) {
    fe_sq(h, f);
#pragma unroll 1
    for (int i = 1; i < k; i++) fe_sq(h, h);
  };
  pow2k(z2, z, 1);
  pow2k(t, z2, 2);
  fe_mul(z9, t, z);
  fe_mul(z11, z9, z2);
  pow2k(t, z11, 1);
  fe_mul(z5, t, z9);  // 2^5 - 1
  pow2k(t, z5, 5);
  fe_mul(z10, t, z5);  // 2^10 - 1
  pow2k(t, z10, 10);
  fe_mul(z20, t, z10);  // 2^20 - 1
  pow2k(t, z20, 20);
  fe_mul(t, t, z20);  // 2^40 - 1
  pow2k(t, t, 10);
  fe_mul(z50, t, z10);  // 2^50 - 1
  pow2k(t, z50, 50);
  fe_mul(z100, t, z50);  // 2^100 - 1
  pow2k(t, z100, 100);
  fe_mul(t, t, z100);  // 2^200 - 1
  pow2k(t, t, 50);
  fe_mul(t, t, z50);  // 2^250 - 1
  pow2k(t, t, 5);
  fe_mul(out, t, z11);  // 2^255 - 21
}

// 32 little-endian bytes (as 8 words) -> limbs; bit 255 is dropped (key.go:50: validPk[31] &= 127)
CB200_XHD void fe_frombytes(Fe& h, const uint32_t (&w)[8]) {
#pragma unroll
  for (int i = 0; i < 10; i++) {
    const int off = (51 * i + 1) / 2, width = (i & 1) ? 25 : 26, wi = off >> 5, sh = off & 31;
    uint32_t x = w[wi] >> sh;
    if (sh + width > 32) x |= w[wi + 1] << (32 - sh);
    h.v[i] = (int32_t)(x & ((1u << width) - 1));
  }
}
// canonical encoding (math/fp25519 ToBytes): subtract p exactly when the value is >= p
CB200_XHD void fe_tobytes(uint32_t (&w)[8], const Fe& f) {
  int32_t h[10];
#pragma unroll
  for (int i = 0; i < 10; i++) h[i] = f.v[i];
  int32_t q = (19 * h[9] + (1 << 24)) >> 25;
#pragma unroll
  for (int i = 0; i < 10; i++) q = (h[i] + q) >> ((i & 1) ? 25 : 26);
  h[0] += 19 * q;
#pragma unroll
  for (int i = 0; i < 9; i++) {
    const int wd = (i & 1) ? 25 : 26;
    const int32_t c = h[i] >> wd;
    h[i + 1] += c;
    h[i] -= c << wd;
  }
  h[9] &= (1 << 25) - 1;
#pragma unroll
  for (int i = 0; i < 8; i++) w[i] = 0;
#pragma unroll
  for (int i = 0; i < 10; i++) {
    const int off = (51 * i + 1) / 2, wi = off >> 5, sh = off & 31;
    const uint64_t x = (uint64_t)(uint32_t)h[i] << sh;
    w[wi] |= (uint32_t)x;
    if (wi + 1 < 8) w[wi + 1] |= (uint32_t)(x >> 32);
  }
}

// the five points of small order of curve.go:89-125, canonical form; key.go:25-32 rejects them after reduction mod p
CB200_XHD bool is_low_order(const uint32_t (&c)[8]) {
  const uint32_t o8a[8] = {0x7c7aebe0u, 0xaeb8413bu, 0xfae35616u, 0x6ac49ff1u, 0xeb8d09dau, 0xfdb1329cu, 0x16056286u, 0x00b8495fu};
  const uint32_t o8b[8] = {0xbc959c5fu, 0x248c50a3u, 0x55b1d0b1u, 0x5bef839cu, 0xc45c4404u, 0x868e1c58u, 0xdd4e22d8u, 0x57119fd0u};
  uint32_t rest = 0, da = 0, db = 0, dm = (c[0] ^ 0xffffffecu) | (c[7] ^ 0x7fffffffu);
#pragma unroll
  for (int i = 0; i < 8; i++) {
    if (i > 0) rest |= c[i];
    da |= c[i] ^ o8a[i];
    db |= c[i] ^ o8b[i];
    if (i > 0 && i < 7) dm |= ~c[i];
  }
  const bool zero_or_one = rest == 0 && c[0] <= 1;
  return zero_or_one || da == 0 || db == 0 || dm == 0;
}

// out = u([clamp(k)] P) as 8 words; returns false when P is of small order (the result is then all zero).
CB200_XHD bool scalarmult(uint32_t (&out)[8], const uint32_t (&kin)[8], const uint32_t (&pin)[8]) {
  uint32_t k[8];
#pragma unroll
  for (int i = 0; i < 8; i++) k[i] = kin[i];
  k[0] &= 0xfffffff8u;
  k[7] = (k[7] & 0x7fffffffu) | 0x40000000u;  // key.go:17-22
  Fe x1, x2, z2, x3, z3;
  fe_frombytes(x1, pin);
  uint32_t canon[8];
  fe_tobytes(canon, x1);
  const bool ok = !is_low_order(canon);
  fe_set(x2, 1);
  fe_set(z2, 0);
  x3 = x1;
  fe_set(z3, 1);
  uint32_t swap = 0;
#pragma unroll 1
  for (int s = 254; s >= 0; s--) {
    uint32_t word = k[0];
#pragma unroll
    for (int q = 1; q < 8; q++) word = ((s >> 5) == q) ? k[q] : word;
    const uint32_t bit = (word >> (s & 31)) & 1;
    swap ^= bit;
    fe_cswap(x2, x3, swap);
    fe_cswap(z2, z3, swap);
    swap = bit;
    Fe a, b, c, d, aa, bb, e, da, cb, t;
    fe_add(a, x2, z2);
    fe_sub(b, x2, z2);
    fe_add(c, x3, z3);
    fe_sub(d, x3, z3);
    fe_sq(aa, a);
    fe_sq(bb, b);
    fe_mul(da, d, a);
    fe_mul(cb, c, b);
    fe_sub(e, aa, bb);
    fe_add(t, da, cb);
    fe_sq(x3, t);
    fe_sub(t, da, cb);
    fe_sq(t, t);
    fe_mul(z3, x1, t);
    fe_mul(x2, aa, bb);
    fe_mul_small(t, e, 121665);
    fe_add(t, t, aa);
    fe_mul(z2, e, t);
  }
  fe_cswap(x2, x3, swap);
  fe_cswap(z2, z3, swap);
  fe_invert(z2, z2);
  fe_mul(x2, x2, z2);
  fe_tobytes(out, x2);
  return ok;
}


// ---------------------------------------------------------------- fixed-base multiplication for KeyGen
// x25519.KeyGen is [clamp(k)] G for the fixed point G (u = 9).  The reference spends a table on it too (Joye ladder
// over precomputed multiples, curve.go:7-37, table.go); here the multiplication runs on the birationally equivalent
// twisted Edwards curve -x^2 + y^2 = 1 + d x^2 y^2 (u = (1 + y) / (1 - y), G <-> B = (x, 4/5)) with radix-16 signed
// digits and a table of the multiples 1..8 of 256^i B, i < 32: 64 mixed additions and 4 doublings instead of 255
// ladder steps.  The result is the same field element, encoded the same way (checked against the ladder in the CPU
// suite and against the oracle on the GPU).  Addition and doubling are the complete a = -1 formulas in extended
// coordinates (Hisil, Wong, Carter, Dawson 2008).
struct GeExt {
  Fe X, Y, Z, T;
};
struct GePre {  // affine multiple prepared for mixed addition: y + x, y - x, 2 d x y
  Fe ypx, ymx, xy2d;
};
constexpr int kBaseTableWords = 32 * 8 * 32;  // [i][j] -> 32 words: ypx (10) | ymx (10) | xy2d (10) | 2 unused

CB200_XHD void fe_renorm(Fe& h) {  // carry a value that went through more than one addition
  int64_t t[10];
#pragma unroll
  for (int i = 0; i < 10; i++) t[i] = h.v[i];
  fe_carry(h, t);
}
// r = p + q (q affine, optionally negated)
CB200_XHD void ge_madd(GeExt& r, const GeExt& p, const GePre& q, bool neg) {
  Fe a, b, c, d, e, f, g, h, ypx = q.ypx, ymx = q.ymx, xy2d = q.xy2d;
  if (neg) {  // -(x, y) = (-x, y): y + x <-> y - x, 2dxy -> -2dxy
    Fe zero;
    fe_set(zero, 0);
    fe_cswap(ypx, ymx, 1);
    fe_sub(xy2d, zero, q.xy2d);
  }
  fe_sub(a, p.Y, p.X);
  fe_mul(a, a, ymx);
  fe_add(b, p.Y, p.X);
  fe_mul(b, b, ypx);
  fe_mul(c, p.T, xy2d);
  fe_add(d, p.Z, p.Z);
  fe_sub(e, b, a);
  fe_sub(f, d, c);
  fe_add(g, d, c);
  fe_add(h, b, a);
  fe_mul(r.X, e, f);
  fe_mul(r.Y, g, h);
  fe_mul(r.Z, f, g);
  fe_mul(r.T, e, h);
}
CB200_XHD void ge_dbl(GeExt& r, const GeExt& p) {
  Fe a, b, c, e, f, g, h, t;
  fe_sq(a, p.X);
  fe_sq(b, p.Y);
  fe_sq(c, p.Z);
  fe_add(c, c, c);
  fe_add(t, p.X, p.Y);
  fe_sq(t, t);
  fe_sub(e, t, a);
  fe_sub(e, e, b);
  fe_renorm(e);
  fe_sub(g, b, a);
  fe_sub(f, g, c);
  fe_renorm(f);
  fe_add(h, a, b);
  fe_set(t, 0);
  fe_sub(h, t, h);
  fe_mul(r.X, e, f);
  fe_mul(r.Y, g, h);
  fe_mul(r.Z, f, g);
  fe_mul(r.T, e, h);
}
CB200_XHD void pre_from_words(GePre& q, const int32_t* w) {
#pragma unroll
  for (int i = 0; i < 10; i++) {
    q.ypx.v[i] = w[i];
    q.ymx.v[i] = w[10 + i];
    q.xy2d.v[i] = w[20 + i];
  }
}

// Host side, once per process: table[i][j] = (j + 1) * 256^i * B in GePre form.
inline void build_base_table(int32_t* table) {
  static const uint32_t kD[8] = {0x135978a3u, 0x75eb4dcau, 0x4141d8abu, 0x00700a4du, 0x7779e898u, 0x8cc74079u, 0x2b6ffe73u, 0x52036ceeu};
  static const uint32_t kBx[8] = {0x8f25d51au, 0xc9562d60u, 0x9525a7b2u, 0x692cc760u, 0xfdd6dc5cu, 0xc0a4e231u, 0xcd6e53feu, 0x216936d3u};
  static const uint32_t kBy[8] = {0x66666658u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u};
  Fe d, d2;
  fe_frombytes(d, kD);
  fe_add(d2, d, d);
  fe_renorm(d2);
  auto to_pre = [&](GePre& q, const GeExt& p) {  // affine coordinates, then (y + x, y - x, 2 d x y), all carried
    Fe zi, x, y, t;
    fe_invert(zi, p.Z);
    fe_mul(x, p.X, zi);
    fe_mul(y, p.Y, zi);
    fe_add(q.ypx, y, x);
    fe_renorm(q.ypx);
    fe_sub(q.ymx, y, x);
    fe_renorm(q.ymx);
    fe_mul(t, x, y);
    fe_mul(q.xy2d, t, d2);
  };
  GeExt P;
  fe_frombytes(P.X, kBx);
  fe_frombytes(P.Y, kBy);
  fe_set(P.Z, 1);
  fe_mul(P.T, P.X, P.Y);
  for (int i = 0; i < 32; i++) {
    GePre base, q;
    to_pre(base, P);
    GeExt M = P;
    for (int j = 0; j < 8; j++) {
      if (j > 0) {
        GeExt s;
        ge_madd(s, M, base, false);
        M = s;
      }
      to_pre(q, M);
      int32_t* w = table + (i * 8 + j) * 32;
      for (int c = 0; c < 10; c++) {
        w[c] = q.ypx.v[c];
        w[10 + c] = q.ymx.v[c];
        w[20 + c] = q.xy2d.v[c];
      }
      w[30] = w[31] = 0;
    }
    for (int k = 0; k < 8; k++) {  // P <- 256 P
      GeExt s;
      ge_dbl(s, P);
      P = s;
    }
  }
}

// h = [k] B in extended coordinates for k < 2^255 (the top digit then stays within 1..8), from the table (device
// pointer on the GPU, host pointer in the CPU test).  The caller prepares the scalar: X25519 KeyGen clamps it, Ed25519
// passes a clamped or a reduced one.
CB200_XHD void ge_scalarmult_base(GeExt& h, const uint32_t (&kin)[8], const int32_t* __restrict__ table) {
  uint32_t k[8];
#pragma unroll
  for (int i = 0; i < 8; i++) k[i] = kin[i];
  // signed radix-16 digits: nibble i of k + 0x88...8 minus 8; the carry out of the top nibble stays in digit 63
  uint32_t carry = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint64_t s = (uint64_t)k[i] + 0x88888888u + carry;
    k[i] = (uint32_t)s;
    carry = (uint32_t)(s >> 32);
  }
  auto digit = [&](int i) -> int {
    uint32_t word = k[0];
#pragma unroll
    for (int q = 1; q < 8; q++) word = ((i >> 3) == q) ? k[q] : word;
    int e = (int)((word >> (4 * (i & 7))) & 15) - 8;
    if (i == 63) e += 16 * (int)carry;
    return e;
  };
  fe_set(h.X, 0);
  fe_set(h.Y, 1);
  fe_set(h.Z, 1);
  fe_set(h.T, 0);
  // Constant-time use of the secret digit, as the reference's KeyGen keeps it (ladderJoye indexes its table by the loop
  // counter only and uses cswap, dh/x25519/curve.go:7-37): all eight multiples of the row are read and the one wanted
  // -- or the neutral element (1, 1, 0) for digit 0 -- is kept by masks; the sign is applied by a masked swap of
  // y + x / y - x and a masked negation of 2dxy.  No branch and no address depends on the scalar.
  auto add_digit = [&](int i) {
    const int e = digit(i);
    const uint32_t neg = (uint32_t)(e >> 31);             // all ones for a negative digit
    const uint32_t m = ((uint32_t)e ^ neg) - neg;         // |e| in 0..8
    GePre q;
    fe_set(q.ypx, 1);
    fe_set(q.ymx, 1);
    fe_set(q.xy2d, 0);
    const int32_t* row = table + (i >> 1) * 8 * 32;
#pragma unroll 1
    for (int j = 0; j < 8; j++) {
      const uint32_t mask = (uint32_t)((int32_t)((m ^ (uint32_t)(j + 1)) - 1u) >> 31);  // all ones iff m == j + 1
#pragma unroll
      for (int c = 0; c < 10; c++) {
        q.ypx.v[c] = (int32_t)(((uint32_t)q.ypx.v[c] & ~mask) | ((uint32_t)row[j * 32 + c] & mask));
        q.ymx.v[c] = (int32_t)(((uint32_t)q.ymx.v[c] & ~mask) | ((uint32_t)row[j * 32 + 10 + c] & mask));
        q.xy2d.v[c] = (int32_t)(((uint32_t)q.xy2d.v[c] & ~mask) | ((uint32_t)row[j * 32 + 20 + c] & mask));
      }
    }
#pragma unroll
    for (int c = 0; c < 10; c++) {
      const uint32_t t = neg & ((uint32_t)q.ypx.v[c] ^ (uint32_t)q.ymx.v[c]);
      q.ypx.v[c] = (int32_t)((uint32_t)q.ypx.v[c] ^ t);
      q.ymx.v[c] = (int32_t)((uint32_t)q.ymx.v[c] ^ t);
      q.xy2d.v[c] = (int32_t)(((uint32_t)q.xy2d.v[c] ^ neg) - neg);
    }
    GeExt s;
    ge_madd(s, h, q, false);
    h = s;
  };
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 1; i < 64; i += 2) add_digit(i);
  for (int q = 0; q < 4; q++) {
    GeExt s;
    ge_dbl(s, h);
    h = s;
  }
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 0; i < 64; i += 2) add_digit(i);
}

// out = u([clamp(k)] G) from the table
CB200_XHD void scalarmult_base(uint32_t (&out)[8], const uint32_t (&kin)[8], const int32_t* __restrict__ table) {
  uint32_t k[8];
#pragma unroll
  for (int i = 0; i < 8; i++) k[i] = kin[i];
  k[0] &= 0xfffffff8u;
  k[7] = (k[7] & 0x7fffffffu) | 0x40000000u;  // key.go:17-22
  GeExt h;
  ge_scalarmult_base(h, k, table);
  Fe num, den;
  fe_add(num, h.Z, h.Y);
  fe_sub(den, h.Z, h.Y);
  fe_invert(den, den);
  fe_mul(num, num, den);
  fe_tobytes(out, num);
}

}  // namespace x25519
}  // namespace cb200
