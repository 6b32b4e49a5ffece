// P-256 (secp256r1, y^2 = x^3 - 3x + b over GF(p), p = 2^256 - 2^224 + 2^192 + 2^96 - 1) on one thread.
//
// Mirrors what Go's crypto/ecdh.P256() computes for the reference's DHKEM(P-256) (hpke/shortkem.go): KeyGen =
// 0x04 || X || Y of [k]G and Shared = X of [k]P, big-endian, for 0 < k < n; NewPublicKey's and NewPrivateKey's
// validation rules (the point on the curve with coordinates below p; 0 < k < n).
//
// Field: eight 32-bit words in Montgomery form (R = 2^256), fully reduced into [0, p) after every operation.  Since
// p = -1 mod 2^32, the Montgomery factor of each reduction step is the low word itself, and p's words are all
// 0, 1 or 2^32 - 1, so the reduction's products by p fold into additions and subtractions.  Products accumulate in
// 64 bits (one IMAD.WIDE per word product on sm_90a).
//
// Group: projective (X : Y : Z) with the complete formulas of Renes, Costello and Batina for a = -3 (ePrint 2015/1060,
// algorithms 4, 5 and 6).  They have no exceptional case -- the identity (0 : 1 : 0), doublings and inverse pairs
// included -- so no branch depends on a point or a scalar.
//
// Plain integer C++ like x25519.cuh: it compiles for the device (kernels), for the host inside the library (the
// fixed-base table is computed once at cb200_init) and for the host-only test of the CPU suite.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define CB200_XHD __host__ __device__ __forceinline__
#define CB200_XHD_NOINLINE static __host__ __device__ __noinline__
#else
#define CB200_XHD inline
#define CB200_XHD_NOINLINE inline
#endif

namespace cb200 {
namespace p256 {

constexpr int kW = 8;
// little-endian 32-bit words
#define CB200_P256_P {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 1u, 0xffffffffu}
#define CB200_P256_N {0xfc632551u, 0xf3b9cac2u, 0xa7179e84u, 0xbce6faadu, 0xffffffffu, 0xffffffffu, 0u, 0xffffffffu}

struct Fe {
  uint32_t v[kW];
};
struct Pt {  // projective (X : Y : Z), Montgomery form
  Fe X, Y, Z;
};
struct Aff {  // affine (x, y), Montgomery form
  Fe x, y;
};

CB200_XHD uint32_t p_word(int i) {
  const uint32_t p[kW] = CB200_P256_P;
  return p[i];
}

CB200_XHD void fe_copy(Fe& h, const Fe& f) {
#pragma unroll
  for (int i = 0; i < kW; i++) h.v[i] = f.v[i];
}
CB200_XHD void fe_set_words(Fe& h, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t w4, uint32_t w5,
                            uint32_t w6, uint32_t w7) {
  h.v[0] = w0, h.v[1] = w1, h.v[2] = w2, h.v[3] = w3, h.v[4] = w4, h.v[5] = w5, h.v[6] = w6, h.v[7] = w7;
}
CB200_XHD void fe_zero(Fe& h) { fe_set_words(h, 0, 0, 0, 0, 0, 0, 0, 0); }
CB200_XHD void fe_one(Fe& h) {  // R mod p
  fe_set_words(h, 1u, 0u, 0u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xfffffffeu, 0u);
}
CB200_XHD void fe_b(Fe& h) {  // b R mod p
  fe_set_words(h, 0x29c4bddfu, 0xd89cdf62u, 0x78843090u, 0xacf005cdu, 0xf7212ed6u, 0xe5a220abu, 0x04874834u, 0xdc30061du);
}
CB200_XHD void fe_r2(Fe& h) {  // R^2 mod p
  fe_set_words(h, 3u, 0u, 0xffffffffu, 0xfffffffbu, 0xfffffffeu, 0xffffffffu, 0xfffffffdu, 4u);
}

// h = t + hi 2^256 - p if that is >= 0, else t (t + hi 2^256 < 2p)
CB200_XHD void fe_reduce_once(Fe& h, const uint32_t (&t)[kW], uint32_t hi) {
  uint32_t u[kW];
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t d = (uint64_t)t[i] - p_word(i) - borrow;
    u[i] = (uint32_t)d;
    borrow = (uint32_t)(d >> 32) & 1u;
  }
  const uint32_t take = 0u - ((hi | (borrow ^ 1u)) & 1u);  // all ones: subtract
#pragma unroll
  for (int i = 0; i < kW; i++) h.v[i] = (u[i] & take) | (t[i] & ~take);
}
CB200_XHD void fe_add(Fe& h, const Fe& f, const Fe& g) {
  uint32_t t[kW];
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    c += (uint64_t)f.v[i] + g.v[i];
    t[i] = (uint32_t)c;
    c >>= 32;
  }
  fe_reduce_once(h, t, (uint32_t)c);
}
CB200_XHD void fe_sub(Fe& h, const Fe& f, const Fe& g) {
  uint32_t t[kW];
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t d = (uint64_t)f.v[i] - g.v[i] - borrow;
    t[i] = (uint32_t)d;
    borrow = (uint32_t)(d >> 32) & 1u;
  }
  const uint32_t m = 0u - borrow;  // add p back after a borrow
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    c += (uint64_t)t[i] + (p_word(i) & m);
    h.v[i] = (uint32_t)c;
    c >>= 32;
  }
}
CB200_XHD void fe_neg(Fe& h, const Fe& f) {
  Fe z;
  fe_zero(z);
  fe_sub(h, z, f);
}

// h = t R^-1 mod p for t < p 2^256 (16 words): eight steps of t += t[i] p 2^(32 i), each clearing word i
CB200_XHD void fe_mont_reduce(Fe& h, uint32_t (&t)[2 * kW]) {
  uint32_t top = 0;  // the bit above word 15
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint32_t m = t[i];
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < kW; j++) {
      c += (uint64_t)t[i + j] + (uint64_t)m * p_word(j);
      t[i + j] = (uint32_t)c;
      c >>= 32;
    }
#pragma unroll
    for (int j = i + kW; j < 2 * kW; j++) {
      c += t[j];
      t[j] = (uint32_t)c;
      c >>= 32;
    }
    top += (uint32_t)c;
  }
  uint32_t r[kW];
#pragma unroll
  for (int i = 0; i < kW; i++) r[i] = t[kW + i];
  fe_reduce_once(h, r, top);
}
CB200_XHD void fe_mul(Fe& h, const Fe& f, const Fe& g) {
  uint32_t t[2 * kW];
#pragma unroll
  for (int i = 0; i < 2 * kW; i++) t[i] = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < kW; j++) {
      c += (uint64_t)t[i + j] + (uint64_t)f.v[i] * g.v[j];
      t[i + j] = (uint32_t)c;
      c >>= 32;
    }
    t[i + kW] = (uint32_t)c;
  }
  fe_mont_reduce(h, t);
}
// squaring: the 28 cross products once, doubled, plus the 8 squares
CB200_XHD void fe_sqr(Fe& h, const Fe& f) {
  uint32_t t[2 * kW];
#pragma unroll
  for (int i = 0; i < 2 * kW; i++) t[i] = 0;
#pragma unroll
  for (int i = 0; i < kW - 1; i++) {
    uint64_t c = 0;
#pragma unroll
    for (int j = i + 1; j < kW; j++) {
      c += (uint64_t)t[i + j] + (uint64_t)f.v[i] * f.v[j];
      t[i + j] = (uint32_t)c;
      c >>= 32;
    }
    t[i + kW] = (uint32_t)c;
  }
  uint32_t carry = 0;
#pragma unroll
  for (int i = 0; i < 2 * kW; i++) {
    const uint32_t v = t[i];
    t[i] = (v << 1) | carry;
    carry = v >> 31;
  }
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t s = (uint64_t)f.v[i] * f.v[i];
    c += (uint64_t)t[2 * i] + (uint32_t)s;
    t[2 * i] = (uint32_t)c;
    c >>= 32;
    c += (uint64_t)t[2 * i + 1] + (uint32_t)(s >> 32);
    t[2 * i + 1] = (uint32_t)c;
    c >>= 32;
  }
  fe_mont_reduce(h, t);
}
CB200_XHD void fe_sqr_n(Fe& h, const Fe& f, int k) {
  fe_sqr(h, f);
  for (int i = 1; i < k; i++) fe_sqr(h, h);
}
// h = f^(p - 2) = f^-1 (0 for f = 0).  p - 2 = 2^256 - 2^224 + 2^192 + 2^96 - 3: the words of p - 2 from the top are
// ffffffff 00000001 00000000 00000000 00000000 ffffffff ffffffff fffffffd; x_k below is f^(2^k - 1).
CB200_XHD_NOINLINE void fe_invert(Fe& h, const Fe& f) {
  Fe x2, x3, x6, x12, x15, x30, x32, t;
  fe_sqr(t, f);
  fe_mul(x2, t, f);
  fe_sqr(t, x2);
  fe_mul(x3, t, f);
  fe_sqr_n(t, x3, 3);
  fe_mul(x6, t, x3);
  fe_sqr_n(t, x6, 6);
  fe_mul(x12, t, x6);
  fe_sqr_n(t, x12, 3);
  fe_mul(x15, t, x3);
  fe_sqr_n(t, x15, 15);
  fe_mul(x30, t, x15);
  fe_sqr_n(t, x30, 2);
  fe_mul(x32, t, x2);
  fe_sqr_n(t, x32, 32);  // ffffffff 00000000
  fe_mul(t, t, f);       // ffffffff 00000001
  fe_sqr_n(t, t, 128);
  fe_mul(t, t, x32);  // ffffffff 00000001 00000000 00000000 00000000 ffffffff
  fe_sqr_n(t, t, 32);
  fe_mul(t, t, x32);  // ... ffffffff ffffffff
  fe_sqr_n(t, t, 30);
  fe_mul(t, t, x30);  // ... ffffffff fffffffc
  fe_sqr_n(t, t, 2);
  fe_mul(h, t, f);  // ... ffffffff fffffffd
}
CB200_XHD void fe_to_mont(Fe& h, const Fe& f) {
  Fe r2;
  fe_r2(r2);
  fe_mul(h, f, r2);
}
CB200_XHD void fe_from_mont(Fe& h, const Fe& f) {
  uint32_t t[2 * kW];
#pragma unroll
  for (int i = 0; i < kW; i++) t[i] = f.v[i], t[kW + i] = 0;
  fe_mont_reduce(h, t);
}
// h = f if mask = 0, g if mask = all ones
CB200_XHD void fe_select(Fe& h, const Fe& f, const Fe& g, uint32_t mask) {
#pragma unroll
  for (int i = 0; i < kW; i++) h.v[i] = (f.v[i] & ~mask) | (g.v[i] & mask);
}
// all ones iff f = g
CB200_XHD uint32_t fe_eq(const Fe& f, const Fe& g) {
  uint32_t d = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) d |= f.v[i] ^ g.v[i];
  return (uint32_t)(((uint64_t)d - 1) >> 32);
}

// big-endian bytes <-> little-endian words; a row may start at any byte
CB200_XHD void words_from_be(uint32_t (&w)[kW], const uint8_t* b) {
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint8_t* q = b + 4 * (kW - 1 - i);
    w[i] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
  }
}
CB200_XHD void words_to_be(uint8_t* b, const uint32_t (&w)[kW], uint32_t mask) {
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint32_t v = w[i] & mask;
    uint8_t* q = b + 4 * (kW - 1 - i);
    q[0] = (uint8_t)(v >> 24), q[1] = (uint8_t)(v >> 16), q[2] = (uint8_t)(v >> 8), q[3] = (uint8_t)v;
  }
}
// all ones iff a < m (a, m little-endian words); constant time
CB200_XHD uint32_t lt_words(const uint32_t (&a)[kW], const uint32_t (&m)[kW]) {
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) borrow = (uint32_t)((((uint64_t)a[i] - m[i] - borrow) >> 32) & 1u);
  return 0u - borrow;
}

// ---------------------------------------------------------------- validation (NewPrivateKey / NewPublicKey)
// all ones iff 0 < k < n
CB200_XHD uint32_t scalar_ok(const uint32_t (&k)[kW]) {
  const uint32_t n[kW] = CB200_P256_N;
  uint32_t nz = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) nz |= k[i];
  return lt_words(k, n) & (0u - (uint32_t)(nz != 0));
}
// Parses 0x04 || X || Y (65 bytes).  Returns all ones iff the prefix is 0x04, X < p, Y < p and the point is on the
// curve; P then holds it in Montgomery form.  Public data: the result may be branched on.
CB200_XHD uint32_t point_decode(Aff& P, const uint8_t* b) {
  const uint32_t p[kW] = CB200_P256_P;
  uint32_t x[kW], y[kW];
  words_from_be(x, b + 1);
  words_from_be(y, b + 33);
  uint32_t ok = (0u - (uint32_t)(b[0] == 4)) & lt_words(x, p) & lt_words(y, p);
  Fe fx, fy, rhs, lhs, t;
#pragma unroll
  for (int i = 0; i < kW; i++) fx.v[i] = x[i], fy.v[i] = y[i];
  fe_to_mont(P.x, fx);
  fe_to_mont(P.y, fy);
  // y^2 = x^3 - 3x + b = (x^2 - 3) x + b
  fe_sqr(lhs, P.y);
  fe_sqr(t, P.x);
  Fe three;
  fe_one(three);
  fe_add(rhs, three, three);
  fe_add(three, rhs, three);
  fe_sub(t, t, three);
  fe_mul(rhs, t, P.x);
  fe_b(t);
  fe_add(rhs, rhs, t);
  return ok & fe_eq(lhs, rhs);
}

// ---------------------------------------------------------------- group law (ePrint 2015/1060, a = -3)
CB200_XHD void pt_identity(Pt& r) {
  fe_zero(r.X);
  fe_one(r.Y);
  fe_zero(r.Z);
}
// algorithm 4: r = p + q (r may alias p or q)
CB200_XHD void pt_add(Pt& r, const Pt& p, const Pt& q) {
  Fe t0, t1, t2, t3, t4, X3, Y3, Z3, b;
  fe_b(b);
  fe_mul(t0, p.X, q.X);
  fe_mul(t1, p.Y, q.Y);
  fe_mul(t2, p.Z, q.Z);
  fe_add(t3, p.X, p.Y);
  fe_add(t4, q.X, q.Y);
  fe_mul(t3, t3, t4);
  fe_add(t4, t0, t1);
  fe_sub(t3, t3, t4);
  fe_add(t4, p.Y, p.Z);
  fe_add(X3, q.Y, q.Z);
  fe_mul(t4, t4, X3);
  fe_add(X3, t1, t2);
  fe_sub(t4, t4, X3);
  fe_add(X3, p.X, p.Z);
  fe_add(Y3, q.X, q.Z);
  fe_mul(X3, X3, Y3);
  fe_add(Y3, t0, t2);
  fe_sub(Y3, X3, Y3);
  fe_mul(Z3, b, t2);
  fe_sub(X3, Y3, Z3);
  fe_add(Z3, X3, X3);
  fe_add(X3, X3, Z3);
  fe_sub(Z3, t1, X3);
  fe_add(X3, t1, X3);
  fe_mul(Y3, b, Y3);
  fe_add(t1, t2, t2);
  fe_add(t2, t1, t2);
  fe_sub(Y3, Y3, t2);
  fe_sub(Y3, Y3, t0);
  fe_add(t1, Y3, Y3);
  fe_add(Y3, t1, Y3);
  fe_add(t1, t0, t0);
  fe_add(t0, t1, t0);
  fe_sub(t0, t0, t2);
  fe_mul(t1, t4, Y3);
  fe_mul(t2, t0, Y3);
  fe_mul(Y3, X3, Z3);
  fe_add(Y3, Y3, t2);
  fe_mul(X3, t3, X3);
  fe_sub(X3, X3, t1);
  fe_mul(Z3, t4, Z3);
  fe_mul(t1, t3, t0);
  fe_add(Z3, Z3, t1);
  fe_copy(r.X, X3);
  fe_copy(r.Y, Y3);
  fe_copy(r.Z, Z3);
}
// algorithm 5: r = p + q for an affine q (which cannot be the identity)
CB200_XHD void pt_add_affine(Pt& r, const Pt& p, const Aff& q) {
  Fe t0, t1, t2, t3, t4, X3, Y3, Z3, b;
  fe_b(b);
  fe_mul(t0, p.X, q.x);
  fe_mul(t1, p.Y, q.y);
  fe_add(t3, q.x, q.y);
  fe_add(t4, p.X, p.Y);
  fe_mul(t3, t3, t4);
  fe_add(t4, t0, t1);
  fe_sub(t3, t3, t4);
  fe_mul(t4, q.y, p.Z);
  fe_add(t4, t4, p.Y);
  fe_mul(Y3, q.x, p.Z);
  fe_add(Y3, Y3, p.X);
  fe_mul(Z3, b, p.Z);
  fe_sub(X3, Y3, Z3);
  fe_add(Z3, X3, X3);
  fe_add(X3, X3, Z3);
  fe_sub(Z3, t1, X3);
  fe_add(X3, t1, X3);
  fe_mul(Y3, b, Y3);
  fe_add(t1, p.Z, p.Z);
  fe_add(t2, t1, p.Z);
  fe_sub(Y3, Y3, t2);
  fe_sub(Y3, Y3, t0);
  fe_add(t1, Y3, Y3);
  fe_add(Y3, t1, Y3);
  fe_add(t1, t0, t0);
  fe_add(t0, t1, t0);
  fe_sub(t0, t0, t2);
  fe_mul(t1, t4, Y3);
  fe_mul(t2, t0, Y3);
  fe_mul(Y3, X3, Z3);
  fe_add(Y3, Y3, t2);
  fe_mul(X3, t3, X3);
  fe_sub(X3, X3, t1);
  fe_mul(Z3, t4, Z3);
  fe_mul(t1, t3, t0);
  fe_add(Z3, Z3, t1);
  fe_copy(r.X, X3);
  fe_copy(r.Y, Y3);
  fe_copy(r.Z, Z3);
}
// algorithm 6: r = 2 p
CB200_XHD void pt_dbl(Pt& r, const Pt& p) {
  Fe t0, t1, t2, t3, X3, Y3, Z3, b;
  fe_b(b);
  fe_sqr(t0, p.X);
  fe_sqr(t1, p.Y);
  fe_sqr(t2, p.Z);
  fe_mul(t3, p.X, p.Y);
  fe_add(t3, t3, t3);
  fe_mul(Z3, p.X, p.Z);
  fe_add(Z3, Z3, Z3);
  fe_mul(Y3, b, t2);
  fe_sub(Y3, Y3, Z3);
  fe_add(X3, Y3, Y3);
  fe_add(Y3, X3, Y3);
  fe_sub(X3, t1, Y3);
  fe_add(Y3, t1, Y3);
  fe_mul(Y3, X3, Y3);
  fe_mul(X3, X3, t3);
  fe_add(t3, t2, t2);
  fe_add(t2, t2, t3);
  fe_mul(Z3, b, Z3);
  fe_sub(Z3, Z3, t2);
  fe_sub(Z3, Z3, t0);
  fe_add(t3, Z3, Z3);
  fe_add(Z3, Z3, t3);
  fe_add(t3, t0, t0);
  fe_add(t0, t3, t0);
  fe_sub(t0, t0, t2);
  fe_mul(t0, t0, Z3);
  fe_add(Y3, Y3, t0);
  fe_mul(t0, p.Y, p.Z);
  fe_add(t0, t0, t0);
  fe_mul(Z3, t0, Z3);
  fe_sub(X3, X3, Z3);
  fe_mul(Z3, t0, t1);
  fe_add(Z3, Z3, Z3);
  fe_add(Z3, Z3, Z3);
  fe_copy(r.X, X3);
  fe_copy(r.Y, Y3);
  fe_copy(r.Z, Z3);
}
// r = p when mask = all ones (r unchanged otherwise)
CB200_XHD void pt_cmov(Pt& r, const Pt& p, uint32_t mask) {
  fe_select(r.X, r.X, p.X, mask);
  fe_select(r.Y, r.Y, p.Y, mask);
  fe_select(r.Z, r.Z, p.Z, mask);
}
// affine coordinates in plain (non-Montgomery) form; the identity gives (0, 0)
CB200_XHD void pt_to_affine(Fe& x, Fe& y, const Pt& p) {
  Fe zi, t;
  fe_invert(zi, p.Z);
  fe_mul(t, p.X, zi);
  fe_from_mont(x, t);
  fe_mul(t, p.Y, zi);
  fe_from_mont(y, t);
}

// ---------------------------------------------------------------- scalar recoding
// For 0 < k < n: k' = min-style choice of k or n - k, whichever is below 2^255 (n < 2^256, so one of them is), and
// flip = all ones when n - k was taken ([k]P = -[n - k]P).  k' is then written as 64 signed radix-16 digits
// d_0..d_63 with d_i in [-8, 7] for i < 63 and d_63 in [0, 8] (the x25519.cuh recoding): the nibbles of
// k' + 0x88...8, minus 8, with the carry out of the top nibble kept in d_63.  All of it by masks.
struct Digits {
  uint32_t k[kW];  // k' + 0x88...8
  uint32_t carry;
};
CB200_XHD uint32_t recode(Digits& d, const uint32_t (&k)[kW]) {
  const uint32_t n[kW] = CB200_P256_N;
  uint32_t nk[kW];
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t t = (uint64_t)n[i] - k[i] - borrow;
    nk[i] = (uint32_t)t;
    borrow = (uint32_t)(t >> 32) & 1u;
  }
  const uint32_t flip = 0u - (k[kW - 1] >> 31);
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    c += (uint64_t)((k[i] & ~flip) | (nk[i] & flip)) + 0x88888888u;
    d.k[i] = (uint32_t)c;
    c >>= 32;
  }
  d.carry = (uint32_t)c;
  return flip;
}
// digit i, as (|d_i| in 0..8, all ones when d_i < 0); i is a loop counter, not secret
CB200_XHD void digit(const Digits& d, int i, uint32_t& mag, uint32_t& neg) {
  uint32_t word = d.k[0];
#pragma unroll
  for (int q = 1; q < kW; q++) word = ((i >> 3) == q) ? d.k[q] : word;
  int e = (int)((word >> (4 * (i & 7))) & 15) - 8;
  if (i == 63) e += 16 * (int)d.carry;
  neg = (uint32_t)(e >> 31);
  mag = ((uint32_t)e ^ neg) - neg;
}
// all ones iff a == b (small values)
CB200_XHD uint32_t eq_mask(uint32_t a, uint32_t b) { return (uint32_t)((int32_t)((a ^ b) - 1u) >> 31); }

// ---------------------------------------------------------------- variable base: r = [k] P, 0 < k < n
// The multiples 1..8 P sit in `tab` (local memory on the device); every entry is read for every digit and the one
// wanted -- or the identity for digit 0 -- kept by masks, then Y is negated by mask for a negative digit.
CB200_XHD void scalarmult(Pt& r, const uint32_t (&k)[kW], const Aff& P) {
  Pt tab[8];
  fe_copy(tab[0].X, P.x);
  fe_copy(tab[0].Y, P.y);
  fe_one(tab[0].Z);
  pt_dbl(tab[1], tab[0]);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int j = 2; j < 8; j++) pt_add(tab[j], tab[j - 1], tab[0]);
  Digits d;
  const uint32_t flip = recode(d, k);
  auto pick = [&](Pt& s, int i) {
    uint32_t mag, neg;
    digit(d, i, mag, neg);
    pt_identity(s);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int j = 0; j < 8; j++) pt_cmov(s, tab[j], eq_mask(mag, (uint32_t)(j + 1)));
    Fe ny;
    fe_neg(ny, s.Y);
    fe_select(s.Y, s.Y, ny, neg);
  };
  pick(r, 63);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 62; i >= 0; i--) {
    pt_dbl(r, r);
    pt_dbl(r, r);
    pt_dbl(r, r);
    pt_dbl(r, r);
    Pt s;
    pick(s, i);
    pt_add(r, r, s);
  }
  Fe ny;
  fe_neg(ny, r.Y);
  fe_select(r.Y, r.Y, ny, flip);
}

// ---------------------------------------------------------------- fixed base: r = [k] G, 0 < k < n
// table[i][j] = (j + 1) 16^i G in affine Montgomery form: 64 rows of 8 entries of 16 words (32 KiB).
constexpr int kTableWords = 64 * 8 * 16;
CB200_XHD void table_entry(Aff& a, const uint32_t* __restrict__ w) {
#pragma unroll
  for (int c = 0; c < kW; c++) a.x.v[c] = w[c], a.y.v[c] = w[kW + c];
}
// Every digit costs one complete mixed addition; for digit 0 its result is dropped by mask.  As in the variable-base
// case, the eight entries of a row are all read, so no address depends on the scalar.
CB200_XHD void scalarmult_base(Pt& r, const uint32_t (&k)[kW], const uint32_t* __restrict__ table) {
  Digits d;
  const uint32_t flip = recode(d, k);
  pt_identity(r);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 0; i < 64; i++) {
    uint32_t mag, neg;
    digit(d, i, mag, neg);
    Aff q;
    table_entry(q, table + i * 8 * 16);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int j = 1; j < 8; j++) {
      Aff e;
      table_entry(e, table + (i * 8 + j) * 16);
      const uint32_t m = eq_mask(mag, (uint32_t)(j + 1));
      fe_select(q.x, q.x, e.x, m);
      fe_select(q.y, q.y, e.y, m);
    }
    Fe ny;
    fe_neg(ny, q.y);
    fe_select(q.y, q.y, ny, neg ^ flip);
    Pt s;
    pt_add_affine(s, r, q);
    pt_cmov(r, s, ~eq_mask(mag, 0));
  }
}

// ---------------------------------------------------------------- the two operations on byte rows
// Rows are big-endian and may start at any byte.  The result is a status: bit 0 = the point is not a valid public
// key, bit 1 = the scalar is not a valid private key; a failed operation writes an all-zero output row.

// out = 0x04 || X || Y of [k]G (65 bytes): ecdh.PrivateKey.PublicKey
CB200_XHD uint32_t keygen(uint8_t* out, const uint8_t* sk, const uint32_t* __restrict__ table) {
  uint32_t k[kW];
  words_from_be(k, sk);
  const uint32_t ok = scalar_ok(k);
  Pt r;
  scalarmult_base(r, k, table);
  Fe x, y;
  pt_to_affine(x, y, r);
  out[0] = (uint8_t)(4u & ok);
  words_to_be(out + 1, x.v, ok);
  words_to_be(out + 33, y.v, ok);
  return ok ? 0u : 2u;
}
// out = X of [k]P (32 bytes): ecdh.PrivateKey.ECDH after NewPublicKey(P)
CB200_XHD uint32_t shared(uint8_t* out, const uint8_t* sk, const uint8_t* pt) {
  uint32_t k[kW];
  words_from_be(k, sk);
  Aff P;
  const uint32_t pok = point_decode(P, pt), kok = scalar_ok(k);
  Pt r;
  scalarmult(r, k, P);
  Fe x, y;
  pt_to_affine(x, y, r);
  words_to_be(out, x.v, pok & kok);
  return (pok ? 0u : 1u) | (kok ? 0u : 2u);
}

// Host side, once per process: the fixed-base table.
inline void build_base_table(uint32_t* table) {
  Fe gx, gy;
  fe_set_words(gx, 0xd898c296u, 0xf4a13945u, 0x2deb33a0u, 0x77037d81u, 0x63a440f2u, 0xf8bce6e5u, 0xe12c4247u, 0x6b17d1f2u);
  fe_set_words(gy, 0x37bf51f5u, 0xcbb64068u, 0x6b315eceu, 0x2bce3357u, 0x7c0f9e16u, 0x8ee7eb4au, 0xfe1a7f9bu, 0x4fe342e2u);
  Pt P;
  fe_to_mont(P.X, gx);
  fe_to_mont(P.Y, gy);
  fe_one(P.Z);
  for (int i = 0; i < 64; i++) {
    Pt M = P;
    for (int j = 0; j < 8; j++) {
      if (j > 0) pt_add(M, M, P);
      Fe x, y, zi;
      fe_invert(zi, M.Z);
      fe_mul(x, M.X, zi);
      fe_mul(y, M.Y, zi);
      uint32_t* w = table + (i * 8 + j) * 16;
      for (int c = 0; c < kW; c++) w[c] = x.v[c], w[kW + c] = y.v[c];
    }
    for (int q = 0; q < 4; q++) pt_dbl(P, P);
  }
}

#undef CB200_P256_P
#undef CB200_P256_N

}  // namespace p256
}  // namespace cb200
