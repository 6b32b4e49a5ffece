// The NIST prime curves y^2 = x^3 - 3x + b over GF(p) -- P-256, P-384 and P-521 -- on one thread, generic over a curve
// type C (p256.cuh, p384.cuh, p521.cuh define one each).
//
// Mirrors what Go's crypto/ecdh computes for the reference's NIST DHKEMs (hpke/shortkem.go): KeyGen = 0x04 || X || Y of
// [k]G and Shared = X of [k]P, big-endian rows of ceil(bits / 8) bytes per coordinate, for 0 < k < n; NewPublicKey's
// and NewPrivateKey's validation rules (the point on the curve with coordinates below p; 0 < k < n).
//
// Field: C::kW 32-bit words in Montgomery form (R = 2^(32 kW)), fully reduced into [0, p) after every operation.  All
// three primes are -1 mod 2^32, so the Montgomery factor of each reduction step is the low word itself, and a product
// by a word of p that is 0, 1 or 2^32 - 1 folds into additions and subtractions.  Products accumulate in 64 bits (one
// IMAD.WIDE per word product on sm_90a).  Inversion is Fermat's, by a fixed addition chain for p - 2 per curve.
//
// Group: projective (X : Y : Z) with the complete formulas of Renes, Costello and Batina for a = -3 (ePrint 2015/1060,
// algorithms 4, 5 and 6).  They have no exceptional case -- the identity (0 : 1 : 0), doublings and inverse pairs
// included -- so no branch depends on a point or a scalar.
//
// A curve type C supplies:
//   kW, kBytes, kDigits    words of an element, bytes of a row (ceil(bits / 8)), signed radix-16 digits of a scalar
//   kFlipWord, kFlipShift  the position of bit bitlen(n) - 1 of a scalar
//   kOutlineMul            the field product and square are calls rather than inlined (see fe_mul)
//   p(i) n(i) b(i) one(i) r2(i) gx(i) gy(i)
//                          word i of p, n, b R mod p, R mod p, R^2 mod p and of G (plain, not Montgomery)
//   invert(h, f)           h = f^(p - 2)
//
// Plain integer C++ like x25519.cuh: it compiles for the device (kernels), for the host inside the library (the
// fixed-base tables are computed once at cb200_init) and for the host-only tests of the CPU suite.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define CB200_XHD __host__ __device__ __forceinline__
#define CB200_XHD_NOINLINE static __host__ __device__ __noinline__
#else
#define CB200_XHD inline
#define CB200_XHD_NOINLINE inline
#endif
// a curve type's static member functions that stay calls (the inversion chains)
#if defined(__CUDACC__)
#define CB200_NISTP_NOINLINE static __host__ __device__ __noinline__
#else
#define CB200_NISTP_NOINLINE static inline
#endif

namespace cb200 {
namespace nistp {

template <class C>
struct Fe {
  uint32_t v[C::kW];
};
template <class C>
struct Pt {  // projective (X : Y : Z), Montgomery form
  Fe<C> X, Y, Z;
};
template <class C>
struct Aff {  // affine (x, y), Montgomery form
  Fe<C> x, y;
};

template <class C>
CB200_XHD void fe_copy(Fe<C>& h, const Fe<C>& f) {
#pragma unroll
  for (int i = 0; i < C::kW; i++) h.v[i] = f.v[i];
}
template <class C>
CB200_XHD void fe_zero(Fe<C>& h) {
#pragma unroll
  for (int i = 0; i < C::kW; i++) h.v[i] = 0;
}
template <class C>
CB200_XHD void fe_one(Fe<C>& h) {  // R mod p
#pragma unroll
  for (int i = 0; i < C::kW; i++) h.v[i] = C::one(i);
}
template <class C>
CB200_XHD void fe_b(Fe<C>& h) {  // b R mod p
#pragma unroll
  for (int i = 0; i < C::kW; i++) h.v[i] = C::b(i);
}
template <class C>
CB200_XHD void fe_r2(Fe<C>& h) {  // R^2 mod p
#pragma unroll
  for (int i = 0; i < C::kW; i++) h.v[i] = C::r2(i);
}

// h = t + hi 2^(32 kW) - p if that is >= 0, else t (t + hi 2^(32 kW) < 2p)
template <class C>
CB200_XHD void fe_reduce_once(Fe<C>& h, const uint32_t (&t)[C::kW], uint32_t hi) {
  constexpr int kW = C::kW;
  uint32_t u[kW];
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t d = (uint64_t)t[i] - C::p(i) - borrow;
    u[i] = (uint32_t)d;
    borrow = (uint32_t)(d >> 32) & 1u;
  }
  const uint32_t take = 0u - ((hi | (borrow ^ 1u)) & 1u);  // all ones: subtract
#pragma unroll
  for (int i = 0; i < kW; i++) h.v[i] = (u[i] & take) | (t[i] & ~take);
}
template <class C>
CB200_XHD void fe_add(Fe<C>& h, const Fe<C>& f, const Fe<C>& g) {
  constexpr int kW = C::kW;
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
template <class C>
CB200_XHD void fe_sub(Fe<C>& h, const Fe<C>& f, const Fe<C>& g) {
  constexpr int kW = C::kW;
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
    c += (uint64_t)t[i] + (C::p(i) & m);
    h.v[i] = (uint32_t)c;
    c >>= 32;
  }
}
template <class C>
CB200_XHD void fe_neg(Fe<C>& h, const Fe<C>& f) {
  Fe<C> z;
  fe_zero(z);
  fe_sub(h, z, f);
}

// h = t R^-1 mod p for t < p R (2 kW words): kW steps of t += t[i] p 2^(32 i), each clearing word i
template <class C>
CB200_XHD void fe_mont_reduce(Fe<C>& h, uint32_t (&t)[2 * C::kW]) {
  constexpr int kW = C::kW;
  uint32_t top = 0;  // the bit above word 2 kW - 1
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint32_t m = t[i];
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < kW; j++) {
      c += (uint64_t)t[i + j] + (uint64_t)m * C::p(j);
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
template <class C>
CB200_XHD void fe_mul_inl(Fe<C>& h, const Fe<C>& f, const Fe<C>& g) {
  constexpr int kW = C::kW;
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
// squaring: the kW (kW - 1) / 2 cross products once, doubled, plus the kW squares
template <class C>
CB200_XHD void fe_sqr_inl(Fe<C>& h, const Fe<C>& f) {
  constexpr int kW = C::kW;
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
// A curve with kOutlineMul set (P-384, P-521) calls one copy of the product and the square instead of inlining them at
// every use: their 12- and 17-word bodies, inlined into the ladders, make kernels that take ptxas many minutes.  P-256
// inlines them.
template <class C>
CB200_NISTP_NOINLINE void fe_mul_out(Fe<C>& h, const Fe<C>& f, const Fe<C>& g) {
  fe_mul_inl(h, f, g);
}
template <class C>
CB200_NISTP_NOINLINE void fe_sqr_out(Fe<C>& h, const Fe<C>& f) {
  fe_sqr_inl(h, f);
}
template <class C>
CB200_XHD void fe_mul(Fe<C>& h, const Fe<C>& f, const Fe<C>& g) {
  if constexpr (C::kOutlineMul)
    fe_mul_out(h, f, g);
  else
    fe_mul_inl(h, f, g);
}
template <class C>
CB200_XHD void fe_sqr(Fe<C>& h, const Fe<C>& f) {
  if constexpr (C::kOutlineMul)
    fe_sqr_out(h, f);
  else
    fe_sqr_inl(h, f);
}
template <class C>
CB200_XHD void fe_sqr_n(Fe<C>& h, const Fe<C>& f, int k) {
  fe_sqr(h, f);
  for (int i = 1; i < k; i++) fe_sqr(h, h);
}
// h = f^(p - 2) = f^-1 (0 for f = 0), by the curve's addition chain
template <class C>
CB200_XHD void fe_invert(Fe<C>& h, const Fe<C>& f) {
  C::invert(h, f);
}
template <class C>
CB200_XHD void fe_to_mont(Fe<C>& h, const Fe<C>& f) {
  Fe<C> r2;
  fe_r2(r2);
  fe_mul(h, f, r2);
}
template <class C>
CB200_XHD void fe_from_mont(Fe<C>& h, const Fe<C>& f) {
  constexpr int kW = C::kW;
  uint32_t t[2 * kW];
#pragma unroll
  for (int i = 0; i < kW; i++) t[i] = f.v[i], t[kW + i] = 0;
  fe_mont_reduce(h, t);
}
// h = f if mask = 0, g if mask = all ones
template <class C>
CB200_XHD void fe_select(Fe<C>& h, const Fe<C>& f, const Fe<C>& g, uint32_t mask) {
#pragma unroll
  for (int i = 0; i < C::kW; i++) h.v[i] = (f.v[i] & ~mask) | (g.v[i] & mask);
}
// all ones iff f = g
template <class C>
CB200_XHD uint32_t fe_eq(const Fe<C>& f, const Fe<C>& g) {
  uint32_t d = 0;
#pragma unroll
  for (int i = 0; i < C::kW; i++) d |= f.v[i] ^ g.v[i];
  return (uint32_t)(((uint64_t)d - 1) >> 32);
}

// Big-endian rows of C::kBytes bytes <-> little-endian words; a row may start at any byte.  When kBytes is not a
// multiple of 4 (P-521's 66), the top word holds the leading kBytes mod 4 bytes and its excess high bits are zero.
template <class C>
CB200_XHD void words_from_be(uint32_t (&w)[C::kW], const uint8_t* b) {
  constexpr int kW = C::kW, kB = C::kBytes;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    if (4 * (i + 1) <= kB) {
      const uint8_t* q = b + kB - 4 * (i + 1);
      w[i] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    } else {
      uint32_t v = 0;
#pragma unroll
      for (int j = 0; j < kB - 4 * i; j++) v = (v << 8) | b[j];
      w[i] = v;
    }
  }
}
template <class C>
CB200_XHD void words_to_be(uint8_t* b, const uint32_t (&w)[C::kW], uint32_t mask) {
  constexpr int kW = C::kW, kB = C::kBytes;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint32_t v = w[i] & mask;
    if (4 * (i + 1) <= kB) {
      uint8_t* q = b + kB - 4 * (i + 1);
      q[0] = (uint8_t)(v >> 24), q[1] = (uint8_t)(v >> 16), q[2] = (uint8_t)(v >> 8), q[3] = (uint8_t)v;
    } else {
#pragma unroll
      for (int j = 0; j < kB - 4 * i; j++) b[j] = (uint8_t)(v >> (8 * (kB - 4 * i - 1 - j)));
    }
  }
}
// all ones iff a < m (a, m little-endian words); constant time
template <int kW>
CB200_XHD uint32_t lt_words(const uint32_t (&a)[kW], const uint32_t (&m)[kW]) {
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) borrow = (uint32_t)((((uint64_t)a[i] - m[i] - borrow) >> 32) & 1u);
  return 0u - borrow;
}

// ---------------------------------------------------------------- validation (NewPrivateKey / NewPublicKey)
// all ones iff 0 < k < n
template <class C>
CB200_XHD uint32_t scalar_ok(const uint32_t (&k)[C::kW]) {
  constexpr int kW = C::kW;
  uint32_t n[kW];
#pragma unroll
  for (int i = 0; i < kW; i++) n[i] = C::n(i);
  uint32_t nz = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) nz |= k[i];
  return lt_words(k, n) & (0u - (uint32_t)(nz != 0));
}
// Parses 0x04 || X || Y (1 + 2 kBytes bytes).  Returns all ones iff the prefix is 0x04, X < p, Y < p and the point is
// on the curve; P then holds it in Montgomery form.  Public data: the result may be branched on.
template <class C>
CB200_XHD uint32_t point_decode(Aff<C>& P, const uint8_t* b) {
  constexpr int kW = C::kW;
  uint32_t p[kW];
#pragma unroll
  for (int i = 0; i < kW; i++) p[i] = C::p(i);
  uint32_t x[kW], y[kW];
  words_from_be<C>(x, b + 1);
  words_from_be<C>(y, b + 1 + C::kBytes);
  uint32_t ok = (0u - (uint32_t)(b[0] == 4)) & lt_words(x, p) & lt_words(y, p);
  Fe<C> fx, fy, rhs, lhs, t;
#pragma unroll
  for (int i = 0; i < kW; i++) fx.v[i] = x[i], fy.v[i] = y[i];
  fe_to_mont(P.x, fx);
  fe_to_mont(P.y, fy);
  // y^2 = x^3 - 3x + b = (x^2 - 3) x + b
  fe_sqr(lhs, P.y);
  fe_sqr(t, P.x);
  Fe<C> three;
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
template <class C>
CB200_XHD void pt_identity(Pt<C>& r) {
  fe_zero(r.X);
  fe_one(r.Y);
  fe_zero(r.Z);
}
// algorithm 4: r = p + q (r may alias p or q)
template <class C>
CB200_XHD void pt_add(Pt<C>& r, const Pt<C>& p, const Pt<C>& q) {
  Fe<C> t0, t1, t2, t3, t4, X3, Y3, Z3, b;
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
template <class C>
CB200_XHD void pt_add_affine(Pt<C>& r, const Pt<C>& p, const Aff<C>& q) {
  Fe<C> t0, t1, t2, t3, t4, X3, Y3, Z3, b;
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
template <class C>
CB200_XHD void pt_dbl(Pt<C>& r, const Pt<C>& p) {
  Fe<C> t0, t1, t2, t3, X3, Y3, Z3, b;
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
template <class C>
CB200_XHD void pt_cmov(Pt<C>& r, const Pt<C>& p, uint32_t mask) {
  fe_select(r.X, r.X, p.X, mask);
  fe_select(r.Y, r.Y, p.Y, mask);
  fe_select(r.Z, r.Z, p.Z, mask);
}
// affine coordinates in plain (non-Montgomery) form; the identity gives (0, 0)
template <class C>
CB200_XHD void pt_to_affine(Fe<C>& x, Fe<C>& y, const Pt<C>& p) {
  Fe<C> zi, t;
  fe_invert(zi, p.Z);
  fe_mul(t, p.X, zi);
  fe_from_mont(x, t);
  fe_mul(t, p.Y, zi);
  fe_from_mont(y, t);
}

// ---------------------------------------------------------------- scalar recoding
// For 0 < k < n: k' = k or n - k, whichever is below 2^(bitlen(n) - 1) (one of them is), and flip = all ones when
// n - k was taken ([k]P = -[n - k]P).  k' is then written as kDigits signed radix-16 digits d_0..d_(kDigits - 1), with
// d_i in [-8, 7] below the top digit: the nibbles of k' + 0x88...8 (kDigits nibbles of 8), minus 8, with the carry out
// of the word array kept for the top digit.  P-256 (64 digits) and P-384 (96) fill their words: k' < 2^255 / 2^383
// leaves the top digit in [0, 8], through that carry.  P-521's k' < 2^520 fills 130 nibbles whose top one can be 15,
// so it has a 131st digit (0 or 1) of its own and its last word adds 0x888, never carrying out.  All of it by masks.
template <class C>
struct Digits {
  uint32_t k[C::kW];  // k' + 0x88...8
  uint32_t carry;
};
// the word i of 0x88...8 (kDigits nibbles)
template <class C>
CB200_XHD constexpr uint32_t eights(int i) {
  return i < C::kDigits / 8 ? 0x88888888u : 0x88888888u & ((1u << (4 * (C::kDigits % 8))) - 1u);
}
template <class C>
CB200_XHD uint32_t recode(Digits<C>& d, const uint32_t (&k)[C::kW]) {
  constexpr int kW = C::kW;
  uint32_t nk[kW];
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t t = (uint64_t)C::n(i) - k[i] - borrow;
    nk[i] = (uint32_t)t;
    borrow = (uint32_t)(t >> 32) & 1u;
  }
  const uint32_t flip = 0u - ((k[C::kFlipWord] >> C::kFlipShift) & 1u);
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    c += (uint64_t)((k[i] & ~flip) | (nk[i] & flip)) + eights<C>(i);
    d.k[i] = (uint32_t)c;
    c >>= 32;
  }
  d.carry = (uint32_t)c;
  return flip;
}
// digit i, as (|d_i| in 0..8, all ones when d_i < 0); i is a loop counter, not secret
template <class C>
CB200_XHD void digit(const Digits<C>& d, int i, uint32_t& mag, uint32_t& neg) {
  uint32_t word = d.k[0];
#pragma unroll
  for (int q = 1; q < C::kW; q++) word = ((i >> 3) == q) ? d.k[q] : word;
  int e = (int)((word >> (4 * (i & 7))) & 15) - 8;
  if (i == C::kDigits - 1) e += 16 * (int)d.carry;
  neg = (uint32_t)(e >> 31);
  mag = ((uint32_t)e ^ neg) - neg;
}
// all ones iff a == b (small values)
CB200_XHD uint32_t eq_mask(uint32_t a, uint32_t b) { return (uint32_t)((int32_t)((a ^ b) - 1u) >> 31); }

// ---------------------------------------------------------------- variable base: r = [k] P, 0 < k < n
// The multiples 1..8 P sit in `tab` (local memory on the device); every entry is read for every digit and the one
// wanted -- or the identity for digit 0 -- kept by masks, then Y is negated by mask for a negative digit.
template <class C>
CB200_XHD void scalarmult(Pt<C>& r, const uint32_t (&k)[C::kW], const Aff<C>& P) {
  Pt<C> tab[8];
  fe_copy(tab[0].X, P.x);
  fe_copy(tab[0].Y, P.y);
  fe_one(tab[0].Z);
  pt_dbl(tab[1], tab[0]);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int j = 2; j < 8; j++) pt_add(tab[j], tab[j - 1], tab[0]);
  Digits<C> d;
  const uint32_t flip = recode(d, k);
  auto pick = [&](Pt<C>& s, int i) {
    uint32_t mag, neg;
    digit(d, i, mag, neg);
    pt_identity(s);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int j = 0; j < 8; j++) pt_cmov(s, tab[j], eq_mask(mag, (uint32_t)(j + 1)));
    Fe<C> ny;
    fe_neg(ny, s.Y);
    fe_select(s.Y, s.Y, ny, neg);
  };
  pick(r, C::kDigits - 1);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = C::kDigits - 2; i >= 0; i--) {
    pt_dbl(r, r);
    pt_dbl(r, r);
    pt_dbl(r, r);
    pt_dbl(r, r);
    Pt<C> s;
    pick(s, i);
    pt_add(r, r, s);
  }
  Fe<C> ny;
  fe_neg(ny, r.Y);
  fe_select(r.Y, r.Y, ny, flip);
}

// ---------------------------------------------------------------- fixed base: r = [k] G, 0 < k < n
// table[i][j] = (j + 1) 16^i G in affine Montgomery form: kDigits rows of 8 entries of 2 kW words.
template <class C>
constexpr int kTableWords = C::kDigits * 8 * 2 * C::kW;
template <class C>
CB200_XHD void table_entry(Aff<C>& a, const uint32_t* __restrict__ w) {
#pragma unroll
  for (int c = 0; c < C::kW; c++) a.x.v[c] = w[c], a.y.v[c] = w[C::kW + c];
}
// Every digit costs one complete mixed addition; for digit 0 its result is dropped by mask.  As in the variable-base
// case, the eight entries of a row are all read, so no address depends on the scalar.
template <class C>
CB200_XHD void scalarmult_base(Pt<C>& r, const uint32_t (&k)[C::kW], const uint32_t* __restrict__ table) {
  constexpr int E = 2 * C::kW;  // words of a table entry
  Digits<C> d;
  const uint32_t flip = recode(d, k);
  pt_identity(r);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 0; i < C::kDigits; i++) {
    uint32_t mag, neg;
    digit(d, i, mag, neg);
    Aff<C> q;
    table_entry(q, table + i * 8 * E);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int j = 1; j < 8; j++) {
      Aff<C> e;
      table_entry(e, table + (i * 8 + j) * E);
      const uint32_t m = eq_mask(mag, (uint32_t)(j + 1));
      fe_select(q.x, q.x, e.x, m);
      fe_select(q.y, q.y, e.y, m);
    }
    Fe<C> ny;
    fe_neg(ny, q.y);
    fe_select(q.y, q.y, ny, neg ^ flip);
    Pt<C> s;
    pt_add_affine(s, r, q);
    pt_cmov(r, s, ~eq_mask(mag, 0));
  }
}

// ---------------------------------------------------------------- the two operations on byte rows
// Rows are big-endian and may start at any byte.  The result is a status: bit 0 = the point is not a valid public
// key, bit 1 = the scalar is not a valid private key; a failed operation writes an all-zero output row.

// out = 0x04 || X || Y of [k]G (1 + 2 kBytes bytes): ecdh.PrivateKey.PublicKey
template <class C>
CB200_XHD uint32_t keygen(uint8_t* out, const uint8_t* sk, const uint32_t* __restrict__ table) {
  uint32_t k[C::kW];
  words_from_be<C>(k, sk);
  const uint32_t ok = scalar_ok<C>(k);
  Pt<C> r;
  scalarmult_base(r, k, table);
  Fe<C> x, y;
  pt_to_affine(x, y, r);
  out[0] = (uint8_t)(4u & ok);
  words_to_be<C>(out + 1, x.v, ok);
  words_to_be<C>(out + 1 + C::kBytes, y.v, ok);
  return ok ? 0u : 2u;
}
// out = X of [k]P (kBytes bytes): ecdh.PrivateKey.ECDH after NewPublicKey(P)
template <class C>
CB200_XHD uint32_t shared(uint8_t* out, const uint8_t* sk, const uint8_t* pt) {
  uint32_t k[C::kW];
  words_from_be<C>(k, sk);
  Aff<C> P;
  const uint32_t pok = point_decode(P, pt), kok = scalar_ok<C>(k);
  Pt<C> r;
  scalarmult(r, k, P);
  Fe<C> x, y;
  pt_to_affine(x, y, r);
  words_to_be<C>(out, x.v, pok & kok);
  return (pok ? 0u : 1u) | (kok ? 0u : 2u);
}

// DeriveKeyPair's range test on one candidate (hpke/shortkem.go:63-90): byte(j), j < kBytes, is the candidate's
// byte j; byte 0 is ANDed with mask0 (shortkem.go's bitmask: 0xff for P-256 and P-384, 0x01 for P-521).  Leaves
// the masked candidate in k and returns all ones iff 0 < k < n.
template <class C, class B>
CB200_XHD uint32_t candidate(uint32_t (&k)[C::kW], const B& byte, uint8_t mask0) {
  constexpr int kW = C::kW, kB = C::kBytes;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    uint32_t v = 0;
#pragma unroll
    for (int j = kB - 4 * (i + 1) < 0 ? 0 : kB - 4 * (i + 1); j < kB - 4 * i; j++)
      v = (v << 8) | (j == 0 ? (uint8_t)(byte(0) & mask0) : byte(j));
    k[i] = v;
  }
  return scalar_ok<C>(k);
}

// Host side, once per process: the fixed-base table.  Each row of eight projective multiples goes to affine form with
// one inversion (Montgomery's trick).
template <class C>
inline void build_base_table(uint32_t* table) {
  constexpr int kW = C::kW;
  Fe<C> gx, gy;
  for (int c = 0; c < kW; c++) gx.v[c] = C::gx(c), gy.v[c] = C::gy(c);
  Pt<C> P;
  fe_to_mont(P.X, gx);
  fe_to_mont(P.Y, gy);
  fe_one(P.Z);
  for (int i = 0; i < C::kDigits; i++) {
    Pt<C> M[8];
    Fe<C> pre[8];  // pre[j] = Z_0 ... Z_j
    M[0] = P;
    for (int j = 1; j < 8; j++) pt_add(M[j], M[j - 1], P);
    pre[0] = M[0].Z;
    for (int j = 1; j < 8; j++) fe_mul(pre[j], pre[j - 1], M[j].Z);
    Fe<C> inv;  // (Z_0 ... Z_j)^-1, going down
    fe_invert(inv, pre[7]);
    for (int j = 7; j >= 0; j--) {
      Fe<C> zi, x, y;
      if (j > 0) {
        fe_mul(zi, inv, pre[j - 1]);
        fe_mul(inv, inv, M[j].Z);
      } else {
        zi = inv;
      }
      fe_mul(x, M[j].X, zi);
      fe_mul(y, M[j].Y, zi);
      uint32_t* w = table + (i * 8 + j) * 2 * kW;
      for (int c = 0; c < kW; c++) w[c] = x.v[c], w[kW + c] = y.v[c];
    }
    for (int q = 0; q < 4; q++) pt_dbl(P, P);
  }
}

}  // namespace nistp
}  // namespace cb200
