// RFC 9497 OPRF server arithmetic over the NIST curves (suites P256-SHA256, P384-SHA384, P521-SHA512), one thread per
// element or request, generic over nistp.cuh's curve types.  Mirrors the reference's oprf/{oprf,server,keys}.go,
// zk/dleq/dleq.go (the prover), group/short.go (compressed points, HashToElement, HashToScalar) and
// expander/expander.go (expand_message_xmd).
//
//   scalars mod n     Montgomery form with their own n0' (n is not -1 mod 2^32, unlike p); add, sub, mul, Fermat
//                     inversion by n - 2, and the reduction of a hash_to_field string (48, 72 or 98 bytes) mod n
//   compressed points 0x02 | 0x03 || X; decoding takes the square root as x^((p + 1) / 4) and rejects another prefix,
//                     X >= p and an X with no square root
//   hash_to_curve     expand_message_xmd, hash_to_field mod p and mod n, the simplified SWU map with sqrt_ratio for
//                     p = 3 mod 4 (RFC 9380 appendix F.2), straight-line: no branch depends on the input
//   DLEQ              ComputeComposites with the prover's shortcut Z = [k] M, and the challenge
//
// Every exponent here ((p - 3) / 4 and n - 2) is public and fixed, so square-and-multiply may branch on its bits.
// Secret values (k, t, t^-1, r, the FullEvaluate input) go through the masked multiplications of nistp.cuh and reach no
// branch or address.  A hash-derived scalar (a composite weight d_j, the challenge c) of 0 and a HashToGroup result at
// the identity each happen with probability below 2^-250; they take no path of their own.
//
// Plain integer C++ like nistp.cuh: it compiles for the device and for the host-only test of the CPU suite.
#pragma once
#include <cstdint>

#include "nistp.cuh"
#include "p256.cuh"
#include "p384.cuh"
#include "p521.cuh"
#include "sha2.cuh"

namespace cb200 {
namespace oprf {

using nistp::Aff;
using nistp::Fe;
using nistp::Pt;

// ---------------------------------------------------------------- the suites
template <class C>
struct Suite;
template <>
struct Suite<nistp::P256> {
  using H = sha2::Sha256;
  static constexpr int kL = 48, kIdLen = 11;
  CB200_XHD static const char* id() { return "P256-SHA256"; }
};
template <>
struct Suite<nistp::P384> {
  using H = sha2::Sha384;
  static constexpr int kL = 72, kIdLen = 11;
  CB200_XHD static const char* id() { return "P384-SHA384"; }
};
template <>
struct Suite<nistp::P521> {
  using H = sha2::Sha512;
  static constexpr int kL = 98, kIdLen = 11;
  CB200_XHD static const char* id() { return "P521-SHA512"; }
};
template <class C>
constexpr int kNe = 1 + C::kBytes;  // compressed element
template <class C>
constexpr int kNh = Suite<C>::H::kDigest;

// ---------------------------------------------------------------- scalars mod n (Montgomery, R = 2^(32 kW))
template <class C>
struct Sc {
  uint32_t v[C::kW];
};
template <class C>
CB200_XHD constexpr uint32_t n0inv() {  // -n^-1 mod 2^32
  uint32_t x = C::n(0);
  for (int i = 0; i < 5; i++) x *= 2u - C::n(0) * x;
  return 0u - x;
}
template <class C>
CB200_XHD void sc_reduce_once(Sc<C>& h, const uint32_t (&t)[C::kW], uint32_t hi) {
  constexpr int kW = C::kW;
  uint32_t u[kW];
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t d = (uint64_t)t[i] - C::n(i) - borrow;
    u[i] = (uint32_t)d;
    borrow = (uint32_t)(d >> 32) & 1u;
  }
  const uint32_t take = 0u - ((hi | (borrow ^ 1u)) & 1u);
#pragma unroll
  for (int i = 0; i < kW; i++) h.v[i] = (u[i] & take) | (t[i] & ~take);
}
template <class C>
CB200_XHD void sc_add(Sc<C>& h, const Sc<C>& f, const Sc<C>& g) {
  uint32_t t[C::kW];
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < C::kW; i++) {
    c += (uint64_t)f.v[i] + g.v[i];
    t[i] = (uint32_t)c;
    c >>= 32;
  }
  sc_reduce_once(h, t, (uint32_t)c);
}
template <class C>
CB200_XHD void sc_sub(Sc<C>& h, const Sc<C>& f, const Sc<C>& g) {
  constexpr int kW = C::kW;
  uint32_t t[kW];
  uint32_t borrow = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t d = (uint64_t)f.v[i] - g.v[i] - borrow;
    t[i] = (uint32_t)d;
    borrow = (uint32_t)(d >> 32) & 1u;
  }
  const uint32_t m = 0u - borrow;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    c += (uint64_t)t[i] + (C::n(i) & m);
    h.v[i] = (uint32_t)c;
    c >>= 32;
  }
}
// h = t R^-1 mod n for t < n R (2 kW words)
template <class C>
CB200_XHD void sc_mont_reduce(Sc<C>& h, uint32_t (&t)[2 * C::kW]) {
  constexpr int kW = C::kW;
  uint32_t top = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint32_t m = t[i] * n0inv<C>();
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < kW; j++) {
      c += (uint64_t)t[i + j] + (uint64_t)m * C::n(j);
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
  sc_reduce_once(h, r, top);
}
template <class C>
CB200_NISTP_NOINLINE void sc_mul(Sc<C>& h, const Sc<C>& f, const Sc<C>& g) {
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
  sc_mont_reduce(h, t);
}
template <class C>
CB200_XHD void sc_rn2(Sc<C>& h) {
#pragma unroll
  for (int i = 0; i < C::kW; i++) h.v[i] = C::rn2(i);
}
// plain words (< n) -> Montgomery form, and back
template <class C>
CB200_XHD void sc_to_mont(Sc<C>& h, const uint32_t (&k)[C::kW]) {
  Sc<C> f, r2;
#pragma unroll
  for (int i = 0; i < C::kW; i++) f.v[i] = k[i];
  sc_rn2(r2);
  sc_mul(h, f, r2);
}
template <class C>
CB200_XHD void sc_from_mont(uint32_t (&k)[C::kW], const Sc<C>& f) {
  constexpr int kW = C::kW;
  uint32_t t[2 * kW];
#pragma unroll
  for (int i = 0; i < kW; i++) t[i] = f.v[i], t[kW + i] = 0;
  Sc<C> h;
  sc_mont_reduce(h, t);
#pragma unroll
  for (int i = 0; i < kW; i++) k[i] = h.v[i];
}
// h = f^(n - 2) = f^-1 (0 for f = 0)
template <class C>
CB200_NISTP_NOINLINE void sc_invert(Sc<C>& h, const Sc<C>& f) {
  Sc<C> r = f;
  // the top bit of n - 2 (n's low word is odd and above 2, so n - 2 borrows nothing), then square-and-multiply
  int top = 32 * C::kW - 1;
  while (top > 0 && !((C::n(top / 32) >> (top % 32)) & 1u)) top--;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int b = top - 1; b >= 0; b--) {
    sc_mul(r, r, r);
    const uint32_t w = b / 32 == 0 ? C::n(0) - 2u : C::n(b / 32);
    if ((w >> (b % 32)) & 1u) sc_mul(r, r, f);
  }
  h = r;
}
// all ones iff f = 0
template <class C>
CB200_XHD uint32_t sc_is_zero(const Sc<C>& f) {
  uint32_t d = 0;
#pragma unroll
  for (int i = 0; i < C::kW; i++) d |= f.v[i];
  return (uint32_t)(((uint64_t)d - 1) >> 32);
}

// A big-endian string of kL bytes (kL < 8 * 2 kW) as 2 kW little-endian words
template <class C>
CB200_XHD void wide_from_be(uint32_t (&t)[2 * C::kW], const uint8_t* b) {
  constexpr int L = Suite<C>::kL;
#pragma unroll
  for (int i = 0; i < 2 * C::kW; i++) {
    uint32_t v = 0;
#pragma unroll
    for (int q = 3; q >= 0; q--) {
      const int j = L - 1 - (4 * i + q);
      v = (v << 8) | (j >= 0 ? b[j] : 0u);
    }
    t[i] = v;
  }
}
// hash_to_field mod n: the kL-byte string b reduced mod n, in Montgomery form.  REDC(b) = b R^-1 (b < n R), and two
// products by R^2 give b R.
template <class C>
CB200_NISTP_NOINLINE void sc_from_wide(Sc<C>& h, const uint8_t* b) {
  uint32_t t[2 * C::kW];
  wide_from_be<C>(t, b);
  Sc<C> r2;
  sc_rn2(r2);
  sc_mont_reduce(h, t);
  sc_mul(h, h, r2);
  sc_mul(h, h, r2);
}
// hash_to_field mod p: plain and Montgomery forms
template <class C>
CB200_NISTP_NOINLINE void fe_from_wide(Fe<C>& plain, Fe<C>& mont, const uint8_t* b) {
  uint32_t t[2 * C::kW];
  wide_from_be<C>(t, b);
  Fe<C> r2;
  nistp::fe_r2(r2);
  nistp::fe_mont_reduce(mont, t);
  nistp::fe_mul(plain, mont, r2);
  nistp::fe_mul(mont, plain, r2);
}

// ---------------------------------------------------------------- field helpers
// h = f^((p - 3) / 4); p = 3 mod 4 and p's low word is 2^32 - 1, so the exponent's words are p's shifted right by 2
template <class C>
CB200_XHD uint32_t c1_word(int i) {
  const uint32_t lo = i == 0 ? C::p(0) - 3u : C::p(i);
  const uint32_t hi = i + 1 < C::kW ? C::p(i + 1) : 0u;
  return (lo >> 2) | (hi << 30);
}
template <class C>
CB200_NISTP_NOINLINE void fe_pow_c1(Fe<C>& h, const Fe<C>& f) {
  int top = 32 * C::kW - 1;
  while (top > 0 && !((c1_word<C>(top / 32) >> (top % 32)) & 1u)) top--;
  Fe<C> r = f;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int b = top - 1; b >= 0; b--) {
    nistp::fe_sqr(r, r);
    if ((c1_word<C>(b / 32) >> (b % 32)) & 1u) nistp::fe_mul(r, r, f);
  }
  h = r;
}
template <class C>
CB200_XHD uint32_t fe_parity(const Fe<C>& mont) {
  Fe<C> t;
  nistp::fe_from_mont(t, mont);
  return t.v[0] & 1u;
}
// h = -3 f
template <class C>
CB200_XHD void fe_mul_a(Fe<C>& h, const Fe<C>& f) {
  Fe<C> t;
  nistp::fe_add(t, f, f);
  nistp::fe_add(t, t, f);
  nistp::fe_neg(h, t);
}
// y^2 = x^3 - 3x + b
template <class C>
CB200_XHD void fe_rhs(Fe<C>& h, const Fe<C>& x) {
  Fe<C> t, b;
  nistp::fe_sqr(t, x);
  nistp::fe_mul(t, t, x);
  Fe<C> ax;
  fe_mul_a(ax, x);
  nistp::fe_add(t, t, ax);
  nistp::fe_b(b);
  nistp::fe_add(h, t, b);
}

// ---------------------------------------------------------------- one compiled copy of each multiplication
// The helpers and kernels call these instead of inlining nistp.cuh's ladders at every use, which keeps oprf.cu to one
// compiled body of each per curve.
template <class C>
CB200_NISTP_NOINLINE void mul_var(Pt<C>& r, const uint32_t (&k)[C::kW], const Aff<C>& P) {
  nistp::scalarmult(r, k, P);
}
template <class C>
CB200_NISTP_NOINLINE void mul_base(Pt<C>& r, const uint32_t (&k)[C::kW], const uint32_t* __restrict__ table) {
  nistp::scalarmult_base(r, k, table);
}
template <class C>
CB200_NISTP_NOINLINE void to_affine(Fe<C>& x, Fe<C>& y, const Pt<C>& P) {
  nistp::pt_to_affine(x, y, P);
}
template <class C>
CB200_NISTP_NOINLINE void add(Pt<C>& r, const Pt<C>& p, const Pt<C>& q) {
  nistp::pt_add(r, p, q);
}

// ---------------------------------------------------------------- compressed points
// out = 0x02 | 0x03 || X of P (kNe bytes), masked to zero unless mask is all ones
template <class C>
CB200_NISTP_NOINLINE void encode(uint8_t* out, const Pt<C>& P, uint32_t mask) {
  Fe<C> x, y;
  to_affine(x, y, P);
  out[0] = (uint8_t)((2u | (y.v[0] & 1u)) & mask);
  nistp::words_to_be<C>(out + 1, x.v, mask);
}
// all ones iff b is a valid compressed point; A then holds it (Montgomery form).  Public data.
template <class C>
CB200_NISTP_NOINLINE uint32_t decode(Aff<C>& A, const uint8_t* b) {
  constexpr int kW = C::kW;
  uint32_t x[kW], p[kW];
#pragma unroll
  for (int i = 0; i < kW; i++) p[i] = C::p(i);
  nistp::words_from_be<C>(x, b + 1);
  uint32_t ok = (0u - (uint32_t)((b[0] & 0xfe) == 2)) & nistp::lt_words(x, p);
  Fe<C> fx, rhs, y, y2;
#pragma unroll
  for (int i = 0; i < kW; i++) fx.v[i] = x[i];
  nistp::fe_to_mont(A.x, fx);
  fe_rhs(rhs, A.x);
  fe_pow_c1(y, rhs);
  nistp::fe_mul(y, y, rhs);  // rhs^((p + 1) / 4)
  nistp::fe_sqr(y2, y);
  ok &= nistp::fe_eq(y2, rhs);
  Fe<C> ny;
  nistp::fe_neg(ny, y);
  nistp::fe_select(A.y, y, ny, 0u - (fe_parity(y) ^ (b[0] & 1u)));
  return ok;
}

// ---------------------------------------------------------------- hashing byte sequences
// A message made of up to K segments; a segment with a null pointer is n zero bytes.
struct Seg {
  const uint8_t* p;
  int n;
};
template <int K>
struct Cat {
  Seg s[K];
  CB200_XHD int len() const {
    int l = 0;
#pragma unroll
    for (int k = 0; k < K; k++) l += s[k].n;
    return l;
  }
  CB200_XHD uint8_t operator()(int j) const {
    uint8_t v = 0;
    bool done = false;
#pragma unroll
    for (int k = 0; k < K; k++) {
      if (!done && j < s[k].n) {
        v = s[k].p ? s[k].p[j] : 0;
        done = true;
      }
      j -= s[k].n;
    }
    return v;
  }
};
// H(msg) of a runtime length into the digest words h.  Word by word through a shift register, so that one block's
// code serves every length and every message functor stays small.
template <class S, class M>
CB200_NISTP_NOINLINE void hash(typename S::W (&h)[8], const M& msg) {
  using W = typename S::W;
  constexpr int B = S::kBlock, WB = S::kWordBytes;
  const int len = msg.len();
  const int nwords = (len + 1 + 2 * WB + B - 1) / B * 16;
  S::iv(h);
  W m[16];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int w = 0; w < nwords; w++) {
    W v = 0;
#pragma unroll
    for (int q = 0; q < WB; q++) {
      const int j = w * WB + q;
      const uint8_t x = j < len ? msg(j) : (j == len ? 0x80 : 0);
      v = (v << 8) | x;
    }
    if (w == nwords - 1) v = (W)((uint64_t)len << 3);
#pragma unroll
    for (int k = 0; k < 15; k++) m[k] = m[k + 1];
    m[15] = v;
    if ((w & 15) == 15) S::compress(h, m);
  }
}
template <class S>
CB200_XHD void digest_bytes(uint8_t* out, const typename S::W (&h)[8]) {
#pragma unroll
  for (int j = 0; j < S::kDigest; j++) out[j] = sha2::digest_byte<S>(h, j);
}

// expand_message_xmd(msg, dst, N) into out[0 .. N) for N <= 2 kL (RFC 9380 section 5.3.1; dst of at most 255 bytes)
template <class C, class M>
CB200_NISTP_NOINLINE void expand_xmd(uint8_t* out, int N, const M& msg, const uint8_t* dst, int dlen) {
  using S = typename Suite<C>::H;
  constexpr int D = S::kDigest;
  uint8_t tail[3 + 256];  // I2OSP(N, 2) || 0 || DST || I2OSP(len(DST), 1)
  tail[0] = (uint8_t)(N >> 8), tail[1] = (uint8_t)N, tail[2] = 0;
  for (int i = 0; i < dlen; i++) tail[3 + i] = dst[i];
  tail[3 + dlen] = (uint8_t)dlen;
  struct B0 {
    const M& m;
    const uint8_t* tail;
    int mlen, tlen;
    CB200_XHD int len() const { return S::kBlock + mlen + tlen; }
    CB200_XHD uint8_t operator()(int j) const {
      if (j < S::kBlock) return 0;
      j -= S::kBlock;
      return j < mlen ? m(j) : tail[j - mlen];
    }
  } m0{msg, tail, msg.len(), 4 + dlen};
  typename S::W h[8];
  hash<S>(h, m0);
  uint8_t b0[D], bi[D + 1 + 256];  // b_(i-1) xor b0 || i || DST'
  digest_bytes<S>(b0, h);
  const int ell = (N + D - 1) / D;
  for (int i = 0; i < dlen + 1; i++) bi[D + 1 + i] = tail[3 + i];
  for (int i = 0; i < D; i++) bi[i] = b0[i];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 1; i <= ell; i++) {
    bi[D] = (uint8_t)i;
    Cat<1> mi{{{bi, D + 2 + dlen}}};
    hash<S>(h, mi);
    for (int j = 0; j < D; j++) {
      const uint8_t v = sha2::digest_byte<S>(h, j);
      if ((i - 1) * D + j < N) out[(i - 1) * D + j] = v;
      bi[j] = v ^ b0[j];
    }
  }
}

// HashToScalar(msg, dst): hash_to_field mod n with one element, Montgomery form
template <class C, class M>
CB200_NISTP_NOINLINE void hash_to_scalar(Sc<C>& h, const M& msg, const uint8_t* dst, int dlen) {
  uint8_t u[Suite<C>::kL];
  expand_xmd<C>(u, Suite<C>::kL, msg, dst, dlen);
  sc_from_wide(h, u);
}

// map_to_curve_simple_swu for p = 3 mod 4 (RFC 9380 appendix F.2 with sqrt_ratio_3mod4), as a projective point
// (x_n : y x_d : x_d) -- no inversion.  u: plain (for sgn0) and Montgomery forms.
template <class C>
CB200_NISTP_NOINLINE void sswu(Pt<C>& Q, const Fe<C>& u_plain, const Fe<C>& u) {
  using namespace nistp;
  Fe<C> Z, c2, B, one, tv1, tv2, tv3, tv4, tv5, tv6, x, y, y1;
#pragma unroll
  for (int i = 0; i < C::kW; i++) Z.v[i] = C::sswu_z(i), c2.v[i] = C::sswu_c2(i);
  fe_b(B);
  fe_one(one);
  fe_sqr(tv1, u);
  fe_mul(tv1, Z, tv1);
  fe_sqr(tv2, tv1);
  fe_add(tv2, tv2, tv1);
  fe_add(tv3, tv2, one);
  fe_mul(tv3, B, tv3);
  Fe<C> ntv2, zero;
  fe_neg(ntv2, tv2);
  fe_zero(zero);
  fe_select(tv4, ntv2, Z, fe_eq(tv2, zero));  // CMOV(Z, -tv2, tv2 != 0)
  fe_mul_a(tv4, tv4);
  fe_sqr(tv2, tv3);
  fe_sqr(tv6, tv4);
  fe_mul_a(tv5, tv6);
  fe_add(tv2, tv2, tv5);
  fe_mul(tv2, tv2, tv3);
  fe_mul(tv6, tv6, tv4);
  fe_mul(tv5, B, tv6);
  fe_add(tv2, tv2, tv5);
  fe_mul(x, tv1, tv3);
  // sqrt_ratio_3mod4(tv2, tv6)
  Fe<C> s1, s2, y2, s3;
  fe_sqr(s1, tv6);
  fe_mul(s2, tv2, tv6);
  fe_mul(s1, s1, s2);
  fe_pow_c1(y1, s1);
  fe_mul(y1, y1, s2);
  fe_mul(y2, y1, c2);
  fe_sqr(s3, y1);
  fe_mul(s3, s3, tv6);
  const uint32_t qr = fe_eq(s3, tv2);
  fe_select(y1, y2, y1, qr);
  fe_mul(y, tv1, u);
  fe_mul(y, y, y1);
  fe_select(x, x, tv3, qr);
  fe_select(y, y, y1, qr);
  Fe<C> ny;
  fe_neg(ny, y);
  fe_select(y, ny, y, 0u - (uint32_t)((u_plain.v[0] & 1u) == fe_parity(y)));
  Q.X = x;
  fe_mul(Q.Y, y, tv4);
  Q.Z = tv4;
}

// HashToGroup(msg, dst) = Q0 + Q1 of hash_to_curve (the cofactor is 1); u receives (u0, u1) plain for the tests
template <class C, class M>
CB200_NISTP_NOINLINE void hash_to_group(Pt<C>& P, const M& msg, const uint8_t* dst, int dlen, Fe<C>* u_out = nullptr,
                             Pt<C>* q_out = nullptr) {
  constexpr int L = Suite<C>::kL;
  uint8_t ub[2 * L];
  expand_xmd<C>(ub, 2 * L, msg, dst, dlen);
  Pt<C> Q[2];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 0; i < 2; i++) {
    Fe<C> up, um;
    fe_from_wide(up, um, ub + i * L);
    sswu(Q[i], up, um);
    if (u_out) u_out[i] = up;
    if (q_out) q_out[i] = Q[i];
  }
  add(P, Q[0], Q[1]);
}

// ---------------------------------------------------------------- scalar rows
// a big-endian kBytes row -> plain words and an all-ones mask iff 0 < k < n
template <class C>
CB200_XHD uint32_t scalar_row(uint32_t (&k)[C::kW], const uint8_t* row) {
  nistp::words_from_be<C>(k, row);
  return nistp::scalar_ok<C>(k);
}
template <class C>
CB200_XHD void scalar_out(uint8_t* row, const Sc<C>& s, uint32_t mask) {
  uint32_t k[C::kW];
  sc_from_mont(k, s);
  nistp::words_to_be<C>(row, k, mask);
}

// the I2OSP(v, 2) prefix of a field
struct Len2 {
  uint8_t b[2];
  CB200_XHD explicit Len2(int v) : b{(uint8_t)(v >> 8), (uint8_t)v} {}
};

// ---------------------------------------------------------------- the server's operations, one thread each
// Status bits: 1 = a blinded element does not decode, 2 = sk not in [1, n - 1], 4 = r not in [1, n - 1], 8 = mode 2
// with t = k + HashToScalar(info) = 0.

// The keys of an op from its sk row: kp (the proof's key: k, or t in mode 2) and ke (the evaluation key: k, or t^-1),
// both plain words.  m_info = HashToScalar("Info" || I2OSP(len(info), 2) || info) in Montgomery form (mode 2 only).
template <class C>
CB200_NISTP_NOINLINE uint32_t op_keys(uint32_t (&kp)[C::kW], uint32_t (&ke)[C::kW], const uint8_t* sk_row, int mode,
                           const Sc<C>& m_info) {
  uint32_t k[C::kW];
  const uint32_t ok = scalar_row<C>(k, sk_row);
  uint32_t st = ok ? 0u : 2u;
  if (mode == 2) {
    Sc<C> km, t, ti;
    sc_to_mont(km, k);
    sc_add(t, km, m_info);
    st |= sc_is_zero(t) & 8u;
    sc_invert(ti, t);
    sc_from_mont(kp, t);
    sc_from_mont(ke, ti);
  } else {
#pragma unroll
    for (int i = 0; i < C::kW; i++) kp[i] = ke[i] = k[i];
  }
  return st;
}

// out = [ke] B for the compressed element in (kNe bytes each); an element that does not decode gives status 1 and an
// all-zero row
template <class C>
CB200_NISTP_NOINLINE uint32_t eval_element(uint8_t* out, const uint8_t* in, const uint32_t (&ke)[C::kW]) {
  Aff<C> B;
  const uint32_t ok = decode(B, in);
  Pt<C> D;
  mul_var(D, ke, B);
  encode(out, D, ok);
  return ok ? 0u : 1u;
}

// ComputeComposites (dleq.go:150-220) with Y = [k]G given compressed: M = sum d_j B_j over the m elements B_j (rows
// of kNe bytes at bs, stride b_stride) and C_j (= [k] B_j, at cs); returns M, and in st the OR of the decode
// failures (bit 0).  ctx / clen: the contextString.
template <class C>
CB200_NISTP_NOINLINE void composite(Pt<C>& M, uint32_t& st, const uint8_t* Y, const uint8_t* bs, size_t b_stride, const uint8_t* cs,
                         size_t c_stride, int m, const uint8_t* ctx, int clen) {
  using S = typename Suite<C>::H;
  constexpr int Ne = kNe<C>, D = S::kDigest;
  uint8_t sdst[5 + 24], hdst[13 + 24];
  for (int i = 0; i < 5; i++) sdst[i] = (uint8_t)"Seed-"[i];
  for (int i = 0; i < 13; i++) hdst[i] = (uint8_t)"HashToScalar-"[i];
  for (int i = 0; i < clen; i++) sdst[5 + i] = hdst[13 + i] = ctx[i];
  const Len2 lne(Ne), lsd(5 + clen), ld(D);
  typename S::W h[8];
  hash<S>(h, Cat<4>{{{lne.b, 2}, {Y, Ne}, {lsd.b, 2}, {sdst, 5 + clen}}});
  uint8_t seed[D];
  digest_bytes<S>(seed, h);
  nistp::pt_identity(M);
  st = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int j = 0; j < m; j++) {
    const uint8_t* bj = bs + (size_t)j * b_stride;
    const Len2 lj(j);
    Sc<C> d;
    hash_to_scalar<C>(d, Cat<8>{{{ld.b, 2}, {seed, D}, {lj.b, 2}, {lne.b, 2}, {bj, Ne}, {lne.b, 2},
                                 {cs + (size_t)j * c_stride, Ne}, {(const uint8_t*)"Composite", 9}}},
                      hdst, 13 + clen);
    uint32_t dk[C::kW];
    sc_from_mont(dk, d);
    Aff<C> B;
    st |= decode(B, bj) ? 0u : 1u;
    Pt<C> T;
    mul_var(T, dk, B);
    add(M, M, T);
  }
}

// The proof (dleq.go:93-145) for the key kp (plain), Y = [kp]G compressed, M (plain affine x || y, big-endian rows)
// and the randomness r (plain): out = c || s.  table: the fixed-base table.  Returns all ones iff 0 < r < n.
template <class C>
CB200_NISTP_NOINLINE uint32_t prove(uint8_t* out, const uint32_t (&kp)[C::kW], const uint8_t* Y, const uint8_t* m_xy,
                         const uint8_t* r_row, const uint32_t* __restrict__ table, const uint8_t* ctx, int clen,
                         uint32_t mask) {
  constexpr int Ne = kNe<C>, kW = C::kW;
  uint32_t r[kW];
  const uint32_t rok = scalar_row<C>(r, r_row);
  Aff<C> Ma;
  {
    Fe<C> x, y;
    nistp::words_from_be<C>(x.v, m_xy);
    nistp::words_from_be<C>(y.v, m_xy + C::kBytes);
    nistp::fe_to_mont(Ma.x, x);
    nistp::fe_to_mont(Ma.y, y);
  }
  uint8_t enc[4][Ne];  // M, Z, t2, t3
  {
    Pt<C> Mp;
    Mp.X = Ma.x, Mp.Y = Ma.y;
    nistp::fe_one(Mp.Z);
    encode(enc[0], Mp, ~0u);
  }
  // Z = [kp] M and t3 = [r] M through one call site
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int q = 0; q < 2; q++) {
    uint32_t s[kW];
#pragma unroll
    for (int i = 0; i < kW; i++) s[i] = q ? r[i] : kp[i];
    Pt<C> T;
    mul_var(T, s, Ma);
    encode(enc[q ? 3 : 1], T, ~0u);
  }
  {
    Pt<C> T;
    mul_base(T, r, table);
    encode(enc[2], T, ~0u);
  }
  uint8_t hdst[13 + 24];
  for (int i = 0; i < 13; i++) hdst[i] = (uint8_t)"HashToScalar-"[i];
  for (int i = 0; i < clen; i++) hdst[13 + i] = ctx[i];
  const Len2 lne(Ne);
  Sc<C> c;
  hash_to_scalar<C>(c, Cat<11>{{{lne.b, 2}, {Y, Ne}, {lne.b, 2}, {enc[0], Ne}, {lne.b, 2}, {enc[1], Ne}, {lne.b, 2},
                                {enc[2], Ne}, {lne.b, 2}, {enc[3], Ne}, {(const uint8_t*)"Challenge", 9}}},
                    hdst, 13 + clen);
  Sc<C> rm, km, s;
  sc_to_mont(rm, r);
  sc_to_mont(km, kp);
  sc_mul(km, c, km);
  sc_sub(s, rm, km);
  scalar_out(out, c, mask & rok);
  scalar_out(out + C::kBytes, s, mask & rok);
  return rok;
}

// FullEvaluate (server.go:97-117): out = H(I2OSP(len(in), 2) || in [|| I2OSP(len(info), 2) || info in mode 2] ||
// I2OSP(Ne, 2) || compress([ke] HashToGroup(in)) || "Finalize"), all zero unless mask is all ones
template <class C>
CB200_NISTP_NOINLINE void full_evaluate(uint8_t* out, const uint32_t (&ke)[C::kW], const uint8_t* in, int inlen, const uint8_t* info,
                             int infolen, int mode, const uint8_t* ctx, int clen, uint32_t mask) {
  using S = typename Suite<C>::H;
  constexpr int Ne = kNe<C>;
  uint8_t gdst[12 + 24];
  for (int i = 0; i < 12; i++) gdst[i] = (uint8_t)"HashToGroup-"[i];
  for (int i = 0; i < clen; i++) gdst[12 + i] = ctx[i];
  Pt<C> P;
  hash_to_group<C>(P, Cat<1>{{{in, inlen}}}, gdst, 12 + clen);
  Aff<C> Pa;
  {
    Fe<C> x, y;
    to_affine(x, y, P);
    nistp::fe_to_mont(Pa.x, x);
    nistp::fe_to_mont(Pa.y, y);
  }
  Pt<C> E;
  mul_var(E, ke, Pa);
  uint8_t e[Ne];
  encode(e, E, ~0u);
  const Len2 lin(inlen), linfo(infolen), lne(Ne);
  const int ni = mode == 2 ? infolen : 0, nl = mode == 2 ? 2 : 0;
  typename S::W h[8];
  hash<S>(h, Cat<7>{{{lin.b, 2}, {in, inlen}, {linfo.b, nl}, {info, ni}, {lne.b, 2}, {e, Ne},
                     {(const uint8_t*)"Finalize", 8}}});
#pragma unroll
  for (int j = 0; j < S::kDigest; j++) out[j] = sha2::digest_byte<S>(h, j) & (uint8_t)mask;
}

// DeriveKey (keys.go:103-132): sk = the first nonzero HashToScalar(seed || I2OSP(len(info), 2) || info || counter,
// "DeriveKeyPair" || contextString), pk = compress([sk] G)
template <class C>
CB200_NISTP_NOINLINE void derive_key(uint8_t* sk_out, uint8_t* pk_out, const uint8_t* seed, const uint8_t* info, int infolen,
                          const uint32_t* __restrict__ table, const uint8_t* ctx, int clen) {
  uint8_t dst[13 + 24];
  for (int i = 0; i < 13; i++) dst[i] = (uint8_t)"DeriveKeyPair"[i];
  for (int i = 0; i < clen; i++) dst[13 + i] = ctx[i];
  const Len2 linfo(infolen);
  Sc<C> s;
  for (int ctr = 0; ctr < 256; ctr++) {  // the loop leaves after the first try but with probability below 2^-250
    const uint8_t cb = (uint8_t)ctr;
    hash_to_scalar<C>(s, Cat<4>{{{seed, 32}, {linfo.b, 2}, {info, infolen}, {&cb, 1}}}, dst, 13 + clen);
    if (!sc_is_zero(s)) break;
  }
  uint32_t k[C::kW];
  sc_from_mont(k, s);
  nistp::words_to_be<C>(sk_out, k, ~0u);
  Pt<C> P;
  mul_base(P, k, table);
  encode(pk_out, P, ~0u);
}

// contextString = "OPRFV1-" || mode || "-" || identifier into c (at most 24 bytes); returns its length
template <class C>
CB200_XHD int context(uint8_t* c, int mode) {
  int n = 0;
  for (int i = 0; i < 7; i++) c[n++] = (uint8_t)"OPRFV1-"[i];
  c[n++] = (uint8_t)mode;
  c[n++] = '-';
  for (int i = 0; i < Suite<C>::kIdLen; i++) c[n++] = (uint8_t)Suite<C>::id()[i];
  return n;
}

}  // namespace oprf
}  // namespace cb200
