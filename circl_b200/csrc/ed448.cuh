// Ed448 on one thread (RFC 8032 section 5.2, pure Ed448): SHAKE256 over dom || prefix || message, scalars mod the
// group order, the edwards448 group law, point encoding and decoding, the fixed-base multiplication and the
// verification equation of the reference.
//
// Mirrors sign/ed448/ed448.go (newKeyFromSeed, signAll, verify, deriveSecretScalar, isLessThanOrder, writeDom),
// ecc/goldilocks/point.go (FromBytes, ToBytes) and scalar.go (FromBytes, Mul, Add).  The field is x448.cuh's
// (sixteen signed 28-bit limbs); only functions that x448.cuh does not have are added here, so no existing kernel
// changes.  Plain integer C++ like x448.cuh: it compiles for the device and for the host-only test of the CPU suite.
//
// Group law.  edwards448 is untwisted (a = 1, d = -39081, d not a square mod p), so the unified formulas of Hisil,
// Wong, Carter and Dawson (2008) in extended coordinates (X : Y : Z : T), T = XY / Z, are complete:
//   A = X1 X2, B = Y1 Y2, C = d T1 T2, D = Z1 Z2, E = (X1 + Y1)(X2 + Y2) - A - B, F = D - C, G = D + C, H = B - A,
//   X3 = E F, Y3 = G H, T3 = E H, Z3 = F G,
// and doubling is the same with C = 2 Z^2, F = A + B - C, G = A + B, H = A - B.  The a = -1 shortcut of ed25519.cuh
// ((Y - X)(Y2 - X2) and (Y + X)(Y2 + X2)) does not apply: p = 3 mod 4 has no square root of -1.
//
// Accumulator bound (x448.cuh: a folded column adds at most 38 products, 38 (2^28 + 2^9)^2 < 2^62).  A multiplication
// may take a sum or difference of two carried values on each side.  Here that covers (X1 + Y1)(X2 + Y2) (both factors
// are sums of two carried values), F, G and H (two carried products each), and d T2 of a cached point, which is one
// carried product fe_mul_small.  Two values go beyond it and are carried before they are multiplied: E (three
// carried products) in the addition, and E and F = A + B - 2 Z^2 (four) in the doubling.  Cached points keep Z and
// d T, never 2 Z or 2 d T.  tests/cpp/test_ed448_host.cpp runs every formula on limbs at the carried extreme.
#pragma once
#include <cstdint>
#include <cstring>

#include "x448.cuh"
#if defined(__CUDACC__)
#include "keccak.cuh"
#endif

namespace cb200 {
namespace ed448 {

using x448::Fe;
constexpr int kW = 14;                          // words of a field element or a scalar (56 bytes)
constexpr int kTableWords = 56 * 8 * 48;        // [i][j] = (j + 1) 256^i G as x (16) | y (16) | d x y (16) limbs
constexpr uint32_t kMaxContext = 255;           // ContextMaxSize

// ---------------------------------------------------------------- Keccak-f[1600] for the host build
inline void keccakf_host(uint64_t (&a)[25]) {
  static const int rho[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};
  uint64_t lfsr = 1;
  for (int r = 0; r < 24; r++) {
    uint64_t c[5], b[25];
    for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
    for (int x = 0; x < 5; x++) {
      const uint64_t dd = c[(x + 4) % 5] ^ ((c[(x + 1) % 5] << 1) | (c[(x + 1) % 5] >> 63));
      for (int y = 0; y < 25; y += 5) a[y + x] ^= dd;
    }
    for (int i = 0; i < 25; i++) {
      const int x = i % 5, y = i / 5, n = rho[i];
      b[y + 5 * ((2 * x + 3 * y) % 5)] = n ? (a[i] << n) | (a[i] >> (64 - n)) : a[i];
    }
    for (int y = 0; y < 25; y += 5)
      for (int x = 0; x < 5; x++) a[y + x] = b[y + x] ^ (~b[y + (x + 1) % 5] & b[y + (x + 2) % 5]);
    uint64_t rc = 0;  // the LFSR of FIPS 202
    for (int j = 0; j < 7; j++) {
      if (lfsr & 1) rc ^= 1ull << ((1 << j) - 1);
      lfsr = ((lfsr << 1) ^ ((lfsr & 0x80) ? 0x71 : 0)) & 0xff;
    }
    a[0] ^= rc;
  }
}

CB200_XHD void f1600(uint64_t (&a)[25]) {
#if defined(__CUDA_ARCH__)
  keccak::f1600(a);
#else
  keccakf_host(a);
#endif
}

// 8 little-endian bytes at p (any alignment), all of them message bytes.  The same rule as ed25519.cuh: on the device
// two aligned loads and a shift; the first aligned word starts up to 7 bytes before p (before the message only for
// its first word, and then inside the 8-byte-aligned word that holds msgs[0]); the second ends at most 7 bytes past
// the last message byte, inside the 8 bytes of read padding the entry points require behind the messages.
CB200_XHD uint64_t ld_le64(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
  const uint32_t a = (uint32_t)((uintptr_t)p & 7);
  const uint64_t* q = reinterpret_cast<const uint64_t*>((uintptr_t)p - a);
  const uint64_t lo = q[0];
  if (a == 0) return lo;
  return (lo >> (8 * a)) | (q[1] << (64 - 8 * a));
#else
  uint64_t v;
  memcpy(&v, p, 8);
  return v;
#endif
}

// SHAKE256(dom || h[0 .. nh) || msg[0 .. len)) up to its first permutation of output: the first 136 output bytes are
// lanes 0..16 of a.  dom is writeDom's string for pure Ed448, "SigEd448" || 0 || ctxlen || ctx (ed448.go:407-417), or
// nothing for ctxlen < 0; h is a short prefix (seed, prefix, R || A).  Both are read byte by byte; ctx is shared by
// the batch.  Lanes that lie wholly inside the message are read with ld_le64; a lane that holds the
// message's last bytes reads them one by one, so nothing past the last message byte but the padding above is read.
CB200_XHD void shake256(uint64_t (&a)[25], const uint8_t* ctx, int32_t ctxlen, const uint8_t* h, uint32_t nh,
                        const uint8_t* msg, uint64_t len) {
  const uint64_t kSig = 0x3834346445676953ull;  // "SigEd448"
  const uint32_t ld = ctxlen < 0 ? 0 : 10 + (uint32_t)ctxlen;
#pragma unroll
  for (int i = 0; i < 25; i++) a[i] = 0;
  const uint64_t hl = (uint64_t)ld + nh, total = hl + len;
  const uint64_t nblocks = total / 136 + 1;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (uint64_t blk = 0; blk < nblocks; blk++) {
#pragma unroll
    for (int l = 0; l < 17; l++) {
      const uint64_t o = blk * 136 + 8 * l;
      uint64_t v = 0;
      if (o >= hl && o + 8 <= total) {
        v = ld_le64(msg + (o - hl));
      } else {
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
        for (int b = 0; b < 8; b++) {
          const uint64_t q = o + b;
          uint32_t byte = 0;
          if (q < ld)
            byte = q < 8 ? (uint32_t)(kSig >> (8 * q)) & 0xff : q == 8 ? 0 : q == 9 ? (uint32_t)ctxlen : ctx[q - 10];
          else if (q < hl)
            byte = h[q - ld];
          else if (q < total)
            byte = msg[q - hl];
          else if (q == total)
            byte = 0x1f;  // SHAKE's domain bits and the first padding bit
          v |= (uint64_t)byte << (8 * b);
        }
      }
      if (l == 16 && blk + 1 == nblocks) v |= 0x80ull << 56;
      a[l] ^= v;
    }
    f1600(a);
  }
}

// the first 120 output bytes as little-endian words (the caller uses 114 or fewer)
CB200_XHD void lanes_to_words(uint32_t (&w)[30], const uint64_t (&a)[25]) {
#pragma unroll
  for (int i = 0; i < 15; i++) {
    w[2 * i] = (uint32_t)a[i];
    w[2 * i + 1] = (uint32_t)(a[i] >> 32);
  }
}
CB200_XHD uint8_t byte_of(const uint32_t* w, int i) { return (uint8_t)(w[i >> 2] >> (8 * (i & 3))); }

// ---------------------------------------------------------------- scalars mod l = 2^446 - 13818066809895115352007386748515426880336692474882178609894547503885
// Fourteen little-endian 32-bit words.  The reduction is the reference's (scalar.go reduceOneWord / FromBytes), with
// 32-bit instead of 64-bit words: the value is folded from the top one word at a time with 2^448 = R mod l
// (R < 2^226), then four masked subtractions of l bring it below l.  Both are exact for every input (DESIGN 6e), so
// the two agree everywhere.  Straight-line code: no branch and no address depends on the value.
CB200_XHD void sc_order(uint32_t (&l)[kW]) {
  const uint32_t L[kW] = {0xab5844f3u, 0x2378c292u, 0x8dc58f55u, 0x216cc272u, 0xaed63690u, 0xc44edb49u, 0x7cca23e9u,
                          0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu};
#pragma unroll
  for (int i = 0; i < kW; i++) l[i] = L[i];
}

// z += hi 2^448 mod l, z < 2^448 before and after (reduceOneWord): hi R < 2^258, so a carry out of the first sum
// leaves z < 2^258 and the second sum cannot carry again
CB200_XHD void sc_fold(uint32_t (&z)[kW], uint32_t hi) {
  const uint32_t R[8] = {0x529eec34u, 0x721cf5b5u, 0xc8e9c2abu, 0x7a4cf635u, 0x44a725bfu, 0xeec492d9u, 0x0cd77058u, 0x00000002u};
  uint64_t carry = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t t = (uint64_t)z[i] + (i < 8 ? (uint64_t)hi * R[i < 8 ? i : 0] : 0) + carry;
    z[i] = (uint32_t)t;
    carry = t >> 32;
  }
  const uint32_t cc = (uint32_t)carry;  // 0 or 1
  carry = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t t = (uint64_t)z[i] + (i < 8 ? (uint64_t)(R[i < 8 ? i : 0] & (0u - cc)) : 0) + carry;
    z[i] = (uint32_t)t;
    carry = t >> 32;
  }
}

// z < 2^448 < 5 l: z - 4 l < 2^448 - 4 l < l, so four masked subtractions leave z mod l
CB200_XHD void sc_final(uint32_t (&z)[kW]) {
  uint32_t L[kW];
  sc_order(L);
#pragma unroll
  for (int pass = 0; pass < 4; pass++) {
    uint32_t s[kW];
    uint64_t borrow = 0;
#pragma unroll
    for (int i = 0; i < kW; i++) {
      const uint64_t t = (uint64_t)z[i] - L[i] - borrow;
      s[i] = (uint32_t)t;
      borrow = (t >> 32) & 1;
    }
    const uint32_t keep = 0u - (uint32_t)borrow;  // all ones: z < l, keep z
#pragma unroll
    for (int i = 0; i < kW; i++) z[i] = (z[i] & keep) | (s[i] & ~keep);
  }
}

// out = x mod l for an N-word x (Scalar.FromBytes)
template <int N>
CB200_XHD void sc_reduce(uint32_t (&out)[kW], const uint32_t (&x)[N]) {
  static_assert(N >= kW, "at least 14 words");
  uint32_t z[kW];
#pragma unroll
  for (int i = 0; i < kW; i++) z[i] = x[N - kW + i];
#pragma unroll
  for (int w = N - kW - 1; w >= 0; w--) {
    const uint32_t hi = z[kW - 1];
#pragma unroll
    for (int i = kW - 1; i > 0; i--) z[i] = z[i - 1];
    z[0] = x[w];
    sc_fold(z, hi);
  }
  sc_final(z);
#pragma unroll
  for (int i = 0; i < kW; i++) out[i] = z[i];
}

// S = (k s + r) mod l for k, s, r < l (S.Mul(k, s); S.Add(S, r)): the 28-word k s + r, reduced as above
CB200_XHD void sc_muladd(uint32_t (&S)[kW], const uint32_t (&k)[kW], const uint32_t (&s)[kW], const uint32_t (&r)[kW]) {
  uint32_t x[2 * kW];
#pragma unroll
  for (int i = 0; i < 2 * kW; i++) x[i] = i < kW ? r[i < kW ? i : 0] : 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    uint64_t carry = 0;
#pragma unroll
    for (int j = 0; j < kW; j++) {
      const uint64_t t = (uint64_t)k[i] * s[j] + x[i + j] + carry;
      x[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
#pragma unroll
    for (int j = i + kW; j < 2 * kW; j++) {  // k s + r < 2^896: the carry never leaves the 28 words
      const uint64_t t = (uint64_t)x[j] + carry;
      x[j] = (uint32_t)t;
      carry = t >> 32;
    }
  }
  sc_reduce<2 * kW>(S, x);
}

// isLessThanOrder (ed448.go:397-405) on the 57 bytes of S as 14 words and byte 56; S is public
CB200_XHD bool sc_is_canonical(const uint32_t (&s)[kW], uint32_t top_byte) {
  uint32_t L[kW];
  sc_order(L);
  if (top_byte != 0) return false;
  for (int i = kW - 1; i >= 0; i--)
    if (s[i] != L[i]) return s[i] < L[i];
  return false;
}

// ---------------------------------------------------------------- field helpers
CB200_XHD void fe_renorm(Fe& h) {  // carry a value that went through more than one addition
  int64_t t[16];
#pragma unroll
  for (int i = 0; i < 16; i++) t[i] = h.v[i];
  x448::fe_carry(h, t);
}
CB200_XHD void fe_neg(Fe& h, const Fe& f) {
#pragma unroll
  for (int i = 0; i < 16; i++) h.v[i] = -f.v[i];
}
CB200_XHD bool fe_is_zero(const Fe& f) {
  uint32_t w[kW];
  x448::fe_tobytes(w, f);
  uint32_t acc = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) acc |= w[i];
  return acc == 0;
}
CB200_XHD void fe_mul_d(Fe& h, const Fe& f) { x448::fe_mul_small(h, f, -39081); }

// z^((p - 3) / 4) = z^(2^446 - 2^222 - 1) = z^([223 ones] 0 [222 ones]): the chain of x448::fe_invert up to that point
CB200_XHD_NOINLINE void fe_pow_p34(Fe& out, const Fe& z) {
  using namespace x448;
  Fe t, z2, z3, z6, z12, z24, z30, z48, z96, z192, z222, z223;
  auto pow2k = [](Fe& h, const Fe& f, int k) {
    fe_sq(h, f);
#pragma unroll 1
    for (int i = 1; i < k; i++) fe_sq(h, h);
  };
  pow2k(t, z, 1);
  fe_mul(z2, t, z);
  pow2k(t, z2, 1);
  fe_mul(z3, t, z);
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
  fe_mul(out, t, z222);
}

// ---------------------------------------------------------------- points
struct GeExt {
  Fe X, Y, Z, T;
};
struct GePre {  // affine multiple for mixed addition: x, y, d x y (carried)
  Fe x, y, dxy;
};
struct GeCached {  // general point for addition: X, Y, Z, d T (carried)
  Fe X, Y, Z, dT;
};

CB200_XHD void ge_identity(GeExt& P) {
  x448::fe_set(P.X, 0);
  x448::fe_set(P.Y, 1);
  x448::fe_set(P.Z, 1);
  x448::fe_set(P.T, 0);
}
// the tail shared by the additions: E (uncarried), A, B, C, D -> r
CB200_XHD void ge_finish(GeExt& r, Fe& e, const Fe& a, const Fe& b, const Fe& c, const Fe& d) {
  using namespace x448;
  Fe f, g, h;
  fe_sub(e, e, a);
  fe_sub(e, e, b);
  fe_renorm(e);
  fe_sub(f, d, c);
  fe_add(g, d, c);
  fe_sub(h, b, a);
  fe_mul(r.X, e, f);
  fe_mul(r.Y, g, h);
  fe_mul(r.Z, f, g);
  fe_mul(r.T, e, h);
}
// r = p + q, q affine (Z = 1)
CB200_XHD void ge_madd(GeExt& r, const GeExt& p, const GePre& q) {
  using namespace x448;
  Fe a, b, c, e, s1, s2;
  fe_mul(a, p.X, q.x);
  fe_mul(b, p.Y, q.y);
  fe_mul(c, p.T, q.dxy);
  fe_add(s1, p.X, p.Y);
  fe_add(s2, q.x, q.y);
  fe_mul(e, s1, s2);
  ge_finish(r, e, a, b, c, p.Z);
}
// r = p + q
CB200_XHD void ge_add(GeExt& r, const GeExt& p, const GeCached& q) {
  using namespace x448;
  Fe a, b, c, d, e, s1, s2;
  fe_mul(a, p.X, q.X);
  fe_mul(b, p.Y, q.Y);
  fe_mul(c, p.T, q.dT);
  fe_mul(d, p.Z, q.Z);
  fe_add(s1, p.X, p.Y);
  fe_add(s2, q.X, q.Y);
  fe_mul(e, s1, s2);
  ge_finish(r, e, a, b, c, d);
}
// r = 2 p
CB200_XHD void ge_dbl(GeExt& r, const GeExt& p) {
  using namespace x448;
  Fe a, b, c, e, f, g, h, t;
  fe_sq(a, p.X);
  fe_sq(b, p.Y);
  fe_sq(c, p.Z);
  fe_add(c, c, c);
  fe_add(t, p.X, p.Y);
  fe_sq(e, t);
  fe_sub(e, e, a);
  fe_sub(e, e, b);
  fe_renorm(e);
  fe_add(g, a, b);
  fe_sub(f, g, c);
  fe_renorm(f);
  fe_sub(h, a, b);
  fe_mul(r.X, e, f);
  fe_mul(r.Y, g, h);
  fe_mul(r.Z, f, g);
  fe_mul(r.T, e, h);
}
CB200_XHD void ge_to_cached(GeCached& c, const GeExt& p) {
  c.X = p.X;
  c.Y = p.Y;
  c.Z = p.Z;
  fe_mul_d(c.dT, p.T);
}

// Point.ToBytes (point.go:124-131): y canonical in bytes 0..55 (words 0..13), x mod 2 in bit 7 of byte 56 (*top)
CB200_XHD void ge_encode(uint32_t (&out)[kW], uint32_t& top, const GeExt& P) {
  using namespace x448;
  Fe zi, x, y;
  fe_invert(zi, P.Z);
  fe_mul(x, P.X, zi);
  fe_mul(y, P.Y, zi);
  uint32_t xb[kW];
  fe_tobytes(xb, x);
  fe_tobytes(out, y);
  top = (xb[0] & 1) << 7;
}

// FromBytes (point.go:42-80): false if byte 56 has any of its low 7 bits set, y >= p, (y^2 - 1) / (d y^2 - 1) is not
// a square, or x = 0 with the sign bit set.  x = u^3 v (u^5 v^3)^((p - 3) / 4) (RFC 8032 5.2.3), accepted iff
// v x^2 = u.  Variable time: only public keys are decoded.
CB200_XHD bool ge_decode(GeExt& P, const uint32_t (&yw)[kW], uint32_t top) {
  using namespace x448;
  if (top & 0x7f) return false;
  const uint32_t sign = top >> 7;
  Fe y, u, v, one, t, u2, x, chk;
  fe_frombytes(y, yw);
  uint32_t canon[kW], diff = 0;
  fe_tobytes(canon, y);
#pragma unroll
  for (int i = 0; i < kW; i++) diff |= canon[i] ^ yw[i];
  if (diff) return false;  // y >= p: its canonical form differs from the input
  fe_set(one, 1);
  fe_sq(u, y);
  fe_mul_d(v, u);
  fe_sub(u, u, one);  // u = y^2 - 1
  fe_sub(v, v, one);  // v = d y^2 - 1
  fe_sq(u2, u);
  fe_mul(t, u2, u);   // u^3
  fe_mul(x, t, v);    // u^3 v
  fe_mul(t, t, u2);   // u^5
  fe_sq(chk, v);
  fe_mul(chk, chk, v);  // v^3
  fe_mul(t, t, chk);    // u^5 v^3
  fe_pow_p34(t, t);
  fe_mul(x, x, t);
  fe_sq(chk, x);
  fe_mul(chk, chk, v);
  fe_sub(chk, chk, u);
  if (!fe_is_zero(chk)) return false;  // u / v is not a square
  uint32_t xb[kW];
  fe_tobytes(xb, x);
  uint32_t nz = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) nz |= xb[i];
  if (nz == 0 && sign) return false;
  if ((xb[0] & 1) != sign) fe_neg(x, x);
  P.X = x;
  P.Y = y;
  fe_set(P.Z, 1);
  fe_mul(P.T, x, y);
  return true;
}

// ---------------------------------------------------------------- fixed base
// Host side, once per process: table[i][j] = (j + 1) 256^i G in affine (x, y, d x y), i < 56 -- 56 x 8 points of
// 192 bytes, 84 KiB.  Computed with the same limb code the kernels use.
inline void build_base_table(int32_t* table) {
  using namespace x448;
  static const uint32_t kGx[kW] = {0xc70cc05eu, 0x2626a82bu, 0x8b00938eu, 0x433b80e1u, 0x2ab66511u, 0x12ae1af7u, 0xa3d3a464u,
                                   0xea6de324u, 0x470f1767u, 0x9e146570u, 0x22bf36dau, 0x221d15a6u, 0x6bed0dedu, 0x4f1970c6u};
  static const uint32_t kGy[kW] = {0xf230fa14u, 0x9808795bu, 0x4ed7c8adu, 0xfdbd132cu, 0xe67c39c4u, 0x3ad3ff1cu, 0x05a0c2d7u,
                                   0x87789c1eu, 0x6ca39840u, 0x4bea7373u, 0x56c9c762u, 0x88762037u, 0x6eb6bc24u, 0x693f4671u};
  auto to_pre = [](GePre& q, const GeExt& p) {
    Fe zi, t;
    fe_invert(zi, p.Z);
    fe_mul(q.x, p.X, zi);
    fe_mul(q.y, p.Y, zi);
    fe_mul(t, q.x, q.y);
    fe_mul_d(q.dxy, t);
  };
  GeExt P;
  fe_frombytes(P.X, kGx);
  fe_frombytes(P.Y, kGy);
  fe_set(P.Z, 1);
  fe_mul(P.T, P.X, P.Y);
  for (int i = 0; i < 56; i++) {
    GePre base, q;
    to_pre(base, P);
    GeExt M = P;
    for (int j = 0; j < 8; j++) {
      if (j > 0) {
        GeExt s;
        ge_madd(s, M, base);
        M = s;
      }
      to_pre(q, M);
      int32_t* w = table + (i * 8 + j) * 48;
      for (int c = 0; c < 16; c++) {
        w[c] = q.x.v[c];
        w[16 + c] = q.y.v[c];
        w[32 + c] = q.dxy.v[c];
      }
    }
    for (int k = 0; k < 8; k++) {  // P <- 256 P
      GeExt s;
      ge_dbl(s, P);
      P = s;
    }
  }
}

// h = [k] G for k < 2^447 (the top digit then stays within -8..8): signed radix-16 digits e_i in -8..7 (the top one
// takes the carry), odd digits first against rows i / 2, four doublings, then the even digits.  The digit is secret on
// the signing path: all eight multiples of a row are read and the wanted one -- or the neutral (0, 1, 0) for digit 0 --
// is kept by masks, and the sign is applied by masked negations of x and d x y.  No branch and no address depends on
// the scalar.
CB200_XHD void ge_scalarmult_base(GeExt& h, const uint32_t (&kin)[kW], const int32_t* __restrict__ table) {
  uint32_t k[kW];
  uint32_t carry = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t s = (uint64_t)kin[i] + 0x88888888u + carry;
    k[i] = (uint32_t)s;
    carry = (uint32_t)(s >> 32);
  }
  auto digit = [&](int i) -> int {
    uint32_t word = k[0];
#pragma unroll
    for (int q = 1; q < kW; q++) word = ((i >> 3) == q) ? k[q] : word;
    int e = (int)((word >> (4 * (i & 7))) & 15) - 8;
    if (i == 111) e += 16 * (int)carry;
    return e;
  };
  ge_identity(h);
  auto add_digit = [&](int i) {
    const int e = digit(i);
    const uint32_t neg = (uint32_t)(e >> 31);      // all ones for a negative digit
    const uint32_t m = ((uint32_t)e ^ neg) - neg;  // |e| in 0..8
    GePre q;
    x448::fe_set(q.x, 0);
    x448::fe_set(q.y, 1);
    x448::fe_set(q.dxy, 0);
    const int32_t* row = table + (i >> 1) * 8 * 48;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int j = 0; j < 8; j++) {
      const uint32_t mask = (uint32_t)((int32_t)((m ^ (uint32_t)(j + 1)) - 1u) >> 31);  // all ones iff m == j + 1
#pragma unroll
      for (int c = 0; c < 16; c++) {
        q.x.v[c] = (int32_t)(((uint32_t)q.x.v[c] & ~mask) | ((uint32_t)row[j * 48 + c] & mask));
        q.y.v[c] = (int32_t)(((uint32_t)q.y.v[c] & ~mask) | ((uint32_t)row[j * 48 + 16 + c] & mask));
        q.dxy.v[c] = (int32_t)(((uint32_t)q.dxy.v[c] & ~mask) | ((uint32_t)row[j * 48 + 32 + c] & mask));
      }
    }
#pragma unroll
    for (int c = 0; c < 16; c++) {  // -(x, y) = (-x, y)
      q.x.v[c] = (int32_t)(((uint32_t)q.x.v[c] ^ neg) - neg);
      q.dxy.v[c] = (int32_t)(((uint32_t)q.dxy.v[c] ^ neg) - neg);
    }
    GeExt s;
    ge_madd(s, h, q);
    h = s;
  };
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 1; i < 112; i += 2) add_digit(i);
  for (int q = 0; q < 4; q++) {
    GeExt s;
    ge_dbl(s, h);
    h = s;
  }
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 0; i < 112; i += 2) add_digit(i);
}

// Q = [s] G + [k] N for public s < l, k < 2^448: [s] G from the table, [k] N by a left-to-right signed radix-16
// window over the multiples 1..8 of N held by the thread (113 digits, the last one the carry; variable time).
CB200_XHD void ge_double_mult(GeExt& Q, const uint32_t (&s)[kW], const uint32_t (&kin)[kW], const GeExt& N,
                              const int32_t* __restrict__ table) {
  GeCached tab[8];
  ge_to_cached(tab[0], N);
  GeExt m = N;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int j = 1; j < 8; j++) {
    GeExt t;
    ge_add(t, m, tab[0]);
    m = t;
    ge_to_cached(tab[j], m);
  }
  uint32_t k[kW];
  uint32_t carry = 0;
#pragma unroll
  for (int i = 0; i < kW; i++) {
    const uint64_t t = (uint64_t)kin[i] + 0x88888888u + carry;
    k[i] = (uint32_t)t;
    carry = (uint32_t)(t >> 32);
  }
  ge_identity(Q);
  if (carry) Q = N;  // digit 112
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 111; i >= 0; i--) {
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int q = 0; q < 4; q++) {
      GeExt t;
      ge_dbl(t, Q);
      Q = t;
    }
    uint32_t word = k[0];
#pragma unroll
    for (int q = 1; q < kW; q++) word = ((i >> 3) == q) ? k[q] : word;
    const int e = (int)((word >> (4 * (i & 7))) & 15) - 8;
    if (e != 0) {
      GeCached c = tab[(e < 0 ? -e : e) - 1];
      if (e < 0) {
        fe_neg(c.X, c.X);
        fe_neg(c.dT, c.dT);
      }
      GeExt t;
      ge_add(t, Q, c);
      Q = t;
    }
  }
  GeExt sb;
  ge_scalarmult_base(sb, s, table);
  GeCached c;
  ge_to_cached(c, sb);
  GeExt t;
  ge_add(t, Q, c);
  Q = t;
}

// ---------------------------------------------------------------- the three operations
// 57-byte values (seed, A, R, S) travel as 14 words plus byte 56; the hashes read them as bytes.
CB200_XHD void to_bytes57(uint8_t* b, const uint32_t (&w)[kW], uint32_t top) {
#pragma unroll
  for (int i = 0; i < 56; i++) b[i] = byte_of(w, i);
  b[56] = (uint8_t)top;
}

// h = SHAKE256(seed, 114); s = clamp(h[0:57]) mod l (deriveSecretScalar), prefix = h[57:114]
CB200_XHD void expand_seed(uint32_t (&s)[kW], uint8_t (&prefix)[57], const uint8_t* seed) {
  uint64_t a[25];
  uint32_t h[30];
  shake256(a, nullptr, -1, seed, 57, nullptr, 0);
  lanes_to_words(h, a);
#pragma unroll
  for (int i = 0; i < kW; i++) s[i] = h[i];
  s[0] &= 0xfffffffcu;
  s[13] |= 0x80000000u;  // byte 56 is cleared: s < 2^448
  sc_reduce<kW>(s, s);
#pragma unroll
  for (int i = 0; i < 57; i++) prefix[i] = byte_of(h, 57 + i);
}

// r = SHAKE256(dom || pre || M, 114) mod l, pre = prefix (57 bytes) or R || A (114 bytes)
CB200_XHD void hash_to_scalar(uint32_t (&r)[kW], const uint8_t* ctx, int32_t ctxlen, const uint8_t* pre, uint32_t npre,
                              const uint8_t* msg, uint64_t len) {
  uint64_t a[25];
  uint32_t h[30];
  shake256(a, ctx, ctxlen, pre, npre, msg, len);
  lanes_to_words(h, a);
  h[28] &= 0xffffu;  // 114 bytes
  h[29] = 0;
  sc_reduce<30>(r, h);
}

// newKeyFromSeed (ed448.go:191-205): A = encode([s] G)
CB200_XHD void public_from_seed(uint32_t (&A)[kW], uint32_t& top, const uint8_t* seed, const int32_t* __restrict__ table) {
  uint32_t s[kW];
  uint8_t prefix[57];
  expand_seed(s, prefix, seed);
  GeExt P;
  ge_scalarmult_base(P, s, table);
  ge_encode(A, top, P);
}

// signAll (ed448.go:207-271), pure Ed448, with A (57 bytes) as given by the caller and ctxlen <= 255.
// sig: R (57 bytes) || S (56 bytes) || 0.
CB200_XHD void sign(uint8_t* sig, const uint8_t* seed, const uint8_t* A, const uint8_t* ctx, int32_t ctxlen, const uint8_t* msg,
                    uint64_t len, const int32_t* __restrict__ table) {
  uint32_t s[kW], r[kW], k[kW], S[kW], Rw[kW], rtop;
  uint8_t buf[114];
  {
    uint8_t prefix[57];
    expand_seed(s, prefix, seed);
    hash_to_scalar(r, ctx, ctxlen, prefix, 57, msg, len);
  }
  GeExt P;
  ge_scalarmult_base(P, r, table);
  ge_encode(Rw, rtop, P);
  to_bytes57(buf, Rw, rtop);
#pragma unroll
  for (int i = 0; i < 57; i++) buf[57 + i] = A[i];
  hash_to_scalar(k, ctx, ctxlen, buf, 114, msg, len);
  sc_muladd(S, k, s, r);
  to_bytes57(sig, Rw, rtop);
  to_bytes57(sig + 57, S, 0);
}

// verify (ed448.go:294-339): S < l with byte 113 = 0, A decodes, and encode(Q) == R for the reference's
// Q = CombinedMult(S, k, -A).  That runs on the 4-isogenous twist with S / 4 and k / 4 mod l and maps back, which
// gives Q = [S] G - [4 ((k / 4) mod l)] A: the 4-torsion part of A drops out.  4 ((k / 4) mod l) = k + (k mod 4) l
// (l = 3 mod 4), below 4 l < 2^448.  sig: R || S (114 bytes); ctxlen <= 255 (the caller rejects longer ones).
CB200_XHD bool verify(const uint8_t* A, const uint8_t* ctx, int32_t ctxlen, const uint8_t* msg, uint64_t len, const uint8_t* sig,
                      const int32_t* __restrict__ table) {
  uint32_t S[kW], Aw[kW];
#pragma unroll
  for (int i = 0; i < kW; i++) {
    S[i] = (uint32_t)sig[57 + 4 * i] | ((uint32_t)sig[58 + 4 * i] << 8) | ((uint32_t)sig[59 + 4 * i] << 16) |
           ((uint32_t)sig[60 + 4 * i] << 24);
    Aw[i] = (uint32_t)A[4 * i] | ((uint32_t)A[4 * i + 1] << 8) | ((uint32_t)A[4 * i + 2] << 16) | ((uint32_t)A[4 * i + 3] << 24);
  }
  if (!sc_is_canonical(S, sig[113])) return false;
  GeExt P;
  if (!ge_decode(P, Aw, A[56])) return false;
  fe_neg(P.X, P.X);  // -A
  fe_neg(P.T, P.T);
  uint8_t buf[114];
#pragma unroll
  for (int i = 0; i < 57; i++) {
    buf[i] = sig[i];
    buf[57 + i] = A[i];
  }
  uint32_t k[kW], L[kW];
  hash_to_scalar(k, ctx, ctxlen, buf, 114, msg, len);
  sc_order(L);
  {  // k += (k mod 4) l
    const uint32_t j = k[0] & 3;
    uint64_t carry = 0;
#pragma unroll
    for (int i = 0; i < kW; i++) {
      const uint64_t t = (uint64_t)k[i] + (uint64_t)j * L[i] + carry;
      k[i] = (uint32_t)t;
      carry = t >> 32;
    }
  }
  GeExt Q;
  ge_double_mult(Q, S, k, P, table);
  uint32_t enc[kW], top;
  ge_encode(enc, top, Q);
  uint32_t diff = top ^ sig[56];
#pragma unroll
  for (int i = 0; i < 56; i++) diff |= (uint32_t)(byte_of(enc, i) ^ sig[i]);
  return diff == 0;
}

}  // namespace ed448
}  // namespace cb200
