// Ed25519 on one thread (RFC 8032 section 5.1, pure Ed25519): SHA-512, scalars mod L, point encoding and decoding,
// the fixed-base and the verification double multiplication.
//
// Mirrors sign/ed25519/ed25519.go (NewKeyFromSeed, Sign, Verify), point.go (ToBytes, FromBytes) and modular.go
// (reduceModOrder, calculateS, isLessThanOrder).  The field and the group law are those of x25519.cuh (ten signed
// limbs, complete a = -1 formulas in extended coordinates), and [k]B runs on its table of multiples of 256^i B.
// Plain integer C++ like x25519.cuh: it compiles for the device and for the host-only test of the CPU suite.
#pragma once
#include <cstdint>
#include <cstring>

#include "x25519.cuh"

namespace cb200 {
namespace ed25519 {

using x25519::Fe;
using x25519::GeExt;

// ---------------------------------------------------------------- SHA-512 (FIPS 180-4), one message per thread
#define CB200_SHA512_K_BODY                                                                                                    \
  0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull, 0x3956c25bf348b538ull,          \
      0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull, 0xd807aa98a3030242ull, 0x12835b0145706fbeull,      \
      0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull, 0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull,      \
      0xc19bf174cf692694ull, 0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull,      \
      0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull, 0x983e5152ee66dfabull,      \
      0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull, 0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull,      \
      0x06ca6351e003826full, 0x142929670a0e6e70ull, 0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull,      \
      0x53380d139d95b3dfull, 0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull,      \
      0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull, 0xd192e819d6ef5218ull,      \
      0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull, 0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull,      \
      0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull, 0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull,      \
      0x682e6ff3d6b2b8a3ull, 0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull,      \
      0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull, 0xca273eceea26619cull,      \
      0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull, 0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull,      \
      0x113f9804bef90daeull, 0x1b710b35131c471bull, 0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull,      \
      0x431d67c49c100d4cull, 0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull
#if defined(__CUDACC__)
static __constant__ uint64_t kSha512K_dev[80] = {CB200_SHA512_K_BODY};
#endif
static const uint64_t kSha512K_host[80] = {CB200_SHA512_K_BODY};
#undef CB200_SHA512_K_BODY

CB200_XHD uint64_t sha512_k(int i) {
#if defined(__CUDA_ARCH__)
  return kSha512K_dev[i];
#else
  return kSha512K_host[i];
#endif
}

// rotate right by a constant: two funnel shifts on the device
CB200_XHD uint64_t rotr64(uint64_t x, int n) {
#if defined(__CUDA_ARCH__)
  const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
  uint32_t rl, rh;
  if (n < 32) {
    rl = __funnelshift_r(lo, hi, n);
    rh = __funnelshift_r(hi, lo, n);
  } else {
    rl = __funnelshift_r(hi, lo, n - 32);
    rh = __funnelshift_r(lo, hi, n - 32);
  }
  return ((uint64_t)rh << 32) | rl;
#else
  return (x >> n) | (x << (64 - n));
#endif
}
CB200_XHD uint64_t bswap64(uint64_t x) {
#if defined(__CUDA_ARCH__)
  const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
  return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
#else
  return __builtin_bswap64(x);
#endif
}

CB200_XHD void sha512_block(uint64_t (&H)[8], uint64_t (&W)[16]) {
  uint64_t a = H[0], b = H[1], c = H[2], d = H[3], e = H[4], f = H[5], g = H[6], h = H[7];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int r = 0; r < 80; r += 16) {
#pragma unroll
    for (int j = 0; j < 16; j++) {
      if (r > 0) {
        const uint64_t w1 = W[(j + 1) & 15], w14 = W[(j + 14) & 15];
        W[j] += (rotr64(w14, 19) ^ rotr64(w14, 61) ^ (w14 >> 6)) + W[(j + 9) & 15] +
                (rotr64(w1, 1) ^ rotr64(w1, 8) ^ (w1 >> 7));
      }
      const uint64_t t1 = h + (rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41)) + ((e & f) ^ (~e & g)) + sha512_k(r + j) + W[j];
      const uint64_t t2 = (rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
      h = g;
      g = f;
      f = e;
      e = d + t1;
      d = c;
      c = b;
      b = a;
      a = t1 + t2;
    }
  }
  H[0] += a;
  H[1] += b;
  H[2] += c;
  H[3] += d;
  H[4] += e;
  H[5] += f;
  H[6] += g;
  H[7] += h;
}

// 8 little-endian bytes at p (any alignment), all of them message bytes.  On the device two aligned loads and a shift:
// the first aligned word starts up to 7 bytes before p (before the message only for its first word, and then inside
// the 8-byte-aligned word that holds msgs[0]); the second ends at most 14 bytes after p, i.e. at most 7 bytes past the
// last message byte, inside the 8 bytes of read padding the entry points require behind the messages.
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

// out = SHA-512(pre || msg[0 .. len)), pre = NPRE 64-bit words (4: a 32-byte prefix, 8: R || A).  pre and out are
// little-endian 32-bit words of the byte strings.  msg needs 8 readable bytes after its end.
template <int NPRE>
CB200_XHD void sha512(uint32_t (&out)[16], const uint32_t (&pre)[2 * NPRE], const uint8_t* msg, uint64_t len) {
  uint64_t H[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                   0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
  const uint64_t total = 8 * NPRE + len;
  const uint64_t nblocks = (total + 17 + 127) / 128;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (uint64_t blk = 0; blk < nblocks; blk++) {
    uint64_t W[16];
#pragma unroll
    for (int w = 0; w < 16; w++) {
      uint64_t v;
      if (w < NPRE && blk == 0) {
        v = (uint64_t)pre[2 * (w < NPRE ? w : 0)] | ((uint64_t)pre[2 * (w < NPRE ? w : 0) + 1] << 32);
      } else {
        const int64_t o = (int64_t)(16 * blk + w - NPRE) * 8;  // byte offset of the word in msg
        const int64_t rem = (int64_t)len - o;
        v = 0;
        if (rem >= 8) {
          v = ld_le64(msg + o);
        } else if (rem > 0) {  // the tail word: byte loads, nothing past the last message byte
          for (int b = 0; b < 7; b++)
            if (b < rem) v |= (uint64_t)msg[o + b] << (8 * b);
        }
        if (rem < 8 && rem >= 0) v = (v & ((1ull << (8 * rem)) - 1)) | (0x80ull << (8 * rem));  // rem = 0: 0x80 only
      }
      W[w] = bswap64(v);
    }
    if (blk + 1 == nblocks) W[15] = total << 3;  // the 0x80 byte is at most in word 13 of the last block
    sha512_block(H, W);
  }
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint64_t le = bswap64(H[i]);
    out[2 * i] = (uint32_t)le;
    out[2 * i + 1] = (uint32_t)(le >> 32);
  }
}

// ---------------------------------------------------------------- scalars mod L = 2^252 + 27742317777372353535851937790883648493
// Eight little-endian 32-bit words.  Reduction is Barrett's (HAC 14.42, base 2^32, k = 8) with two masked final
// subtractions: straight-line code, no branch and no address depends on the value.
CB200_XHD void sc_order(uint32_t (&l)[9]) {
  const uint32_t L[9] = {0x5cf5d3edu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu, 0, 0, 0, 0x10000000u, 0};
#pragma unroll
  for (int i = 0; i < 9; i++) l[i] = L[i];
}

// out = x mod L for x < 2^512 (16 words)
CB200_XHD void sc_reduce(uint32_t (&out)[8], const uint32_t (&x)[16]) {
  const uint32_t mu[9] = {0x0a2c131bu, 0xed9ce5a3u, 0x086329a7u, 0x2106215du, 0xffffffebu,
                          0xffffffffu, 0xffffffffu, 0xffffffffu, 0x0000000fu};  // floor(2^512 / L)
  uint32_t L[9];
  sc_order(L);
  // q3 = floor(floor(x / 2^224) * mu / 2^288)
  uint32_t q2[18];
#pragma unroll
  for (int i = 0; i < 18; i++) q2[i] = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {
    uint64_t carry = 0;
#pragma unroll
    for (int j = 0; j < 9; j++) {
      const uint64_t t = (uint64_t)x[7 + i] * mu[j] + q2[i + j] + carry;
      q2[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
    q2[i + 9] = (uint32_t)carry;
  }
  // r = (x - q3 L) mod 2^288
  uint32_t r2[9];
#pragma unroll
  for (int i = 0; i < 9; i++) r2[i] = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {
    uint64_t carry = 0;
#pragma unroll
    for (int j = 0; j + i < 9; j++) {
      const uint64_t t = (uint64_t)q2[9 + i] * L[j] + r2[i + j] + carry;
      r2[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
  }
  uint32_t r[9];
  uint64_t borrow = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {
    const uint64_t t = (uint64_t)x[i] - r2[i] - borrow;
    r[i] = (uint32_t)t;
    borrow = (t >> 32) & 1;
  }
  // now r < 3L: subtract L twice where it does not go negative
#pragma unroll
  for (int pass = 0; pass < 2; pass++) {
    uint32_t s[9];
    borrow = 0;
#pragma unroll
    for (int i = 0; i < 9; i++) {
      const uint64_t t = (uint64_t)r[i] - L[i] - borrow;
      s[i] = (uint32_t)t;
      borrow = (t >> 32) & 1;
    }
    const uint32_t keep = (uint32_t)0 - (uint32_t)borrow;  // all ones: r < L, keep r
#pragma unroll
    for (int i = 0; i < 9; i++) r[i] = (r[i] & keep) | (s[i] & ~keep);
  }
#pragma unroll
  for (int i = 0; i < 8; i++) out[i] = r[i];
}

// S = (r + k a) mod L (modular.go calculateS): r, k < L, a < 2^256 (the clamped, unreduced secret scalar)
CB200_XHD void sc_muladd(uint32_t (&S)[8], const uint32_t (&r)[8], const uint32_t (&k)[8], const uint32_t (&a)[8]) {
  uint32_t x[16];
#pragma unroll
  for (int i = 0; i < 16; i++) x[i] = i < 8 ? r[i < 8 ? i : 0] : 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint64_t carry = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const uint64_t t = (uint64_t)k[i] * a[j] + x[i + j] + carry;
      x[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
#pragma unroll
    for (int j = i + 8; j < 16; j++) {  // propagate the carry (k a + r < 2^512)
      const uint64_t t = (uint64_t)x[j] + carry;
      x[j] = (uint32_t)t;
      carry = t >> 32;
    }
  }
  sc_reduce(S, x);
}

// isLessThanOrder (ed25519.go:437-443); S is public
CB200_XHD bool sc_is_canonical(const uint32_t (&s)[8]) {
  uint32_t L[9];
  sc_order(L);
  for (int i = 7; i >= 0; i--)
    if (s[i] != L[i]) return s[i] < L[i];
  return false;
}

// ---------------------------------------------------------------- field and points
CB200_XHD void fe_const(Fe& h, const uint32_t (&w)[8]) { x25519::fe_frombytes(h, w); }
CB200_XHD void fe_d2(Fe& h) {
  const uint32_t w[8] = {0x26b2f159u, 0xebd69b94u, 0x8283b156u, 0x00e0149au, 0xeef3d130u, 0x198e80f2u, 0x56dffce7u, 0x2406d9dcu};
  fe_const(h, w);
}
CB200_XHD bool fe_is_zero(const Fe& f) {
  uint32_t w[8];
  x25519::fe_tobytes(w, f);
  uint32_t acc = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) acc |= w[i];
  return acc == 0;
}

// z^((p - 5) / 8) = z^(2^252 - 3): the chain of fe_invert up to 2^250 - 1, then two squarings and one multiplication
CB200_XHD_NOINLINE void fe_pow22523(Fe& out, const Fe& z) {
  using namespace x25519;
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
  fe_mul(z5, t, z9);
  pow2k(t, z5, 5);
  fe_mul(z10, t, z5);
  pow2k(t, z10, 10);
  fe_mul(z20, t, z10);
  pow2k(t, z20, 20);
  fe_mul(t, t, z20);
  pow2k(t, t, 10);
  fe_mul(z50, t, z10);
  pow2k(t, z50, 50);
  fe_mul(z100, t, z50);
  pow2k(t, z100, 100);
  fe_mul(t, t, z100);
  pow2k(t, t, 50);
  fe_mul(t, t, z50);  // 2^250 - 1
  pow2k(t, t, 2);
  fe_mul(out, t, z);  // 2^252 - 3
}

// pointR1.ToBytes (point.go:38-52): canonical y with the low bit of x in bit 255
CB200_XHD void ge_encode(uint32_t (&out)[8], const GeExt& P) {
  using namespace x25519;
  Fe zi, x, y;
  fe_invert(zi, P.Z);
  fe_mul(x, P.X, zi);
  fe_mul(y, P.Y, zi);
  uint32_t xb[8];
  fe_tobytes(xb, x);
  fe_tobytes(out, y);
  out[7] |= (xb[0] & 1) << 31;
}

// pointR1.FromBytes (point.go:54-87): false for y >= p, for a y without a square root x, and for x = 0 with the sign
// bit set.  Variable time: only public keys are decoded.
CB200_XHD bool ge_decode(GeExt& P, const uint32_t (&in)[8]) {
  using namespace x25519;
  const uint32_t sign = in[7] >> 31;
  uint32_t yw[8];
#pragma unroll
  for (int i = 0; i < 8; i++) yw[i] = in[i];
  yw[7] &= 0x7fffffffu;
  uint32_t top = yw[7] ^ 0x7fffffffu;
#pragma unroll
  for (int i = 1; i < 7; i++) top |= ~yw[i];
  if (top == 0 && yw[0] >= 0xffffffedu) return false;  // y >= p
  const uint32_t dw[8] = {0x135978a3u, 0x75eb4dcau, 0x4141d8abu, 0x00700a4du, 0x7779e898u, 0x8cc74079u, 0x2b6ffe73u, 0x52036ceeu};
  const uint32_t iw[8] = {0x4a0ea0b0u, 0xc4ee1b27u, 0xad2fe478u, 0x2f431806u, 0x3dfbd7a7u, 0x2b4d0099u, 0x4fc1df0bu, 0x2b832480u};
  Fe y, u, v, d, one, v3, t, x, chk;
  fe_frombytes(y, yw);
  fe_const(d, dw);
  fe_set(one, 1);
  fe_sq(u, y);
  fe_mul(v, u, d);
  fe_sub(u, u, one);  // u = y^2 - 1
  fe_add(v, v, one);  // v = d y^2 + 1
  fe_renorm(u);
  fe_renorm(v);
  // x = u v^3 (u v^7)^((p - 5) / 8)
  fe_sq(v3, v);
  fe_mul(v3, v3, v);
  fe_sq(t, v3);
  fe_mul(t, t, v);
  fe_mul(t, t, u);
  fe_pow22523(t, t);
  fe_mul(t, t, v3);
  fe_mul(x, t, u);
  fe_sq(chk, x);
  fe_mul(chk, chk, v);  // v x^2
  fe_sub(t, chk, u);
  fe_renorm(t);
  if (!fe_is_zero(t)) {
    fe_add(t, chk, u);
    fe_renorm(t);
    if (!fe_is_zero(t)) return false;  // u / v is not a square
    Fe i;
    fe_const(i, iw);
    fe_mul(x, x, i);
  }
  uint32_t xb[8];
  fe_tobytes(xb, x);
  uint32_t nz = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) nz |= xb[i];
  if (nz == 0 && sign) return false;
  if ((xb[0] & 1) != sign) {
    Fe zero;
    fe_set(zero, 0);
    fe_sub(x, zero, x);
    fe_renorm(x);
  }
  P.X = x;
  P.Y = y;
  fe_set(P.Z, 1);
  fe_mul(P.T, x, y);
  return true;
}

// a point prepared for a general addition: y + x, y - x, 2 z, 2 d t (all carried)
struct GeCached {
  Fe ypx, ymx, z2, t2d;
};
CB200_XHD void ge_to_cached(GeCached& c, const GeExt& p, const Fe& d2) {
  using namespace x25519;
  fe_add(c.ypx, p.Y, p.X);
  fe_renorm(c.ypx);
  fe_sub(c.ymx, p.Y, p.X);
  fe_renorm(c.ymx);
  fe_add(c.z2, p.Z, p.Z);
  fe_renorm(c.z2);
  fe_mul(c.t2d, p.T, d2);
}
// r = p + q (complete a = -1 formulas, as ge_madd with a general Z)
CB200_XHD void ge_add(GeExt& r, const GeExt& p, const GeCached& q) {
  using namespace x25519;
  Fe a, b, c, d, e, f, g, h;
  fe_sub(a, p.Y, p.X);
  fe_mul(a, a, q.ymx);
  fe_add(b, p.Y, p.X);
  fe_mul(b, b, q.ypx);
  fe_mul(c, p.T, q.t2d);
  fe_mul(d, p.Z, q.z2);
  fe_sub(e, b, a);
  fe_sub(f, d, c);
  fe_add(g, d, c);
  fe_add(h, b, a);
  fe_mul(r.X, e, f);
  fe_mul(r.Y, g, h);
  fe_mul(r.Z, f, g);
  fe_mul(r.T, e, h);
}
CB200_XHD void ge_cached_neg(GeCached& c) {
  Fe t = c.ypx;
  c.ypx = c.ymx;
  c.ymx = t;
  Fe zero;
  x25519::fe_set(zero, 0);
  x25519::fe_sub(c.t2d, zero, c.t2d);
}

// Q = [s] B + [k] N for public s < 2^256, k < 2^253 (the verification equation with N = -A, pointR1.doubleMult).
// [s] B comes from the fixed-base table; [k] N is a left-to-right signed radix-16 window over the multiples
// 1..8 N held by the thread (variable time: every input is public).
CB200_XHD void ge_double_mult(GeExt& Q, const uint32_t (&s)[8], const uint32_t (&kin)[8], const GeExt& N,
                              const int32_t* __restrict__ table) {
  using namespace x25519;
  Fe d2;
  fe_d2(d2);
  GeCached tab[8];
  ge_to_cached(tab[0], N, d2);
  GeExt m = N;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int j = 1; j < 8; j++) {
    GeExt t;
    ge_add(t, m, tab[0]);
    m = t;
    ge_to_cached(tab[j], m, d2);
  }
  uint32_t k[8];
  uint32_t carry = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {  // same recoding as ge_scalarmult_base: nibble i of k + 0x88...8, minus 8
    const uint64_t t = (uint64_t)kin[i] + 0x88888888u + carry;
    k[i] = (uint32_t)t;
    carry = (uint32_t)(t >> 32);
  }
  fe_set(Q.X, 0);
  fe_set(Q.Y, 1);
  fe_set(Q.Z, 1);
  fe_set(Q.T, 0);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 63; i >= 0; i--) {
    if (i < 63) {
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
      for (int q = 0; q < 4; q++) {
        GeExt t;
        ge_dbl(t, Q);
        Q = t;
      }
    }
    uint32_t word = k[0];
#pragma unroll
    for (int q = 1; q < 8; q++) word = ((i >> 3) == q) ? k[q] : word;
    int e = (int)((word >> (4 * (i & 7))) & 15) - 8;
    if (i == 63) e += 16 * (int)carry;
    if (e != 0) {
      GeCached c = tab[(e < 0 ? -e : e) - 1];
      if (e < 0) ge_cached_neg(c);
      GeExt t;
      ge_add(t, Q, c);
      Q = t;
    }
  }
  GeExt sb;
  ge_scalarmult_base(sb, s, table);
  GeCached c;
  ge_to_cached(c, sb, d2);
  GeExt t;
  ge_add(t, Q, c);
  Q = t;
}

// ---------------------------------------------------------------- the three operations
// h = SHA-512(seed): s = clamp(h[0:32]) (ed25519.go:431-434), prefix = h[32:64]
CB200_XHD void expand_seed(uint32_t (&s)[8], uint32_t (&prefix)[8], const uint32_t (&seed)[8]) {
  uint32_t h[16];
  sha512<4>(h, seed, nullptr, 0);
#pragma unroll
  for (int i = 0; i < 8; i++) {
    s[i] = h[i];
    prefix[i] = h[8 + i];
  }
  s[0] &= 0xfffffff8u;
  s[7] = (s[7] & 0x7fffffffu) | 0x40000000u;
}

// NewKeyFromSeed (ed25519.go:206-223): A = encode([s] B)
CB200_XHD void public_from_seed(uint32_t (&A)[8], const uint32_t (&seed)[8], const int32_t* __restrict__ table) {
  uint32_t s[8], prefix[8];
  expand_seed(s, prefix, seed);
  GeExt P;
  ge_scalarmult_base(P, s, table);
  ge_encode(A, P);
}

// Sign (ed25519.go:225-294) with A as given by the caller (the second half of the private key)
CB200_XHD void sign(uint32_t (&R)[8], uint32_t (&S)[8], const uint32_t (&seed)[8], const uint32_t (&A)[8], const uint8_t* msg,
                    uint64_t len, const int32_t* __restrict__ table) {
  uint32_t s[8], prefix[8], h[16], r[8], k[8], ra[16];
  expand_seed(s, prefix, seed);
  sha512<4>(h, prefix, msg, len);
  sc_reduce(r, h);
  GeExt P;
  ge_scalarmult_base(P, r, table);
  ge_encode(R, P);
#pragma unroll
  for (int i = 0; i < 8; i++) {
    ra[i] = R[i];
    ra[8 + i] = A[i];
  }
  sha512<8>(h, ra, msg, len);
  sc_reduce(k, h);
  sc_muladd(S, r, k, s);
}

// Verify (ed25519.go:329-368), cofactorless: S < L, A decodes, encode([S] B - [k] A) == R byte for byte
CB200_XHD bool verify(const uint32_t (&A)[8], const uint8_t* msg, uint64_t len, const uint32_t (&R)[8], const uint32_t (&S)[8],
                      const int32_t* __restrict__ table) {
  using namespace x25519;
  if (!sc_is_canonical(S)) return false;
  GeExt P;
  if (!ge_decode(P, A)) return false;
  Fe zero;
  fe_set(zero, 0);
  fe_sub(P.X, zero, P.X);  // -A
  fe_renorm(P.X);
  fe_sub(P.T, zero, P.T);
  fe_renorm(P.T);
  uint32_t ra[16], h[16], k[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    ra[i] = R[i];
    ra[8 + i] = A[i];
  }
  sha512<8>(h, ra, msg, len);
  sc_reduce(k, h);
  GeExt Q;
  ge_double_mult(Q, S, k, P, table);
  uint32_t enc[8];
  ge_encode(enc, Q);
  uint32_t diff = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) diff |= enc[i] ^ R[i];
  return diff == 0;
}

}  // namespace ed25519
}  // namespace cb200
