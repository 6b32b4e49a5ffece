// RSA blind signatures (RFC 9474, RSABSSA-SHA384), the server side of the reference's blindsign/blindrsa package:
// BlindSign (brsa.go:237-257 with DecryptAndCheck, internal/common/common.go:80-93) and Verify (brsa.go:214, verifyPSS
// and emsaPSSVerify, internal/common/common.go:121-137 and pss.go:132-221), one thread per operation.
//
//   Mod<W>        an odd modulus of W 32-bit words with its Montgomery constants (R = 2^(32 W)), prepared on the host
//   mont_mul      CIOS Montgomery product a b R^-1 mod m for a b < m R, with a masked final subtraction; one outlined
//                 copy per word count (32, 48, 64 for the CRT halves, 64, 96, 128 for the full modulus)
//   exp_secret    x^d by fixed 4-bit windows over every window of the modulus' bit length, the 16-entry table read
//                 whole under a mask at each window
//   exp_public    x^e by left-to-right square-and-multiply on the bits of the public e < 2^32
//   blind_sign    s_p = c^dp mod p, s_q = c^dq mod q, Garner's recombination with qinv, the check s^e mod N == c
//   verify        s^e mod N and the EMSA-PSS decode with MGF1-SHA-384
//
// Secret values (p, q, dp, dq, qinv, s_p, s_q) reach no branch and no address: every loop count and index comes from
// the word counts and the public bit lengths of p and q, the window digit only forms masks, and the final subtraction
// of mont_mul and the modular subtraction of Garner's step select with masks.  Public values (N, e, c, a Verify
// signature, the bit lengths) may branch.
//
// Plain integer C++ like nistp.cuh: it compiles for the device and for the host-only test of the CPU suite, and the
// library's host code prepares the constants with the same functions.
#pragma once
#include <cstdint>

#include "sha2.cuh"

#if defined(__CUDACC__)
#define CB200_RSA_NOINLINE static __host__ __device__ __noinline__
#else
#define CB200_RSA_NOINLINE static inline
#endif

namespace cb200 {
namespace rsa {

constexpr int kHash = 48;  // SHA-384

template <int W>
struct Mod {
  uint32_t m[W];   // the modulus, little-endian words
  uint32_t r2[W];  // R^2 mod m
  uint32_t r3[W];  // R^3 mod m
  uint32_t n0;     // -m^-1 mod 2^32
  int bits;        // bit length of m
};

// one private key under its word counts: the CRT halves at WP words, N at WN (WP <= WN <= 2 WP)
template <int WP, int WN>
struct SignKey {
  Mod<WP> p, q;
  uint32_t dp[WP], dq[WP], qinv[WP];
  Mod<WN> n;
  uint32_t e;
  int klen;  // bytes of N
};
template <int WN>
struct VerifyKey {
  Mod<WN> n;
  uint32_t e;
  int klen;
  int slen;  // salt length: 48 or 0
};

// a word of the key: the key is one read-only struct in global memory, and every thread of a warp reads the same word
CB200_XHD uint32_t ldk(const uint32_t* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}

// r = a b R^-1 mod m for a b < m R (a < R and b < m, or a < m and b < R), r < m.  r may alias a or b.
template <int W>
CB200_RSA_NOINLINE void mont_mul(uint32_t* r, const uint32_t* a, const uint32_t* b, const Mod<W>* M) {
  // b stays in registers where they suffice; the 96- and 128-word products read it from memory
  constexpr bool kReg = W <= 64;
  uint32_t bb[kReg ? W : 1];
  if constexpr (kReg) {
#pragma unroll
    for (int j = 0; j < W; j++) bb[j] = b[j];
  }
  const uint32_t n0 = ldk(&M->n0);
  uint32_t t[W + 2];
#pragma unroll
  for (int j = 0; j < W + 2; j++) t[j] = 0;
#pragma unroll 1
  for (int i = 0; i < W; i++) {
    const uint32_t ai = a[i];
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < W; j++) {
      c += (uint64_t)ai * (kReg ? bb[kReg ? j : 0] : b[j]) + t[j];
      t[j] = (uint32_t)c;
      c >>= 32;
    }
    c += t[W];
    t[W] = (uint32_t)c;
    t[W + 1] = (uint32_t)(c >> 32);
    const uint32_t u = t[0] * n0;
    c = ((uint64_t)u * ldk(&M->m[0]) + t[0]) >> 32;
#pragma unroll
    for (int j = 1; j < W; j++) {
      c += (uint64_t)u * ldk(&M->m[j]) + t[j];
      t[j - 1] = (uint32_t)c;
      c >>= 32;
    }
    c += t[W];
    t[W - 1] = (uint32_t)c;
    t[W] = t[W + 1] + (uint32_t)(c >> 32);
  }
  // t < 2m: keep t - m unless it borrows
  uint32_t d[W];
  uint32_t br = 0;
#pragma unroll
  for (int j = 0; j < W; j++) {
    const uint64_t x = (uint64_t)t[j] - ldk(&M->m[j]) - br;
    d[j] = (uint32_t)x;
    br = (uint32_t)(x >> 63);
  }
  const uint32_t keep = 0u - (uint32_t)(((uint64_t)t[W] - br) >> 63);
#pragma unroll
  for (int j = 0; j < W; j++) r[j] = (t[j] & keep) | (d[j] & ~keep);
}

// r = a - b mod m for a, b < m, the correction added under a mask
template <int W>
CB200_XHD void sub_mod(uint32_t* r, const uint32_t* a, const uint32_t* b, const Mod<W>* M) {
  uint32_t br = 0;
  for (int j = 0; j < W; j++) {
    const uint64_t x = (uint64_t)a[j] - b[j] - br;
    r[j] = (uint32_t)x;
    br = (uint32_t)(x >> 63);
  }
  const uint32_t mask = 0u - br;
  uint64_t c = 0;
  for (int j = 0; j < W; j++) {
    c += (uint64_t)r[j] + (ldk(&M->m[j]) & mask);
    r[j] = (uint32_t)c;
    c >>= 32;
  }
}

// r = a + b mod m for a, b < m, the subtraction kept under a mask
template <int W>
CB200_XHD void add_mod(uint32_t* r, const uint32_t* a, const uint32_t* b, const Mod<W>* M) {
  uint32_t s[W], d[W];
  uint64_t c = 0;
  for (int j = 0; j < W; j++) {
    c += (uint64_t)a[j] + b[j];
    s[j] = (uint32_t)c;
    c >>= 32;
  }
  uint32_t br = 0;
  for (int j = 0; j < W; j++) {
    const uint64_t x = (uint64_t)s[j] - ldk(&M->m[j]) - br;
    d[j] = (uint32_t)x;
    br = (uint32_t)(x >> 63);
  }
  const uint32_t keep = 0u - (uint32_t)(((uint64_t)(uint32_t)c - br) >> 63);
  for (int j = 0; j < W; j++) r[j] = (s[j] & keep) | (d[j] & ~keep);
}

// r = x^d R mod m from xm = x R mod m, for the secret d of W words of which the low M->bits count (d < m).  Every
// one of the ceil(bits / 4) windows costs four squarings and one product with a table entry selected by masks.
template <int W>
CB200_RSA_NOINLINE void exp_secret(uint32_t* r, const uint32_t* xm, const uint32_t* d, const Mod<W>* M) {
  uint32_t tbl[16][W], one[W];
  for (int j = 0; j < W; j++) one[j] = j == 0;
  mont_mul<W>(tbl[0], M->r2, one, M);  // R mod m
  for (int j = 0; j < W; j++) tbl[1][j] = xm[j];
#pragma unroll 1
  for (int k = 2; k < 16; k++) mont_mul<W>(tbl[k], tbl[k - 1], xm, M);
  for (int j = 0; j < W; j++) r[j] = tbl[0][j];
  const int nwin = (ldk((const uint32_t*)&M->bits) + 3) / 4;
  uint32_t sel[W];
#pragma unroll 1
  for (int w = nwin - 1; w >= 0; w--) {
#pragma unroll 1
    for (int s = 0; s < 4; s++) mont_mul<W>(r, r, r, M);
    const uint32_t digit = (ldk(&d[w >> 3]) >> (4 * (w & 7))) & 15;
#pragma unroll
    for (int j = 0; j < W; j++) sel[j] = 0;
#pragma unroll 1
    for (uint32_t k = 0; k < 16; k++) {
      const uint32_t mask = 0u - (uint32_t)(((k ^ digit) - 1u) >> 31);
#pragma unroll
      for (int j = 0; j < W; j++) sel[j] |= tbl[k][j] & mask;
    }
    mont_mul<W>(r, r, sel, M);
  }
}

// r = x^e R mod m from xm = x R mod m for a public e >= 1
template <int W>
CB200_RSA_NOINLINE void exp_public(uint32_t* r, const uint32_t* xm, uint32_t e, const Mod<W>* M) {
  int top = 31;
  while (!((e >> top) & 1)) top--;
  for (int j = 0; j < W; j++) r[j] = xm[j];
  for (int b = top - 1; b >= 0; b--) {
    mont_mul<W>(r, r, r, M);
    if ((e >> b) & 1) mont_mul<W>(r, r, xm, M);
  }
}

// ---------------------------------------------------------------- byte strings
// x (W words) = the len-byte big-endian string s, len <= 4 W
template <int W>
CB200_XHD void from_be(uint32_t* x, const uint8_t* s, int len) {
  for (int j = 0; j < W; j++) x[j] = 0;
  for (int i = 0; i < len; i++) {
    const int k = len - 1 - i;
    x[k >> 2] |= (uint32_t)s[i] << (8 * (k & 3));
  }
}
// byte i of the len-byte big-endian string of x
CB200_XHD uint8_t be_byte(const uint32_t* x, int len, int i) {
  const int k = len - 1 - i;
  return (uint8_t)(x[k >> 2] >> (8 * (k & 3)));
}
// compares two public W-word values: -1, 0, 1
template <int W>
CB200_XHD int cmp(const uint32_t* a, const uint32_t* b) {
  for (int j = W - 1; j >= 0; j--)
    if (a[j] != b[j]) return a[j] < b[j] ? -1 : 1;
  return 0;
}

// ---------------------------------------------------------------- BlindSign
// s = q h + s_q, with h = (s_p - s_q) qinv mod p (Garner), from spm = s_p R mod p and sq = s_q (< q); s has WN words
template <int WP, int WN>
CB200_XHD void garner(uint32_t* s, const uint32_t* spm, const uint32_t* sq, const SignKey<WP, WN>& K) {
  uint32_t sqm[WP], h[WP], qinv[WP];
  mont_mul<WP>(sqm, sq, K.p.r2, &K.p);  // s_q R mod p (s_q < q may exceed p)
  sub_mod<WP>(h, spm, sqm, &K.p);       // (s_p - s_q) R mod p
  for (int j = 0; j < WP; j++) qinv[j] = ldk(&K.qinv[j]);
  mont_mul<WP>(h, h, qinv, &K.p);  // (s_p - s_q) qinv mod p
  // s = q h + s_q < N: the product's words above WN are zero
  uint32_t acc[2 * WP];
  for (int j = 0; j < 2 * WP; j++) acc[j] = j < WP ? sq[j] : 0;
#pragma unroll 1
  for (int i = 0; i < WP; i++) {
    const uint32_t hi = h[i];
    uint64_t c = 0;
    for (int j = 0; j < WP; j++) {
      c += (uint64_t)hi * ldk(&K.q.m[j]) + acc[i + j];
      acc[i + j] = (uint32_t)c;
      c >>= 32;
    }
    acc[i + WP] = (uint32_t)c;  // no earlier row reached this word
  }
  for (int j = 0; j < WN; j++) s[j] = acc[j];
}

// BlindSign of the kLen-byte blinded message c under K: status 0 and s = c^d mod N in out (kLen bytes), or 1 for c > N
// (ErrInvalidMessageLength) and 2 for s^e mod N != c ("rsa: internal error"), with out all zero
template <int WP, int WN>
CB200_XHD uint32_t blind_sign(uint8_t* out, const uint8_t* in, const SignKey<WP, WN>& K) {
  const int klen = K.klen;
  uint32_t c[WN], nw[WN];
  from_be<WN>(c, in, klen);
  for (int j = 0; j < WN; j++) nw[j] = ldk(&K.n.m[j]);
  uint32_t st = cmp<WN>(c, nw) > 0 ? 1u : 0u;
  // c R mod p = c_hi R^3 R^-1 + c_lo R^2 R^-1 with c = c_hi R + c_lo (both below R = 2^(32 WP))
  uint32_t lo[WP], hi[WP], x[WP], y[WP], sp[WP], sq[WP];
  for (int j = 0; j < WP; j++) {
    lo[j] = c[j];
    hi[j] = j + WP < WN ? c[j + WP] : 0;
  }
  mont_mul<WP>(x, hi, K.p.r3, &K.p);
  mont_mul<WP>(y, lo, K.p.r2, &K.p);
  add_mod<WP>(x, x, y, &K.p);
  exp_secret<WP>(sp, x, K.dp, &K.p);  // s_p R mod p
  mont_mul<WP>(x, hi, K.q.r3, &K.q);
  mont_mul<WP>(y, lo, K.q.r2, &K.q);
  add_mod<WP>(x, x, y, &K.q);
  exp_secret<WP>(y, x, K.dq, &K.q);  // s_q R mod q
  for (int j = 0; j < WP; j++) x[j] = j == 0;
  mont_mul<WP>(sq, y, x, &K.q);  // s_q
  uint32_t s[WN], sm[WN], v[WN];
  garner<WP, WN>(s, sp, sq, K);
  // the check on the full modulus (DecryptAndCheck): s^e mod N must equal c
  mont_mul<WN>(sm, s, K.n.r2, &K.n);
  exp_public<WN>(v, sm, ldk(&K.e), &K.n);
  for (int j = 0; j < WN; j++) sm[j] = j == 0;
  mont_mul<WN>(v, v, sm, &K.n);
  uint32_t diff = 0;
  for (int j = 0; j < WN; j++) diff |= v[j] ^ c[j];
  if (!st && diff) st = 2;
  const uint32_t keep = st ? 0u : ~0u;
  for (int i = 0; i < klen; i++) out[i] = be_byte(s, klen, i) & keep;
  return st;
}

// ---------------------------------------------------------------- Verify
// SHA-384(0x00 * 8 || mHash || salt) for sLen salt bytes
CB200_XHD void pss_hash(uint64_t (&H)[8], const uint64_t (&mh)[8], const uint8_t* salt, int slen) {
  sha2::Sha384::iv(H);
  sha2::absorb<sha2::Sha384>(H, 0, 8 + kHash + slen, [&](int j) -> uint8_t {
    if (j < 8) return 0;
    if (j < 8 + kHash) return sha2::digest_byte<sha2::Sha384>(mh, j - 8);
    return salt[j - 8 - kHash];
  });
}

// EMSA-PSS-VERIFY (RFC 8017 section 9.1.2, pss.go:132-221) of m = s^e mod N (WN words, kLen bytes) against mHash:
// 0 if consistent, else 2.  emBits = bitlen(N) - 1; when that is a multiple of 8 the encoded message is the low
// kLen - 1 bytes of m, whose top byte must then be zero.
template <int WN>
CB200_XHD uint32_t emsa_pss_verify(const uint32_t* m, int klen, int nbits, const uint64_t (&mh)[8], int slen) {
  const int embits = nbits - 1, emlen = (embits + 7) / 8, off = klen - emlen;
  if (off && be_byte(m, klen, 0)) return 2;
  auto em = [&](int i) { return be_byte(m, klen, off + i); };
  if (emlen < kHash + slen + 2) return 2;
  if (em(emlen - 1) != 0xbc) return 2;
  const uint8_t bitmask = (uint8_t)(0xff >> (8 * emlen - embits));
  if (em(0) & ~bitmask) return 2;
  const int dblen = emlen - kHash - 1, pslen = dblen - slen - 1;
  uint8_t salt[kHash];
  uint32_t bad = 0;
  for (int blk = 0; blk * kHash < dblen; blk++) {
    uint64_t H[8];
    sha2::Sha384::iv(H);
    sha2::absorb<sha2::Sha384>(H, 0, kHash + 4, [&](int j) -> uint8_t {
      return j < kHash ? em(dblen + j) : (uint8_t)((uint32_t)blk >> (8 * (kHash + 3 - j)));
    });
    for (int k = 0; k < kHash; k++) {
      const int i = blk * kHash + k;
      if (i >= dblen) break;
      uint8_t db = em(i) ^ sha2::digest_byte<sha2::Sha384>(H, k);
      if (i == 0) db &= bitmask;
      if (i < pslen) bad |= db;
      else if (i == pslen) bad |= db ^ 1;
      else salt[i - pslen - 1] = db;
    }
  }
  uint64_t h2[8];
  pss_hash(h2, mh, salt, slen);
  for (int j = 0; j < kHash; j++) bad |= sha2::digest_byte<sha2::Sha384>(h2, j) ^ em(dblen + j);
  return bad ? 2 : 0;
}

// Verify of the message msg[0 .. len) and the kLen-byte signature sig under K: 0, 1 for s >= N, 2 for an inconsistent
// encoding (both rsa.ErrVerification in the reference)
template <int WN>
CB200_XHD uint32_t verify(const uint8_t* msg, uint64_t len, const uint8_t* sig, const VerifyKey<WN>& K) {
  const int klen = K.klen;
  uint32_t s[WN], nw[WN], sm[WN], v[WN];
  from_be<WN>(s, sig, klen);
  for (int j = 0; j < WN; j++) nw[j] = ldk(&K.n.m[j]);
  if (cmp<WN>(s, nw) >= 0) return 1;
  mont_mul<WN>(sm, s, K.n.r2, &K.n);
  exp_public<WN>(v, sm, ldk(&K.e), &K.n);
  for (int j = 0; j < WN; j++) sm[j] = j == 0;
  mont_mul<WN>(v, v, sm, &K.n);
  uint64_t mh[8];
  sha2::Sha384::iv(mh);
  sha2::absorb<sha2::Sha384>(mh, 0, (int)len, [&](int j) -> uint8_t { return msg[j]; });
  return emsa_pss_verify<WN>(v, klen, ldk((const uint32_t*)&K.n.bits), mh, ldk((const uint32_t*)&K.slen));
}

// ---------------------------------------------------------------- host preparation
// M from the odd modulus m > 1 of W words: n0 by Newton's iteration, R^2 mod m from R mod m (32 W modular doublings of
// 1) by t more doublings and s Montgomery squarings with t 2^s = 32 W (each squaring doubles the exponent of 2 over R),
// R^3 = R^2 R^2 R^-1.  The doublings keep their subtraction under a mask.
template <int W>
inline void mod_init(Mod<W>& M, const uint32_t* m) {
  for (int j = 0; j < W; j++) M.m[j] = m[j];
  uint32_t inv = m[0];
  for (int i = 0; i < 5; i++) inv *= 2u - m[0] * inv;
  M.n0 = 0u - inv;
  M.bits = 0;
  for (int j = W - 1; j >= 0 && !M.bits; j--)
    if (m[j])
      for (int b = 31; b >= 0; b--)
        if ((m[j] >> b) & 1) {
          M.bits = 32 * j + b + 1;
          break;
        }
  int s = 0, t = 32 * W;
  while (!(t & 1)) t >>= 1, s++;
  uint32_t x[W];
  for (int j = 0; j < W; j++) x[j] = j == 0;
  for (int i = 0; i < 32 * W + t; i++) add_mod<W>(x, x, x, &M);  // x < m after the first step since m > 1
  for (int i = 0; i < s; i++) mont_mul<W>(x, x, x, &M);
  for (int j = 0; j < W; j++) M.r2[j] = x[j];
  mont_mul<W>(M.r3, M.r2, M.r2, &M);
}

}  // namespace rsa
}  // namespace cb200
