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
//   crt_sign      the BlindSign body: s_p = c^d_p mod p and s_q = c^d_q mod q by the caller's exponentiations,
//                 Garner's recombination with qinv, the check s^e mod N == c by the caller's public exponentiation
//   pss_verify    the Verify body: s^e mod N by the caller's exponentiation, SHA-384 of the message bytes the caller
//                 gives and the EMSA-PSS decode with MGF1-SHA-384
//   blind_sign    crt_sign with dp and dq from the key and its 32-bit e
//   verify        pss_verify with the 32-bit e and the message as it is
//   pb_*          partially blind RSA (RSAPBSSA-SHA384, partiallyblindrsa/pbrsa.go): e' from the metadata by
//                 HKDF-SHA-384, d' by Fermat inversion mod p' = (p - 1) / 2 and q', exp_public_words for the
//                 multi-word e', on the same two bodies; see that section
//   tss_*         threshold RSA (tss/rsa): signature shares by exp_windows over a public bound, and the combination of
//                 k shares with mod_inverse for the public values it inverts; see that section
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

// r = x^d R mod m from xm = x R mod m, for the secret d below 2^bits(), with bits() public: bitlen(m) for an exponent
// reduced mod m, a public bound otherwise (read once, after the table is built).  Every one of the ceil(bits / 4)
// windows costs four squarings and one product with a table entry selected by masks.  digit(w) reads window w of d.
template <int W, class Digit, class Bits>
CB200_XHD void exp_windows(uint32_t* r, const uint32_t* xm, const Digit& digit_of, const Bits& bits, const Mod<W>* M) {
  uint32_t tbl[16][W], one[W];
  for (int j = 0; j < W; j++) one[j] = j == 0;
  mont_mul<W>(tbl[0], M->r2, one, M);  // R mod m
  for (int j = 0; j < W; j++) tbl[1][j] = xm[j];
#pragma unroll 1
  for (int k = 2; k < 16; k++) mont_mul<W>(tbl[k], tbl[k - 1], xm, M);
  for (int j = 0; j < W; j++) r[j] = tbl[0][j];
  const int nwin = (bits() + 3) / 4;
  uint32_t sel[W];
#pragma unroll 1
  for (int w = nwin - 1; w >= 0; w--) {
#pragma unroll 1
    for (int s = 0; s < 4; s++) mont_mul<W>(r, r, r, M);
    const uint32_t digit = digit_of(w);
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
// d in the key (global memory on the device)
template <int W>
CB200_RSA_NOINLINE void exp_secret(uint32_t* r, const uint32_t* xm, const uint32_t* d, const Mod<W>* M) {
  exp_windows<W>(r, xm, [&](int w) { return (ldk(&d[w >> 3]) >> (4 * (w & 7))) & 15; },
                 [&] { return ldk((const uint32_t*)&M->bits); }, M);
}
// d in the thread's own memory (an exponent computed per operation)
template <int W>
CB200_RSA_NOINLINE void exp_secret_own(uint32_t* r, const uint32_t* xm, const uint32_t* d, const Mod<W>* M) {
  exp_windows<W>(r, xm, [&](int w) { return (d[w >> 3] >> (4 * (w & 7))) & 15; },
                 [&] { return ldk((const uint32_t*)&M->bits); }, M);
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
// s = q h + s_q, with h = (s_p - s_q) qinv mod p (Garner), from spm = s_p R mod p and sq = s_q (< q); s has WN words.
// K: a key with the members p, q (Mod<WP>) and qinv.
template <int WP, int WN, class Key>
CB200_XHD void garner(uint32_t* s, const uint32_t* spm, const uint32_t* sq, const Key& K) {
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

// CRT BlindSign of the kLen-byte blinded message c under K (members p, q, qinv, n, klen), the body of blind_sign and
// pb_blind_sign: status 0 and s = c^d mod N in out (kLen bytes), or 1 for c > N (ErrInvalidMessageLength) and 2 for
// s^e mod N != c ("rsa: internal error"), with out all zero.  The caller supplies the exponentiations:
//   prep()            runs once after the c > N test
//   half_p(r, cm)     r = c^d_p R mod p from cm = c R mod p; half_q the same mod q
//   pub(v, sm)        v = s^e R mod N from sm = s R mod N
template <int WP, int WN, class Key, class Prep, class HalfP, class HalfQ, class Pub>
CB200_XHD uint32_t crt_sign(uint8_t* out, const uint8_t* in, const Key& K, const Prep& prep, const HalfP& half_p,
                            const HalfQ& half_q, const Pub& pub) {
  const int klen = K.klen;
  uint32_t c[WN], nw[WN];
  from_be<WN>(c, in, klen);
  for (int j = 0; j < WN; j++) nw[j] = ldk(&K.n.m[j]);
  uint32_t st = cmp<WN>(c, nw) > 0 ? 1u : 0u;
  prep();
  // c R mod p = c_hi R^3 R^-1 + c_lo R^2 R^-1 with c = c_hi R + c_lo (both below R = 2^(32 WP))
  uint32_t lo[WP], hi[WP], x[WP], y[WP], sp[WP], sq[WP];
  for (int j = 0; j < WP; j++) {
    lo[j] = c[j];
    hi[j] = j + WP < WN ? c[j + WP] : 0;
  }
  auto to_mont = [&](const Mod<WP>& P) {  // x = c R mod P
    mont_mul<WP>(x, hi, P.r3, &P);
    mont_mul<WP>(y, lo, P.r2, &P);
    add_mod<WP>(x, x, y, &P);
  };
  to_mont(K.p);
  half_p(sp, x);  // s_p R mod p
  to_mont(K.q);
  half_q(y, x);  // s_q R mod q
  for (int j = 0; j < WP; j++) x[j] = j == 0;
  mont_mul<WP>(sq, y, x, &K.q);  // s_q
  uint32_t s[WN], sm[WN], v[WN];
  garner<WP, WN>(s, sp, sq, K);
  // the check on the full modulus (DecryptAndCheck): s^e mod N must equal c
  mont_mul<WN>(sm, s, K.n.r2, &K.n);
  pub(v, sm);
  for (int j = 0; j < WN; j++) sm[j] = j == 0;
  mont_mul<WN>(v, v, sm, &K.n);
  uint32_t diff = 0;
  for (int j = 0; j < WN; j++) diff |= v[j] ^ c[j];
  if (!st && diff) st = 2;
  const uint32_t keep = st ? 0u : ~0u;
  for (int i = 0; i < klen; i++) out[i] = be_byte(s, klen, i) & keep;
  return st;
}

// BlindSign of the kLen-byte blinded message c under K: crt_sign with s_p = c^dp mod p, s_q = c^dq mod q and the
// 32-bit e
template <int WP, int WN>
CB200_XHD uint32_t blind_sign(uint8_t* out, const uint8_t* in, const SignKey<WP, WN>& K) {
  return crt_sign<WP, WN>(
      out, in, K, [] {}, [&](uint32_t* r, const uint32_t* cm) { exp_secret<WP>(r, cm, K.dp, &K.p); },
      [&](uint32_t* r, const uint32_t* cm) { exp_secret<WP>(r, cm, K.dq, &K.q); },
      [&](uint32_t* v, const uint32_t* sm) { exp_public<WN>(v, sm, ldk(&K.e), &K.n); });
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

// Verify of the kLen-byte signature sig under K (members n, klen), the body of verify and pb_verify, for the message
// of len bytes whose byte j is msg(j), with a salt of salt_len(K) bytes: 0, 1 for s >= N, 2 for an inconsistent
// encoding (both rsa.ErrVerification in the reference).  prep() runs once after the s >= N test; pub(v, sm) gives
// v = s^e R mod N from sm = s R mod N.
template <int WN, class Key, class Prep, class Pub, class Msg>
CB200_XHD uint32_t pss_verify(const uint8_t* sig, const Key& K, const Prep& prep, const Pub& pub, uint64_t len,
                              const Msg& msg) {
  const int klen = K.klen;
  uint32_t s[WN], nw[WN], sm[WN], v[WN];
  from_be<WN>(s, sig, klen);
  for (int j = 0; j < WN; j++) nw[j] = ldk(&K.n.m[j]);
  if (cmp<WN>(s, nw) >= 0) return 1;
  prep();
  mont_mul<WN>(sm, s, K.n.r2, &K.n);
  pub(v, sm);
  for (int j = 0; j < WN; j++) sm[j] = j == 0;
  mont_mul<WN>(v, v, sm, &K.n);
  uint64_t mh[8];
  sha2::Sha384::iv(mh);
  sha2::absorb<sha2::Sha384>(mh, 0, (int)len, msg);
  return emsa_pss_verify<WN>(v, klen, ldk((const uint32_t*)&K.n.bits), mh, salt_len(K));
}

// RSABSSA-SHA384's salt: 48 bytes or none by the variant
template <int WN>
CB200_XHD int salt_len(const VerifyKey<WN>& K) { return ldk((const uint32_t*)&K.slen); }
// Verify of the message msg[0 .. len) and the kLen-byte signature sig under K: pss_verify with the 32-bit e
template <int WN>
CB200_XHD uint32_t verify(const uint8_t* msg, uint64_t len, const uint8_t* sig, const VerifyKey<WN>& K) {
  return pss_verify<WN>(
      sig, K, [] {}, [&](uint32_t* v, const uint32_t* sm) { exp_public<WN>(v, sm, ldk(&K.e), &K.n); }, len,
      [&](int j) -> uint8_t { return msg[j]; });
}

// ---------------------------------------------------------------- partially blind RSA (RSAPBSSA-SHA384)
// draft-amjad-cfrg-partially-blind-rsa as the reference's blindsign/blindrsa/partiallyblindrsa (pbrsa.go): every
// metadata value selects the key (N, e') and d' = e'^-1 mod phi(N), derived per operation.  The primes are safe,
// p = 2 p' + 1 with p' prime and p = 3 mod 4.  e' has fewer than lambda = bitlen(N) / 2 bits, so it fits in WN / 2
// words, never more than WP.  p', q', p' - 2, q' - 2, d'_p, d'_q, s_p and s_q are secret under the rules above; e'
// and the metadata are public.
template <int WN>
struct PbVerifyKey {
  Mod<WN> n;
  uint64_t si[8], so[8];  // HMAC-SHA-384 pad states of HKDF's salt N (kLen bytes, longer than a block: SHA-384(N))
  int klen;
};
template <int WP, int WN>
struct PbSignKey {
  Mod<WP> p, q;
  Mod<WP> ph, qh;             // p' = (p - 1) / 2, q' = (q - 1) / 2
  uint32_t ph2[WP], qh2[WP];  // p' - 2, q' - 2: Fermat's exponents
  uint32_t qinv[WP];
  Mod<WN> n;
  uint64_t si[8], so[8];
  int klen;
};

// bits of e' that can be set: the first lambda / 8 bytes, bits lambda - 1 and lambda - 2 clear
CB200_XHD int pb_exp_bits(int nbits) {
  const int lambda = nbits / 2;
  return lambda - 2 < 8 * (lambda / 8) ? lambda - 2 : 8 * (lambda / 8);
}

// e' (WN / 2 words) of derivePublicKey (pbrsa.go:81-117) for the metadata meta[0 .. mlen): HKDF-SHA-384 with salt N,
// IKM "key" || meta || 0x00 and info "PBRSA", its first lambda / 8 bytes read big-endian, bit 0 set and bits lambda - 1
// and lambda - 2 cleared.  Only the Expand blocks holding those bytes are computed: a block does not depend on the
// output length.  si / so: the salt's pad states (PbVerifyKey).
template <int WN>
CB200_XHD void derive_exponent(uint32_t* e, int nbits, const uint8_t* meta, int mlen, const uint64_t (&si)[8],
                               const uint64_t (&so)[8]) {
  using S = sha2::Sha384;
  uint64_t prk[8], ki[8], ko[8], t[8], prev[8];
  sha2::hmac<S>(prk, si, so, mlen + 4, [&](int j) -> uint8_t {
    if (j < 3) return (uint8_t)"key"[j];
    return j - 3 < mlen ? meta[j - 3] : 0;
  });
  sha2::hmac_key<S>(ki, ko, prk);
  const int lambda = nbits / 2, nb = lambda / 8;
  for (int j = 0; j < WN / 2; j++) e[j] = 0;
#pragma unroll 1
  for (int blk = 0; blk * kHash < nb; blk++) {
    const int tl = blk ? kHash : 0;  // T(0) is empty
    for (int i = 0; i < 8; i++) prev[i] = t[i];
    sha2::hmac<S>(t, ki, ko, tl + 6, [&](int j) -> uint8_t {
      if (j < tl) return sha2::digest_byte<S>(prev, j);
      return j < tl + 5 ? (uint8_t)"PBRSA"[j - tl] : (uint8_t)(blk + 1);
    });
    for (int k = 0; k < kHash && blk * kHash + k < nb; k++) {
      const int i = nb - 1 - (blk * kHash + k);  // byte index from the least significant end
      e[i >> 2] |= (uint32_t)sha2::digest_byte<S>(t, k) << (8 * (i & 3));
    }
  }
  e[0] |= 1;
  for (int b = lambda - 2; b < lambda; b++)
    if (b < 8 * nb) e[b >> 5] &= ~(1u << (b & 31));
}

// r = x^e R mod m from xm = x R mod m for a public e below 2^bits: fixed windows of kPubWin bits from the top, each
// kPubWin squarings and one product with the table entry of its digit (entry 0 is R mod m, so a zero digit costs the
// same product).  The sequence of products depends on `bits` alone, so the threads of a warp, which share N, run in
// step whatever their e.
constexpr int kPubWin = 5;
template <int W>
CB200_RSA_NOINLINE void exp_public_words(uint32_t* r, const uint32_t* xm, const uint32_t* e, int bits, const Mod<W>* M) {
  uint32_t tbl[1 << kPubWin][W], one[W];
  for (int j = 0; j < W; j++) one[j] = j == 0;
  mont_mul<W>(tbl[0], M->r2, one, M);
  for (int j = 0; j < W; j++) tbl[1][j] = xm[j];
#pragma unroll 1
  for (int k = 2; k < (1 << kPubWin); k++) mont_mul<W>(tbl[k], tbl[k - 1], xm, M);
  const int nw = (bits + 31) / 32, nwin = (bits + kPubWin - 1) / kPubWin;
  auto digit = [&](int b) {  // bits b .. b + kPubWin - 1 of e
    uint32_t v = e[b >> 5] >> (b & 31);
    if ((b & 31) > 32 - kPubWin && (b >> 5) + 1 < nw) v |= e[(b >> 5) + 1] << (32 - (b & 31));
    return v & ((1u << kPubWin) - 1);
  };
  const uint32_t* top = tbl[digit(kPubWin * (nwin - 1))];
  for (int j = 0; j < W; j++) r[j] = top[j];
#pragma unroll 1
  for (int w = nwin - 2; w >= 0; w--) {
#pragma unroll 1
    for (int s = 0; s < kPubWin; s++) mont_mul<W>(r, r, r, M);
    mont_mul<W>(r, r, tbl[digit(kPubWin * w)], M);
  }
}

// s_p R mod p = c^d'_p R mod p from cm = c R mod p, with d'_p = e'^-1 mod (p - 1) = 2 p': x = e'^(p' - 2) mod p'
// (Fermat's inverse, p' prime), lifted to its odd representative below 2 p' (e' is odd, so is d'_p) by adding p' under
// a mask.  e: e' in WP words; H: p'; h2: p' - 2.
template <int WP>
CB200_XHD void pb_half(uint32_t* sm, const uint32_t* cm, const uint32_t* e, const Mod<WP>& P, const Mod<WP>& H,
                       const uint32_t* h2) {
  uint32_t x[WP], d[WP];
  mont_mul<WP>(x, e, H.r2, &H);  // e' R mod p' (e' < R)
  exp_secret<WP>(d, x, h2, &H);
  for (int j = 0; j < WP; j++) x[j] = j == 0;
  mont_mul<WP>(d, d, x, &H);
  const uint32_t even = (d[0] & 1) - 1u;
  uint64_t c = 0;
  for (int j = 0; j < WP; j++) {
    c += (uint64_t)d[j] + (ldk(&H.m[j]) & even);
    d[j] = (uint32_t)c;
    c >>= 32;
  }
  exp_secret_own<WP>(sm, cm, d, &P);
}

// BlindSign (pbrsa.go:350-375) of the kLen-byte blinded message c under the key of meta[0 .. mlen): crt_sign with e'
// derived once c has been read, d'_p and d'_q by pb_half, and the check s^e' mod N == c
template <int WP, int WN>
CB200_XHD uint32_t pb_blind_sign(uint8_t* out, const uint8_t* in, const uint8_t* meta, int mlen,
                                 const PbSignKey<WP, WN>& K) {
  const int nbits = ldk((const uint32_t*)&K.n.bits);
  uint32_t e[WP];
  return crt_sign<WP, WN>(
      out, in, K,
      [&] {
        derive_exponent<WN>(e, nbits, meta, mlen, K.si, K.so);
        for (int j = WN / 2; j < WP; j++) e[j] = 0;
      },
      [&](uint32_t* r, const uint32_t* cm) { pb_half<WP>(r, cm, e, K.p, K.ph, K.ph2); },
      [&](uint32_t* r, const uint32_t* cm) { pb_half<WP>(r, cm, e, K.q, K.qh, K.qh2); },
      [&](uint32_t* v, const uint32_t* sm) { exp_public_words<WN>(v, sm, e, pb_exp_bits(nbits), &K.n); });
}

// RSAPBSSA-SHA384's salt: 48 bytes
template <int WN>
CB200_XHD int salt_len(const PbVerifyKey<WN>&) { return kHash; }
// Verify (pbrsa.go:244-251) of msg[0 .. len) under the metadata meta[0 .. mlen) and the kLen-byte signature: the
// message framed as "msg" || I2OSP(mlen, 4) || meta || msg, pss_verify under (N, e').  7 + mlen + len < 2^31.
template <int WN>
CB200_XHD uint32_t pb_verify(const uint8_t* msg, int len, const uint8_t* meta, int mlen, const uint8_t* sig,
                             const PbVerifyKey<WN>& K) {
  const int nbits = ldk((const uint32_t*)&K.n.bits);
  uint32_t e[WN / 2];
  return pss_verify<WN>(
      sig, K, [&] { derive_exponent<WN>(e, nbits, meta, mlen, K.si, K.so); },
      [&](uint32_t* v, const uint32_t* sm) { exp_public_words<WN>(v, sm, e, pb_exp_bits(nbits), &K.n); },
      7 + mlen + len, [&](int j) -> uint8_t {
        if (j < 3) return (uint8_t)"msg"[j];
        if (j < 7) return (uint8_t)((uint32_t)mlen >> (8 * (6 - j)));
        return j - 7 < mlen ? meta[j - 7] : msg[j - 7 - mlen];
      });
}

// ---------------------------------------------------------------- threshold RSA (tss/rsa, Shoup's protocol 1)
// The reference's tss/rsa package: a party holding the key share s_i signs x with x^(2 Delta s_i) mod N
// (KeyShare.Sign, keyshare.go:188-256), and a combiner turns k >= threshold such shares into the RSA signature
// (CombineSignShares, rsa_threshold.go:207-293), with Delta = players!.  Served: 2 <= players <= kTssMaxPlayers,
// u16 indices, k <= kTssMaxPlayers shares per op.  Then 2 Delta < 2^297 (kDeltaWords), e' = 4 Delta^2 < 2^594
// (kEpWords) and |2 lambda| < 2 Delta 65535^63 < 2^1305 (kLambdaWords).
//   tss_sign_share  x^E mod N for the secret E = 2 Delta s_i (or the share's cached value) by exp_windows over the
//                   public bound bitlen(N) - 2 + bitlen(2 Delta) on bitlen(E); E reaches no branch and no address
//   mod_inverse     a^-1 R mod m from a R mod m for a public a and an odd composite m, by binary extended Euclid
//                   (variable-time: every value Combine inverts is public)
//   tss_lambda      lambda_j of computeLambda (rsa_threshold.go:315-349) for i = 0
//   tss_combine     CombineSignShares of one op from the k shares, its index set and x
constexpr int kTssMaxPlayers = 64;
constexpr int kDeltaWords = 10;
constexpr int kEpWords = 19;
constexpr int kLambdaWords = 41;

template <int WN>
struct TssSignKey {
  Mod<WN> n;
  uint32_t e[WN + kDeltaWords];  // E, little-endian
  int ebits;                     // the public bound on bitlen(E) the windows run over
  int klen;
};
template <int WN>
struct TssCombineKey {
  Mod<WN> n;
  uint32_t e;                    // the public exponent
  uint32_t delta[kDeltaWords];   // Delta = players!
  uint32_t a;                    // |a| and |b| of e' a + e b = gcd(e', e), with their signs and bit lengths
  uint32_t b[kEpWords];
  int a_neg, b_neg, a_bits, b_bits;
  int k;                         // shares per op
  int klen;
};

// xi = x^E mod N (kLen bytes) of the kLen-byte x (x < R, so x R mod N = x R^2 R^-1 reduces it, as Exp does)
template <int WN>
CB200_XHD void tss_sign_share(uint8_t* out, const uint8_t* in, const TssSignKey<WN>& K) {
  const int klen = K.klen;
  uint32_t x[WN], r[WN];
  from_be<WN>(x, in, klen);
  mont_mul<WN>(x, x, K.n.r2, &K.n);
  exp_windows<WN>(r, x, [&](int w) { return (ldk(&K.e[w >> 3]) >> (4 * (w & 7))) & 15; },
                  [&] { return ldk((const uint32_t*)&K.ebits); }, &K.n);
  for (int j = 0; j < WN; j++) x[j] = j == 0;
  mont_mul<WN>(r, r, x, &K.n);
  for (int i = 0; i < klen; i++) out[i] = be_byte(r, klen, i);
}

// trailing and leading zero bits of x != 0
CB200_XHD int ctz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __ffs(x) - 1;
#else
  return __builtin_ctz(x);
#endif
}
CB200_XHD int clz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __clz(x);
#else
  return __builtin_clz(x);
#endif
}

// r = a^-1 R mod m from a = a' R mod m (a < m), for the odd m: true, or false if gcd(a, m) != 1 (a = 0 included).
// Binary extended Euclid on (u, v) = (a, m) with x1 a = u, x2 a = v mod m: strip u's (v's) trailing zeros, up to 32 a
// step, dividing x1 (x2) by 2^s mod m as Montgomery's reduction does (add k m with k = x1 (-m^-1) mod 2^s), then
// subtract the smaller of u, v from the larger.  Ends at u = 1 or v = 1 with x = (a' R)^-1, and x R^3 R^-1 = a'^-1 R.
// Every value it sees is public, so it branches freely.
template <int W>
CB200_RSA_NOINLINE bool mod_inverse(uint32_t* r, const uint32_t* a, const Mod<W>* M) {
  uint32_t u[W], v[W], x1[W], x2[W];
  for (int j = 0; j < W; j++) u[j] = a[j], v[j] = ldk(&M->m[j]), x1[j] = j == 0, x2[j] = 0;
  const uint32_t n0 = ldk(&M->n0);
  auto is_small = [](const uint32_t* x, uint32_t c) {
    if (x[0] != c) return false;
    for (int j = 1; j < W; j++)
      if (x[j]) return false;
    return true;
  };
  auto strip = [&](uint32_t* x, uint32_t* c) {  // x even and not zero: x >>= s, c = c 2^-s mod m
    while (!(x[0] & 1)) {
      const int s = x[0] ? ctz32(x[0]) : 32;
      for (int j = 0; j < W; j++)
        x[j] = (uint32_t)(((uint64_t)(j + 1 < W ? x[j + 1] : 0) << 32 | x[j]) >> s);
      const uint32_t k = (c[0] * n0) & (s == 32 ? ~0u : (1u << s) - 1);
      uint64_t cy = 0;
      uint32_t lo = 0;
      for (int j = 0; j < W; j++) {  // (c + k m) >> s < m
        cy += (uint64_t)k * ldk(&M->m[j]) + c[j];
        const uint32_t t = (uint32_t)cy;
        cy >>= 32;
        if (j) c[j - 1] = (uint32_t)(((uint64_t)t << 32 | lo) >> s);
        lo = t;
      }
      c[W - 1] = (uint32_t)((cy << 32 | lo) >> s);
    }
  };
  auto sub = [](uint32_t* x, const uint32_t* y) {
    uint32_t br = 0;
    for (int j = 0; j < W; j++) {
      const uint64_t d = (uint64_t)x[j] - y[j] - br;
      x[j] = (uint32_t)d;
      br = (uint32_t)(d >> 63);
    }
  };
  if (is_small(u, 0)) return false;
  while (!is_small(u, 1) && !is_small(v, 1)) {
    if (is_small(u, 0) || is_small(v, 0)) return false;  // the gcd is the other one, above 1
    strip(u, x1);
    strip(v, x2);
    if (cmp<W>(u, v) >= 0) {
      sub(u, v);
      sub_mod<W>(x1, x1, x2, M);
    } else {
      sub(v, u);
      sub_mod<W>(x2, x2, x1, M);
    }
  }
  mont_mul<W>(r, is_small(u, 1) ? x1 : x2, M->r3, M);
  return true;
}

// |lambda_j| (kLambdaWords words, returned in lam) and its sign for j = idx(t) over the index set idx(0 .. k) with
// i = 0: lambda = Delta prod_{j' != j} (0 - j') / prod_{j' != j} (j - j'), as computeLambda.  Returns 1 (ErrInvalidCalc)
// if an index is 0 (checkIndices: i = 0 must not be in S) or the quotient is not an integer, else 0.  Delta prod j' is
// formed first, then divided by each |j - j'| in turn: the divisions are all exact iff the product of the divisors
// divides it.  A repeated index is skipped like j itself, as the reference does, so the denominator is never zero.
template <class Idx>
CB200_XHD uint32_t tss_lambda(uint32_t* lam, bool* neg, const Idx& idx, int t, int k, const uint32_t* delta) {
  const uint32_t j = idx(t);
  for (int i = 0; i < kLambdaWords; i++) lam[i] = i < kDeltaWords ? ldk(&delta[i]) : 0;
  bool s = false;
  for (int u = 0; u < k; u++) {
    const uint32_t jp = idx(u);
    if (jp == 0) return 1;
    if (jp == j) continue;
    s = s != (jp < j);  // (0 - j') / (j - j') < 0 iff j' < j: the sign flips exactly then
    uint64_t c = 0;
    for (int i = 0; i < kLambdaWords; i++) {
      c += (uint64_t)lam[i] * jp;
      lam[i] = (uint32_t)c;
      c >>= 32;
    }
  }
  for (int u = 0; u < k; u++) {
    const uint32_t jp = idx(u);
    if (jp == j) continue;
    const uint32_t d = jp > j ? jp - j : j - jp;
    uint64_t rem = 0;
    for (int i = kLambdaWords - 1; i >= 0; i--) {
      const uint64_t cur = rem << 32 | lam[i];
      lam[i] = (uint32_t)(cur / d);
      rem = cur % d;
    }
    if (rem) return 1;
  }
  *neg = s;
  return 0;
}

// bit length of a public value of n words
CB200_XHD int bits_of(const uint32_t* x, int n) {
  for (int j = n - 1; j >= 0; j--)
    if (x[j]) return 32 * j + 32 - clz32(x[j]);
  return 0;
}

// CombineSignShares (rsa_threshold.go:207-293) of one op: the k shares xi(t) (kLen bytes each) of the indices idx(t)
// and the kLen-byte x -> y (kLen bytes) and 0, or 1 (ErrInvalidCalc from computeLambda) or 2 ("rsa: internal error":
// y^e mod N != x, x unreduced), with out all zero.  The parameter checks before the lambdas are the host's.
//   w = prod_t xi_t^(2 lambda_t) = P / Q with P the product of the terms of positive lambda and Q of the negative ones,
//   y = w^a x^b mod N.
// The reference inverts each negative term, then w if a < 0, then x if b < 0.  All of them are invertible iff
// D = Q (P if a < 0) (x if b < 0) is, and one inverse of D then gives each of them.  Otherwise the reference's
// sequence runs as it is: a term whose inverse fails stays as it was (ModInverse leaves it unchanged), and a power
// with a negative exponent of a base without an inverse is 0 (Exp leaves its fresh result at 0).
template <int WN, class Idx, class Xi>
CB200_XHD uint32_t tss_combine(uint8_t* out, const Idx& idx, const Xi& xi, const uint8_t* msg,
                               const TssCombineKey<WN>& K) {
  const int klen = K.klen, k = ldk((const uint32_t*)&K.k);
  const Mod<WN>* M = &K.n;
  uint32_t lam[kLambdaWords];
  bool neg;
  for (int i = 0; i < klen; i++) out[i] = 0;
  for (int t = 0; t < k; t++)
    if (tss_lambda(lam, &neg, idx, t, k, K.delta)) return 1;
  uint32_t one[WN], mone[WN], P[WN], Q[WN], x[WN], xm[WN], tm[WN];
  for (int j = 0; j < WN; j++) one[j] = j == 0;
  mont_mul<WN>(mone, M->r2, one, M);  // R mod N
  // tm = xi_t^|2 lambda_t| R mod N
  auto term = [&](int t) {
    tss_lambda(lam, &neg, idx, t, k, K.delta);
    for (int i = kLambdaWords - 1; i > 0; i--) lam[i] = lam[i] << 1 | lam[i - 1] >> 31;
    lam[0] <<= 1;
    from_be<WN>(tm, xi(t), klen);
    mont_mul<WN>(tm, tm, M->r2, M);
    exp_public_words<WN>(tm, tm, lam, bits_of(lam, kLambdaWords), M);
  };
  for (int j = 0; j < WN; j++) P[j] = Q[j] = mone[j];
  for (int t = 0; t < k; t++) {
    term(t);
    mont_mul<WN>(neg ? Q : P, neg ? Q : P, tm, M);
  }
  from_be<WN>(x, msg, klen);
  mont_mul<WN>(xm, x, M->r2, M);
  const bool a_neg = ldk((const uint32_t*)&K.a_neg), b_neg = ldk((const uint32_t*)&K.b_neg);
  uint32_t D[WN], ba[WN], bb[WN];  // the bases of |a| and |b|
  bool za = false, zb = false;     // a base that is 0 (a failed inverse of Exp)
  for (int j = 0; j < WN; j++) D[j] = Q[j];
  if (a_neg) mont_mul<WN>(D, D, P, M);
  if (b_neg) mont_mul<WN>(D, D, xm, M);
  if (mod_inverse<WN>(D, D, M)) {
    // D^-1 Q = (P if a < 0)^-1 (x if b < 0)^-1, D^-1 (D / Q) = Q^-1
    mont_mul<WN>(tm, D, Q, M);
    if (b_neg) mont_mul<WN>(bb, tm, a_neg ? P : mone, M);  // x^-1
    else for (int j = 0; j < WN; j++) bb[j] = xm[j];
    if (a_neg) {  // w^-1 = Q P^-1 = Q (D^-1 Q (x if b < 0))
      mont_mul<WN>(ba, tm, b_neg ? xm : mone, M);
      mont_mul<WN>(ba, ba, Q, M);
    } else {  // w = P Q^-1 = P D^-1 (x if b < 0)
      mont_mul<WN>(ba, D, b_neg ? xm : mone, M);
      mont_mul<WN>(ba, ba, P, M);
    }
  } else {
    for (int j = 0; j < WN; j++) ba[j] = mone[j];
    for (int t = 0; t < k; t++) {
      term(t);
      if (neg) mod_inverse<WN>(tm, tm, M);  // unchanged when there is no inverse
      mont_mul<WN>(ba, ba, tm, M);
    }
    if (a_neg) za = !mod_inverse<WN>(ba, ba, M);
    for (int j = 0; j < WN; j++) bb[j] = xm[j];
    if (b_neg) zb = !mod_inverse<WN>(bb, bb, M);
  }
  // w^a and x^b: Exp by 0 is 1
  uint32_t ea[1] = {ldk(&K.a)};
  const int abits = ldk((const uint32_t*)&K.a_bits), bbits = ldk((const uint32_t*)&K.b_bits);
  if (abits) exp_public_words<WN>(ba, ba, ea, abits, M);
  else for (int j = 0; j < WN; j++) ba[j] = mone[j];
  if (bbits) {
    uint32_t eb[kEpWords];
    for (int j = 0; j < kEpWords; j++) eb[j] = ldk(&K.b[j]);
    exp_public_words<WN>(bb, bb, eb, bbits, M);
  } else {
    for (int j = 0; j < WN; j++) bb[j] = mone[j];
  }
  uint32_t y[WN];
  mont_mul<WN>(y, ba, bb, M);
  if (za || zb)
    for (int j = 0; j < WN; j++) y[j] = 0;
  exp_public<WN>(tm, y, ldk(&K.e), M);  // y^e R
  mont_mul<WN>(tm, tm, one, M);
  mont_mul<WN>(y, y, one, M);
  if (cmp<WN>(tm, x)) return 2;
  for (int i = 0; i < klen; i++) out[i] = be_byte(y, klen, i);
  return 0;
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

// the HMAC-SHA-384 pad states of HKDF's salt, the klen-byte big-endian N (longer than a block, so HMAC keys with
// SHA-384(N))
inline void pb_salt_states(uint64_t (&si)[8], uint64_t (&so)[8], const uint8_t* n, int klen) {
  uint64_t h[8];
  sha2::Sha384::iv(h);
  sha2::absorb<sha2::Sha384>(h, 0, klen, [&](int j) { return n[j]; });
  sha2::hmac_key<sha2::Sha384>(si, so, h);
}

// Miller-Rabin on the odd n >= 3 of W words with `rounds` random bases below 2^(bitlen(n) - 1), drawn from rnd() (32
// random bits a call): false if a round proves n composite
template <int W, class Rnd>
inline bool probably_prime(const uint32_t* n, int rounds, Rnd& rnd) {
  Mod<W> M;
  mod_init<W>(M, n);
  if (M.bits == 2) return true;  // n = 3
  uint32_t d[W], one[W], m1[W], a[W], x[W];
  for (int j = 0; j < W; j++) d[j] = n[j], one[j] = j == 0;
  d[0] -= 1;  // n - 1 = 2^s d, d odd
  int s = 0;
  while (!(d[0] & 1)) {
    for (int j = 0; j < W; j++) d[j] = (d[j] >> 1) | (j + 1 < W ? d[j + 1] << 31 : 0);
    s++;
  }
  mont_mul<W>(one, M.r2, one, &M);  // R mod n, 1 in Montgomery form
  uint32_t zero[W] = {0};
  sub_mod<W>(m1, zero, one, &M);  // -1
  for (int r = 0; r < rounds; r++) {
    const int top = M.bits - 1;  // a < 2^top < n
    for (int j = 0; j < W; j++)
      a[j] = 32 * j >= top ? 0 : 32 * j + 32 <= top ? (uint32_t)rnd() : (uint32_t)rnd() & ((1u << (top & 31)) - 1);
    bool small = a[0] < 2;
    for (int j = 1; j < W; j++) small = small && !a[j];
    if (small) {  // bases 0 and 1 prove nothing: draw again
      r--;
      continue;
    }
    mont_mul<W>(x, a, M.r2, &M);
    exp_secret<W>(x, x, d, &M);
    if (!cmp<W>(x, one) || !cmp<W>(x, m1)) continue;
    bool witness = true;
    for (int i = 1; i < s && witness; i++) {
      mont_mul<W>(x, x, x, &M);
      if (!cmp<W>(x, m1)) witness = false;
    }
    if (witness) return false;
  }
  return true;
}

// (a, b) with e' a + e b = gcd(e', e) for e' = ep (kEpWords words) and e < 2^32: the classical extended Euclid
// coefficients, as Go's GCD gives them.  Its first step is e' = q e + r; the rest runs on (e, r) in 64-bit integers,
// giving s e + t r = g, so a = t and b = s - t q.  |a| < 2^32 and |b| <= e' fit their fields.
inline void tss_bezout(uint32_t* a, int* a_neg, uint32_t* b, int* b_neg, const uint32_t* ep, uint32_t e) {
  uint32_t q[kEpWords];
  uint64_t rem = 0;
  for (int i = kEpWords - 1; i >= 0; i--) {
    const uint64_t cur = rem << 32 | ep[i];
    q[i] = (uint32_t)(cur / e);
    rem = cur % e;
  }
  int64_t r0 = e, r1 = (int64_t)rem, s0 = 1, s1 = 0, t0 = 0, t1 = 1;
  while (r1) {
    const int64_t qq = r0 / r1, r2 = r0 - qq * r1, s2 = s0 - qq * s1, t2 = t0 - qq * t1;
    r0 = r1, r1 = r2, s0 = s1, s1 = s2, t0 = t1, t1 = t2;
  }
  *a_neg = t0 < 0;
  *a = (uint32_t)(t0 < 0 ? -t0 : t0);
  // b = s - t q from |t| q and |s| (both below 2^32 in magnitude for t and s)
  const uint64_t at = (uint64_t)(t0 < 0 ? -t0 : t0), as = (uint64_t)(s0 < 0 ? -s0 : s0);
  uint32_t tq[kEpWords];
  uint64_t c = 0;
  for (int i = 0; i < kEpWords; i++) {
    c += (uint64_t)q[i] * at;
    tq[i] = (uint32_t)c;
    c >>= 32;
  }
  // -t q and s: the same sign (add magnitudes) or opposite (subtract the smaller)
  const bool tq_neg = t0 > 0, s_neg = s0 < 0;
  uint32_t sw[kEpWords] = {(uint32_t)as, (uint32_t)(as >> 32)};
  if (tq_neg == s_neg || !at) {
    uint64_t cy = 0;
    for (int i = 0; i < kEpWords; i++) {
      cy += (uint64_t)tq[i] + sw[i];
      b[i] = (uint32_t)cy;
      cy >>= 32;
    }
    *b_neg = at ? tq_neg : s_neg;
  } else {
    const bool big = cmp<kEpWords>(tq, sw) >= 0;
    const uint32_t* hi = big ? tq : sw;
    const uint32_t* lo = big ? sw : tq;
    uint32_t br = 0;
    for (int i = 0; i < kEpWords; i++) {
      const uint64_t d = (uint64_t)hi[i] - lo[i] - br;
      b[i] = (uint32_t)d;
      br = (uint32_t)(d >> 63);
    }
    *b_neg = big ? tq_neg : s_neg;
  }
  bool zero = true;
  for (int i = 0; i < kEpWords; i++) zero = zero && !b[i];
  if (zero) *b_neg = 0;
}

}  // namespace rsa
}  // namespace cb200
