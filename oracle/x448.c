/* oracle/x448.c -- TEST INFRASTRUCTURE ONLY (see oracle.h): CPU restatement of dh/x448 (RFC 7748 X448):
 *   dh/x448/key.go:15-46        clamp, KeyGen, Shared, isValidPubKey (reduce mod p, then compare)
 *   dh/x448/curve.go:50-104     Montgomery ladder, toAffine, the three low-order points
 *   math/fp448 (generic)        GF(2^448 - 2^224 - 1), canonical ToBytes
 *   kem/hybrid/hybrid.go:83-93,197-283, xkem.go   Kyber768-X448, Kyber1024-X448 (X448 || round-3 Kyber)
 * The reference computes KeyGen with a Joye ladder over a precomputed table (curve.go:9-48); like Shared it returns
 * the affine u-coordinate of [clamp(k)]P in canonical form, which is what the plain RFC 7748 ladder below returns.
 * Pinned by the RFC 7748 vectors the reference's own tests use (dh/x448/testdata) and by OpenSSL's X448.
 * Built on its own into liboracle_x448.so (oracle/x448.py), linked against liboracle.so for SHAKE256 and the
 * round-3 Kyber KEM.
 */
#include <string.h>

#include "oracle.h"

int orc_x448(uint8_t out[56], const uint8_t scalar[56], const uint8_t *point);

/* ---------------------------------------------------------------- GF(2^448 - 2^224 - 1), eight 56-bit limbs */
typedef uint64_t fq[8];
typedef unsigned __int128 u128;
#define M56 ((1ull << 56) - 1)

static void fq_frombytes(fq h, const uint8_t s[56]) { /* all 448 bits */
  for (int i = 0; i < 8; i++) {
    uint64_t x = 0;
    for (int b = 6; b >= 0; b--) x = (x << 8) | s[7 * i + b];
    h[i] = x;
  }
}
/* one pass of carries; the carry out of limb 7 re-enters at limbs 0 and 4 (2^448 = 2^224 + 1) */
static void fq_carry(fq h) {
  for (int i = 0; i < 7; i++) { h[i + 1] += h[i] >> 56; h[i] &= M56; }
  uint64_t c = h[7] >> 56;
  h[7] &= M56;
  h[0] += c;
  h[4] += c;
}
static void fq_tobytes(uint8_t s[56], const fq f) { /* canonical encoding */
  fq h;
  memcpy(h, f, sizeof(fq));
  for (int r = 0; r < 3; r++) fq_carry(h);
  /* h < 2^448; subtract p if h >= p: h + 2^224 + 1 reaches 2^448 exactly then */
  fq t;
  memcpy(t, h, sizeof(fq));
  t[0] += 1;
  t[4] += 1;
  for (int i = 0; i < 7; i++) { t[i + 1] += t[i] >> 56; t[i] &= M56; }
  if (t[7] >> 56) { t[7] &= M56; memcpy(h, t, sizeof(fq)); }
  for (int i = 0; i < 8; i++)
    for (int b = 0; b < 7; b++) s[7 * i + b] = (uint8_t)(h[i] >> (8 * b));
}
static void fq_add(fq h, const fq f, const fq g) { for (int i = 0; i < 8; i++) h[i] = f[i] + g[i]; }
static void fq_sub(fq h, const fq f, const fq g) { /* f - g + 2p keeps limbs positive */
  for (int i = 0; i < 8; i++) h[i] = f[i] + (i == 4 ? 0x1fffffffffffffcull : 0x1fffffffffffffeull) - g[i];
}
static void fq_mul(fq h, const fq f, const fq g) {
  u128 t[15] = {0};
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 8; j++) t[i + j] += (u128)f[i] * g[j];
  for (int k = 14; k >= 8; k--) { t[k - 8] += t[k]; t[k - 4] += t[k]; } /* top down: k - 4 >= 8 folds again */
  u128 c = 0;
  for (int k = 0; k < 8; k++) { t[k] += c; h[k] = (uint64_t)t[k] & M56; c = t[k] >> 56; }
  u128 a = (u128)h[0] + c, b = (u128)h[4] + c;
  h[0] = (uint64_t)a & M56; h[1] += (uint64_t)(a >> 56);
  h[4] = (uint64_t)b & M56; h[5] += (uint64_t)(b >> 56);
}
static void fq_mul_small(fq h, const fq f, uint64_t s) {
  u128 c = 0;
  for (int k = 0; k < 8; k++) { c += (u128)f[k] * s; h[k] = (uint64_t)c & M56; c >>= 56; }
  h[0] += (uint64_t)c;
  h[4] += (uint64_t)c;
  fq_carry(h);
}
static void fq_pow2k(fq h, const fq f, int k) { fq_mul(h, f, f); for (int i = 1; i < k; i++) fq_mul(h, h, h); }
static void fq_invert(fq out, const fq z) { /* z^(p-2), p - 2 = [223 ones] 0 [222 ones] 0 1 */
  fq t, z2, z3, z6, z12, z24, z30, z48, z96, z192, z222, z223;
  fq_pow2k(t, z, 1); fq_mul(z2, t, z);
  fq_pow2k(t, z2, 1); fq_mul(z3, t, z);
  fq_pow2k(t, z3, 3); fq_mul(z6, t, z3);
  fq_pow2k(t, z6, 6); fq_mul(z12, t, z6);
  fq_pow2k(t, z12, 12); fq_mul(z24, t, z12);
  fq_pow2k(t, z24, 6); fq_mul(z30, t, z6);
  fq_pow2k(t, z24, 24); fq_mul(z48, t, z24);
  fq_pow2k(t, z48, 48); fq_mul(z96, t, z48);
  fq_pow2k(t, z96, 96); fq_mul(z192, t, z96);
  fq_pow2k(t, z192, 30); fq_mul(z222, t, z30);
  fq_pow2k(t, z222, 1); fq_mul(z223, t, z);
  fq_pow2k(t, z223, 223); fq_mul(t, t, z222);
  fq_pow2k(t, t, 2); fq_mul(out, t, z);
}
static void fq_cswap(fq a, fq b, uint64_t bit) {
  uint64_t m = 0 - bit;
  for (int i = 0; i < 8; i++) { uint64_t x = m & (a[i] ^ b[i]); a[i] ^= x; b[i] ^= x; }
}

/* out = u([clamp(scalar)] P); point == NULL: P = u 5 (KeyGen, key.go:33-35), else Shared (key.go:41-46).
 * Returns 1 unless `point` (reduced mod p) is one of the low-order values 0, 1, p - 1 of curve.go:76-104. */
int orc_x448(uint8_t out[56], const uint8_t scalar[56], const uint8_t *point) {
  static const uint8_t base[56] = {5};
  uint8_t k[56], canon[56];
  memcpy(k, scalar, 56);
  k[0] &= 252; k[55] |= 128; /* key.go:15-20 */
  fq x1, x2 = {1}, z2 = {0}, x3, z3 = {1}, a, aa, b, bb, e, c, d, da, cb, t;
  fq_frombytes(x1, point ? point : base);
  memcpy(x3, x1, sizeof(fq));
  uint64_t swap = 0;
  for (int s = 447; s >= 0; s--) {
    uint64_t bit = (k[s >> 3] >> (s & 7)) & 1;
    swap ^= bit;
    fq_cswap(x2, x3, swap); fq_cswap(z2, z3, swap);
    swap = bit;
    fq_add(a, x2, z2); fq_mul(aa, a, a);
    fq_sub(b, x2, z2); fq_mul(bb, b, b);
    fq_sub(e, aa, bb);
    fq_add(c, x3, z3); fq_sub(d, x3, z3);
    fq_mul(da, d, a); fq_mul(cb, c, b);
    fq_add(t, da, cb); fq_mul(x3, t, t);
    fq_sub(t, da, cb); fq_mul(t, t, t); fq_mul(z3, x1, t);
    fq_mul(x2, aa, bb);
    fq_mul_small(t, e, 39081); fq_add(t, t, aa); fq_mul(z2, e, t); /* RFC 7748: a24 = (A - 2) / 4 */
  }
  fq_cswap(x2, x3, swap); fq_cswap(z2, z3, swap);
  fq_invert(z2, z2);
  fq_mul(x2, x2, z2);
  fq_tobytes(out, x2);
  if (!point) return 1;
  uint8_t low[3][56];
  memset(low, 0, sizeof(low));
  low[1][0] = 1;
  memset(low[2], 0xff, 56); /* p - 1 */
  low[2][0] = 0xfe;
  low[2][28] = 0xfe;
  fq_tobytes(canon, x1); /* reduced mod p, as isValidPubKey does (key.go:22-30) */
  int ok = 1;
  for (int i = 0; i < 3; i++) ok &= memcmp(canon, low[i], 56) != 0;
  return ok;
}

/* ---------------------------------------------------------------- kem/hybrid over X448 (hybrid.go, xkem.go)
 * k = 3: Kyber768-X448, k = 4: Kyber1024-X448 (first = X448, second = round-3 Kyber, hybrid.go:83-93).
 * Sizes: pk = 56 + ek, sk = 56 + dk, ct = 56 + ct, ss = 56 + 32 (hybrid.go:141-143); key seed 64 = max(56, 64),
 * encapsulation seed 56 = max(56, 32) (hybrid.go:131-157). */
/* xScheme.DeriveKeyPair (xkem.go:112-123): sk = SHAKE256(seed, 56), pk = KeyGen(sk) */
static void xkem448_derive(uint8_t pk[56], uint8_t sk[56], const uint8_t seed[56]) {
  orc_shake256(sk, 56, seed, 56);
  orc_x448(pk, sk, NULL);
}
/* scheme.DeriveKeyPair (hybrid.go:197-212): SHAKE256(seed) -> X seed (56) || Kyber seed (64) */
void orc_x448_hybrid_keygen(int k, uint8_t *pk, uint8_t *sk, const uint8_t seed[64]) {
  uint8_t ex[56 + 64];
  orc_shake256(ex, sizeof(ex), seed, 64);
  xkem448_derive(pk, sk, ex);
  orc_kyber_kem_keygen(k, pk + 56, sk + 56, ex + 56);
}
/* EncapsulateDeterministically (hybrid.go:233-261, xkem.go:160-178): SHAKE256(seed) -> X seed (56) || Kyber seed (32).
 * rc: 0 ok, 1 kem.ErrPubKey (low-order X448 share) */
int orc_x448_hybrid_encaps(int k, uint8_t *ct, uint8_t *ss, const uint8_t *pk, const uint8_t seed[56]) {
  uint8_t ex[56 + 32], esk[56];
  orc_shake256(ex, sizeof(ex), seed, 56);
  xkem448_derive(ct, esk, ex);
  const int ok = orc_x448(ss, esk, pk);
  orc_kyber_kem_encaps(k, ct + 56, ss + 56, pk + 56, ex + 56);
  return ok ? 0 : 1;
}
/* Decapsulate (hybrid.go:263-283, xkem.go:180-196).  rc: 0 ok, 1 kem.ErrPubKey (low-order X448 share in ct) */
int orc_x448_hybrid_decaps(int k, uint8_t *ss, const uint8_t *sk, const uint8_t *ct) {
  orc_kyber_kem_decaps(k, ss + 56, sk + 56, ct + 56);
  return orc_x448(ss, sk, ct) ? 0 : 1;
}
