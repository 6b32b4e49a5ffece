/* oracle/p256.c -- TEST INFRASTRUCTURE ONLY (see oracle.h): CPU restatement of HPKE's DHKEM(P-256, HKDF-SHA256)
 * (RFC 9180 section 4.1, kem_id 0x10) as the reference computes it:
 *   hpke/shortkem.go:31-55     sizes, calcDH (the x-coordinate of [sk]pk)
 *   hpke/shortkem.go:63-90     DeriveKeyPair: candidates LabeledExpand(dkp_prk, "candidate", I2OSP(ctr, 1), 32) for
 *                              ctr = 0..255, the first in [1, n - 1] is the key
 *   hpke/shortkem.go:103-130   UnmarshalBinaryPrivateKey / PublicKey (crypto/ecdh NewPrivateKey / NewPublicKey rules)
 *   hpke/kembase.go:94-241     ExtractAndExpand, Encap, AuthEncap, Decap, AuthDecap
 * The curve arithmetic is written for obviousness and is deliberately unlike circl_b200/csrc/p256.cuh: plain
 * residues (no Montgomery form) reduced with the NIST fast reduction of FIPS 186-4 D.2.3, Jacobian coordinates with
 * the textbook formulas and their special cases, double-and-add over the bits of the scalar and inversion by
 * square-and-multiply over the bits of p - 2.  SHA-256 is oracle/hpke.c's (orc_sha256 of liboracle_hpke.so); HMAC and
 * HKDF with HPKE's labels are written out again below.  Built into liboracle_p256.so (oracle/p256.py).
 */
#include <string.h>

#include "oracle.h"

void orc_sha256(uint8_t out[32], const uint8_t *m, size_t len);

typedef struct {
  uint32_t w[8]; /* little-endian words */
} u256;

static const u256 P = {{0xffffffff, 0xffffffff, 0xffffffff, 0, 0, 0, 1, 0xffffffff}};
static const u256 NN = {{0xfc632551, 0xf3b9cac2, 0xa7179e84, 0xbce6faad, 0xffffffff, 0xffffffff, 0, 0xffffffff}};
static const u256 B = {{0x27d2604b, 0x3bce3c3e, 0xcc53b0f6, 0x651d06b0, 0x769886bc, 0xb3ebbd55, 0xaa3a93e7, 0x5ac635d8}};
static const u256 GX = {{0xd898c296, 0xf4a13945, 0x2deb33a0, 0x77037d81, 0x63a440f2, 0xf8bce6e5, 0xe12c4247, 0x6b17d1f2}};
static const u256 GY = {{0x37bf51f5, 0xcbb64068, 0x6b315ece, 0x2bce3357, 0x7c0f9e16, 0x8ee7eb4a, 0xfe1a7f9b, 0x4fe342e2}};

static int cmp(const u256 *a, const u256 *b) {
  for (int i = 7; i >= 0; i--)
    if (a->w[i] != b->w[i]) return a->w[i] < b->w[i] ? -1 : 1;
  return 0;
}
static int is_zero(const u256 *a) {
  for (int i = 0; i < 8; i++)
    if (a->w[i]) return 0;
  return 1;
}
static uint32_t add_raw(u256 *r, const u256 *a, const u256 *b) {
  uint64_t c = 0;
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)a->w[i] + b->w[i];
    r->w[i] = (uint32_t)c;
    c >>= 32;
  }
  return (uint32_t)c;
}
static uint32_t sub_raw(u256 *r, const u256 *a, const u256 *b) {
  int64_t c = 0;
  for (int i = 0; i < 8; i++) {
    c += (int64_t)a->w[i] - b->w[i];
    r->w[i] = (uint32_t)c;
    c >>= 32; /* arithmetic: 0 or -1 */
  }
  return (uint32_t)(c != 0);
}
static void from_be(u256 *a, const uint8_t *b) {
  for (int i = 0; i < 8; i++) {
    const uint8_t *q = b + 4 * (7 - i);
    a->w[i] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
  }
}
static void to_be(uint8_t *b, const u256 *a) {
  for (int i = 0; i < 8; i++) {
    uint8_t *q = b + 4 * (7 - i);
    q[0] = (uint8_t)(a->w[i] >> 24), q[1] = (uint8_t)(a->w[i] >> 16), q[2] = (uint8_t)(a->w[i] >> 8), q[3] = (uint8_t)a->w[i];
  }
}

/* ---------------------------------------------------------------- GF(p) */
static void fadd(u256 *r, const u256 *a, const u256 *b) {
  const uint32_t c = add_raw(r, a, b);
  if (c || cmp(r, &P) >= 0) sub_raw(r, r, &P);
}
static void fsub(u256 *r, const u256 *a, const u256 *b) {
  if (sub_raw(r, a, b)) add_raw(r, r, &P);
}
/* FIPS 186-4 D.2.3: c = c15..c0 (32-bit words) reduced as s1 + 2 s2 + 2 s3 + s4 + s5 - s6 - s7 - s8 - s9 */
static void reduce(u256 *r, const uint32_t c[16]) {
  static const int8_t T[9][8] = {
      /* word index of each term, from word 0 up; -1 = zero */
      {0, 1, 2, 3, 4, 5, 6, 7},          {-1, -1, -1, 11, 12, 13, 14, 15}, {-1, -1, -1, 12, 13, 14, 15, -1},
      {8, 9, 10, -1, -1, -1, 14, 15},     {9, 10, 11, 13, 14, 15, 13, 8},  {11, 12, 13, -1, -1, -1, 8, 10},
      {12, 13, 14, 15, -1, -1, 9, 11},    {13, 14, 15, 8, 9, 10, -1, 12},  {14, 15, -1, 9, 10, 11, -1, 13}};
  static const int K[9] = {1, 2, 2, 1, 1, -1, -1, -1, -1};
  int64_t acc[8] = {0};
  for (int t = 0; t < 9; t++)
    for (int i = 0; i < 8; i++)
      if (T[t][i] >= 0) acc[i] += K[t] * (int64_t)c[T[t][i]];
  int64_t carry = 0;
  for (int i = 0; i < 8; i++) {
    acc[i] += carry;
    r->w[i] = (uint32_t)acc[i];
    carry = (acc[i] - (int64_t)r->w[i]) >> 32;
  }
  /* value = r + carry 2^256 with -4 <= carry <= 6: fold whole multiples of p back in */
  while (carry < 0) carry += add_raw(r, r, &P);
  while (carry > 0) carry -= sub_raw(r, r, &P);
  while (cmp(r, &P) >= 0) sub_raw(r, r, &P);
}
static void fmul(u256 *r, const u256 *a, const u256 *b) {
  uint32_t c[16] = {0};
  for (int i = 0; i < 8; i++) {
    uint64_t carry = 0;
    for (int j = 0; j < 8; j++) {
      carry += (uint64_t)c[i + j] + (uint64_t)a->w[i] * b->w[j];
      c[i + j] = (uint32_t)carry;
      carry >>= 32;
    }
    c[i + 8] = (uint32_t)carry;
  }
  reduce(r, c);
}
static void finv(u256 *r, const u256 *a) { /* a^(p - 2), square-and-multiply over the bits of p - 2 */
  u256 e = P, x = {{1}};
  e.w[0] -= 2;
  for (int bit = 255; bit >= 0; bit--) {
    fmul(&x, &x, &x);
    if ((e.w[bit / 32] >> (bit % 32)) & 1) fmul(&x, &x, a);
  }
  *r = x;
}

/* ---------------------------------------------------------------- the group, Jacobian (X / Z^2, Y / Z^3) */
typedef struct {
  u256 X, Y, Z; /* Z = 0: the point at infinity */
} jac;

static void jdbl(jac *r, const jac *p) { /* dbl-2001-b (a = -3) */
  if (is_zero(&p->Z) || is_zero(&p->Y)) {
    memset(r, 0, sizeof *r);
    return;
  }
  u256 delta, gamma, beta, alpha, t, u, X3, Y3, Z3;
  fmul(&delta, &p->Z, &p->Z);
  fmul(&gamma, &p->Y, &p->Y);
  fmul(&beta, &p->X, &gamma);
  fsub(&t, &p->X, &delta);
  fadd(&u, &p->X, &delta);
  fmul(&alpha, &t, &u);
  fadd(&t, &alpha, &alpha);
  fadd(&alpha, &t, &alpha); /* 3 (X - delta)(X + delta) */
  fmul(&X3, &alpha, &alpha);
  fadd(&t, &beta, &beta);
  fadd(&t, &t, &t);
  fadd(&u, &t, &t); /* 8 beta */
  fsub(&X3, &X3, &u);
  fadd(&Z3, &p->Y, &p->Z);
  fmul(&Z3, &Z3, &Z3);
  fsub(&Z3, &Z3, &gamma);
  fsub(&Z3, &Z3, &delta);
  fsub(&u, &t, &X3); /* 4 beta - X3 */
  fmul(&Y3, &alpha, &u);
  fmul(&t, &gamma, &gamma);
  fadd(&t, &t, &t);
  fadd(&t, &t, &t);
  fadd(&t, &t, &t); /* 8 gamma^2 */
  fsub(&Y3, &Y3, &t);
  r->X = X3, r->Y = Y3, r->Z = Z3;
}
static void jadd(jac *r, const jac *p, const jac *q) { /* add-2007-bl with its special cases */
  if (is_zero(&p->Z)) {
    *r = *q;
    return;
  }
  if (is_zero(&q->Z)) {
    *r = *p;
    return;
  }
  u256 z1z1, z2z2, u1, u2, s1, s2, h, i, j, rr, v, t, X3, Y3, Z3;
  fmul(&z1z1, &p->Z, &p->Z);
  fmul(&z2z2, &q->Z, &q->Z);
  fmul(&u1, &p->X, &z2z2);
  fmul(&u2, &q->X, &z1z1);
  fmul(&t, &q->Z, &z2z2);
  fmul(&s1, &p->Y, &t);
  fmul(&t, &p->Z, &z1z1);
  fmul(&s2, &q->Y, &t);
  if (cmp(&u1, &u2) == 0) {
    if (cmp(&s1, &s2) == 0) {
      jdbl(r, p);
    } else {
      memset(r, 0, sizeof *r);
    }
    return;
  }
  fsub(&h, &u2, &u1);
  fadd(&i, &h, &h);
  fmul(&i, &i, &i);
  fmul(&j, &h, &i);
  fsub(&rr, &s2, &s1);
  fadd(&rr, &rr, &rr);
  fmul(&v, &u1, &i);
  fmul(&X3, &rr, &rr);
  fsub(&X3, &X3, &j);
  fsub(&X3, &X3, &v);
  fsub(&X3, &X3, &v);
  fsub(&t, &v, &X3);
  fmul(&Y3, &rr, &t);
  fmul(&t, &s1, &j);
  fadd(&t, &t, &t);
  fsub(&Y3, &Y3, &t);
  fadd(&Z3, &p->Z, &q->Z);
  fmul(&Z3, &Z3, &Z3);
  fsub(&Z3, &Z3, &z1z1);
  fsub(&Z3, &Z3, &z2z2);
  fmul(&Z3, &Z3, &h);
  r->X = X3, r->Y = Y3, r->Z = Z3;
}
/* (x, y) = [k](px, py); returns 0 for the point at infinity */
static int smul(u256 *x, u256 *y, const u256 *k, const u256 *px, const u256 *py) {
  jac r, p;
  memset(&r, 0, sizeof r);
  p.X = *px, p.Y = *py;
  memset(&p.Z, 0, sizeof p.Z);
  p.Z.w[0] = 1;
  for (int bit = 255; bit >= 0; bit--) {
    jdbl(&r, &r);
    if ((k->w[bit / 32] >> (bit % 32)) & 1) jadd(&r, &r, &p);
  }
  if (is_zero(&r.Z)) return 0;
  u256 zi, z2, z3;
  finv(&zi, &r.Z);
  fmul(&z2, &zi, &zi);
  fmul(&z3, &z2, &zi);
  fmul(x, &r.X, &z2);
  fmul(y, &r.Y, &z3);
  return 1;
}

/* ---------------------------------------------------------------- the crypto/ecdh rules */
/* NewPrivateKey: 0 < k < n */
int orc_p256_scalar_ok(const uint8_t sk[32]) {
  u256 k;
  from_be(&k, sk);
  return !is_zero(&k) && cmp(&k, &NN) < 0;
}
/* NewPublicKey: 0x04 || X || Y, X < p, Y < p, y^2 = x^3 - 3x + b */
int orc_p256_point_ok(const uint8_t pk[65]) {
  if (pk[0] != 4) return 0;
  u256 x, y, l, r, t;
  from_be(&x, pk + 1);
  from_be(&y, pk + 33);
  if (cmp(&x, &P) >= 0 || cmp(&y, &P) >= 0) return 0;
  fmul(&l, &y, &y);
  fmul(&r, &x, &x);
  fmul(&r, &r, &x);
  fadd(&t, &x, &x);
  fadd(&t, &t, &x);
  fsub(&r, &r, &t);
  fadd(&r, &r, &B);
  return cmp(&l, &r) == 0;
}
/* KeyGen (pt NULL: out = 0x04 || X || Y, 65 bytes) or Shared (out = X, 32 bytes).  Returns a status: bit 0 = invalid
 * point, bit 1 = invalid scalar; out is then all zero. */
int orc_p256(uint8_t *out, const uint8_t sk[32], const uint8_t *pt) {
  int st = 0;
  if (!orc_p256_scalar_ok(sk)) st |= 2;
  if (pt && !orc_p256_point_ok(pt)) st |= 1;
  memset(out, 0, pt ? 32 : 65);
  if (st) return st;
  u256 k, px = GX, py = GY, x, y;
  from_be(&k, sk);
  if (pt) from_be(&px, pt + 1), from_be(&py, pt + 33);
  smul(&x, &y, &k, &px, &py); /* never the point at infinity for 0 < k < n and a point of the prime-order group */
  if (pt) {
    to_be(out, &x);
  } else {
    out[0] = 4;
    to_be(out + 1, &x);
    to_be(out + 33, &y);
  }
  return 0;
}

/* ---------------------------------------------------------------- HMAC-SHA256, HPKE's labeled HKDF */
#define MAXMSG 512
static void hmac(uint8_t out[32], const uint8_t *key, size_t keylen, const uint8_t *m, size_t len) {
  uint8_t buf[64 + MAXMSG], inner[32];
  memset(buf, 0, 64);
  memcpy(buf, key, keylen);
  for (int i = 0; i < 64; i++) buf[i] ^= 0x36;
  memcpy(buf + 64, m, len);
  orc_sha256(inner, buf, 64 + len);
  memset(buf, 0, 64);
  memcpy(buf, key, keylen);
  for (int i = 0; i < 64; i++) buf[i] ^= 0x5c;
  memcpy(buf + 64, inner, 32);
  orc_sha256(out, buf, 96);
}
static size_t put_prefix(uint8_t *m) { /* "HPKE-v1" || "KEM" || I2OSP(0x10, 2) */
  memcpy(m, "HPKE-v1KEM\x00\x10", 12);
  return 12;
}
static void labeled_extract(uint8_t prk[32], const char *label, const uint8_t *ikm, size_t ikmlen) {
  uint8_t m[MAXMSG];
  size_t o = put_prefix(m);
  memcpy(m + o, label, strlen(label)), o += strlen(label);
  memcpy(m + o, ikm, ikmlen), o += ikmlen;
  hmac(prk, NULL, 0, m, o);
}
/* L <= 32: the first block of HKDF-Expand */
static void labeled_expand(uint8_t *out, const uint8_t prk[32], const char *label, const uint8_t *info, size_t infolen,
                           size_t L) {
  uint8_t m[MAXMSG], t[32];
  size_t o = 0;
  m[o++] = (uint8_t)(L >> 8);
  m[o++] = (uint8_t)L;
  o += put_prefix(m + o);
  memcpy(m + o, label, strlen(label)), o += strlen(label);
  memcpy(m + o, info, infolen), o += infolen;
  m[o++] = 1;
  hmac(t, prk, 32, m, o);
  memcpy(out, t, L);
}

/* DeriveKeyPair (shortkem.go:63-90); returns the counter of the key, or -1 after 256 candidates (the reference panics) */
int orc_p256_derive(uint8_t pk[65], uint8_t sk[32], const uint8_t seed[32]) {
  uint8_t prk[32];
  labeled_extract(prk, "dkp_prk", seed, 32);
  for (int ctr = 0; ctr < 256; ctr++) {
    const uint8_t c = (uint8_t)ctr;
    labeled_expand(sk, prk, "candidate", &c, 1, 32);
    if (orc_p256_scalar_ok(sk)) {
      orc_p256(pk, sk, NULL);
      return ctr;
    }
  }
  memset(sk, 0, 32);
  memset(pk, 0, 65);
  return -1;
}

static void kdf(uint8_t ss[32], const uint8_t *dh, size_t dhlen, const uint8_t *ctx, size_t ctxlen) {
  uint8_t prk[32];
  labeled_extract(prk, "eae_prk", dh, dhlen);
  labeled_expand(ss, prk, "shared_secret", ctx, ctxlen, 32);
}

/* Encap / AuthEncap (kembase.go:120-183; skS NULL for Encap).  Returns a status: bit 0 = pkR invalid
 * (ErrInvalidKEMPublicKey), bit 1 = skS invalid (ErrInvalidKEMPrivateKey); ss is then all zero.  enc is written
 * either way. */
int orc_p256_encaps(uint8_t enc[65], uint8_t ss[32], const uint8_t pkR[65], const uint8_t *skS, const uint8_t seed[32]) {
  uint8_t skE[32], dh[64], ctx[195];
  orc_p256_derive(enc, skE, seed);
  int st = orc_p256(dh, skE, pkR);
  memcpy(ctx, enc, 65);
  memcpy(ctx + 65, pkR, 65);
  size_t dhlen = 32, ctxlen = 130;
  if (skS) {
    st |= orc_p256(dh + 32, skS, pkR);
    st |= orc_p256(ctx + 130, skS, NULL);
    dhlen = 64, ctxlen = 195;
  }
  memset(ss, 0, 32);
  if (st) return st;
  kdf(ss, dh, dhlen, ctx, ctxlen);
  return 0;
}

/* Decap / AuthDecap (kembase.go:185-241; pkS NULL for Decap): pkR = KeyGen(skR).  Status as orc_p256_encaps, with
 * bit 0 for enc or pkS and bit 1 for skR. */
int orc_p256_decaps(uint8_t ss[32], const uint8_t skR[32], const uint8_t enc[65], const uint8_t *pkS) {
  uint8_t dh[64], ctx[195];
  int st = orc_p256(dh, skR, enc);
  memcpy(ctx, enc, 65);
  st |= orc_p256(ctx + 65, skR, NULL);
  size_t dhlen = 32, ctxlen = 130;
  if (pkS) {
    st |= orc_p256(dh + 32, skR, pkS);
    memcpy(ctx + 130, pkS, 65);
    dhlen = 64, ctxlen = 195;
  }
  memset(ss, 0, 32);
  if (st) return st;
  kdf(ss, dh, dhlen, ctx, ctxlen);
  return 0;
}
