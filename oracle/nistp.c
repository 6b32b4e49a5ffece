/* oracle/nistp.c -- TEST INFRASTRUCTURE ONLY (see oracle.h): CPU restatement of HPKE's DHKEM(P-384, HKDF-SHA384)
 * (kem_id 0x11) and DHKEM(P-521, HKDF-SHA512) (kem_id 0x12) as the reference computes them:
 *   hpke/shortkem.go:31-55     sizes, calcDH (the x-coordinate of [sk]pk)
 *   hpke/shortkem.go:63-90     DeriveKeyPair: candidates LabeledExpand(dkp_prk, "candidate", I2OSP(ctr, 1), Nsk) with
 *                              byte 0 ANDed with the bitmask (0xff for P-384, 0x01 for P-521), for ctr = 0..255; the
 *                              first in [1, n - 1] is the key
 *   hpke/shortkem.go:103-130   UnmarshalBinaryPrivateKey / PublicKey (crypto/ecdh NewPrivateKey / NewPublicKey rules)
 *   hpke/kembase.go:94-241     ExtractAndExpand, Encap, AuthEncap, Decap, AuthDecap
 * The curve arithmetic is written for obviousness and is deliberately unlike circl_b200/csrc/nistp.cuh: plain residues
 * (no Montgomery form) reduced by folding, since p = 2^k - c with a short c (P-384: c = 2^128 + 2^96 - 2^32 + 1;
 * P-521: c = 1, the Mersenne fold), Jacobian coordinates with the textbook formulas and their special cases,
 * double-and-add over the bits of the scalar and inversion by square-and-multiply over the bits of p - 2.  SHA-384 and
 * SHA-512, HMAC and HKDF with HPKE's labels (HKDF-Expand over as many blocks as L needs) are written out below.  Built
 * into liboracle_nistp.so (oracle/nistp.py).  `bits` selects the curve: 384 or 521.
 */
#include <string.h>

#include "oracle.h"

#define MW 17 /* words of the largest field element */
typedef struct {
  uint32_t w[MW]; /* little-endian words, the unused ones zero */
} fe;

typedef struct {
  int nw, nbytes, k, kem_id, nh; /* words, bytes of a row, p = 2^k - c, kem_id, digest bytes */
  uint8_t mask0;                  /* DeriveKeyPair's bitmask */
  const char *p, *n, *b, *gx, *gy, *c; /* big-endian hex */
} curve;

static const curve P384 = {
    12, 48, 384, 0x11, 48, 0xff,
    "fffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffeffffffff0000000000000000ffffffff",
    "ffffffffffffffffffffffffffffffffffffffffffffffffc7634d81f4372ddf581a0db248b0a77aecec196accc52973",
    "b3312fa7e23ee7e4988e056be3f82d19181d9c6efe8141120314088f5013875ac656398d8a2ed19d2a85c8edd3ec2aef",
    "aa87ca22be8b05378eb1c71ef320ad746e1d3b628ba79b9859f741e082542a385502f25dbf55296c3a545e3872760ab7",
    "3617de4a96262c6f5d9e98bf9292dc29f8f41dbd289a147ce9da3113b5f0b8c00a60b1ce1d7e819d7a431d7c90ea0e5f",
    "0100000000ffffffffffffffff00000001"};
static const curve P521 = {
    17, 66, 521, 0x12, 64, 0x01,
    "01ffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffff",
    "01fffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffa51868783bf2f966b7fcc0148f709a5d03bb5c9b8899c47aebb6fb71e91386409",
    "0051953eb9618e1c9a1f929a21a0b68540eea2da725b99b315f3b8b489918ef109e156193951ec7e937b1652c0bd3bb1bf073573df883d2c34f1ef451fd46b503f00",
    "00c6858e06b70404e9cd9e3ecb662395b4429c648139053fb521f828af606b4d3dbaa14b5e77efe75928fe1dc127a2ffa8de3348b3c1856a429bf97e7e31c2e5bd66",
    "011839296a789a3bc0045c8a5fb42c7d1bd998f54449579b446817afbd17273e662c97ee72995ef42640c550b9013fad0761353c7086a272c24088be94769fd16650",
    "01"};

typedef struct {
  const curve *cv;
  fe p, n, b, gx, gy, c;
} ctx;

static void from_hex(fe *a, const char *h) {
  memset(a, 0, sizeof *a);
  size_t len = strlen(h);
  for (size_t i = 0; i < len; i++) {
    const char ch = h[len - 1 - i];
    const uint32_t v = (uint32_t)(ch <= '9' ? ch - '0' : ch - 'a' + 10);
    a->w[i / 8] |= v << (4 * (i % 8));
  }
}
static int setup(ctx *x, int bits) {
  x->cv = bits == 384 ? &P384 : bits == 521 ? &P521 : NULL;
  if (!x->cv) return 0;
  from_hex(&x->p, x->cv->p), from_hex(&x->n, x->cv->n), from_hex(&x->b, x->cv->b);
  from_hex(&x->gx, x->cv->gx), from_hex(&x->gy, x->cv->gy), from_hex(&x->c, x->cv->c);
  return 1;
}

static int cmp(const fe *a, const fe *b) {
  for (int i = MW - 1; i >= 0; i--)
    if (a->w[i] != b->w[i]) return a->w[i] < b->w[i] ? -1 : 1;
  return 0;
}
static int is_zero(const fe *a) {
  for (int i = 0; i < MW; i++)
    if (a->w[i]) return 0;
  return 1;
}
static void add_raw(fe *r, const fe *a, const fe *b) { /* no overflow: values stay below 2^544 */
  uint64_t c = 0;
  for (int i = 0; i < MW; i++) {
    c += (uint64_t)a->w[i] + b->w[i];
    r->w[i] = (uint32_t)c;
    c >>= 32;
  }
}
static void sub_raw(fe *r, const fe *a, const fe *b) { /* a >= b */
  int64_t c = 0;
  for (int i = 0; i < MW; i++) {
    c += (int64_t)a->w[i] - b->w[i];
    r->w[i] = (uint32_t)c;
    c >>= 32;
  }
}
static void from_be(const ctx *x, fe *a, const uint8_t *b) {
  memset(a, 0, sizeof *a);
  for (int j = 0; j < x->cv->nbytes; j++) a->w[j / 4] |= (uint32_t)b[x->cv->nbytes - 1 - j] << (8 * (j % 4));
}
static void to_be(const ctx *x, uint8_t *b, const fe *a) {
  for (int j = 0; j < x->cv->nbytes; j++) b[x->cv->nbytes - 1 - j] = (uint8_t)(a->w[j / 4] >> (8 * (j % 4)));
}

/* ---------------------------------------------------------------- GF(p), p = 2^k - c */
static void fadd(const ctx *x, fe *r, const fe *a, const fe *b) {
  add_raw(r, a, b);
  if (cmp(r, &x->p) >= 0) sub_raw(r, r, &x->p);
}
static void fsub(const ctx *x, fe *r, const fe *a, const fe *b) {
  if (cmp(a, b) >= 0) {
    sub_raw(r, a, b);
  } else {
    fe t;
    add_raw(&t, a, &x->p);
    sub_raw(r, &t, b);
  }
}
/* t (2 MW + 2 words) mod p: t = hi 2^k + lo = hi c + lo (mod p), repeated until hi = 0 */
#define TW (2 * MW + 2)
static void reduce(const ctx *x, fe *r, uint32_t t[TW]) {
  const int k = x->cv->k;
  for (;;) {
    uint32_t hi[TW] = {0}, lo[TW] = {0};
    int nz = 0;
    for (int i = 0; i < TW; i++) {
      const int bit = 32 * i;
      if (bit + 32 <= k) lo[i] = t[i];
      else if (bit < k) lo[i] = t[i] & ((1u << (k - bit)) - 1);
    }
    for (int i = 0; i < TW; i++) { /* hi = t >> k */
      const int src = i + k / 32, sh = k % 32;
      uint64_t v = src < TW ? t[src] : 0;
      if (sh && src + 1 < TW) v |= (uint64_t)t[src + 1] << 32;
      hi[i] = (uint32_t)(v >> sh);
      nz |= hi[i] != 0;
    }
    if (!nz) break;
    uint32_t s[TW] = {0}; /* s = hi c + lo */
    for (int i = 0; i < TW; i++) {
      uint64_t carry = 0;
      for (int j = 0; j < MW && i + j < TW; j++) {
        carry += (uint64_t)s[i + j] + (uint64_t)hi[i] * x->c.w[j];
        s[i + j] = (uint32_t)carry;
        carry >>= 32;
      }
    }
    uint64_t carry = 0;
    for (int i = 0; i < TW; i++) {
      carry += (uint64_t)s[i] + lo[i];
      t[i] = (uint32_t)carry;
      carry >>= 32;
    }
  }
  memcpy(r->w, t, sizeof r->w);
  while (cmp(r, &x->p) >= 0) sub_raw(r, r, &x->p);
}
static void fmul(const ctx *x, fe *r, const fe *a, const fe *b) {
  uint32_t t[TW] = {0};
  for (int i = 0; i < MW; i++) {
    uint64_t carry = 0;
    for (int j = 0; j < MW; j++) {
      carry += (uint64_t)t[i + j] + (uint64_t)a->w[i] * b->w[j];
      t[i + j] = (uint32_t)carry;
      carry >>= 32;
    }
    t[i + MW] = (uint32_t)carry;
  }
  reduce(x, r, t);
}
static void finv(const ctx *x, fe *r, const fe *a) { /* a^(p - 2), square-and-multiply over the bits of p - 2 */
  fe e = x->p, one, y;
  memset(&one, 0, sizeof one);
  one.w[0] = 2;
  sub_raw(&e, &e, &one);
  memset(&y, 0, sizeof y);
  y.w[0] = 1;
  for (int bit = x->cv->k - 1; bit >= 0; bit--) {
    fmul(x, &y, &y, &y);
    if ((e.w[bit / 32] >> (bit % 32)) & 1) fmul(x, &y, &y, a);
  }
  *r = y;
}

/* ---------------------------------------------------------------- the group, Jacobian (X / Z^2, Y / Z^3) */
typedef struct {
  fe X, Y, Z; /* Z = 0: the point at infinity */
} jac;

static void jdbl(const ctx *x, jac *r, const jac *p) { /* dbl-2001-b (a = -3) */
  if (is_zero(&p->Z) || is_zero(&p->Y)) {
    memset(r, 0, sizeof *r);
    return;
  }
  fe delta, gamma, beta, alpha, t, u, X3, Y3, Z3;
  fmul(x, &delta, &p->Z, &p->Z);
  fmul(x, &gamma, &p->Y, &p->Y);
  fmul(x, &beta, &p->X, &gamma);
  fsub(x, &t, &p->X, &delta);
  fadd(x, &u, &p->X, &delta);
  fmul(x, &alpha, &t, &u);
  fadd(x, &t, &alpha, &alpha);
  fadd(x, &alpha, &t, &alpha); /* 3 (X - delta)(X + delta) */
  fmul(x, &X3, &alpha, &alpha);
  fadd(x, &t, &beta, &beta);
  fadd(x, &t, &t, &t);
  fadd(x, &u, &t, &t); /* 8 beta */
  fsub(x, &X3, &X3, &u);
  fadd(x, &Z3, &p->Y, &p->Z);
  fmul(x, &Z3, &Z3, &Z3);
  fsub(x, &Z3, &Z3, &gamma);
  fsub(x, &Z3, &Z3, &delta);
  fsub(x, &u, &t, &X3); /* 4 beta - X3 */
  fmul(x, &Y3, &alpha, &u);
  fmul(x, &t, &gamma, &gamma);
  fadd(x, &t, &t, &t);
  fadd(x, &t, &t, &t);
  fadd(x, &t, &t, &t); /* 8 gamma^2 */
  fsub(x, &Y3, &Y3, &t);
  r->X = X3, r->Y = Y3, r->Z = Z3;
}
static void jadd(const ctx *x, jac *r, const jac *p, const jac *q) { /* add-2007-bl with its special cases */
  if (is_zero(&p->Z)) {
    *r = *q;
    return;
  }
  if (is_zero(&q->Z)) {
    *r = *p;
    return;
  }
  fe z1z1, z2z2, u1, u2, s1, s2, h, i, j, rr, v, t, X3, Y3, Z3;
  fmul(x, &z1z1, &p->Z, &p->Z);
  fmul(x, &z2z2, &q->Z, &q->Z);
  fmul(x, &u1, &p->X, &z2z2);
  fmul(x, &u2, &q->X, &z1z1);
  fmul(x, &t, &q->Z, &z2z2);
  fmul(x, &s1, &p->Y, &t);
  fmul(x, &t, &p->Z, &z1z1);
  fmul(x, &s2, &q->Y, &t);
  if (cmp(&u1, &u2) == 0) {
    if (cmp(&s1, &s2) == 0) {
      jdbl(x, r, p);
    } else {
      memset(r, 0, sizeof *r);
    }
    return;
  }
  fsub(x, &h, &u2, &u1);
  fadd(x, &i, &h, &h);
  fmul(x, &i, &i, &i);
  fmul(x, &j, &h, &i);
  fsub(x, &rr, &s2, &s1);
  fadd(x, &rr, &rr, &rr);
  fmul(x, &v, &u1, &i);
  fmul(x, &X3, &rr, &rr);
  fsub(x, &X3, &X3, &j);
  fsub(x, &X3, &X3, &v);
  fsub(x, &X3, &X3, &v);
  fsub(x, &t, &v, &X3);
  fmul(x, &Y3, &rr, &t);
  fmul(x, &t, &s1, &j);
  fadd(x, &t, &t, &t);
  fsub(x, &Y3, &Y3, &t);
  fadd(x, &Z3, &p->Z, &q->Z);
  fmul(x, &Z3, &Z3, &Z3);
  fsub(x, &Z3, &Z3, &z1z1);
  fsub(x, &Z3, &Z3, &z2z2);
  fmul(x, &Z3, &Z3, &h);
  r->X = X3, r->Y = Y3, r->Z = Z3;
}
/* (ox, oy) = [k](px, py) for a k that is not a multiple of the order */
static void smul(const ctx *x, fe *ox, fe *oy, const fe *k, const fe *px, const fe *py) {
  jac r, p;
  memset(&r, 0, sizeof r);
  p.X = *px, p.Y = *py;
  memset(&p.Z, 0, sizeof p.Z);
  p.Z.w[0] = 1;
  for (int bit = 32 * MW - 1; bit >= 0; bit--) {
    jdbl(x, &r, &r);
    if ((k->w[bit / 32] >> (bit % 32)) & 1) jadd(x, &r, &r, &p);
  }
  fe zi, z2, z3;
  finv(x, &zi, &r.Z);
  fmul(x, &z2, &zi, &zi);
  fmul(x, &z3, &z2, &zi);
  fmul(x, ox, &r.X, &z2);
  fmul(x, oy, &r.Y, &z3);
}

/* ---------------------------------------------------------------- the crypto/ecdh rules */
static int scalar_ok(const ctx *x, const uint8_t *sk) { /* NewPrivateKey: 0 < k < n */
  fe k;
  from_be(x, &k, sk);
  /* every byte of the row is part of k: a leading byte above 0x01 (P-521) makes k >= n */
  return !is_zero(&k) && cmp(&k, &x->n) < 0;
}
static int point_ok(const ctx *x, const uint8_t *pk) { /* NewPublicKey: 0x04 || X || Y, X, Y < p, on the curve */
  if (pk[0] != 4) return 0;
  const int nb = x->cv->nbytes;
  fe px, py, l, r, t;
  from_be(x, &px, pk + 1);
  from_be(x, &py, pk + 1 + nb);
  if (cmp(&px, &x->p) >= 0 || cmp(&py, &x->p) >= 0) return 0;
  fmul(x, &l, &py, &py);
  fmul(x, &r, &px, &px);
  fmul(x, &r, &r, &px);
  fadd(x, &t, &px, &px);
  fadd(x, &t, &t, &px);
  fsub(x, &r, &r, &t);
  fadd(x, &r, &r, &x->b);
  return cmp(&l, &r) == 0;
}
int orc_nistp_scalar_ok(int bits, const uint8_t *sk) {
  ctx x;
  return setup(&x, bits) && scalar_ok(&x, sk);
}
int orc_nistp_point_ok(int bits, const uint8_t *pk) {
  ctx x;
  return setup(&x, bits) && point_ok(&x, pk);
}
/* KeyGen (pt NULL: out = 0x04 || X || Y) or Shared (out = X).  Returns a status: bit 0 = invalid point, bit 1 =
 * invalid scalar; out is then all zero.  -1 for an unknown curve. */
static int ecdh(const ctx *x, uint8_t *out, const uint8_t *sk, const uint8_t *pt) {
  const int nb = x->cv->nbytes;
  int st = 0;
  if (!scalar_ok(x, sk)) st |= 2;
  if (pt && !point_ok(x, pt)) st |= 1;
  memset(out, 0, pt ? (size_t)nb : (size_t)(1 + 2 * nb));
  if (st) return st;
  fe k, px = x->gx, py = x->gy, ox, oy;
  from_be(x, &k, sk);
  if (pt) from_be(x, &px, pt + 1), from_be(x, &py, pt + 1 + nb);
  smul(x, &ox, &oy, &k, &px, &py); /* never the point at infinity for 0 < k < n on a prime-order curve */
  if (pt) {
    to_be(x, out, &ox);
  } else {
    out[0] = 4;
    to_be(x, out + 1, &ox);
    to_be(x, out + 1 + nb, &oy);
  }
  return 0;
}
int orc_nistp(int bits, uint8_t *out, const uint8_t *sk, const uint8_t *pt) {
  ctx x;
  if (!setup(&x, bits)) return -1;
  return ecdh(&x, out, sk, pt);
}

/* ---------------------------------------------------------------- SHA-384 / SHA-512 (FIPS 180-4) */
static const uint64_t K512[80] = {
    0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull, 0x3956c25bf348b538ull,
    0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull, 0xd807aa98a3030242ull, 0x12835b0145706fbeull,
    0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull, 0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull,
    0xc19bf174cf692694ull, 0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull,
    0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull, 0x983e5152ee66dfabull,
    0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull, 0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull,
    0x06ca6351e003826full, 0x142929670a0e6e70ull, 0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull,
    0x53380d139d95b3dfull, 0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull,
    0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull, 0xd192e819d6ef5218ull,
    0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull, 0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull,
    0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull, 0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull,
    0x682e6ff3d6b2b8a3ull, 0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull,
    0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull, 0xca273eceea26619cull,
    0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull, 0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull,
    0x113f9804bef90daeull, 0x1b710b35131c471bull, 0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull,
    0x431d67c49c100d4cull, 0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull};
static const uint64_t IV384[8] = {0xcbbb9d5dc1059ed8ull, 0x629a292a367cd507ull, 0x9159015a3070dd17ull,
                                  0x152fecd8f70e5939ull, 0x67332667ffc00b31ull, 0x8eb44a8768581511ull,
                                  0xdb0c2e0d64f98fa7ull, 0x47b5481dbefa4fa4ull};
static const uint64_t IV512[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull,
                                  0xa54ff53a5f1d36f1ull, 0x510e527fade682d1ull, 0x9b05688c2b3e6c1full,
                                  0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
static uint64_t ror(uint64_t v, int n) { return (v >> n) | (v << (64 - n)); }
static void block(uint64_t H[8], const uint8_t *m) {
  uint64_t w[80], a[8];
  for (int t = 0; t < 16; t++) {
    w[t] = 0;
    for (int b = 0; b < 8; b++) w[t] = (w[t] << 8) | m[8 * t + b];
  }
  for (int t = 16; t < 80; t++)
    w[t] = (ror(w[t - 2], 19) ^ ror(w[t - 2], 61) ^ (w[t - 2] >> 6)) + w[t - 7] +
           (ror(w[t - 15], 1) ^ ror(w[t - 15], 8) ^ (w[t - 15] >> 7)) + w[t - 16];
  memcpy(a, H, sizeof a);
  for (int t = 0; t < 80; t++) {
    const uint64_t t1 = a[7] + (ror(a[4], 14) ^ ror(a[4], 18) ^ ror(a[4], 41)) + ((a[4] & a[5]) ^ (~a[4] & a[6])) +
                        K512[t] + w[t];
    const uint64_t t2 = (ror(a[0], 28) ^ ror(a[0], 34) ^ ror(a[0], 39)) + ((a[0] & a[1]) ^ (a[0] & a[2]) ^ (a[1] & a[2]));
    memmove(a + 1, a, 7 * sizeof(uint64_t));
    a[4] += t1;
    a[0] = t1 + t2;
  }
  for (int i = 0; i < 8; i++) H[i] += a[i];
}
/* SHA-384 (nh = 48) or SHA-512 (nh = 64) of m */
static void sha(int nh, uint8_t *out, const uint8_t *m, size_t len) {
  uint64_t H[8];
  memcpy(H, nh == 48 ? IV384 : IV512, sizeof H);
  size_t off = 0;
  for (; off + 128 <= len; off += 128) block(H, m + off);
  uint8_t last[256] = {0};
  const size_t rest = len - off, nl = rest + 17 <= 128 ? 128 : 256;
  memcpy(last, m + off, rest);
  last[rest] = 0x80;
  for (int b = 0; b < 8; b++) last[nl - 1 - b] = (uint8_t)(((uint64_t)len << 3) >> (8 * b));
  for (size_t o = 0; o < nl; o += 128) block(H, last + o);
  for (int i = 0; i < nh; i++) out[i] = (uint8_t)(H[i / 8] >> (56 - 8 * (i % 8)));
}
void orc_sha384(uint8_t out[48], const uint8_t *m, size_t len) { sha(48, out, m, len); }

/* ---------------------------------------------------------------- HMAC, HPKE's labeled HKDF */
#define MAXMSG 1024
static void hmac(const ctx *x, uint8_t *out, const uint8_t *key, size_t keylen, const uint8_t *m, size_t len) {
  const int nh = x->cv->nh;
  uint8_t buf[128 + MAXMSG], inner[64];
  memset(buf, 0, 128);
  memcpy(buf, key, keylen);
  for (int i = 0; i < 128; i++) buf[i] ^= 0x36;
  memcpy(buf + 128, m, len);
  sha(nh, inner, buf, 128 + len);
  memset(buf, 0, 128);
  memcpy(buf, key, keylen);
  for (int i = 0; i < 128; i++) buf[i] ^= 0x5c;
  memcpy(buf + 128, inner, (size_t)nh);
  sha(nh, out, buf, 128 + (size_t)nh);
}
static size_t put_prefix(const ctx *x, uint8_t *m) { /* "HPKE-v1" || "KEM" || I2OSP(kem_id, 2) */
  memcpy(m, "HPKE-v1KEM", 10);
  m[10] = (uint8_t)(x->cv->kem_id >> 8), m[11] = (uint8_t)x->cv->kem_id;
  return 12;
}
static void labeled_extract(const ctx *x, uint8_t *prk, const char *label, const uint8_t *ikm, size_t ikmlen) {
  uint8_t m[MAXMSG];
  size_t o = put_prefix(x, m);
  memcpy(m + o, label, strlen(label)), o += strlen(label);
  memcpy(m + o, ikm, ikmlen), o += ikmlen;
  hmac(x, prk, NULL, 0, m, o);
}
/* HKDF-Expand over ceil(L / Nh) blocks: T(i) = HMAC(prk, T(i - 1) || info || i) */
static void labeled_expand(const ctx *x, uint8_t *out, const uint8_t *prk, const char *label, const uint8_t *info,
                           size_t infolen, size_t L) {
  const size_t nh = (size_t)x->cv->nh;
  uint8_t linfo[MAXMSG], m[MAXMSG], t[64];
  size_t o = 0;
  linfo[o++] = (uint8_t)(L >> 8);
  linfo[o++] = (uint8_t)L;
  o += put_prefix(x, linfo + o);
  memcpy(linfo + o, label, strlen(label)), o += strlen(label);
  memcpy(linfo + o, info, infolen), o += infolen;
  size_t done = 0, tlen = 0;
  for (uint8_t i = 1; done < L; i++) {
    memcpy(m, t, tlen);
    memcpy(m + tlen, linfo, o);
    m[tlen + o] = i;
    hmac(x, t, prk, nh, m, tlen + o + 1);
    tlen = nh;
    const size_t take = L - done < nh ? L - done : nh;
    memcpy(out + done, t, take);
    done += take;
  }
}

/* DeriveKeyPair (shortkem.go:63-90); returns the counter of the key, or -1 after 256 candidates (the reference
 * panics) or for an unknown curve */
int orc_nistp_derive(int bits, uint8_t *pk, uint8_t *sk, const uint8_t *seed) {
  ctx x;
  if (!setup(&x, bits)) return -1;
  const int nb = x.cv->nbytes;
  uint8_t prk[64];
  labeled_extract(&x, prk, "dkp_prk", seed, (size_t)nb);
  for (int ctr = 0; ctr < 256; ctr++) {
    const uint8_t c = (uint8_t)ctr;
    labeled_expand(&x, sk, prk, "candidate", &c, 1, (size_t)nb);
    sk[0] &= x.cv->mask0;
    if (scalar_ok(&x, sk)) {
      ecdh(&x, pk, sk, NULL);
      return ctr;
    }
  }
  memset(sk, 0, (size_t)nb);
  memset(pk, 0, (size_t)(1 + 2 * nb));
  return -1;
}

static void kdf(const ctx *x, uint8_t *ss, const uint8_t *dh, size_t dhlen, const uint8_t *c, size_t clen) {
  uint8_t prk[64];
  labeled_extract(x, prk, "eae_prk", dh, dhlen);
  labeled_expand(x, ss, prk, "shared_secret", c, clen, (size_t)x->cv->nh);
}

/* Encap / AuthEncap (kembase.go:120-183; skS NULL for Encap).  Returns a status: bit 0 = pkR invalid
 * (ErrInvalidKEMPublicKey), bit 1 = skS invalid (ErrInvalidKEMPrivateKey); ss is then all zero.  enc is written
 * either way. */
int orc_nistp_encaps(int bits, uint8_t *enc, uint8_t *ss, const uint8_t *pkR, const uint8_t *skS, const uint8_t *seed) {
  ctx x;
  if (!setup(&x, bits)) return -1;
  const size_t nb = (size_t)x.cv->nbytes, npk = 1 + 2 * nb;
  uint8_t skE[66], dh[132], c[3 * 133];
  orc_nistp_derive(bits, enc, skE, seed);
  int st = ecdh(&x, dh, skE, pkR);
  memcpy(c, enc, npk);
  memcpy(c + npk, pkR, npk);
  size_t dhlen = nb, clen = 2 * npk;
  if (skS) {
    st |= ecdh(&x, dh + nb, skS, pkR);
    st |= ecdh(&x, c + 2 * npk, skS, NULL);
    dhlen = 2 * nb, clen = 3 * npk;
  }
  memset(ss, 0, (size_t)x.cv->nh);
  if (st) return st;
  kdf(&x, ss, dh, dhlen, c, clen);
  return 0;
}

/* Decap / AuthDecap (kembase.go:185-241; pkS NULL for Decap): pkR = KeyGen(skR).  Status as orc_nistp_encaps, with
 * bit 0 for enc or pkS and bit 1 for skR. */
int orc_nistp_decaps(int bits, uint8_t *ss, const uint8_t *skR, const uint8_t *enc, const uint8_t *pkS) {
  ctx x;
  if (!setup(&x, bits)) return -1;
  const size_t nb = (size_t)x.cv->nbytes, npk = 1 + 2 * nb;
  uint8_t dh[132], c[3 * 133];
  int st = ecdh(&x, dh, skR, enc);
  memcpy(c, enc, npk);
  st |= ecdh(&x, c + npk, skR, NULL);
  size_t dhlen = nb, clen = 2 * npk;
  if (pkS) {
    st |= ecdh(&x, dh + nb, skR, pkS);
    memcpy(c + 2 * npk, pkS, npk);
    dhlen = 2 * nb, clen = 3 * npk;
  }
  memset(ss, 0, (size_t)x.cv->nh);
  if (st) return st;
  kdf(&x, ss, dh, dhlen, c, clen);
  return 0;
}
