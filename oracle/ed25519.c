/* oracle/ed25519.c -- TEST INFRASTRUCTURE ONLY: a plain-C restatement of sign/ed25519 (pure Ed25519, RFC 8032
 * section 5.1: ed25519.go NewKeyFromSeed / Sign / Verify, point.go ToBytes / FromBytes, modular.go) and of
 * sign/eddilithium2 (eddilithium.go NewKeyFromSeed / SignTo / Verify) on top of liboracle.so's SHAKE256 and round-3
 * Dilithium2.
 *
 * Written for obviousness, not speed, and independent of circl_b200/csrc/ed25519.cuh: five 51-bit limbs with 128-bit
 * products, exponentiation by square-and-multiply, bit-serial double-and-add, scalars reduced mod L by binary long
 * division.  Nothing here is constant time. */
#include <stdint.h>
#include <string.h>

#include "oracle.h"

/* ------------------------------------------------------------------ SHA-512 (FIPS 180-4) */
typedef struct {
  uint64_t h[8];
  uint8_t buf[128];
  size_t fill;
  uint64_t total;
} sha512_ctx;

static const uint64_t K512[80] = {
    0x428a2f98d728ae22ULL, 0x7137449123ef65cdULL, 0xb5c0fbcfec4d3b2fULL, 0xe9b5dba58189dbbcULL, 0x3956c25bf348b538ULL,
    0x59f111f1b605d019ULL, 0x923f82a4af194f9bULL, 0xab1c5ed5da6d8118ULL, 0xd807aa98a3030242ULL, 0x12835b0145706fbeULL,
    0x243185be4ee4b28cULL, 0x550c7dc3d5ffb4e2ULL, 0x72be5d74f27b896fULL, 0x80deb1fe3b1696b1ULL, 0x9bdc06a725c71235ULL,
    0xc19bf174cf692694ULL, 0xe49b69c19ef14ad2ULL, 0xefbe4786384f25e3ULL, 0x0fc19dc68b8cd5b5ULL, 0x240ca1cc77ac9c65ULL,
    0x2de92c6f592b0275ULL, 0x4a7484aa6ea6e483ULL, 0x5cb0a9dcbd41fbd4ULL, 0x76f988da831153b5ULL, 0x983e5152ee66dfabULL,
    0xa831c66d2db43210ULL, 0xb00327c898fb213fULL, 0xbf597fc7beef0ee4ULL, 0xc6e00bf33da88fc2ULL, 0xd5a79147930aa725ULL,
    0x06ca6351e003826fULL, 0x142929670a0e6e70ULL, 0x27b70a8546d22ffcULL, 0x2e1b21385c26c926ULL, 0x4d2c6dfc5ac42aedULL,
    0x53380d139d95b3dfULL, 0x650a73548baf63deULL, 0x766a0abb3c77b2a8ULL, 0x81c2c92e47edaee6ULL, 0x92722c851482353bULL,
    0xa2bfe8a14cf10364ULL, 0xa81a664bbc423001ULL, 0xc24b8b70d0f89791ULL, 0xc76c51a30654be30ULL, 0xd192e819d6ef5218ULL,
    0xd69906245565a910ULL, 0xf40e35855771202aULL, 0x106aa07032bbd1b8ULL, 0x19a4c116b8d2d0c8ULL, 0x1e376c085141ab53ULL,
    0x2748774cdf8eeb99ULL, 0x34b0bcb5e19b48a8ULL, 0x391c0cb3c5c95a63ULL, 0x4ed8aa4ae3418acbULL, 0x5b9cca4f7763e373ULL,
    0x682e6ff3d6b2b8a3ULL, 0x748f82ee5defb2fcULL, 0x78a5636f43172f60ULL, 0x84c87814a1f0ab72ULL, 0x8cc702081a6439ecULL,
    0x90befffa23631e28ULL, 0xa4506cebde82bde9ULL, 0xbef9a3f7b2c67915ULL, 0xc67178f2e372532bULL, 0xca273eceea26619cULL,
    0xd186b8c721c0c207ULL, 0xeada7dd6cde0eb1eULL, 0xf57d4f7fee6ed178ULL, 0x06f067aa72176fbaULL, 0x0a637dc5a2c898a6ULL,
    0x113f9804bef90daeULL, 0x1b710b35131c471bULL, 0x28db77f523047d84ULL, 0x32caab7b40c72493ULL, 0x3c9ebe0a15c9bebcULL,
    0x431d67c49c100d4cULL, 0x4cc5d4becb3e42b6ULL, 0x597f299cfc657e2aULL, 0x5fcb6fab3ad6faecULL, 0x6c44198c4a475817ULL};

static uint64_t ror(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

static void sha512_block(sha512_ctx *c, const uint8_t *p) {
  uint64_t w[80], s[8];
  for (int i = 0; i < 16; i++) {
    w[i] = 0;
    for (int j = 0; j < 8; j++) w[i] = (w[i] << 8) | p[8 * i + j];
  }
  for (int i = 16; i < 80; i++)
    w[i] = (ror(w[i - 2], 19) ^ ror(w[i - 2], 61) ^ (w[i - 2] >> 6)) + w[i - 7] +
           (ror(w[i - 15], 1) ^ ror(w[i - 15], 8) ^ (w[i - 15] >> 7)) + w[i - 16];
  memcpy(s, c->h, sizeof s);
  for (int i = 0; i < 80; i++) {
    uint64_t t1 = s[7] + (ror(s[4], 14) ^ ror(s[4], 18) ^ ror(s[4], 41)) + ((s[4] & s[5]) ^ (~s[4] & s[6])) + K512[i] + w[i];
    uint64_t t2 = (ror(s[0], 28) ^ ror(s[0], 34) ^ ror(s[0], 39)) + ((s[0] & s[1]) ^ (s[0] & s[2]) ^ (s[1] & s[2]));
    memmove(s + 1, s, 7 * sizeof(uint64_t));
    s[4] += t1;
    s[0] = t1 + t2;
  }
  for (int i = 0; i < 8; i++) c->h[i] += s[i];
}
static void sha512_init(sha512_ctx *c) {
  static const uint64_t iv[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                                 0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
  memcpy(c->h, iv, sizeof iv);
  c->fill = 0;
  c->total = 0;
}
static void sha512_update(sha512_ctx *c, const uint8_t *p, size_t n) {
  c->total += n;
  while (n) {
    size_t k = 128 - c->fill < n ? 128 - c->fill : n;
    memcpy(c->buf + c->fill, p, k);
    c->fill += k;
    p += k;
    n -= k;
    if (c->fill == 128) {
      sha512_block(c, c->buf);
      c->fill = 0;
    }
  }
}
static void sha512_final(sha512_ctx *c, uint8_t out[64]) {
  const uint64_t bits = c->total * 8;
  uint8_t pad = 0x80, zero = 0;
  sha512_update(c, &pad, 1);
  while (c->fill != 112) sha512_update(c, &zero, 1);
  uint8_t len[16] = {0};
  for (int i = 0; i < 8; i++) len[15 - i] = (uint8_t)(bits >> (8 * i));
  sha512_update(c, len, 16);
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 8; j++) out[8 * i + j] = (uint8_t)(c->h[i] >> (56 - 8 * j));
}
void orc_sha512(uint8_t out[64], const uint8_t *in, size_t n) {
  sha512_ctx c;
  sha512_init(&c);
  sha512_update(&c, in, n);
  sha512_final(&c, out);
}

/* ------------------------------------------------------------------ GF(2^255 - 19), five 51-bit limbs */
typedef struct {
  uint64_t v[5];
} fe;
#define M51 ((1ULL << 51) - 1)

static void fe_frombytes(fe *h, const uint8_t b[32]) { /* bit 255 is dropped */
  uint8_t t[32];
  memcpy(t, b, 32);
  t[31] &= 127;
  for (int i = 0; i < 5; i++) {
    uint64_t x = 0;
    for (int k = 0; k < 64; k++) {
      const int bit = 51 * i + k;
      if (k >= 51 || bit > 254) break;
      x |= (uint64_t)((t[bit >> 3] >> (bit & 7)) & 1) << k;
    }
    h->v[i] = x;
  }
}
static void fe_carry(fe *h) {
  for (int r = 0; r < 2; r++) {
    for (int i = 0; i < 4; i++) {
      h->v[i + 1] += h->v[i] >> 51;
      h->v[i] &= M51;
    }
    h->v[0] += 19 * (h->v[4] >> 51);
    h->v[4] &= M51;
  }
}
static void fe_tobytes(uint8_t b[32], const fe *f) { /* canonical */
  fe h = *f;
  fe_carry(&h);
  /* subtract p if h >= p: h + 19 overflows 2^255 exactly then */
  uint64_t q = (h.v[0] + 19) >> 51;
  for (int i = 1; i < 5; i++) q = (h.v[i] + q) >> 51;
  h.v[0] += 19 * q;
  for (int i = 0; i < 4; i++) {
    h.v[i + 1] += h.v[i] >> 51;
    h.v[i] &= M51;
  }
  h.v[4] &= M51;
  memset(b, 0, 32);
  for (int bit = 0; bit < 255; bit++)
    if ((h.v[bit / 51] >> (bit % 51)) & 1) b[bit >> 3] |= (uint8_t)(1u << (bit & 7));
}
static void fe_add(fe *h, const fe *f, const fe *g) {
  for (int i = 0; i < 5; i++) h->v[i] = f->v[i] + g->v[i];
  fe_carry(h);
}
static void fe_sub(fe *h, const fe *f, const fe *g) { /* f + 4p - g */
  static const uint64_t p4[5] = {4 * (M51 - 18), 4 * M51, 4 * M51, 4 * M51, 4 * M51};
  for (int i = 0; i < 5; i++) h->v[i] = f->v[i] + p4[i] - g->v[i];
  fe_carry(h);
}
static void fe_mul(fe *h, const fe *f, const fe *g) {
  unsigned __int128 t[5] = {0};
  for (int i = 0; i < 5; i++)
    for (int j = 0; j < 5; j++) {
      const unsigned __int128 p = (unsigned __int128)f->v[i] * g->v[j];
      if (i + j < 5)
        t[i + j] += p;
      else
        t[i + j - 5] += p * 19;
    }
  uint64_t c = 0;
  for (int i = 0; i < 5; i++) {
    t[i] += c;
    h->v[i] = (uint64_t)t[i] & M51;
    c = (uint64_t)(t[i] >> 51);
  }
  h->v[0] += 19 * c;
  fe_carry(h);
}
static void fe_set(fe *h, uint64_t x) {
  memset(h, 0, sizeof *h);
  h->v[0] = x;
}
static void fe_pow(fe *out, const fe *a, const uint8_t e[32]) { /* a^e, e little endian */
  fe r, b = *a;
  fe_set(&r, 1);
  for (int bit = 0; bit < 256; bit++) {
    if ((e[bit >> 3] >> (bit & 7)) & 1) fe_mul(&r, &r, &b);
    fe_mul(&b, &b, &b);
  }
  *out = r;
}
static int fe_iszero(const fe *f) {
  uint8_t b[32], acc = 0;
  fe_tobytes(b, f);
  for (int i = 0; i < 32; i++) acc |= b[i];
  return acc == 0;
}
static void fe_invert(fe *out, const fe *a) { /* a^(p - 2) */
  uint8_t e[32];
  memset(e, 0xff, 32);
  e[0] = 0xeb;
  e[31] = 0x7f;
  fe_pow(out, a, e);
}
static void fe_neg(fe *h, const fe *f) {
  fe z;
  fe_set(&z, 0);
  fe_sub(h, &z, f);
}
/* d = -121665 / 121666, sqrt(-1) = 2^((p - 1) / 4) */
static void fe_d(fe *d) {
  fe a, b;
  fe_set(&a, 121665);
  fe_neg(&a, &a);
  fe_set(&b, 121666);
  fe_invert(&b, &b);
  fe_mul(d, &a, &b);
}
static void fe_sqrtm1(fe *r) {
  uint8_t e[32];
  memset(e, 0xff, 32);
  e[0] = 0xfb;
  e[31] = 0x1f; /* (p - 1) / 4 = 2^253 - 5 */
  fe two;
  fe_set(&two, 2);
  fe_pow(r, &two, e);
}

/* ------------------------------------------------------------------ edwards25519, extended coordinates */
typedef struct {
  fe X, Y, Z, T;
} ge;

static void ge_identity(ge *p) {
  fe_set(&p->X, 0);
  fe_set(&p->Y, 1);
  fe_set(&p->Z, 1);
  fe_set(&p->T, 0);
}
/* complete addition on -x^2 + y^2 = 1 + d x^2 y^2 (Hisil, Wong, Carter, Dawson 2008, a = -1); also doubles */
static void ge_add(ge *r, const ge *p, const ge *q) {
  fe d, a, b, c, dd, e, f, g, h, t;
  fe_d(&d);
  fe_sub(&a, &p->Y, &p->X);
  fe_sub(&t, &q->Y, &q->X);
  fe_mul(&a, &a, &t);
  fe_add(&b, &p->Y, &p->X);
  fe_add(&t, &q->Y, &q->X);
  fe_mul(&b, &b, &t);
  fe_mul(&c, &p->T, &q->T);
  fe_mul(&c, &c, &d);
  fe_add(&c, &c, &c);
  fe_mul(&dd, &p->Z, &q->Z);
  fe_add(&dd, &dd, &dd);
  fe_sub(&e, &b, &a);
  fe_sub(&f, &dd, &c);
  fe_add(&g, &dd, &c);
  fe_add(&h, &b, &a);
  fe_mul(&r->X, &e, &f);
  fe_mul(&r->Y, &g, &h);
  fe_mul(&r->T, &e, &h);
  fe_mul(&r->Z, &f, &g);
}
/* [k] P for a 256-bit little-endian k, bit by bit from the top */
static void ge_scalarmult(ge *r, const uint8_t k[32], const ge *p) {
  ge q;
  ge_identity(&q);
  for (int bit = 255; bit >= 0; bit--) {
    ge_add(&q, &q, &q);
    if ((k[bit >> 3] >> (bit & 7)) & 1) ge_add(&q, &q, p);
  }
  *r = q;
}
/* pointR1.ToBytes (point.go:38-52) */
static void ge_tobytes(uint8_t out[32], const ge *p) {
  fe zi, x, y;
  uint8_t xb[32];
  fe_invert(&zi, &p->Z);
  fe_mul(&x, &p->X, &zi);
  fe_mul(&y, &p->Y, &zi);
  fe_tobytes(out, &y);
  fe_tobytes(xb, &x);
  out[31] |= (uint8_t)((xb[0] & 1) << 7);
}
/* pointR1.FromBytes (point.go:54-87): 0 for y >= p, a non-square u / v, or x = 0 with the sign bit set */
static int ge_frombytes(ge *p, const uint8_t in[32]) {
  static const uint8_t P[32] = {0xed, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0x7f};
  const int sign = in[31] >> 7;
  uint8_t yb[32];
  memcpy(yb, in, 32);
  yb[31] &= 127;
  int i = 31;
  while (i > 0 && yb[i] == P[i]) i--;
  if (!(yb[i] < P[i])) return 0;
  fe y, u, v, d, one, x, chk, t;
  fe_frombytes(&y, yb);
  fe_d(&d);
  fe_set(&one, 1);
  fe_mul(&u, &y, &y);
  fe_mul(&v, &u, &d);
  fe_sub(&u, &u, &one);
  fe_add(&v, &v, &one);
  /* x^2 = u / v; a root is w^((p + 3) / 8) with w = u / v, times sqrt(-1) if that squares to -w */
  fe w;
  fe_invert(&w, &v);
  fe_mul(&w, &w, &u);
  uint8_t e[32];
  memset(e, 0xff, 32);
  e[0] = 0xfe;
  e[31] = 0x0f; /* (p + 3) / 8 = 2^252 - 2 */
  fe_pow(&x, &w, e);
  fe_mul(&chk, &x, &x);
  fe_sub(&t, &chk, &w);
  if (!fe_iszero(&t)) {
    fe_add(&t, &chk, &w);
    if (!fe_iszero(&t)) return 0;
    fe s;
    fe_sqrtm1(&s);
    fe_mul(&x, &x, &s);
  }
  uint8_t xb[32];
  fe_tobytes(xb, &x);
  if (fe_iszero(&x) && sign) return 0;
  if ((xb[0] & 1) != sign) fe_neg(&x, &x);
  p->X = x;
  p->Y = y;
  fe_set(&p->Z, 1);
  fe_mul(&p->T, &x, &y);
  return 1;
}
/* B = (x, 4/5) with x even (RFC 8032 section 5.1) */
static void ge_base(ge *b) {
  fe four, five;
  fe_set(&four, 4);
  fe_set(&five, 5);
  fe_invert(&five, &five);
  fe_mul(&four, &four, &five);
  uint8_t yb[32];
  fe_tobytes(yb, &four);
  ge_frombytes(b, yb);
}

/* ------------------------------------------------------------------ scalars mod L */
static const uint8_t L_BYTES[32] = {0xed, 0xd3, 0xf5, 0x5c, 0x1a, 0x63, 0x12, 0x58, 0xd6, 0x9c, 0xf7, 0xa2, 0xde, 0xf9, 0xde, 0x14,
                                    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0x10};

/* out = x mod L for an n-byte little-endian x, by binary long division */
static void sc_reduce(uint8_t out[32], const uint8_t *x, size_t n) {
  uint64_t r[5] = {0}, l[5] = {0};
  for (int i = 0; i < 32; i++) l[i / 8] |= (uint64_t)L_BYTES[i] << (8 * (i % 8));
  for (long bit = (long)(8 * n) - 1; bit >= 0; bit--) {
    for (int i = 4; i > 0; i--) r[i] = (r[i] << 1) | (r[i - 1] >> 63);
    r[0] = (r[0] << 1) | ((x[bit >> 3] >> (bit & 7)) & 1);
    int ge_l = 1; /* r >= L ? */
    for (int i = 4; i >= 0; i--)
      if (r[i] != l[i]) {
        ge_l = r[i] > l[i];
        break;
      }
    if (ge_l) {
      unsigned __int128 borrow = 0;
      for (int i = 0; i < 5; i++) {
        const unsigned __int128 t = (unsigned __int128)r[i] - l[i] - borrow;
        r[i] = (uint64_t)t;
        borrow = (t >> 64) & 1;
      }
    }
  }
  for (int i = 0; i < 32; i++) out[i] = (uint8_t)(r[i / 8] >> (8 * (i % 8)));
}
/* calculateS (modular.go): (r + k a) mod L */
static void sc_muladd(uint8_t out[32], const uint8_t r[32], const uint8_t k[32], const uint8_t a[32]) {
  uint8_t t[65] = {0};
  unsigned acc[65] = {0};
  for (int i = 0; i < 32; i++)
    for (int j = 0; j < 32; j++) acc[i + j] += (unsigned)k[i] * a[j];
  for (int i = 0; i < 32; i++) acc[i] += r[i];
  unsigned c = 0;
  for (int i = 0; i < 65; i++) {
    acc[i] += c;
    t[i] = (uint8_t)acc[i];
    c = acc[i] >> 8;
  }
  sc_reduce(out, t, 65);
}
/* isLessThanOrder (ed25519.go:437-443) */
static int sc_less_than_order(const uint8_t s[32]) {
  int i = 31;
  while (i > 0 && s[i] == L_BYTES[i]) i--;
  return s[i] < L_BYTES[i];
}

/* ------------------------------------------------------------------ Ed25519 */
static void expand(uint8_t s[32], uint8_t prefix[32], const uint8_t seed[32]) {
  uint8_t h[64];
  orc_sha512(h, seed, 32);
  memcpy(s, h, 32);
  memcpy(prefix, h + 32, 32);
  s[0] &= 248;
  s[31] = (uint8_t)((s[31] & 127) | 64);
}
void orc_ed25519_keygen(uint8_t pk[32], uint8_t sk[64], const uint8_t seed[32]) {
  uint8_t s[32], prefix[32];
  ge B, A;
  expand(s, prefix, seed);
  ge_base(&B);
  ge_scalarmult(&A, s, &B);
  ge_tobytes(pk, &A);
  memcpy(sk, seed, 32);
  memcpy(sk + 32, pk, 32);
}
/* Sign (ed25519.go:225-294): A is read from sk[32:64] as given */
void orc_ed25519_sign(uint8_t sig[64], const uint8_t sk[64], const uint8_t *msg, size_t len) {
  uint8_t s[32], prefix[32], h[64], r[32], k[32];
  sha512_ctx c;
  expand(s, prefix, sk);
  sha512_init(&c);
  sha512_update(&c, prefix, 32);
  sha512_update(&c, msg, len);
  sha512_final(&c, h);
  sc_reduce(r, h, 64);
  ge B, R;
  ge_base(&B);
  ge_scalarmult(&R, r, &B);
  ge_tobytes(sig, &R);
  sha512_init(&c);
  sha512_update(&c, sig, 32);
  sha512_update(&c, sk + 32, 32);
  sha512_update(&c, msg, len);
  sha512_final(&c, h);
  sc_reduce(k, h, 64);
  sc_muladd(sig + 32, r, k, s);
}
/* Verify (ed25519.go:329-368), cofactorless */
int orc_ed25519_verify(const uint8_t pk[32], const uint8_t *msg, size_t len, const uint8_t *sig, size_t siglen) {
  if (siglen != 64 || !sc_less_than_order(sig + 32)) return 0;
  ge A, B, sB, kA, Q;
  if (!ge_frombytes(&A, pk)) return 0;
  uint8_t h[64], k[32], enc[32];
  sha512_ctx c;
  sha512_init(&c);
  sha512_update(&c, sig, 32);
  sha512_update(&c, pk, 32);
  sha512_update(&c, msg, len);
  sha512_final(&c, h);
  sc_reduce(k, h, 64);
  fe_neg(&A.X, &A.X);
  fe_neg(&A.T, &A.T);
  ge_base(&B);
  ge_scalarmult(&sB, sig + 32, &B);
  ge_scalarmult(&kA, k, &A);
  ge_add(&Q, &sB, &kA);
  ge_tobytes(enc, &Q);
  return memcmp(enc, sig, 32) == 0;
}

/* ------------------------------------------------------------------ Ed25519-Dilithium2 (eddilithium.go) */
void orc_eddilithium2_keygen(uint8_t pk[1344], uint8_t sk[2560], const uint8_t seed[32]) {
  uint8_t ex[64], esk[64];
  orc_shake256(ex, 64, seed, 32); /* Dilithium2 seed || Ed25519 seed */
  orc_mldsa_keygen(2, pk, sk, ex);
  orc_ed25519_keygen(pk + 1312, esk, ex + 32);
  memcpy(sk + 2528, ex + 32, 32);
}
/* SignTo: the Ed25519 key is rebuilt from the stored seed (PrivateKey.Unpack); returns orc_mldsa_sign's result */
int orc_eddilithium2_sign(uint8_t sig[2484], const uint8_t sk[2560], const uint8_t *msg, size_t len) {
  static const uint8_t zero[32] = {0};
  uint8_t epk[32], esk[64];
  const int rc = orc_mldsa_sign(2, sig, sk, msg, len, NULL, 0, zero, 0);
  orc_ed25519_keygen(epk, esk, sk + 2528);
  orc_ed25519_sign(sig + 2420, esk, msg, len);
  return rc;
}
int orc_eddilithium2_verify(const uint8_t pk[1344], const uint8_t *msg, size_t len, const uint8_t *sig, size_t siglen) {
  if (siglen != 2484) return 0;
  if (!orc_mldsa_verify(2, pk, msg, len, NULL, 0, sig, 2420, 0)) return 0;
  return orc_ed25519_verify(pk + 1312, msg, len, sig + 2420, 64);
}
