/* oracle/ed448.c -- TEST INFRASTRUCTURE ONLY: a plain-C restatement of sign/ed448 (pure Ed448, RFC 8032 section 5.2:
 * ed448.go newKeyFromSeed / signAll / verify), of ecc/goldilocks (point.go FromBytes / ToBytes, the isogeny route of
 * curve.go ScalarBaseMult / CombinedMult, scalar.go FromBytes / Mul / Add with reduceOneWord and modOrder) and of
 * sign/eddilithium3 (eddilithium.go NewKeyFromSeed / SignTo / Verify) on top of liboracle.so's SHAKE256 and round-3
 * Dilithium3.
 *
 * Written for obviousness, not speed, and independent of circl_b200/csrc/ed448.cuh: eight 56-bit limbs with 128-bit
 * products, exponentiation by square-and-multiply, bit-serial double-and-add on the curve and on its 4-isogenous
 * twist, and the reference's 64-bit scalar arithmetic word for word.  Nothing here is constant time. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

typedef unsigned __int128 u128;

/* ------------------------------------------------------------------ GF(p), p = 2^448 - 2^224 - 1 */
typedef struct {
  uint64_t v[8]; /* 56-bit limbs, value = sum v[i] 2^(56 i), not necessarily reduced */
} fe;
static const uint64_t M56 = ((uint64_t)1 << 56) - 1;

static void fe_carry(fe *h) { /* until every limb is below 2^56 */
  for (;;) {
    uint64_t c = 0;
    for (int i = 0; i < 8; i++) {
      h->v[i] += c;
      c = h->v[i] >> 56;
      h->v[i] &= M56;
    }
    if (!c) return;
    h->v[0] += c; /* 2^448 = 2^224 + 1 */
    h->v[4] += c;
  }
}
static void fe_set(fe *h, uint64_t x) {
  memset(h, 0, sizeof *h);
  h->v[0] = x;
}
static void fe_add(fe *h, const fe *f, const fe *g) {
  for (int i = 0; i < 8; i++) h->v[i] = f->v[i] + g->v[i];
  fe_carry(h);
}
/* h = f - g: f + 2p - g limb-wise (2p in limbs: 2^57 - 2 everywhere but limb 4, 2^57 - 4) */
static void fe_sub(fe *h, const fe *f, const fe *g) {
  for (int i = 0; i < 8; i++) h->v[i] = f->v[i] + ((i == 4 ? (M56 - 1) : M56) << 1) - g->v[i];
  fe_carry(h);
}
static void fe_neg(fe *h, const fe *f) {
  fe z;
  fe_set(&z, 0);
  fe_sub(h, &z, f);
}
static void fe_mul(fe *h, const fe *f, const fe *g) {
  u128 t[16] = {0};
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 8; j++) t[i + j] += (u128)f->v[i] * g->v[j];
  /* fold 2^(56 k), k >= 8: 2^448 = 2^224 + 1 */
  for (int k = 15; k >= 8; k--) {
    t[k - 8] += t[k];
    t[k - 4] += t[k];
    t[k] = 0;
  }
  u128 c = 0;
  for (int i = 0; i < 8; i++) {
    t[i] += c;
    c = t[i] >> 56;
    h->v[i] = (uint64_t)t[i] & M56;
  }
  h->v[0] += (uint64_t)c;
  h->v[4] += (uint64_t)c;
  fe_carry(h);
}
static void fe_pow(fe *h, const fe *f, const uint8_t e[56]) {
  fe r, b = *f;
  fe_set(&r, 1);
  for (int i = 447; i >= 0; i--) {
    fe_mul(&r, &r, &r);
    if ((e[i >> 3] >> (i & 7)) & 1) fe_mul(&r, &r, &b);
  }
  *h = r;
}
static void p_bytes(uint8_t p[56]) {
  memset(p, 0xff, 56);
  p[28] = 0xfe;
}
static void fe_tobytes(uint8_t out[56], const fe *f) {
  fe t = *f;
  fe_carry(&t);
  uint8_t b[56], p[56];
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 7; j++) b[7 * i + j] = (uint8_t)(t.v[i] >> (8 * j));
  p_bytes(p);
  for (int pass = 0; pass < 2; pass++) { /* the carried value is below 2p */
    int i = 55;
    while (i > 0 && b[i] == p[i]) i--;
    if (b[i] >= p[i]) {
      int borrow = 0;
      for (int k = 0; k < 56; k++) {
        int d = b[k] - p[k] - borrow;
        borrow = d < 0;
        b[k] = (uint8_t)(d & 0xff);
      }
    }
  }
  memcpy(out, b, 56);
}
static void fe_frombytes(fe *h, const uint8_t in[56]) {
  for (int i = 0; i < 8; i++) {
    h->v[i] = 0;
    for (int j = 0; j < 7; j++) h->v[i] |= (uint64_t)in[7 * i + j] << (8 * j);
  }
}
static int fe_iszero(const fe *f) {
  uint8_t b[56];
  fe_tobytes(b, f);
  uint8_t acc = 0;
  for (int i = 0; i < 56; i++) acc |= b[i];
  return acc == 0;
}
static void fe_inv(fe *h, const fe *f) {
  uint8_t e[56];
  p_bytes(e);
  e[0] = 0xfd; /* p - 2 */
  fe_pow(h, f, e);
}
static void fe_small(fe *h, int64_t s) { /* s mod p for |s| < 2^56 */
  fe t;
  fe_set(&t, (uint64_t)(s < 0 ? -s : s));
  if (s < 0)
    fe_neg(h, &t);
  else
    *h = t;
}

/* ------------------------------------------------------------------ curves: a x^2 + y^2 = 1 + d x^2 y^2
 * goldilocks: a = 1, d = -39081; its 4-isogenous twist: a = -1, d = -39082 */
typedef struct {
  fe x, y, z, t;
} pt;
typedef struct {
  int a;
  int64_t d;
} curve;
static const curve TWIST = {-1, -39082}; /* the goldilocks curve itself only appears through FromBytes and the isogeny */

static void pt_identity(pt *p) {
  fe_set(&p->x, 0);
  fe_set(&p->y, 1);
  fe_set(&p->z, 1);
  fe_set(&p->t, 0);
}
/* extended coordinates, Hisil-Wong-Carter-Dawson 2008 (unified: also used for doubling) */
static void pt_add(pt *r, const pt *p, const pt *q, const curve *c) {
  fe A, B, C, D, E, F, G, H, t, u, dd;
  fe_mul(&A, &p->x, &q->x);
  fe_mul(&B, &p->y, &q->y);
  fe_small(&dd, c->d);
  fe_mul(&C, &p->t, &q->t);
  fe_mul(&C, &C, &dd);
  fe_mul(&D, &p->z, &q->z);
  fe_add(&t, &p->x, &p->y);
  fe_add(&u, &q->x, &q->y);
  fe_mul(&E, &t, &u);
  fe_sub(&E, &E, &A);
  fe_sub(&E, &E, &B);
  fe_sub(&F, &D, &C);
  fe_add(&G, &D, &C);
  if (c->a == 1)
    fe_sub(&H, &B, &A);
  else
    fe_add(&H, &B, &A);
  fe_mul(&r->x, &E, &F);
  fe_mul(&r->y, &G, &H);
  fe_mul(&r->t, &E, &H);
  fe_mul(&r->z, &F, &G);
}
/* [k] P, k little-endian of n bytes, bit-serial */
static void pt_mul(pt *r, const uint8_t *k, int n, const pt *P, const curve *c) {
  pt acc;
  pt_identity(&acc);
  for (int i = 8 * n - 1; i >= 0; i--) {
    pt_add(&acc, &acc, &acc, c);
    if ((k[i >> 3] >> (i & 7)) & 1) pt_add(&acc, &acc, P, c);
  }
  *r = acc;
}
/* isogeny.go push: goldilocks -> twist (sign = +1, D = A) and twist -> goldilocks (sign = -1, D = -A) */
static void pt_push(pt *q, const pt *p, int sign) {
  fe A, B, C, D, E, F, G, H, s;
  fe_add(&s, &p->x, &p->y);
  fe_mul(&A, &p->x, &p->x);
  fe_mul(&B, &p->y, &p->y);
  fe_mul(&C, &p->z, &p->z);
  fe_add(&C, &C, &C);
  if (sign > 0)
    D = A;
  else
    fe_neg(&D, &A);
  fe_mul(&E, &s, &s);
  fe_sub(&E, &E, &A);
  fe_sub(&E, &E, &B);
  fe_add(&H, &B, &D);
  fe_sub(&G, &B, &D);
  fe_sub(&F, &C, &H);
  fe_mul(&q->z, &F, &G);
  fe_mul(&q->x, &E, &F);
  fe_mul(&q->y, &G, &H);
  fe_mul(&q->t, &E, &H);
}
static const uint8_t GX[56] = {
    0x5e, 0xc0, 0x0c, 0xc7, 0x2b, 0xa8, 0x26, 0x26, 0x8e, 0x93, 0x00, 0x8b, 0xe1, 0x80, 0x3b, 0x43, 0x11, 0x65, 0xb6, 0x2a,
    0xf7, 0x1a, 0xae, 0x12, 0x64, 0xa4, 0xd3, 0xa3, 0x24, 0xe3, 0x6d, 0xea, 0x67, 0x17, 0x0f, 0x47, 0x70, 0x65, 0x14, 0x9e,
    0xda, 0x36, 0xbf, 0x22, 0xa6, 0x15, 0x1d, 0x22, 0xed, 0x0d, 0xed, 0x6b, 0xc6, 0x70, 0x19, 0x4f};
static const uint8_t GY[56] = {
    0x14, 0xfa, 0x30, 0xf2, 0x5b, 0x79, 0x08, 0x98, 0xad, 0xc8, 0xd7, 0x4e, 0x2c, 0x13, 0xbd, 0xfd, 0xc4, 0x39, 0x7c, 0xe6,
    0x1c, 0xff, 0xd3, 0x3a, 0xd7, 0xc2, 0xa0, 0x05, 0x1e, 0x9c, 0x78, 0x87, 0x40, 0x98, 0xa3, 0x6c, 0x73, 0x73, 0xea, 0x4b,
    0x62, 0xc7, 0xc9, 0x56, 0x37, 0x20, 0x76, 0x88, 0x24, 0xbc, 0xb6, 0x6e, 0x71, 0x46, 0x3f, 0x69};
static void gen(pt *g) {
  fe_frombytes(&g->x, GX);
  fe_frombytes(&g->y, GY);
  fe_set(&g->z, 1);
  fe_mul(&g->t, &g->x, &g->y);
}
/* ToBytes */
static void pt_tobytes(uint8_t out[57], const pt *p) {
  fe zi, x, y;
  uint8_t xb[56];
  fe_inv(&zi, &p->z);
  fe_mul(&x, &p->x, &zi);
  fe_mul(&y, &p->y, &zi);
  fe_tobytes(xb, &x);
  fe_tobytes(out, &y);
  out[56] = (uint8_t)((xb[0] & 1) << 7);
}
/* FromBytes: InvSqrt gives x = u^3 v (u^5 v^3)^((p-3)/4), a square root of u / v iff v x^2 = u */
static int pt_frombytes(pt *p, const uint8_t in[57]) {
  uint8_t pb[56], e[56];
  if (in[56] & 0x7f) return 0;
  const int sign = in[56] >> 7;
  p_bytes(pb);
  int i = 55;
  while (i > 0 && in[i] == pb[i]) i--;
  if (!(in[i] < pb[i])) return 0;
  fe y, u, v, one, d, x, t, w;
  fe_frombytes(&y, in);
  fe_set(&one, 1);
  fe_small(&d, -39081);
  fe_mul(&u, &y, &y);
  fe_mul(&v, &u, &d);
  fe_sub(&u, &u, &one);
  fe_sub(&v, &v, &one);
  fe_mul(&t, &u, &u);
  fe_mul(&t, &t, &u);  /* u^3 */
  fe_mul(&x, &t, &v);  /* u^3 v */
  fe_mul(&t, &t, &u);
  fe_mul(&t, &t, &u);  /* u^5 */
  fe_mul(&w, &v, &v);
  fe_mul(&w, &w, &v);  /* v^3 */
  fe_mul(&t, &t, &w);
  memset(e, 0xff, 56); /* (p - 3) / 4 = 2^446 - 2^222 - 1 */
  e[55] = 0x3f;
  e[27] = 0xbf;
  fe_pow(&t, &t, e);
  fe_mul(&x, &x, &t);
  fe_mul(&w, &x, &x);
  fe_mul(&w, &w, &v);
  fe_sub(&w, &w, &u);
  if (!fe_iszero(&w)) return 0;
  uint8_t xb[56];
  fe_tobytes(xb, &x);
  int nz = 0;
  for (int k = 0; k < 56; k++) nz |= xb[k];
  if (!nz && sign) return 0;
  if ((xb[0] & 1) != sign) fe_neg(&x, &x);
  p->x = x;
  p->y = y;
  fe_set(&p->z, 1);
  fe_mul(&p->t, &x, &y);
  return 1;
}

/* ------------------------------------------------------------------ scalars (scalar.go, 64-bit words) */
#define N 7
static const uint8_t ORDER[56] = {
    0xf3, 0x44, 0x58, 0xab, 0x92, 0xc2, 0x78, 0x23, 0x55, 0x8f, 0xc5, 0x8d, 0x72, 0xc2, 0x6c, 0x21, 0x90, 0x36, 0xd6, 0xae,
    0x49, 0xdb, 0x4e, 0xc4, 0xe9, 0x23, 0xca, 0x7c, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
    0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0x3f};
static uint64_t ld64(const uint8_t *p) {
  uint64_t v = 0;
  for (int i = 7; i >= 0; i--) v = (v << 8) | p[i];
  return v;
}
static void st64(uint8_t *p, uint64_t v) {
  for (int i = 0; i < 8; i++) p[i] = (uint8_t)(v >> (8 * i));
}
static void from_scalar(uint64_t z[N], const uint8_t x[56]) {
  for (int i = 0; i < N; i++) z[i] = ld64(x + 8 * i);
}
static void to_scalar(uint8_t x[56], const uint64_t z[N]) {
  for (int i = 0; i < N; i++) st64(x + 8 * i, z[i]);
}
static uint64_t add_w(uint64_t *z, const uint64_t *x, int lx, const uint64_t *y, int ly) { /* add(): z = x + y */
  const uint64_t *zz = y;
  int l = lx, Lm = ly;
  if (lx > ly) {
    l = ly;
    Lm = lx;
    zz = x;
  }
  uint64_t c = 0;
  for (int i = 0; i < l; i++) {
    u128 s = (u128)x[i] + y[i] + c;
    z[i] = (uint64_t)s;
    c = (uint64_t)(s >> 64);
  }
  for (int i = l; i < Lm; i++) {
    u128 s = (u128)zz[i] + c;
    z[i] = (uint64_t)s;
    c = (uint64_t)(s >> 64);
  }
  return c;
}
static uint64_t sub_w(uint64_t *z, const uint64_t *x, const uint64_t *y, int l) {
  uint64_t c = 0;
  for (int i = 0; i < l; i++) {
    u128 d = (u128)x[i] - y[i] - c;
    z[i] = (uint64_t)d;
    c = (uint64_t)(d >> 64) & 1;
  }
  return c;
}
static void mul_word(uint64_t *z, int lz, const uint64_t *x, int lx, uint64_t y) { /* mulWord: z = x * y */
  for (int i = 0; i < lz; i++) z[i] = 0;
  uint64_t carry = 0;
  for (int i = 0; i < lx; i++) {
    u128 t = (u128)x[i] * y + z[i] + carry;
    z[i] = (uint64_t)t;
    carry = (uint64_t)(t >> 64);
  }
  z[lx] = carry;
}
static uint64_t RES448[N]; /* residue448 = 2^448 mod order */
static uint64_t O64[N];
static void scalar_init(void) {
  static int done = 0;
  if (done) return;
  from_scalar(O64, ORDER);
  /* 2^448 - 4 order (the order is below 2^446 and 2^448 < 5 order) */
  uint64_t four[N], zero[N] = {0};
  uint64_t c = 0;
  for (int i = 0; i < N; i++) {
    u128 t = (u128)O64[i] * 4 + c;
    four[i] = (uint64_t)t;
    c = (uint64_t)(t >> 64);
  }
  sub_w(RES448, zero, four, N); /* 2^448 - 4 order as a 448-bit value */
  done = 1;
}
static void reduce_one_word(uint64_t z[N], uint64_t x) { /* reduceOneWord */
  uint64_t prod[N + 1];
  mul_word(prod, N + 1, RES448, N, x);
  uint64_t cc = add_w(z, z, N, prod, N);
  mul_word(prod, N + 1, RES448, N, cc);
  add_w(z, z, N, prod, N);
}
static void mod_order(uint64_t z[N]) { /* modOrder: eight masked subtractions */
  for (int i = 0; i < 8; i++) {
    uint64_t x[N];
    uint64_t c = sub_w(x, z, O64, N);
    if (c == 0) memcpy(z, x, sizeof x);
  }
}
static void left_shift(uint64_t z[N], uint64_t low, uint64_t *high) {
  *high = z[N - 1];
  for (int i = N - 1; i > 0; i--) z[i] = z[i - 1];
  z[0] = low;
}
/* Scalar.FromBytes */
static void sc_from_bytes(uint8_t z[56], const uint8_t *x, int n) {
  scalar_init();
  const int nceil = (n + 7) >> 3;
  memset(z, 0, 56);
  if (nceil < N) {
    memcpy(z, x, (size_t)n);
    return;
  }
  const int from = 8 * (nceil - N);
  memcpy(z, x + from, (size_t)(n - from < 56 ? n - from : 56));
  uint64_t z64[N];
  from_scalar(z64, z);
  for (int i = nceil - N - 1; i >= 0; i--) {
    uint64_t high;
    left_shift(z64, ld64(x + 8 * i), &high);
    reduce_one_word(z64, high);
  }
  mod_order(z64);
  to_scalar(z, z64);
}
/* Scalar.Mul */
static void sc_mul(uint8_t z[56], const uint8_t x[56], const uint8_t y[56]) {
  scalar_init();
  uint64_t z64[N], x64[N], y64[N], prod[N + 1], h;
  from_scalar(x64, x);
  from_scalar(y64, y);
  mul_word(prod, N + 1, x64, N, y64[N - 1]);
  memcpy(z64, prod, sizeof z64);
  reduce_one_word(z64, prod[N]);
  for (int i = N - 2; i >= 0; i--) {
    left_shift(z64, 0, &h);
    reduce_one_word(z64, h);
    mul_word(prod, N + 1, x64, N, y64[i]);
    uint64_t c = add_w(z64, z64, N, prod, N);
    reduce_one_word(z64, prod[N] + c);
  }
  mod_order(z64);
  to_scalar(z, z64);
}
/* Scalar.Add */
static void sc_add(uint8_t z[56], const uint8_t x[56], const uint8_t y[56]) {
  scalar_init();
  uint64_t z64[N], x64[N], y64[N], t[N];
  from_scalar(x64, x);
  from_scalar(y64, y);
  uint64_t c = add_w(z64, x64, N, y64, N);
  add_w(t, z64, N, RES448, N);
  if (c) memcpy(z64, t, sizeof t);
  mod_order(z64);
  to_scalar(z, z64);
}
/* divBy4: x * invFour, invFour = (order + 1) / 4 (order = 3 mod 4) */
static void sc_div4(uint8_t z[56], const uint8_t x[56]) {
  uint8_t inv4[56];
  int c = 1;
  for (int i = 0; i < 56; i++) {
    int s = ORDER[i] + c;
    inv4[i] = (uint8_t)s;
    c = s >> 8;
  }
  for (int i = 0; i < 56; i++) inv4[i] = (uint8_t)((inv4[i] >> 2) | (i < 55 ? inv4[i + 1] << 6 : 0));
  sc_mul(z, x, inv4);
}

/* ------------------------------------------------------------------ goldilocks Curve */
/* ScalarBaseMult(k) = pull([k / 4] push(G)) */
static void base_mult(pt *r, const uint8_t k[56]) {
  uint8_t k4[56];
  pt g, gt, q;
  sc_div4(k4, k);
  gen(&g);
  pt_push(&gt, &g, +1);
  pt_mul(&q, k4, 56, &gt, &TWIST);
  pt_push(r, &q, -1);
}
/* CombinedMult(m, n, P) = pull([m / 4] push(G) + [n / 4] push(P)) */
static void combined_mult(pt *r, const uint8_t m[56], const uint8_t n[56], const pt *P) {
  uint8_t m4[56], n4[56];
  pt g, gt, pt_, a, b, s;
  sc_div4(m4, m);
  sc_div4(n4, n);
  gen(&g);
  pt_push(&gt, &g, +1);
  pt_push(&pt_, P, +1);
  pt_mul(&a, m4, 56, &gt, &TWIST);
  pt_mul(&b, n4, 56, &pt_, &TWIST);
  pt_add(&s, &a, &b, &TWIST);
  pt_push(r, &s, -1);
}

void orc_ed448_base_mult(uint8_t out[57], const uint8_t k[56]) {
  pt r;
  base_mult(&r, k);
  pt_tobytes(out, &r);
}

/* ------------------------------------------------------------------ Ed448 */
static void expand(uint8_t s[56], uint8_t prefix[57], const uint8_t seed[57]) {
  uint8_t h[114];
  orc_shake256(h, 114, seed, 57);
  h[0] &= 0xfc; /* deriveSecretScalar */
  h[56] = 0;
  h[55] |= 0x80;
  sc_from_bytes(s, h, 57);
  memcpy(prefix, h + 57, 57);
}
/* SHAKE256(dom4 || a || b || M, 114) */
static void hash4(uint8_t out[114], const uint8_t *ctx, size_t ctxlen, const uint8_t *a, size_t la, const uint8_t *b, size_t lb,
                  const uint8_t *msg, size_t len) {
  uint8_t buf[10 + 255 + 114 + 4096];
  uint8_t *big = NULL, *p = buf;
  const size_t total = 10 + ctxlen + la + lb + len;
  if (total > sizeof buf) p = big = (uint8_t *)malloc(total);
  memcpy(p, "SigEd448", 8);
  p[8] = 0;
  p[9] = (uint8_t)ctxlen;
  size_t o = 10;
  if (ctxlen) memcpy(p + o, ctx, ctxlen);
  o += ctxlen;
  if (la) memcpy(p + o, a, la);
  o += la;
  if (lb) memcpy(p + o, b, lb);
  o += lb;
  if (len) memcpy(p + o, msg, len);
  orc_shake256(out, 114, p, total);
  if (big) free(big);
}
void orc_ed448_keygen(uint8_t pk[57], uint8_t sk[114], const uint8_t seed[57]) {
  uint8_t s[56], prefix[57];
  pt A;
  expand(s, prefix, seed);
  base_mult(&A, s);
  pt_tobytes(pk, &A);
  memcpy(sk, seed, 57);
  memcpy(sk + 57, pk, 57);
}
/* signAll: A is read from sk[57:114] as given; returns -1 for a context longer than 255 bytes (the reference panics) */
int orc_ed448_sign(uint8_t sig[114], const uint8_t sk[114], const uint8_t *msg, size_t len, const uint8_t *ctx, size_t ctxlen) {
  if (ctxlen > 255) return -1;
  uint8_t s[56], prefix[57], h[114], r[56], k[56], S[56];
  pt R;
  expand(s, prefix, sk);
  hash4(h, ctx, ctxlen, prefix, 57, NULL, 0, msg, len);
  sc_from_bytes(r, h, 114);
  base_mult(&R, r);
  pt_tobytes(sig, &R);
  hash4(h, ctx, ctxlen, sig, 57, sk + 57, 57, msg, len);
  sc_from_bytes(k, h, 114);
  sc_mul(S, k, s);
  sc_add(S, S, r);
  memcpy(sig + 57, S, 56);
  sig[113] = 0;
  return 0;
}
/* isLessThanOrder */
static int less_than_order(const uint8_t x[57]) {
  int i = 55;
  while (i > 0 && x[i] == ORDER[i]) i--;
  return x[56] == 0 && x[i] < ORDER[i];
}
int orc_ed448_verify(const uint8_t pk[57], const uint8_t *msg, size_t len, const uint8_t *sig, size_t siglen, const uint8_t *ctx,
                     size_t ctxlen) {
  if (siglen != 114 || ctxlen > 255 || !less_than_order(sig + 57)) return 0;
  pt A, Q;
  if (!pt_frombytes(&A, pk)) return 0;
  uint8_t h[114], k[56], S[56], enc[57];
  hash4(h, ctx, ctxlen, sig, 57, pk, 57, msg, len);
  sc_from_bytes(k, h, 114);
  sc_from_bytes(S, sig + 57, 57);
  fe_neg(&A.x, &A.x); /* P.Neg() */
  fe_neg(&A.t, &A.t);
  combined_mult(&Q, S, k, &A);
  pt_tobytes(enc, &Q);
  return memcmp(enc, sig, 57) == 0;
}

/* ------------------------------------------------------------------ Ed448-Dilithium3 (eddilithium.go) */
void orc_eddilithium3_keygen(uint8_t pk[2009], uint8_t sk[4057], const uint8_t seed[57]) {
  uint8_t ex[89], esk[114];
  orc_shake256(ex, 89, seed, 57); /* Dilithium3 seed (32) || Ed448 seed (57) */
  orc_mldsa_keygen(3, pk, sk, ex);
  orc_ed448_keygen(pk + 1952, esk, ex + 32);
  memcpy(sk + 4000, ex + 32, 57);
}
/* SignTo: the Ed448 key is rebuilt from the stored seed (PrivateKey.Unpack); returns orc_mldsa_sign's result */
int orc_eddilithium3_sign(uint8_t sig[3407], const uint8_t sk[4057], const uint8_t *msg, size_t len) {
  static const uint8_t zero[32] = {0};
  uint8_t epk[57], esk[114];
  const int rc = orc_mldsa_sign(3, sig, sk, msg, len, NULL, 0, zero, 0);
  orc_ed448_keygen(epk, esk, sk + 4000);
  orc_ed448_sign(sig + 3293, esk, msg, len, NULL, 0);
  return rc;
}
int orc_eddilithium3_verify(const uint8_t pk[2009], const uint8_t *msg, size_t len, const uint8_t *sig, size_t siglen) {
  if (siglen != 3407) return 0;
  if (!orc_mldsa_verify(3, pk, msg, len, NULL, 0, sig, 3293, 0)) return 0;
  return orc_ed448_verify(pk + 1952, msg, len, sig + 3293, 114, NULL, 0);
}
