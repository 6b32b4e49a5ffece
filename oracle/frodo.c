/*
 * oracle/frodo.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C restatement of FrodoKEM-640-SHAKE (kem/frodo/frodo640shake/{frodo,matrix_shake,noise,util}.go), one
 * function per reference function.  SHAKE128 is liboracle.so's sponge.  All file:line citations are relative to
 * kem/frodo/frodo640shake/ in the reference repository.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

#define N 640
#define NBAR 8
#define LOGQ 15
#define QMASK ((1u << LOGQ) - 1)
#define SEEDA 16
#define SS 16
#define PK 9616
#define SK 19888
#define CT 9720
#define BP_PACKED 9600 /* (logQ * N * NBAR) / 8, frodo.go:29 */

/* sha3.NewShake128 + Write + Read of one message made of up to three parts */
static void shake128(uint8_t *out, size_t outlen, const uint8_t *a, size_t al, const uint8_t *b, size_t bl,
                     const uint8_t *c, size_t cl) {
  orc_sponge s;
  orc_sponge_init(&s, 168, 0x1F);
  if (al) orc_sponge_write(&s, a, al);
  if (bl) orc_sponge_write(&s, b, bl);
  if (cl) orc_sponge_write(&s, c, cl);
  orc_sponge_read(&s, out, outlen);
}

static uint16_t le16(const uint8_t *p) { return (uint16_t)(p[0] | (p[1] << 8)); }

/* noise.go:5 */
static const uint16_t cdf_table[13] = {4643, 13363, 20579, 25843, 29227, 31145, 32103,
                                       32525, 32689, 32745, 32762, 32766, 32767};

/* sample, noise.go:9-26 */
static void sample(uint16_t *v, size_t n) {
  for (size_t i = 0; i < n; i++) {
    uint16_t g = 0, sign = v[i] & 1, u = v[i] >> 1;
    for (int j = 0; j < 12; j++) g += (uint16_t)((uint16_t)(cdf_table[j] - u) >> 15);
    v[i] = (uint16_t)((((uint16_t)-sign) ^ g) + sign);
  }
}

/* pack, util.go:15-51 */
static void pack(uint8_t *out, const uint16_t *in, size_t n) {
  for (size_t i = 0, j = 0; i * 8 < n; i++, j += 15) {
    uint16_t a[8];
    for (int k = 0; k < 8; k++) a[k] = in[i * 8 + k] & QMASK;
    out[j] = (uint8_t)(a[0] >> 7);
    out[j + 1] = (uint8_t)(((a[0] & 0x7F) << 1) | (a[1] >> 14));
    out[j + 2] = (uint8_t)(a[1] >> 6);
    out[j + 3] = (uint8_t)(((a[1] & 0x3F) << 2) | (a[2] >> 13));
    out[j + 4] = (uint8_t)(a[2] >> 5);
    out[j + 5] = (uint8_t)(((a[2] & 0x1F) << 3) | (a[3] >> 12));
    out[j + 6] = (uint8_t)(a[3] >> 4);
    out[j + 7] = (uint8_t)(((a[3] & 0x0F) << 4) | (a[4] >> 11));
    out[j + 8] = (uint8_t)(a[4] >> 3);
    out[j + 9] = (uint8_t)(((a[4] & 0x07) << 5) | (a[5] >> 10));
    out[j + 10] = (uint8_t)(a[5] >> 2);
    out[j + 11] = (uint8_t)(((a[5] & 0x03) << 6) | (a[6] >> 9));
    out[j + 12] = (uint8_t)(a[6] >> 1);
    out[j + 13] = (uint8_t)(((a[6] & 0x01) << 7) | (a[7] >> 8));
    out[j + 14] = (uint8_t)a[7];
  }
}

/* unpack, util.go:53-85 */
static void unpack(uint16_t *out, const uint8_t *in, size_t inlen) {
  for (size_t i = 0, j = 0; i * 15 < inlen; i++, j += 8) {
    const uint8_t *b = in + i * 15;
    out[j] = (uint16_t)((b[0] << 7) | ((b[1] & 0xFE) >> 1));
    out[j + 1] = (uint16_t)(((b[1] & 0x1) << 14) | (b[2] << 6) | ((b[3] & 0xFC) >> 2));
    out[j + 2] = (uint16_t)(((b[3] & 0x03) << 13) | (b[4] << 5) | ((b[5] & 0xF8) >> 3));
    out[j + 3] = (uint16_t)(((b[5] & 0x07) << 12) | (b[6] << 4) | ((b[7] & 0xF0) >> 4));
    out[j + 4] = (uint16_t)(((b[7] & 0x0F) << 11) | (b[8] << 3) | ((b[9] & 0xE0) >> 5));
    out[j + 5] = (uint16_t)(((b[9] & 0x1F) << 10) | (b[10] << 2) | ((b[11] & 0xC0) >> 6));
    out[j + 6] = (uint16_t)(((b[11] & 0x3F) << 9) | (b[12] << 1) | ((b[13] & 0x80) >> 7));
    out[j + 7] = (uint16_t)(((b[13] & 0x7F) << 8) | b[14]);
  }
}

/* encodeMessage, util.go:87-100 */
static void encode_message(uint16_t out[64], const uint8_t msg[16]) {
  int pos = 0;
  for (int i = 0; i * 2 < 16; i++) {
    uint16_t in = le16(msg + 2 * i);
    for (int j = 0; j < 8; j++) {
      out[pos++] = (uint16_t)((in & 3) << (LOGQ - 2));
      in >>= 2;
    }
  }
}

/* decodeMessage, util.go:102-115 */
static void decode_message(uint8_t out[16], const uint16_t msg[64]) {
  int pos = 0;
  memset(out, 0, 16);
  for (int i = 0; i < 16; i++)
    for (int j = 0; j < 4; j++) {
      uint16_t t = (uint16_t)((msg[pos] & QMASK) + (1u << (LOGQ - 3)));
      t = (uint16_t)((t >> (LOGQ - 2)) & 3);
      out[i] |= (uint8_t)(t << (2 * j));
      pos++;
    }
}

/* add / sub, util.go:3-13 */
static void add(uint16_t *out, const uint16_t *l, const uint16_t *r) {
  for (int i = 0; i < 64; i++) out[i] = (uint16_t)((l[i] + r[i]) & QMASK);
}
static void sub(uint16_t *out, const uint16_t *l, const uint16_t *r) {
  for (int i = 0; i < 64; i++) out[i] = (uint16_t)((l[i] - r[i]) & QMASK);
}

/* mulAddSBPlusE, util.go:117-131 */
static void mul_add_sb_plus_e(uint16_t *out, const uint16_t *s, const uint16_t *b, const uint16_t *e) {
  for (int k = 0; k < NBAR; k++)
    for (int i = 0; i < NBAR; i++) {
      uint16_t v = e[k * NBAR + i];
      for (int j = 0; j < N; j++) v = (uint16_t)(v + s[k * N + j] * b[j * NBAR + i]);
      out[k * NBAR + i] = v & QMASK;
    }
}

/* mulBS, util.go:133-143 */
static void mul_bs(uint16_t *out, const uint16_t *b, const uint16_t *s) {
  for (int i = 0; i < NBAR; i++)
    for (int j = 0; j < NBAR; j++) {
      uint16_t v = 0;
      for (int k = 0; k < N; k++) v = (uint16_t)(v + b[i * N + k] * s[j * N + k]);
      out[i * NBAR + j] = v & QMASK;
    }
}

/* ctCompareU16, util.go:145-159 */
static int ct_compare_u16(const uint16_t *l, const uint16_t *r, size_t n) {
  uint16_t v = 0;
  for (size_t i = 0; i < n; i++) v |= l[i] ^ r[i];
  return (uint16_t)(v | (uint16_t)-v) >> 15;
}

/* expandSeedIntoA, matrix_shake.go:7-27 (A is 640 x 640, 800 KiB) */
static void expand_seed_into_a(uint16_t *A, const uint8_t seed[SEEDA]) {
  uint8_t sep[2 + SEEDA], row[2 * N];
  memcpy(sep + 2, seed, SEEDA);
  for (int i = 0; i < N; i++) {
    sep[0] = (uint8_t)i;
    sep[1] = (uint8_t)(i >> 8);
    shake128(row, sizeof row, sep, sizeof sep, NULL, 0, NULL, 0);
    for (int j = 0; j < N; j++) A[i * N + j] = le16(row + 2 * j);
  }
}

/* mulAddASPlusE, matrix_shake.go:29-41 (out is zero-initialised by the caller, as the Go array is) */
static void mul_add_as_plus_e(uint16_t *out, const uint16_t *A, const uint16_t *s, const uint16_t *e) {
  for (int i = 0; i < N; i++)
    for (int k = 0; k < NBAR; k++) {
      uint16_t sum = e[i * NBAR + k];
      for (int j = 0; j < N; j++) sum = (uint16_t)(sum + A[i * N + j] * s[k * N + j]);
      out[i * NBAR + k] = (uint16_t)(out[i * NBAR + k] + sum);
    }
}

/* mulAddSAPlusE, matrix_shake.go:43-55 */
static void mul_add_sa_plus_e(uint16_t *out, const uint16_t *s, const uint16_t *A, const uint16_t *e) {
  for (int i = 0; i < N; i++)
    for (int k = 0; k < NBAR; k++) {
      uint16_t sum = e[k * N + i];
      for (int j = 0; j < N; j++) sum = (uint16_t)(sum + A[j * N + i] * s[k * N + j]);
      out[k * N + i] = (uint16_t)(out[k * N + i] + sum);
    }
}

/* newKeyFromSeed, frodo.go:84-135, with PrivateKey.Pack / PublicKey.Pack (frodo.go:334-389) */
void orc_frodo_keygen(uint8_t pk[PK], uint8_t sk[SK], const uint8_t seed[48]) {
  uint16_t *A = malloc(sizeof(uint16_t) * N * N);
  uint16_t S[N * NBAR], E[N * NBAR], B[N * NBAR];
  uint8_t byteSE[2 * (N * NBAR + N * NBAR)];
  uint8_t seedA[SEEDA];
  shake128(seedA, SEEDA, seed + 2 * SS, 16, NULL, 0, NULL, 0);
  const uint8_t ds = 0x5F;
  shake128(byteSE, sizeof byteSE, &ds, 1, seed + SS, SS, NULL, 0);
  for (int i = 0; i < N * NBAR; i++) S[i] = le16(byteSE + 2 * i);
  sample(S, N * NBAR);
  for (int i = 0; i < N * NBAR; i++) E[i] = le16(byteSE + 2 * (N * NBAR + i));
  sample(E, N * NBAR);
  expand_seed_into_a(A, seedA);
  memset(B, 0, sizeof B);
  mul_add_as_plus_e(B, A, S, E);
  free(A);
  memcpy(pk, seedA, SEEDA);
  pack(pk + SEEDA, B, N * NBAR);
  memcpy(sk, seed, SS);
  memcpy(sk + SS, pk, PK);
  for (int i = 0; i < N * NBAR; i++) {
    sk[SS + PK + 2 * i] = (uint8_t)S[i];
    sk[SS + PK + 2 * i + 1] = (uint8_t)(S[i] >> 8);
  }
  shake128(sk + SS + PK + 2 * N * NBAR, 16, pk, PK, NULL, 0, NULL, 0);
}

/* EncapsulateTo, frodo.go:160-240, on PublicKey.Unpack of pk (frodo.go:394-401) */
void orc_frodo_encaps(uint8_t ct[CT], uint8_t ss[SS], const uint8_t pk[PK], const uint8_t seed[16]) {
  uint16_t *A = malloc(sizeof(uint16_t) * N * N);
  uint16_t B[N * NBAR], SpEpEpp[2 * N * NBAR + NBAR * NBAR], Bp[N * NBAR], V[64], C[64];
  uint8_t byteSE[2 * (2 * N * NBAR + NBAR * NBAR)];
  uint8_t hpk[16], G2out[32];
  unpack(B, pk + SEEDA, PK - SEEDA);
  shake128(hpk, 16, pk, PK, NULL, 0, NULL, 0);
  shake128(G2out, 32, hpk, 16, seed, 16, NULL, 0);
  const uint8_t ds = 0x96;
  shake128(byteSE, sizeof byteSE, &ds, 1, G2out, SS, NULL, 0);
  for (size_t i = 0; i < 2 * N * NBAR + NBAR * NBAR; i++) SpEpEpp[i] = le16(byteSE + 2 * i);
  sample(SpEpEpp, 2 * N * NBAR + NBAR * NBAR);
  const uint16_t *Sp = SpEpEpp, *Ep = SpEpEpp + N * NBAR, *Epp = SpEpEpp + 2 * N * NBAR;
  expand_seed_into_a(A, pk);
  memset(Bp, 0, sizeof Bp);
  mul_add_sa_plus_e(Bp, Sp, A, Ep);
  free(A);
  mul_add_sb_plus_e(V, Sp, B, Epp);
  encode_message(C, seed);
  add(C, V, C);
  pack(ct, Bp, N * NBAR);
  pack(ct + BP_PACKED, C, 64);
  shake128(ss, SS, ct, CT, G2out + SS, SS, NULL, 0);
}

/* DecapsulateTo, frodo.go:247-329, on PrivateKey.Unpack of sk (frodo.go:359-377) */
void orc_frodo_decaps(uint8_t ss[SS], const uint8_t sk[SK], const uint8_t ct[CT]) {
  uint16_t *A = malloc(sizeof(uint16_t) * N * N);
  uint16_t S[N * NBAR], B[N * NBAR], Bp[N * NBAR], C[64], W[64], CC[64], BBp[N * NBAR];
  uint16_t SpEpEpp[2 * N * NBAR + NBAR * NBAR];
  uint8_t byteSE[2 * (2 * N * NBAR + NBAR * NBAR)];
  uint8_t mu[16], G2out[32], kp[SS];
  const uint8_t *s = sk, *pk = sk + SS, *hpk = sk + SS + PK + 2 * N * NBAR;
  unpack(B, pk + SEEDA, PK - SEEDA);
  for (int i = 0; i < N * NBAR; i++) S[i] = le16(sk + SS + PK + 2 * i);
  unpack(Bp, ct, BP_PACKED);
  unpack(C, ct + BP_PACKED, CT - BP_PACKED);
  mul_bs(W, Bp, S);
  sub(W, C, W);
  decode_message(mu, W);
  shake128(G2out, 32, hpk, 16, mu, 16, NULL, 0);
  const uint8_t ds = 0x96;
  shake128(byteSE, sizeof byteSE, &ds, 1, G2out, SS, NULL, 0);
  for (size_t i = 0; i < 2 * N * NBAR + NBAR * NBAR; i++) SpEpEpp[i] = le16(byteSE + 2 * i);
  sample(SpEpEpp, 2 * N * NBAR + NBAR * NBAR);
  const uint16_t *Sp = SpEpEpp, *Ep = SpEpEpp + N * NBAR, *Epp = SpEpEpp + 2 * N * NBAR;
  expand_seed_into_a(A, pk);
  memset(BBp, 0, sizeof BBp);
  mul_add_sa_plus_e(BBp, Sp, A, Ep);
  free(A);
  for (int i = 0; i < N * NBAR; i++) BBp[i] &= QMASK;
  mul_add_sb_plus_e(W, Sp, B, Epp);
  encode_message(CC, mu);
  add(CC, W, CC);
  const int selector = ct_compare_u16(Bp, BBp, N * NBAR) | ct_compare_u16(C, CC, 64);
  /* subtle.ConstantTimeCopy(selector, kprime, s) */
  const uint8_t mask = (uint8_t)(0 - selector);
  for (int i = 0; i < SS; i++) kp[i] = (uint8_t)(G2out[SS + i] ^ (mask & (G2out[SS + i] ^ s[i])));
  shake128(ss, SS, ct, CT, kp, SS, NULL, 0);
}

/* the sampler on one value, for the host test of the device header */
uint16_t orc_frodo_sample(uint16_t r) {
  sample(&r, 1);
  return r;
}
void orc_frodo_pack(uint8_t *out, const uint16_t *in, size_t n) { pack(out, in, n); }
void orc_frodo_unpack(uint16_t *out, const uint8_t *in, size_t inlen) { unpack(out, in, inlen); }
void orc_frodo_encode(uint16_t out[64], const uint8_t msg[16]) { encode_message(out, msg); }
void orc_frodo_decode(uint8_t out[16], const uint16_t msg[64]) { decode_message(out, msg); }

/* ---- batches over host threads (op = 0 keygen, 1 encaps, 2 decaps); key stride 0 = one key for the batch ---- */
typedef struct {
  int op;
  const uint8_t *key, *in;
  size_t key_stride;
  uint8_t *out0, *out1;
  size_t first, count;
} job;

static void *run_job(void *p) {
  job *j = p;
  for (size_t i = j->first; i < j->first + j->count; i++) {
    if (j->op == 0)
      orc_frodo_keygen(j->out0 + i * PK, j->out1 + i * SK, j->in + i * 48);
    else if (j->op == 1)
      orc_frodo_encaps(j->out0 + i * CT, j->out1 + i * SS, j->key + i * j->key_stride, j->in + i * 16);
    else
      orc_frodo_decaps(j->out1 + i * SS, j->key + i * j->key_stride, j->in + i * CT);
  }
  return NULL;
}

void orc_frodo_batch(int op, const uint8_t *key, size_t key_stride, const uint8_t *in, uint8_t *out0, uint8_t *out1,
                     size_t n, int nthreads) {
  if (nthreads < 1) nthreads = 1;
  pthread_t th[256];
  job jobs[256];
  if (nthreads > 256) nthreads = 256;
  size_t per = (n + (size_t)nthreads - 1) / (size_t)nthreads, first = 0;
  int used = 0;
  for (int t = 0; t < nthreads && first < n; t++, used++) {
    size_t c = per < n - first ? per : n - first;
    jobs[t] = (job){op, key, in, key_stride, out0, out1, first, c};
    pthread_create(&th[t], NULL, run_job, &jobs[t]);
    first += c;
  }
  for (int t = 0; t < used; t++) pthread_join(th[t], NULL);
}
