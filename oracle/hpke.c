/* oracle/hpke.c -- TEST INFRASTRUCTURE ONLY (see oracle.h): CPU restatement of HPKE's two Montgomery-curve DHKEMs
 * (RFC 9180 section 4.1) as the reference computes them:
 *   hpke/kembase.go:36-80        LabeledExtract / LabeledExpand, suite_id = "KEM" || I2OSP(kem_id, 2)
 *   hpke/kembase.go:94-241       ExtractAndExpand, Encap, AuthEncap, Decap, AuthDecap
 *   hpke/xkem.go:20-163          sizes, DeriveKeyPair (sk stored unclamped), calcDH (Shared returning false ->
 *                                hpke.ErrInvalidKEMSharedSecret), KeyGen for the public key
 * with SHA-256 and SHA-512 (FIPS 180-4), HMAC (RFC 2104) and HKDF (RFC 5869) written out below, over orc_x25519
 * (liboracle.so) and orc_x448 (liboracle_x448.so).  Written for obviousness, not speed, and independent of
 * circl_b200/csrc/sha2.cuh.  Built on its own into liboracle_hpke.so (oracle/hpke.py).
 */
#include <string.h>

#include "oracle.h"

int orc_x448(uint8_t out[56], const uint8_t scalar[56], const uint8_t *point);

/* ---------------------------------------------------------------- SHA-256 */
static const uint32_t K256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
    0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
    0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
    0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
    0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
    0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
static uint32_t ror32(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
static void sha256_compress(uint32_t h[8], const uint8_t blk[64]) {
  uint32_t w[64];
  for (int t = 0; t < 16; t++)
    w[t] = ((uint32_t)blk[4 * t] << 24) | ((uint32_t)blk[4 * t + 1] << 16) | ((uint32_t)blk[4 * t + 2] << 8) | blk[4 * t + 3];
  for (int t = 16; t < 64; t++) {
    const uint32_t s0 = ror32(w[t - 15], 7) ^ ror32(w[t - 15], 18) ^ (w[t - 15] >> 3);
    const uint32_t s1 = ror32(w[t - 2], 17) ^ ror32(w[t - 2], 19) ^ (w[t - 2] >> 10);
    w[t] = w[t - 16] + s0 + w[t - 7] + s1;
  }
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
  for (int t = 0; t < 64; t++) {
    const uint32_t t1 = hh + (ror32(e, 6) ^ ror32(e, 11) ^ ror32(e, 25)) + ((e & f) ^ (~e & g)) + K256[t] + w[t];
    const uint32_t t2 = (ror32(a, 2) ^ ror32(a, 13) ^ ror32(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
    hh = g, g = f, f = e, e = d + t1, d = c, c = b, b = a, a = t1 + t2;
  }
  h[0] += a, h[1] += b, h[2] += c, h[3] += d, h[4] += e, h[5] += f, h[6] += g, h[7] += hh;
}
static void sha256(uint8_t out[32], const uint8_t *m, size_t len) {
  uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  uint8_t blk[64];
  size_t off = 0;
  for (; off + 64 <= len; off += 64) sha256_compress(h, m + off);
  const size_t rem = len - off;
  memset(blk, 0, 64);
  memcpy(blk, m + off, rem);
  blk[rem] = 0x80;
  if (rem >= 56) {
    sha256_compress(h, blk);
    memset(blk, 0, 64);
  }
  const uint64_t bits = (uint64_t)len * 8;
  for (int i = 0; i < 8; i++) blk[63 - i] = (uint8_t)(bits >> (8 * i));
  sha256_compress(h, blk);
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 4; j++) out[4 * i + j] = (uint8_t)(h[i] >> (24 - 8 * j));
}

/* ---------------------------------------------------------------- SHA-512 */
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
static uint64_t ror64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
static void sha512_compress(uint64_t h[8], const uint8_t blk[128]) {
  uint64_t w[80];
  for (int t = 0; t < 16; t++) {
    w[t] = 0;
    for (int j = 0; j < 8; j++) w[t] = (w[t] << 8) | blk[8 * t + j];
  }
  for (int t = 16; t < 80; t++) {
    const uint64_t s0 = ror64(w[t - 15], 1) ^ ror64(w[t - 15], 8) ^ (w[t - 15] >> 7);
    const uint64_t s1 = ror64(w[t - 2], 19) ^ ror64(w[t - 2], 61) ^ (w[t - 2] >> 6);
    w[t] = w[t - 16] + s0 + w[t - 7] + s1;
  }
  uint64_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
  for (int t = 0; t < 80; t++) {
    const uint64_t t1 = hh + (ror64(e, 14) ^ ror64(e, 18) ^ ror64(e, 41)) + ((e & f) ^ (~e & g)) + K512[t] + w[t];
    const uint64_t t2 = (ror64(a, 28) ^ ror64(a, 34) ^ ror64(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
    hh = g, g = f, f = e, e = d + t1, d = c, c = b, b = a, a = t1 + t2;
  }
  h[0] += a, h[1] += b, h[2] += c, h[3] += d, h[4] += e, h[5] += f, h[6] += g, h[7] += hh;
}
static void sha512(uint8_t out[64], const uint8_t *m, size_t len) {
  uint64_t h[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                   0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
  uint8_t blk[128];
  size_t off = 0;
  for (; off + 128 <= len; off += 128) sha512_compress(h, m + off);
  const size_t rem = len - off;
  memset(blk, 0, 128);
  memcpy(blk, m + off, rem);
  blk[rem] = 0x80;
  if (rem >= 112) {
    sha512_compress(h, blk);
    memset(blk, 0, 128);
  }
  const uint64_t bits = (uint64_t)len * 8;
  for (int i = 0; i < 8; i++) blk[127 - i] = (uint8_t)(bits >> (8 * i));
  sha512_compress(h, blk);
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 8; j++) out[8 * i + j] = (uint8_t)(h[i] >> (56 - 8 * j));
}

/* ---------------------------------------------------------------- HMAC, HKDF with HPKE's labels */
typedef struct {
  int id;         /* kem_id */
  size_t n;       /* Nsk = Npk = Nenc = Nsecret seed (xkem.go:20-24) */
  size_t nh;      /* digest size; the shared secret's size (kembase.go:34) */
  size_t block;   /* hash block size */
  void (*hash)(uint8_t *out, const uint8_t *m, size_t len);
} kem_t;

static void hash256(uint8_t *out, const uint8_t *m, size_t len) { sha256(out, m, len); }
static void hash512(uint8_t *out, const uint8_t *m, size_t len) { sha512(out, m, len); }

static int kem_of(int id, kem_t *k) {
  if (id == 0x20) {
    *k = (kem_t){0x20, 32, 32, 64, hash256};
    return 1;
  }
  if (id == 0x21) {
    *k = (kem_t){0x21, 56, 64, 128, hash512};
    return 1;
  }
  return 0;
}

#define MAXMSG 512
/* HMAC(key, m), key at most one block (every key here is a digest or the empty salt) */
static void hmac(const kem_t *k, uint8_t *out, const uint8_t *key, size_t keylen, const uint8_t *m, size_t len) {
  uint8_t buf[128 + MAXMSG], inner[64];
  memset(buf, 0, k->block);
  memcpy(buf, key, keylen);
  for (size_t i = 0; i < k->block; i++) buf[i] ^= 0x36;
  memcpy(buf + k->block, m, len);
  k->hash(inner, buf, k->block + len);
  memset(buf, 0, k->block);
  memcpy(buf, key, keylen);
  for (size_t i = 0; i < k->block; i++) buf[i] ^= 0x5c;
  memcpy(buf + k->block, inner, k->nh);
  k->hash(out, buf, k->block + k->nh);
}
/* "HPKE-v1" || suite_id, suite_id = "KEM" || I2OSP(kem_id, 2) (kembase.go:36-48) */
static size_t put_prefix(const kem_t *k, uint8_t *m) {
  memcpy(m, "HPKE-v1KEM", 10);
  m[10] = (uint8_t)(k->id >> 8);
  m[11] = (uint8_t)k->id;
  return 12;
}
/* LabeledExtract("", label, ikm) = HKDF-Extract(salt = "", labeled ikm) (kembase.go:50-62) */
static void labeled_extract(const kem_t *k, uint8_t *prk, const char *label, const uint8_t *ikm, size_t ikmlen) {
  uint8_t m[MAXMSG];
  size_t o = put_prefix(k, m);
  memcpy(m + o, label, strlen(label)), o += strlen(label);
  memcpy(m + o, ikm, ikmlen), o += ikmlen;
  hmac(k, prk, NULL, 0, m, o); /* an empty salt is a key of zeros */
}
/* LabeledExpand(prk, label, info, L) = HKDF-Expand(prk, I2OSP(L, 2) || labeled info, L) (kembase.go:64-80) */
static void labeled_expand(const kem_t *k, uint8_t *out, const uint8_t *prk, const char *label, const uint8_t *info,
                           size_t infolen, size_t L) {
  uint8_t m[MAXMSG], t[64];
  size_t o = 0;
  m[o++] = (uint8_t)(L >> 8);
  m[o++] = (uint8_t)L;
  o += put_prefix(k, m + o);
  memcpy(m + o, label, strlen(label)), o += strlen(label);
  memcpy(m + o, info, infolen), o += infolen;
  /* HKDF-Expand: T(i) = HMAC(prk, T(i-1) || info || i) */
  uint8_t blk[64 + MAXMSG];
  size_t done = 0, tl = 0;
  for (uint8_t i = 1; done < L; i++) {
    memcpy(blk, t, tl);
    memcpy(blk + tl, m, o);
    blk[tl + o] = i;
    hmac(k, t, prk, k->nh, blk, tl + o + 1);
    tl = k->nh;
    const size_t take = L - done < k->nh ? L - done : k->nh;
    memcpy(out + done, t, take);
    done += take;
  }
}

/* x25519 / x448 KeyGen (pt NULL) or Shared; returns 0 when Shared returns false */
static int dh(const kem_t *k, uint8_t *out, const uint8_t *sk, const uint8_t *pt) {
  return k->n == 32 ? orc_x25519(out, sk, pt) : orc_x448(out, sk, pt);
}

/* DeriveKeyPair (xkem.go:55-71): sk unclamped, pk = KeyGen(sk) */
int orc_hpke_keygen(int id, uint8_t *pk, uint8_t *sk, const uint8_t *seed) {
  kem_t k;
  if (!kem_of(id, &k)) return -1;
  uint8_t prk[64];
  labeled_extract(&k, prk, "dkp_prk", seed, k.n);
  labeled_expand(&k, sk, prk, "sk", NULL, 0, k.n);
  dh(&k, pk, sk, NULL);
  return 0;
}

/* ExtractAndExpand (kembase.go:94-118) */
static void kdf(const kem_t *k, uint8_t *ss, const uint8_t *dhv, size_t dhlen, const uint8_t *ctx, size_t ctxlen) {
  uint8_t prk[64];
  labeled_extract(k, prk, "eae_prk", dhv, dhlen);
  labeled_expand(k, ss, prk, "shared_secret", ctx, ctxlen, k->nh);
}

/* Encap / AuthEncap (kembase.go:120-159; skS NULL for Encap): 0, or 1 = hpke.ErrInvalidKEMSharedSecret (ss zeroed) */
int orc_hpke_encaps(int id, uint8_t *enc, uint8_t *ss, const uint8_t *pkR, const uint8_t *skS, const uint8_t *seed) {
  kem_t k;
  if (!kem_of(id, &k)) return -1;
  uint8_t skE[56], dhv[112], ctx[168];
  orc_hpke_keygen(id, enc, skE, seed);
  int ok = dh(&k, dhv, skE, pkR);
  memcpy(ctx, enc, k.n);
  memcpy(ctx + k.n, pkR, k.n);
  size_t dhlen = k.n, ctxlen = 2 * k.n;
  if (skS) {
    ok &= dh(&k, dhv + k.n, skS, pkR);
    dh(&k, ctx + 2 * k.n, skS, NULL);
    dhlen += k.n, ctxlen += k.n;
  }
  if (!ok) {
    memset(ss, 0, k.nh);
    return 1;
  }
  kdf(&k, ss, dhv, dhlen, ctx, ctxlen);
  return 0;
}

/* Decap / AuthDecap (kembase.go:185-241; pkS NULL for Decap): pkR = KeyGen(skR) */
int orc_hpke_decaps(int id, uint8_t *ss, const uint8_t *skR, const uint8_t *enc, const uint8_t *pkS) {
  kem_t k;
  if (!kem_of(id, &k)) return -1;
  uint8_t dhv[112], ctx[168];
  int ok = dh(&k, dhv, skR, enc);
  memcpy(ctx, enc, k.n);
  dh(&k, ctx + k.n, skR, NULL);
  size_t dhlen = k.n, ctxlen = 2 * k.n;
  if (pkS) {
    ok &= dh(&k, dhv + k.n, skR, pkS);
    memcpy(ctx + 2 * k.n, pkS, k.n);
    dhlen += k.n, ctxlen += k.n;
  }
  if (!ok) {
    memset(ss, 0, k.nh);
    return 1;
  }
  kdf(&k, ss, dhv, dhlen, ctx, ctxlen);
  return 0;
}

/* the raw hashes, for the oracle's own tests */
void orc_sha256(uint8_t out[32], const uint8_t *m, size_t len) { sha256(out, m, len); }
void orc_sha512(uint8_t out[64], const uint8_t *m, size_t len) { sha512(out, m, len); }
