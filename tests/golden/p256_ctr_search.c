/* Searches for DeriveKeyPair seeds of DHKEM(P-256, HKDF-SHA256) whose first candidate (ctr = 0) is not a private key
 * (candidate >= n), so that the key comes from ctr >= 1.  About one seed in 2^32 qualifies.
 *
 * seed = prefix (24 bytes, argv[1] in hex) || I2OSP(i, 8) for i = 0, 1, ...; each of the threads takes every
 * nthreads-th i.  Prints "hex(seed)" for the first `want` seeds found (in no particular order) and exits.
 * Build: cc -O2 -pthread p256_ctr_search.c -lcrypto.  Used by make_golden_hpke_p256.py.
 */
#include <openssl/sha.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static const uint8_t kN[32] = {0xff, 0xff, 0xff, 0xff, 0x00, 0x00, 0x00, 0x00, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                               0xbc, 0xe6, 0xfa, 0xad, 0xa7, 0x17, 0x9e, 0x84, 0xf3, 0xb9, 0xca, 0xc2, 0xfc, 0x63, 0x25, 0x51};
static uint8_t prefix[24];
static int nthreads, want;
static volatile int found;
static pthread_mutex_t mu = PTHREAD_MUTEX_INITIALIZER;

static void pad_ctx(SHA256_CTX *c, const uint8_t *key, size_t keylen, uint8_t pad) {
  uint8_t b[64];
  memset(b, 0, 64);
  memcpy(b, key, keylen);
  for (int i = 0; i < 64; i++) b[i] ^= pad;
  SHA256_Init(c);
  SHA256_Update(c, b, 64);
}

static void *run(void *arg) {
  const uint64_t t = (uint64_t)(uintptr_t)arg;
  SHA256_CTX i0, o0, c;
  pad_ctx(&i0, NULL, 0, 0x36);
  pad_ctx(&o0, NULL, 0, 0x5c);
  /* LabeledExtract("", "dkp_prk", seed) and LabeledExpand(prk, "candidate", I2OSP(0, 1), 32) messages */
  uint8_t ext[51], exp[25] = {0, 32, 'H', 'P', 'K', 'E', '-', 'v', '1', 'K', 'E', 'M', 0, 0x10,
                              'c', 'a', 'n', 'd', 'i', 'd', 'a', 't', 'e', 0, 1};
  memcpy(ext, "HPKE-v1KEM\x00\x10" "dkp_prk", 19);
  memcpy(ext + 19, prefix, 24);
  uint8_t prk[32], in[32], cand[32];
  for (uint64_t i = t; !found; i += (uint64_t)nthreads) {
    for (int b = 0; b < 8; b++) ext[43 + b] = (uint8_t)(i >> (56 - 8 * b));
    c = i0;
    SHA256_Update(&c, ext, sizeof ext);
    SHA256_Final(in, &c);
    c = o0;
    SHA256_Update(&c, in, 32);
    SHA256_Final(prk, &c);
    pad_ctx(&c, prk, 32, 0x36);
    SHA256_Update(&c, exp, sizeof exp);
    SHA256_Final(in, &c);
    pad_ctx(&c, prk, 32, 0x5c);
    SHA256_Update(&c, in, 32);
    SHA256_Final(cand, &c);
    if (cand[0] != 0xff || cand[1] != 0xff || cand[2] != 0xff || cand[3] != 0xff) continue;
    if (memcmp(cand, kN, 32) < 0) continue;
    pthread_mutex_lock(&mu);
    if (found < want) {
      for (int b = 0; b < 24; b++) printf("%02x", prefix[b]);
      for (int b = 0; b < 8; b++) printf("%02x", ext[43 + b]);
      printf("\n");
      fflush(stdout);
      found++;
    }
    pthread_mutex_unlock(&mu);
  }
  return NULL;
}

int main(int argc, char **argv) {
  if (argc != 4 || strlen(argv[1]) != 48) {
    fprintf(stderr, "usage: %s prefix_hex(24 bytes) threads count\n", argv[0]);
    return 2;
  }
  for (int b = 0; b < 24; b++) sscanf(argv[1] + 2 * b, "%2hhx", &prefix[b]);
  nthreads = atoi(argv[2]);
  want = atoi(argv[3]);
  pthread_t th[256];
  for (int t = 0; t < nthreads && t < 256; t++) pthread_create(&th[t], NULL, run, (void *)(uintptr_t)t);
  for (int t = 0; t < nthreads && t < 256; t++) pthread_join(th[t], NULL);
  return 0;
}
