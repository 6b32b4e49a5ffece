// Host-side check of the lane mapping of the K-PKE kernels' noise (csrc/kyber.cuh: noise_select, noise_pairs, noise_cbd;
// compiled by nvcc as host code, no GPU needed): for random seeds and nonces, the PRF output SHAKE256(seed || nonce) is
// gathered and turned into coefficients lane by lane, and lane v's r[2 s + b] must equal coefficient 16 s + 2 v + b of
// the oracle's DeriveNoise for eta = 2 and 3, for every v, s and b.  The kernels around these functions are covered by
// the GPU suite (tests/test_gpu_mlkem.py, tests/test_gpu_mlkem_subbatch.py).
#include <cstdint>
#include <cstdio>
#include <cstring>

#include "../../circl_b200/csrc/kyber.cuh"

extern "C" {
void orc_shake256(uint8_t* out, size_t outlen, const uint8_t* in, size_t n);
void orc_kyber_derive_noise(int16_t p[256], const uint8_t* seed, size_t seedlen, uint8_t nonce, int eta);
}
using namespace cb200::kyber;

static uint64_t st = 0x243f6a8885a308d3ull;
static uint64_t rnd() { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return st; }

template <int ETA>
static long check(const uint8_t seed[32], uint8_t nonce) {
  uint8_t in[33];
  memcpy(in, seed, 32);
  in[32] = nonce;
  uint32_t w[48];  // the squeezed words as a lane reads them from shared memory (little-endian)
  uint8_t b[192];
  orc_shake256(b, 64 * ETA, in, 33);
  for (int i = 0; i < 16 * ETA; i++) w[i] = b[4 * i] | (b[4 * i + 1] << 8) | (b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
  int16_t ref[256];
  orc_kyber_derive_noise(ref, seed, 32, nonce, ETA);
  long bad = 0;
  for (int v = 0; v < 8; v++) {
    uint32_t x[kNoiseWords<ETA>];
    noise_select<ETA>(w, v, x);
    int32_t r[32];
    noise_cbd<ETA>(x, r);
    for (int s = 0; s < 16; s++)
      for (int bb = 0; bb < 2; bb++) {
        const int c = 16 * s + 2 * v + bb;
        if (r[2 * s + bb] != ref[c]) {
          if (bad < 5) printf("eta=%d nonce=%d v=%d s=%d b=%d: %d != %d\n", ETA, nonce, v, s, bb, r[2 * s + bb], ref[c]);
          bad++;
        }
      }
  }
  return bad;
}

int main() {
  long bad = 0, polys = 0;
  for (int t = 0; t < 2000; t++) {
    uint8_t seed[32];
    for (int i = 0; i < 32; i++) seed[i] = (uint8_t)rnd();
    const uint8_t nonce = (uint8_t)(t < 256 ? t : rnd());
    bad += check<2>(seed, nonce);
    bad += check<3>(seed, nonce);
    polys += 2;
  }
  printf("polys=%ld bad=%ld\n", polys, bad);
  return bad != 0;
}
