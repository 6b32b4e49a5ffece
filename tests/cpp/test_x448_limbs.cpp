// Host-side check of the X448 limb arithmetic of csrc/x448.cuh against the oracle: the header is plain C++ once the
// CUDA qualifiers are defined away, so the field code is compared in the CPU suite (no GPU needed); the kernel around
// it is covered by tests/test_gpu_x448.py.
#include <cstdio>
#include <cstdint>
#include <cstring>
#define __device__
#define __forceinline__ inline
#define __noinline__
#include "../../circl_b200/csrc/x448.cuh"
extern "C" int orc_x448(uint8_t out[56], const uint8_t scalar[56], const uint8_t *point);
using namespace cb200::x448;

static int bad = 0;
static void expect(bool c, const char* what, int t) {
  if (!c) { bad++; printf("FAIL %s t=%d\n", what, t); }
}
static void enc(uint8_t (&b)[56], const Fe& f) {
  uint32_t w[kWords];
  fe_tobytes(w, f);
  memcpy(b, w, 56);
}
static void dec(Fe& f, const uint8_t (&b)[56]) {
  uint32_t w[kWords];
  memcpy(w, b, 56);
  fe_frombytes(f, w);
}
static bool same(const Fe& f, const Fe& g) {
  uint8_t a[56], b[56];
  enc(a, f);
  enc(b, g);
  return memcmp(a, b, 56) == 0;
}

int main() {
  uint64_t st = 88172645463325252ull;
  auto rnd = [&]() { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return st; };
  // edge values as 56-byte strings: 0, 1, p - 1, p, p + 1, 2^448 - 1 and their canonical residues
  uint8_t e[6][56], want[6][56];
  memset(e, 0, sizeof(e));
  memset(want, 0, sizeof(want));
  e[1][0] = 1;
  memset(e[2], 0xff, 56); e[2][0] = 0xfe; e[2][28] = 0xfe;  // p - 1
  memset(e[3], 0xff, 56); e[3][28] = 0xfe;                  // p
  memset(e[4] + 28, 0xff, 28);                              // p + 1 = 2^448 - 2^224
  memset(e[5], 0xff, 56);                                   // 2^448 - 1
  want[1][0] = 1;
  memcpy(want[2], e[2], 56);
  // p = 0, p + 1 = 1, 2^448 - 1 = 2^224 (mod p)
  want[4][0] = 1;
  want[5][28] = 1;
  for (int i = 0; i < 6; i++) {
    Fe f;
    dec(f, e[i]);
    uint8_t got[56];
    enc(got, f);
    expect(memcmp(got, want[i], 56) == 0, "ToBytes of an edge value", i);
    // f * f^-1 = 1 for the non-zero residues, and f^2 = f * f
    Fe inv, prod, sq, mm, one;
    fe_set(one, 1);
    fe_invert(inv, f);
    fe_mul(prod, f, inv);
    const bool zero = (i == 0 || i == 3);
    Fe zero_fe;
    fe_set(zero_fe, 0);
    expect(same(prod, zero ? zero_fe : one), "f * inv(f)", i);
    fe_sq(sq, f);
    fe_mul(mm, f, f);
    expect(same(sq, mm), "sqr == mul", i);
  }
  {  // (p - 1)^2 = 1
    Fe f, sq, one;
    dec(f, e[2]);
    fe_sq(sq, f);
    fe_set(one, 1);
    expect(same(sq, one), "(p-1)^2 == 1", 0);
  }
  // limbs at the accumulator bound (a sum or difference of two carried values, |v| <= 2^28 + 2^8): the product
  // must equal the product of the same values carried first (exact), which stays far below the bound
  for (int t = 0; t < 2000; t++) {
    const int32_t B = (1 << 28) + (1 << 8);
    Fe f, g, fc, gc, h1, h2, s1, s2;
    for (int i = 0; i < 16; i++) {
      const uint64_t r = rnd();
      f.v[i] = t < 4 ? ((t & 1) ? -B : B) : (int32_t)(r % (2 * (uint64_t)B + 1)) - B;
      g.v[i] = t < 4 ? ((t & 2) ? -B : B) : (int32_t)((r >> 32) % (2 * (uint64_t)B + 1)) - B;
    }
    int64_t tf[16], tg[16];
    for (int i = 0; i < 16; i++) { tf[i] = f.v[i]; tg[i] = g.v[i]; }
    fe_carry(fc, tf);
    fe_carry(gc, tg);
    fe_mul(h1, f, g);
    fe_mul(h2, fc, gc);
    expect(same(h1, h2), "mul at the accumulator bound", t);
    fe_sq(s1, f);
    fe_sq(s2, fc);
    expect(same(s1, s2), "sqr at the accumulator bound", t);
  }
  // double-width products of non-canonical inputs reaching the fold: (2^448 - 1)(p + 1) and (2^448 - 1)^2
  {
    Fe a, b, r1, r2;
    dec(a, e[5]);
    dec(b, e[4]);
    fe_mul(r1, a, b);  // 2^224 * 1
    uint8_t got[56];
    enc(got, r1);
    expect(memcmp(got, want[5], 56) == 0, "(2^448-1)(p+1)", 0);
    fe_sq(r2, a);      // 2^448 = 2^224 + 1
    uint8_t w2[56] = {1};
    w2[28] = 1;
    enc(got, r2);
    expect(memcmp(got, w2, 56) == 0, "(2^448-1)^2", 0);
  }
  // ladder and low-order test against the oracle: random scalars and points, non-canonical and low-order points
  for (int t = 0; t < 300; t++) {
    uint32_t k[kWords], p[kWords], r[kWords];
    for (int i = 0; i < kWords; i++) { k[i] = (uint32_t)rnd(); p[i] = (uint32_t)rnd(); }
    if (t < 6) memcpy(p, e[t], 56);
    if (t == 6) { memset(p, 0, 56); ((uint8_t*)p)[0] = 5; }
    if (t == 7) for (int i = 0; i < kWords; i++) k[i] = 0xffffffffu;
    if (t == 8) for (int i = 0; i < kWords; i++) k[i] = 0;
    const bool ok = scalarmult(r, k, p);
    uint8_t w[56];
    const int wok = orc_x448(w, (const uint8_t*)k, (const uint8_t*)p);
    if (memcmp(w, r, 56) || (int)ok != wok) { bad++; printf("ladder mismatch t=%d ok=%d wok=%d\n", t, (int)ok, wok); }
    if (t < 6) expect(ok == !(t == 0 || t == 1 || t == 2 || t == 3 || t == 4), "low-order status", t);
  }
  printf("bad=%d\n", bad);
  return bad != 0;
}
