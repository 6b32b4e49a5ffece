// SHA-256 (FIPS 180-4), and HMAC (RFC 2104) and HPKE's labeled HKDF (RFC 9180 section 4) over SHA-256, SHA-384 and
// SHA-512, one message per thread.  SHA-512's compression function is ed25519.cuh's; SHA-384 is the same compression
// from its own initial value, with the digest cut to six words.
//
// The HPKE KEMs hash short messages of fixed, public lengths whose bytes come from a few places: constant labels,
// rows in memory and values held in registers.  A message is therefore a functor msg(j) returning byte j; the block
// loops are unrolled, so once a caller's lengths are constants every position is known at compile time and a label
// byte becomes an immediate.  No branch or address depends on a message byte.
//
// HMAC keys are at most one block here: the all-zero salt of LabeledExtract (its two pad states are constants below,
// so an Extract costs its message blocks plus one outer block) and a pseudorandom key of one digest.
// Plain integer C++ like ed25519.cuh: it compiles for the device and for the host-only test of the CPU suite.
#pragma once
#include <cstdint>

#include "ed25519.cuh"

namespace cb200 {
namespace sha2 {

#define CB200_SHA256_K_BODY                                                                                              \
  0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u, 0xd807aa98u,    \
      0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, 0xe49b69c1u, 0xefbe4786u,\
      0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau, 0x983e5152u, 0xa831c66du, 0xb00327c8u,\
      0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u, 0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u,\
      0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u, 0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u,\
      0xd6990624u, 0xf40e3585u, 0x106aa070u, 0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au,\
      0x5b9cca4fu, 0x682e6ff3u, 0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u,\
      0xc67178f2u
#if defined(__CUDACC__)
static __constant__ uint32_t kSha256K_dev[64] = {CB200_SHA256_K_BODY};
#endif
static const uint32_t kSha256K_host[64] = {CB200_SHA256_K_BODY};
#undef CB200_SHA256_K_BODY

CB200_XHD uint32_t sha256_k(int i) {
#if defined(__CUDA_ARCH__)
  return kSha256K_dev[i];
#else
  return kSha256K_host[i];
#endif
}
CB200_XHD uint32_t rotr32(uint32_t x, int n) {
#if defined(__CUDA_ARCH__)
  return __funnelshift_r(x, x, n);
#else
  return (x >> n) | (x << (32 - n));
#endif
}

CB200_XHD void sha256_block(uint32_t (&H)[8], uint32_t (&W)[16]) {
  uint32_t a = H[0], b = H[1], c = H[2], d = H[3], e = H[4], f = H[5], g = H[6], h = H[7];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int r = 0; r < 64; r += 16) {
#pragma unroll
    for (int j = 0; j < 16; j++) {
      if (r > 0) {
        const uint32_t w1 = W[(j + 1) & 15], w14 = W[(j + 14) & 15];
        W[j] += (rotr32(w14, 17) ^ rotr32(w14, 19) ^ (w14 >> 10)) + W[(j + 9) & 15] +
                (rotr32(w1, 7) ^ rotr32(w1, 18) ^ (w1 >> 3));
      }
      const uint32_t t1 = h + (rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25)) + ((e & f) ^ (~e & g)) + sha256_k(r + j) + W[j];
      const uint32_t t2 = (rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
      h = g;
      g = f;
      f = e;
      e = d + t1;
      d = c;
      c = b;
      b = a;
      a = t1 + t2;
    }
  }
  H[0] += a;
  H[1] += b;
  H[2] += c;
  H[3] += d;
  H[4] += e;
  H[5] += f;
  H[6] += g;
  H[7] += h;
}

// The three hashes behind one interface.  W: state and message word; the state is 8 words and a digest its first
// kDigest bytes, big-endian within each word.  ipad0 / opad0: the state after the first block of HMAC with the
// all-zero key (any zero key up to a block long), i.e. the compression of 0x36... / 0x5c... from the initial value.
struct Sha256 {
  using W = uint32_t;
  static constexpr int kBlock = 64, kWordBytes = 4, kDigest = 32;
  CB200_XHD static void iv(W (&H)[8]) {
    H[0] = 0x6a09e667u, H[1] = 0xbb67ae85u, H[2] = 0x3c6ef372u, H[3] = 0xa54ff53au;
    H[4] = 0x510e527fu, H[5] = 0x9b05688cu, H[6] = 0x1f83d9abu, H[7] = 0x5be0cd19u;
  }
  CB200_XHD static void ipad0(W (&H)[8]) {
    H[0] = 0xf454deadu, H[1] = 0x9725214fu, H[2] = 0x90daf2a0u, H[3] = 0xdf1228eau;
    H[4] = 0x64e5750fu, H[5] = 0xa3924181u, H[6] = 0x824a932bu, H[7] = 0xf8e04e32u;
  }
  CB200_XHD static void opad0(W (&H)[8]) {
    H[0] = 0xd385480fu, H[1] = 0x7abb6477u, H[2] = 0x37c9c538u, H[3] = 0x5dd82467u;
    H[4] = 0x8e043a72u, H[5] = 0x753434b0u, H[6] = 0xdeb82818u, H[7] = 0x361d45a6u;
  }
  CB200_XHD static void compress(W (&H)[8], W (&M)[16]) { sha256_block(H, M); }
};
struct Sha512 {
  using W = uint64_t;
  static constexpr int kBlock = 128, kWordBytes = 8, kDigest = 64;
  CB200_XHD static void iv(W (&H)[8]) {
    H[0] = 0x6a09e667f3bcc908ull, H[1] = 0xbb67ae8584caa73bull, H[2] = 0x3c6ef372fe94f82bull, H[3] = 0xa54ff53a5f1d36f1ull;
    H[4] = 0x510e527fade682d1ull, H[5] = 0x9b05688c2b3e6c1full, H[6] = 0x1f83d9abfb41bd6bull, H[7] = 0x5be0cd19137e2179ull;
  }
  CB200_XHD static void ipad0(W (&H)[8]) {
    H[0] = 0x1aa8caac196aa9cfull, H[1] = 0x157bc66ffacbb113ull, H[2] = 0x2f5813b01a6d99fbull, H[3] = 0x6b15a0122ed28282ull;
    H[4] = 0xb31bdcd996d81fa6ull, H[5] = 0x151961af57cb87c1ull, H[6] = 0xdb05ba3a642721c9ull, H[7] = 0x3aa11644c5429812ull;
  }
  CB200_XHD static void opad0(W (&H)[8]) {
    H[0] = 0x1efe832e03f7255bull, H[1] = 0x2b9bb33f32f60445ull, H[2] = 0xf9d607f52ec5b0a3ull, H[3] = 0x11afe3481f43b83dull;
    H[4] = 0x68dee3ab8db272b7ull, H[5] = 0x815ffb34f560a851ull, H[6] = 0xfc6950d7e19a3529ull, H[7] = 0x23f2e1e9645f0fe6ull;
  }
  CB200_XHD static void compress(W (&H)[8], W (&M)[16]) { ed25519::sha512_block(H, M); }
};
struct Sha384 {
  using W = uint64_t;
  static constexpr int kBlock = 128, kWordBytes = 8, kDigest = 48;
  CB200_XHD static void iv(W (&H)[8]) {
    H[0] = 0xcbbb9d5dc1059ed8ull, H[1] = 0x629a292a367cd507ull, H[2] = 0x9159015a3070dd17ull, H[3] = 0x152fecd8f70e5939ull;
    H[4] = 0x67332667ffc00b31ull, H[5] = 0x8eb44a8768581511ull, H[6] = 0xdb0c2e0d64f98fa7ull, H[7] = 0x47b5481dbefa4fa4ull;
  }
  CB200_XHD static void ipad0(W (&H)[8]) {
    H[0] = 0x53f869327560c3a2ull, H[1] = 0xc237b05164a5bbe8ull, H[2] = 0xe581f7394cfa66b8ull, H[3] = 0x846fa61922faad62ull;
    H[4] = 0xdd0b37ce462cff5eull, H[5] = 0x7ee8a4bdc87567f3ull, H[6] = 0x39bda99c75a047f7ull, H[7] = 0xc7bd628bd3f9a734ull;
  }
  CB200_XHD static void opad0(W (&H)[8]) {
    H[0] = 0xff6ce3f9ca86c81cull, H[1] = 0x585559c2ae0fc15cull, H[2] = 0xcf0d5686fb65a54eull, H[3] = 0xf1d54ee19e8cfd02ull;
    H[4] = 0xa5c720ab778ff100ull, H[5] = 0xdeb3e5f667573e8cull, H[6] = 0xc1bfc7ec16b591f3ull, H[7] = 0x34d487c1c79d59ebull;
  }
  CB200_XHD static void compress(W (&H)[8], W (&M)[16]) { ed25519::sha512_block(H, M); }
};

// Hashes msg(0 .. len) with FIPS 180-4 padding into H, which already holds `done` bytes (a whole number of blocks).
// Message lengths stay below 2^32 bits, so the length field is its last word alone.
template <class S, class M>
CB200_XHD void absorb(typename S::W (&H)[8], uint32_t done, int len, const M& msg) {
  using W = typename S::W;
  constexpr int B = S::kBlock, WB = S::kWordBytes;
  const int nblocks = (len + 1 + 2 * WB + B - 1) / B;
#pragma unroll
  for (int blk = 0; blk < nblocks; blk++) {
    W m[16];
#pragma unroll
    for (int w = 0; w < 16; w++) {
      W v = 0;
#pragma unroll
      for (int b = 0; b < WB; b++) {
        const int j = blk * B + w * WB + b;
        const uint8_t x = j < len ? msg(j) : (j == len ? 0x80 : 0);
        v |= (W)x << (8 * (WB - 1 - b));
      }
      m[w] = v;
    }
    if (blk + 1 == nblocks) m[15] = (W)(((uint64_t)done + (uint64_t)len) << 3);
    S::compress(H, m);
  }
}

// HMAC(key, msg) from the two pad states of the key
template <class S, class M>
CB200_XHD void hmac(typename S::W (&out)[8], const typename S::W (&ki)[8], const typename S::W (&ko)[8], int len, const M& msg) {
  using W = typename S::W;
  constexpr int WB = S::kWordBytes, DW = S::kDigest / WB;
  W h[8];
#pragma unroll
  for (int i = 0; i < 8; i++) h[i] = ki[i];
  absorb<S>(h, S::kBlock, len, msg);
  // outer hash: one block holding the inner digest (DW words), the padding and the length of block + digest
  W m[16];
#pragma unroll
  for (int i = 0; i < DW; i++) m[i] = h[i];
  m[DW] = (W)0x80 << (8 * (WB - 1));
#pragma unroll
  for (int i = DW + 1; i < 15; i++) m[i] = 0;
  m[15] = (W)((uint64_t)(S::kBlock + S::kDigest) << 3);
#pragma unroll
  for (int i = 0; i < 8; i++) out[i] = ko[i];
  S::compress(out, m);
}

// the pad states of a one-digest key (a PRK): (key || 0...) ^ 0x36... and ^ 0x5c..., each compressed from the IV
template <class S>
CB200_XHD void hmac_key(typename S::W (&ki)[8], typename S::W (&ko)[8], const typename S::W (&key)[8]) {
  using W = typename S::W;
  constexpr int DW = S::kDigest / S::kWordBytes;
  const W i36 = (W)0x3636363636363636ull, i5c = (W)0x5c5c5c5c5c5c5c5cull;
  W m[16];
#pragma unroll
  for (int i = 0; i < 16; i++) m[i] = (i < DW ? key[i] : 0) ^ i36;
  S::iv(ki);
  S::compress(ki, m);
#pragma unroll
  for (int i = 0; i < 16; i++) m[i] = (i < DW ? key[i] : 0) ^ i5c;
  S::iv(ko);
  S::compress(ko, m);
}

// byte j of a digest
template <class S>
CB200_XHD uint8_t digest_byte(const typename S::W (&h)[8], int j) {
  constexpr int WB = S::kWordBytes;
  return (uint8_t)(h[j / WB] >> (8 * (WB - 1 - j % WB)));
}

// ---------------------------------------------------------------- HPKE's labeled messages (RFC 9180 section 4)
// LabeledExtract:  "HPKE-v1" || suite_id || label || ikm
// LabeledExpand:   I2OSP(L, 2) || "HPKE-v1" || suite_id || label || info || 0x01 (the first HKDF-Expand block; the
//                  only one where L is at most one digest, else ExpandNext gives the second)
// suite_id = "KEM" || I2OSP(kem_id, 2).  ikm / info are up to three rows of r0n, r1n, r2n bytes.
struct Labeled {
  int expand;         // 1: LabeledExpand's message, 0: LabeledExtract's
  int outlen;         // L of LabeledExpand
  int kem_id;
  const char* label;  // a string literal
  int lablen;
  const uint8_t *r0, *r1, *r2;
  int r0n, r1n, r2n;
  CB200_XHD int len() const { return (expand ? 3 : 0) + 12 + lablen + r0n + r1n + r2n; }
  CB200_XHD uint8_t operator()(int j) const {
    if (expand) {
      if (j == 0) return (uint8_t)(outlen >> 8);
      if (j == 1) return (uint8_t)outlen;
      j -= 2;
    }
    if (j < 7) return (uint8_t)"HPKE-v1"[j];
    if (j < 10) return (uint8_t)"KEM"[j - 7];
    if (j == 10) return (uint8_t)(kem_id >> 8);
    if (j == 11) return (uint8_t)kem_id;
    j -= 12;
    if (j < lablen) return (uint8_t)label[j];
    j -= lablen;
    if (j < r0n) return r0[j];
    j -= r0n;
    if (j < r1n) return r1[j];
    j -= r1n;
    if (j < r2n) return r2[j];
    return 1;  // the HKDF-Expand counter
  }
};

// HKDF-Expand's second block message T(1) || m' || 0x02, where m = m' || 0x01 is the first block's message: T(1) (one
// digest, in registers) and m (a functor like Labeled) as given.
template <class S, class M>
struct ExpandNext {
  const typename S::W (&t1)[8];
  const M& m;
  CB200_XHD int len() const { return S::kDigest + m.len(); }
  CB200_XHD uint8_t operator()(int j) const {
    if (j < S::kDigest) return digest_byte<S>(t1, j);
    j -= S::kDigest;
    return j == m.len() - 1 ? 2 : m(j);
  }
};

// prk = LabeledExtract("", label, ikm): HMAC with the all-zero salt of one digest
template <class S>
CB200_XHD void labeled_extract(typename S::W (&prk)[8], const Labeled& m) {
  typename S::W ki[8], ko[8];
  S::ipad0(ki);
  S::opad0(ko);
  hmac<S>(prk, ki, ko, m.len(), m);
}
// out = LabeledExpand(prk, label, info, L) for L <= one digest (the first L bytes of out)
template <class S>
CB200_XHD void labeled_expand(typename S::W (&out)[8], const typename S::W (&prk)[8], const Labeled& m) {
  typename S::W ki[8], ko[8];
  hmac_key<S>(ki, ko, prk);
  hmac<S>(out, ki, ko, m.len(), m);
}

}  // namespace sha2
}  // namespace cb200
