// FrodoKEM-640-SHAKE building blocks (kem/frodo/frodo640shake): the parameters, 15-bit packing, the CDF sampler,
// message encoding and the masks of the constant-time compare.  Plain integer C++ like x448.cuh: it compiles for the
// device (frodo.cu) and for the host-only test of the CPU suite.  No branch or address depends on a secret value.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define CB200_FHD __host__ __device__ __forceinline__
#else
#define CB200_FHD inline
#endif

namespace cb200 {
namespace frodo {

// frodo.go:14-51
constexpr int kN = 640, kNbar = 8, kLogQ = 15;
constexpr uint16_t kQMask = (1u << kLogQ) - 1;
constexpr int kPk = 9616, kSk = 19888, kCt = 9720, kSs = 16, kSeed = 48, kEseed = 16;
constexpr int kBpBytes = kLogQ * kN * kNbar / 8;  // 9600: the packed B' part of a ciphertext (and B of a public key)
// private key: s (16) | pk (9616) | S^T as 5120 little-endian uint16 | H(pk) (16)   (frodo.go:334-354)
constexpr int kSkPk = 16, kSkS = 16 + kPk, kSkHpk = kSkS + 2 * kN * kNbar;
// A's rows are SHAKE128(uint16_le(i) || seedA) squeezed to 1280 bytes: 8 blocks of the 168-byte rate, 84 coefficients
// per block, the last block partly used (matrix_shake.go:7-27)
constexpr int kRate = 168, kRowBlocks = 8, kPerBlock = kRate / 2;

// 8 coefficients <-> 15 bytes, big-endian bit order within the group (util.go:15-85)
CB200_FHD void pack8(uint8_t* out, const uint16_t (&v)[8]) {
  uint16_t a[8];
  for (int k = 0; k < 8; k++) a[k] = v[k] & kQMask;
  out[0] = (uint8_t)(a[0] >> 7);
  out[1] = (uint8_t)(((a[0] & 0x7F) << 1) | (a[1] >> 14));
  out[2] = (uint8_t)(a[1] >> 6);
  out[3] = (uint8_t)(((a[1] & 0x3F) << 2) | (a[2] >> 13));
  out[4] = (uint8_t)(a[2] >> 5);
  out[5] = (uint8_t)(((a[2] & 0x1F) << 3) | (a[3] >> 12));
  out[6] = (uint8_t)(a[3] >> 4);
  out[7] = (uint8_t)(((a[3] & 0x0F) << 4) | (a[4] >> 11));
  out[8] = (uint8_t)(a[4] >> 3);
  out[9] = (uint8_t)(((a[4] & 0x07) << 5) | (a[5] >> 10));
  out[10] = (uint8_t)(a[5] >> 2);
  out[11] = (uint8_t)(((a[5] & 0x03) << 6) | (a[6] >> 9));
  out[12] = (uint8_t)(a[6] >> 1);
  out[13] = (uint8_t)(((a[6] & 0x01) << 7) | (a[7] >> 8));
  out[14] = (uint8_t)a[7];
}
CB200_FHD void unpack8(uint16_t (&v)[8], const uint8_t* in) {
  v[0] = (uint16_t)((in[0] << 7) | (in[1] >> 1));
  v[1] = (uint16_t)(((in[1] & 0x01) << 14) | (in[2] << 6) | (in[3] >> 2));
  v[2] = (uint16_t)(((in[3] & 0x03) << 13) | (in[4] << 5) | (in[5] >> 3));
  v[3] = (uint16_t)(((in[5] & 0x07) << 12) | (in[6] << 4) | (in[7] >> 4));
  v[4] = (uint16_t)(((in[7] & 0x0F) << 11) | (in[8] << 3) | (in[9] >> 5));
  v[5] = (uint16_t)(((in[9] & 0x1F) << 10) | (in[10] << 2) | (in[11] >> 6));
  v[6] = (uint16_t)(((in[11] & 0x3F) << 9) | (in[12] << 1) | (in[13] >> 7));
  v[7] = (uint16_t)(((in[13] & 0x7F) << 8) | in[14]);
}

// The CDF sampler (noise.go:3-26): 12 arithmetic comparisons against the table, no table index that depends on the
// sample, and the sign from bit 0.  The result is in [-12, 12] as a 16-bit two's complement value.
CB200_FHD uint16_t sample(uint16_t r) {
  const uint16_t sign = r & 1, u = r >> 1;
  uint16_t g = 0;
#define CB200_FRODO_CDF(t) g += (uint16_t)(((uint16_t)((t) - u)) >> 15);
  CB200_FRODO_CDF(4643) CB200_FRODO_CDF(13363) CB200_FRODO_CDF(20579) CB200_FRODO_CDF(25843) CB200_FRODO_CDF(29227)
  CB200_FRODO_CDF(31145) CB200_FRODO_CDF(32103) CB200_FRODO_CDF(32525) CB200_FRODO_CDF(32689) CB200_FRODO_CDF(32745)
  CB200_FRODO_CDF(32762) CB200_FRODO_CDF(32766)
#undef CB200_FRODO_CDF
  return (uint16_t)((((uint16_t)-sign) ^ g) + sign);
}

// message coefficient q of a 16-byte message, B = 2 bits per coefficient (util.go:87-100)
CB200_FHD uint16_t encode_coef(const uint8_t* msg, int q) {
  return (uint16_t)(((msg[q >> 2] >> (2 * (q & 3))) & 3) << (kLogQ - 2));
}
// the two message bits a coefficient decodes to (util.go:102-115)
CB200_FHD uint32_t decode_coef(uint16_t w) { return (uint32_t)((((w & kQMask) + (1u << (kLogQ - 3))) >> (kLogQ - 2)) & 3); }

// ctCompareU16's final step (util.go:145-159): 0 for v == 0, else 1; and that bit as an all-ones byte mask, which
// selects s over k' as subtle.ConstantTimeCopy does (frodo.go:321-323)
CB200_FHD uint32_t nonzero_bit(uint32_t v) { return (v | (0u - v)) >> 31; }
CB200_FHD uint8_t select_mask(uint32_t v) { return (uint8_t)(0u - nonzero_bit(v)); }

}  // namespace frodo
}  // namespace cb200
