// P-521 (secp521r1, p = 2^521 - 1): the curve type of nistp.cuh.  Seventeen words of 32 bits (R = 2^544), 66-byte rows
// whose top word holds two bytes, 131 signed radix-16 digits (k' < 2^520 fills 130 nibbles, the top one up to 15, so
// the carry out of them is a digit of its own).  A scalar row whose leading byte is above 0x01 is >= n.
#pragma once
#include "nistp.cuh"

namespace cb200 {
namespace nistp {

struct P521 {
  static constexpr int kW = 17, kBytes = 66, kDigits = 131, kFlipWord = 16, kFlipShift = 8;
  static constexpr bool kOutlineMul = true;
  // little-endian 32-bit words
  CB200_XHD static uint32_t p(int i) { return i < 16 ? 0xffffffffu : 0x1ffu; }
  CB200_XHD static uint32_t n(int i) {
    const uint32_t w[kW] = {0x91386409u, 0xbb6fb71eu, 0x899c47aeu, 0x3bb5c9b8u, 0xf709a5d0u, 0x7fcc0148u,
                            0xbf2f966bu, 0x51868783u, 0xfffffffau, 0xffffffffu, 0xffffffffu, 0xffffffffu,
                            0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x1ffu};
    return w[i];
  }
  CB200_XHD static uint32_t b(int i) {  // b R mod p
    const uint32_t w[kW] = {0x8014654fu, 0xea35a81fu, 0x78f7a28fu, 0xc41e961au, 0x839ab9efu, 0x5e9dd8dfu,
                            0xbd8b2960u, 0xa8f63f49u, 0xf0ab0c9cu, 0xc8c77884u, 0xf9dc5a44u, 0x2dccd98au,
                            0x77516d39u, 0xd05b42a0u, 0x0fc94d10u, 0xb0c70e4du, 0x15cu};
    return w[i];
  }
  CB200_XHD static uint32_t one(int i) { return i == 0 ? 0x00800000u : 0u; }  // R mod p = 2^23
  CB200_XHD static uint32_t r2(int i) { return i == 1 ? 0x00004000u : 0u; }   // R^2 mod p = 2^46
  CB200_XHD static uint32_t gx(int i) {
    const uint32_t w[kW] = {0xc2e5bd66u, 0xf97e7e31u, 0x856a429bu, 0x3348b3c1u, 0xa2ffa8deu, 0xfe1dc127u,
                            0xefe75928u, 0xa14b5e77u, 0x6b4d3dbau, 0xf828af60u, 0x053fb521u, 0x9c648139u,
                            0x2395b442u, 0x9e3ecb66u, 0x0404e9cdu, 0x858e06b7u, 0xc6u};
    return w[i];
  }
  CB200_XHD static uint32_t gy(int i) {
    const uint32_t w[kW] = {0x9fd16650u, 0x88be9476u, 0xa272c240u, 0x353c7086u, 0x3fad0761u, 0xc550b901u,
                            0x5ef42640u, 0x97ee7299u, 0x273e662cu, 0x17afbd17u, 0x579b4468u, 0x98f54449u,
                            0x2c7d1bd9u, 0x5c8a5fb4u, 0x9a3bc004u, 0x39296a78u, 0x118u};
    return w[i];
  }
  // for oprf.cuh: R^2 mod n, and the SSWU map's Z = -4 and c2 = sqrt(-Z) = 2 (RFC 9380 F.2) times R mod p
  CB200_XHD static uint32_t rn2(int i) {
    const uint32_t w[kW] = {0x61c64ca7u, 0x1163115au, 0x4374a642u, 0x18354a56u, 0x0791d9dcu, 0x5d4dd6d3u,
                            0xd3402705u, 0x4fb35b72u, 0xb7756e3au, 0xcff3d142u, 0xa8e567bcu, 0x5bcc6d61u,
                            0x492d0d45u, 0x2d8e03d1u, 0x8c44383du, 0x5b5a3afeu, 0x19au};
    return w[i];
  }
  CB200_XHD static uint32_t sswu_z(int i) { return i == 0 ? 0xfdffffffu : i < 16 ? 0xffffffffu : 0x1ffu; }
  CB200_XHD static uint32_t sswu_c2(int i) { return i == 0 ? 0x01000000u : 0u; }
  // h = f^(p - 2).  p - 2 = 2^521 - 3: 519 ones, then 0, 1; x_k below is f^(2^k - 1).
  CB200_NISTP_NOINLINE void invert(Fe<P521>& h, const Fe<P521>& f) {
    Fe<P521> x2, x3, x4, x7, t;
    fe_sqr(t, f);
    fe_mul(x2, t, f);
    fe_sqr(t, x2);
    fe_mul(x3, t, f);
    fe_sqr(t, x3);
    fe_mul(x4, t, f);
    fe_sqr_n(t, x4, 3);
    fe_mul(x7, t, x3);
    fe_sqr_n(t, x4, 4);
    fe_mul(t, t, x4);  // x8
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int k = 8; k < 512; k *= 2) {  // x_2k = x_k^(2^k) x_k
      Fe<P521> s;
      fe_sqr_n(s, t, k);
      fe_mul(t, s, t);
    }
    fe_sqr_n(t, t, 7);
    fe_mul(t, t, x7);  // 519 ones
    fe_sqr_n(t, t, 2);
    fe_mul(h, t, f);  // ... 0, 1
  }
};

}  // namespace nistp
}  // namespace cb200
