// P-384 (secp384r1, p = 2^384 - 2^128 - 2^96 + 2^32 - 1): the curve type of nistp.cuh.  Twelve words of 32 bits, 48-byte
// rows, 96 signed radix-16 digits (k' < 2^383 fills them with the top digit in [0, 8]).
#pragma once
#include "nistp.cuh"

namespace cb200 {
namespace nistp {

struct P384 {
  static constexpr int kW = 12, kBytes = 48, kDigits = 96, kFlipWord = 11, kFlipShift = 31;
  static constexpr bool kOutlineMul = true;
  // little-endian 32-bit words
  CB200_XHD static uint32_t p(int i) {
    const uint32_t w[kW] = {0xffffffffu, 0u, 0u, 0xffffffffu, 0xfffffffeu, 0xffffffffu,
                            0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
    return w[i];
  }
  CB200_XHD static uint32_t n(int i) {
    const uint32_t w[kW] = {0xccc52973u, 0xecec196au, 0x48b0a77au, 0x581a0db2u, 0xf4372ddfu, 0xc7634d81u,
                            0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
    return w[i];
  }
  CB200_XHD static uint32_t b(int i) {  // b R mod p
    const uint32_t w[kW] = {0x9d412dccu, 0x08118871u, 0x7a4c32ecu, 0xf729add8u, 0x1920022eu, 0x77f2209bu,
                            0x94938ae2u, 0xe3374beeu, 0x1f022094u, 0xb62b21f4u, 0x604fbff9u, 0xcd08114bu};
    return w[i];
  }
  CB200_XHD static uint32_t one(int i) {  // R mod p
    const uint32_t w[kW] = {1u, 0xffffffffu, 0xffffffffu, 0u, 1u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    return w[i];
  }
  CB200_XHD static uint32_t r2(int i) {  // R^2 mod p
    const uint32_t w[kW] = {1u, 0xfffffffeu, 0u, 2u, 0u, 0xfffffffeu, 0u, 2u, 1u, 0u, 0u, 0u};
    return w[i];
  }
  CB200_XHD static uint32_t gx(int i) {
    const uint32_t w[kW] = {0x72760ab7u, 0x3a545e38u, 0xbf55296cu, 0x5502f25du, 0x82542a38u, 0x59f741e0u,
                            0x8ba79b98u, 0x6e1d3b62u, 0xf320ad74u, 0x8eb1c71eu, 0xbe8b0537u, 0xaa87ca22u};
    return w[i];
  }
  CB200_XHD static uint32_t gy(int i) {
    const uint32_t w[kW] = {0x90ea0e5fu, 0x7a431d7cu, 0x1d7e819du, 0x0a60b1ceu, 0xb5f0b8c0u, 0xe9da3113u,
                            0x289a147cu, 0xf8f41dbdu, 0x9292dc29u, 0x5d9e98bfu, 0x96262c6fu, 0x3617de4au};
    return w[i];
  }
  // for oprf.cuh: R^2 mod n, and the SSWU map's Z = -12 and c2 = sqrt(-Z) (RFC 9380 F.2) times R mod p
  CB200_XHD static uint32_t rn2(int i) {
    const uint32_t w[kW] = {0x19b409a9u, 0x2d319b24u, 0xdf1aa419u, 0xff3d81e5u, 0xfcb82947u, 0xbc3e483au,
                            0x4aab1cc5u, 0xd40d4917u, 0x28266895u, 0x3fb05b7au, 0x2b39bf21u, 0x0c84ee01u};
    return w[i];
  }
  CB200_XHD static uint32_t sswu_z(int i) {
    const uint32_t w[kW] = {0xfffffff3u, 0x0000000cu, 0u, 0xfffffff3u, 0xfffffff2u, 0xffffffffu,
                            0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
    return w[i];
  }
  CB200_XHD static uint32_t sswu_c2(int i) {
    const uint32_t w[kW] = {0xc0a3f1f8u, 0x1cdf6f1cu, 0x4c08f647u, 0xfdf2313bu, 0xd4183d32u, 0x89cb6776u,
                            0x476b11b6u, 0xacb3a761u, 0xc093fceau, 0xe428a383u, 0x3ae40b98u, 0xd78fa36bu};
    return w[i];
  }
  // h = f^(p - 2).  The bits of p - 2 from the top: 255 ones, a zero, 32 ones, 64 zeros, 30 ones, 0, 1 (words
  // ffffffff x 7, fffffffe, ffffffff, 00000000, 00000000, fffffffd); x_k below is f^(2^k - 1).
  CB200_NISTP_NOINLINE void invert(Fe<P384>& h, const Fe<P384>& f) {
    Fe<P384> x2, x3, x6, x12, x15, x30, x32, x60, x120, t;
    fe_sqr(t, f);
    fe_mul(x2, t, f);
    fe_sqr(t, x2);
    fe_mul(x3, t, f);
    fe_sqr_n(t, x3, 3);
    fe_mul(x6, t, x3);
    fe_sqr_n(t, x6, 6);
    fe_mul(x12, t, x6);
    fe_sqr_n(t, x12, 3);
    fe_mul(x15, t, x3);
    fe_sqr_n(t, x15, 15);
    fe_mul(x30, t, x15);
    fe_sqr_n(t, x30, 2);
    fe_mul(x32, t, x2);
    fe_sqr_n(t, x30, 30);
    fe_mul(x60, t, x30);
    fe_sqr_n(t, x60, 60);
    fe_mul(x120, t, x60);
    fe_sqr_n(t, x120, 120);
    fe_mul(t, t, x120);  // x240
    fe_sqr_n(t, t, 15);
    fe_mul(t, t, x15);  // 255 ones
    fe_sqr_n(t, t, 33);
    fe_mul(t, t, x32);  // ... 0, 32 ones
    fe_sqr_n(t, t, 94);
    fe_mul(t, t, x30);  // ... 64 zeros, 30 ones
    fe_sqr_n(t, t, 2);
    fe_mul(h, t, f);  // ... 0, 1
  }
};

}  // namespace nistp
}  // namespace cb200
