// P-256 (secp256r1, p = 2^256 - 2^224 + 2^192 + 2^96 - 1): the curve type of nistp.cuh and the names the P-256 kernels
// and the host-only test use.  Eight words of 32 bits; p's words are all 0, 1 or 2^32 - 1.
#pragma once
#include "nistp.cuh"

namespace cb200 {
namespace nistp {

struct P256 {
  static constexpr int kW = 8, kBytes = 32, kDigits = 64, kFlipWord = 7, kFlipShift = 31;
  static constexpr bool kOutlineMul = false;
  // little-endian 32-bit words
  CB200_XHD static uint32_t p(int i) {
    const uint32_t w[kW] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 1u, 0xffffffffu};
    return w[i];
  }
  CB200_XHD static uint32_t n(int i) {
    const uint32_t w[kW] = {0xfc632551u, 0xf3b9cac2u, 0xa7179e84u, 0xbce6faadu, 0xffffffffu, 0xffffffffu, 0u, 0xffffffffu};
    return w[i];
  }
  CB200_XHD static uint32_t b(int i) {  // b R mod p
    const uint32_t w[kW] = {0x29c4bddfu, 0xd89cdf62u, 0x78843090u, 0xacf005cdu,
                            0xf7212ed6u, 0xe5a220abu, 0x04874834u, 0xdc30061du};
    return w[i];
  }
  CB200_XHD static uint32_t one(int i) {  // R mod p
    const uint32_t w[kW] = {1u, 0u, 0u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xfffffffeu, 0u};
    return w[i];
  }
  CB200_XHD static uint32_t r2(int i) {  // R^2 mod p
    const uint32_t w[kW] = {3u, 0u, 0xffffffffu, 0xfffffffbu, 0xfffffffeu, 0xffffffffu, 0xfffffffdu, 4u};
    return w[i];
  }
  CB200_XHD static uint32_t gx(int i) {
    const uint32_t w[kW] = {0xd898c296u, 0xf4a13945u, 0x2deb33a0u, 0x77037d81u,
                            0x63a440f2u, 0xf8bce6e5u, 0xe12c4247u, 0x6b17d1f2u};
    return w[i];
  }
  CB200_XHD static uint32_t gy(int i) {
    const uint32_t w[kW] = {0x37bf51f5u, 0xcbb64068u, 0x6b315eceu, 0x2bce3357u,
                            0x7c0f9e16u, 0x8ee7eb4au, 0xfe1a7f9bu, 0x4fe342e2u};
    return w[i];
  }
  // for oprf.cuh: R^2 mod n, and the SSWU map's Z = -10 and c2 = sqrt(-Z) (RFC 9380 F.2) times R mod p
  CB200_XHD static uint32_t rn2(int i) {
    const uint32_t w[kW] = {0xbe79eea2u, 0x83244c95u, 0x49bd6fa6u, 0x4699799cu,
                            0x2b6bec59u, 0x2845b239u, 0xf3d95620u, 0x66e12d94u};
    return w[i];
  }
  CB200_XHD static uint32_t sswu_z(int i) {
    const uint32_t w[kW] = {0xfffffff5u, 0xffffffffu, 0xffffffffu, 0x0000000au, 0u, 0u, 0x0000000bu, 0xfffffff5u};
    return w[i];
  }
  CB200_XHD static uint32_t sswu_c2(int i) {
    const uint32_t w[kW] = {0x98a195fdu, 0xa1fd38eeu, 0x423dcf70u, 0x78400ad7u,
                            0x9ea8dfeeu, 0x6913c88fu, 0x12a8f304u, 0x9051d26eu};
    return w[i];
  }
  // h = f^(p - 2).  p - 2 = 2^256 - 2^224 + 2^192 + 2^96 - 3: the words of p - 2 from the top are
  // ffffffff 00000001 00000000 00000000 00000000 ffffffff ffffffff fffffffd; x_k below is f^(2^k - 1).
  CB200_NISTP_NOINLINE void invert(Fe<P256>& h, const Fe<P256>& f) {
    Fe<P256> x2, x3, x6, x12, x15, x30, x32, t;
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
    fe_sqr_n(t, x32, 32);  // ffffffff 00000000
    fe_mul(t, t, f);       // ffffffff 00000001
    fe_sqr_n(t, t, 128);
    fe_mul(t, t, x32);  // ffffffff 00000001 00000000 00000000 00000000 ffffffff
    fe_sqr_n(t, t, 32);
    fe_mul(t, t, x32);  // ... ffffffff ffffffff
    fe_sqr_n(t, t, 30);
    fe_mul(t, t, x30);  // ... ffffffff fffffffc
    fe_sqr_n(t, t, 2);
    fe_mul(h, t, f);  // ... ffffffff fffffffd
  }
};

}  // namespace nistp

namespace p256 {
using C = nistp::P256;
constexpr int kW = C::kW;
constexpr int kTableWords = nistp::kTableWords<C>;  // 32 KiB
using Fe = nistp::Fe<C>;
using Pt = nistp::Pt<C>;
using Aff = nistp::Aff<C>;
using nistp::fe_add;
using nistp::fe_from_mont;
using nistp::fe_invert;
using nistp::fe_mul;
using nistp::fe_sqr;
using nistp::fe_sub;
using nistp::fe_to_mont;
using nistp::point_decode;
CB200_XHD void words_from_be(uint32_t (&w)[kW], const uint8_t* b) { nistp::words_from_be<C>(w, b); }
CB200_XHD void words_to_be(uint8_t* b, const uint32_t (&w)[kW], uint32_t mask) { nistp::words_to_be<C>(b, w, mask); }
CB200_XHD uint32_t scalar_ok(const uint32_t (&k)[kW]) { return nistp::scalar_ok<C>(k); }
CB200_XHD uint32_t keygen(uint8_t* out, const uint8_t* sk, const uint32_t* __restrict__ table) {
  return nistp::keygen<C>(out, sk, table);
}
CB200_XHD uint32_t shared(uint8_t* out, const uint8_t* sk, const uint8_t* pt) { return nistp::shared<C>(out, sk, pt); }
inline void build_base_table(uint32_t* table) { nistp::build_base_table<C>(table); }
}  // namespace p256

}  // namespace cb200
