// circl_b200/csrc/frodo.cuh compiled for the host: a line-oriented driver for tests/test_frodo_host.py.
// Each input line produces one output line:
//   sample                 the sampler on every 16-bit input, 65536 hex values of 4 digits, concatenated
//   pack <hex of 8 x u16le>        the 15 packed bytes
//   unpack <hex of 15 bytes>       the 8 coefficients as u16le
//   encode <hex of 16 bytes>       the 64 message coefficients as u16le
//   decode <hex of 64 x u16le>     the 16 message bytes
//   mask <u32 decimal>             nonzero_bit and select_mask of the value, as "<bit> <mask>"
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../circl_b200/csrc/frodo.cuh"

using namespace cb200::frodo;

static std::vector<uint8_t> unhex(const std::string& s) {
  std::vector<uint8_t> out(s.size() / 2);
  for (size_t i = 0; i < out.size(); i++) out[i] = (uint8_t)std::stoul(s.substr(2 * i, 2), nullptr, 16);
  return out;
}
static void hex(const uint8_t* p, size_t n) {
  for (size_t i = 0; i < n; i++) printf("%02x", p[i]);
  printf("\n");
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, a;
    in >> op >> a;
    std::vector<uint8_t> b = unhex(a);
    if (op == "sample") {
      for (uint32_t r = 0; r < 65536; r++) printf("%04x", sample((uint16_t)r));
      printf("\n");
    } else if (op == "pack") {
      uint16_t v[8];
      for (int k = 0; k < 8; k++) v[k] = (uint16_t)(b[2 * k] | (b[2 * k + 1] << 8));
      uint8_t o[15];
      pack8(o, v);
      hex(o, 15);
    } else if (op == "unpack") {
      uint16_t v[8];
      unpack8(v, b.data());
      hex(reinterpret_cast<uint8_t*>(v), 16);
    } else if (op == "encode") {
      uint16_t v[64];
      for (int q = 0; q < 64; q++) v[q] = encode_coef(b.data(), q);
      hex(reinterpret_cast<uint8_t*>(v), 128);
    } else if (op == "decode") {
      uint8_t m[16] = {0};
      for (int q = 0; q < 64; q++) m[q >> 2] |= (uint8_t)(decode_coef((uint16_t)(b[2 * q] | (b[2 * q + 1] << 8))) << (2 * (q & 3)));
      hex(m, 16);
    } else if (op == "mask") {
      const uint32_t v = (uint32_t)std::stoul(a);
      printf("%u %u\n", nonzero_bit(v), (unsigned)select_mask(v));
    }
  }
  return 0;
}
