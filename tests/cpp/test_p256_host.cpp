// circl_b200/csrc/p256.cuh compiled for the host (the CUDA qualifiers defined away).  Reads one command per line on
// stdin and prints one result line; tests/test_p256_host.py compares the results with Python integers.
//   add|sub|mul|sqr|inv a [b]   field operations on values below p (hex), through the Montgomery form
//   scalar k                    1 iff 0 < k < n (k 32 bytes, hex)
//   point P                     1 iff P (65 bytes, hex) is a valid public key
//   base k                      status and 0x04 || X || Y of [k]G from the fixed-base table
//   shared k P                  status and X of [k]P
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>
#define __device__
#define __forceinline__ inline
#define __noinline__
#include "../../circl_b200/csrc/p256.cuh"
using namespace cb200::p256;

static std::vector<uint8_t> unhex(const std::string& s) {
  std::vector<uint8_t> b(s.size() / 2);
  for (size_t i = 0; i < b.size(); i++) b[i] = (uint8_t)std::stoi(s.substr(2 * i, 2), nullptr, 16);
  return b;
}
static std::string hex(const uint8_t* b, size_t n) {
  std::string s;
  char t[3];
  for (size_t i = 0; i < n; i++) snprintf(t, 3, "%02x", b[i]), s += t;
  return s;
}
static Fe fe_in(const std::string& s) {  // 32 bytes big-endian -> Montgomery form
  Fe f, m;
  words_from_be(f.v, unhex(s).data());
  fe_to_mont(m, f);
  return m;
}
static std::string fe_out(const Fe& m) {
  Fe f;
  fe_from_mont(f, m);
  uint8_t b[32];
  words_to_be(b, f.v, 0xffffffffu);
  return hex(b, 32);
}

int main() {
  std::vector<uint32_t> table(kTableWords);
  build_base_table(table.data());
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, a, b;
    in >> op >> a >> b;
    Fe h;
    if (op == "add") fe_add(h, fe_in(a), fe_in(b)), std::cout << fe_out(h) << "\n";
    else if (op == "sub") fe_sub(h, fe_in(a), fe_in(b)), std::cout << fe_out(h) << "\n";
    else if (op == "mul") fe_mul(h, fe_in(a), fe_in(b)), std::cout << fe_out(h) << "\n";
    else if (op == "sqr") fe_sqr(h, fe_in(a)), std::cout << fe_out(h) << "\n";
    else if (op == "inv") fe_invert(h, fe_in(a)), std::cout << fe_out(h) << "\n";
    else if (op == "scalar") {
      uint32_t k[kW];
      words_from_be(k, unhex(a).data());
      std::cout << (scalar_ok(k) ? 1 : 0) << "\n";
    } else if (op == "point") {
      Aff P;
      std::cout << (point_decode(P, unhex(a).data()) ? 1 : 0) << "\n";
    } else if (op == "base") {
      uint8_t out[65];
      const uint32_t st = keygen(out, unhex(a).data(), table.data());
      std::cout << st << " " << hex(out, 65) << "\n";
    } else if (op == "shared") {
      uint8_t out[32];
      const uint32_t st = shared(out, unhex(a).data(), unhex(b).data());
      std::cout << st << " " << hex(out, 32) << "\n";
    } else {
      std::cerr << "unknown op " << op << "\n";
      return 1;
    }
  }
  return 0;
}
