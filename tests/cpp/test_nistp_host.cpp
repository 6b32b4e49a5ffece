// circl_b200/csrc/nistp.cuh with the P-384 and P-521 curve types compiled for the host (the CUDA qualifiers defined
// away).  argv[1] is 384 or 521.  Reads one command per line on stdin and prints one result line;
// tests/test_nistp_host.py compares the results with Python integers.  Values are big-endian hex of kBytes bytes.
//   add|sub|mul|sqr|inv a [b]   field operations on values below p, through the Montgomery form
//   scalar k                    1 iff 0 < k < n
//   point P                     1 iff P (1 + 2 kBytes bytes) is a valid public key
//   base k                      status and 0x04 || X || Y of [k]G from the fixed-base table
//   shared k P                  status and X of [k]P
//   candidate c mask0           DeriveKeyPair's range test: 1 iff 0 < (c with byte 0 & mask0) < n, and that value
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>
#define __device__
#define __forceinline__ inline
#define __noinline__
#include "../../circl_b200/csrc/p384.cuh"
#include "../../circl_b200/csrc/p521.cuh"
using namespace cb200::nistp;

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

template <class C>
static int run() {
  constexpr int kB = C::kBytes;
  std::vector<uint32_t> table(kTableWords<C>);
  build_base_table<C>(table.data());
  auto fe_in = [](const std::string& s) {
    Fe<C> f, m;
    words_from_be<C>(f.v, unhex(s).data());
    fe_to_mont(m, f);
    return m;
  };
  auto fe_out = [](const Fe<C>& m) {
    Fe<C> f;
    fe_from_mont(f, m);
    uint8_t b[kB];
    words_to_be<C>(b, f.v, 0xffffffffu);
    return hex(b, kB);
  };
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, a, b;
    in >> op >> a >> b;
    Fe<C> h;
    if (op == "add") fe_add(h, fe_in(a), fe_in(b)), std::cout << fe_out(h) << "\n";
    else if (op == "sub") fe_sub(h, fe_in(a), fe_in(b)), std::cout << fe_out(h) << "\n";
    else if (op == "mul") fe_mul(h, fe_in(a), fe_in(b)), std::cout << fe_out(h) << "\n";
    else if (op == "sqr") fe_sqr(h, fe_in(a)), std::cout << fe_out(h) << "\n";
    else if (op == "inv") fe_invert(h, fe_in(a)), std::cout << fe_out(h) << "\n";
    else if (op == "scalar") {
      uint32_t k[C::kW];
      words_from_be<C>(k, unhex(a).data());
      std::cout << (scalar_ok<C>(k) ? 1 : 0) << "\n";
    } else if (op == "point") {
      Aff<C> P;
      std::cout << (point_decode(P, unhex(a).data()) ? 1 : 0) << "\n";
    } else if (op == "base") {
      uint8_t out[1 + 2 * kB];
      const uint32_t st = keygen<C>(out, unhex(a).data(), table.data());
      std::cout << st << " " << hex(out, sizeof out) << "\n";
    } else if (op == "shared") {
      uint8_t out[kB];
      const uint32_t st = shared<C>(out, unhex(a).data(), unhex(b).data());
      std::cout << st << " " << hex(out, kB) << "\n";
    } else if (op == "candidate") {
      const std::vector<uint8_t> c = unhex(a);
      uint32_t k[C::kW];
      const uint32_t ok = candidate<C>(k, [&](int j) { return c[j]; }, (uint8_t)std::stoi(b, nullptr, 16));
      uint8_t out[kB];
      words_to_be<C>(out, k, 0xffffffffu);
      std::cout << (ok ? 1 : 0) << " " << hex(out, kB) << "\n";
    } else {
      std::cerr << "unknown op " << op << "\n";
      return 1;
    }
  }
  return 0;
}

int main(int argc, char** argv) {
  const int bits = argc > 1 ? std::atoi(argv[1]) : 0;
  if (bits == 384) return run<P384>();
  if (bits == 521) return run<P521>();
  std::cerr << "usage: test_nistp_host 384|521\n";
  return 2;
}
