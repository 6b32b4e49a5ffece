// The C++ tssrsa mirror (include/circl_b200.hpp), driven by tests/test_cpp_tssrsa.py.  With CB200_SIZES_ONLY set:
// argv[1..2] are the hex N and e of a good key; the checks are the argument and size errors that hold without a device.
// Otherwise, after circl::init(), one command per stdin line (hex):
//   sign N players E rows                              -> "xi=.." (rows: digests back to back)
//   combine N e players threshold k j1,j2,.. xi msgs   -> "sig=.." or "err=<calc|internal> st=.." (idx: the same k
//                                                         indices for every op; xi: n rows of k kLen bytes)
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

#include "circl_b200.hpp"

using circl::Bytes;
namespace t = circl::tssrsa;

static Bytes unhex(const std::string& s) {
  Bytes r;
  for (size_t i = 0; i + 1 < s.size(); i += 2) r.push_back((uint8_t)std::stoul(s.substr(i, 2), nullptr, 16));
  return r;
}
static std::string hex(const Bytes& v) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (uint8_t x : v) s += d[x >> 4], s += d[x & 15];
  return s;
}
#define CHECK(c)                                             \
  do {                                                       \
    if (!(c)) {                                              \
      std::cout << "FAIL line " << __LINE__ << ": " #c "\n"; \
      return 1;                                              \
    }                                                        \
  } while (0)

template <class E, class F>
static bool throws(F f) {
  try {
    f();
  } catch (const E&) {
    return true;
  } catch (...) {
    return false;
  }
  return false;
}

static int sizes_only(const Bytes& N, const Bytes& e) {
  const t::PublicKey pub{N, e};
  const size_t kl = pub.Size();
  CHECK(kl >= 256);
  const Bytes row(kl, 1), two(2 * kl, 1);
  const std::vector<uint16_t> idx{1, 2};
  // sizes
  CHECK(throws<t::ErrUnexpectedSize>([&] { t::SignShareBatch(pub, 3, Bytes{5}, Bytes(kl + 1)); }));
  CHECK(throws<std::logic_error>([&] { t::SignShareBatch(t::PublicKey{}, 3, Bytes{5}, row); }));
  CHECK(throws<t::ErrUnexpectedSize>([&] { t::CombineSignSharesBatch(pub, 3, 2, 2, idx, Bytes(kl), row); }));
  CHECK(throws<t::ErrUnexpectedSize>([&] { t::CombineSignSharesBatch(pub, 3, 2, 2, {1}, two, row); }));
  // argument rules of the C ABI, before any device work
  CHECK(throws<std::logic_error>([&] { t::SignShareBatch(pub, 1, Bytes{5}, row); }));
  CHECK(throws<std::logic_error>([&] { t::SignShareBatch(pub, 65, Bytes{5}, row); }));
  Bytes big(kl + 40, 0xff);
  CHECK(throws<std::logic_error>([&] { t::SignShareBatch(pub, 3, big, row); }));
  CHECK(throws<std::logic_error>([&] { t::CombineSignSharesBatch(t::PublicKey{N, Bytes{1, 0}}, 3, 2, 2, idx, two, row); }));
  CHECK(throws<std::logic_error>([&] { t::CombineSignSharesBatch(pub, 3, 4, 2, idx, two, row); }));
  CHECK(throws<std::logic_error>([&] { t::CombineSignSharesBatch(pub, 3, 0, 2, idx, two, row); }));
  CHECK(throws<std::logic_error>([&] { t::CombineSignSharesBatch(pub, 5, 3, 2, idx, two, row); }));
  Bytes small(N.begin(), N.begin() + 64);
  CHECK(throws<std::logic_error>([&] { t::SignShareBatch(t::PublicKey{small, e}, 3, Bytes{5}, Bytes(64)); }));
  // good arguments without a device: the library's error, not an argument error
  CHECK(throws<circl::Error>([&] { t::SignShareBatch(pub, 3, Bytes{5}, row); }));
  CHECK(!throws<std::logic_error>([&] { t::SignShareBatch(pub, 3, Bytes{5}, row); }));
  CHECK(!throws<std::logic_error>([&] { t::CombineSignSharesBatch(pub, 3, 2, 2, idx, two, row); }));
  std::cout << "ALL OK\n";
  return 0;
}

int main(int argc, char** argv) {
  if (std::getenv("CB200_SIZES_ONLY")) return argc > 2 ? sizes_only(unhex(argv[1]), unhex(argv[2])) : 1;
  circl::init();
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string cmd;
    in >> cmd;
    if (cmd == "sign") {
      std::string n, e, rows;
      int players;
      in >> n >> players >> e >> rows;
      std::cout << "xi=" << hex(t::SignShareBatch(t::PublicKey{unhex(n), {}}, players, unhex(e), unhex(rows))) << "\n";
    } else if (cmd == "combine") {
      std::string n, e, js, xi, msgs;
      int players, threshold, k;
      in >> n >> e >> players >> threshold >> k >> js >> xi >> msgs;
      const t::PublicKey pub{unhex(n), unhex(e)};
      std::vector<uint16_t> one, idx;
      std::stringstream ss(js);
      std::string tok;
      while (std::getline(ss, tok, ',')) one.push_back((uint16_t)std::stoul(tok));
      const size_t ops = unhex(msgs).size() / pub.Size();
      for (size_t i = 0; i < ops; i++) idx.insert(idx.end(), one.begin(), one.end());
      try {
        const Bytes sig = t::CombineSignSharesBatch(pub, players, threshold, k, idx, unhex(xi), unhex(msgs));
        std::cout << "sig=" << hex(sig) << "\n";
      } catch (const t::ErrInvalidCalc& err) {
        std::cout << "err=calc st=" << hex(err.status) << "\n";
      } catch (const t::ErrInternal& err) {
        std::cout << "err=internal st=" << hex(err.status) << "\n";
      }
    } else {
      std::cout << "?\n";
    }
  }
  std::cout << "ALL OK\n";
  return 0;
}
