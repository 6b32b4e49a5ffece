// The C++ oprf mirror (include/circl_b200.hpp), driven by tests/test_cpp_oprf.py.  With CB200_SIZES_ONLY set: suites,
// sizes and the errors that hold without a device.  Otherwise, after circl::init(), one command per stdin line:
//   vec suite mode seed keyInfo info r input blinded   -> "sk=.. pk=.. ev=.. proof=.. out=.. ok=0|1"
// (hex, "-" for empty; r "-" lets the server draw it, the proof is then printed as "rand").
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

#include "circl_b200.hpp"

using circl::Bytes;
namespace o = circl::oprf;

static Bytes unhex(const std::string& s) {
  Bytes b;
  if (s == "-") return b;
  for (size_t i = 0; i + 1 < s.size(); i += 2) b.push_back((uint8_t)std::stoul(s.substr(i, 2), nullptr, 16));
  return b;
}
static std::string hex(const Bytes& b) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (uint8_t v : b) s += d[v >> 4], s += d[v & 15];
  return b.empty() ? "-" : s;
}
#define CHECK(c)                                          \
  do {                                                    \
    if (!(c)) {                                           \
      std::cout << "FAIL line " << __LINE__ << ": " #c "\n"; \
      return 1;                                           \
    }                                                     \
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

static int sizes_only() {
  CHECK(o::GetSuite("P256-SHA256").Ne() == 33 && o::GetSuite("P256-SHA256").ProofSize() == 64);
  CHECK(o::GetSuite("P384-SHA384").Ns() == 48 && o::GetSuite("P384-SHA384").Nh() == 48);
  CHECK(o::GetSuite("P521-SHA512").Ne() == 67 && o::GetSuite("P521-SHA512").Nh() == 64);
  CHECK(throws<o::ErrInvalidSuite>([] { o::GetSuite("ristretto255-SHA512"); }));
  CHECK(throws<o::ErrInvalidSeed>([] { o::DeriveKey(o::SuiteP256, 0, Bytes(31)); }));
  CHECK(throws<o::ErrInvalidMode>([] { o::DeriveKey(o::SuiteP256, 3, Bytes(32)); }));
  CHECK(throws<o::ErrInvalidInfo>([] { o::DeriveKey(o::SuiteP384, 2, Bytes(32), Bytes(65536)); }));
  CHECK(throws<circl::Error>([] { o::DeriveKey(o::SuiteP521, 1, Bytes(32)); }));  // no device: not initialised
  std::cout << "ALL OK\n";
  return 0;
}

int main() {
  if (std::getenv("CB200_SIZES_ONLY")) return sizes_only();
  circl::init();
  std::string l;
  while (std::getline(std::cin, l)) {
    std::istringstream in(l);
    std::string op, suite, seed, ki, info, r, input, bl;
    int mode;
    in >> op >> suite >> mode >> seed >> ki >> info >> r >> input >> bl;
    const o::Suite s = o::GetSuite(suite);
    const o::PrivateKey key = o::DeriveKey(s, mode, unhex(seed), unhex(ki));
    const Bytes inf = unhex(info), inp = unhex(input), b = unhex(bl);
    Bytes ev(b.size()), proof(mode ? s.ProofSize() : 0), out;
    bool ok;
    if (r != "-" || mode == 0) {
      o::ServerBase srv(s, key, mode);
      Bytes rb = unhex(r);
      srv.EvaluateBatch(b.data(), b.size() / s.Ne(), mode ? rb.data() : nullptr, inf, ev.data(),
                        mode ? proof.data() : nullptr, 1);
    }
    if (mode == 0) {
      o::Server srv = o::NewServer(s, key);
      out = srv.FullEvaluate(inp);
      ok = srv.VerifyFinalize(inp, out) && !srv.VerifyFinalize(inp, Bytes(out.size()));
    } else if (mode == 1) {
      o::VerifiableServer srv = o::NewVerifiableServer(s, key);
      if (r == "-") ev = srv.Evaluate({b}).Elements[0], proof = {};
      out = srv.FullEvaluate(inp);
      ok = srv.VerifyFinalize(inp, out) && !srv.VerifyFinalize(inp, Bytes(out.size()));
    } else {
      o::PartialObliviousServer srv = o::NewPartialObliviousServer(s, key);
      if (r == "-") ev = srv.Evaluate({b}, inf).Elements[0], proof = {};
      out = srv.FullEvaluate(inp, inf);
      ok = srv.VerifyFinalize(inp, inf, out) && !srv.VerifyFinalize(inp, inf, Bytes(out.size()));
    }
    std::cout << "sk=" << hex(key.k) << " pk=" << hex(key.Public()) << " ev=" << hex(ev)
              << " proof=" << (r == "-" && mode ? std::string("rand") : hex(proof)) << " out=" << hex(out)
              << " ok=" << ok << "\n";
  }
  std::cout << "ALL OK\n";
  return 0;
}
