// The C++ blindrsa mirror (include/circl_b200.hpp), driven by tests/test_cpp_brsa.py.  With CB200_SIZES_ONLY set:
// argv[1..7] are the hex fields N e p q dp dq qinv of a good key; the checks are the key, variant and size errors that
// hold without a device.  Otherwise, after circl::init(), one command per stdin line (hex, "-" for empty):
//   sign N e p q dp dq qinv rows      -> "sig=.." or "err=<class> st=.." (rows: blinded messages back to back)
//   verify variant N e sig msg...     -> "ok" or "err=<class> st=.." (sig: one row per message)
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

#include "circl_b200.hpp"

using circl::Bytes;
namespace b = circl::blindrsa;

static Bytes unhex(const std::string& s) {
  Bytes r;
  if (s == "-") return r;
  for (size_t i = 0; i + 1 < s.size(); i += 2) r.push_back((uint8_t)std::stoul(s.substr(i, 2), nullptr, 16));
  return r;
}
static std::string hex(const Bytes& v) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (uint8_t x : v) s += d[x >> 4], s += d[x & 15];
  return v.empty() ? "-" : s;
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

static b::PrivateKey key(char** f) {
  return b::PrivateKey{{unhex(f[0]), unhex(f[1])}, unhex(f[2]), unhex(f[3]), unhex(f[4]), unhex(f[5]), unhex(f[6])};
}

static int sizes_only(char** f) {
  const b::PrivateKey sk = key(f);
  const b::Signer s(sk);  // a good key constructs without a device
  CHECK(s.KLen() == (size_t)sk.pub.N.size());
  CHECK(throws<b::ErrUnexpectedSize>([&] { s.BlindSign(Bytes(s.KLen() - 1)); }));
  CHECK(throws<circl::Error>([&] { s.BlindSign(Bytes(s.KLen())); }));  // no device: not initialised
  b::PrivateKey bad = sk;
  bad.P.back() ^= 2;  // p q != N
  CHECK(throws<b::ErrInvalidKey>([&] { b::Signer x(bad); }));
  bad = sk;
  bad.pub.E = {0x01, 0x00, 0x00};  // even e
  CHECK(throws<b::ErrInvalidKey>([&] { b::Signer x(bad); }));
  CHECK(throws<b::ErrInvalidKey>([&] { b::Verifier x(b::SHA384PSSRandomized, bad.pub); }));
  CHECK(throws<b::ErrInvalidVariant>([&] { b::Verifier x((b::Variant)4, sk.pub); }));
  const b::Verifier v(b::SHA384PSSZeroDeterministic, sk.pub);
  CHECK(throws<b::ErrVerification>([&] { v.Verify(Bytes(3), Bytes(v.KLen() + 1)); }));
  std::cout << "ALL OK\n";
  return 0;
}

template <class F>
static std::string run(F f) {
  try {
    return f();
  } catch (const b::ErrInvalidMessageLength& e) {
    return "err=length st=" + hex(e.status);
  } catch (const b::ErrInternal& e) {
    return "err=internal st=" + hex(e.status);
  } catch (const b::ErrVerification& e) {
    return "err=verification st=" + hex(e.status);
  }
}

int main(int argc, char** argv) {
  if (std::getenv("CB200_SIZES_ONLY")) return argc == 8 ? sizes_only(argv + 1) : 1;
  circl::init();
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op;
    in >> op;
    if (op == "sign") {
      std::string f[7], rows;
      for (auto& x : f) in >> x;
      in >> rows;
      char* p[7];
      for (int i = 0; i < 7; i++) p[i] = &f[i][0];
      const b::Signer s = b::NewSigner(key(p));
      std::cout << run([&] { return "sig=" + hex(s.BlindSignBatch(unhex(rows))); }) << "\n";
    } else {
      int variant;
      std::string n, e, sig, m;
      in >> variant >> n >> e >> sig;
      std::vector<Bytes> msgs;
      while (in >> m) msgs.push_back(unhex(m));
      const b::Verifier v = b::NewVerifier((b::Variant)variant, {unhex(n), unhex(e)});
      std::cout << run([&] { v.VerifyBatch(msgs, unhex(sig)); return std::string("ok"); }) << "\n";
    }
  }
  std::cout << "ALL OK\n";
  return 0;
}
