// The C++ partiallyblindrsa mirror (include/circl_b200.hpp), driven by tests/test_cpp_pbrsa.py.  With CB200_SIZES_ONLY
// set: argv[1..4] are the hex fields N p q qinv of a good safe-prime key and argv[5..8] those of a key whose primes are
// not safe; the checks are the key and size errors that hold without a device.  Otherwise, after circl::init(), one
// command per stdin line (hex, "-" for empty):
//   sign N p q qinv rows meta...        -> "sig=.." or "err=<class> st=.." (rows back to back, one metadata per row)
//   verify N sigs msg meta msg meta...  -> "ok" or "err=<class> st=.." (sigs: one row per message)
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

#include "circl_b200.hpp"

using circl::Bytes;
namespace pb = circl::partiallyblindrsa;

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

static pb::PrivateKey key(const std::string& n, const std::string& p, const std::string& q, const std::string& qinv) {
  return pb::PrivateKey{{unhex(n), {0x01, 0x00, 0x01}}, unhex(p), unhex(q), {}, {}, unhex(qinv)};
}

static int sizes_only(char** f) {
  const pb::PrivateKey sk = key(f[0], f[1], f[2], f[3]);
  const pb::Signer s(sk);  // a good key constructs without a device
  CHECK(s.KLen() == (size_t)sk.pub.N.size());
  CHECK(throws<pb::ErrUnexpectedSize>([&] { s.BlindSign(Bytes(s.KLen() - 1), {}); }));
  CHECK(throws<pb::ErrUnexpectedSize>([&] { s.BlindSignBatch(Bytes(s.KLen()), {}); }));
  CHECK(throws<circl::Error>([&] { s.BlindSign(Bytes(s.KLen()), {}); }));  // no device: not initialised
  CHECK(throws<pb::ErrInvalidPrivateKey>([&] { pb::Signer x(key(f[4], f[5], f[6], f[7])); }));  // primes not safe
  pb::PrivateKey bad = sk;
  bad.P.back() ^= 2;  // p q != N
  CHECK(throws<pb::ErrInvalidPrivateKey>([&] { pb::Signer x(bad); }));
  bad = sk;
  bad.Qinv = bad.P;  // qinv >= p
  CHECK(throws<pb::ErrInvalidPrivateKey>([&] { pb::Signer x(bad); }));
  CHECK(throws<pb::ErrInvalidPublicKey>([&] { pb::Verifier x({Bytes(100, 0xff), {3}}); }));  // 800-bit N
  const pb::Verifier v(sk.pub);
  CHECK(throws<pb::ErrVerification>([&] { v.Verify(Bytes(3), Bytes(1), Bytes(v.KLen() + 1)); }));
  CHECK(throws<pb::ErrUnexpectedSize>([&] { v.VerifyBatch({Bytes(3)}, {}, Bytes(v.KLen())); }));
  std::cout << "ALL OK\n";
  return 0;
}

template <class F>
static std::string run(F f) {
  try {
    return f();
  } catch (const pb::ErrInvalidMessageLength& e) {
    return "err=length st=" + hex(e.status);
  } catch (const pb::ErrInternal& e) {
    return "err=internal st=" + hex(e.status);
  } catch (const pb::ErrVerification& e) {
    return "err=verification st=" + hex(e.status);
  }
}

int main(int argc, char** argv) {
  if (std::getenv("CB200_SIZES_ONLY")) return argc == 9 ? sizes_only(argv + 1) : 1;
  circl::init();
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, n;
    in >> op >> n;
    if (op == "sign") {
      std::string p, q, qinv, rows, m;
      in >> p >> q >> qinv >> rows;
      std::vector<Bytes> meta;
      while (in >> m) meta.push_back(unhex(m));
      const pb::Signer s = pb::NewSigner(key(n, p, q, qinv));
      std::cout << run([&] { return "sig=" + hex(s.BlindSignBatch(unhex(rows), meta)); }) << "\n";
    } else {
      std::string sig, m, md;
      in >> sig;
      std::vector<Bytes> msgs, meta;
      while (in >> m >> md) msgs.push_back(unhex(m)), meta.push_back(unhex(md));
      const pb::Verifier v = pb::NewVerifier({unhex(n), {0x01, 0x00, 0x01}});
      std::cout << run([&] { v.VerifyBatch(msgs, meta, unhex(sig)); return std::string("ok"); }) << "\n";
    }
  }
  std::cout << "ALL OK\n";
  return 0;
}
