// DHKEM(P-384, HKDF-SHA384) and DHKEM(P-521, HKDF-SHA512) of the C++ kem::Scheme (include/circl_b200.hpp), driven by
// tests/test_cpp_nistp.py; argv[1] is 384 or 521.  With CB200_SIZES_ONLY set: the kem::p384 / kem::p521 registries,
// the sizes, the registries that must not change and the errors raised before any device work (no GPU needed).
// Otherwise, on the GPU: a random round trip (plain and authenticated), invalid keys, then one line of output per input
// line "base <ikmR> <ikmE>" or "auth <ikmR> <ikmS> <ikmE>" (hex):
//   pk=<pkR> enc=<enc> ss=<ss> dec=<ss from decapsulation>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

#include "circl_b200.hpp"

using circl::Bytes;
namespace kem = circl::kem;

static int fails = 0;
#define CHECK(c)                                              \
  do {                                                        \
    if (!(c)) {                                               \
      std::printf("FAIL line %d: %s\n", __LINE__, #c);        \
      fails++;                                                \
    }                                                         \
  } while (0)

static Bytes unhex(const std::string& s) {
  Bytes out(s.size() / 2);
  for (size_t i = 0; i < out.size(); i++) out[i] = (uint8_t)std::stoul(s.substr(2 * i, 2), nullptr, 16);
  return out;
}
static std::string hex(const Bytes& b) {
  std::string out;
  char buf[3];
  for (uint8_t v : b) {
    std::snprintf(buf, sizeof buf, "%02x", v);
    out += buf;
  }
  return out;
}
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

struct Curve {
  const char* name;
  const std::vector<const kem::Scheme*>& (*all)();
  const kem::Scheme* (*by_name)(const std::string&);
  size_t sk, pk, ss;
  const char* n;  // the group order, big-endian hex
};
static const Curve kP384 = {"HPKE_KEM_P384_HKDF_SHA384", kem::p384::All, kem::p384::ByName, 48, 97, 48,
                            "ffffffffffffffffffffffffffffffffffffffffffffffffc7634d81f4372ddf581a0db248b0a77aecec196accc52973"};
static const Curve kP521 = {"HPKE_KEM_P521_HKDF_SHA512", kem::p521::All, kem::p521::ByName, 66, 133, 64,
                            "01fffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffa51868783bf2f966b7fcc0148f709a5d"
                            "03bb5c9b8899c47aebb6fb71e91386409"};

static void sizes_only(const Curve& c) {
  CHECK(kem::All().size() == 12 && kem::hpke::All().size() == 2 && kem::p256::All().size() == 1);
  CHECK(kem::ByName(c.name) == nullptr && kem::hpke::ByName(c.name) == nullptr && kem::p256::ByName(c.name) == nullptr);
  CHECK(c.all().size() == 1);
  const kem::Scheme* s = c.by_name(kem::lower(c.name));
  CHECK(s == c.all()[0] && s->Name() == c.name && c.by_name("HPKE_KEM_P256_HKDF_SHA256") == nullptr);
  CHECK(s->nist() != nullptr && !s->p256());
  CHECK(s->PublicKeySize() == c.pk && s->PrivateKeySize() == c.sk && s->CiphertextSize() == c.pk &&
        s->SharedKeySize() == c.ss && s->SeedSize() == c.sk && s->EncapsulationSeedSize() == c.sk);
  CHECK(throws<kem::ErrInvalidKEMPrivateKey>([&] { s->UnmarshalBinaryPrivateKey(Bytes(c.sk)); }));
  CHECK(throws<kem::ErrInvalidKEMPrivateKey>([&] { s->UnmarshalBinaryPrivateKey(unhex(c.n)); }));
  Bytes top(c.sk, 0xff);  // above n (for P-521: a leading byte above 0x01)
  CHECK(throws<kem::ErrInvalidKEMPrivateKey>([&] { s->UnmarshalBinaryPrivateKey(top); }));
  CHECK(throws<kem::ErrPrivKeySize>([&] { s->UnmarshalBinaryPrivateKey(Bytes(c.pk)); }));
  Bytes nm1 = unhex(c.n);
  nm1.back() -= 1;
  CHECK(s->UnmarshalBinaryPrivateKey(nm1).MarshalBinary() == nm1);
  Bytes one(c.sk);
  one.back() = 1;
  kem::PrivateKey sk = s->UnmarshalBinaryPrivateKey(one);
  CHECK(throws<kem::ErrPubKeySize>([&] { s->Decapsulate(sk, Bytes(32)); }));
  CHECK(throws<std::logic_error>([&] { s->DeriveKeyPair(Bytes(c.pk)); }));
  const kem::Scheme* x = kem::hpke::All()[0];
  CHECK(throws<kem::ErrTypeMismatch>([&] { s->Decapsulate(x->UnmarshalBinaryPrivateKey(Bytes(32)), Bytes(c.pk)); }));
}

static void round_trips(const Curve& c) {
  const kem::Scheme* s = c.all()[0];
  auto [pkR, skR] = s->GenerateKeyPair();
  auto [pkS, skS] = s->GenerateKeyPair();
  CHECK(skR.Public().Equal(pkR) && pkR.MarshalBinary()[0] == 4 && pkR.MarshalBinary().size() == c.pk);
  auto [ct, ss] = s->Encapsulate(pkR);
  CHECK(ss.size() == c.ss && s->Decapsulate(skR, ct) == ss);
  auto [act, ass] = s->AuthEncapsulate(pkR, skS);
  CHECK(s->AuthDecapsulate(skR, act, pkS) == ass && ass != ss);
  CHECK(throws<kem::ErrInvalidKEMPublicKey>([&] { s->Decapsulate(skR, Bytes(c.pk)); }));
}

int main(int argc, char** argv) {
  const int bits = argc > 1 ? std::atoi(argv[1]) : 0;
  if (bits != 384 && bits != 521) {
    std::printf("usage: test_kem_nistp 384|521\n");
    return 2;
  }
  const Curve& c = bits == 384 ? kP384 : kP521;
  if (std::getenv("CB200_SIZES_ONLY")) {
    sizes_only(c);
    std::printf(fails ? "FAILED\n" : "ALL OK\n");
    return fails != 0;
  }
  circl::init(0);
  sizes_only(c);
  round_trips(c);
  const kem::Scheme* s = c.all()[0];
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream is(line);
    std::string mode, ikmR, ikmS, ikmE;
    is >> mode >> ikmR;
    if (mode == "auth") is >> ikmS;
    is >> ikmE;
    auto [pkR, skR] = s->DeriveKeyPair(unhex(ikmR));
    Bytes enc, ss, dec;
    if (mode == "auth") {
      auto [pkS, skS] = s->DeriveKeyPair(unhex(ikmS));
      std::tie(enc, ss) = s->AuthEncapsulateDeterministically(pkR, skS, unhex(ikmE));
      dec = s->AuthDecapsulate(skR, enc, pkS);
    } else {
      std::tie(enc, ss) = s->EncapsulateDeterministically(pkR, unhex(ikmE));
      dec = s->Decapsulate(skR, enc);
    }
    std::cout << "pk=" << hex(pkR.MarshalBinary()) << " enc=" << hex(enc) << " ss=" << hex(ss) << " dec=" << hex(dec) << "\n";
  }
  std::printf(fails ? "FAILED\n" : "ALL OK\n");
  return fails != 0;
}
