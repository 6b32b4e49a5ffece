// DHKEM(P-256, HKDF-SHA256) of the C++ kem::Scheme (include/circl_b200.hpp), driven by tests/test_cpp_p256.py.
// With CB200_SIZES_ONLY set: the kem::p256 registry, the sizes, the registries that must not change and the errors
// raised before any device work (no GPU needed).  Otherwise, on the GPU: a random round trip (plain and authenticated),
// invalid keys, then one line of output per input line "base <ikmR> <ikmE>" or "auth <ikmR> <ikmS> <ikmE>" (hex):
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
static const char* kN = "ffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551";

static void sizes_only() {
  CHECK(kem::All().size() == 12 && kem::hpke::All().size() == 2);
  CHECK(kem::ByName("HPKE_KEM_P256_HKDF_SHA256") == nullptr && kem::hpke::ByName("HPKE_KEM_P256_HKDF_SHA256") == nullptr);
  CHECK(kem::p256::All().size() == 1);
  const kem::Scheme* s = kem::p256::ByName("hpke_kem_p256_hkdf_sha256");
  CHECK(s == kem::p256::All()[0] && s->Name() == "HPKE_KEM_P256_HKDF_SHA256" && kem::p256::ByName("X-Wing") == nullptr);
  CHECK(s->PublicKeySize() == 65 && s->PrivateKeySize() == 32 && s->CiphertextSize() == 65 && s->SharedKeySize() == 32 &&
        s->SeedSize() == 32 && s->EncapsulationSeedSize() == 32);
  CHECK(throws<kem::ErrInvalidKEMPrivateKey>([&] { s->UnmarshalBinaryPrivateKey(Bytes(32)); }));
  CHECK(throws<kem::ErrInvalidKEMPrivateKey>([&] { s->UnmarshalBinaryPrivateKey(unhex(kN)); }));
  CHECK(throws<kem::ErrPrivKeySize>([&] { s->UnmarshalBinaryPrivateKey(Bytes(65)); }));
  Bytes one(32);
  one[31] = 1;
  kem::PrivateKey sk = s->UnmarshalBinaryPrivateKey(one);
  CHECK(throws<kem::ErrPubKeySize>([&] { s->Decapsulate(sk, Bytes(32)); }));
  CHECK(throws<std::logic_error>([&] { s->DeriveKeyPair(Bytes(65)); }));
  const kem::Scheme* x = kem::hpke::All()[0];
  CHECK(throws<kem::ErrTypeMismatch>([&] { s->Decapsulate(x->UnmarshalBinaryPrivateKey(Bytes(32)), Bytes(65)); }));
}

static void round_trips() {
  const kem::Scheme* s = kem::p256::All()[0];
  auto [pkR, skR] = s->GenerateKeyPair();
  auto [pkS, skS] = s->GenerateKeyPair();
  CHECK(skR.Public().Equal(pkR) && pkR.MarshalBinary()[0] == 4);
  auto [ct, ss] = s->Encapsulate(pkR);
  CHECK(ss.size() == 32 && s->Decapsulate(skR, ct) == ss);
  auto [act, ass] = s->AuthEncapsulate(pkR, skS);
  CHECK(s->AuthDecapsulate(skR, act, pkS) == ass && ass != ss);
  // an encapsulation that is not a point: hpke.ErrInvalidKEMPublicKey
  CHECK(throws<kem::ErrInvalidKEMPublicKey>([&] { s->Decapsulate(skR, Bytes(65)); }));
}

int main() {
  if (std::getenv("CB200_SIZES_ONLY")) {
    sizes_only();
    std::printf(fails ? "FAILED\n" : "ALL OK\n");
    return fails != 0;
  }
  circl::init(0);
  sizes_only();
  round_trips();
  const kem::Scheme* s = kem::p256::All()[0];
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
