// The HPKE DHKEMs of the C++ kem::Scheme (include/circl_b200.hpp), driven by tests/test_cpp_hpke.py.
// With CB200_SIZES_ONLY set: the registry, the sizes and the errors raised before any device work (no GPU needed).
// Otherwise, on the GPU: a random round trip per scheme (plain and authenticated), then one line of output per input
// line "base <kem_id> <ikmR> <ikmE>" or "auth <kem_id> <ikmR> <ikmS> <ikmE>" (hex):
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

static void sizes_only() {
  CHECK(kem::All().size() == 12);
  CHECK(kem::ByName("HPKE_KEM_X25519_HKDF_SHA256") == nullptr);
  CHECK(kem::hpke::All().size() == 2);
  const kem::Scheme* a = kem::hpke::ByName("hpke_kem_x25519_hkdf_sha256");
  const kem::Scheme* b = kem::hpke::ByName("HPKE_KEM_X448_HKDF_SHA512");
  CHECK(a == kem::hpke::All()[0] && b == kem::hpke::All()[1] && kem::hpke::ByName("X-Wing") == nullptr);
  CHECK(a->Name() == "HPKE_KEM_X25519_HKDF_SHA256" && b->Name() == "HPKE_KEM_X448_HKDF_SHA512");
  CHECK(a->PublicKeySize() == 32 && a->PrivateKeySize() == 32 && a->CiphertextSize() == 32 && a->SharedKeySize() == 32 &&
        a->SeedSize() == 32 && a->EncapsulationSeedSize() == 32);
  CHECK(b->PublicKeySize() == 56 && b->PrivateKeySize() == 56 && b->CiphertextSize() == 56 && b->SharedKeySize() == 64 &&
        b->SeedSize() == 56 && b->EncapsulationSeedSize() == 56);
  kem::PrivateKey sk = a->UnmarshalBinaryPrivateKey(Bytes(32));
  CHECK(throws<kem::ErrPubKeySize>([&] { a->Decapsulate(sk, Bytes(31)); }));
  CHECK(throws<kem::ErrPrivKeySize>([&] { b->UnmarshalBinaryPrivateKey(Bytes(32)); }));
  CHECK(throws<kem::ErrTypeMismatch>([&] { b->Decapsulate(sk, Bytes(56)); }));
  CHECK(throws<std::logic_error>([&] { a->DeriveKeyPair(Bytes(56)); }));
  // seed and encapsulation lengths are checked before the key's type, as the reference does; for HPKE a wrong seed is
  // DeriveKeyPair's panic and a wrong encapsulation kem.ErrPubKeySize
  kem::PublicKey pb = b->UnmarshalBinaryPublicKey(Bytes(56));
  kem::PrivateKey sb = b->UnmarshalBinaryPrivateKey(Bytes(56));
  CHECK(throws<std::logic_error>([&] { a->EncapsulateDeterministically(pb, Bytes(31)); }));
  CHECK(throws<std::logic_error>([&] { a->AuthEncapsulateDeterministically(pb, sb, Bytes(31)); }));
  CHECK(throws<kem::ErrPubKeySize>([&] { a->Decapsulate(sb, Bytes(31)); }));
  CHECK(throws<kem::ErrPubKeySize>([&] { a->AuthDecapsulate(sb, Bytes(31), pb); }));
  // the other schemes keep their order: seed size first in encapsulation, key type first in decapsulation
  const kem::Scheme* m768 = kem::ByName("ML-KEM-768");
  CHECK(throws<kem::ErrSeedSize>([&] { m768->EncapsulateDeterministically(pb, Bytes(31)); }));
  CHECK(throws<kem::ErrTypeMismatch>([&] { m768->Decapsulate(sb, Bytes(31)); }));
  const kem::Scheme* xw = kem::ByName("X-Wing");
  CHECK(throws<std::logic_error>(
      [&] { xw->AuthEncapsulate(xw->UnmarshalBinaryPublicKey(Bytes(1216)), xw->UnmarshalBinaryPrivateKey(Bytes(32))); }));
}

static void round_trips() {
  for (const kem::Scheme* s : kem::hpke::All()) {
    auto [pkR, skR] = s->GenerateKeyPair();
    auto [pkS, skS] = s->GenerateKeyPair();
    CHECK(skR.Public().Equal(pkR));
    auto [ct, ss] = s->Encapsulate(pkR);
    CHECK(ss.size() == s->SharedKeySize() && s->Decapsulate(skR, ct) == ss);
    auto [act, ass] = s->AuthEncapsulate(pkR, skS);
    CHECK(s->AuthDecapsulate(skR, act, pkS) == ass && ass != ss);
    // a low-order encapsulation: hpke.ErrInvalidKEMSharedSecret
    CHECK(throws<kem::ErrInvalidKEMSharedSecret>([&] { s->Decapsulate(skR, Bytes(s->CiphertextSize())); }));
  }
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
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream is(line);
    std::string mode, ikmR, ikmS, ikmE;
    int id;
    is >> mode >> std::hex >> id >> ikmR;
    if (mode == "auth") is >> ikmS;
    is >> ikmE;
    const kem::Scheme* s = kem::hpke::All()[id == CB200_HPKE_X25519_HKDF_SHA256 ? 0 : 1];
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
