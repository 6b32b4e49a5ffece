// FrodoKEM-640-SHAKE through the C++ kem::Scheme (include/circl_b200.hpp), driven by tests/test_cpp_frodo.py.
// With CB200_SIZES_ONLY set: the registry, the sizes and the errors raised before any device work (no GPU needed).
// Otherwise, on the GPU: one line of output per input line "<48-byte key seed> <16-byte encapsulation seed>" (hex):
//   pk=<first 32 bytes of pk> ss=<ss> dec=<ss from decapsulation>; a shared-key batch of two is checked in place
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
static std::string hex(const Bytes& b, size_t n) {
  std::string s;
  char t[3];
  for (size_t i = 0; i < n && i < b.size(); i++) {
    std::snprintf(t, sizeof t, "%02x", b[i]);
    s += t;
  }
  return s;
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

int main() {
  const kem::Scheme* s = kem::frodo::ByName("frodokem-640-shake");
  CHECK(s && s == kem::frodo::All()[0] && kem::frodo::All().size() == 1 && s->Name() == "FrodoKEM-640-SHAKE");
  CHECK(kem::All().size() == 12 && !kem::ByName("FrodoKEM-640-SHAKE") && !kem::hpke::ByName("FrodoKEM-640-SHAKE"));
  CHECK(s->PublicKeySize() == 9616 && s->PrivateKeySize() == 19888 && s->CiphertextSize() == 9720 &&
        s->SharedKeySize() == 16 && s->SeedSize() == 48 && s->EncapsulationSeedSize() == 16);
  const kem::Scheme* other = kem::ByName("ML-KEM-768");
  auto pk = s->UnmarshalBinaryPublicKey(Bytes(9616, 7));
  auto sk = s->UnmarshalBinaryPrivateKey(Bytes(19888, 9));
  CHECK(sk.Public().MarshalBinary() == Bytes(9616, 9));
  CHECK(throws<kem::ErrPubKeySize>([&] { s->UnmarshalBinaryPublicKey(Bytes(9615)); }));
  CHECK(throws<kem::ErrCiphertextSize>([&] { s->Decapsulate(other->UnmarshalBinaryPrivateKey(Bytes(2400)), Bytes(1)); }));
  CHECK(throws<kem::ErrTypeMismatch>([&] { s->Decapsulate(other->UnmarshalBinaryPrivateKey(Bytes(2400)), Bytes(9720)); }));
  CHECK(throws<kem::ErrSeedSize>([&] { s->EncapsulateDeterministically(pk, Bytes(32)); }));
  CHECK(throws<std::logic_error>([&] { s->DeriveKeyPair(Bytes(32)); }));
  if (!std::getenv("CB200_SIZES_ONLY")) {
    if (cb200_init(0)) {
      std::printf("init failed: %s\n", cb200_last_error());
      return 1;
    }
    std::string line;
    while (std::getline(std::cin, line)) {
      std::istringstream in(line);
      std::string ks, es;
      in >> ks >> es;
      auto kp = s->DeriveKeyPair(unhex(ks));
      auto enc = s->EncapsulateDeterministically(kp.first, unhex(es));
      Bytes dec = s->Decapsulate(kp.second, enc.first);
      Bytes cts, sss;
      Bytes seeds = unhex(es);
      seeds.insert(seeds.end(), seeds.begin(), seeds.end());
      s->EncapsulateBatch(kp.first.MarshalBinary(), seeds, cts, sss);  // one key shared by two operations
      CHECK(Bytes(sss.begin() + 16, sss.end()) == enc.second && Bytes(cts.begin(), cts.begin() + 9720) == enc.first);
      std::printf("pk=%s ss=%s dec=%s\n", hex(kp.first.MarshalBinary(), 32).c_str(), hex(enc.second, 16).c_str(),
                  hex(dec, 16).c_str());
    }
    cb200_shutdown();
  }
  if (fails) return 1;
  std::printf("ALL OK\n");
  return 0;
}
