// tests/cpp/test_sign_eddsa.cpp -- the Ed25519 and Ed25519-Dilithium2 entries of sign::Scheme in
// include/circl_b200.hpp, exercised as sign/schemes/schemes_test.go exercises the Go API.  Prints hex transcripts for
// fixed seeds; tests/test_cpp_eddsa.py compares them with OpenSSL and the oracle.
#include <cstdio>
#include <cstdlib>

#include "circl_b200.hpp"

using namespace circl;

static void hex(const char* tag, const Bytes& b) {
  printf("%s=", tag);
  for (uint8_t x : b) printf("%02x", x);
  printf("\n");
}
#define REQUIRE(c)                                                                   \
  do {                                                                               \
    if (!(c)) {                                                                      \
      fprintf(stderr, "REQUIRE failed: %s (%s:%d)\n", #c, __FILE__, __LINE__);       \
      return 1;                                                                      \
    }                                                                                \
  } while (0)

int main() {
  // sign/schemes/schemes.go:31-44 order for the schemes served here
  const std::vector<const char*> names = {"Ed25519", "Ed25519-Dilithium2", "ML-DSA-44", "ML-DSA-65",
                                          "ML-DSA-87", "Dilithium2", "Dilithium3", "Dilithium5"};
  REQUIRE(sign::All().size() == names.size());
  for (size_t i = 0; i < names.size(); i++) REQUIRE(sign::All()[i]->Name() == names[i]);
  REQUIRE(sign::ByName("ed25519") == sign::All()[0] && sign::ByName("ED25519-DILITHIUM2") == sign::All()[1]);
  REQUIRE(sign::ByName("Ed448") == nullptr);
  const sign::Scheme* e = sign::ByName("Ed25519");
  const sign::Scheme* c = sign::ByName("Ed25519-Dilithium2");
  REQUIRE(e->PublicKeySize() == 32 && e->PrivateKeySize() == 64 && e->SignatureSize() == 64 && e->SeedSize() == 32);
  REQUIRE(c->PublicKeySize() == 1344 && c->PrivateKeySize() == 2560 && c->SignatureSize() == 2484 && c->SeedSize() == 32);
  REQUIRE(!e->SupportsContext() && !c->SupportsContext());
  if (getenv("CB200_SIZES_ONLY")) {  // the CPU suite: sizes and registry need no device
    printf("ALL OK\n");
    return 0;
  }
  init(0);
  Bytes seed(32), msg = {'h', 'e', 'l', 'l', 'o'};
  for (size_t i = 0; i < 32; i++) seed[i] = (uint8_t)(5 * i + 2);
  sign::SignatureOpts opts{"ctx"};
  for (const sign::Scheme* s : {e, c}) {
    auto kp = s->DeriveKey(seed);
    REQUIRE(kp.first.MarshalBinary().size() == s->PublicKeySize());
    Bytes sig = s->Sign(kp.second, msg);
    REQUIRE(sig.size() == s->SignatureSize() && s->Verify(kp.first, msg, sig));
    Bytes bad = sig;
    bad[bad.size() - 40] ^= 1;  // the Ed25519 S of both layouts
    REQUIRE(!s->Verify(kp.first, msg, bad));
    REQUIRE(!s->Verify(kp.first, msg, Bytes(sig.begin(), sig.end() - 1)));
    bool threw = false;
    try { s->Sign(kp.second, msg, &opts); } catch (const sign::ErrContextNotSupported&) { threw = true; }
    REQUIRE(threw);
    threw = false;
    try { s->Verify(kp.first, msg, sig, &opts); } catch (const sign::ErrContextNotSupported&) { threw = true; }
    REQUIRE(threw);
    threw = false;
    try { s->UnmarshalBinaryPrivateKey(Bytes(10)); } catch (const sign::ErrPrivKeySize&) { threw = true; }
    REQUIRE(threw);
    // batch: 30 keys, growing messages, one tampered signature
    const size_t nb = 30;
    Bytes seeds(32 * nb), pks, sks, msgs, sigs, okv;
    for (size_t i = 0; i < seeds.size(); i++) seeds[i] = (uint8_t)(i * 11 + 7);
    s->DeriveKeyBatch(seeds, pks, sks);
    std::vector<uint64_t> off(nb + 1, 0);
    for (size_t i = 0; i < nb; i++) {
      for (size_t j = 0; j < 9 * i; j++) msgs.push_back((uint8_t)(i + 5 * j));
      off[i + 1] = msgs.size();
    }
    s->SignBatch(sks, msgs, off, "", sigs);
    sigs[4 * s->SignatureSize() + 3] ^= 1;
    s->VerifyBatch(pks, msgs, off, "", sigs, okv);
    for (size_t i = 0; i < nb; i++) REQUIRE((okv[i] != 0) == (i != 4));
    printf("scheme=%s\n", s->Name().c_str());
    hex("pk", kp.first.MarshalBinary());
    hex("sk", kp.second.MarshalBinary());
    hex("sig", sig);
  }
  {  // PrivateKey -> public key (ed25519.PrivateKey.Public: the second half of the key)
    auto kp = e->DeriveKey(seed);
    REQUIRE(e->Public(kp.second).Equal(kp.first));
  }
  printf("ALL OK\n");
  cb200_shutdown();
  return 0;
}
