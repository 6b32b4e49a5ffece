// tests/cpp/test_sign_ed448.cpp -- the Ed448 and Ed448-Dilithium3 entries of sign::Scheme in include/circl_b200.hpp,
// served through their own registry sign::ed448::All() / ByName().  Prints hex transcripts for fixed seeds;
// tests/test_cpp_ed448.py compares them with OpenSSL and the oracle.
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
  REQUIRE(sign::ed448::All().size() == 2);
  REQUIRE(sign::ed448::All()[0]->Name() == "Ed448" && sign::ed448::All()[1]->Name() == "Ed448-Dilithium3");
  REQUIRE(sign::ed448::ByName("ED448") == sign::ed448::All()[0]);
  REQUIRE(sign::ed448::ByName("ed448-dilithium3") == sign::ed448::All()[1]);
  REQUIRE(sign::ed448::ByName("Ed25519") == nullptr);
  REQUIRE(sign::All().size() == 8 && sign::ByName("Ed448") == nullptr);  // the main registry is unchanged
  const sign::Scheme* e = sign::ed448::ByName("Ed448");
  const sign::Scheme* c = sign::ed448::ByName("Ed448-Dilithium3");
  REQUIRE(e->PublicKeySize() == 57 && e->PrivateKeySize() == 114 && e->SignatureSize() == 114 && e->SeedSize() == 57);
  REQUIRE(c->PublicKeySize() == 2009 && c->PrivateKeySize() == 4057 && c->SignatureSize() == 3407 && c->SeedSize() == 57);
  REQUIRE(e->SupportsContext() && !c->SupportsContext());
  if (getenv("CB200_SIZES_ONLY")) {  // the CPU suite: sizes and registry need no device
    printf("ALL OK\n");
    return 0;
  }
  init(0);
  Bytes seed(57), msg = {'h', 'e', 'l', 'l', 'o'};
  for (size_t i = 0; i < 57; i++) seed[i] = (uint8_t)(5 * i + 2);
  sign::SignatureOpts opts{"ctx"};
  for (const sign::Scheme* s : {e, c}) {
    auto kp = s->DeriveKey(seed);
    REQUIRE(kp.first.MarshalBinary().size() == s->PublicKeySize());
    Bytes sig = s->Sign(kp.second, msg);
    REQUIRE(sig.size() == s->SignatureSize() && s->Verify(kp.first, msg, sig));
    Bytes bad = sig;
    bad[bad.size() - 40] ^= 1;  // the Ed448 S of both layouts
    REQUIRE(!s->Verify(kp.first, msg, bad));
    REQUIRE(!s->Verify(kp.first, msg, Bytes(sig.begin(), sig.end() - 1)));
    if (s == e) {  // Ed448 takes a context; over 255 bytes signing throws and verifying is false
      Bytes csig = s->Sign(kp.second, msg, &opts);
      REQUIRE(s->Verify(kp.first, msg, csig, &opts) && !s->Verify(kp.first, msg, csig));
      hex("ctxsig", csig);
      sign::SignatureOpts longctx{std::string(256, 'x')};
      bool threw = false;
      try { s->Sign(kp.second, msg, &longctx); } catch (const sign::ErrContextTooLong&) { threw = true; }
      REQUIRE(threw);
      REQUIRE(!s->Verify(kp.first, msg, sig, &longctx));
      REQUIRE(s->Public(kp.second).Equal(kp.first));  // ed448.PrivateKey.Public: the second half of the key
    } else {
      bool threw = false;
      try { s->Sign(kp.second, msg, &opts); } catch (const sign::ErrContextNotSupported&) { threw = true; }
      REQUIRE(threw);
    }
    // batch: 30 keys, growing messages, one tampered signature
    const size_t nb = 30;
    Bytes seeds(57 * nb), pks, sks, msgs, sigs, okv;
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
  printf("ALL OK\n");
  cb200_shutdown();
  return 0;
}
