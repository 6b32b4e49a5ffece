// include/circl_b200.hpp -- C++ host-side mirror of CIRCL's kem.Scheme / sign.Scheme over the C ABI.
//
// CIRCL is Go and this build image has no Go toolchain, so besides the cgo shim delivered as source
// (go/), this header is the *compiled* host side above libcirclb200.so: same method names, argument
// meaning and error behaviour as
//   kem/kem.go:14-121            kem.Scheme, kem.PublicKey/PrivateKey, kem.Err*
//   kem/mlkem/mlkem768/kyber.go:267-407   (scheme boilerplate; mlkem512/1024 identical)
//   sign/sign.go:14-119          sign.Scheme, sign.SignatureOpts, sign.Err*
//   sign/mldsa/mldsa65/dilithium.go:256-366
//   kem/schemes/schemes.go:57-72, sign/schemes/schemes.go:56-71   (ByName, case-insensitive)
// Go's (value, error) returns become exceptions; Go panics (programmer errors) become std::logic_error.
// Batch methods are added beside the single-op ones (SURVEY.md 8(b)).  Header-only; link with -lcirclb200.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <cerrno>
#include <string>
#include <utility>
#include <vector>

#include <sys/random.h>

#include "circl_b200.h"

namespace circl {

using Bytes = std::vector<uint8_t>;

struct Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};
inline void init(int device = 0) {
  if (cb200_init(device) != 0) throw Error(cb200_last_error());
}
// one process, GPUs 0..ndev-1 (0: all): host-pointer batches are sharded by index inside the library
inline void init_devices(int ndev = 0) {
  if (cb200_init_devices(ndev) != 0) throw Error(cb200_last_error());
}
// crypto/rand of the mirror: the kernel's CSPRNG (getrandom(2)), as Go's crypto/rand reads it on Linux
inline void fill_random(uint8_t* p, size_t n) {
  size_t got = 0;
  while (got < n) {
    const ssize_t r = getrandom(p + got, n - got, 0);
    if (r < 0) {
      if (errno == EINTR) continue;
      throw Error("getrandom failed");
    }
    got += (size_t)r;
  }
}

namespace kem {

struct ErrTypeMismatch : Error { ErrTypeMismatch() : Error("kem: type mismatch") {} };
struct ErrSeedSize : Error { ErrSeedSize() : Error("kem: invalid seed size") {} };
struct ErrPubKeySize : Error { ErrPubKeySize() : Error("kem: invalid public key size") {} };
struct ErrCiphertextSize : Error { ErrCiphertextSize() : Error("kem: invalid ciphertext size") {} };
struct ErrPrivKeySize : Error { ErrPrivKeySize() : Error("kem: invalid private key size") {} };
struct ErrPubKey : Error { ErrPubKey() : Error("kem: invalid public key") {} };
struct ErrPrivKey : Error { ErrPrivKey() : Error("kem: invalid private key") {} };
// hpke.ErrInvalidKEMSharedSecret (hpke/hpke.go:280): a DH step of an HPKE DHKEM met a low-order point
struct ErrInvalidKEMSharedSecret : Error { ErrInvalidKEMSharedSecret() : Error("hpke: invalid KEM shared secret") {} };
// hpke.ErrInvalidKEMPublicKey / ErrInvalidKEMPrivateKey (hpke/hpke.go:278-279): DHKEM(P-256) keys that crypto/ecdh rejects
struct ErrInvalidKEMPublicKey : Error { ErrInvalidKEMPublicKey() : Error("hpke: invalid KEM public key") {} };
struct ErrInvalidKEMPrivateKey : Error { ErrInvalidKEMPrivateKey() : Error("hpke: invalid KEM private key") {} };

class Scheme;

class PublicKey {  // kem.PublicKey (kem/kem.go:14-20)
 public:
  PublicKey(const Scheme* s, Bytes b) : scheme_(s), packed_(std::move(b)) {}
  const Scheme* GetScheme() const { return scheme_; }
  const Bytes& MarshalBinary() const { return packed_; }
  bool Equal(const PublicKey& o) const { return scheme_ == o.scheme_ && packed_ == o.packed_; }

 private:
  const Scheme* scheme_;
  Bytes packed_;
};

class PrivateKey {  // kem.PrivateKey (kem/kem.go:22-30)
 public:
  PrivateKey(const Scheme* s, Bytes b) : scheme_(s), packed_(std::move(b)) {}
  const Scheme* GetScheme() const { return scheme_; }
  const Bytes& MarshalBinary() const { return packed_; }
  bool Equal(const PrivateKey& o) const { return scheme_ == o.scheme_ && packed_ == o.packed_; }
  PublicKey Public() const;

 private:
  const Scheme* scheme_;
  Bytes packed_;
};

// The entry points of one NIST DHKEM (cb200_hpke_p256_* / p384_* / p521_*), its raw ECDH (cb200_p256 / p384 / p521)
// and its group order n (big-endian, Nsk bytes); nullptr for any other id.
struct NistOps {
  size_t (*pk_size)(void), (*sk_size)(void), (*ss_size)(void);
  int (*keygen)(const uint8_t*, uint8_t*, uint8_t*, size_t);
  int (*encaps)(const uint8_t*, size_t, const uint8_t*, uint8_t*, uint8_t*, uint8_t*, size_t);
  int (*decaps)(const uint8_t*, size_t, const uint8_t*, uint8_t*, uint8_t*, size_t);
  int (*auth_encaps)(const uint8_t*, size_t, const uint8_t*, size_t, const uint8_t*, uint8_t*, uint8_t*, uint8_t*, size_t);
  int (*auth_decaps)(const uint8_t*, size_t, const uint8_t*, const uint8_t*, size_t, uint8_t*, uint8_t*, size_t);
  int (*ecdh)(const uint8_t*, const uint8_t*, uint8_t*, uint8_t*, size_t);
  const uint8_t* n;
};
inline const NistOps* nist_ops(int id) {
  static const uint8_t n256[32] = {0xff, 0xff, 0xff, 0xff, 0x00, 0x00, 0x00, 0x00, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                   0xff, 0xff, 0xbc, 0xe6, 0xfa, 0xad, 0xa7, 0x17, 0x9e, 0x84, 0xf3, 0xb9, 0xca, 0xc2,
                                   0xfc, 0x63, 0x25, 0x51};
  static const uint8_t n384[48] = {0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                   0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xc7, 0x63, 0x4d, 0x81,
                                   0xf4, 0x37, 0x2d, 0xdf, 0x58, 0x1a, 0x0d, 0xb2, 0x48, 0xb0, 0xa7, 0x7a, 0xec, 0xec,
                                   0x19, 0x6a, 0xcc, 0xc5, 0x29, 0x73};
  static const uint8_t n521[66] = {0x01, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                   0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                   0xff, 0xff, 0xff, 0xff, 0xff, 0xfa, 0x51, 0x86, 0x87, 0x83, 0xbf, 0x2f, 0x96, 0x6b,
                                   0x7f, 0xcc, 0x01, 0x48, 0xf7, 0x09, 0xa5, 0xd0, 0x3b, 0xb5, 0xc9, 0xb8, 0x89, 0x9c,
                                   0x47, 0xae, 0xbb, 0x6f, 0xb7, 0x1e, 0x91, 0x38, 0x64, 0x09};
#define CIRCL_NIST_OPS(c, n)                                                                                         \
  {cb200_hpke_##c##_public_key_size, cb200_hpke_##c##_private_key_size, cb200_hpke_##c##_shared_key_size,            \
   cb200_hpke_##c##_keygen, cb200_hpke_##c##_encaps, cb200_hpke_##c##_decaps, cb200_hpke_##c##_auth_encaps,          \
   cb200_hpke_##c##_auth_decaps, cb200_##c, n}
  static const NistOps p256 = CIRCL_NIST_OPS(p256, n256), p384 = CIRCL_NIST_OPS(p384, n384),
                       p521 = CIRCL_NIST_OPS(p521, n521);
#undef CIRCL_NIST_OPS
  switch (id) {
    case CB200_HPKE_P256_HKDF_SHA256: return &p256;
    case CB200_HPKE_P384_HKDF_SHA384: return &p384;
    case CB200_HPKE_P521_HKDF_SHA512: return &p521;
  }
  return nullptr;
}

// kem.Scheme (kem/kem.go:33-82).  One class serves the four families behind the C ABI:
//   MLKEM   ML-KEM-512/768/1024            kem/mlkem/mlkem768/kyber.go:267-407
//   KYBER3  round-3 Kyber512/768/1024      kem/kyber/kyber768/kyber.go:267-407
//   XWING   X-Wing                         kem/xwing/scheme.go:1-140
//   HYBRID  X25519MLKEM768, Kyber768-X25519, Kyber512-X25519,
//           Kyber768-X448, Kyber1024-X448                      kem/hybrid/hybrid.go:76-315
//   HPKE    HPKE_KEM_X25519_HKDF_SHA256, HPKE_KEM_X448_HKDF_SHA512   hpke/kembase.go, hpke/xkem.go, and the NIST
//           DHKEMs HPKE_KEM_P256/P384/P521_* (hpke/shortkem.go, their own entry points: nist()); these are also
//           kem.AuthScheme (kem/kem.go:84-90): the Auth* methods below serve them only
//   FRODO   FrodoKEM-640-SHAKE             kem/frodo/frodo640shake/frodo.go:405-547
class Scheme {
 public:
  enum Kind { MLKEM, KYBER3, XWING, HYBRID, HPKE, FRODO };
  Scheme(std::string name, int k, bool round3 = false) : name_(std::move(name)), kind_(round3 ? KYBER3 : MLKEM), k_(k) {}
  Scheme(std::string name, Kind kind, int id) : name_(std::move(name)), kind_(kind), k_(id) {}
  const std::string& Name() const { return name_; }
  size_t CiphertextSize() const {
    if (kind_ == HPKE) return nist() ? nist()->pk_size() : cb200_hpke_ciphertext_size(k_);
    if (kind_ == FRODO) return cb200_frodo640shake_ciphertext_size();
    return kind_ == XWING ? 1120 : kind_ == HYBRID ? cb200_hybrid_ciphertext_size(k_) : cb200_mlkem_ciphertext_size(k_);
  }
  size_t SharedKeySize() const {
    if (kind_ == HPKE) return nist() ? nist()->ss_size() : cb200_hpke_shared_key_size(k_);
    if (kind_ == FRODO) return cb200_frodo640shake_shared_key_size();
    return kind_ == HYBRID ? cb200_hybrid_shared_key_size(k_) : 32;
  }
  size_t PrivateKeySize() const {
    if (kind_ == HPKE) return nist() ? nist()->sk_size() : cb200_hpke_private_key_size(k_);
    if (kind_ == FRODO) return cb200_frodo640shake_private_key_size();
    return kind_ == XWING ? 32 : kind_ == HYBRID ? cb200_hybrid_private_key_size(k_) : cb200_mlkem_private_key_size(k_);
  }
  size_t PublicKeySize() const {
    if (kind_ == HPKE) return nist() ? nist()->pk_size() : cb200_hpke_public_key_size(k_);
    if (kind_ == FRODO) return cb200_frodo640shake_public_key_size();
    return kind_ == XWING ? 1216 : kind_ == HYBRID ? cb200_hybrid_public_key_size(k_) : cb200_mlkem_public_key_size(k_);
  }
  size_t SeedSize() const {
    if (kind_ == HPKE) return nist() ? nist()->sk_size() : cb200_hpke_seed_size(k_);
    if (kind_ == FRODO) return cb200_frodo640shake_seed_size();
    return kind_ == XWING ? 32 : kind_ == HYBRID ? cb200_hybrid_seed_size(k_) : 64;
  }
  size_t EncapsulationSeedSize() const {
    if (kind_ == HPKE) return nist() ? nist()->sk_size() : cb200_hpke_encapsulation_seed_size(k_);
    if (kind_ == FRODO) return cb200_frodo640shake_encapsulation_seed_size();
    return kind_ == XWING ? 64 : kind_ == HYBRID ? cb200_hybrid_encapsulation_seed_size(k_) : 32;
  }

  std::pair<PublicKey, PrivateKey> DeriveKeyPair(const Bytes& seed) const {  // kyber.go:337-346
    if (seed.size() != SeedSize()) throw std::logic_error("kem: invalid seed size");  // Go panics here
    Bytes ek, dk;
    DeriveKeyPairBatch(seed, ek, dk);
    return {PublicKey(this, std::move(ek)), PrivateKey(this, std::move(dk))};
  }
  std::pair<PublicKey, PrivateKey> GenerateKeyPair() const;  // kyber.go:281-283; a random sk for HPKE (xkem.go:73-80)
  std::pair<PublicKey, PrivateKey> GenerateFromSeed() const {
    Bytes seed(SeedSize());
    fill_random(seed.data(), seed.size());
    return DeriveKeyPair(seed);
  }
  PublicKey UnmarshalBinaryPublicKey(const Bytes& buf) const {  // kyber.go:390-396
    if (buf.size() != PublicKeySize()) throw ErrPubKeySize();
    return PublicKey(this, buf);
  }
  PrivateKey UnmarshalBinaryPrivateKey(const Bytes& buf) const {  // kyber.go:398-407
    if (buf.size() != PrivateKeySize()) throw ErrPrivKeySize();
    if (nist() && !nist_scalar_ok(buf)) throw ErrInvalidKEMPrivateKey();  // shortkem.go:103-113
    return PrivateKey(this, buf);
  }
  // (ct, ss)
  std::pair<Bytes, Bytes> EncapsulateDeterministically(const PublicKey& pk, const Bytes& seed) const {  // kyber.go:359-374
    if (seed.size() != EncapsulationSeedSize()) {
      if (kind_ == HPKE) throw std::logic_error("kem: invalid seed size");  // DeriveKeyPair panics (xkem.go:60-62)
      throw ErrSeedSize();
    }
    if (pk.GetScheme() != this) throw ErrTypeMismatch();
    Bytes ct, ss;
    EncapsulateBatch(pk.MarshalBinary(), seed, ct, ss);
    return {std::move(ct), std::move(ss)};
  }
  std::pair<Bytes, Bytes> Encapsulate(const PublicKey& pk) const {  // kyber.go:348-357
    Bytes seed(EncapsulationSeedSize());
    fill_random(seed.data(), seed.size());
    return EncapsulateDeterministically(pk, seed);
  }
  Bytes Decapsulate(const PrivateKey& sk, const Bytes& ct) const {  // kyber.go:376-388
    // HPKE parses ct as a public key before it looks at the key's type (kembase.go:222)
    if (kind_ == HPKE && ct.size() != CiphertextSize()) throw ErrPubKeySize();
    // FrodoKEM checks the ciphertext length before the key's type (frodo.go:517-525)
    if (kind_ == FRODO && ct.size() != CiphertextSize()) throw ErrCiphertextSize();
    if (sk.GetScheme() != this) throw ErrTypeMismatch();
    if (ct.size() != CiphertextSize()) throw ErrCiphertextSize();
    Bytes ss;
    DecapsulateBatch(sk.MarshalBinary(), ct, ss);
    return ss;
  }
  // ---- batch entry points (keys: one packed key = shared by the batch, or n keys back to back)
  void EncapsulateBatch(const Bytes& eks, const Bytes& seeds, Bytes& cts, Bytes& sss) const {
    const size_t es = EncapsulationSeedSize(), pks = PublicKeySize();
    if (seeds.size() % es) throw ErrSeedSize();
    const size_t n = seeds.size() / es;
    const bool shared = eks.size() == pks;
    if (!shared && eks.size() != n * pks) throw ErrPubKeySize();
    const size_t stride = shared ? 0 : pks;
    cts.resize(n * CiphertextSize());
    sss.resize(n * SharedKeySize());
    switch (kind_) {
      case MLKEM: check(cb200_mlkem_encaps(k_, eks.data(), stride, seeds.data(), cts.data(), sss.data(), nullptr, n)); break;
      case KYBER3: check(cb200_kyber_kem_encaps(k_, eks.data(), stride, seeds.data(), cts.data(), sss.data(), n)); break;
      case XWING: check(cb200_xwing_encaps(eks.data(), stride, seeds.data(), cts.data(), sss.data(), nullptr, n)); break;
      case HYBRID: check(cb200_hybrid_encaps(k_, eks.data(), stride, seeds.data(), cts.data(), sss.data(), nullptr, n)); break;
      case HPKE:
        check(nist() ? nist()->encaps(eks.data(), stride, seeds.data(), cts.data(), sss.data(), nullptr, n)
                     : cb200_hpke_encaps(k_, eks.data(), stride, seeds.data(), cts.data(), sss.data(), nullptr, n));
        break;
      case FRODO: check(cb200_frodo640shake_encaps(eks.data(), stride, seeds.data(), cts.data(), sss.data(), n)); break;
    }
  }
  void DecapsulateBatch(const Bytes& dks, const Bytes& cts, Bytes& sss) const {
    const size_t sks = PrivateKeySize();
    if (cts.size() % CiphertextSize()) throw ErrCiphertextSize();
    const size_t n = cts.size() / CiphertextSize();
    const bool shared = dks.size() == sks;
    if (!shared && dks.size() != n * sks) throw ErrPrivKeySize();
    const size_t stride = shared ? 0 : sks;
    sss.resize(n * SharedKeySize());
    switch (kind_) {
      case MLKEM: check(cb200_mlkem_decaps(k_, dks.data(), stride, cts.data(), sss.data(), nullptr, n)); break;
      case KYBER3: check(cb200_kyber_kem_decaps(k_, dks.data(), stride, cts.data(), sss.data(), n)); break;
      case XWING: check(cb200_xwing_decaps(dks.data(), stride, cts.data(), sss.data(), n)); break;
      case HYBRID: {
        if (!shared || n == 1) {
          check(cb200_hybrid_decaps(k_, dks.data(), sks, cts.data(), sss.data(), nullptr, n));
        } else {  // the hybrid decapsulation flow takes one key per operation
          Bytes rep(n * sks);
          for (size_t i = 0; i < n; i++) std::copy(dks.begin(), dks.end(), rep.begin() + i * sks);
          check(cb200_hybrid_decaps(k_, rep.data(), sks, cts.data(), sss.data(), nullptr, n));
        }
        break;
      }
      case HPKE:
        check(nist() ? nist()->decaps(dks.data(), stride, cts.data(), sss.data(), nullptr, n)
                     : cb200_hpke_decaps(k_, dks.data(), stride, cts.data(), sss.data(), nullptr, n));
        break;
      case FRODO: check(cb200_frodo640shake_decaps(dks.data(), stride, cts.data(), sss.data(), n)); break;
    }
  }
  void DeriveKeyPairBatch(const Bytes& seeds, Bytes& eks, Bytes& dks) const {
    if (seeds.size() % SeedSize()) throw ErrSeedSize();
    const size_t n = seeds.size() / SeedSize();
    eks.resize(n * PublicKeySize());
    dks.resize(n * PrivateKeySize());
    switch (kind_) {
      case MLKEM: check(cb200_mlkem_keygen(k_, seeds.data(), eks.data(), dks.data(), n)); break;
      case KYBER3: check(cb200_kyber_kem_keygen(k_, seeds.data(), eks.data(), dks.data(), n)); break;
      case XWING:  // the packed private key is the seed itself (xwing.go:68-73)
        check(cb200_xwing_keygen(seeds.data(), eks.data(), n));
        dks = seeds;
        break;
      case HYBRID: check(cb200_hybrid_keygen(k_, seeds.data(), eks.data(), dks.data(), n)); break;
      case HPKE:
        check(nist() ? nist()->keygen(seeds.data(), eks.data(), dks.data(), n)
                     : cb200_hpke_keygen(k_, seeds.data(), eks.data(), dks.data(), n));
        break;
      case FRODO: check(cb200_frodo640shake_keygen(seeds.data(), eks.data(), dks.data(), n)); break;
    }
  }
  // ---- kem.AuthScheme (HPKE only): (ct, ss) and ss
  std::pair<Bytes, Bytes> AuthEncapsulateDeterministically(const PublicKey& pkr, const PrivateKey& sks,
                                                           const Bytes& seed) const {  // kembase.go:108-112
    auth_only();
    if (seed.size() != EncapsulationSeedSize()) throw std::logic_error("kem: invalid seed size");
    if (pkr.GetScheme() != this || sks.GetScheme() != this) throw ErrTypeMismatch();
    Bytes ct, ss;
    AuthEncapsulateBatch(pkr.MarshalBinary(), sks.MarshalBinary(), seed, ct, ss);
    return {std::move(ct), std::move(ss)};
  }
  std::pair<Bytes, Bytes> AuthEncapsulate(const PublicKey& pkr, const PrivateKey& sks) const {
    Bytes seed(EncapsulationSeedSize());
    fill_random(seed.data(), seed.size());
    return AuthEncapsulateDeterministically(pkr, sks, seed);
  }
  Bytes AuthDecapsulate(const PrivateKey& skr, const Bytes& ct, const PublicKey& pks) const {  // kembase.go:194-217
    auth_only();
    if (ct.size() != CiphertextSize()) throw ErrPubKeySize();
    if (skr.GetScheme() != this || pks.GetScheme() != this) throw ErrTypeMismatch();
    Bytes ss;
    AuthDecapsulateBatch(skr.MarshalBinary(), ct, pks.MarshalBinary(), ss);
    return ss;
  }
  // keys: one key (shared by the batch) or n keys back to back
  void AuthEncapsulateBatch(const Bytes& pkrs, const Bytes& skss, const Bytes& seeds, Bytes& cts, Bytes& sss) const {
    auth_only();
    const size_t n = rows(seeds, EncapsulationSeedSize(), ErrSeedSize());
    const size_t ps = key_stride(pkrs, n, PublicKeySize(), ErrPubKeySize()), ss = key_stride(skss, n, PrivateKeySize(), ErrPrivKeySize());
    cts.resize(n * CiphertextSize());
    sss.resize(n * SharedKeySize());
    check(nist() ? nist()->auth_encaps(pkrs.data(), ps, skss.data(), ss, seeds.data(), cts.data(), sss.data(), nullptr, n)
                 : cb200_hpke_auth_encaps(k_, pkrs.data(), ps, skss.data(), ss, seeds.data(), cts.data(), sss.data(), nullptr, n));
  }
  void AuthDecapsulateBatch(const Bytes& skrs, const Bytes& cts, const Bytes& pkss, Bytes& sss) const {
    auth_only();
    const size_t n = rows(cts, CiphertextSize(), ErrPubKeySize());
    const size_t ss = key_stride(skrs, n, PrivateKeySize(), ErrPrivKeySize()), ps = key_stride(pkss, n, PublicKeySize(), ErrPubKeySize());
    sss.resize(n * SharedKeySize());
    check(nist() ? nist()->auth_decaps(skrs.data(), ss, cts.data(), pkss.data(), ps, sss.data(), nullptr, n)
                 : cb200_hpke_auth_decaps(k_, skrs.data(), ss, cts.data(), pkss.data(), ps, sss.data(), nullptr, n));
  }
  int k() const { return k_; }
  Kind kind() const { return kind_; }
  // DHKEM(P-256, HKDF-SHA256): an HPKE scheme on the cb200_hpke_p256_* entry points (kem::p256::All())
  bool p256() const { return kind_ == HPKE && k_ == CB200_HPKE_P256_HKDF_SHA256; }
  // a NIST DHKEM (P-256, P-384 or P-521; kem::p256 / p384 / p521::All()): its entry points, else nullptr
  const NistOps* nist() const { return kind_ == HPKE ? nist_ops(k_) : nullptr; }

 private:
  bool nist_scalar_ok(const Bytes& k) const {  // 0 < k < n, big-endian (crypto/ecdh NewPrivateKey)
    const uint8_t* n = nist()->n;
    return std::any_of(k.begin(), k.end(), [](uint8_t b) { return b != 0; }) &&
           std::lexicographical_compare(k.begin(), k.end(), n, n + k.size());
  }
  void auth_only() const {
    if (kind_ != HPKE) throw std::logic_error("kem: " + name_ + " is not a kem.AuthScheme");
  }
  template <class E>
  static size_t rows(const Bytes& b, size_t unit, E err) {
    if (b.size() % unit) throw err;
    return b.size() / unit;
  }
  template <class E>
  static size_t key_stride(const Bytes& keys, size_t n, size_t unit, E err) {
    if (keys.size() == unit) return 0;
    if (keys.size() != n * unit) throw err;
    return unit;
  }
  void check(int rc) const {
    if (rc == 0) return;
    if (rc == CB200_ERR_PUBKEY && nist()) throw ErrInvalidKEMPublicKey();
    if (rc == CB200_ERR_PRIVKEY && nist()) throw ErrInvalidKEMPrivateKey();
    if (rc == CB200_ERR_PUBKEY && kind_ == HPKE) throw ErrInvalidKEMSharedSecret();
    if (rc == CB200_ERR_PUBKEY) throw ErrPubKey();
    if (rc == CB200_ERR_PRIVKEY) throw ErrPrivKey();
    if (rc == CB200_ERR_ARG) throw std::logic_error(cb200_last_error());
    throw Error(cb200_last_error());
  }
  std::string name_;
  Kind kind_;
  int k_;  // K of the lattice scheme, or the hybrid / HPKE KEM identifier
};

inline PublicKey PrivateKey::Public() const {
  const Scheme* s = scheme_;
  if (s->kind() == Scheme::HPKE) {  // KeyGen of the stored (unclamped) key (xkem.go:146-163, shortkem.go:151-157)
    Bytes pk(s->PublicKeySize());
    if ((s->nist() ? s->nist()->ecdh : pk.size() == 56 ? cb200_x448 : cb200_x25519)(packed_.data(), nullptr, pk.data(), nullptr, 1))
      throw Error(cb200_last_error());
    return PublicKey(s, std::move(pk));
  }
  if (s->kind() == Scheme::FRODO)  // the embedded public key (frodo.go:466-468)
    return PublicKey(s, Bytes(packed_.begin() + 16, packed_.begin() + 16 + s->PublicKeySize()));
  if (s->kind() == Scheme::XWING) {  // sk is the seed: derive again (xwing.go:278-281)
    Bytes pk, sk;
    s->DeriveKeyPairBatch(packed_, pk, sk);
    return PublicKey(s, std::move(pk));
  }
  if (s->kind() == Scheme::HYBRID) {  // {first.Public(), second.Public()} (hybrid.go:151-153, xkem.go:68-84)
    const size_t xs = s->SharedKeySize() - 32;  // size of the X half: 32 (X25519) or 56 (X448)
    const size_t dk = s->PrivateKeySize() - xs, ek = s->PublicKeySize() - xs, kk = (dk - 96) / 768;
    const bool x_first = s->k() != CB200_HYBRID_X25519MLKEM768;
    Bytes pk(s->PublicKeySize());
    const uint8_t* skm = packed_.data() + (x_first ? xs : 0);
    const uint8_t* skx = packed_.data() + (x_first ? 0 : dk);
    std::copy(skm + 384 * kk, skm + 384 * kk + ek, pk.begin() + (x_first ? xs : 0));
    uint8_t* pkx = pk.data() + (x_first ? 0 : ek);
    if ((xs == 56 ? cb200_x448 : cb200_x25519)(skx, nullptr, pkx, nullptr, 1)) throw Error(cb200_last_error());
    return PublicKey(s, std::move(pk));
  }
  const int k = s->k();
  return PublicKey(s, Bytes(packed_.begin() + 384 * k, packed_.begin() + 384 * k + 384 * k + 32));
}

inline std::pair<PublicKey, PrivateKey> Scheme::GenerateKeyPair() const {
  if (kind_ != HPKE || nist()) return GenerateFromSeed();  // NIST curves: a uniform key in [1, n - 1] from DeriveKeyPair
  Bytes sk(PrivateKeySize());
  fill_random(sk.data(), sk.size());
  PrivateKey priv(this, std::move(sk));
  return {priv.Public(), priv};
}

inline std::string lower(std::string s) {
  std::transform(s.begin(), s.end(), s.begin(), [](unsigned char c) { return (char)std::tolower(c); });
  return s;
}
inline const std::vector<const Scheme*>& All() {  // kem/schemes/schemes.go:75
  static const Scheme s512("ML-KEM-512", 2), s768("ML-KEM-768", 3), s1024("ML-KEM-1024", 4);
  static const Scheme k512("Kyber512", 2, true), k768("Kyber768", 3, true), k1024("Kyber1024", 4, true);
  static const Scheme xw("X-Wing", Scheme::XWING, 0), xm("X25519MLKEM768", Scheme::HYBRID, CB200_HYBRID_X25519MLKEM768),
      k7x("Kyber768-X25519", Scheme::HYBRID, CB200_HYBRID_KYBER768_X25519),
      k5x("Kyber512-X25519", Scheme::HYBRID, CB200_HYBRID_KYBER512_X25519),
      k7x4("Kyber768-X448", Scheme::HYBRID, CB200_HYBRID_KYBER768_X448),
      k10x4("Kyber1024-X448", Scheme::HYBRID, CB200_HYBRID_KYBER1024_X448);
  static const std::vector<const Scheme*> all = {&s512, &s768, &s1024, &k512, &k768, &k1024, &k5x, &k7x, &k7x4, &k10x4, &xm, &xw};
  return all;
}
inline const Scheme* ByName(const std::string& name) {  // kem/schemes/schemes.go:70 (nullptr = no such scheme)
  for (const Scheme* s : All())
    if (lower(s->Name()) == lower(name)) return s;
  return nullptr;
}

// HPKE's two Montgomery-curve DHKEMs (kem/schemes/schemes.go:35-55) are registered on their own so that All()
// above keeps its twelve schemes.
namespace hpke {
inline const std::vector<const Scheme*>& All() {
  static const Scheme x25519("HPKE_KEM_X25519_HKDF_SHA256", Scheme::HPKE, CB200_HPKE_X25519_HKDF_SHA256),
      x448("HPKE_KEM_X448_HKDF_SHA512", Scheme::HPKE, CB200_HPKE_X448_HKDF_SHA512);
  static const std::vector<const Scheme*> all = {&x25519, &x448};
  return all;
}
inline const Scheme* ByName(const std::string& name) {  // case-insensitive; nullptr = no such scheme
  for (const Scheme* s : All())
    if (lower(s->Name()) == lower(name)) return s;
  return nullptr;
}
}  // namespace hpke

// DHKEM(P-256, HKDF-SHA256) (kem/schemes/schemes.go, HPKE_KEM_P256_HKDF_SHA256), registered on its own so that
// hpke::All() keeps its two Montgomery-curve schemes.  UnmarshalBinaryPrivateKey checks the scalar range; a public key
// or encapsulation that is not a P-256 point is reported by the call that uses it (ErrInvalidKEMPublicKey).
namespace p256 {
inline const std::vector<const Scheme*>& All() {
  static const Scheme s("HPKE_KEM_P256_HKDF_SHA256", Scheme::HPKE, CB200_HPKE_P256_HKDF_SHA256);
  static const std::vector<const Scheme*> all = {&s};
  return all;
}
inline const Scheme* ByName(const std::string& name) {  // case-insensitive; nullptr = no such scheme
  for (const Scheme* s : All())
    if (lower(s->Name()) == lower(name)) return s;
  return nullptr;
}
}  // namespace p256

// DHKEM(P-384, HKDF-SHA384) and DHKEM(P-521, HKDF-SHA512) (kem/schemes/schemes.go), registered like P-256's and with
// its checks.
namespace p384 {
inline const std::vector<const Scheme*>& All() {
  static const Scheme s("HPKE_KEM_P384_HKDF_SHA384", Scheme::HPKE, CB200_HPKE_P384_HKDF_SHA384);
  static const std::vector<const Scheme*> all = {&s};
  return all;
}
inline const Scheme* ByName(const std::string& name) {  // case-insensitive; nullptr = no such scheme
  for (const Scheme* s : All())
    if (lower(s->Name()) == lower(name)) return s;
  return nullptr;
}
}  // namespace p384
namespace p521 {
inline const std::vector<const Scheme*>& All() {
  static const Scheme s("HPKE_KEM_P521_HKDF_SHA512", Scheme::HPKE, CB200_HPKE_P521_HKDF_SHA512);
  static const std::vector<const Scheme*> all = {&s};
  return all;
}
inline const Scheme* ByName(const std::string& name) {  // case-insensitive; nullptr = no such scheme
  for (const Scheme* s : All())
    if (lower(s->Name()) == lower(name)) return s;
  return nullptr;
}
}  // namespace p521

// FrodoKEM-640-SHAKE (kem/schemes/schemes.go entry 6), registered on its own like the HPKE DHKEMs.
namespace frodo {
inline const std::vector<const Scheme*>& All() {
  static const Scheme f("FrodoKEM-640-SHAKE", Scheme::FRODO, 0);
  static const std::vector<const Scheme*> all = {&f};
  return all;
}
inline const Scheme* ByName(const std::string& name) {  // case-insensitive; nullptr = no such scheme
  for (const Scheme* s : All())
    if (lower(s->Name()) == lower(name)) return s;
  return nullptr;
}
}  // namespace frodo

}  // namespace kem

namespace sign {

struct ErrContextTooLong : Error { ErrContextTooLong() : Error("sign: context string too long") {} };
struct ErrContextNotSupported : Error { ErrContextNotSupported() : Error("sign: context not supported") {} };
struct ErrPubKeySize : Error { ErrPubKeySize() : Error("sign: invalid public key size") {} };
struct ErrPrivKeySize : Error { ErrPrivKeySize() : Error("sign: invalid private key size") {} };
struct ErrSeedSize : Error { ErrSeedSize() : Error("sign: invalid seed size") {} };

struct SignatureOpts {  // sign/sign.go:14-18
  std::string Context;
};

class Scheme;
class PublicKey {
 public:
  PublicKey(const Scheme* s, Bytes b) : scheme_(s), packed_(std::move(b)) {}
  const Scheme* GetScheme() const { return scheme_; }
  const Bytes& MarshalBinary() const { return packed_; }
  bool Equal(const PublicKey& o) const { return packed_ == o.packed_; }

 private:
  const Scheme* scheme_;
  Bytes packed_;
};
class PrivateKey {
 public:
  PrivateKey(const Scheme* s, Bytes b) : scheme_(s), packed_(std::move(b)) {}
  const Scheme* GetScheme() const { return scheme_; }
  const Bytes& MarshalBinary() const { return packed_; }
  bool Equal(const PrivateKey& o) const { return packed_ == o.packed_; }

 private:
  const Scheme* scheme_;
  Bytes packed_;
};

class Scheme {  // sign.Scheme (sign/sign.go:48-94) for ML-DSA-44/65/87 (modes 44, 65, 87), round-3 Dilithium2/3/5 (2, 3, 5),
                // Ed25519 (sign/ed25519/signapi.go), Ed25519-Dilithium2 (sign/eddilithium2/signapi.go), Ed448
                // (sign/ed448/signapi.go) and Ed448-Dilithium3 (sign/eddilithium3/signapi.go)
 public:
  enum Family { kMLDSA, kEd25519, kEdDilithium2, kEd448, kEdDilithium3 };
  Scheme(std::string name, int mode, Family family = kMLDSA) : name_(std::move(name)), mode_(mode), family_(family) {}
  const std::string& Name() const { return name_; }
  size_t PublicKeySize() const {
    return family_ == kEd25519 ? cb200_ed25519_public_key_size()
           : family_ == kEdDilithium2 ? cb200_eddilithium2_public_key_size()
           : family_ == kEd448 ? cb200_ed448_public_key_size()
           : family_ == kEdDilithium3 ? cb200_eddilithium3_public_key_size() : cb200_mldsa_public_key_size(mode_);
  }
  size_t PrivateKeySize() const {
    return family_ == kEd25519 ? cb200_ed25519_private_key_size()
           : family_ == kEdDilithium2 ? cb200_eddilithium2_private_key_size()
           : family_ == kEd448 ? cb200_ed448_private_key_size()
           : family_ == kEdDilithium3 ? cb200_eddilithium3_private_key_size() : cb200_mldsa_private_key_size(mode_);
  }
  size_t SignatureSize() const {
    return family_ == kEd25519 ? cb200_ed25519_signature_size()
           : family_ == kEdDilithium2 ? cb200_eddilithium2_signature_size()
           : family_ == kEd448 ? cb200_ed448_signature_size()
           : family_ == kEdDilithium3 ? cb200_eddilithium3_signature_size() : cb200_mldsa_signature_size(mode_);
  }
  size_t SeedSize() const { return family_ == kEd448 || family_ == kEdDilithium3 ? 57 : 32; }
  // round 3, Ed25519, Ed25519-Dilithium2 and Ed448-Dilithium3: sign.ErrContextNotSupported; Ed448 takes a context
  bool SupportsContext() const { return (family_ == kMLDSA && mode_ > 10) || family_ == kEd448; }

  std::pair<PublicKey, PrivateKey> DeriveKey(const Bytes& seed) const {  // dilithium.go:266-276, ed25519 signapi.go
    if (seed.size() != SeedSize()) throw std::logic_error("sign: invalid seed size");  // Go panics here
    Bytes pk, sk;
    DeriveKeyBatch(seed, pk, sk);
    return {PublicKey(this, std::move(pk)), PrivateKey(this, std::move(sk))};
  }
  std::pair<PublicKey, PrivateKey> GenerateKey() const {
    Bytes seed(SeedSize());
    fill_random(seed.data(), seed.size());
    return DeriveKey(seed);
  }
  PublicKey UnmarshalBinaryPublicKey(const Bytes& b) const {
    if (b.size() != PublicKeySize()) throw ErrPubKeySize();
    return PublicKey(this, b);
  }
  PrivateKey UnmarshalBinaryPrivateKey(const Bytes& b) const {
    if (b.size() != PrivateKeySize()) throw ErrPrivKeySize();
    return PrivateKey(this, b);
  }
  // PrivateKey.Public() of Ed25519 and Ed448 (ed25519.go, ed448.go: the second half of the private key).  The ML-DSA
  // and composite private keys do not hold their public key; their Public() needs the seed (DeriveKey).
  PublicKey Public(const PrivateKey& sk) const {
    if (family_ != kEd25519 && family_ != kEd448)
      throw std::logic_error("sign: Public() from a packed private key is served for Ed25519 and Ed448 only");
    const Bytes& b = sk.MarshalBinary();
    return PublicKey(this, Bytes(b.begin() + PublicKeySize(), b.end()));
  }
  // deterministic signing, as sign.Scheme.Sign does (dilithium.go:282-303, ed25519 signapi.go)
  Bytes Sign(const PrivateKey& sk, const Bytes& msg, const SignatureOpts* opts = nullptr) const {
    const std::string ctx = opts ? opts->Context : std::string();
    Bytes sigs;
    SignBatch(sk.MarshalBinary(), msg, {0, msg.size()}, ctx, sigs);
    return sigs;
  }
  bool Verify(const PublicKey& pk, const Bytes& msg, const Bytes& sig, const SignatureOpts* opts = nullptr) const {
    const std::string ctx = opts ? opts->Context : std::string();
    if (!ctx.empty() && family_ != kMLDSA && family_ != kEd448) throw ErrContextNotSupported();
    if (ctx.size() > 255 || sig.size() != SignatureSize()) return false;  // dilithium.go:116-118, ed25519.go:330-334
    uint8_t ok = 0;
    const uint64_t off[2] = {0, msg.size()};
    Bytes padded(msg);
    padded.resize(msg.size() + 8);
    if (family_ == kEd25519)
      check(cb200_ed25519_verify(pk.MarshalBinary().data(), 0, padded.data(), off, sig.data(), &ok, 1));
    else if (family_ == kEdDilithium2)
      check(cb200_eddilithium2_verify(pk.MarshalBinary().data(), 0, padded.data(), off, sig.data(), &ok, 1));
    else if (family_ == kEd448)
      check(cb200_ed448_verify(pk.MarshalBinary().data(), 0, padded.data(), off, (const uint8_t*)ctx.data(), ctx.size(),
                               sig.data(), &ok, 1));
    else if (family_ == kEdDilithium3)
      check(cb200_eddilithium3_verify(pk.MarshalBinary().data(), 0, padded.data(), off, sig.data(), &ok, 1));
    else
      check(cb200_mldsa_verify(mode_, pk.MarshalBinary().data(), 0, padded.data(), off, (const uint8_t*)ctx.data(), ctx.size(),
                               sig.data(), &ok, 1, 0));
    return ok != 0;
  }
  // batch: messages back to back with n+1 offsets; sks: one key (shared) or n keys
  void SignBatch(const Bytes& sks, const Bytes& msgs, const std::vector<uint64_t>& off, const std::string& ctx, Bytes& sigs) const {
    if (!ctx.empty() && !SupportsContext()) throw ErrContextNotSupported();
    if (ctx.size() > 255) throw ErrContextTooLong();
    const size_t n = off.size() - 1;
    const bool shared = sks.size() == PrivateKeySize();
    if (!shared && sks.size() != n * PrivateKeySize()) throw ErrPrivKeySize();
    sigs.resize(n * SignatureSize());
    Bytes padded(msgs);
    padded.resize(msgs.size() + 8);
    const size_t stride = shared ? 0 : PrivateKeySize();
    if (family_ == kEd25519)
      check(cb200_ed25519_sign(sks.data(), stride, padded.data(), off.data(), sigs.data(), n));
    else if (family_ == kEdDilithium2)
      check(cb200_eddilithium2_sign(sks.data(), stride, padded.data(), off.data(), sigs.data(), nullptr, n));
    else if (family_ == kEd448)
      check(cb200_ed448_sign(sks.data(), stride, padded.data(), off.data(), (const uint8_t*)ctx.data(), ctx.size(), sigs.data(),
                             n));
    else if (family_ == kEdDilithium3)
      check(cb200_eddilithium3_sign(sks.data(), stride, padded.data(), off.data(), sigs.data(), nullptr, n));
    else
      check(cb200_mldsa_sign(mode_, sks.data(), stride, padded.data(), off.data(), (const uint8_t*)ctx.data(), ctx.size(), nullptr,
                             sigs.data(), nullptr, n, 0, nullptr));
  }
  // ok[i] = 1 where signature i verifies; pks: one key (shared) or n keys
  void VerifyBatch(const Bytes& pks, const Bytes& msgs, const std::vector<uint64_t>& off, const std::string& ctx,
                   const Bytes& sigs, Bytes& ok) const {
    if (!ctx.empty() && !SupportsContext()) throw ErrContextNotSupported();
    const size_t n = off.size() - 1;
    const bool shared = pks.size() == PublicKeySize();
    if (!shared && pks.size() != n * PublicKeySize()) throw ErrPubKeySize();
    ok.assign(n, 0);
    if (ctx.size() > 255 || sigs.size() != n * SignatureSize()) return;  // dilithium.go:116-118: such signatures are invalid
    Bytes padded(msgs);
    padded.resize(msgs.size() + 8);
    const size_t stride = shared ? 0 : PublicKeySize();
    if (family_ == kEd25519)
      check(cb200_ed25519_verify(pks.data(), stride, padded.data(), off.data(), sigs.data(), ok.data(), n));
    else if (family_ == kEdDilithium2)
      check(cb200_eddilithium2_verify(pks.data(), stride, padded.data(), off.data(), sigs.data(), ok.data(), n));
    else if (family_ == kEd448)
      check(cb200_ed448_verify(pks.data(), stride, padded.data(), off.data(), (const uint8_t*)ctx.data(), ctx.size(), sigs.data(),
                               ok.data(), n));
    else if (family_ == kEdDilithium3)
      check(cb200_eddilithium3_verify(pks.data(), stride, padded.data(), off.data(), sigs.data(), ok.data(), n));
    else
      check(cb200_mldsa_verify(mode_, pks.data(), stride, padded.data(), off.data(), (const uint8_t*)ctx.data(), ctx.size(),
                               sigs.data(), ok.data(), n, 0));
  }
  void DeriveKeyBatch(const Bytes& seeds, Bytes& pks, Bytes& sks) const {
    if (seeds.size() % SeedSize()) throw ErrSeedSize();
    const size_t n = seeds.size() / SeedSize();
    pks.resize(n * PublicKeySize());
    sks.resize(n * PrivateKeySize());
    if (family_ == kEd25519)
      check(cb200_ed25519_keygen(seeds.data(), pks.data(), sks.data(), n));
    else if (family_ == kEdDilithium2)
      check(cb200_eddilithium2_keygen(seeds.data(), pks.data(), sks.data(), n));
    else if (family_ == kEd448)
      check(cb200_ed448_keygen(seeds.data(), pks.data(), sks.data(), n));
    else if (family_ == kEdDilithium3)
      check(cb200_eddilithium3_keygen(seeds.data(), pks.data(), sks.data(), n));
    else
      check(cb200_mldsa_keygen(mode_, seeds.data(), pks.data(), sks.data(), n));
  }

 private:
  static void check(int rc) {
    if (rc == 0) return;
    if (rc == CB200_ERR_ARG) throw std::logic_error(cb200_last_error());
    throw Error(cb200_last_error());  // includes CB200_ERR_SIGN_ATTEMPTS (the reference panics after 576 attempts)
  }
  std::string name_;
  int mode_;
  Family family_;
};

// in the order of sign/schemes/schemes.go:31-44 for the schemes served here
inline const std::vector<const Scheme*>& All() {
  static const Scheme e25519("Ed25519", 0, Scheme::kEd25519), ed2("Ed25519-Dilithium2", 2, Scheme::kEdDilithium2);
  static const Scheme s44("ML-DSA-44", 44), s65("ML-DSA-65", 65), s87("ML-DSA-87", 87);
  static const Scheme d2("Dilithium2", 2), d3("Dilithium3", 3), d5("Dilithium5", 5);
  static const std::vector<const Scheme*> all = {&e25519, &ed2, &s44, &s65, &s87, &d2, &d3, &d5};
  return all;
}
inline const Scheme* ByName(const std::string& name) {  // sign/schemes/schemes.go:69 (nullptr = no such scheme)
  for (const Scheme* s : All())
    if (kem::lower(s->Name()) == kem::lower(name)) return s;
  return nullptr;
}

// Ed448 and Ed448-Dilithium3 (sign/schemes/schemes.go:31-54 lists them second and fourth).  They have a registry of
// their own so that All() above keeps its eight schemes.
namespace ed448 {
inline const std::vector<const Scheme*>& All() {
  static const Scheme e448("Ed448", 0, Scheme::kEd448), ed3("Ed448-Dilithium3", 3, Scheme::kEdDilithium3);
  static const std::vector<const Scheme*> all = {&e448, &ed3};
  return all;
}
inline const Scheme* ByName(const std::string& name) {  // case-insensitive; nullptr = no such scheme
  for (const Scheme* s : All())
    if (kem::lower(s->Name()) == kem::lower(name)) return s;
  return nullptr;
}
}  // namespace ed448

}  // namespace sign

// ---------------------------------------------------------------- oprf: RFC 9497 servers (oprf/{oprf,server,keys}.go)
// The suites P256-SHA256, P384-SHA384 and P521-SHA512; Server, VerifiableServer and PartialObliviousServer with
// Evaluate, FullEvaluate, VerifyFinalize and PublicKey, plus batch forms on host rows.  The proof randomness
// of Evaluate comes from fill_random (the reference's rand.Reader) unless the batch form is given rows of it.
namespace oprf {
enum Mode : int { BaseMode = 0, VerifiableMode = 1, PartialObliviousMode = 2 };
struct OprfError : Error {
  std::vector<uint8_t> status;  // per-op bits of a failed batch: 1 element, 2 key, 4 r, 8 t = 0, 16 input length
  explicit OprfError(const std::string& m, std::vector<uint8_t> st = {}) : Error(m), status(std::move(st)) {}
};
#define CIRCL_OPRF_ERROR(name, text) \
  struct name : OprfError {          \
    explicit name(std::vector<uint8_t> st = {}) : OprfError(text, std::move(st)) {} \
  };
CIRCL_OPRF_ERROR(ErrInvalidSuite, "oprf: invalid suite")
CIRCL_OPRF_ERROR(ErrInvalidMode, "oprf: invalid mode")
CIRCL_OPRF_ERROR(ErrInvalidSeed, "oprf: invalid seed size")
CIRCL_OPRF_ERROR(ErrInvalidInfo, "oprf: invalid info")
CIRCL_OPRF_ERROR(ErrInvalidInput, "oprf: invalid input")
CIRCL_OPRF_ERROR(ErrInvalidPrivateKey, "oprf: invalid private key")
CIRCL_OPRF_ERROR(ErrInverseZero, "oprf: inverting a zero value")
CIRCL_OPRF_ERROR(ErrInvalidRandomness, "oprf: invalid proof randomness")
#undef CIRCL_OPRF_ERROR

struct Suite {
  int id;
  const char* identifier;
  std::string Identifier() const { return identifier; }
  size_t Ne() const { return cb200_oprf_element_size(id); }
  size_t Ns() const { return cb200_oprf_scalar_size(id); }
  size_t Nh() const { return cb200_oprf_output_size(id); }
  size_t ProofSize() const { return cb200_oprf_proof_size(id); }
};
inline const Suite SuiteP256{CB200_OPRF_P256_SHA256, "P256-SHA256"};
inline const Suite SuiteP384{CB200_OPRF_P384_SHA384, "P384-SHA384"};
inline const Suite SuiteP521{CB200_OPRF_P521_SHA512, "P521-SHA512"};
inline Suite GetSuite(const std::string& identifier) {
  for (const Suite* s : {&SuiteP256, &SuiteP384, &SuiteP521})
    if (identifier == s->identifier) return *s;
  throw ErrInvalidSuite();
}

namespace detail {
inline void check_call(int rc) {
  if (rc == CB200_ERR_ARG) throw std::logic_error(cb200_last_error());
  if (rc != 0) throw Error(cb200_last_error());
}
// the error of the first failure class, as circl_b200.oprf raises it
inline void check_status(const uint8_t* st, size_t n) {
  uint8_t any = 0;
  for (size_t i = 0; i < n; i++) any |= st[i];
  if (!any) return;
  std::vector<uint8_t> v(st, st + n);
  if (any & 2) throw ErrInvalidPrivateKey(v);
  if (any & 8) throw ErrInverseZero(v);
  if (any & (1 | 16)) throw ErrInvalidInput(v);
  throw ErrInvalidRandomness(v);
}
inline void check_mode_info(int mode, const Bytes& info) {
  if (mode < 0 || mode > 2) throw ErrInvalidMode();
  if (info.size() > 65535) throw ErrInvalidInfo();
}
}  // namespace detail

struct PrivateKey {
  Suite suite;
  Bytes k, pk;
  Bytes MarshalBinary() const { return k; }
  Bytes Public() const { return pk; }
};
// DeriveKey (keys.go:103-132)
inline PrivateKey DeriveKey(const Suite& s, int mode, const Bytes& seed, const Bytes& info = {}) {
  detail::check_mode_info(mode, info);
  if (seed.size() != 32) throw ErrInvalidSeed();
  PrivateKey key{s, Bytes(s.Ns()), Bytes(s.Ne())};
  detail::check_call(cb200_oprf_derive_key(s.id, mode, seed.data(), info.data(), info.size(), key.k.data(),
                                           key.pk.data(), 1));
  return key;
}

struct Evaluation {
  std::vector<Bytes> Elements;
  Bytes Proof;  // c || s; empty in mode 0
};

class ServerBase {
 public:
  ServerBase(Suite s, PrivateKey key, int mode) : s_(s), key_(std::move(key)), mode_(mode) {}
  Bytes PublicKey() const { return key_.Public(); }
  // n requests of m elements (n * m rows of Ne at `blinded`), rnd: n rows of Ns (modes 1, 2) -> evaluated (n * m rows
  // of Ne) and proof (n rows of 2 Ns).  Host buffers (the key and the status bytes are host memory); a failed op raises
  // after the batch, rows zeroed.
  void EvaluateBatch(const uint8_t* blinded, size_t m, const uint8_t* rnd, const Bytes& info, uint8_t* evaluated,
                     uint8_t* proof, size_t n) const {
    detail::check_mode_info(mode_, info);
    std::vector<uint8_t> st(n);
    detail::check_call(cb200_oprf_evaluate(s_.id, mode_, key_.k.data(), 0, blinded, m, rnd, info.data(), info.size(),
                                           evaluated, proof, st.data(), n));
    detail::check_status(st.data(), n);
  }
  // inputs msgs[off[i] .. off[i + 1]) -> n rows of Nh
  void FullEvaluateBatch(const uint8_t* msgs, const uint64_t* off, const Bytes& info, uint8_t* out, size_t n) const {
    detail::check_mode_info(mode_, info);
    std::vector<uint8_t> st(n);
    detail::check_call(cb200_oprf_full_evaluate(s_.id, mode_, key_.k.data(), 0, msgs, off, info.data(), info.size(), out,
                                                st.data(), n));
    detail::check_status(st.data(), n);
  }

 protected:
  Evaluation evaluate(const std::vector<Bytes>& elements, const Bytes& info) const {
    const size_t Ne = s_.Ne(), Ns = s_.Ns();
    Bytes b;
    for (const Bytes& e : elements) {
      if (e.size() != Ne) throw ErrInvalidInput();
      b.insert(b.end(), e.begin(), e.end());
    }
    if (elements.empty()) throw ErrInvalidInput();
    Bytes r(Ns), ev(b.size()), proof(mode_ ? 2 * Ns : 0);
    if (mode_) random_scalar(r);
    EvaluateBatch(b.data(), elements.size(), mode_ ? r.data() : nullptr, info, ev.data(), mode_ ? proof.data() : nullptr,
                  1);
    Evaluation out{{}, proof};
    for (size_t j = 0; j < elements.size(); j++) out.Elements.emplace_back(ev.begin() + j * Ne, ev.begin() + (j + 1) * Ne);
    return out;
  }
  Bytes full(const Bytes& input, const Bytes& info) const {
    if (input.size() > 65535) throw ErrInvalidInput();
    const uint64_t off[2] = {0, input.size()};
    Bytes out(s_.Nh());
    const uint8_t zero = 0;
    FullEvaluateBatch(input.empty() ? &zero : input.data(), off, info, out.data(), 1);
    return out;
  }
  bool verify(const Bytes& input, const Bytes& info, const Bytes& expected) const {
    Bytes got;
    try {
      got = full(input, info);
    } catch (const OprfError&) {
      return false;
    }
    if (got.size() != expected.size()) return false;
    uint8_t d = 0;
    for (size_t i = 0; i < got.size(); i++) d |= got[i] ^ expected[i];
    return d == 0;
  }
  // a uniform r in [1, n - 1]: the leading byte masked to the order's bit length, then rejection against the device's
  // own range test (an r the call would flag is drawn again)
  void random_scalar(Bytes& r) const {
    const uint8_t top = s_.Ns() == 66 ? 0x01 : 0xff;
    for (;;) {
      fill_random(r.data(), r.size());
      r[0] &= top;
      if (lt_order(r)) return;
    }
  }
  bool lt_order(const Bytes& r) const {
    static const uint8_t n256[32] = {0xff, 0xff, 0xff, 0xff, 0x00, 0x00, 0x00, 0x00, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                     0xff, 0xff, 0xbc, 0xe6, 0xfa, 0xad, 0xa7, 0x17, 0x9e, 0x84, 0xf3, 0xb9, 0xca, 0xc2,
                                     0xfc, 0x63, 0x25, 0x51};
    static const uint8_t n384[48] = {0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                     0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xc7, 0x63, 0x4d, 0x81,
                                     0xf4, 0x37, 0x2d, 0xdf, 0x58, 0x1a, 0x0d, 0xb2, 0x48, 0xb0, 0xa7, 0x7a, 0xec, 0xec,
                                     0x19, 0x6a, 0xcc, 0xc5, 0x29, 0x73};
    static const uint8_t n521[66] = {0x01, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                     0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff,
                                     0xff, 0xff, 0xff, 0xff, 0xff, 0xfa, 0x51, 0x86, 0x87, 0x83, 0xbf, 0x2f, 0x96, 0x6b,
                                     0x7f, 0xcc, 0x01, 0x48, 0xf7, 0x09, 0xa5, 0xd0, 0x3b, 0xb5, 0xc9, 0xb8, 0x89, 0x9c,
                                     0x47, 0xae, 0xbb, 0x6f, 0xb7, 0x1e, 0x91, 0x38, 0x64, 0x09};
    const uint8_t* n = r.size() == 32 ? n256 : r.size() == 48 ? n384 : n521;
    bool nz = false;
    for (uint8_t v : r) nz |= v != 0;
    return nz && std::lexicographical_compare(r.begin(), r.end(), n, n + r.size());
  }
  Suite s_;
  PrivateKey key_;
  int mode_;
};

class Server : public ServerBase {
 public:
  Server(Suite s, PrivateKey key) : ServerBase(s, std::move(key), BaseMode) {}
  Evaluation Evaluate(const std::vector<Bytes>& elements) const { return evaluate(elements, {}); }
  Bytes FullEvaluate(const Bytes& input) const { return full(input, {}); }
  bool VerifyFinalize(const Bytes& input, const Bytes& expected) const { return verify(input, {}, expected); }
};
class VerifiableServer : public ServerBase {
 public:
  VerifiableServer(Suite s, PrivateKey key) : ServerBase(s, std::move(key), VerifiableMode) {}
  Evaluation Evaluate(const std::vector<Bytes>& elements) const { return evaluate(elements, {}); }
  Bytes FullEvaluate(const Bytes& input) const { return full(input, {}); }
  bool VerifyFinalize(const Bytes& input, const Bytes& expected) const { return verify(input, {}, expected); }
};
class PartialObliviousServer : public ServerBase {
 public:
  PartialObliviousServer(Suite s, PrivateKey key) : ServerBase(s, std::move(key), PartialObliviousMode) {}
  Evaluation Evaluate(const std::vector<Bytes>& elements, const Bytes& info) const { return evaluate(elements, info); }
  Bytes FullEvaluate(const Bytes& input, const Bytes& info) const { return full(input, info); }
  bool VerifyFinalize(const Bytes& input, const Bytes& info, const Bytes& expected) const {
    return verify(input, info, expected);
  }
};
inline Server NewServer(const Suite& s, const PrivateKey& k) { return Server(s, k); }
inline VerifiableServer NewVerifiableServer(const Suite& s, const PrivateKey& k) { return VerifiableServer(s, k); }
inline PartialObliviousServer NewPartialObliviousServer(const Suite& s, const PrivateKey& k) {
  return PartialObliviousServer(s, k);
}
}  // namespace oprf

// RSA blind signatures (RFC 9474, RSABSSA-SHA384), server side: the reference's blindsign/blindrsa package (brsa.go).
// Keys are big-endian byte strings; a private key carries the PKCS #1 CRT fields (Go's Precomputed Dp, Dq, Qinv).
// The constructors check the key without a device (cb200_brsa_* with n = 0) and throw ErrInvalidKey for one outside
// the served range; a batch whose ops fail throws the error of the first failure class with the per-op status bytes.
namespace blindrsa {
enum Variant : int {
  SHA384PSSRandomized = CB200_BRSA_SHA384_PSS_RANDOMIZED,
  SHA384PSSZeroRandomized = CB200_BRSA_SHA384_PSSZERO_RANDOMIZED,
  SHA384PSSDeterministic = CB200_BRSA_SHA384_PSS_DETERMINISTIC,
  SHA384PSSZeroDeterministic = CB200_BRSA_SHA384_PSSZERO_DETERMINISTIC,
};
struct BlindRSAError : Error {
  std::vector<uint8_t> status;  // per-op bytes of a failed batch
  explicit BlindRSAError(const std::string& m, std::vector<uint8_t> st = {}) : Error(m), status(std::move(st)) {}
};
#define CIRCL_BRSA_ERROR(name, text) \
  struct name : BlindRSAError {      \
    explicit name(std::vector<uint8_t> st = {}) : BlindRSAError(text, std::move(st)) {} \
  };
CIRCL_BRSA_ERROR(ErrInvalidVariant, "blindrsa: invalid BRSA variant")
CIRCL_BRSA_ERROR(ErrUnexpectedSize, "blindrsa: unexpected input size")
CIRCL_BRSA_ERROR(ErrInvalidMessageLength, "blindrsa: invalid message length")
CIRCL_BRSA_ERROR(ErrInternal, "rsa: internal error")
CIRCL_BRSA_ERROR(ErrVerification, "crypto/rsa: verification error")
#undef CIRCL_BRSA_ERROR
struct ErrInvalidKey : BlindRSAError {
  explicit ErrInvalidKey(const std::string& m) : BlindRSAError(m) {}
};

struct PublicKey {
  Bytes N, E;
  size_t Size() const { return N.empty() ? 0 : cb200_brsa_modulus_bytes(N.data(), N.size()); }
};
struct PrivateKey {
  PublicKey pub;
  Bytes P, Q, Dp, Dq, Qinv;
  const PublicKey& Public() const { return pub; }
};

namespace detail {
inline const uint8_t* p(const Bytes& b) { return b.empty() ? nullptr : b.data(); }
inline void check_call(int rc) {
  if (rc == CB200_ERR_ARG) throw std::logic_error(cb200_last_error());
  if (rc != 0) throw Error(cb200_last_error());
}
// strings back to back with their n + 1 offsets; the blob is never empty
inline void pack(const std::vector<Bytes>& v, Bytes* blob, std::vector<uint64_t>* off) {
  off->assign(v.size() + 1, 0);
  for (size_t i = 0; i < v.size(); i++) {
    blob->insert(blob->end(), v[i].begin(), v[i].end());
    (*off)[i + 1] = blob->size();
  }
  blob->push_back(0);
}
// BlindSign status bytes: throws ErrInvalidMessageLength if any op has status 1, else ErrInternal if any has 2
inline void throw_sign_status(const std::vector<uint8_t>& st) {
  for (uint8_t bit : {1, 2})
    for (uint8_t s : st)
      if (s == bit) {
        if (bit == 1) throw ErrInvalidMessageLength(st);
        throw ErrInternal(st);
      }
}
}  // namespace detail

class Signer {
 public:
  explicit Signer(PrivateKey sk) : sk_(std::move(sk)) {
    uint8_t z[1] = {0};
    if (call(z, z, z, 0) == CB200_ERR_ARG) throw ErrInvalidKey(cb200_last_error());
  }
  size_t KLen() const { return sk_.pub.Size(); }
  // n blinded rows of KLen bytes back to back -> n blind signatures; throws ErrInvalidMessageLength (c > N) or
  // ErrInternal (the s^e mod N == c check) with the status bytes; failed rows are zero
  Bytes BlindSignBatch(const Bytes& blinded) const {
    const size_t k = KLen();
    if (blinded.size() % k) throw ErrUnexpectedSize();
    const size_t n = blinded.size() / k;
    Bytes sig(n * k);
    std::vector<uint8_t> st(n);
    if (n) detail::check_call(call(blinded.data(), sig.data(), st.data(), n));
    detail::throw_sign_status(st);
    return sig;
  }
  Bytes BlindSign(const Bytes& data) const {  // brsa.go:237-257
    if (data.size() != KLen()) throw ErrUnexpectedSize();
    return BlindSignBatch(data);
  }

 private:
  int call(const uint8_t* in, uint8_t* out, uint8_t* st, size_t n) const {
    using detail::p;
    const PublicKey& k = sk_.pub;
    return cb200_brsa_blind_sign(p(k.N), k.N.size(), p(k.E), k.E.size(), p(sk_.P), sk_.P.size(), p(sk_.Q), sk_.Q.size(),
                                 p(sk_.Dp), sk_.Dp.size(), p(sk_.Dq), sk_.Dq.size(), p(sk_.Qinv), sk_.Qinv.size(), in,
                                 out, st, n);
  }
  PrivateKey sk_;
};

class Verifier {
 public:
  Verifier(Variant v, PublicKey pk) : v_(v), pk_(std::move(pk)) {
    if (v < SHA384PSSRandomized || v > SHA384PSSZeroDeterministic) throw ErrInvalidVariant();
    uint8_t z[1] = {0};
    uint64_t off[1] = {0};
    if (call(z, off, z, z, 0) == CB200_ERR_ARG) throw ErrInvalidKey(cb200_last_error());
  }
  size_t KLen() const { return pk_.Size(); }
  // status bytes of messages[i] against signature row i (KLen bytes each, back to back): 0 valid, 1 s >= N, 2 an
  // inconsistent encoding; throws ErrVerification with them if any op fails
  std::vector<uint8_t> VerifyBatch(const std::vector<Bytes>& messages, const Bytes& sigs) const {
    const size_t n = messages.size(), k = KLen();
    if (sigs.size() != n * k) throw ErrUnexpectedSize();
    Bytes blob;
    std::vector<uint64_t> off;
    detail::pack(messages, &blob, &off);
    std::vector<uint8_t> st(n);
    if (n) detail::check_call(call(blob.data(), off.data(), sigs.data(), st.data(), n));
    for (uint8_t s : st)
      if (s) throw ErrVerification(st);
    return st;
  }
  void Verify(const Bytes& message, const Bytes& signature) const {  // brsa.go:214
    if (signature.size() != KLen()) throw ErrVerification();
    VerifyBatch({message}, signature);
  }

 private:
  int call(const uint8_t* msgs, const uint64_t* off, const uint8_t* sigs, uint8_t* st, size_t n) const {
    using detail::p;
    return cb200_brsa_verify(v_, p(pk_.N), pk_.N.size(), p(pk_.E), pk_.E.size(), msgs, off, sigs, st, n);
  }
  Variant v_;
  PublicKey pk_;
};
inline Signer NewSigner(const PrivateKey& sk) { return Signer(sk); }
inline Verifier NewVerifier(Variant v, const PublicKey& pk) { return Verifier(v, pk); }
}  // namespace blindrsa

// Partially blind RSA signatures (RSAPBSSA-SHA384), server side: the reference's blindsign/blindrsa/partiallyblindrsa
// package (pbrsa.go).  Each op's metadata selects the key it is signed and verified under.  Keys are blindrsa's;
// a private key needs N, P, Q and Qinv (E, Dp and Dq are not used).  Signer runs NewSigner's safe-prime test once
// (cb200_pbrsa_check_key) and throws ErrInvalidPrivateKey for a key that fails it or lies outside the served range;
// Verifier throws ErrInvalidPublicKey for a modulus outside the range.  Errors are blindrsa's otherwise.
namespace partiallyblindrsa {
using blindrsa::BlindRSAError;
using blindrsa::ErrInternal;
using blindrsa::ErrInvalidMessageLength;
using blindrsa::ErrUnexpectedSize;
using blindrsa::ErrVerification;
using blindrsa::PrivateKey;
using blindrsa::PublicKey;
struct ErrInvalidPrivateKey : BlindRSAError {
  explicit ErrInvalidPrivateKey(const std::string& m) : BlindRSAError(m) {}
};
struct ErrInvalidPublicKey : BlindRSAError {
  explicit ErrInvalidPublicKey(const std::string& m) : BlindRSAError(m) {}
};

class Signer {
 public:
  explicit Signer(PrivateKey sk) : sk_(std::move(sk)) {
    using blindrsa::detail::p;
    uint8_t z[1] = {0};
    uint64_t off[1] = {0};
    const PublicKey& k = sk_.pub;
    if (call(z, z, off, z, z, 0) == CB200_ERR_ARG ||
        cb200_pbrsa_check_key(p(k.N), k.N.size(), p(sk_.P), sk_.P.size(), p(sk_.Q), sk_.Q.size()) == CB200_ERR_ARG)
      throw ErrInvalidPrivateKey(cb200_last_error());
  }
  size_t KLen() const { return sk_.pub.Size(); }
  // n blinded rows of KLen bytes back to back, op i under metadata[i] -> n blind signatures; throws
  // ErrInvalidMessageLength (c > N) or ErrInternal (the s^e' mod N == c check) with the status bytes
  Bytes BlindSignBatch(const Bytes& blinded, const std::vector<Bytes>& metadata) const {
    const size_t k = KLen();
    if (blinded.size() % k || blinded.size() / k != metadata.size()) throw ErrUnexpectedSize();
    const size_t n = metadata.size();
    Bytes sig(n * k), meta;
    std::vector<uint64_t> off;
    blindrsa::detail::pack(metadata, &meta, &off);
    std::vector<uint8_t> st(n);
    if (n) blindrsa::detail::check_call(call(blinded.data(), meta.data(), off.data(), sig.data(), st.data(), n));
    blindrsa::detail::throw_sign_status(st);
    return sig;
  }
  Bytes BlindSign(const Bytes& data, const Bytes& metadata) const {  // pbrsa.go:350-375
    if (data.size() != KLen()) throw ErrUnexpectedSize();
    return BlindSignBatch(data, {metadata});
  }

 private:
  int call(const uint8_t* in, const uint8_t* meta, const uint64_t* off, uint8_t* out, uint8_t* st, size_t n) const {
    using blindrsa::detail::p;
    const PublicKey& k = sk_.pub;
    return cb200_pbrsa_blind_sign(p(k.N), k.N.size(), p(sk_.P), sk_.P.size(), p(sk_.Q), sk_.Q.size(), p(sk_.Qinv),
                                  sk_.Qinv.size(), in, meta, off, out, st, n);
  }
  PrivateKey sk_;
};

class Verifier {
 public:
  explicit Verifier(PublicKey pk) : pk_(std::move(pk)) {
    uint8_t z[1] = {0};
    uint64_t off[1] = {0};
    if (call(z, off, z, off, z, z, 0) == CB200_ERR_ARG) throw ErrInvalidPublicKey(cb200_last_error());
  }
  size_t KLen() const { return pk_.Size(); }
  // status bytes of messages[i] under metadata[i] against signature row i: 0 valid, 1 s >= N, 2 an inconsistent
  // encoding; throws ErrVerification with them if any op fails
  std::vector<uint8_t> VerifyBatch(const std::vector<Bytes>& messages, const std::vector<Bytes>& metadata,
                                   const Bytes& sigs) const {
    const size_t n = messages.size();
    if (sigs.size() != n * KLen() || metadata.size() != n) throw ErrUnexpectedSize();
    Bytes msgs, meta;
    std::vector<uint64_t> off, moff;
    blindrsa::detail::pack(messages, &msgs, &off);
    blindrsa::detail::pack(metadata, &meta, &moff);
    std::vector<uint8_t> st(n);
    if (n) blindrsa::detail::check_call(call(msgs.data(), off.data(), meta.data(), moff.data(), sigs.data(), st.data(), n));
    for (uint8_t s : st)
      if (s) throw ErrVerification(st);
    return st;
  }
  void Verify(const Bytes& message, const Bytes& metadata, const Bytes& signature) const {  // pbrsa.go:244-251
    if (signature.size() != KLen()) throw ErrVerification();
    VerifyBatch({message}, {metadata}, signature);
  }

 private:
  int call(const uint8_t* msgs, const uint64_t* off, const uint8_t* meta, const uint64_t* moff, const uint8_t* sigs,
           uint8_t* st, size_t n) const {
    using blindrsa::detail::p;
    return cb200_pbrsa_verify(p(pk_.N), pk_.N.size(), msgs, off, meta, moff, sigs, st, n);
  }
  PublicKey pk_;
};
inline Signer NewSigner(const PrivateKey& sk) { return Signer(sk); }
inline Verifier NewVerifier(const PublicKey& pk) { return Verifier(pk); }
}  // namespace partiallyblindrsa

// Threshold RSA (the reference's tss/rsa, Shoup's protocol 1): a party's signature shares x^E mod N under its key
// share, E = 2 Delta s_i (or the share's cached twoDeltaSi, as KeyShare.Sign uses it), and the combination of k shares
// per op into the RSA signature (CombineSignShares after its share parameter checks).  Byte strings are big-endian;
// rows are kLen = ceil(bitlen(N) / 8) bytes back to back.  Served: N of 2048 to 4096 bits, an odd e with
// 3 <= e < 2^32, 2 <= players <= 64, threshold <= k <= 64 shares per op, u16 indices, E of at most
// bitlen(N) - 2 + bitlen(2 players!) bits.  Arguments outside these throw std::logic_error with the library's message.
namespace tssrsa {
struct TSSRSAError : Error {
  std::vector<uint8_t> status;  // per-op bytes of a failed batch
  explicit TSSRSAError(const std::string& m, std::vector<uint8_t> st = {}) : Error(m), status(std::move(st)) {}
};
struct ErrUnexpectedSize : TSSRSAError {
  ErrUnexpectedSize() : TSSRSAError("tssrsa: unexpected input size") {}
};
// status 1: an index 0 or a Lagrange coefficient that is not an integer (computeLambda)
struct ErrInvalidCalc : TSSRSAError {
  explicit ErrInvalidCalc(std::vector<uint8_t> st = {}) : TSSRSAError("tss/rsa: invalid calculation", std::move(st)) {}
};
// status 2: y^e mod N != x
struct ErrInternal : TSSRSAError {
  explicit ErrInternal(std::vector<uint8_t> st = {}) : TSSRSAError("rsa: internal error", std::move(st)) {}
};

struct PublicKey {
  Bytes N, E;
  size_t Size() const { return N.empty() ? 0 : cb200_brsa_modulus_bytes(N.data(), N.size()); }
};

// KeyShare.Sign on a batch: digests (n rows of kLen, reduced mod N as Exp does) -> the shares xi (n rows of kLen)
inline Bytes SignShareBatch(const PublicKey& pub, int players, const Bytes& E, const Bytes& digests) {
  const size_t k = pub.Size();
  uint8_t z = 0;
  auto call = [&](const uint8_t* in, uint8_t* out, size_t n) {
    blindrsa::detail::check_call(cb200_tssrsa_sign_share(blindrsa::detail::p(pub.N), pub.N.size(), players,
                                                         E.empty() ? &z : E.data(), E.size(), in, out, n));
  };
  if (!k) call(&z, &z, 0);  // a modulus outside the served range: the library's argument error
  if (!k || digests.size() % k) throw ErrUnexpectedSize();
  const size_t n = digests.size() / k;
  Bytes xi(n * k);
  call(n ? digests.data() : &z, n ? xi.data() : &z, n);
  return xi;
}

// CombineSignShares on a batch of n ops, each with its k indices (idx: n * k values), its k shares (xi: n rows of
// k kLen bytes) and its padded message (msgs: n rows of kLen) -> n signatures; throws ErrInvalidCalc if any op has
// status 1, else ErrInternal if any has status 2, with the status bytes (failed rows are zero)
inline Bytes CombineSignSharesBatch(const PublicKey& pub, int players, int threshold, int k,
                                    const std::vector<uint16_t>& idx, const Bytes& xi, const Bytes& msgs) {
  const size_t kl = pub.Size();
  const uint16_t zi = 0;
  uint8_t z = 0;
  auto call = [&](const uint16_t* ix, const uint8_t* x, const uint8_t* m, uint8_t* out, uint8_t* st, size_t n) {
    using blindrsa::detail::p;
    blindrsa::detail::check_call(
        cb200_tssrsa_combine(p(pub.N), pub.N.size(), p(pub.E), pub.E.size(), players, threshold, k, ix, x, m, out, st, n));
  };
  if (!kl) call(&zi, &z, &z, &z, &z, 0);  // a modulus outside the served range: the library's argument error
  if (!kl || k < 1 || msgs.size() % kl) throw ErrUnexpectedSize();
  const size_t n = msgs.size() / kl;
  if (idx.size() != n * (size_t)k || xi.size() != n * (size_t)k * kl) throw ErrUnexpectedSize();
  Bytes sig(n * kl);
  std::vector<uint8_t> st(n);
  call(n ? idx.data() : &zi, n ? xi.data() : &z, n ? msgs.data() : &z, n ? sig.data() : &z, n ? st.data() : &z, n);
  for (uint8_t s : st)
    if (s == 1) throw ErrInvalidCalc(st);
  for (uint8_t s : st)
    if (s == 2) throw ErrInternal(st);
  return sig;
}
}  // namespace tssrsa
// Prio3 aggregators (draft-irtf-cfrg-vdaf-14): the reference's vdaf/prio3 packages count, sum, sumvec, histogram and
// mhcv, aggregator side, on host buffers.  The constructors validate as the reference's New does and throw
// std::invalid_argument with the library's message.  Rows are the reference's wire encodings, one per report, back to
// back.  The batch calls return the per-report status bytes (1 an element >= p, 2 ErrJointRand, 4 ErrInvalidEval, 8
// ErrProofVerify; failed rows are zero); the per-report calls throw the error of the status instead.
namespace prio3 {
struct Prio3Error : Error {
  uint8_t status;
  Prio3Error(const std::string& m, uint8_t st) : Error(m), status(st) {}
};
#define CIRCL_PRIO3_ERR(name)                                        \
  struct name : Prio3Error {                                         \
    explicit name(uint8_t st) : Prio3Error("prio3: " #name, st) {} \
  };
CIRCL_PRIO3_ERR(ErrDecode)
CIRCL_PRIO3_ERR(ErrJointRand)
CIRCL_PRIO3_ERR(ErrInvalidEval)
CIRCL_PRIO3_ERR(ErrProofVerify)
#undef CIRCL_PRIO3_ERR

class Prio3 {
 public:
  const cb200_prio3_sizes& Params() const { return z_; }
  unsigned Shares() const { return cfg_.num_shares; }
  // n reports as aggregator aggID -> prep states and prep shares (n rows each)
  std::vector<uint8_t> PrepInitBatch(const Bytes& verifyKey, uint8_t aggID, const Bytes& nonces,
                                     const Bytes& publicShares, const Bytes& inputShares, Bytes* states,
                                     Bytes* shares) const {
    const size_t n = nonces.size() / 16;
    const size_t in = aggID ? z_.input_share_helper : z_.input_share_leader;
    if (verifyKey.size() != 32 || nonces.size() != 16 * n || inputShares.size() != in * n ||
        publicShares.size() != z_.public_share * n)
      throw std::invalid_argument("prio3: row sizes do not match the configuration");
    states->assign(n * z_.prep_state, 0);
    shares->assign(n * z_.prep_share, 0);
    std::vector<uint8_t> st(n);
    check(cb200_prio3_prep_init(&cfg_, verifyKey.data(), aggID, nonces.data(), ptr(publicShares), inputShares.data(),
                                states->data(), shares->data(), st.data(), n));
    return st;
  }
  // row i of prepShares: the Shares() prep shares of report i -> prep messages
  std::vector<uint8_t> PrepSharesToPrepBatch(const Bytes& prepShares, Bytes* msgs) const {
    const size_t row = cfg_.num_shares * z_.prep_share, n = prepShares.size() / row;
    if (prepShares.size() != n * row) throw std::invalid_argument("prio3: row sizes do not match the configuration");
    msgs->assign(n * z_.prep_msg, 0);
    std::vector<uint8_t> st(n);
    check(cb200_prio3_prep_shares_to_prep(&cfg_, prepShares.data(), ptr(*msgs), st.data(), n));
    return st;
  }
  std::vector<uint8_t> PrepNextBatch(const Bytes& states, const Bytes& msgs, Bytes* outShares) const {
    const size_t n = states.size() / z_.prep_state;
    if (states.size() != n * z_.prep_state || msgs.size() != n * z_.prep_msg)
      throw std::invalid_argument("prio3: row sizes do not match the configuration");
    outShares->assign(n * z_.out_share, 0);
    std::vector<uint8_t> st(n);
    check(cb200_prio3_prep_next(&cfg_, states.data(), ptr(msgs), outShares->data(), st.data(), n));
    return st;
  }
  // the agg share of the out shares whose status byte is 0 (all of them for an empty status)
  Bytes AggregateBatch(const Bytes& outShares, const std::vector<uint8_t>& status = {}) const {
    const size_t n = outShares.size() / z_.out_share;
    if (outShares.size() != n * z_.out_share || (!status.empty() && status.size() != n))
      throw std::invalid_argument("prio3: row sizes do not match the configuration");
    Bytes agg(z_.agg_share);
    check(cb200_prio3_aggregate(&cfg_, outShares.data(), status.empty() ? nullptr : status.data(), agg.data(), n));
    return agg;
  }
  // one report (prio3.go:245-403)
  void PrepInit(const Bytes& verifyKey, const Bytes& nonce, uint8_t aggID, const Bytes& publicShare,
                const Bytes& inputShare, Bytes* state, Bytes* share) const {
    throw_status(PrepInitBatch(verifyKey, aggID, nonce, publicShare, inputShare, state, share)[0]);
  }
  Bytes PrepSharesToPrep(const std::vector<Bytes>& prepShares) const {
    if (prepShares.size() != cfg_.num_shares) throw std::invalid_argument("prio3: invalid prep shares length");
    Bytes rows, msg;
    for (const Bytes& b : prepShares) rows.insert(rows.end(), b.begin(), b.end());
    throw_status(PrepSharesToPrepBatch(rows, &msg)[0]);
    return msg;
  }
  Bytes PrepNext(const Bytes& state, const Bytes& msg) const {
    Bytes out;
    throw_status(PrepNextBatch(state, msg, &out)[0]);
    return out;
  }
  Bytes AggregateInit() const { return Bytes(z_.agg_share); }
  void AggregateUpdate(Bytes* aggShare, const Bytes& outShare) const {
    *aggShare = AggregateBatch(merge_rows({*aggShare, outShare}));
  }
  // the sum of the agg shares, as integers (Decode of every circuit: one element for Count and Sum)
  std::vector<uint64_t> Unshard(const std::vector<Bytes>& aggShares, uint64_t numMeas) const {
    if (aggShares.size() != cfg_.num_shares) throw std::invalid_argument("prio3: invalid aggregate shares length");
    if (cfg_.kind == CB200_PRIO3_SUM) {
      const unsigned __int128 bound = (unsigned __int128)numMeas * cfg_.max_measurement;
      if (bound >= 0xffffffff00000001ull) throw std::invalid_argument("prio3: sum aggregate bound is not representable");
    }
    const Bytes s = AggregateBatch(merge_rows(aggShares));
    const size_t B = cfg_.kind <= CB200_PRIO3_SUM ? 8 : 16;
    std::vector<uint64_t> out(s.size() / B);
    for (size_t i = 0; i < out.size(); i++) {  // GetUint64: a Field128 element must fit in 64 bits
      uint64_t v = 0, hi = 0;
      for (int j = 0; j < 8; j++) v |= (uint64_t)s[B * i + j] << (8 * j);
      for (size_t j = 8; j < B; j++) hi |= s[B * i + j];
      if (hi) throw std::range_error("prio3: number of bits is not enough to represent the number");
      out[i] = v;
    }
    return out;
  }

 protected:
  Prio3(uint32_t kind, uint8_t shares, const Bytes& context) : ctx_(context) {
    cfg_ = cb200_prio3_config{};
    cfg_.kind = kind;
    cfg_.num_shares = shares;
  }
  void finish() {
    cfg_.context = ctx_.empty() ? nullptr : ctx_.data();
    cfg_.context_len = ctx_.size();
    if (cb200_prio3_get_sizes(&cfg_, &z_) != 0) throw std::invalid_argument(cb200_last_error());
  }
  cb200_prio3_config cfg_;

 private:
  static const uint8_t* ptr(const Bytes& b) { return b.empty() ? nullptr : b.data(); }
  static uint8_t* ptr(Bytes& b) { return b.empty() ? nullptr : b.data(); }
  static void check(int rc) {
    if (rc == CB200_ERR_ARG) throw std::invalid_argument(cb200_last_error());
    if (rc != 0) throw Error(cb200_last_error());
  }
  static void throw_status(uint8_t st) {
    if (st & 1) throw ErrDecode(st);
    if (st & 2) throw ErrJointRand(st);
    if (st & 4) throw ErrInvalidEval(st);
    if (st & 8) throw ErrProofVerify(st);
  }
  Bytes merge_rows(const std::vector<Bytes>& rows) const {
    Bytes all;
    for (const Bytes& b : rows) {
      if (b.size() != z_.agg_share) throw std::invalid_argument("prio3: agg share size");
      all.insert(all.end(), b.begin(), b.end());
    }
    return all;
  }
  Bytes ctx_;
  cb200_prio3_sizes z_{};
};

struct Count : Prio3 {
  Count(uint8_t numShares, const Bytes& context) : Prio3(CB200_PRIO3_COUNT, numShares, context) { finish(); }
};
struct Sum : Prio3 {
  Sum(uint8_t numShares, uint64_t maxMeasurement, const Bytes& context) : Prio3(CB200_PRIO3_SUM, numShares, context) {
    cfg_.max_measurement = maxMeasurement;
    finish();
  }
};
struct SumVec : Prio3 {
  SumVec(uint8_t numShares, uint64_t length, uint64_t bits, uint64_t chunkLength, const Bytes& context)
      : Prio3(CB200_PRIO3_SUMVEC, numShares, context) {
    cfg_.length = length;
    cfg_.bits = bits;
    cfg_.chunk_length = chunkLength;
    finish();
  }
};
struct Histogram : Prio3 {
  Histogram(uint8_t numShares, uint64_t length, uint64_t chunkLength, const Bytes& context)
      : Prio3(CB200_PRIO3_HISTOGRAM, numShares, context) {
    cfg_.length = length;
    cfg_.chunk_length = chunkLength;
    finish();
  }
};
struct MultiHotCountVec : Prio3 {
  MultiHotCountVec(uint8_t numShares, uint64_t length, uint64_t maxWeight, uint64_t chunkLength, const Bytes& context)
      : Prio3(CB200_PRIO3_MULTIHOT, numShares, context) {
    cfg_.length = length;
    cfg_.max_weight = maxWeight;
    cfg_.chunk_length = chunkLength;
    finish();
  }
};
}  // namespace prio3
}  // namespace circl
