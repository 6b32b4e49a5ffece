//go:build cuda && cgo

// Package hpkecuda backs the kem/schemes entries "HPKE_KEM_X25519_HKDF_SHA256", "HPKE_KEM_X448_HKDF_SHA512",
// "HPKE_KEM_P256_HKDF_SHA256", "HPKE_KEM_P384_HKDF_SHA384" and "HPKE_KEM_P521_HKDF_SHA512" (hpke/algs.go:248-277) with
// the cb200 engine.  All are kem.AuthScheme (kem/kem.go:84-90): DeriveKeyPair, the
// (authenticated) encapsulations and decapsulations run on the GPU as batches of one, everything else (key parsing,
// GenerateKeyPair, marshalling) delegates to CIRCL's own scheme.  EncapsulateBatch and DecapsulateBatch are the entry
// points that make a GPU worthwhile.
//
// hpke.Suite keeps calling CIRCL's own KEM: only kem/schemes callers reach these schemes (see INTEGRATION.md).
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package hpkecuda

import (
	"crypto/rand"

	"github.com/cloudflare/circl/hpke"
	"github.com/cloudflare/circl/kem"

	"example.com/circl_b200/go/cb200"
)

type scheme struct {
	kem.AuthScheme // CIRCL's DHKEM (hpke/xkem.go, hpke/shortkem.go)
	id             int
}

var (
	x25519 = &scheme{hpke.KEM_X25519_HKDF_SHA256.Scheme().(kem.AuthScheme), cb200.HPKEX25519HKDFSHA256}
	x448   = &scheme{hpke.KEM_X448_HKDF_SHA512.Scheme().(kem.AuthScheme), cb200.HPKEX448HKDFSHA512}
	p256   = &scheme{hpke.KEM_P256_HKDF_SHA256.Scheme().(kem.AuthScheme), cb200.HPKEP256HKDFSHA256}
	p384   = &scheme{hpke.KEM_P384_HKDF_SHA384.Scheme().(kem.AuthScheme), cb200.HPKEP384HKDFSHA384}
	p521   = &scheme{hpke.KEM_P521_HKDF_SHA512.Scheme().(kem.AuthScheme), cb200.HPKEP521HKDFSHA512}
)

// X25519, X448, P256, P384 and P521 return the GPU-backed schemes; Name() is unchanged so kem/schemes.ByName keeps
// working.
func X25519() kem.AuthScheme { return x25519 }
func X448() kem.AuthScheme   { return x448 }
func P256() kem.AuthScheme   { return p256 }
func P384() kem.AuthScheme   { return p384 }
func P521() kem.AuthScheme   { return p521 }

// isNIST: the NIST curves have entry points of their own and validate points and scalars
func (s *scheme) isNIST() bool {
	return s.id == cb200.HPKEP256HKDFSHA256 || s.id == cb200.HPKEP384HKDFSHA384 || s.id == cb200.HPKEP521HKDFSHA512
}

// The engine calls of a scheme.
func (s *scheme) keygen(seeds, pk, sk []byte) error {
	switch s.id {
	case cb200.HPKEP256HKDFSHA256:
		return cb200.HPKEP256Keygen(seeds, pk, sk)
	case cb200.HPKEP384HKDFSHA384:
		return cb200.HPKEP384Keygen(seeds, pk, sk)
	case cb200.HPKEP521HKDFSHA512:
		return cb200.HPKEP521Keygen(seeds, pk, sk)
	}
	return cb200.HPKEKeygen(s.id, seeds, pk, sk)
}
func (s *scheme) encaps(pkR, skS, seeds, enc, ss []byte, ok []bool) error {
	switch s.id {
	case cb200.HPKEP256HKDFSHA256:
		return s.mapErr(cb200.HPKEP256Encaps(pkR, skS, seeds, enc, ss, ok))
	case cb200.HPKEP384HKDFSHA384:
		return s.mapErr(cb200.HPKEP384Encaps(pkR, skS, seeds, enc, ss, ok))
	case cb200.HPKEP521HKDFSHA512:
		return s.mapErr(cb200.HPKEP521Encaps(pkR, skS, seeds, enc, ss, ok))
	}
	return s.mapErr(cb200.HPKEEncaps(s.id, pkR, skS, seeds, enc, ss, ok))
}
func (s *scheme) decaps(skR, enc, pkS, ss []byte, ok []bool) error {
	switch s.id {
	case cb200.HPKEP256HKDFSHA256:
		return s.mapErr(cb200.HPKEP256Decaps(skR, enc, pkS, ss, ok))
	case cb200.HPKEP384HKDFSHA384:
		return s.mapErr(cb200.HPKEP384Decaps(skR, enc, pkS, ss, ok))
	case cb200.HPKEP521HKDFSHA512:
		return s.mapErr(cb200.HPKEP521Decaps(skR, enc, pkS, ss, ok))
	}
	return s.mapErr(cb200.HPKEDecaps(s.id, skR, enc, pkS, ss, ok))
}

func mustMarshal(k interface{ MarshalBinary() ([]byte, error) }) []byte {
	b, err := k.MarshalBinary()
	if err != nil {
		panic(err)
	}
	return b
}

// mapErr maps the engine's per-batch failures to the reference's errors: for X25519 / X448 a low-order point is
// hpke.ErrInvalidKEMSharedSecret (hpke/hpke.go:280); for the NIST curves an invalid point or scalar is
// hpke.ErrInvalidKEMPublicKey / ErrInvalidKEMPrivateKey (hpke/hpke.go:278-279)
func (s *scheme) mapErr(err error) error {
	switch {
	case err == cb200.ErrPubKey && s.isNIST():
		return hpke.ErrInvalidKEMPublicKey
	case err == cb200.ErrPrivKey && s.isNIST():
		return hpke.ErrInvalidKEMPrivateKey
	case err == cb200.ErrPubKey:
		return hpke.ErrInvalidKEMSharedSecret
	}
	return err
}

func (s *scheme) checkPub(pk kem.PublicKey) []byte {
	if pk == nil || pk.Scheme().Name() != s.Name() {
		panic(kem.ErrTypeMismatch) // the reference's type assertion in calcDH (xkem.go:28-29)
	}
	return mustMarshal(pk)
}

func (s *scheme) checkPriv(sk kem.PrivateKey) []byte {
	if sk == nil || sk.Scheme().Name() != s.Name() {
		panic(kem.ErrTypeMismatch)
	}
	return mustMarshal(sk)
}

func (s *scheme) DeriveKeyPair(seed []byte) (kem.PublicKey, kem.PrivateKey) {
	if len(seed) != s.SeedSize() {
		panic(kem.ErrSeedSize) // xkem.go:60-62
	}
	pk, sk := make([]byte, s.PublicKeySize()), make([]byte, s.PrivateKeySize())
	if err := s.keygen(seed, pk, sk); err != nil {
		panic(err)
	}
	pub, err := s.UnmarshalBinaryPublicKey(pk)
	if err != nil {
		panic(err)
	}
	priv, err := s.UnmarshalBinaryPrivateKey(sk)
	if err != nil {
		panic(err)
	}
	return pub, priv
}

func (s *scheme) encap(pkr kem.PublicKey, sks kem.PrivateKey, seed []byte) (ct, ss []byte, err error) {
	if len(seed) != s.SeedSize() {
		panic(kem.ErrSeedSize) // DeriveKeyPair of the ephemeral key (kembase.go:166)
	}
	var skS []byte
	if sks != nil {
		skS = s.checkPriv(sks)
	}
	ct, ss = make([]byte, s.CiphertextSize()), make([]byte, s.SharedKeySize())
	if err = s.encaps(s.checkPub(pkr), skS, seed, ct, ss, nil); err != nil {
		return nil, nil, err
	}
	return ct, ss, nil
}

func (s *scheme) decap(skr kem.PrivateKey, ct []byte, pks kem.PublicKey) ([]byte, error) {
	if len(ct) != s.PublicKeySize() {
		return nil, kem.ErrPubKeySize // ct is parsed as a public key (kembase.go:222, xkem.go:95-101)
	}
	if s.isNIST() { // shortkem.go:115-130 also checks the point
		if _, err := s.AuthScheme.UnmarshalBinaryPublicKey(ct); err != nil {
			return nil, err
		}
	}
	var pkS []byte
	if pks != nil {
		pkS = s.checkPub(pks)
	}
	ss := make([]byte, s.SharedKeySize())
	if err := s.decaps(s.checkPriv(skr), ct, pkS, ss, nil); err != nil {
		return nil, err
	}
	return ss, nil
}

func (s *scheme) EncapsulateDeterministically(pkr kem.PublicKey, seed []byte) (ct, ss []byte, err error) {
	return s.encap(pkr, nil, seed)
}

func (s *scheme) Decapsulate(skr kem.PrivateKey, ct []byte) ([]byte, error) { return s.decap(skr, ct, nil) }

func (s *scheme) AuthEncapsulateDeterministically(pkr kem.PublicKey, sks kem.PrivateKey, seed []byte) (ct, ss []byte,
	err error) {
	return s.encap(pkr, sks, seed)
}

func (s *scheme) AuthDecapsulate(skr kem.PrivateKey, ct []byte, pks kem.PublicKey) ([]byte, error) {
	return s.decap(skr, ct, pks)
}

// The embedded scheme's Encapsulate / AuthEncapsulate would call its own deterministic variants: draw the seed here.
func (s *scheme) Encapsulate(pkr kem.PublicKey) (ct, ss []byte, err error) {
	seed := make([]byte, s.SeedSize())
	if _, err = rand.Read(seed); err != nil {
		return nil, nil, err
	}
	return s.encap(pkr, nil, seed)
}

func (s *scheme) AuthEncapsulate(pkr kem.PublicKey, sks kem.PrivateKey) (ct, ss []byte, err error) {
	seed := make([]byte, s.SeedSize())
	if _, err = rand.Read(seed); err != nil {
		return nil, nil, err
	}
	return s.encap(pkr, sks, seed)
}

// EncapsulateBatch encapsulates len(seeds)/N times against one packed pkR (N bytes) or one per operation; skS (nil for
// plain encapsulation) likewise.  ok[i] (may be nil) is false for the operations that failed.
func EncapsulateBatch(s kem.AuthScheme, pkR, skS, seeds []byte, ok []bool) (enc, ss []byte, err error) {
	g := s.(*scheme)
	n := len(seeds) / g.SeedSize()
	enc, ss = make([]byte, n*g.CiphertextSize()), make([]byte, n*g.SharedKeySize())
	return enc, ss, g.encaps(pkR, skS, seeds, enc, ss, ok)
}

// DecapsulateBatch decapsulates len(enc)/N encapsulations with one packed skR (its public key is computed once: the
// gateway case) or one per operation; pkS (nil for plain decapsulation) likewise.
func DecapsulateBatch(s kem.AuthScheme, skR, enc, pkS []byte, ok []bool) ([]byte, error) {
	g := s.(*scheme)
	ss := make([]byte, len(enc)/g.CiphertextSize()*g.SharedKeySize())
	return ss, g.decaps(skR, enc, pkS, ss, ok)
}
