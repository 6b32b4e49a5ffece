//go:build cuda && cgo

// Package frodo640shakecuda backs the kem/schemes entry "FrodoKEM-640-SHAKE" (kem/frodo/frodo640shake) with the cb200
// engine.  DeriveKeyPair, the encapsulations and Decapsulate run on the GPU as batches of one; key parsing and
// marshalling delegate to CIRCL's own scheme.  EncapsulateBatch and DecapsulateBatch are the entry points that make a
// GPU worthwhile: with one key for the whole batch, A and H(pk) are computed once per call and S'A runs as one
// tensor-core GEMM.
//
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package frodo640shakecuda

import (
	cryptoRand "crypto/rand"

	"github.com/cloudflare/circl/kem"
	"github.com/cloudflare/circl/kem/frodo/frodo640shake"

	"example.com/circl_b200/go/cb200"
)

type scheme struct{ kem.Scheme } // embeds CIRCL's stateless singleton (frodo.go:405-410)

var sch kem.Scheme = &scheme{frodo640shake.Scheme()}

// Scheme returns the GPU-backed FrodoKEM-640-SHAKE scheme; Name() is unchanged so kem/schemes.ByName keeps working.
func Scheme() kem.Scheme { return sch }

func mustMarshal(k interface{ MarshalBinary() ([]byte, error) }) []byte {
	b, err := k.MarshalBinary()
	if err != nil {
		panic(err)
	}
	return b
}

func (s *scheme) DeriveKeyPair(seed []byte) (kem.PublicKey, kem.PrivateKey) {
	if len(seed) != frodo640shake.KeySeedSize {
		panic(kem.ErrSeedSize) // frodo.go:480-483
	}
	pk, sk := make([]byte, frodo640shake.PublicKeySize), make([]byte, frodo640shake.PrivateKeySize)
	if err := cb200.Frodo640SHAKEKeygen(seed, pk, sk); err != nil {
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

func (s *scheme) GenerateKeyPair() (kem.PublicKey, kem.PrivateKey, error) {
	var seed [frodo640shake.KeySeedSize]byte
	if _, err := cryptoRand.Read(seed[:]); err != nil {
		return nil, nil, err
	}
	pk, sk := s.DeriveKeyPair(seed[:])
	return pk, sk, nil
}

// the reference's order: the seed length, then the key's type (frodo.go:499-515)
func (s *scheme) EncapsulateDeterministically(pk kem.PublicKey, seed []byte) (ct, ss []byte, err error) {
	if len(seed) != frodo640shake.EncapsulationSeedSize {
		return nil, nil, kem.ErrSeedSize
	}
	pub, ok := pk.(*frodo640shake.PublicKey)
	if !ok {
		return nil, nil, kem.ErrTypeMismatch
	}
	ct, ss = make([]byte, frodo640shake.CiphertextSize), make([]byte, frodo640shake.SharedKeySize)
	if err = cb200.Frodo640SHAKEEncaps(mustMarshal(pub), seed, ct, ss); err != nil {
		return nil, nil, err
	}
	return ct, ss, nil
}

func (s *scheme) Encapsulate(pk kem.PublicKey) (ct, ss []byte, err error) {
	if _, ok := pk.(*frodo640shake.PublicKey); !ok {
		return nil, nil, kem.ErrTypeMismatch // frodo.go:491-494
	}
	var seed [frodo640shake.EncapsulationSeedSize]byte
	if _, err = cryptoRand.Read(seed[:]); err != nil {
		return nil, nil, err
	}
	return s.EncapsulateDeterministically(pk, seed[:])
}

// the reference's order: the ciphertext length, then the key's type (frodo.go:517-529)
func (s *scheme) Decapsulate(sk kem.PrivateKey, ct []byte) ([]byte, error) {
	if len(ct) != frodo640shake.CiphertextSize {
		return nil, kem.ErrCiphertextSize
	}
	priv, ok := sk.(*frodo640shake.PrivateKey)
	if !ok {
		return nil, kem.ErrTypeMismatch
	}
	ss := make([]byte, frodo640shake.SharedKeySize)
	if err := cb200.Frodo640SHAKEDecaps(mustMarshal(priv), ct, ss); err != nil {
		return nil, err
	}
	return ss, nil
}

// EncapsulateBatch encapsulates len(seeds)/16 times.  packedKeys holds either one 9616-byte key (shared by the batch)
// or one key per operation.  Errors follow kem.Scheme: kem.ErrSeedSize / kem.ErrPubKeySize.
func EncapsulateBatch(packedKeys, seeds []byte) (cts, sss []byte, err error) {
	if len(seeds)%frodo640shake.EncapsulationSeedSize != 0 {
		return nil, nil, kem.ErrSeedSize
	}
	n := len(seeds) / frodo640shake.EncapsulationSeedSize
	if len(packedKeys) != frodo640shake.PublicKeySize && len(packedKeys) != n*frodo640shake.PublicKeySize {
		return nil, nil, kem.ErrPubKeySize
	}
	cts, sss = make([]byte, n*frodo640shake.CiphertextSize), make([]byte, n*frodo640shake.SharedKeySize)
	return cts, sss, cb200.Frodo640SHAKEEncaps(packedKeys, seeds, cts, sss)
}

// DecapsulateBatch decapsulates len(cts)/9720 ciphertexts with one packed 19888-byte key (shared by the batch: the
// server case) or one key per operation.  Errors: kem.ErrCiphertextSize / kem.ErrPrivKeySize.
func DecapsulateBatch(packedKeys, cts []byte) ([]byte, error) {
	if len(cts)%frodo640shake.CiphertextSize != 0 {
		return nil, kem.ErrCiphertextSize
	}
	n := len(cts) / frodo640shake.CiphertextSize
	if len(packedKeys) != frodo640shake.PrivateKeySize && len(packedKeys) != n*frodo640shake.PrivateKeySize {
		return nil, kem.ErrPrivKeySize
	}
	sss := make([]byte, n*frodo640shake.SharedKeySize)
	return sss, cb200.Frodo640SHAKEDecaps(packedKeys, cts, sss)
}
