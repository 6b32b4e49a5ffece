//go:build cuda && cgo

// Package eddilithium3cuda registers "Ed448-Dilithium3" backed by the cb200 engine, keeping sign.Scheme
// (sign/sign.go:48-94) intact: Sign / Verify / DeriveKey go through the GPU (batch of one), everything else
// delegates to CIRCL's own eddilithium3 scheme (sign/eddilithium3/signapi.go); SignBatch and VerifyBatch are the
// entry points that make a GPU worthwhile.
//
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package eddilithium3cuda

import (
	"github.com/cloudflare/circl/sign"
	"github.com/cloudflare/circl/sign/eddilithium3"

	"example.com/circl_b200/go/cb200"
)

type scheme struct{ sign.Scheme } // embeds CIRCL's stateless singleton (signapi.go)

var sch sign.Scheme = &scheme{eddilithium3.Scheme()}

// Scheme returns the GPU-backed Ed448-Dilithium3 scheme; Name() is unchanged so sign/schemes.ByName keeps working.
func Scheme() sign.Scheme { return sch }

func (s *scheme) DeriveKey(seed []byte) (sign.PublicKey, sign.PrivateKey) {
	if len(seed) != eddilithium3.SeedSize {
		panic(sign.ErrSeedSize)
	}
	pk, sk := make([]byte, eddilithium3.PublicKeySize), make([]byte, eddilithium3.PrivateKeySize)
	if err := cb200.EdDilithium3KeyGen(seed, pk, sk); err != nil {
		panic(err)
	}
	pub, _ := s.UnmarshalBinaryPublicKey(pk)
	priv, _ := s.UnmarshalBinaryPrivateKey(sk)
	return pub, priv
}

func (s *scheme) Sign(sk sign.PrivateKey, message []byte, opts *sign.SignatureOpts) []byte {
	priv, ok := sk.(*eddilithium3.PrivateKey)
	if !ok {
		panic(sign.ErrTypeMismatch)
	}
	if opts != nil && opts.Context != "" {
		panic(sign.ErrContextNotSupported)
	}
	packed, _ := priv.MarshalBinary()
	sig := make([]byte, eddilithium3.SignatureSize)
	if err := cb200.EdDilithium3SignBatch(packed, true, [][]byte{message}, sig); err != nil {
		panic(err)
	}
	return sig
}

func (s *scheme) Verify(pk sign.PublicKey, message, signature []byte, opts *sign.SignatureOpts) bool {
	pub, ok := pk.(*eddilithium3.PublicKey)
	if !ok {
		panic(sign.ErrTypeMismatch)
	}
	if opts != nil && opts.Context != "" {
		panic(sign.ErrContextNotSupported)
	}
	if len(signature) != eddilithium3.SignatureSize {
		return false // eddilithium.go:97-99
	}
	packed, _ := pub.MarshalBinary()
	res := make([]bool, 1)
	if err := cb200.EdDilithium3VerifyBatch(packed, true, [][]byte{message}, signature, res); err != nil {
		panic(err)
	}
	return res[0]
}

// SignBatch signs every message with its own packed key (len(sks) == n*4057) or one shared key.
func SignBatch(sks []byte, msgs [][]byte) ([]byte, error) {
	shared := len(sks) == eddilithium3.PrivateKeySize
	if !shared && len(sks) != len(msgs)*eddilithium3.PrivateKeySize {
		return nil, sign.ErrTypeMismatch
	}
	sigs := make([]byte, len(msgs)*eddilithium3.SignatureSize)
	return sigs, cb200.EdDilithium3SignBatch(sks, shared, msgs, sigs)
}

// VerifyBatch verifies n signatures (len(sigs) == n*3407) under their own keys (len(pks) == n*2009) or one shared key.
func VerifyBatch(pks []byte, msgs [][]byte, sigs []byte) ([]bool, error) {
	shared := len(pks) == eddilithium3.PublicKeySize
	if (!shared && len(pks) != len(msgs)*eddilithium3.PublicKeySize) || len(sigs) != len(msgs)*eddilithium3.SignatureSize {
		return nil, sign.ErrTypeMismatch
	}
	ok := make([]bool, len(msgs))
	return ok, cb200.EdDilithium3VerifyBatch(pks, shared, msgs, sigs, ok)
}
