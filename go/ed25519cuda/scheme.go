//go:build cuda && cgo

// Package ed25519cuda registers "Ed25519" backed by the cb200 engine, keeping sign.Scheme (sign/sign.go:48-94)
// intact: Sign / Verify / DeriveKey go through the GPU (batch of one), everything else (marshalling, crypto.Signer
// plumbing) delegates to CIRCL's own ed25519 scheme (sign/ed25519/signapi.go); SignBatch and VerifyBatch are the entry
// points that make a GPU worthwhile.
//
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package ed25519cuda

import (
	"github.com/cloudflare/circl/sign"
	"github.com/cloudflare/circl/sign/ed25519"

	"example.com/circl_b200/go/cb200"
)

type scheme struct{ sign.Scheme } // embeds CIRCL's stateless singleton (signapi.go)

var sch sign.Scheme = &scheme{ed25519.Scheme()}

// Scheme returns the GPU-backed Ed25519 scheme; Name() is unchanged so sign/schemes.ByName keeps working.
func Scheme() sign.Scheme { return sch }

func (s *scheme) DeriveKey(seed []byte) (sign.PublicKey, sign.PrivateKey) {
	if len(seed) != ed25519.SeedSize {
		panic(sign.ErrSeedSize)
	}
	pk, sk := make([]byte, ed25519.PublicKeySize), make([]byte, ed25519.PrivateKeySize)
	if err := cb200.Ed25519KeyGen(seed, pk, sk); err != nil {
		panic(err)
	}
	return ed25519.PublicKey(pk), ed25519.PrivateKey(sk)
}

func (s *scheme) Sign(sk sign.PrivateKey, message []byte, opts *sign.SignatureOpts) []byte {
	priv, ok := sk.(ed25519.PrivateKey)
	if !ok {
		panic(sign.ErrTypeMismatch) // signapi.go: Sign
	}
	if opts != nil && opts.Context != "" {
		panic(sign.ErrContextNotSupported)
	}
	if len(priv) != ed25519.PrivateKeySize {
		panic("ed25519: bad private key length") // ed25519.go:226-228
	}
	sig := make([]byte, ed25519.SignatureSize)
	if err := cb200.Ed25519SignBatch(priv, true, [][]byte{message}, sig); err != nil {
		panic(err)
	}
	return sig
}

func (s *scheme) Verify(pk sign.PublicKey, message, signature []byte, opts *sign.SignatureOpts) bool {
	pub, ok := pk.(ed25519.PublicKey)
	if !ok {
		panic(sign.ErrTypeMismatch)
	}
	if opts != nil && opts.Context != "" {
		panic(sign.ErrContextNotSupported)
	}
	if len(pub) != ed25519.PublicKeySize || len(signature) != ed25519.SignatureSize {
		return false // ed25519.go:330-334
	}
	res := make([]bool, 1)
	if err := cb200.Ed25519VerifyBatch(pub, true, [][]byte{message}, signature, res); err != nil {
		panic(err)
	}
	return res[0]
}

// SignBatch signs every message with its own key (len(sks) == n*64) or one shared key.
func SignBatch(sks []byte, msgs [][]byte) ([]byte, error) {
	shared := len(sks) == ed25519.PrivateKeySize
	if !shared && len(sks) != len(msgs)*ed25519.PrivateKeySize {
		return nil, sign.ErrTypeMismatch
	}
	sigs := make([]byte, len(msgs)*ed25519.SignatureSize)
	return sigs, cb200.Ed25519SignBatch(sks, shared, msgs, sigs)
}

// VerifyBatch verifies n signatures (len(sigs) == n*64) under their own keys (len(pks) == n*32) or one shared key.
func VerifyBatch(pks []byte, msgs [][]byte, sigs []byte) ([]bool, error) {
	shared := len(pks) == ed25519.PublicKeySize
	if (!shared && len(pks) != len(msgs)*ed25519.PublicKeySize) || len(sigs) != len(msgs)*ed25519.SignatureSize {
		return nil, sign.ErrTypeMismatch
	}
	ok := make([]bool, len(msgs))
	return ok, cb200.Ed25519VerifyBatch(pks, shared, msgs, sigs, ok)
}
