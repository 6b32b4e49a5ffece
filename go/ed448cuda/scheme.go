//go:build cuda && cgo

// Package ed448cuda registers "Ed448" backed by the cb200 engine, keeping sign.Scheme (sign/sign.go:48-94) intact:
// Sign / Verify / DeriveKey go through the GPU (batch of one), everything else (marshalling, crypto.Signer plumbing)
// delegates to CIRCL's own ed448 scheme (sign/ed448/signapi.go); SignBatch and VerifyBatch are the entry points that
// make a GPU worthwhile.  Ed448 takes a context string (SupportsContext() is true).
//
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package ed448cuda

import (
	"github.com/cloudflare/circl/sign"
	"github.com/cloudflare/circl/sign/ed448"

	"example.com/circl_b200/go/cb200"
)

type scheme struct{ sign.Scheme } // embeds CIRCL's stateless singleton (signapi.go)

var sch sign.Scheme = &scheme{ed448.Scheme()}

// Scheme returns the GPU-backed Ed448 scheme; Name() is unchanged so sign/schemes.ByName keeps working.
func Scheme() sign.Scheme { return sch }

func (s *scheme) DeriveKey(seed []byte) (sign.PublicKey, sign.PrivateKey) {
	if len(seed) != ed448.SeedSize {
		panic(sign.ErrSeedSize)
	}
	pk, sk := make([]byte, ed448.PublicKeySize), make([]byte, ed448.PrivateKeySize)
	if err := cb200.Ed448KeyGen(seed, pk, sk); err != nil {
		panic(err)
	}
	return ed448.PublicKey(pk), ed448.PrivateKey(sk)
}

func (s *scheme) Sign(sk sign.PrivateKey, message []byte, opts *sign.SignatureOpts) []byte {
	priv, ok := sk.(ed448.PrivateKey)
	if !ok {
		panic(sign.ErrTypeMismatch) // signapi.go: Sign
	}
	ctx := ""
	if opts != nil {
		ctx = opts.Context
	}
	if len(ctx) > ed448.ContextMaxSize {
		panic(sign.ErrContextTooLong) // ed448.go:208-210 panics on a long context
	}
	if len(priv) != ed448.PrivateKeySize {
		panic("ed448: bad private key length")
	}
	sig := make([]byte, ed448.SignatureSize)
	if err := cb200.Ed448SignBatch(priv, true, [][]byte{message}, []byte(ctx), sig); err != nil {
		panic(err)
	}
	return sig
}

func (s *scheme) Verify(pk sign.PublicKey, message, signature []byte, opts *sign.SignatureOpts) bool {
	pub, ok := pk.(ed448.PublicKey)
	if !ok {
		panic(sign.ErrTypeMismatch)
	}
	ctx := ""
	if opts != nil {
		ctx = opts.Context
	}
	if len(pub) != ed448.PublicKeySize || len(signature) != ed448.SignatureSize || len(ctx) > ed448.ContextMaxSize {
		return false // ed448.go:295-300
	}
	res := make([]bool, 1)
	if err := cb200.Ed448VerifyBatch(pub, true, [][]byte{message}, []byte(ctx), signature, res); err != nil {
		panic(err)
	}
	return res[0]
}

// SignBatch signs every message with its own key (len(sks) == n*114) or one shared key, under one context.
func SignBatch(sks []byte, msgs [][]byte, ctx []byte) ([]byte, error) {
	shared := len(sks) == ed448.PrivateKeySize
	if !shared && len(sks) != len(msgs)*ed448.PrivateKeySize {
		return nil, sign.ErrTypeMismatch
	}
	if len(ctx) > ed448.ContextMaxSize {
		return nil, sign.ErrContextTooLong
	}
	sigs := make([]byte, len(msgs)*ed448.SignatureSize)
	return sigs, cb200.Ed448SignBatch(sks, shared, msgs, ctx, sigs)
}

// VerifyBatch verifies n signatures (len(sigs) == n*114) under their own keys (len(pks) == n*57) or one shared key.
func VerifyBatch(pks []byte, msgs [][]byte, ctx []byte, sigs []byte) ([]bool, error) {
	shared := len(pks) == ed448.PublicKeySize
	if (!shared && len(pks) != len(msgs)*ed448.PublicKeySize) || len(sigs) != len(msgs)*ed448.SignatureSize {
		return nil, sign.ErrTypeMismatch
	}
	ok := make([]bool, len(msgs))
	return ok, cb200.Ed448VerifyBatch(pks, shared, msgs, ctx, sigs, ok)
}
