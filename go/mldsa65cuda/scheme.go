//go:build cuda && cgo

// Package mldsa65cuda registers "ML-DSA-65" backed by the cb200 engine, keeping sign.Scheme
// (sign/sign.go:48-94) intact: Sign / Verify / DeriveKey go through the GPU (batch of one), everything
// else (marshalling, crypto.Signer plumbing) delegates to CIRCL's own mldsa65 scheme; SignBatch and
// VerifyBatch are the entry points that make a GPU worthwhile.
//
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package mldsa65cuda

import (
	"github.com/cloudflare/circl/sign"
	"github.com/cloudflare/circl/sign/mldsa/mldsa65"

	"example.com/circl_b200/go/cb200"
)

type scheme struct{ sign.Scheme } // embeds CIRCL's stateless singleton (dilithium.go:258)

var sch sign.Scheme = &scheme{mldsa65.Scheme()}

// Scheme returns the GPU-backed ML-DSA-65 scheme; Name() is unchanged so sign/schemes.ByName keeps working.
func Scheme() sign.Scheme { return sch }

func (s *scheme) Sign(sk sign.PrivateKey, message []byte, opts *sign.SignatureOpts) []byte {
	priv, ok := sk.(*mldsa65.PrivateKey)
	if !ok {
		panic(sign.ErrTypeMismatch) // dilithium.go:290-293
	}
	var ctx []byte
	if opts != nil && opts.Context != "" {
		ctx = []byte(opts.Context)
	}
	if len(ctx) > 255 {
		panic(sign.ErrContextTooLong)
	}
	packed, _ := priv.MarshalBinary()
	sig := make([]byte, mldsa65.SignatureSize)
	if err := cb200.MLDSA65Sign(packed, true, [][]byte{message}, ctx, nil, sig); err != nil {
		panic(err) // the reference panics if 576 attempts are exhausted (internal/dilithium.go:372-377)
	}
	return sig
}

// SignBatch signs every message with its own key (len(sks) == n*4032) or one shared key.
func SignBatch(sks []byte, msgs [][]byte, ctx []byte) ([]byte, error) {
	if len(ctx) > 255 {
		return nil, sign.ErrContextTooLong
	}
	shared := len(sks) == mldsa65.PrivateKeySize
	if !shared && len(sks) != len(msgs)*mldsa65.PrivateKeySize {
		return nil, sign.ErrTypeMismatch
	}
	sigs := make([]byte, len(msgs)*mldsa65.SignatureSize)
	return sigs, cb200.MLDSA65Sign(sks, shared, msgs, ctx, nil, sigs)
}
