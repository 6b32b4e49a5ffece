//go:build cuda && cgo

// Package xwingcuda backs kem/xwing's scheme (kem/xwing/scheme.go:1-140) with the cb200 engine.  As in
// mlkem768cuda, everything off the accelerated path delegates to CIRCL's own singleton; the deterministic
// encapsulation is a batch of one and EncapsulateBatch is the entry point that makes a GPU worthwhile.  The
// same pattern applies to kem/hybrid's X25519MLKEM768 with cb200.HybridEncaps (64-byte shared secrets).
//
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package xwingcuda

import (
	"github.com/cloudflare/circl/kem"
	"github.com/cloudflare/circl/kem/xwing"

	"example.com/circl_b200/go/cb200"
)

type scheme struct{ kem.Scheme }

var sch kem.Scheme = &scheme{xwing.Scheme()}

// Scheme returns the GPU-backed X-Wing scheme; Name() stays "X-Wing" (kem/schemes/schemes.go:54).
func Scheme() kem.Scheme { return sch }

func (s *scheme) EncapsulateDeterministically(pk kem.PublicKey, seed []byte) (ct, ss []byte, err error) {
	if len(seed) != xwing.EncapsulationSeedSize {
		return nil, nil, kem.ErrSeedSize // scheme.go:96-98
	}
	pub, ok := pk.(*xwing.PublicKey)
	if !ok {
		return nil, nil, kem.ErrTypeMismatch // scheme.go:91-94
	}
	var packed [xwing.PublicKeySize]byte
	pub.Pack(packed[:])
	ct = make([]byte, xwing.CiphertextSize)
	ss = make([]byte, xwing.SharedKeySize)
	if err = cb200.XWingEncaps(packed[:], true, seed, ct, ss); err == cb200.ErrPubKey {
		err = kem.ErrPubKey // the ML-KEM-768 half failed the FIPS 203 modulus check (xwing.go:173-177)
	}
	return
}

// EncapsulateBatch encapsulates len(seeds)/64 times against one packed key (len 1216) or one key per operation.
func EncapsulateBatch(packedKeys, seeds []byte) (cts, sss []byte, err error) {
	if len(seeds)%xwing.EncapsulationSeedSize != 0 {
		return nil, nil, kem.ErrSeedSize
	}
	n := len(seeds) / xwing.EncapsulationSeedSize
	shared := len(packedKeys) == xwing.PublicKeySize
	if !shared && len(packedKeys) != n*xwing.PublicKeySize {
		return nil, nil, kem.ErrPubKeySize
	}
	cts = make([]byte, n*xwing.CiphertextSize)
	sss = make([]byte, n*xwing.SharedKeySize)
	if err = cb200.XWingEncaps(packedKeys, shared, seeds, cts, sss); err == cb200.ErrPubKey {
		err = kem.ErrPubKey
	}
	return
}
