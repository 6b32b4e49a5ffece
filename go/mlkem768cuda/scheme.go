//go:build cuda && cgo

// Package mlkem768cuda registers "ML-KEM-768" backed by the cb200 engine.  It keeps
// kem.Scheme (kem/kem.go:33-82) intact: every method that is not on the accelerated
// path delegates to CIRCL's own mlkem768 scheme; Encapsulate* go through the GPU
// (batch of one), and EncapsulateBatch is the entry point that makes a GPU worthwhile.
//
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package mlkem768cuda

import (
	cryptoRand "crypto/rand"

	"github.com/cloudflare/circl/kem"
	"github.com/cloudflare/circl/kem/mlkem/mlkem768"

	"example.com/circl_b200/go/cb200"
)

type scheme struct{ kem.Scheme } // embeds CIRCL's stateless singleton (kyber.go:269)

var sch kem.Scheme = &scheme{mlkem768.Scheme()}

// Scheme returns the GPU-backed ML-KEM-768 scheme; Name() is unchanged so registries keep working.
func Scheme() kem.Scheme { return sch }

func (s *scheme) EncapsulateDeterministically(pk kem.PublicKey, seed []byte) (ct, ss []byte, err error) {
	if len(seed) != mlkem768.EncapsulationSeedSize {
		return nil, nil, kem.ErrSeedSize // kyber.go:362-364
	}
	pub, ok := pk.(*mlkem768.PublicKey)
	if !ok {
		return nil, nil, kem.ErrTypeMismatch // kyber.go:366-369
	}
	packed, _ := pub.MarshalBinary()
	ct = make([]byte, mlkem768.CiphertextSize)
	ss = make([]byte, mlkem768.SharedKeySize)
	if err = cb200.MLKEMEncaps(3, packed, true, seed, ct, ss); err == cb200.ErrPubKey {
		err = kem.ErrPubKey
	}
	return
}

func (s *scheme) Encapsulate(pk kem.PublicKey) (ct, ss []byte, err error) {
	var seed [mlkem768.EncapsulationSeedSize]byte
	if _, err = cryptoRand.Read(seed[:]); err != nil {
		return nil, nil, err
	}
	return s.EncapsulateDeterministically(pk, seed[:])
}

// EncapsulateBatch encapsulates len(seeds)/32 times.  packedKeys holds either one
// 1184-byte key (shared) or one key per operation.  Errors follow kem.Scheme:
// kem.ErrPubKeySize / kem.ErrPubKey / kem.ErrSeedSize.
func EncapsulateBatch(packedKeys, seeds []byte) (cts, sss []byte, err error) {
	if len(seeds)%32 != 0 {
		return nil, nil, kem.ErrSeedSize
	}
	n := len(seeds) / 32
	shared := len(packedKeys) == mlkem768.PublicKeySize
	if !shared && len(packedKeys) != n*mlkem768.PublicKeySize {
		return nil, nil, kem.ErrPubKeySize
	}
	cts = make([]byte, n*mlkem768.CiphertextSize)
	sss = make([]byte, n*mlkem768.SharedKeySize)
	if err = cb200.MLKEMEncaps(3, packedKeys, shared, seeds, cts, sss); err == cb200.ErrPubKey {
		err = kem.ErrPubKey
	}
	return
}
