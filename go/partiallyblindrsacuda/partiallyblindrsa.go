//go:build cuda && cgo

// Package partiallyblindrsacuda serves batches of partially blind RSA signatures (RSAPBSSA-SHA384) for the reference's
// blindsign/blindrsa/partiallyblindrsa package with the cb200 engine: BlindSign under one *rsa.PrivateKey and Verify
// under one *rsa.PublicKey, each op with its own public metadata.  Clients keep using partiallyblindrsa.Verifier's
// Blind and Finalize unchanged.  Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package partiallyblindrsacuda

import (
	"crypto"
	"crypto/rsa"
	"errors"
	"math/big"

	"github.com/cloudflare/circl/blindsign/blindrsa/partiallyblindrsa"

	"example.com/circl_b200/go/cb200"
)

// ErrBatch reports the ops of a batch that failed, with the per-op status bytes of the C ABI.
type ErrBatch struct{ Status []byte }

func (e *ErrBatch) Error() string { return "partiallyblindrsacuda: some operations failed" }

// ErrHash: only crypto.SHA384 is served.
var ErrHash = errors.New("partiallyblindrsacuda: only crypto.SHA384 is served")

func be(x *big.Int) []byte {
	if x.Sign() == 0 {
		return []byte{0}
	}
	return x.Bytes()
}

// Signer signs blinded messages under one two-prime key whose primes are safe.
type Signer struct {
	n, p, q, qinv []byte
	kLen          int
}

// NewSigner takes a key whose Precompute has run (Precomputed.Qinv set) and runs the reference's safe-prime test
// once; a key that fails it, or lies outside the served range, is partiallyblindrsa.ErrInvalidPrivateKey.
func NewSigner(sk *rsa.PrivateKey, h crypto.Hash) (*Signer, error) {
	if h != crypto.SHA384 {
		return nil, ErrHash
	}
	if len(sk.Primes) != 2 || sk.Precomputed.Qinv == nil {
		return nil, partiallyblindrsa.ErrInvalidPrivateKey
	}
	s := &Signer{n: be(sk.N), p: be(sk.Primes[0]), q: be(sk.Primes[1]), qinv: be(sk.Precomputed.Qinv)}
	s.kLen = cb200.BRSAModulusBytes(s.n)
	if s.kLen == 0 || cb200.PBRSACheckKey(s.n, s.p, s.q) != nil {
		return nil, partiallyblindrsa.ErrInvalidPrivateKey
	}
	return s, nil
}

// BlindSign is partiallyblindrsa.Signer.BlindSign on a batch: one kLen-byte blind signature per blinded message,
// op i under metadata[i].  A message of the wrong length is partiallyblindrsa.ErrUnexpectedSize for the whole batch;
// failed ops are reported by *ErrBatch (status 1 = ErrInvalidMessageLength, 2 = "rsa: internal error") and their rows
// are nil.
func (s *Signer) BlindSign(blinded, metadata [][]byte) ([][]byte, error) {
	n := len(blinded)
	if len(metadata) != n {
		return nil, errors.New("partiallyblindrsacuda: one metadata string per blinded message")
	}
	in := make([]byte, n*s.kLen)
	for i, b := range blinded {
		if len(b) != s.kLen {
			return nil, partiallyblindrsa.ErrUnexpectedSize
		}
		copy(in[i*s.kLen:], b)
	}
	out, st := make([]byte, n*s.kLen), make([]byte, n)
	if err := cb200.PBRSABlindSign(s.n, s.p, s.q, s.qinv, in, metadata, out, st); err != nil {
		return nil, err
	}
	sigs := make([][]byte, n)
	bad := false
	for i := range sigs {
		if st[i] != 0 {
			bad = true
			continue
		}
		sigs[i] = out[i*s.kLen : (i+1)*s.kLen]
	}
	if bad {
		return sigs, &ErrBatch{Status: st}
	}
	return sigs, nil
}

// Verifier verifies signatures under one public key.
type Verifier struct {
	n    []byte
	kLen int
}

func NewVerifier(pk *rsa.PublicKey, h crypto.Hash) (*Verifier, error) {
	if h != crypto.SHA384 {
		return nil, ErrHash
	}
	if pk == nil || pk.N == nil {
		return nil, partiallyblindrsa.ErrInvalidPublicKey
	}
	v := &Verifier{n: be(pk.N)}
	v.kLen = cb200.BRSAModulusBytes(v.n)
	if v.kLen == 0 {
		return nil, partiallyblindrsa.ErrInvalidPublicKey
	}
	return v, nil
}

// Verify is partiallyblindrsa.Verifier.Verify on a batch: one result per (message, metadata, signature); a nil entry
// is a valid signature, rsa.ErrVerification an invalid one (a signature of the wrong length included).
func (v *Verifier) Verify(messages, metadata, signatures [][]byte) ([]error, error) {
	n := len(messages)
	if len(signatures) != n || len(metadata) != n {
		return nil, errors.New("partiallyblindrsacuda: one metadata string and one signature per message")
	}
	sigs, wrong := make([]byte, n*v.kLen), make([]bool, n)
	for i, s := range signatures {
		if len(s) != v.kLen {
			wrong[i] = true
			continue
		}
		copy(sigs[i*v.kLen:], s)
	}
	st := make([]byte, n)
	if err := cb200.PBRSAVerify(v.n, messages, metadata, sigs, st); err != nil {
		return nil, err
	}
	res := make([]error, n)
	for i := range res {
		if wrong[i] || st[i] != 0 {
			res[i] = rsa.ErrVerification
		}
	}
	return res, nil
}
