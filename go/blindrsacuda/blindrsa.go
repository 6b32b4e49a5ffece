//go:build cuda && cgo

// Package blindrsacuda serves batches of RFC 9474 blind signatures (RSABSSA-SHA384) for the reference's
// blindsign/blindrsa package with the cb200 engine: BlindSign under one *rsa.PrivateKey and Verify under one
// *rsa.PublicKey, each for many independent messages.  Clients keep using blindrsa.Client unchanged.
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package blindrsacuda

import (
	"crypto/rsa"
	"errors"
	"math/big"

	"github.com/cloudflare/circl/blindsign/blindrsa"

	"example.com/circl_b200/go/cb200"
)

// ErrBatch reports the ops of a batch that failed, with the per-op status bytes of the C ABI.
type ErrBatch struct{ Status []byte }

func (e *ErrBatch) Error() string { return "blindrsacuda: some operations failed" }

var ErrKey = errors.New("blindrsacuda: only two-prime keys with precomputed CRT values are served")

func be(x *big.Int) []byte {
	if x.Sign() == 0 {
		return []byte{0}
	}
	return x.Bytes()
}

// Signer signs blinded messages under one two-prime key.
type Signer struct {
	n, e, p, q, dp, dq, qinv []byte
	kLen                     int
}

// NewSigner takes a key whose Precompute has run (Precomputed.Dp, Dq and Qinv set).
func NewSigner(sk *rsa.PrivateKey) (*Signer, error) {
	if len(sk.Primes) != 2 || sk.Precomputed.Dp == nil || sk.Precomputed.Dq == nil || sk.Precomputed.Qinv == nil {
		return nil, ErrKey
	}
	s := &Signer{n: be(sk.N), e: be(big.NewInt(int64(sk.E))), p: be(sk.Primes[0]), q: be(sk.Primes[1]),
		dp: be(sk.Precomputed.Dp), dq: be(sk.Precomputed.Dq), qinv: be(sk.Precomputed.Qinv)}
	s.kLen = cb200.BRSAModulusBytes(s.n)
	if s.kLen == 0 {
		return nil, ErrKey
	}
	return s, nil
}

// BlindSign is blindrsa.Signer.BlindSign on a batch: one kLen-byte blind signature per blinded message.  A message
// of the wrong length is blindrsa.ErrUnexpectedSize for the whole batch; failed ops are reported by *ErrBatch (status
// 1 = blindrsa.ErrInvalidMessageLength, 2 = "rsa: internal error") and their rows are nil.
func (s *Signer) BlindSign(blinded [][]byte) ([][]byte, error) {
	n := len(blinded)
	in := make([]byte, n*s.kLen)
	for i, b := range blinded {
		if len(b) != s.kLen {
			return nil, blindrsa.ErrUnexpectedSize
		}
		copy(in[i*s.kLen:], b)
	}
	out, st := make([]byte, n*s.kLen), make([]byte, n)
	if err := cb200.BRSABlindSign(s.n, s.e, s.p, s.q, s.dp, s.dq, s.qinv, in, out, st); err != nil {
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

// Verifier verifies signatures of one variant under one public key.
type Verifier struct {
	variant int
	n, e    []byte
	kLen    int
}

func NewVerifier(v blindrsa.Variant, pk *rsa.PublicKey) (*Verifier, error) {
	if v < blindrsa.SHA384PSSRandomized || v > blindrsa.SHA384PSSZeroDeterministic {
		return nil, blindrsa.ErrInvalidVariant
	}
	vf := &Verifier{variant: int(v), n: be(pk.N), e: be(big.NewInt(int64(pk.E)))}
	vf.kLen = cb200.BRSAModulusBytes(vf.n)
	if vf.kLen == 0 {
		return nil, ErrKey
	}
	return vf, nil
}

// Verify is blindrsa.Verifier.Verify on a batch: one result per (message, signature); a nil entry is a valid
// signature, rsa.ErrVerification an invalid one (a signature of the wrong length included).
func (v *Verifier) Verify(messages, signatures [][]byte) ([]error, error) {
	n := len(messages)
	if len(signatures) != n {
		return nil, errors.New("blindrsacuda: one signature per message")
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
	if err := cb200.BRSAVerify(v.variant, v.n, v.e, messages, sigs, st); err != nil {
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
