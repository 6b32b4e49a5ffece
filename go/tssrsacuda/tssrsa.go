//go:build cuda && cgo

// Package tssrsacuda serves batches of threshold RSA (the reference's tss/rsa package) with the cb200 engine: a party's
// signature shares of many digests under its one KeyShare, and the combination of many independent sets of shares.
// KeyShare's s_i and cached twoDeltaSi and SignShare's xi are unexported, so they travel through the reference's own
// MarshalBinary / UnmarshalBinary encodings.  Delivered as source (no Go toolchain in the build image) -- see
// INTEGRATION.md.
package tssrsacuda

import (
	"crypto/rsa"
	"encoding/binary"
	"errors"
	"math/big"

	tss "github.com/cloudflare/circl/tss/rsa"

	"example.com/circl_b200/go/cb200"
)

var (
	ErrInvalidCalc = tss.ErrInvalidCalc
	ErrInternal    = errors.New("rsa: internal error")
	errEncoding    = errors.New("tssrsacuda: unexpected KeyShare encoding")
)

func kLen(pub *rsa.PublicKey) int { return (pub.N.BitLen() + 7) / 8 }

// row: x as kLen big-endian bytes, reduced mod N when it is longer (Exp reduces it)
func row(x []byte, pub *rsa.PublicKey, k int) []byte {
	v := new(big.Int).SetBytes(x)
	if len(x) > k {
		v.Mod(v, pub.N)
	}
	return v.FillBytes(make([]byte, k))
}

// exponent returns Players, Threshold, Index and 2 Delta s_i (or the cached twoDeltaSi) of a KeyShare.
func exponent(share *tss.KeyShare) (uint16, uint16, uint16, []byte, error) {
	b, err := share.MarshalBinary()
	if err != nil {
		return 0, 0, 0, nil, err
	}
	if len(b) < 8 {
		return 0, 0, 0, nil, errEncoding
	}
	players, threshold, index := binary.BigEndian.Uint16(b[0:2]), binary.BigEndian.Uint16(b[2:4]),
		binary.BigEndian.Uint16(b[4:6])
	sl := int(binary.BigEndian.Uint16(b[6:8]))
	if len(b) < 8+sl+3 {
		return 0, 0, 0, nil, errEncoding
	}
	si := new(big.Int).SetBytes(b[8 : 8+sl])
	if b[8+sl] != 0 {
		tl := int(binary.BigEndian.Uint16(b[8+sl+1 : 8+sl+3]))
		if len(b) < 8+sl+3+tl {
			return 0, 0, 0, nil, errEncoding
		}
		return players, threshold, index, append([]byte{0}, b[8+sl+3:8+sl+3+tl]...), nil
	}
	e := new(big.Int).MulRange(1, int64(players))
	e.Lsh(e, 1).Mul(e, si)
	return players, threshold, index, append([]byte{0}, e.Bytes()...), nil
}

// SignBatch: share.Sign(nil, pub, digests[i], false) for every digest (the exponentiation is constant-time, so no
// randomness is taken).
func SignBatch(share *tss.KeyShare, pub *rsa.PublicKey, digests [][]byte) ([]tss.SignShare, error) {
	players, threshold, index, e, err := exponent(share)
	if err != nil {
		return nil, err
	}
	k := kLen(pub)
	in := make([]byte, 0, len(digests)*k)
	for _, d := range digests {
		in = append(in, row(d, pub, k)...)
	}
	xi := make([]byte, len(in))
	if err := cb200.TSSRSASignShare(pub.N.Bytes(), int(players), e, in, xi); err != nil {
		return nil, err
	}
	out := make([]tss.SignShare, len(digests))
	for i := range out {
		v := new(big.Int).SetBytes(xi[i*k : (i+1)*k]).Bytes()
		if len(v) == 0 {
			v = []byte{0}
		}
		enc := make([]byte, 8, 8+len(v))
		binary.BigEndian.PutUint16(enc[0:2], players)
		binary.BigEndian.PutUint16(enc[2:4], threshold)
		binary.BigEndian.PutUint16(enc[4:6], index)
		binary.BigEndian.PutUint16(enc[6:8], uint16(len(v)))
		if err := out[i].UnmarshalBinary(append(enc, v...)); err != nil {
			return nil, err
		}
	}
	return out, nil
}

// paramsFail: the checks CombineSignShares makes before any arithmetic (rsa_threshold.go:83-93, 211-230)
func paramsFail(ss []tss.SignShare, players, threshold uint) bool {
	if players <= 1 || threshold < 1 || threshold > players || len(ss) == 0 || uint(len(ss)) < threshold {
		return true
	}
	for j := range ss {
		if ss[j].Players != players || ss[j].Threshold != threshold {
			return true
		}
	}
	return false
}

func xiOf(s *tss.SignShare) ([]byte, error) {
	b, err := s.MarshalBinary()
	if err != nil {
		return nil, err
	}
	return b[8:], nil
}

// CombineBatch: tss.CombineSignShares(pub, players, threshold, shares[i], msgs[i]) for every op, with the reference's
// parameter errors per op; ops with the same number of shares run in one call.
func CombineBatch(pub *rsa.PublicKey, players, threshold uint, shares [][]tss.SignShare, msgs [][]byte) ([]tss.Signature, []error) {
	k := kLen(pub)
	sigs := make([]tss.Signature, len(shares))
	errs := make([]error, len(shares))
	groups := map[int][]int{}
	for i, ss := range shares {
		if paramsFail(ss, players, threshold) {
			// the reference returns its parameter error before any arithmetic
			_, errs[i] = tss.CombineSignShares(pub, players, threshold, ss, msgs[i])
			continue
		}
		if len(ss) > 64 {
			errs[i] = errors.New("tssrsacuda: at most 64 shares per op are served")
			continue
		}
		groups[len(ss)] = append(groups[len(ss)], i)
	}
	e := big.NewInt(int64(pub.E)).Bytes()
	for kk, ops := range groups {
		n := len(ops)
		idx := make([]uint16, 0, n*kk)
		xi := make([]byte, 0, n*kk*k)
		in := make([]byte, 0, n*k)
		for _, i := range ops {
			for j := range shares[i] {
				if shares[i][j].Index > 0xffff {
					errs[i] = errors.New("tssrsacuda: share indices above 65535 are not served")
				}
				idx = append(idx, uint16(shares[i][j].Index))
				v, err := xiOf(&shares[i][j])
				if err != nil {
					errs[i] = err
				}
				xi = append(xi, row(v, pub, k)...)
			}
			m := msgs[i]
			if len(m) > k { // x >= N: fails the final check as 2^(8 kLen) - 1 does
				m = make([]byte, k)
				for j := range m {
					m[j] = 0xff
				}
			}
			in = append(in, row(m, pub, k)...)
		}
		sig := make([]byte, n*k)
		st := make([]byte, n)
		if err := cb200.TSSRSACombine(pub.N.Bytes(), e, int(players), int(threshold), kk, idx, xi, in, sig, st); err != nil {
			for _, i := range ops {
				errs[i] = err
			}
			continue
		}
		for r, i := range ops {
			if errs[i] != nil {
				continue
			}
			switch st[r] {
			case 0:
				sigs[i] = sig[r*k : (r+1)*k]
			case 1:
				errs[i] = ErrInvalidCalc
			default:
				errs[i] = ErrInternal
			}
		}
	}
	return sigs, errs
}
