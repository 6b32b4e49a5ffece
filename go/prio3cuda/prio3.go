//go:build cuda && cgo

// Package prio3cuda answers batches of Prio3 aggregator work (draft-irtf-cfrg-vdaf-14) for the reference's
// vdaf/prio3 packages (count, sum, sumvec, histogram, mhcv) with the cb200 engine, on the reference's own types:
// inputs are pointers to values of count.InputShare, count.PrepShare, ... (any of the five packages), and outputs are
// filled into values the caller made with the package's New methods and Params, through their MarshalBinary /
// UnmarshalBinary.  Nonces and the verify key are passed as (*[16]byte)(nonce) and (*[32]byte)(verifyKey).
// Clients keep using the reference's Shard; the collector keeps its Unshard.  Delivered as source (no Go toolchain in
// the build image) -- see INTEGRATION.md.
package prio3cuda

import (
	"encoding"
	"errors"

	"example.com/circl_b200/go/cb200"
)

// The reference's per-report errors, by status bit.
var (
	ErrDecode       = errors.New("prio3cuda: field element is not canonical") // UnmarshalBinary's error
	ErrJointRand    = errors.New("invalid joint randomness")                  // prio3.ErrJointRand
	ErrInvalidEval  = errors.New("invalid evaluation point")                  // flp.ErrInvalidEval
	ErrProofVerify  = errors.New("proof verifier check failed")               // prio3.ErrProofVerify
	ErrBatchLengths = errors.New("prio3cuda: batch slices have different lengths")
)

// StatusErr maps one report's status byte to the reference's error (nil for 0).
func StatusErr(st byte) error {
	switch {
	case st == 0:
		return nil
	case st&1 != 0:
		return ErrDecode
	case st&2 != 0:
		return ErrJointRand
	case st&4 != 0:
		return ErrInvalidEval
	default:
		return ErrProofVerify
	}
}

// Aggregator is one Prio3 instance.
type Aggregator struct {
	cfg   cb200.Prio3Config
	sizes cb200.Prio3Sizes
}

func newAggregator(c cb200.Prio3Config) (*Aggregator, error) {
	z, err := cb200.Prio3GetSizes(&c)
	if err != nil {
		return nil, err
	}
	return &Aggregator{c, z}, nil
}

// NewCount, NewSum, NewSumVec, NewHistogram and NewMultiHotCountVec take the arguments of the reference's New of
// count, sum, sumvec, histogram and mhcv, and return its errors' conditions as an error.
func NewCount(numShares uint8, context []byte) (*Aggregator, error) {
	return newAggregator(cb200.Prio3Config{Kind: 1, NumShares: uint32(numShares), Context: context})
}

func NewSum(numShares uint8, maxMeasurement uint64, context []byte) (*Aggregator, error) {
	return newAggregator(cb200.Prio3Config{Kind: 2, NumShares: uint32(numShares), MaxMeasurement: maxMeasurement,
		Context: context})
}

func NewSumVec(numShares uint8, length, bits, chunkLength uint, context []byte) (*Aggregator, error) {
	return newAggregator(cb200.Prio3Config{Kind: 3, NumShares: uint32(numShares), Length: uint64(length),
		Bits: uint64(bits), ChunkLength: uint64(chunkLength), Context: context})
}

func NewHistogram(numShares uint8, length, chunkLength uint, context []byte) (*Aggregator, error) {
	return newAggregator(cb200.Prio3Config{Kind: 4, NumShares: uint32(numShares), Length: uint64(length),
		ChunkLength: uint64(chunkLength), Context: context})
}

func NewMultiHotCountVec(numShares uint8, length, maxWeight, chunkLength uint, context []byte) (*Aggregator, error) {
	return newAggregator(cb200.Prio3Config{Kind: 5, NumShares: uint32(numShares), Length: uint64(length),
		MaxWeight: uint64(maxWeight), ChunkLength: uint64(chunkLength), Context: context})
}

// Sizes returns the wire sizes of the instance.
func (a *Aggregator) Sizes() cb200.Prio3Sizes { return a.sizes }

// pack marshals n values of `width` bytes each back to back.
func pack[T encoding.BinaryMarshaler](vs []T, width int) ([]byte, error) {
	out := make([]byte, 0, len(vs)*width)
	for _, v := range vs {
		b, err := v.MarshalBinary()
		if err != nil {
			return nil, err
		}
		if len(b) != width {
			return nil, errors.New("prio3cuda: a value does not have the configuration's size")
		}
		out = append(out, b...)
	}
	return out, nil
}

// unpack fills the values of the reports whose status is 0 from rows of `width` bytes.
func unpack[T encoding.BinaryUnmarshaler](rows []byte, width int, status []byte, out []T) error {
	for i := range out {
		if status[i] != 0 {
			continue
		}
		if err := out[i].UnmarshalBinary(rows[i*width : (i+1)*width]); err != nil {
			return err
		}
	}
	return nil
}

// PrepInit is the reference's PrepInit on a batch under one verify key as aggregator aggID: nonces[i],
// publicShares[i] (nil values for circuits without joint randomness) and inputShares[i] give report i; states[i] and
// shares[i] (made with the package's New(&params)) receive its outputs.  The result holds each report's error (nil
// when it succeeded); the outputs of a failed report are left untouched.
func PrepInit[PS, IS encoding.BinaryMarshaler, ST, SH encoding.BinaryUnmarshaler](a *Aggregator, verifyKey *[32]byte,
	aggID uint8, nonces []*[16]byte, publicShares []PS, inputShares []IS, states []ST, shares []SH) ([]error, error) {
	n := len(nonces)
	if len(inputShares) != n || len(states) != n || len(shares) != n || (a.sizes.PublicShare > 0 && len(publicShares) != n) {
		return nil, ErrBatchLengths
	}
	z := a.sizes
	in := z.InputShareLeader
	if aggID != 0 {
		in = z.InputShareHelper
	}
	nb := make([]byte, 0, 16*n)
	for _, x := range nonces {
		nb = append(nb, x[:]...)
	}
	ib, err := pack(inputShares, in)
	if err != nil {
		return nil, err
	}
	var pb []byte
	if z.PublicShare > 0 {
		if pb, err = pack(publicShares, z.PublicShare); err != nil {
			return nil, err
		}
	}
	sb, hb, st := make([]byte, n*z.PrepState), make([]byte, n*z.PrepShare), make([]byte, n)
	if err := cb200.Prio3PrepInit(&a.cfg, z, verifyKey[:], aggID, nb, pb, ib, sb, hb, st); err != nil {
		return nil, err
	}
	if err := unpack(sb, z.PrepState, st, states); err != nil {
		return nil, err
	}
	if err := unpack(hb, z.PrepShare, st, shares); err != nil {
		return nil, err
	}
	return errs(st), nil
}

// PrepSharesToPrep is the reference's PrepSharesToPrep on a batch: prepShares[i] holds the NumShares prep shares of
// report i in aggregator order; msgs[i] receives its prep message.
func PrepSharesToPrep[SH encoding.BinaryMarshaler, M encoding.BinaryUnmarshaler](a *Aggregator, prepShares [][]SH,
	msgs []M) ([]error, error) {
	n := len(prepShares)
	if len(msgs) != n {
		return nil, ErrBatchLengths
	}
	z := a.sizes
	rows := make([]byte, 0, n*int(a.cfg.NumShares)*z.PrepShare)
	for _, r := range prepShares {
		if len(r) != int(a.cfg.NumShares) {
			return nil, errors.New("invalid prep shares length") // prio3.ErrPrepShareSize
		}
		b, err := pack(r, z.PrepShare)
		if err != nil {
			return nil, err
		}
		rows = append(rows, b...)
	}
	mb, st := make([]byte, n*z.PrepMsg), make([]byte, n)
	if err := cb200.Prio3PrepSharesToPrep(&a.cfg, z, rows, mb, st); err != nil {
		return nil, err
	}
	if err := unpack(mb, z.PrepMsg, st, msgs); err != nil {
		return nil, err
	}
	return errs(st), nil
}

// PrepNext is the reference's PrepNext on a batch; outShares[i] receives report i's out share.
func PrepNext[ST, M encoding.BinaryMarshaler, O encoding.BinaryUnmarshaler](a *Aggregator, states []ST, msgs []M,
	outShares []O) ([]error, error) {
	n := len(states)
	if len(msgs) != n || len(outShares) != n {
		return nil, ErrBatchLengths
	}
	z := a.sizes
	sb, err := pack(states, z.PrepState)
	if err != nil {
		return nil, err
	}
	mb, err := pack(msgs, z.PrepMsg)
	if err != nil {
		return nil, err
	}
	ob, st := make([]byte, n*z.OutShare), make([]byte, n)
	if err := cb200.Prio3PrepNext(&a.cfg, z, sb, mb, ob, st); err != nil {
		return nil, err
	}
	if err := unpack(ob, z.OutShare, st, outShares); err != nil {
		return nil, err
	}
	return errs(st), nil
}

// Aggregate is AggregateInit followed by AggregateUpdate with every out share, on the device; aggShare (made with
// the package's AggregateInit) receives the sum.
func Aggregate[O encoding.BinaryMarshaler, A encoding.BinaryUnmarshaler](a *Aggregator, outShares []O,
	aggShare A) error {
	z := a.sizes
	ob, err := pack(outShares, z.OutShare)
	if err != nil {
		return err
	}
	agg := make([]byte, z.AggShare)
	if err := cb200.Prio3Aggregate(&a.cfg, z, ob, nil, agg); err != nil {
		return err
	}
	return aggShare.UnmarshalBinary(agg)
}

func errs(st []byte) []error {
	out := make([]error, len(st))
	for i, s := range st {
		out[i] = StatusErr(s)
	}
	return out
}
