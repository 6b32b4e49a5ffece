//go:build cuda && cgo

// Package oprfcuda evaluates batches of RFC 9497 OPRF requests for the reference's oprf package (suites P256-SHA256,
// P384-SHA384 and P521-SHA512) with the cb200 engine: one server key, many independent client requests, each with its
// own proof.  Keys come from oprf.DeriveKey or oprf.GenerateKey and are used as their MarshalBinary bytes; requests and
// evaluations stay CIRCL's own types, so clients are unchanged.
// Delivered as source (no Go toolchain in the build image) -- see INTEGRATION.md.
package oprfcuda

import (
	"crypto/rand"
	"errors"

	"github.com/cloudflare/circl/oprf"
	"github.com/cloudflare/circl/zk/dleq"

	"example.com/circl_b200/go/cb200"
)

// ErrRequest reports the requests of a batch that failed (status bits: 1 element, 2 key, 4 randomness, 8 t = 0).
type ErrRequest struct{ Status []byte }

func (e *ErrRequest) Error() string { return "oprfcuda: some requests failed" }

var ErrSuite = errors.New("oprfcuda: suite not served")

func suiteID(s oprf.Suite) (int, error) {
	switch s.Identifier() {
	case "P256-SHA256":
		return cb200.OPRFP256SHA256, nil
	case "P384-SHA384":
		return cb200.OPRFP384SHA384, nil
	case "P521-SHA512":
		return cb200.OPRFP521SHA512, nil
	}
	return 0, ErrSuite
}

// Server is a batched server of one mode (oprf.BaseMode, VerifiableMode or PartialObliviousMode) under one key.
type Server struct {
	suite oprf.Suite
	id    int
	mode  oprf.Mode
	sk    []byte
}

func NewServer(s oprf.Suite, mode oprf.Mode, key *oprf.PrivateKey) (*Server, error) {
	id, err := suiteID(s)
	if err != nil {
		return nil, err
	}
	sk, err := key.MarshalBinary()
	if err != nil {
		return nil, err
	}
	return &Server{s, id, mode, sk}, nil
}

// Evaluate answers every request (all with the same number of elements) as the reference's Server, VerifiableServer
// or PartialObliviousServer.Evaluate would, info being used in the partially oblivious mode.
func (s *Server) Evaluate(reqs []*oprf.EvaluationRequest, info []byte) ([]*oprf.Evaluation, error) {
	n := len(reqs)
	if n == 0 {
		return nil, nil
	}
	m := len(reqs[0].Elements)
	ne, ns, _, np := cb200.OPRFSizes(s.id)
	blinded := make([]byte, 0, n*m*ne)
	for _, r := range reqs {
		if len(r.Elements) != m {
			return nil, errors.New("oprfcuda: requests must hold the same number of elements")
		}
		for _, e := range r.Elements {
			b, err := e.MarshalBinaryCompress()
			if err != nil {
				return nil, err
			}
			blinded = append(blinded, b...)
		}
	}
	g := s.suite.Group()
	var rnd, proof []byte
	if s.mode != oprf.BaseMode {
		rnd = make([]byte, 0, n*ns)
		for i := 0; i < n; i++ {
			b, err := g.RandomNonZeroScalar(rand.Reader).MarshalBinary()
			if err != nil {
				return nil, err
			}
			rnd = append(rnd, b...)
		}
		proof = make([]byte, n*np)
	}
	ev, status := make([]byte, n*m*ne), make([]byte, n)
	if err := cb200.OPRFEvaluate(s.id, int(s.mode), s.sk, true, blinded, m, rnd, info, ev, proof, status); err != nil {
		return nil, err
	}
	for _, st := range status {
		if st != 0 {
			return nil, &ErrRequest{status}
		}
	}
	out := make([]*oprf.Evaluation, n)
	for i := range out {
		e := &oprf.Evaluation{Elements: make([]oprf.Evaluated, m)}
		for j := 0; j < m; j++ {
			e.Elements[j] = g.NewElement()
			if err := e.Elements[j].UnmarshalBinary(ev[(i*m+j)*ne : (i*m+j+1)*ne]); err != nil {
				return nil, err
			}
		}
		if proof != nil {
			e.Proof = new(dleq.Proof)
			if err := e.Proof.UnmarshalBinary(g, proof[i*np:(i+1)*np]); err != nil {
				return nil, err
			}
		}
		out[i] = e
	}
	return out, nil
}

// FullEvaluate is the servers' FullEvaluate on a batch of inputs.
func (s *Server) FullEvaluate(inputs [][]byte, info []byte) ([][]byte, error) {
	_, _, nh, _ := cb200.OPRFSizes(s.id)
	out, status := make([]byte, len(inputs)*nh), make([]byte, len(inputs))
	if err := cb200.OPRFFullEvaluate(s.id, int(s.mode), s.sk, true, inputs, info, out, status); err != nil {
		return nil, err
	}
	for _, st := range status {
		if st != 0 {
			return nil, &ErrRequest{status}
		}
	}
	res := make([][]byte, len(inputs))
	for i := range res {
		res[i] = out[i*nh : (i+1)*nh]
	}
	return res, nil
}
