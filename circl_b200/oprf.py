"""RFC 9497 OPRF servers over the C ABI: the reference's oprf package (oprf/oprf.go, server.go, keys.go) for the
suites P256-SHA256, P384-SHA384 and P521-SHA512, in modes 0x00 (Server), 0x01 (VerifiableServer) and 0x02
(PartialObliviousServer).  The client side is not served here.

  GetSuite, DeriveKey                                  keys.go:103-132
  NewServer / NewVerifiableServer / NewPartialObliviousServer
      .PublicKey(), .Evaluate, .FullEvaluate, .VerifyFinalize      server.go
      .EvaluateBatch, .FullEvaluateBatch                           the same on batches (numpy or CUDA tensors)
  DeriveKeyBatch, EvaluateBatch, FullEvaluateBatch                 batches with per-op keys (or one shared key)

Elements are compressed points (0x02 | 0x03 || X, Ne bytes), scalars Ns big-endian bytes.  The proof randomness r is
an argument (one Ns row per request; the reference draws it from rand.Reader): Evaluate draws it with os.urandom when
none is given.  A batch whose ops fail raises the error of the first failure class below, with .status holding the
per-op bits (1 an element that does not decode, 2 an invalid key, 4 an invalid r, 8 t = 0 in mode 2, 16 a
FullEvaluate input over 65535 bytes on CUDA buffers) and .results
the outputs, whose failed rows are all zero.
"""
from __future__ import annotations

import hmac
import os

import numpy as np

from ._ffi import check, lib
from .hybrid import _is_torch, _new, _prep, _ptr

__all__ = ["BaseMode", "VerifiableMode", "PartialObliviousMode", "GetSuite", "SuiteP256", "SuiteP384", "SuiteP521",
           "DeriveKey", "DeriveKeyBatch", "EvaluateBatch", "FullEvaluateBatch", "NewServer", "NewVerifiableServer",
           "NewPartialObliviousServer", "PrivateKey", "PublicKey", "OprfError", "ErrInvalidSuite", "ErrInvalidMode",
           "ErrInvalidSeed", "ErrInvalidInfo", "ErrInvalidInput", "ErrInvalidPrivateKey", "ErrInverseZero",
           "ErrInvalidRandomness"]

BaseMode, VerifiableMode, PartialObliviousMode = 0x00, 0x01, 0x02


class OprfError(ValueError):
    def __init__(self, msg="", status=None, results=None):
        super().__init__(msg)
        self.status, self.results = status, results


class ErrInvalidSuite(OprfError):  # oprf.ErrInvalidSuite
    pass


class ErrInvalidMode(OprfError):  # oprf.ErrInvalidMode
    pass


class ErrInvalidSeed(OprfError):  # oprf.ErrInvalidSeed
    pass


class ErrInvalidInfo(OprfError):  # oprf.ErrInvalidInfo: more than 65535 bytes
    pass


class ErrInvalidInput(OprfError):  # group.UnmarshalBinary's error on a blinded element; an input over 65535 bytes
    pass


class ErrInvalidPrivateKey(OprfError):  # oprf.ErrInvalidPrivateKey
    pass


class ErrInverseZero(OprfError):  # oprf.ErrInverseZero
    pass


class ErrInvalidRandomness(OprfError):  # r = 0 or r >= n (r = 0 would reveal the key through s)
    pass


class Suite:
    def __init__(self, identifier: str, sid: int):
        self.identifier, self.id = identifier, sid

    def Identifier(self) -> str:
        return self.identifier

    def __repr__(self):
        return self.identifier

    @property
    def Ne(self):
        return lib().cb200_oprf_element_size(self.id)

    @property
    def Ns(self):
        return lib().cb200_oprf_scalar_size(self.id)

    @property
    def Nh(self):
        return lib().cb200_oprf_output_size(self.id)

    @property
    def proof_size(self):
        return lib().cb200_oprf_proof_size(self.id)


SuiteP256 = Suite("P256-SHA256", 3)
SuiteP384 = Suite("P384-SHA384", 4)
SuiteP521 = Suite("P521-SHA512", 5)


def GetSuite(identifier: str) -> Suite:
    for s in (SuiteP256, SuiteP384, SuiteP521):
        if s.identifier == identifier:
            return s
    raise ErrInvalidSuite("oprf: invalid suite")


def _mode(mode):
    if mode not in (BaseMode, VerifiableMode, PartialObliviousMode):
        raise ErrInvalidMode("oprf: invalid mode")
    return mode


def _info(info):
    info = bytes(info or b"")
    if len(info) > 65535:
        raise ErrInvalidInfo("oprf: invalid info")
    return info, (info or b"\0")


def _raise(status, results):
    st = status.cpu().numpy() if _is_torch(status) else status
    if not st.any():
        return
    for bit, cls, what in ((2, ErrInvalidPrivateKey, "invalid private key"), (8, ErrInverseZero, "inverting a zero value"),
                           (1 | 16, ErrInvalidInput, "invalid blinded element or input"),
                           (4, ErrInvalidRandomness, "invalid r")):
        if (st & bit).any():
            raise cls(f"oprf: {what} in {int(((st & bit) != 0).sum())} of {len(st)} ops", status, results)


class PublicKey:
    def __init__(self, suite: Suite, b: bytes):
        self.suite, self.e = suite, bytes(b)

    def MarshalBinary(self) -> bytes:
        return self.e


class PrivateKey:
    def __init__(self, suite: Suite, k: bytes, pub: bytes):
        self.suite, self.k, self.pub = suite, bytes(k), bytes(pub)

    def MarshalBinary(self) -> bytes:
        return self.k

    def Public(self) -> PublicKey:
        return PublicKey(self.suite, self.pub)


def DeriveKeyBatch(suite: Suite, mode: int, seeds, info: bytes = b""):
    """(sk (n, Ns), pk (n, Ne)) from 32-byte seeds and one info."""
    _mode(mode)
    info, ib = _info(info)
    seeds = _prep(seeds, 32, ErrInvalidSeed("oprf: invalid seed size"))
    n = seeds.shape[0]
    sk, pk = _new(seeds, (n, suite.Ns)), _new(seeds, (n, suite.Ne))
    check(lib().cb200_oprf_derive_key(suite.id, mode, _ptr(seeds), ib, len(info), _ptr(sk), _ptr(pk), n))
    return sk, pk


def DeriveKey(suite: Suite, mode: int, seed: bytes, info: bytes = b"") -> PrivateKey:
    """keys.go:103-132."""
    if len(seed) != 32:
        raise ErrInvalidSeed("oprf: invalid seed size")
    sk, pk = DeriveKeyBatch(suite, mode, np.frombuffer(bytes(seed), dtype=np.uint8).reshape(1, 32), info)
    return PrivateKey(suite, sk[0].tobytes(), pk[0].tobytes())


def _keys(suite, sk, like):
    """(rows, stride): one key for the batch (a 1-D row or bytes) or one per op."""
    if isinstance(sk, (bytes, bytearray)):
        sk = np.frombuffer(bytes(sk), dtype=np.uint8)
    if _is_torch(like) and not _is_torch(sk):
        import torch
        sk = torch.as_tensor(np.asarray(sk, dtype=np.uint8)).to(like.device)
    if sk.ndim == 1:
        sk = _prep(sk.reshape(1, -1), suite.Ns, ErrInvalidPrivateKey("oprf: invalid private key size"))
        return sk, 0
    return _prep(sk, suite.Ns, ErrInvalidPrivateKey("oprf: invalid private key size")), suite.Ns


def EvaluateBatch(suite: Suite, mode: int, sk, blinded, m: int = 1, rnd=None, info: bytes = b""):
    """n requests of m elements each: blinded is (n, m * Ne) (or (n * m, Ne) rows in request order), rnd (n, Ns) in
    modes 1 and 2.  Returns (evaluated (n, m * Ne), proof (n, 2 Ns) or None)."""
    _mode(mode)
    info, ib = _info(info)
    if not 1 <= m <= 65535:
        raise ErrInvalidInput("oprf: 1 <= m <= 65535")
    Ne = suite.Ne
    if blinded.ndim == 2 and blinded.shape[1] == Ne and m > 1:
        blinded = blinded.reshape(-1, m * Ne)
    blinded = _prep(blinded, m * Ne, ErrInvalidInput("oprf: blinded elements must be (n, m * Ne) uint8"))
    n = blinded.shape[0]
    keys, ks = _keys(suite, sk, blinded)
    ev, st = _new(blinded, (n, m * Ne)), _new(blinded, (n,))
    proof = rp = None
    if mode != BaseMode:
        rnd = _prep(rnd, suite.Ns, ErrInvalidRandomness("oprf: r must be (n, Ns) uint8"))
        if rnd.shape[0] != n:
            raise ErrInvalidRandomness("oprf: one r per request")
        proof = _new(blinded, (n, suite.proof_size))
        rp = _ptr(rnd)
    if ks and keys.shape[0] != n:
        raise ErrInvalidPrivateKey("oprf: one key per request")
    check(lib().cb200_oprf_evaluate(suite.id, mode, _ptr(keys), ks, _ptr(blinded), m, rp, ib, len(info), _ptr(ev),
                                    _ptr(proof) if proof is not None else None, _ptr(st), n))
    _raise(st, (ev, proof))
    return ev, proof


def _msgs(inputs):
    lens = [len(x) for x in inputs]
    if any(v > 65535 for v in lens):
        raise ErrInvalidInput("oprf: input longer than 65535 bytes")
    off = np.zeros(len(inputs) + 1, dtype=np.uint64)
    np.cumsum(lens, out=off[1:])
    return np.frombuffer(b"".join(bytes(x) for x in inputs) or b"\0", dtype=np.uint8).copy(), off


def FullEvaluateBatch(suite: Suite, mode: int, sk, inputs, info: bytes = b""):
    """outputs (n, Nh) for a list of inputs (host), or for (msgs, msg_off) CUDA tensors (uint8 bytes, n + 1 int64
    offsets)."""
    _mode(mode)
    info, ib = _info(info)
    if isinstance(inputs, tuple) and _is_torch(inputs[0]):
        msgs, off = inputs
        like, n = msgs, off.shape[0] - 1
        import torch
        check(lib().cb200_set_stream(torch.cuda.current_stream().cuda_stream))
    else:
        msgs, off = _msgs(inputs)
        like, n = msgs, len(inputs)
    keys, ks = _keys(suite, sk, like)
    if ks and keys.shape[0] != n:
        raise ErrInvalidPrivateKey("oprf: one key per op")
    out, st = _new(like, (n, suite.Nh)), _new(like, (n,))
    if n:
        check(lib().cb200_oprf_full_evaluate(suite.id, mode, _ptr(keys), ks, _ptr(msgs), _ptr(off), ib, len(info),
                                             _ptr(out), _ptr(st), n))
    _raise(st, out)
    return out


class _Server:
    mode = BaseMode

    def __init__(self, suite: Suite, key: PrivateKey):
        if key is None:
            raise OprfError("oprf: must provide a key")
        self.suite, self.key = suite, key

    def PublicKey(self) -> PublicKey:
        return self.key.Public()

    def _sk(self):
        return np.frombuffer(self.key.k, dtype=np.uint8)

    def EvaluateBatch(self, blinded, m: int = 1, rnd=None, info: bytes = b""):
        return EvaluateBatch(self.suite, self.mode, self._sk(), blinded, m, rnd, info)

    def FullEvaluateBatch(self, inputs, info: bytes = b""):
        return FullEvaluateBatch(self.suite, self.mode, self._sk(), inputs, info)

    def _evaluate(self, elements, info, rnd):
        els = [bytes(e) for e in elements]
        if not els or any(len(e) != self.suite.Ne for e in els):
            raise ErrInvalidInput("oprf: invalid blinded element")
        b = np.frombuffer(b"".join(els), dtype=np.uint8).reshape(1, -1)
        r = None
        if self.mode != BaseMode:
            r = np.frombuffer(bytes(rnd) if rnd is not None else self._random_scalar(), dtype=np.uint8).reshape(1, -1)
        ev, proof = EvaluateBatch(self.suite, self.mode, self._sk(), b, len(els), r, info)
        Ne = self.suite.Ne
        out = [ev[0, j * Ne:(j + 1) * Ne].tobytes() for j in range(len(els))]
        return out, (proof[0].tobytes() if proof is not None else None)

    def _random_scalar(self):
        n = _ORDERS[self.suite.identifier]
        while True:
            k = int.from_bytes(os.urandom(self.suite.Ns), "big") % (1 << n.bit_length())
            if 0 < k < n:
                return k.to_bytes(self.suite.Ns, "big")

    def _full(self, inp, info):
        return FullEvaluateBatch(self.suite, self.mode, self._sk(), [bytes(inp)], info)[0].tobytes()

    def _verify(self, inp, info, expected):
        try:
            got = self._full(inp, info)
        except OprfError:
            return False
        return hmac.compare_digest(got, bytes(expected))


class Server(_Server):
    mode = BaseMode

    def Evaluate(self, elements, rnd=None):
        """(evaluated elements, None)."""
        return self._evaluate(elements, b"", rnd)

    def FullEvaluate(self, inp: bytes) -> bytes:
        return self._full(inp, b"")

    def VerifyFinalize(self, inp: bytes, expected: bytes) -> bool:
        return self._verify(inp, b"", expected)


class VerifiableServer(Server):
    mode = VerifiableMode

    def Evaluate(self, elements, rnd=None):
        """(evaluated elements, proof c || s)."""
        return self._evaluate(elements, b"", rnd)


class PartialObliviousServer(_Server):
    mode = PartialObliviousMode

    def Evaluate(self, elements, info: bytes, rnd=None):
        return self._evaluate(elements, info, rnd)

    def FullEvaluate(self, inp: bytes, info: bytes) -> bytes:
        return self._full(inp, info)

    def VerifyFinalize(self, inp: bytes, info: bytes, expected: bytes) -> bool:
        return self._verify(inp, info, expected)


_ORDERS = {
    "P256-SHA256": 0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551,
    "P384-SHA384": 0xffffffffffffffffffffffffffffffffffffffffffffffffc7634d81f4372ddf581a0db248b0a77aecec196accc52973,
    "P521-SHA512": 0x01fffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffa51868783bf2f966b7fcc0148f709a5d03bb5c9b8899c47aebb6fb71e91386409,
}


def NewServer(suite: Suite, key: PrivateKey) -> Server:
    return Server(suite, key)


def NewVerifiableServer(suite: Suite, key: PrivateKey) -> VerifiableServer:
    return VerifiableServer(suite, key)


def NewPartialObliviousServer(suite: Suite, key: PrivateKey) -> PartialObliviousServer:
    return PartialObliviousServer(suite, key)
