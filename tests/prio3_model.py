"""Prio3 (draft-irtf-cfrg-vdaf-14) in Python integers, as the reference's vdaf/prio3 computes it: TurboSHAKE128 and the
VDAF XOF (internal/prio3/xof.go), Field64 / Field128 and their NTTs (arith/fp64, arith/fp128), the FLP's Prove, Query and
Decide (internal/flp/flp.go), the five circuits (count, sum, sumvec, histogram, mhcv) and the whole VDAF: Shard, PrepInit,
PrepSharesToPrep, PrepNext, Aggregate and Unshard (internal/prio3/prio3.go).  Field elements are plain ints < p; every
wire format is the reference's (little-endian elements, seeds of 32 bytes)."""
from __future__ import annotations

SEED = 32
NONCE = 16

# ---------------------------------------------------------------- TurboSHAKE128 (Keccak-p[1600, 12], rate 168)
_RC = []
_lfsr = 1
for _r in range(24):
    _c = 0
    for _j in range(7):
        if _lfsr & 1:
            _c ^= 1 << ((1 << _j) - 1)
        _lfsr = ((_lfsr << 1) ^ (0x171 if _lfsr & 0x80 else 0)) & 0xff
    _RC.append(_c)
_ROT = [0] * 25
_x, _y = 1, 0
for _t in range(24):
    _ROT[_x + 5 * _y] = ((_t + 1) * (_t + 2) // 2) % 64
    _x, _y = _y, (2 * _x + 3 * _y) % 5
_M64 = (1 << 64) - 1


def p1600_12(a):
    """Keccak-p[1600, 12]: rounds 12..23 of Keccak-f[1600], in place on 25 lanes (index x + 5y)."""
    for r in range(12, 24):
        c = [a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20] for x in range(5)]
        d = [c[(x + 4) % 5] ^ (((c[(x + 1) % 5] << 1) | (c[(x + 1) % 5] >> 63)) & _M64) for x in range(5)]
        b = [0] * 25
        for i in range(25):
            x, y = i % 5, i // 5
            v = a[i] ^ d[x]
            s = _ROT[i]
            b[y + 5 * ((2 * x + 3 * y) % 5)] = ((v << s) | (v >> (64 - s))) & _M64 if s else v
        for y in range(0, 25, 5):
            for x in range(5):
                a[y + x] = b[y + x] ^ (~b[y + (x + 1) % 5] & b[y + (x + 2) % 5] & _M64)
        a[0] ^= _RC[r]


class TurboShake128:
    """Incremental TurboSHAKE128 with domain byte D: absorb with write(), then read() squeezes."""
    RATE = 168

    def __init__(self, d=1):
        self.d = d
        self.buf = bytearray()
        self.st = None
        self.out = b""

    def write(self, b):
        assert self.st is None
        self.buf += b
        return self

    def _absorb(self):
        m = bytes(self.buf) + bytes([self.d])
        m += bytes(-len(m) % self.RATE)
        m = bytearray(m)
        m[-1] ^= 0x80
        a = [0] * 25
        for o in range(0, len(m), self.RATE):
            for i in range(21):
                a[i] ^= int.from_bytes(m[o + 8 * i:o + 8 * i + 8], "little")
            p1600_12(a)
        self.st = a

    def read(self, n):
        if self.st is None:
            self._absorb()
        while len(self.out) < n:
            self.out += b"".join(x.to_bytes(8, "little") for x in self.st[:21])
            p1600_12(self.st)
        r, self.out = self.out[:n], self.out[n:]
        return r


def turboshake128(m, n, d=1):
    return TurboShake128(d).write(m).read(n)


# ---------------------------------------------------------------- fields
class Field:
    def __init__(self, name, p, size, gen, two_adicity):
        self.name, self.p, self.size, self.gen, self.k = name, p, size, gen, two_adicity

    def root(self, n):
        """principal root of unity of order 2^n"""
        assert n <= self.k
        return pow(self.gen, 1 << (self.k - n), self.p)

    def inv(self, x):
        return pow(x, self.p - 2, self.p)

    def enc(self, v):
        return b"".join(x.to_bytes(self.size, "little") for x in v)

    def dec(self, b):
        """elements of b, or None when one is not canonical (UnmarshalBinary)"""
        assert len(b) % self.size == 0
        v = [int.from_bytes(b[i:i + self.size], "little") for i in range(0, len(b), self.size)]
        return None if any(x >= self.p for x in v) else v

    def ntt(self, vals, n):
        """out[k] = sum_j vals[j] w^(jk), w = root(log2 n) (Vec.NTT; vals shorter than n are zero-padded)"""
        w = self.root(n.bit_length() - 1)
        v = list(vals) + [0] * (n - len(vals))
        return [sum(v[j] * pow(w, j * k, self.p) for j in range(n)) % self.p for k in range(n)] if n <= 8 else \
            self._fast_ntt(v, w)

    def _fast_ntt(self, v, w):
        n = len(v)
        if n == 1:
            return v[:]
        p = self.p
        ev, od = self._fast_ntt(v[0::2], w * w % p), self._fast_ntt(v[1::2], w * w % p)
        out, t = [0] * n, 1
        for k in range(n // 2):
            a, b = ev[k], od[k] * t % p
            out[k], out[k + n // 2] = (a + b) % p, (a - b) % p
            t = t * w % p
        return out

    def inv_ntt(self, vals, n):
        """Vec.InvNTT: NTT then reverse out[1:] (no 1/n factor)"""
        o = self.ntt(vals, n)
        return [o[0]] + o[1:][::-1]


F64 = Field("Field64", 2**64 - 2**32 + 1, 8, pow(7, (2**64 - 2**32) >> 32, 2**64 - 2**32 + 1), 32)
_P128 = 2**128 - 28 * 2**64 + 1
F128 = Field("Field128", _P128, 16, pow(7, (_P128 - 1) >> 66, _P128), 66)


def next_pow2(n):
    """math.NextPow2: (N, log2 N) with N the least power of two >= n"""
    if n & (n - 1) == 0:
        return n, n.bit_length() - 1
    return 1 << n.bit_length(), n.bit_length()


def poly_eval(c, x, p):
    r = 0
    for a in reversed(c):
        r = (r * x + a) % p
    return r


def poly_mul(a, b, p):
    out = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            out[i + j] = (out[i + j] + x * y) % p
    return out


# ---------------------------------------------------------------- gadgets
class Mul:
    arity, degree = 2, 2

    def eval(self, F, x):
        return x[0] * x[1] % F.p

    def eval_poly(self, F, polys):
        return poly_mul(polys[0], polys[1], F.p)


class PolyEvalX2X:
    arity, degree = 1, 2

    def eval(self, F, x):
        return (x[0] * x[0] - x[0]) % F.p

    def eval_poly(self, F, polys):
        sq = poly_mul(polys[0], polys[0], F.p)
        return [(sq[i] - (polys[0][i] if i < len(polys[0]) else 0)) % F.p for i in range(len(sq))]


class ParallelSumMul:
    degree = 2

    def __init__(self, count):
        self.count = count
        self.arity = 2 * count

    def eval(self, F, x):
        return sum(x[2 * j] * x[2 * j + 1] for j in range(self.count)) % F.p

    def eval_poly(self, F, polys):
        out = None
        for j in range(self.count):
            t = poly_mul(polys[2 * j], polys[2 * j + 1], F.p)
            out = t if out is None else [(a + b) % F.p for a, b in zip(out, t)]
        return out


class _Wrap:
    """the FLP's gadget wrapper: records each call's inputs as wire values at points alpha^k"""

    def __init__(self, F, gadget, calls, seeds):
        self.F, self.g = F, gadget
        self.p, self.log2p = next_pow2(1 + calls)
        self.wires = [[s] + [0] * (self.p - 1) for s in seeds]
        self.k = 0

    def record(self, x):
        self.k += 1
        for i, v in enumerate(x):
            self.wires[i][self.k] = v


class ProveGadget(_Wrap):
    def __call__(self, x):
        self.record(x)
        return self.g.eval(self.F, x)


class QueryGadget(_Wrap):
    def __init__(self, F, gadget, calls, seeds, poly):
        super().__init__(F, gadget, calls, seeds)
        self.poly = poly
        self.alpha = F.root(self.log2p)

    def __call__(self, x):
        self.record(x)
        return poly_eval(self.poly, pow(self.alpha, self.k, self.F.p), self.F.p)


# ---------------------------------------------------------------- circuits
class Circuit:
    """one FLP validity circuit; subclasses set the lengths and define eval / encode / truncate / decode"""
    F = None
    joint_rand_len = 0

    def gadget_poly_len(self):
        p, _ = next_pow2(1 + self.calls)
        return 1 + self.gadget.degree * (p - 1)

    @property
    def prove_rand_len(self):
        return self.gadget.arity

    @property
    def proof_len(self):
        return self.gadget.arity + self.gadget_poly_len()

    @property
    def verifier_len(self):
        return 2 + self.gadget.arity

    @property
    def query_rand_len(self):
        return 1 + self.eval_output_len

    def prove(self, meas, prove_rand, joint_rand):
        F = self.F
        g = ProveGadget(F, self.gadget, self.calls, prove_rand[:self.gadget.arity])
        self.eval(g, meas, joint_rand, 1)
        inv_n = F.inv(g.p)
        polys = [[c * inv_n % F.p for c in F.inv_ntt(w, g.p)] for w in g.wires]
        proof = [w[0] for w in g.wires]
        gp = self.gadget.eval_poly(F, polys)
        gp = gp + [0] * (self.gadget_poly_len() - len(gp))
        return proof + gp[:self.gadget_poly_len()]

    def query(self, meas_share, proof_share, query_rand, joint_rand, shares):
        """the verifier share, or None for ErrInvalidEval (t^p = 1)"""
        F = self.F
        a = self.gadget.arity
        g = QueryGadget(F, self.gadget, self.calls, proof_share[:a], proof_share[a:a + self.gadget_poly_len()])
        out = self.eval(g, meas_share, joint_rand, shares)
        n = self.eval_output_len
        if n > 1:
            v, t = sum(o * r for o, r in zip(out, query_rand[:n])) % F.p, query_rand[n]
        else:
            v, t = out[0], query_rand[0]  # the cursor is not advanced past a single output (flp.go:83-90)
        return self._checks(g, v, t)

    def _checks(self, g, v, t):
        F = self.F
        if pow(t, g.p, F.p) == 1:
            return None
        inv_n = F.inv(g.p)
        checks = [poly_eval(F.inv_ntt(w, g.p), t, F.p) * inv_n % F.p for w in g.wires]
        return [v] + checks + [poly_eval(g.poly, t, F.p)]

    def decide(self, verifier):
        F = self.F
        if verifier[0] != 0:
            return False
        a = self.gadget.arity
        return self.gadget.eval(F, verifier[1:1 + a]) == verifier[1 + a]


def _split_bits(n, bits):
    assert n.bit_length() <= bits
    return [(n >> i) & 1 for i in range(bits)]


def _range_check(F, g, calls, chunk, inv_shares, meas, jr):
    out = 0
    for i in range(calls):
        r, x = 1, []
        for j in range(chunk):
            idx = i * chunk + j
            m = meas[idx] if idx < len(meas) else 0
            r = r * jr[i] % F.p
            x += [r * m % F.p, (m - inv_shares) % F.p]
        out = (out + g(x)) % F.p
    return out


class Count(Circuit):
    ID, F = 1, F64

    def __init__(self):
        self.gadget, self.calls = Mul(), 1
        self.meas_len = self.output_len = self.eval_output_len = 1

    def eval(self, g, meas, jr, shares):
        return [(g([meas[0], meas[0]]) - meas[0]) % self.F.p]

    def encode(self, m):
        return [1 if m else 0]

    def truncate(self, meas):
        return meas

    def decode(self, out, num):
        return out[0]


class Sum(Circuit):
    ID, F = 2, F64

    def __init__(self, max_measurement):
        if max_measurement >= 1 << 63:
            raise ValueError("max measurement")
        self.max = max_measurement
        self.bits = max_measurement.bit_length()
        self.offset = (1 << self.bits) - 1 - max_measurement
        self.gadget, self.calls = PolyEvalX2X(), 2 * self.bits
        self.meas_len, self.output_len, self.eval_output_len = 2 * self.bits, 1, 2 * self.bits + 1

    def eval(self, g, meas, jr, shares):
        F = self.F
        out = [g([m]) for m in meas]
        a, b = poly_eval(meas[:self.bits], 2, F.p), poly_eval(meas[self.bits:], 2, F.p)
        return out + [(self.offset * F.inv(shares) + a - b) % F.p]

    def encode(self, m):
        assert m <= self.max
        return _split_bits(m, self.bits) + _split_bits(m + self.offset, self.bits)

    def truncate(self, meas):
        return [poly_eval(meas[:self.bits], 2, self.F.p)]

    def decode(self, out, num):
        return out[0]


class _RangeChecked(Circuit):
    F = F128

    def _init(self, chunk, meas_len, output_len, eval_output_len, calls):
        self.chunk = chunk
        self.gadget, self.calls = ParallelSumMul(chunk), calls
        self.meas_len, self.output_len, self.eval_output_len = meas_len, output_len, eval_output_len
        self.joint_rand_len = calls

    def decode(self, out, num):
        return list(out)


class SumVec(_RangeChecked):
    ID = 3

    def __init__(self, length, bits, chunk):
        if length == 0 or bits == 0 or bits > 64 or chunk == 0:
            raise ValueError("sumvec parameters")
        self.length, self.bits = length, bits
        self._init(chunk, length * bits, length, 1, (length * bits + chunk - 1) // chunk)

    def eval(self, g, meas, jr, shares):
        return [_range_check(self.F, g, self.calls, self.chunk, self.F.inv(shares), meas, jr)]

    def encode(self, m):
        return [b for x in m for b in _split_bits(x, self.bits)]

    def truncate(self, meas):
        return [poly_eval(meas[i * self.bits:(i + 1) * self.bits], 2, self.F.p) for i in range(self.length)]


class Histogram(_RangeChecked):
    ID = 4

    def __init__(self, length, chunk):
        if length == 0 or chunk == 0:
            raise ValueError("histogram parameters")
        self.length = length
        self._init(chunk, length, length, 2, (length + chunk - 1) // chunk)

    def eval(self, g, meas, jr, shares):
        F = self.F
        inv = F.inv(shares)
        return [_range_check(F, g, self.calls, self.chunk, inv, meas, jr), (sum(meas) - inv) % F.p]

    def encode(self, m):
        assert m < self.length
        return [1 if i == m else 0 for i in range(self.length)]

    def truncate(self, meas):
        return meas


class MultiHotCountVec(_RangeChecked):
    ID = 5

    def __init__(self, length, max_weight, chunk):
        if length == 0 or max_weight > length or chunk == 0:
            raise ValueError("mhcv parameters")
        self.length, self.bits = length, max_weight.bit_length()
        self.offset = (1 << self.bits) - 1 - max_weight
        if F128.p - self.offset <= length:
            raise ValueError("field size")
        self._init(chunk, length + self.bits, length, 2, (length + self.bits + chunk - 1) // chunk)

    def eval(self, g, meas, jr, shares):
        F = self.F
        inv = F.inv(shares)
        rc = _range_check(F, g, self.calls, self.chunk, inv, meas, jr)
        w = sum(meas[:self.length]) % F.p
        rep = poly_eval(meas[self.length:], 2, F.p)
        return [rc, (self.offset * inv + w - rep) % F.p]

    def encode(self, m):
        assert len(m) == self.length
        return [1 if b else 0 for b in m] + _split_bits(self.offset + sum(1 for b in m if b), self.bits)

    def truncate(self, meas):
        return meas[:self.length]


# ---------------------------------------------------------------- the VDAF
(U_MEAS_SHARE, U_PROOF_SHARE, U_JOINT_RAND, U_PROVE_RAND, U_QUERY_RAND, U_JOINT_RAND_SEED,
 U_JOINT_RAND_PART) = range(1, 8)

ERR_DECODE, ERR_JOINT_RAND, ERR_INVALID_EVAL, ERR_PROOF_VERIFY = 1, 2, 4, 8


class Prio3:
    def __init__(self, circuit, shares, ctx=b""):
        if shares < 2 or shares > 255:
            raise ValueError("ErrNumShares")
        if len(ctx) > 65535 - 8:
            raise ValueError("ErrContextSize")
        self.c, self.shares, self.ctx = circuit, shares, ctx
        self.F = circuit.F
        self.jr = circuit.joint_rand_len > 0

    # ---- XOF (xof.go)
    def xof(self, usage, seed, *binder):
        dst = bytes([12, 0]) + self.c.ID.to_bytes(4, "big") + usage.to_bytes(2, "big") + self.ctx
        x = TurboShake128(1).write(len(dst).to_bytes(2, "little") + dst + bytes([SEED]) + seed)
        for b in binder:
            x.write(b)
        return x

    def vec(self, x, n):
        F, out = self.F, []
        while len(out) < n:
            v = int.from_bytes(x.read(F.size), "little")
            if v < F.p:
                out.append(v)
        return out

    def helper_meas(self, seed, agg):
        return self.vec(self.xof(U_MEAS_SHARE, seed, bytes([agg])), self.c.meas_len)

    def helper_proof(self, seed, agg):
        return self.vec(self.xof(U_PROOF_SHARE, seed, bytes([1, agg])), self.c.proof_len)

    def joint_rand_part(self, blind, agg, nonce, meas_enc):
        return self.xof(U_JOINT_RAND_PART, blind, bytes([agg]), nonce, meas_enc).read(SEED)

    def joint_rand_seed(self, parts):
        return self.xof(U_JOINT_RAND_SEED, bytes(SEED), parts).read(SEED)

    def joint_rands(self, seed):
        return self.vec(self.xof(U_JOINT_RAND, seed, bytes([1])), self.c.joint_rand_len)

    def query_rands(self, vk, nonce):
        return self.vec(self.xof(U_QUERY_RAND, vk, bytes([1]), nonce), self.c.query_rand_len)

    # ---- wire sizes
    def sizes(self):
        F, c, j = self.F.size, self.c, SEED if self.jr else 0
        return dict(input_share_leader=F * (c.meas_len + c.proof_len) + j, input_share_helper=SEED + j,
                    public_share=self.shares * SEED if self.jr else 0, prep_share=F * c.verifier_len + j,
                    prep_msg=j, prep_state=F * c.output_len + j, out_share=F * c.output_len,
                    agg_share=F * c.output_len)

    def rand_size(self):
        return SEED * self.shares * (2 if self.jr else 1)

    # ---- Shard (client)
    def shard(self, measurement, nonce, rand):
        F, c, S = self.F, self.c, self.shares
        assert len(rand) == self.rand_size()
        meas = c.encode(measurement)
        cur = 0

        def nxt():
            nonlocal cur
            cur += SEED
            return rand[cur - SEED:cur]
        helpers = [(nxt(), nxt() if self.jr else None) for _ in range(1, S)]
        leader_blind = nxt() if self.jr else None
        meas_l = list(meas)
        parts = [b""] * S
        for i, (seed, blind) in enumerate(helpers, 1):
            m = self.helper_meas(seed, i)
            if self.jr:
                parts[i] = self.joint_rand_part(blind, i, nonce, F.enc(m))
            meas_l = [(a - b) % F.p for a, b in zip(meas_l, m)]
        if self.jr:
            parts[0] = self.joint_rand_part(leader_blind, 0, nonce, F.enc(meas_l))
        prove_rand = self.vec(self.xof(U_PROVE_RAND, nxt(), bytes([1])), c.prove_rand_len)
        jr = self.joint_rands(self.joint_rand_seed(b"".join(parts))) if self.jr else []
        proof_l = c.prove(meas, prove_rand, jr)
        for i, (seed, _) in enumerate(helpers, 1):
            proof_l = [(a - b) % F.p for a, b in zip(proof_l, self.helper_proof(seed, i))]
        public = b"".join(parts)
        inputs = [F.enc(meas_l) + F.enc(proof_l) + (leader_blind or b"")]
        inputs += [seed + (blind or b"") for seed, blind in helpers]
        return public, inputs

    # ---- PrepInit (aggregator)
    def prep_init(self, vk, agg, nonce, public, input_share):
        """(status, prep_state, prep_share); on a nonzero status both rows are all zero"""
        F, c = self.F, self.c
        sz = self.sizes()
        bad = (0, bytes(sz["prep_state"]), bytes(sz["prep_share"]))
        if agg == 0:
            nm = F.size * c.meas_len
            meas = F.dec(input_share[:nm])
            proof = F.dec(input_share[nm:nm + F.size * c.proof_len])
            if meas is None or proof is None:
                return (ERR_DECODE,) + bad[1:]
            blind = input_share[nm + F.size * c.proof_len:] if self.jr else None
        else:
            seed = input_share[:SEED]
            meas, proof = self.helper_meas(seed, agg), self.helper_proof(seed, agg)
            blind = input_share[SEED:2 * SEED] if self.jr else None
        state = F.enc(c.truncate(meas))
        jr, part = [], b""
        if self.jr:
            part = self.joint_rand_part(blind, agg, nonce, F.enc(meas))
            if public[agg * SEED:(agg + 1) * SEED] != part:
                return (ERR_JOINT_RAND,) + bad[1:]
            corrected = public[:agg * SEED] + part + public[(agg + 1) * SEED:]
            cseed = self.joint_rand_seed(corrected)
            state += cseed
            jr = self.joint_rands(cseed)
        qr = self.query_rands(vk, nonce)
        ver = c.query(meas, proof, qr, jr, self.shares)
        if ver is None:
            return (ERR_INVALID_EVAL,) + bad[1:]
        return 0, state, F.enc(ver) + part

    def prep_shares_to_prep(self, prep_shares):
        """(status, prep_msg)"""
        F, c = self.F, self.c
        n = F.size * c.verifier_len
        vs = [F.dec(s[:n]) for s in prep_shares]
        if any(v is None for v in vs):
            return ERR_DECODE, bytes(self.sizes()["prep_msg"])
        ver = [sum(col) % F.p for col in zip(*vs)]
        if not c.decide(ver):
            return ERR_PROOF_VERIFY, bytes(self.sizes()["prep_msg"])
        if not self.jr:
            return 0, b""
        return 0, self.joint_rand_seed(b"".join(s[n:] for s in prep_shares))

    def prep_next(self, state, msg):
        """(status, out_share)"""
        n = self.F.size * self.c.output_len
        if self.jr and state[n:] != msg:
            return ERR_JOINT_RAND, bytes(n)
        return 0, state[:n]

    def aggregate(self, out_shares):
        F = self.F
        acc = [0] * self.c.output_len
        for o in out_shares:
            acc = [(a + b) % F.p for a, b in zip(acc, F.dec(o))]
        return F.enc(acc)

    def unshard(self, agg_shares, num):
        return self.c.decode(self.F.dec(self.aggregate(agg_shares)), num)


def from_vector(name, v):
    """the Prio3 instance a reference vector file describes"""
    ctx = bytes.fromhex(v["ctx"])
    kind = name.split("_")[0]
    if kind == "Count":
        c = Count()
    elif kind == "Sum":
        c = Sum(v["max_measurement"])
    elif kind == "SumVec":
        c = SumVec(v["length"], v["bits"], v["chunk_length"])
    elif kind == "Histogram":
        c = Histogram(v["length"], v["chunk_length"])
    else:
        c = MultiHotCountVec(v["length"], v["max_weight"], v["chunk_length"])
    return Prio3(c, v["shares"], ctx)


VECTOR_FILES = ["Count_0", "Count_1", "Count_2", "Sum_0", "Sum_1", "Sum_2", "SumVec_0", "SumVec_1", "Histogram_0",
                "Histogram_1", "Histogram_2", "MultihotCountVec_0", "MultihotCountVec_1", "MultihotCountVec_2"]
