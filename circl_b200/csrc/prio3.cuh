// Prio3 aggregator arithmetic (draft-irtf-cfrg-vdaf-14), one thread per report: the reference's vdaf/prio3 for Count,
// Sum, SumVec, Histogram and MultiHotCountVec.  Mirrors arith/fp64 and arith/fp128 (Field64 p = 2^64 - 2^32 + 1,
// Field128 p = 2^128 - 28 * 2^64 + 1), internal/prio3/xof.go (TurboSHAKE128 with the VDAF header), internal/flp/flp.go
// (Query, Decide), internal/flp/gadgets.go and the circuits' Eval.
//
//   fields   Montgomery form in 64-bit limbs (R = 2^64 / 2^128), products through unsigned __int128; every reduction
//            and correction is a mask, not a branch
//   XOF      TurboSHAKE128(D = 1) of LE16(len dst) || dst || 32 || seed || binder, dst = 12 || 0 || BE32(kind) ||
//            BE16(usage) || context; elements by rejection of 8- or 16-byte little-endian strings >= p
//   Query    the reference interpolates each wire over the 2^k-point domain and evaluates at t, and evaluates the
//            gadget polynomial at alpha^k for every call (O(calls * p) by Horner).  Here, with the same exact results:
//              - the gadget polynomial (2p - 1 coefficients) is folded mod x^p - 1 and one forward NTT of size p gives
//                its value at every alpha^k;
//              - every wire check is sum_k wire_k L_k(t) with the Lagrange weights
//                L_k(t) = (t^p - 1) / p * alpha^k / (t - alpha^k), computed once per report with one batched
//                inversion (t^p != 1 makes every t - alpha^k nonzero), so the wires are accumulated as the circuit
//                runs and never stored.
//
// Constant time: a share value (measurement, proof, joint randomness, verify-key output) reaches no branch and no
// address.  Loop bounds and addresses depend only on the public configuration.  The exceptions are public by
// construction: the XOF's rejection test (the reference's too; a rejected string is discarded output), the t^p = 1
// test and the status of a report, which are reported to the caller.
//
// Plain integer C++: the field code compiles for the device and the host.  The XOF and everything above it are device
// code under nvcc (the permutation is keccak.cuh's f1600 with 12 rounds); a host build (the CPU test) supplies
// cb200::keccak::f1600 itself.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#include "keccak.cuh"
#define P3_XHD __host__ __device__ __forceinline__
#define P3_D __device__ __forceinline__
#else
#define P3_XHD inline
#define P3_D inline
namespace cb200 {
namespace keccak {
void f1600(uint64_t (&a)[25], int first_round);
}
}  // namespace cb200
#endif

namespace cb200 {
namespace prio3 {

typedef unsigned __int128 u128;

// kinds (the reference's algorithm IDs) and status bits of a report
enum { kCount = 1, kSum = 2, kSumVec = 3, kHistogram = 4, kMultiHot = 5 };
enum { kErrDecode = 1, kErrJointRand = 2, kErrInvalidEval = 4, kErrProofVerify = 8 };
constexpr int kSeed = 32, kNonce = 16;

// ---------------------------------------------------------------- fields
struct F64 {
  static constexpr int N = 1, kBytes = 8, kTwoAdic = 32;
  P3_XHD static uint64_t p(int) { return 0xffffffff00000001ull; }
  P3_XHD static uint64_t r2(int) { return 0xfffffffe00000001ull; }
  P3_XHD static uint64_t one(int) { return 0x00000000ffffffffull; }
  P3_XHD static uint64_t gen(int) { return 0xda58878b0d514e98ull; }  // root of unity of order 2^32, Montgomery form
  P3_XHD static uint64_t half(int) { return 0x8000000000000000ull; }
  static constexpr uint64_t kNinv = 0xfffffffeffffffffull;  // -p^-1 mod 2^64
};
struct F128 {
  static constexpr int N = 2, kBytes = 16, kTwoAdic = 66;
  P3_XHD static uint64_t p(int i) { return i ? 0xffffffffffffffe4ull : 1ull; }
  P3_XHD static uint64_t r2(int i) { return i ? 0x5587ull : 0xfffffffffffffcf1ull; }
  P3_XHD static uint64_t one(int i) { return i ? 0x1bull : 0xffffffffffffffffull; }
  P3_XHD static uint64_t gen(int i) { return i ? 0x50f8f7f554db309cull : 0xf0111fb98c6b9875ull; }  // order 2^66
  P3_XHD static uint64_t half(int i) { return i ? 0x8000000000000000ull : 0ull; }
  static constexpr uint64_t kNinv = 0xffffffffffffffffull;
};

template <class F>
struct Fe {
  uint64_t v[F::N];
};

// t (N limbs) + carry bit c, known < 2p: t - p if that does not borrow or c is set
template <class F>
P3_XHD Fe<F> reduce_once(const uint64_t* t, uint64_t c) {
  Fe<F> s;
  uint64_t borrow = 0;
  for (int i = 0; i < F::N; i++) {
    const u128 d = (u128)t[i] - F::p(i) - borrow;
    s.v[i] = (uint64_t)d;
    borrow = (uint64_t)(d >> 64) & 1;
  }
  const uint64_t keep = 0 - (borrow & (c ^ 1));  // all ones: t < p, keep t
  for (int i = 0; i < F::N; i++) s.v[i] = (t[i] & keep) | (s.v[i] & ~keep);
  return s;
}
template <class F>
P3_XHD Fe<F> add(const Fe<F>& a, const Fe<F>& b) {
  uint64_t t[F::N], c = 0;
  for (int i = 0; i < F::N; i++) {
    const u128 s = (u128)a.v[i] + b.v[i] + c;
    t[i] = (uint64_t)s;
    c = (uint64_t)(s >> 64);
  }
  return reduce_once<F>(t, c);
}
template <class F>
P3_XHD Fe<F> sub(const Fe<F>& a, const Fe<F>& b) {
  Fe<F> d;
  uint64_t borrow = 0;
  for (int i = 0; i < F::N; i++) {
    const u128 x = (u128)a.v[i] - b.v[i] - borrow;
    d.v[i] = (uint64_t)x;
    borrow = (uint64_t)(x >> 64) & 1;
  }
  const uint64_t m = 0 - borrow;
  uint64_t c = 0;
  for (int i = 0; i < F::N; i++) {
    const u128 s = (u128)d.v[i] + (F::p(i) & m) + c;
    d.v[i] = (uint64_t)s;
    c = (uint64_t)(s >> 64);
  }
  return d;
}
// Montgomery product a b R^-1 (CIOS)
template <class F>
P3_XHD Fe<F> mul(const Fe<F>& a, const Fe<F>& b) {
  constexpr int N = F::N;
  uint64_t t[N + 2];
  for (int i = 0; i < N + 2; i++) t[i] = 0;
  for (int i = 0; i < N; i++) {
    u128 c = 0;
    for (int j = 0; j < N; j++) {
      c += (u128)a.v[j] * b.v[i] + t[j];
      t[j] = (uint64_t)c;
      c >>= 64;
    }
    c += t[N];
    t[N] = (uint64_t)c;
    t[N + 1] = (uint64_t)(c >> 64);
    const uint64_t m = t[0] * F::kNinv;
    c = ((u128)m * F::p(0) + t[0]) >> 64;
    for (int j = 1; j < N; j++) {
      c += (u128)m * F::p(j) + t[j];
      t[j - 1] = (uint64_t)c;
      c >>= 64;
    }
    c += t[N];
    t[N - 1] = (uint64_t)c;
    t[N] = t[N + 1] + (uint64_t)(c >> 64);
  }
  return reduce_once<F>(t, t[N]);
}
template <class F>
P3_XHD Fe<F> zero() {
  Fe<F> z;
  for (int i = 0; i < F::N; i++) z.v[i] = 0;
  return z;
}
template <class F>
P3_XHD Fe<F> one() {
  Fe<F> z;
  for (int i = 0; i < F::N; i++) z.v[i] = F::one(i);
  return z;
}
template <class F>
P3_XHD Fe<F> to_mont(const Fe<F>& a) {
  Fe<F> r2;
  for (int i = 0; i < F::N; i++) r2.v[i] = F::r2(i);
  return mul<F>(a, r2);
}
template <class F>
P3_XHD Fe<F> from_mont(const Fe<F>& a) {
  Fe<F> u = zero<F>();
  u.v[0] = 1;
  return mul<F>(a, u);
}
template <class F>
P3_XHD Fe<F> from_u64(uint64_t n) {  // n < p
  Fe<F> a = zero<F>();
  a.v[0] = n;
  return to_mont<F>(a);
}
template <class F>
P3_XHD uint64_t is_zero(const Fe<F>& a) {  // 1 or 0
  uint64_t acc = 0;
  for (int i = 0; i < F::N; i++) acc |= a.v[i];
  return ((acc | (0 - acc)) >> 63) ^ 1;
}
template <class F>
P3_XHD uint64_t is_equal(const Fe<F>& a, const Fe<F>& b) {
  return is_zero<F>(sub<F>(a, b));
}
// a^e for a public exponent of up to 128 bits (e_hi:e_lo)
template <class F>
P3_XHD Fe<F> pow(const Fe<F>& a, uint64_t e_lo, uint64_t e_hi) {
  Fe<F> r = one<F>();
  for (int i = 127; i >= 0; i--) {
    r = mul<F>(r, r);
    const uint64_t bit = i >= 64 ? (e_hi >> (i - 64)) & 1 : (e_lo >> i) & 1;
    if (bit) r = mul<F>(r, a);
  }
  return r;
}
template <class F>
P3_XHD Fe<F> inv(const Fe<F>& a) {  // a^(p - 2); 0 maps to 0
  if (F::N == 1) return pow<F>(a, F::p(0) - 2, 0);
  return pow<F>(a, F::p(0) - 2, F::p(1) - (F::p(0) < 2));
}
// principal root of unity of order 2^n (n <= kTwoAdic): the generator squared kTwoAdic - n times
template <class F>
P3_XHD Fe<F> root(int n) {
  Fe<F> w;
  for (int i = 0; i < F::N; i++) w.v[i] = F::gen(i);
  for (int i = n; i < F::kTwoAdic; i++) w = mul<F>(w, w);
  return w;
}
template <class F>
P3_XHD Fe<F> inv_two_n(int n) {  // 2^-n
  Fe<F> h, r = one<F>();
  for (int i = 0; i < F::N; i++) h.v[i] = F::half(i);
  for (int i = 0; i < n; i++) r = mul<F>(r, h);
  return r;
}

// little-endian canonical encoding; load returns 1 when the string is < p (UnmarshalBinary), else 0 and some element
template <class F>
P3_XHD void store(uint8_t* out, const Fe<F>& a) {
  const Fe<F> x = from_mont<F>(a);
  for (int i = 0; i < F::N; i++)
    for (int j = 0; j < 8; j++) out[8 * i + j] = (uint8_t)(x.v[i] >> (8 * j));
}
template <class F>
P3_XHD uint64_t in_range(const Fe<F>& x) {  // x < p, as 1 or 0
  uint64_t borrow = 0;
  for (int i = 0; i < F::N; i++) {
    const u128 d = (u128)x.v[i] - F::p(i) - borrow;
    borrow = (uint64_t)(d >> 64) & 1;
  }
  return borrow;
}
template <class F>
P3_XHD uint64_t load(Fe<F>& a, const uint8_t* in) {
  Fe<F> x;
  for (int i = 0; i < F::N; i++) {
    uint64_t w = 0;
    for (int j = 0; j < 8; j++) w |= (uint64_t)in[8 * i + j] << (8 * j);
    x.v[i] = w;
  }
  const uint64_t ok = in_range<F>(x);
  a = to_mont<F>(x);
  return ok;
}

// in-place forward NTT of size n = 2^logn over a[] in natural order: a[k] <- sum_j a[j] w^(jk) (Vec.NTT)
template <class F>
P3_XHD void ntt(Fe<F>* a, int logn) {
  const uint64_t n = 1ull << logn;
  for (uint64_t i = 1, j = 0; i < n; i++) {  // bit-reversal permutation
    uint64_t bit = n >> 1;
    for (; j & bit; bit >>= 1) j ^= bit;
    j ^= bit;
    if (i < j) {
      const Fe<F> t = a[i];
      a[i] = a[j];
      a[j] = t;
    }
  }
  for (int l = 1; l <= logn; l++) {
    const uint64_t y = 1ull << (l - 1);
    const Fe<F> wn = root<F>(l);
    Fe<F> w = one<F>();
    for (uint64_t i = 0; i < y; i++) {
      for (uint64_t x = i; x < n; x += 2 * y) {
        const Fe<F> u = a[x], t = mul<F>(w, a[x + y]);
        a[x] = add<F>(u, t);
        a[x + y] = sub<F>(u, t);
      }
      w = mul<F>(w, wn);
    }
  }
}

// ---------------------------------------------------------------- configuration (public, uniform over a call)
struct Cfg {
  uint32_t kind, shares;
  uint32_t meas_len, out_len, eval_out_len, proof_len, verifier_len, jr_len, arity, calls;
  uint32_t chunk, bits, length, log2p;
  uint64_t offset;          // Sum / MultiHotCountVec: 2^bits - 1 - max
  uint64_t work;            // field elements of work area per report (prep_init)
  const uint8_t* ctx;       // context string (device memory under nvcc)
  uint32_t ctxlen;
  P3_XHD uint32_t poly_len() const { return 1 + 2 * ((1u << log2p) - 1); }
};

// ---------------------------------------------------------------- TurboSHAKE128 XOF
struct Xof {
  uint64_t a[25];
  int pos;  // byte position in the 168-byte rate
};
P3_D void xof_byte(Xof& x, uint8_t b) {
  x.a[x.pos >> 3] ^= (uint64_t)b << (8 * (x.pos & 7));
  if (++x.pos == 168) {
    keccak::f1600(x.a, 12);
    x.pos = 0;
  }
}
P3_D void xof_bytes(Xof& x, const uint8_t* b, int n) {
  for (int i = 0; i < n; i++) xof_byte(x, b[i]);
}
template <class F>
P3_D void xof_elt(Xof& x, const Fe<F>& e) {
  uint8_t b[F::kBytes];
  store<F>(b, e);
  xof_bytes(x, b, F::kBytes);
}
// Init(usage, seed): the header and the seed
P3_D void xof_init(Xof& x, const Cfg& c, int usage, const uint8_t* seed) {
  for (int i = 0; i < 25; i++) x.a[i] = 0;
  x.pos = 0;
  const uint32_t dl = 8 + c.ctxlen;
  const uint8_t h[12] = {(uint8_t)dl, (uint8_t)(dl >> 8), 12, 0, (uint8_t)(c.kind >> 24), (uint8_t)(c.kind >> 16),
                         (uint8_t)(c.kind >> 8), (uint8_t)c.kind, (uint8_t)(usage >> 8), (uint8_t)usage};
  xof_bytes(x, h, 10);
  xof_bytes(x, c.ctx, (int)c.ctxlen);
  xof_byte(x, (uint8_t)kSeed);
  xof_bytes(x, seed, kSeed);
}
// end of the input: domain byte 1 and the final 0x80
P3_D void xof_finish(Xof& x) {
  x.a[x.pos >> 3] ^= (uint64_t)1 << (8 * (x.pos & 7));
  x.a[20] ^= 0x80ull << 56;
  keccak::f1600(x.a, 12);
  x.pos = 0;
}
P3_D uint64_t xof_u64(Xof& x) {
  if (x.pos == 168) {
    keccak::f1600(x.a, 12);
    x.pos = 0;
  }
  const uint64_t v = x.a[x.pos >> 3];
  x.pos += 8;
  return v;
}
P3_D void xof_seed(Xof& x, uint8_t* out) {
  for (int i = 0; i < 4; i++) {
    const uint64_t v = xof_u64(x);
    for (int j = 0; j < 8; j++) out[8 * i + j] = (uint8_t)(v >> (8 * j));
  }
}
// next field element by rejection sampling (RandomSHA3); the test is on public XOF output that is discarded
template <class F>
P3_D Fe<F> xof_fe(Xof& x) {
  for (;;) {
    Fe<F> e;
    for (int i = 0; i < F::N; i++) e.v[i] = xof_u64(x);
    if (in_range<F>(e)) return to_mont<F>(e);
  }
}
enum { kUMeasShare = 1, kUProofShare, kUJointRand, kUProveRand, kUQueryRand, kUJointRandSeed, kUJointRandPart };

// ---------------------------------------------------------------- FLP Query (streaming form)
// Per-report state of the query gadget: wire checks accumulate L_k * input as each call k is made, and call k returns
// the gadget polynomial's value at alpha^k (G[k]).
template <class F>
struct Query {
  const Fe<F>* L;  // p Lagrange weights at t
  const Fe<F>* G;  // p gadget values
  Fe<F>* wc;       // arity wire checks
  uint32_t k;
  P3_D Fe<F> call(const Fe<F>* x, uint32_t n) {
    k++;
    for (uint32_t i = 0; i < n; i++) wc[i] = add<F>(wc[i], mul<F>(L[k], x[i]));
    return G[k];
  }
  // one input at a time, for the ParallelSum gadget's 2 * chunk inputs
  P3_D void wire(uint32_t i, const Fe<F>& x) { wc[i] = add<F>(wc[i], mul<F>(L[k + 1], x)); }
  P3_D Fe<F> done() { return G[++k]; }
};

// sum_i 2^i b[i] (JoinBits), Horner from the top bit
template <class F>
P3_D Fe<F> join_bits(const Fe<F>* b, uint32_t n) {
  const Fe<F> two = add<F>(one<F>(), one<F>());
  Fe<F> r = zero<F>();
  for (uint32_t i = n; i-- > 0;) r = add<F>(mul<F>(r, two), b[i]);
  return r;
}

// the circuit's Eval with the query gadget, reduced to the verifier's first element: the output itself when it has
// one element, else its dot product with the query randomness qr
template <class F>
P3_D Fe<F> eval_circuit(const Cfg& c, Query<F>& g, const Fe<F>* meas, const Fe<F>* jr, const Fe<F>* qr) {
  const Fe<F> inv_sh = inv<F>(from_u64<F>(c.shares));
  if (c.kind == kCount) {
    const Fe<F> x[2] = {meas[0], meas[0]};
    return sub<F>(g.call(x, 2), meas[0]);
  }
  if (c.kind == kSum) {
    Fe<F> v = zero<F>();
    for (uint32_t i = 0; i < c.meas_len; i++) v = add<F>(v, mul<F>(g.call(&meas[i], 1), qr[i]));
    Fe<F> rc = mul<F>(from_u64<F>(c.offset), inv_sh);
    rc = sub<F>(add<F>(rc, join_bits<F>(meas, c.bits)), join_bits<F>(meas + c.bits, c.bits));
    return c.eval_out_len == 1 ? rc : add<F>(v, mul<F>(rc, qr[c.meas_len]));  // max 0: no bits, one output
  }
  // RangeCheck (valid.go:70-97) for SumVec, Histogram and MultiHotCountVec
  Fe<F> rc = zero<F>();
  for (uint32_t i = 0; i < c.calls; i++) {
    Fe<F> r = one<F>();
    for (uint32_t j = 0; j < c.chunk; j++) {
      const uint64_t idx = (uint64_t)i * c.chunk + j;
      const Fe<F> m = idx < c.meas_len ? meas[idx] : zero<F>();
      r = mul<F>(r, jr[i]);
      g.wire(2 * j, mul<F>(r, m));
      g.wire(2 * j + 1, sub<F>(m, inv_sh));
    }
    rc = add<F>(rc, g.done());
  }
  if (c.kind == kSumVec) return rc;
  Fe<F> second;
  if (c.kind == kHistogram) {
    second = sub<F>(zero<F>(), inv_sh);
    for (uint32_t i = 0; i < c.meas_len; i++) second = add<F>(second, meas[i]);
  } else {
    second = mul<F>(from_u64<F>(c.offset), inv_sh);
    for (uint32_t i = 0; i < c.length; i++) second = add<F>(second, meas[i]);
    second = sub<F>(second, join_bits<F>(meas + c.length, c.bits));
  }
  return add<F>(mul<F>(rc, qr[0]), mul<F>(second, qr[1]));
}

// FLP Query at the point t (flp.go:70-121): the verifier share (verifier_len elements) into out, or kErrInvalidEval when
// t^p = 1.  L, G and wc are the work area's p, p and arity elements.
template <class F>
P3_D uint32_t query(const Cfg& c, const Fe<F>& t, const Fe<F>* meas, const Fe<F>* proof, const Fe<F>* jr,
                    const Fe<F>* qr, Fe<F>* L, Fe<F>* G, Fe<F>* wc, uint8_t* out) {
  constexpr int B = F::kBytes;
  const uint32_t p = 1u << c.log2p;
  Fe<F> tp = t;
  for (uint32_t i = 0; i < c.log2p; i++) tp = mul<F>(tp, tp);
  const Fe<F> tp1 = sub<F>(tp, one<F>());
  if (is_zero<F>(tp1)) return kErrInvalidEval;
  // Lagrange weights: den_k = t - alpha^k (held in G), prefix products in L, one inversion, then the backward pass
  const Fe<F> alpha = root<F>((int)c.log2p);
  Fe<F> ak = one<F>(), acc = one<F>();
  for (uint32_t k = 0; k < p; k++) {
    G[k] = sub<F>(t, ak);
    L[k] = acc;
    acc = mul<F>(acc, G[k]);
    ak = mul<F>(ak, alpha);
  }
  Fe<F> iv = inv<F>(acc);
  for (uint32_t k = p; k-- > 0;) {
    const Fe<F> d = G[k];
    L[k] = mul<F>(iv, L[k]);
    iv = mul<F>(iv, d);
  }
  const Fe<F> scale = mul<F>(tp1, inv_two_n<F>((int)c.log2p));
  ak = one<F>();
  for (uint32_t k = 0; k < p; k++) {
    L[k] = mul<F>(mul<F>(L[k], ak), scale);
    ak = mul<F>(ak, alpha);
  }
  // gadget polynomial: its value at t, and at every alpha^k through the fold mod x^p - 1 and one NTT
  const Fe<F>* poly = proof + c.arity;
  const uint32_t plen = c.poly_len();
  Fe<F> gcheck = zero<F>();
  for (uint32_t j = plen; j-- > 0;) gcheck = add<F>(mul<F>(gcheck, t), poly[j]);
  for (uint32_t k = 0; k < p; k++) G[k] = poly[k];
  for (uint32_t k = p; k < plen; k++) G[k - p] = add<F>(G[k - p], poly[k]);
  ntt<F>(G, (int)c.log2p);
  for (uint32_t i = 0; i < c.arity; i++) wc[i] = mul<F>(L[0], proof[i]);
  Query<F> g{L, G, wc, 0};
  const Fe<F> v = eval_circuit<F>(c, g, meas, jr, qr);
  // rows
  store<F>(out, v);
  for (uint32_t i = 0; i < c.arity; i++) store<F>(out + (size_t)B * (1 + i), wc[i]);
  store<F>(out + (size_t)B * (1 + c.arity), gcheck);
  return 0;
}

// Work area of one report, in field elements: meas | proof | jr | qr | L (p) | G (p) | wc (arity)
P3_XHD uint64_t work_elems(const Cfg& c) {
  const uint64_t p = 1ull << c.log2p;
  return (uint64_t)c.meas_len + c.proof_len + c.jr_len + c.eval_out_len + 1 + 2 * p + c.arity;
}

// PrepInit of one report.  in: the input share row (leader: meas || proof || blind; helper: seed || blind); pub: the
// public share (shares x 32 bytes, read only with joint randomness); state: out share || corrected joint-rand seed;
// share: verifier share || joint-rand part.  Returns the status; the caller zeroes the rows of a failed report.
template <class F>
P3_D uint32_t prep_init(const Cfg& c, const uint8_t* vk, uint32_t agg, const uint8_t* nonce, const uint8_t* pub,
                        const uint8_t* in, uint8_t* state, uint8_t* share, Fe<F>* w) {
  constexpr int B = F::kBytes;
  const bool jrd = c.jr_len > 0;
  const uint32_t p = 1u << c.log2p;
  Fe<F>*meas = w, *proof = meas + c.meas_len, *jr = proof + c.proof_len, *qr = jr + c.jr_len;
  Fe<F>*L = qr + c.eval_out_len + 1, *G = L + p, *wc = G + p;
  uint64_t ok = 1;
  const uint8_t* blind;
  if (agg == 0) {
    for (uint32_t i = 0; i < c.meas_len; i++) ok &= load<F>(meas[i], in + (size_t)B * i);
    for (uint32_t i = 0; i < c.proof_len; i++) ok &= load<F>(proof[i], in + (size_t)B * (c.meas_len + i));
    blind = in + (size_t)B * (c.meas_len + c.proof_len);
  } else {
    Xof x;
    const uint8_t b1[1] = {(uint8_t)agg}, b2[2] = {1, (uint8_t)agg};
    xof_init(x, c, kUMeasShare, in);
    xof_bytes(x, b1, 1);
    xof_finish(x);
    for (uint32_t i = 0; i < c.meas_len; i++) meas[i] = xof_fe<F>(x);
    xof_init(x, c, kUProofShare, in);
    xof_bytes(x, b2, 2);
    xof_finish(x);
    for (uint32_t i = 0; i < c.proof_len; i++) proof[i] = xof_fe<F>(x);
    blind = in + kSeed;
  }
  if (!ok) return kErrDecode;
  uint8_t part[kSeed], cseed[kSeed];
  if (jrd) {
    Xof x;
    const uint8_t b1[1] = {(uint8_t)agg};
    xof_init(x, c, kUJointRandPart, blind);
    xof_bytes(x, b1, 1);
    xof_bytes(x, nonce, kNonce);
    for (uint32_t i = 0; i < c.meas_len; i++) xof_elt<F>(x, meas[i]);
    xof_finish(x);
    xof_seed(x, part);
    uint8_t diff = 0;
    for (int i = 0; i < kSeed; i++) diff |= part[i] ^ pub[(size_t)agg * kSeed + i];
    if (diff) return kErrJointRand;
    const uint8_t zeros[kSeed] = {};
    xof_init(x, c, kUJointRandSeed, zeros);
    for (uint32_t s = 0; s < c.shares; s++) xof_bytes(x, s == agg ? part : pub + (size_t)s * kSeed, kSeed);
    xof_finish(x);
    xof_seed(x, cseed);
    const uint8_t one_[1] = {1};
    xof_init(x, c, kUJointRand, cseed);
    xof_bytes(x, one_, 1);
    xof_finish(x);
    for (uint32_t i = 0; i < c.jr_len; i++) jr[i] = xof_fe<F>(x);
  }
  {
    Xof x;
    const uint8_t one_[1] = {1};
    xof_init(x, c, kUQueryRand, vk);
    xof_bytes(x, one_, 1);
    xof_bytes(x, nonce, kNonce);
    xof_finish(x);
    for (uint32_t i = 0; i <= c.eval_out_len; i++) qr[i] = xof_fe<F>(x);
  }
  const uint32_t st = query<F>(c, qr[c.eval_out_len > 1 ? c.eval_out_len : 0], meas, proof, jr, qr, L, G, wc, share);
  if (st) return st;
  if (jrd)
    for (int i = 0; i < kSeed; i++) share[(size_t)B * c.verifier_len + i] = part[i];
  // Truncate
  if (c.kind == kSum) {
    store<F>(state, join_bits<F>(meas, c.bits));
  } else if (c.kind == kSumVec) {
    for (uint32_t i = 0; i < c.length; i++) store<F>(state + (size_t)B * i, join_bits<F>(meas + (size_t)i * c.bits, c.bits));
  } else {
    for (uint32_t i = 0; i < c.out_len; i++) store<F>(state + (size_t)B * i, meas[i]);
  }
  if (jrd)
    for (int i = 0; i < kSeed; i++) state[(size_t)B * c.out_len + i] = cseed[i];
  return 0;
}

// PrepSharesToPrep of one report: rows holds the shares' prep shares back to back (each `ps` bytes).  Sums the
// verifier shares, runs Decide, and derives the joint-rand seed into msg.
template <class F>
P3_D uint32_t prep_shares_to_prep(const Cfg& c, const uint8_t* rows, size_t ps, uint8_t* msg) {
  constexpr int B = F::kBytes;
  uint64_t ok = 1;
  auto sum = [&](uint32_t e) {
    Fe<F> s = zero<F>();
    for (uint32_t i = 0; i < c.shares; i++) {
      Fe<F> x;
      ok &= load<F>(x, rows + i * ps + (size_t)B * e);
      s = add<F>(s, x);
    }
    return s;
  };
  const Fe<F> v = sum(0), gcheck = sum(1 + c.arity);
  Fe<F> gv;
  if (c.kind == kSum) {
    const Fe<F> x = sum(1);
    gv = sub<F>(mul<F>(x, x), x);
  } else {  // Mul, and ParallelSum of Mul
    gv = zero<F>();
    for (uint32_t j = 0; j < c.arity / 2; j++) gv = add<F>(gv, mul<F>(sum(1 + 2 * j), sum(2 + 2 * j)));
  }
  if (!ok) return kErrDecode;
  if (!(is_zero<F>(v) & is_equal<F>(gv, gcheck))) return kErrProofVerify;
  if (c.jr_len) {
    Xof x;
    const uint8_t zeros[kSeed] = {};
    xof_init(x, c, kUJointRandSeed, zeros);
    for (uint32_t i = 0; i < c.shares; i++) xof_bytes(x, rows + i * ps + (size_t)B * c.verifier_len, kSeed);
    xof_finish(x);
    xof_seed(x, msg);
  }
  return 0;
}

}  // namespace prio3
}  // namespace cb200
