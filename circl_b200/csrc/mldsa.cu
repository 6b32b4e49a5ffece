// circl_b200/csrc/mldsa.cu -- batched ML-DSA-65 Sign on sm_90a.
//
// Replaces, per signature and bit-exactly:
//   (*PrivateKey).Unpack        sign/mldsa/mldsa65/internal/dilithium.go:142-163  (ExpandA, NTT of s1, s2, t0)
//   SignTo (ML-DSA.Sign_internal) sign/mldsa/mldsa65/internal/dilithium.go:340-470
//   external framing            sign/mldsa/mldsa65/dilithium.go:56-84  (0x00 || len(ctx) || ctx || msg)
//   samplers                    internal/sample.go:92-123 (ExpandA), :197-209 (ExpandMask), :299-339 (SampleInBall)
//   rounding / packing          internal/rounding.go:13-67, internal/pack.go:77-95,205-252, pack.go:23-86,102-108
//
// The rejection loop (dilithium.go:369-467) is run in *rounds* over the list of
// still-active signatures; every stage is a dense kernel:
//   expand (once)  ExpandA: one thread per SHAKE128 stream; s1/s2/t0: one octet per polynomial (unpack + NTT)
//   mu             one thread per op: mu = SHAKE256(tr || M'), rho' = SHAKE256(key || rnd || mu)
//   per round:     mask (thread per y polynomial) -> yntt (octet) -> w (octet per row: A y, InvNTT, Decompose)
//                  -> challenge (thread per op: c~ = H(mu || w1), SampleInBall) -> cntt (octet)
//                  -> response (octet per output polynomial: norm checks, z packing, hints)
//                  -> finalize (thread per op: accept -> pack c~/hints; reject -> next attempt)
// yNonce advances by L every attempt; the first attempt passing all four checks wins; 576 attempts cap.
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "../../include/circl_b200.h"
#include "context.h"
#include "dilithium.cuh"
#include "flow_internal.h"
#include "keccak.cuh"
#include "mldsa_internal.h"

namespace cb200 {
namespace mldsa {

using namespace dil;

// Parameter sets (sign/dilithium/gen.go:80-162).  44/65/87: ML-DSA (NIST = true, tr = 64 bytes); 2/3/5: the round-3
// Dilithium2/3/5 of sign/dilithium/mode{2,3,5} (NIST = false: tr and c~ are 32 bytes, the key seed is hashed without
// K and L, rho' = H(key || mu) without rnd, and the message is hashed as given).
template <int MODE>
struct Params;
template <>
struct Params<44> {
  static constexpr int K = 4, L = 4, ETA = 2, TAU = 39, G1BITS = 17, OMEGA = 80, CTILDE = 32;
  static constexpr uint32_t GAMMA2 = (Q - 1) / 88;
  static constexpr int TR = 64;
  static constexpr bool NIST = true;
};
template <>
struct Params<65> {
  static constexpr int K = 6, L = 5, ETA = 4, TAU = 49, G1BITS = 19, OMEGA = 55, CTILDE = 48;
  static constexpr uint32_t GAMMA2 = (Q - 1) / 32;
  static constexpr int TR = 64;
  static constexpr bool NIST = true;
};
template <>
struct Params<87> {
  static constexpr int K = 8, L = 7, ETA = 2, TAU = 60, G1BITS = 19, OMEGA = 75, CTILDE = 64;
  static constexpr uint32_t GAMMA2 = (Q - 1) / 32;
  static constexpr int TR = 64;
  static constexpr bool NIST = true;
};
template <>
struct Params<2> : Params<44> {
  static constexpr int CTILDE = 32, TR = 32;
  static constexpr bool NIST = false;
};
template <>
struct Params<3> : Params<65> {
  static constexpr int CTILDE = 32, TR = 32;
  static constexpr bool NIST = false;
};
template <>
struct Params<5> : Params<87> {
  static constexpr int CTILDE = 32, TR = 32;
  static constexpr bool NIST = false;
};
// local aliases of the parameter set inside a templated kernel / function
#define MLDSA_USE(P)                                                                                         \
  constexpr int K = P::K, L = P::L, ETA = P::ETA, TAU = P::TAU, BETA = P::TAU * P::ETA, OMEGA = P::OMEGA,  \
                CTILDE = P::CTILDE, ZBITS = P::G1BITS + 1, W1BITS = 23 - P::G1BITS, POLY_ETA = (P::ETA == 2 ? 96 : 128), \
                POLY_Z = 32 * (P::G1BITS + 1), POLY_W1 = 32 * (23 - P::G1BITS), NKEYPOLY = P::L + 2 * P::K,   \
                TR = P::TR, OFF_S1 = 64 + P::TR, OFF_S2 = OFF_S1 + POLY_ETA * P::L, OFF_T0 = OFF_S2 + POLY_ETA * P::K,                          \
                SK_BYTES = OFF_T0 + 416 * P::K, PK_BYTES = 32 + 320 * P::K,                                    \
                SIG_BYTES = P::CTILDE + P::L * POLY_Z + P::OMEGA + P::K;                                       \
  constexpr uint32_t GAMMA1 = 1u << P::G1BITS, GAMMA2 = P::GAMMA2, ALPHA = 2 * P::GAMMA2;                     \
  (void)K; (void)L; (void)ETA; (void)TAU; (void)BETA; (void)OMEGA; (void)CTILDE; (void)ZBITS; (void)W1BITS;    \
  (void)POLY_ETA; (void)POLY_Z; (void)POLY_W1; (void)NKEYPOLY; (void)OFF_S2; (void)OFF_T0; (void)SK_BYTES;     \
  (void)PK_BYTES; (void)SIG_BYTES; (void)GAMMA1; (void)GAMMA2; (void)ALPHA; (void)TR
constexpr int OFF_KEY = 32, OFF_TR = 64, POLY_T1 = 320;
constexpr int MAX_ATTEMPTS = 576;

// j-th 64-bit word of PackW1(w1) (internal/pack.go:256-271) for one op, built from the byte-per-coefficient
// buffer: 4-bit PackLe16 when gamma1 = 2^19, 6-bit fields when gamma1 = 2^17.
template <class P>
__device__ __forceinline__ uint64_t w1_word(const uint8_t* __restrict__ w1u_op, int j) {
  constexpr int W1BITS = 23 - P::G1BITS, WPP = 4 * W1BITS;  // words per polynomial
  const uint8_t* poly = w1u_op + (j / WPP) * 256;
  const int q = j % WPP;
  if constexpr (W1BITS == 4) {
    const uint4 b = *reinterpret_cast<const uint4*>(poly + 16 * q);
    const uint32_t w[4] = {b.x, b.y, b.z, b.w};
    uint64_t r = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) r |= (uint64_t)((w[i >> 2] >> (8 * (i & 3))) & 15) << (4 * i);
    return r;
  } else {
    const int c0 = (64 * q) / 6, rem = 64 * q - 6 * c0;
    unsigned __int128 acc = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) {
      const int c = c0 + i < 256 ? c0 + i : 255;
      acc |= (unsigned __int128)(poly[c] & 63) << (6 * i);
    }
    return (uint64_t)(acc >> rem);
  }
}

// 32 fields of BITS bits (little-endian bit stream) from nw 32-bit words with static indexing
template <int BITS, int NW>
__device__ __forceinline__ uint32_t field32(const uint32_t (&w)[NW], int i) {
  const int bit = BITS * i, wi = bit >> 5, sh = bit & 31;
  uint32_t f = w[wi] >> sh;
  if (sh + BITS > 32) f |= w[wi + 1] << (32 - sh);
  return f & ((1u << BITS) - 1);
}

// Sign keeps w1 in the final PackW1 byte order when w1 has 4 bits (gamma2 = (q-1)/32: two coefficients per byte, 128
// bytes per polynomial) so the challenge hash absorbs it as is; the 6-bit case keeps one byte per coefficient and is
// packed by w1_word.  Verify always uses the byte-per-coefficient form.
template <class P>
struct SignW1 {
  static constexpr bool packed = (23 - P::G1BITS) == 4;
  static constexpr int stride = packed ? 128 : 256;  // bytes per polynomial
  // coefficients 16s + 2v and 16s + 2v + 1
  static __device__ __forceinline__ void store(uint8_t* poly, int s, int v, uint32_t hi0, uint32_t hi1) {
    if constexpr (packed) poly[8 * s + v] = (uint8_t)(hi0 | (hi1 << 4));
    else *reinterpret_cast<uint16_t*>(poly + 16 * s + 2 * v) = (uint16_t)(hi0 | (hi1 << 8));
  }
  static __device__ __forceinline__ void load(const uint8_t* poly, int s, int v, uint32_t& hi0, uint32_t& hi1) {
    if constexpr (packed) {
      const uint32_t b = poly[8 * s + v];
      hi0 = b & 15;
      hi1 = b >> 4;
    } else {
      const uint32_t b = *reinterpret_cast<const uint16_t*>(poly + 16 * s + 2 * v);
      hi0 = b & 0xff;
      hi1 = b >> 8;
    }
  }
};

struct Work {
  uint32_t *A, *sh;        // per key: A [30][256]; sh = s1h[5] | s2h[6] | t0h[6]
  uint64_t *mu, *rhop;     // per op: 8 words each
  uint32_t *y, *yh, *w0;   // per op: [5][256], [5][256], [6][256]
  uint8_t* w1u;            // per op: K x SignW1::stride bytes: PackW1 layout (4-bit w1) or one byte per coefficient (6-bit)
  uint32_t* cmask;         // per op: 8 words "c[i] != 0" | 8 words "c[i] == -1" from SampleInBall
  uint8_t* zbuf;           // per op: 5 x 640 bytes, z packed (word aligned; copied into the signature on accept)
  uint32_t* c;             // per op: [256] challenge polynomial, then its NTT
  uint64_t* ctilde;        // per op: 6 words
  uint32_t *hintbits, *flags, *hintcnt, *attempt;  // per op: [48], 1, 1, 1
  uint32_t *pass, *list1, *list2;  // per op: 2 interleaved pass counters (stage 0, stage 1); survivors of response stages 0 and 1
  // Speculative attempts: once enough ops are finished, every active op tries T consecutive attempts in one round;
  // attempt t >= 1 of op X runs in the per-op state slot of a finished op (its id comes from `done`), so a slot id
  // indexes all per-round state while owner[slot] = X indexes the key, mu, rho' and the attempt counter.
  uint32_t *owner, *tofs;  // per slot: the op it works for, and its attempt offset t
  uint32_t *best;          // per op: min over accepted slots of (t << 24 | slot), 0xffffffff = none yet
  uint32_t *done, *slots;  // ids of finished ops (free slots); the slot list of the current round
  uint32_t* act[2];        // active lists (op ids)
  uint32_t* count;         // [8] device counters: act[0], act[1], list1, list2, done, -, total attempts (64 bit)
};

// ------------------------------------------------------------------ key expansion
constexpr int kExpThreads = 64;
constexpr int kExpRow = 257;  // 256 words + 1 slack, odd stride

// One SHAKE128 stream of PolyDeriveUniform (sample.go:92-123): `a` holds the absorbed, padded block seed || nonce; the
// 256 accepted coefficients land in this thread's shared-memory row (kExpRow words).
// 56 candidates of 3 bytes per block (23 bits each); every candidate is stored at the write pointer (one slack
// word per row) and only the pointer advance is predicated.  The first four blocks cannot fill the row (224 < 256).
__device__ __forceinline__ void uniform_stream(uint64_t (&a)[25], uint32_t* row) {
  auto parse = [&](uint32_t* wp, auto checked) {
#pragma unroll
    for (int f = 0; f < 56; f++) {
      const int bit = 24 * f, wi = bit >> 5, sh = bit & 31;
      const uint32_t lo = (uint32_t)(a[wi >> 1] >> (32 * (wi & 1)));
      uint32_t d;
      if (sh + 24 <= 32) {
        d = (lo >> sh) & 0x7fffff;
      } else {
        const uint32_t hi = (uint32_t)(a[(wi + 1) >> 1] >> (32 * ((wi + 1) & 1)));
        d = __funnelshift_r(lo, hi, sh) & 0x7fffff;
      }
      *wp = d;
      bool acc = d < Q;
      if (decltype(checked)::value) acc = acc && wp < row + N;
      wp += acc ? 1 : 0;
    }
    return wp;
  };
  uint32_t* wp = row;
#pragma unroll 1
  for (int b = 0; b < 4; b++) {
    keccak::f1600(a);
    wp = parse(wp, std::false_type{});
  }
  do {
    keccak::f1600(a);
    wp = parse(wp, std::true_type{});
  } while (wp < row + N);
}

// ExpandA (mat.go:15-23, sample.go:92-123): A[i][j] = RejNTTPoly(SHAKE128(rho || le16((i<<8)+j)))
template <class P>
__global__ void __launch_bounds__(kExpThreads) expand_a_kernel(const uint8_t* __restrict__ sk, size_t sk_stride,
                                                               size_t nkeys, uint32_t* __restrict__ A) {
  MLDSA_USE(P);
  extern __shared__ __align__(16) uint32_t rows[];
  const size_t s0 = (size_t)blockIdx.x * blockDim.x, total = nkeys * K * L;
  const size_t s = s0 + threadIdx.x;
  const size_t sc = s < total ? s : total - 1;
  const size_t key = sc % nkeys;
  const int ij = (int)(sc / nkeys), i = ij / L, j = ij % L;
  const uint8_t* rho = sk + key * sk_stride;
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll
  for (int w = 0; w < 4; w++) a[w] = keccak::ld64(rho + 8 * w);
  a[4] = (uint64_t)j | ((uint64_t)i << 8) | (0x1full << 16);  // nonce = (i<<8)+j, little endian
  a[20] = 0x8000000000000000ull;                               // SHAKE128 rate 168
  uniform_stream(a, rows + threadIdx.x * kExpRow);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int p = warp; p < kExpThreads; p += kExpThreads / 32) {
    const size_t sp = s0 + p;
    if (sp >= total) break;
    uint32_t* dst = A + ((sp % nkeys) * (K * L) + sp / nkeys) * N;
#pragma unroll
    for (int w = 0; w < 8; w++) dst[32 * w + lane] = rows[p * kExpRow + 32 * w + lane];
  }
}

// s1h, s2h, t0h = NTT(unpack(...)) (dilithium.go:150-162): one octet per (key, polynomial)
template <class P>
__global__ void __launch_bounds__(128) expand_s_kernel(const uint8_t* __restrict__ sk, size_t sk_stride, size_t nkeys,
                                                       uint32_t* __restrict__ sh, const uint32_t* __restrict__ zetas) {
  MLDSA_USE(P);
  __shared__ __align__(16) uint32_t tiles[16 * kPolyWords];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, oct = lane >> 3, v = lane & 7;
  uint32_t* tile = tiles + (warp * 4 + oct) * kPolyWords;
  const size_t total = nkeys * NKEYPOLY;
  const size_t base = ((size_t)blockIdx.x * 4 + warp) * 4;
  if (base >= total) return;
  const size_t u_raw = base + oct;
  const bool active = u_raw < total;
  const size_t u = active ? u_raw : total - 1;
  const size_t key = u / NKEYPOLY;
  const int p = (int)(u % NKEYPOLY);
  const uint8_t* skp = sk + key * sk_stride;
  uint32_t r[32];
  if (p < L + K) {  // PolyUnpackLeqEta (internal/pack.go:49-75): nibbles (eta = 4) or 3-bit fields (eta = 2)
    constexpr int EB = (ETA == 2) ? 3 : 4;
    const uint32_t* src = reinterpret_cast<const uint32_t*>(skp + OFF_S1 + POLY_ETA * p + 4 * EB * v);
    uint32_t w[EB + 1];
#pragma unroll
    for (int i = 0; i < EB; i++) w[i] = __ldg(src + i);
    w[EB] = 0;
#pragma unroll
    for (int i = 0; i < 32; i++) r[i] = Q + ETA - field32<EB>(w, i);
  } else {  // UnpackT0 (pack.go:56-86): 13-bit fields, Q + 2^12 - x
    const uint32_t* src = reinterpret_cast<const uint32_t*>(skp + OFF_T0 + 416 * (p - L - K) + 52 * v);
    uint32_t w[14];
#pragma unroll
    for (int i = 0; i < 13; i++) w[i] = __ldg(src + i);
    w[13] = 0;
#pragma unroll
    for (int i = 0; i < 32; i++) {
      const int bit = 13 * i, wi = bit >> 5, sh = bit & 31;
      uint32_t f = w[wi] >> sh;
      if (sh > 19) f |= w[wi + 1] << (32 - sh);
      r[i] = Q + (1u << 12) - (f & 0x1fff);
    }
  }
  c_to_s(r, tile, v);
  LaneTw t;
  load_lane_tw_fwd(t, zetas, v);
  ntt_octet(r, tile, v, t);
  gstore_C_via_tile(sh + (key * NKEYPOLY + p) * N, tile, v, r, active);
}

// ------------------------------------------------------------------ mu, rho'
struct ByteSponge {  // SHAKE256 absorber for unaligned byte streams (thread-local block buffer)
  uint64_t a[25];
  uint64_t blk[17];
  int pos;
  __device__ __forceinline__ void init() {
    keccak::zero(a);
#pragma unroll
    for (int i = 0; i < 17; i++) blk[i] = 0;
    pos = 0;
  }
  __device__ __forceinline__ void flush() {
#pragma unroll
    for (int i = 0; i < 17; i++) {
      a[i] ^= blk[i];
      blk[i] = 0;
    }
    keccak::f1600(a);
    pos = 0;
  }
  __device__ __forceinline__ void put(uint8_t b) {
    blk[pos >> 3] |= (uint64_t)b << (8 * (pos & 7));
    if (++pos == 136) flush();
  }
  __device__ __forceinline__ void finish() {  // SHAKE pad: 0x1f ... 0x80
    blk[pos >> 3] ^= 0x1full << (8 * (pos & 7));
    blk[16] ^= 0x8000000000000000ull;
    flush();
  }
};

template <class P>
__global__ void __launch_bounds__(128) mu_kernel(const uint8_t* __restrict__ sk, size_t sk_stride,
                                                 const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ msg_off,
                                                 const uint8_t* __restrict__ ctx, int ctxlen, int internal,
                                                 const uint8_t* __restrict__ rnd, size_t n, uint64_t* __restrict__ mu,
                                                 uint64_t* __restrict__ rhop, uint32_t* __restrict__ attempt,
                                                 uint32_t* __restrict__ act, uint32_t* __restrict__ owner,
                                                 uint32_t* __restrict__ tofs) {
  MLDSA_USE(P);
  const size_t op = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (op >= n) return;
  const uint8_t* skp = sk + op * sk_stride;
  ByteSponge sp;
  sp.init();
  for (int i = 0; i < TR; i++) sp.put(skp[OFF_TR + i]);  // mu = H(tr || M')  (dilithium.go:354-357)
  if (!internal && P::NIST) {                              // mldsa65/dilithium.go:71-79
    sp.put(0);
    sp.put((uint8_t)ctxlen);
    for (int i = 0; i < ctxlen; i++) sp.put(ctx[i]);
  }
  const uint64_t lo = msg_off[op], hi = msg_off[op + 1];
  for (uint64_t i = lo; i < hi; i++) sp.put(msgs[i]);
  sp.finish();
  uint64_t m[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    m[i] = sp.a[i];
    mu[8 * op + i] = m[i];
  }
  // rho' = H(key || rnd || mu)  (dilithium.go:360-366): 128 bytes, one block
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll
  for (int i = 0; i < 4; i++) a[i] = keccak::ld64(skp + OFF_KEY + 8 * i);
  if constexpr (P::NIST) {
#pragma unroll
    for (int i = 0; i < 4; i++) a[4 + i] = rnd ? keccak::ld64(rnd + 32 * op + 8 * i) : 0;
#pragma unroll
    for (int i = 0; i < 8; i++) a[8 + i] = m[i];
    a[16] = 0x800000000000001full;
  } else {  // round 3: rho' = H(key || mu), 96 bytes
#pragma unroll
    for (int i = 0; i < 8; i++) a[4 + i] = m[i];
    a[12] = 0x1f;
    a[16] = 0x8000000000000000ull;
  }
  keccak::f1600(a);
#pragma unroll
  for (int i = 0; i < 8; i++) rhop[8 * op + i] = a[i];
  attempt[op] = 0;
  act[op] = (uint32_t)op;
  owner[op] = (uint32_t)op;
  tofs[op] = 0;
}

// PolyDeriveUniformLeGamma1 (sample.go:197-209, internal/pack.go:146-203): `a` holds the absorbed, padded block
// seed || nonce; five SHAKE256 blocks are unpacked to 256 coefficients gamma1 - field (mod q) at `dst`.
template <class P>
__device__ __forceinline__ void legamma1_poly(uint64_t (&a)[25], uint32_t* __restrict__ dst) {
  MLDSA_USE(P);
  uint64_t buf[86];
#pragma unroll
  for (int b = 0; b < 5; b++) {
    keccak::f1600(a);
#pragma unroll
    for (int w = 0; w < 17; w++) buf[17 * b + w] = a[w];
  }
  buf[85] = 0;
  uint4* out = reinterpret_cast<uint4*>(dst);
#pragma unroll 2
  for (int p = 0; p < 64; p++) {  // 4 coefficients of ZBITS bits each (internal/pack.go:146-203)
    uint32_t cf[4];
#pragma unroll
    for (int h = 0; h < 4; h++) {
      const int bit = ZBITS * (4 * p + h), wi = bit >> 6, sh = bit & 63;
      uint64_t f = buf[wi] >> sh;
      if (sh + ZBITS > 64) f |= buf[wi + 1] << (64 - sh);
      uint32_t c = GAMMA1 - ((uint32_t)f & ((1u << ZBITS) - 1));
      c += (uint32_t)((int32_t)c >> 31) & Q;
      cf[h] = c;
    }
    out[p] = make_uint4(cf[0], cf[1], cf[2], cf[3]);
  }
}

// ------------------------------------------------------------------ per-round kernels
// y[i] = ExpandMask(rho', L*attempt + i)  (sample.go:187-209, pack.go:177-195)
template <class P>
__global__ void __launch_bounds__(128) mask_kernel(const uint32_t* __restrict__ act, size_t nact,
                                                   const uint64_t* __restrict__ rhop,
                                                   const uint32_t* __restrict__ attempt,
                                                   const uint32_t* __restrict__ owner, const uint32_t* __restrict__ tofs,
                                                   uint32_t* __restrict__ y) {
  MLDSA_USE(P);
  const size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nact * L) return;
  const size_t op = act[s % nact];  // state slot
  const size_t own = owner[op];
  const int i = (int)(s / nact);
  const uint32_t nonce = L * (attempt[own] + tofs[op]) + i;
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll
  for (int w = 0; w < 8; w++) a[w] = rhop[8 * own + w];
  a[8] = (uint64_t)(nonce & 0xffff) | (0x1full << 16);
  a[16] = 0x8000000000000000ull;
  legamma1_poly<P>(a, y + (op * L + i) * N);
}

struct OctetCtx {
  int lane, warp, oct, v;
  uint32_t* tile;
};
__device__ __forceinline__ OctetCtx octet_ctx(uint32_t* tiles) {
  OctetCtx o;
  o.lane = threadIdx.x & 31;
  o.warp = threadIdx.x >> 5;
  o.oct = o.lane >> 3;
  o.v = o.lane & 7;
  o.tile = tiles + (o.warp * 4 + o.oct) * kPolyWords;
  return o;
}

// yh = NTT(y): octet per (active op, j)
template <class P>
__global__ void __launch_bounds__(128) yntt_kernel(const uint32_t* __restrict__ act, size_t nact,
                                                   const uint32_t* __restrict__ y, uint32_t* __restrict__ yh,
                                                   const uint32_t* __restrict__ zetas) {
  MLDSA_USE(P);
  __shared__ __align__(16) uint32_t tiles[16 * kPolyWords];
  const OctetCtx o = octet_ctx(tiles);
  const size_t total = nact * L, base = ((size_t)blockIdx.x * 4 + o.warp) * 4;
  if (base >= total) return;
  const bool active = base + o.oct < total;
  const size_t u = active ? base + o.oct : total - 1;
  const size_t op = act[u / L];
  const int j = (int)(u % L);
  uint32_t r[32];
  gload_S(y + (op * L + j) * N, o.v, r);
  LaneTw t;
  load_lane_tw_fwd(t, zetas, o.v);
  ntt_octet(r, o.tile, o.v, t);
  gstore_C_via_tile(yh + (op * L + j) * N, o.tile, o.v, r, active);
}

// decompose (rounding.go:13-43): alpha = 523776 (gamma2 = (q-1)/32) or 190464 (gamma2 = (q-1)/88)
template <class P>
__device__ __forceinline__ void decompose(uint32_t a, uint32_t& a0plusq, uint32_t& a1) {
  constexpr uint32_t ALPHA = 2 * P::GAMMA2;
  a1 = (a + 127) >> 7;
  if constexpr (ALPHA == 523776) {
    a1 = (a1 * 1025 + (1u << 21)) >> 22;
    a1 &= 15;
  } else {
    a1 = (a1 * 11275 + (1u << 23)) >> 24;
    a1 ^= (uint32_t)((int32_t)(43 - a1) >> 31) & a1;
  }
  a0plusq = a - a1 * ALPHA;
  a0plusq += (uint32_t)((int32_t)(a0plusq - (Q - 1) / 2) >> 31) & Q;
}

// w[i] = InvNTT(ReduceLe2Q(A[i] . yh)), NormalizeAssumingLe2Q, Decompose (dilithium.go:386-394).
// A unit of work is one row (op, i); the units are dealt to the octets of a persistent grid, adjacent octets taking
// adjacent rows so that the K rows of an op read its y-hat while it is hot in L2.  The row of A -- L polynomials of
// 1 KB, 30 KB per op and by far the largest stream of the signing loop -- does not pass through registers: lane 0 of
// each octet keeps kWSlots 1 KB bulk copies (TMA engine, one mbarrier per slot) in flight into the octet's ring in
// shared memory, always kWSlots polynomials ahead of the arithmetic, also across the end of a row, so the DRAM
// latency of the next row hides behind the inverse NTT and Decompose of the current one.
// The kernel is bound by latency, not by a pipe or by HBM, and resident warps are what it responds to: twiddles read from
// shared memory and a ring of two slots instead of three fit four CTAs per SM instead of three.  Summing the L products
// of a coefficient as 64-bit integers with one Montgomery reduction at the end saves a tenth of the instructions but
// costs 32 registers, and y-hat one polynomial ahead in registers costs another 32: both lose resident warps.
constexpr int kWSlots = 2;
constexpr int kWCtas = 4;  // CTAs per SM the grid and the register allocation are sized for
struct WSm {
  static constexpr int ring = 16 * kWSlots * 1024, tiles = 16 * kPolyWords * 4, bars = 16 * kWSlots * 8;
  static constexpr int bytes = ring + tiles + bars + 2048;  // + the inverse twiddle pairs
};
template <class P>
__global__ void __launch_bounds__(128, kWCtas) w_kernel(const uint32_t* __restrict__ act, size_t nact, int key_shared,
                                                        const uint32_t* __restrict__ A, const uint32_t* __restrict__ yh,
                                                        uint32_t* __restrict__ w0, uint8_t* __restrict__ w1u,
                                                        const uint32_t* __restrict__ owner, const uint32_t* __restrict__ zetas) {
  MLDSA_USE(P);
  using S = WSm;
  constexpr int SLOTS = kWSlots;
  extern __shared__ __align__(128) uint8_t wsm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, oct = lane >> 3, v = lane & 7, ob = warp * 4 + oct;
  uint32_t* ring = reinterpret_cast<uint32_t*>(wsm) + ob * (SLOTS * 256);
  uint32_t* tile = reinterpret_cast<uint32_t*>(wsm + S::ring) + ob * kPolyWords;
  uint64_t* bars = reinterpret_cast<uint64_t*>(wsm + S::ring + S::tiles) + ob * SLOTS;
  if (v == 0) {
#pragma unroll
    for (int q = 0; q < SLOTS; q++) mbar_init(bars + q, 1);
    fence_barrier_init();
  }
  // the per-lane twiddles of the inverse transform are read from shared memory where they are used: thirty registers
  // less across the product loop
  volatile uint2* izs = reinterpret_cast<volatile uint2*>(wsm + S::ring + S::tiles + S::bars);
  stage_inv_pairs(izs, zetas);
  __syncthreads();
  const size_t total = nact * K, G = (size_t)gridDim.x * 16, first = ((size_t)blockIdx.x * 4 + warp) * 4;
  if (first >= total) return;
  const size_t n_it = (total - first + G - 1) / G;  // the same for the four octets of a warp
  const size_t n_chunks = n_it * L;
  auto unit = [&](size_t it) {
    const size_t u = first + it * G + oct;
    return u < total ? u : total - 1;  // octets past the end repeat the last unit and store nothing
  };
  auto issue = [&](size_t c) {  // lane 0 of the octet: fetch polynomial c % L of row unit(c / L) into slot c % SLOTS
    const size_t u = unit(c / L);
    const size_t own = key_shared ? 0 : owner[act[u / K]];
    const uint32_t* src = A + (own * (size_t)(K * L) + (u % K) * L + c % L) * N;
    uint64_t* bar = bars + c % SLOTS;
    mbar_expect_tx(bar, 1024);
    bulk_g2s(ring + (c % SLOTS) * 256, src, 1024, bar);
  };
  if (v == 0)
    for (size_t c = 0; c < (size_t)SLOTS && c < n_chunks; c++) issue(c);
  size_t c = 0;
  for (size_t it = 0; it < n_it; it++) {
    const size_t u = unit(it);
    const bool active = first + it * G + oct < total;
    const size_t op = act[u / K];
    const int i = (int)(u % K);
    uint32_t acc[32];
#pragma unroll
    for (int q = 0; q < 32; q++) acc[q] = 0;
#pragma unroll 1
    for (int j = 0; j < L; j++, c++) {
      uint4 z[8];
      gload_I(yh + (op * L + j) * N, v, z);  // issued before the wait: overlaps the tail of the bulk copy
      const int slot = (int)(c % SLOTS);
      mbar_wait(bars + slot, (uint32_t)((c / SLOTS) & 1));
      const uint4* xs = reinterpret_cast<const uint4*>(ring + slot * 256) + v;
#pragma unroll
      for (int q = 0; q < 8; q++) {
        const uint4 x = xs[8 * q];
        acc[4 * q] += mont_mul(x.x, z[q].x);
        acc[4 * q + 1] += mont_mul(x.y, z[q].y);
        acc[4 * q + 2] += mont_mul(x.z, z[q].z);
        acc[4 * q + 3] += mont_mul(x.w, z[q].w);
      }
      __syncwarp();  // every lane of the octet is done with the slot
      if (v == 0 && c + SLOTS < n_chunks) {
        fence_proxy_async();  // the reads above (generic proxy) before the asynchronous refill of the slot
        issue(c + SLOTS);
      }
    }
#pragma unroll
    for (int q = 0; q < 32; q++) acc[q] = reduce_le2q(acc[q]);
    i_to_c(acc, tile, v);
    invntt_octet_smem(acc, tile, v, izs);  // -> S layout: acc[2s+b] = coefficient 16s + 2v + b
    uint32_t* w0p = w0 + (op * K + i) * N;
    uint8_t* w1b = w1u + (op * K + i) * SignW1<P>::stride;
#pragma unroll
    for (int s = 0; s < 16; s++) {
      uint32_t lo0, hi0, lo1, hi1;
      decompose<P>(le2q_modq(acc[2 * s]), lo0, hi0);
      decompose<P>(le2q_modq(acc[2 * s + 1]), lo1, hi1);
      if (active) {
        *reinterpret_cast<uint2*>(w0p + 16 * s + 2 * v) = make_uint2(lo0, lo1);
        SignW1<P>::store(w1b, s, v, hi0, hi1);
      }
    }
  }
}

// SampleInBall (sample.go:299-339) on c~ = ct: nz = positions with c != 0, ng = positions with c == -1; `a` is scratch.
template <class P>
__device__ __forceinline__ void sample_in_ball(const uint64_t (&ct)[P::CTILDE / 8], uint64_t (&a)[25], uint64_t (&nz)[4],
                                               uint64_t (&ng)[4]) {
  MLDSA_USE(P);
  constexpr int CTW = CTILDE / 8;
  // SampleInBall: nz = positions with c != 0, ng = positions with c == -1.  Every i of the loop lies in the top
  // 64-bit word (i >= 256 - TAU >= 192) and is untouched before its iteration.
  keccak::zero(a);
#pragma unroll
  for (int i = 0; i < CTW; i++) a[i] = ct[i];
  a[CTW] = 0x1f;
  a[16] = 0x8000000000000000ull;
  keccak::f1600(a);
  uint64_t buf[17];
#pragma unroll
  for (int i = 0; i < 17; i++) buf[i] = a[i];
  uint64_t signs = buf[0];
  int off = 8;
#pragma unroll
  for (int q = 0; q < 4; q++) nz[q] = ng[q] = 0;
  static_assert(256 - TAU >= 192, "SampleInBall indices must stay in the top word");
  for (int i = N - TAU; i < N; i++) {
    uint32_t b;
    for (;;) {
      if (off >= 136) {
        keccak::f1600(a);
#pragma unroll
        for (int q = 0; q < 17; q++) buf[q] = a[q];
        off = 0;
      }
      uint64_t wsel = buf[0];
#pragma unroll
      for (int q = 1; q < 17; q++) wsel = ((off >> 3) == q) ? buf[q] : wsel;
      b = (uint32_t)(wsel >> (8 * (off & 7))) & 0xff;
      off++;
      if (b <= (uint32_t)i) break;
    }
    const int bq = b >> 6, br = b & 63;
    uint64_t wn = nz[0], wg = ng[0];
#pragma unroll
    for (int q = 1; q < 4; q++) {
      wn = (bq == q) ? nz[q] : wn;
      wg = (bq == q) ? ng[q] : wg;
    }
    // c[i] = c[b]
    nz[3] |= ((wn >> br) & 1) << (i - 192);
    ng[3] |= ((wg >> br) & 1) << (i - 192);
    // c[b] = 1 - 2 * sign
    const uint64_t bit = 1ull << br, sg = (signs & 1) << br;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      nz[q] |= (bq == q) ? bit : 0;
      ng[q] = (bq == q) ? ((ng[q] & ~bit) | sg) : ng[q];
    }
    signs >>= 1;
  }
}

// c~ = H(mu || w1) (dilithium.go:397-401), c = SampleInBall(c~) (sample.go:299-339): thread per op.
// With packed w1 the hash input is staged through shared memory: two rate blocks at a time, each warp copies that
// slice of the (mu || w1) rows of its 32 ops with coalesced loads into rows of odd stride, from which the per-thread
// absorb reads are bank-conflict free.  c never exists as 256 words in memory: SampleInBall keeps it as two 256-bit
// masks in registers and cntt_mask_kernel expands them.
constexpr int kChThreads = 64;
template <class P>
struct ChLayout {
  static constexpr int WORDS = 8 + P::K * 4 * (23 - P::G1BITS);  // 64-bit words of mu || PackW1(w1)
  static constexpr int FULL = WORDS / 17, REM = WORDS % 17;
  static constexpr int BPP = 2, NPH = (FULL + BPP - 1) / BPP;     // rate blocks per phase, phases
  static constexpr int PHW = BPP * 17 + REM;                       // 64-bit words a phase may hold
  static constexpr int ROWP = (2 * PHW) | 1;                       // 32-bit words per row
  static constexpr int smem = (23 - P::G1BITS) == 4 ? kChThreads * ROWP * 4 : 0;
};
template <class P>
__global__ void __launch_bounds__(kChThreads) challenge_kernel(const uint32_t* __restrict__ act, size_t nact,
                                                               const uint64_t* __restrict__ mu,
                                                               const uint8_t* __restrict__ w1u, uint64_t* __restrict__ ctilde,
                                                               uint32_t* __restrict__ cmask, uint32_t* __restrict__ flags,
                                                               uint32_t* __restrict__ hintcnt, uint32_t* __restrict__ pass,
                                                               const uint32_t* __restrict__ owner) {
  MLDSA_USE(P);
  using CL = ChLayout<P>;
  extern __shared__ __align__(16) uint32_t rows[];
  constexpr int ROWP = CL::ROWP, WORDS = CL::WORDS, FULL = CL::FULL, REM = CL::REM, CTW = CTILDE / 8;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t s0 = (size_t)blockIdx.x * kChThreads + warp * 32;
  if (s0 >= nact) return;
  const size_t s = s0 + lane;
  const bool valid = s < nact;
  const size_t op = act[valid ? s : nact - 1];
  const size_t own = owner[op];
  uint64_t a[25];
  keccak::zero(a);
  if constexpr (SignW1<P>::packed) {
    uint32_t* wrows = rows + warp * 32 * ROWP;
    const uint32_t* myrow = wrows + lane * ROWP;
#pragma unroll 1
    for (int ph = 0; ph < CL::NPH; ph++) {
      const int first = ph * CL::BPP * 17;                                       // first 64-bit word of this phase
      const int nw = (ph == CL::NPH - 1) ? WORDS - first : CL::BPP * 17;         // 64-bit words staged
      __syncwarp();
      const int nrows = nact - s0 < 32 ? (int)(nact - s0) : 32;
#pragma unroll 8
      for (int t = 0; t < nrows; t++) {
        const size_t ot = __shfl_sync(0xffffffffu, (uint32_t)op, t), wt = __shfl_sync(0xffffffffu, (uint32_t)own, t);
        const uint32_t* m32 = reinterpret_cast<const uint32_t*>(mu + 8 * wt);
        const uint32_t* w32 = reinterpret_cast<const uint32_t*>(w1u + ot * (K * 128));
        for (int x = lane; x < 2 * nw; x += 32) {
          const int g = 2 * first + x;  // 32-bit word of the stream
          wrows[t * ROWP + x] = g < 16 ? m32[g] : ldg_stream32(w32 + (g - 16));
        }
      }
      __syncwarp();
      const int b_end = (ph + 1) * CL::BPP < FULL ? (ph + 1) * CL::BPP : FULL;
#pragma unroll 1
      for (int b = ph * CL::BPP; b < b_end; b++) {
        const uint32_t* src = myrow + 2 * (17 * b - first);
#pragma unroll
        for (int w = 0; w < 17; w++) a[w] ^= (uint64_t)src[2 * w] | ((uint64_t)src[2 * w + 1] << 32);
        keccak::f1600(a);
      }
      if (ph == CL::NPH - 1) {
        const uint32_t* src = myrow + 2 * (17 * FULL - first);
#pragma unroll
        for (int w = 0; w < REM; w++) a[w] ^= (uint64_t)src[2 * w] | ((uint64_t)src[2 * w + 1] << 32);
      }
    }
  } else {
    const uint8_t* w1o = w1u + op * (K * SignW1<P>::stride);
#pragma unroll 1
    for (int b = 0; b < FULL; b++) {
#pragma unroll
      for (int w = 0; w < 17; w++) {
        const int k = 17 * b + w;
        a[w] ^= (k < 8) ? mu[8 * own + k] : w1_word<P>(w1o, k - 8);
      }
      keccak::f1600(a);
    }
#pragma unroll
    for (int w = 0; w < REM; w++) a[w] ^= w1_word<P>(w1o, 17 * FULL + w - 8);
  }
  if (!valid) return;
  a[REM] ^= 0x1f;
  a[16] ^= 0x8000000000000000ull;
  keccak::f1600(a);
  uint64_t ct[CTW];
#pragma unroll
  for (int i = 0; i < CTW; i++) {
    ct[i] = a[i];
    ctilde[CTW * op + i] = ct[i];
  }
  uint64_t nz[4], ng[4];
  sample_in_ball<P>(ct, a, nz, ng);
  uint4* cm = reinterpret_cast<uint4*>(cmask + 16 * op);
  cm[0] = make_uint4((uint32_t)nz[0], (uint32_t)(nz[0] >> 32), (uint32_t)nz[1], (uint32_t)(nz[1] >> 32));
  cm[1] = make_uint4((uint32_t)nz[2], (uint32_t)(nz[2] >> 32), (uint32_t)nz[3], (uint32_t)(nz[3] >> 32));
  cm[2] = make_uint4((uint32_t)ng[0], (uint32_t)(ng[0] >> 32), (uint32_t)ng[1], (uint32_t)(ng[1] >> 32));
  cm[3] = make_uint4((uint32_t)ng[2], (uint32_t)(ng[2] >> 32), (uint32_t)ng[3], (uint32_t)(ng[3] >> 32));
  flags[op] = 1;  // cleared when the op passes response stage 1
  hintcnt[op] = 0;
  pass[2 * op] = 0;
  pass[2 * op + 1] = 0;
}

// c-hat = NTT(c) for Sign: octet per active op; c is expanded from the SampleInBall masks
__global__ void __launch_bounds__(128) cntt_mask_kernel(const uint32_t* __restrict__ act, size_t nact,
                                                        const uint32_t* __restrict__ cmask, uint32_t* __restrict__ cpoly,
                                                        const uint32_t* __restrict__ zetas) {
  __shared__ __align__(16) uint32_t tiles[16 * kPolyWords];
  const OctetCtx o = octet_ctx(tiles);
  const size_t base = ((size_t)blockIdx.x * 4 + o.warp) * 4;
  if (base >= nact) return;
  const bool active = base + o.oct < nact;
  const size_t op = act[active ? base + o.oct : nact - 1];
  const uint4* cm = reinterpret_cast<const uint4*>(cmask + 16 * op);
  const uint4 n0 = cm[0], n1 = cm[1], g0 = cm[2], g1 = cm[3];
  const uint32_t nzw[8] = {n0.x, n0.y, n0.z, n0.w, n1.x, n1.y, n1.z, n1.w};
  const uint32_t ngw[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
  uint32_t r[32];
#pragma unroll
  for (int s = 0; s < 16; s++) {  // S layout: r[2s + b] = coefficient 16s + 2v + b = bit 16 (s & 1) + 2v + b of word s >> 1
#pragma unroll
    for (int b = 0; b < 2; b++) {
      const int sh = 16 * (s & 1) + 2 * o.v + b;
      const uint32_t isnz = (nzw[s >> 1] >> sh) & 1, isng = (ngw[s >> 1] >> sh) & 1;
      r[2 * s + b] = isnz ? (isng ? Q - 1 : 1u) : 0u;
    }
  }
  LaneTw t;
  load_lane_tw_fwd(t, zetas, o.v);
  ntt_octet(r, o.tile, o.v, t);
  __syncwarp();
  gstore_C_via_tile(cpoly + op * N, o.tile, o.v, r, active);
}

// c-hat = NTT(c): octet per active op
__global__ void __launch_bounds__(128) cntt_kernel(const uint32_t* __restrict__ act, size_t nact,
                                                   uint32_t* __restrict__ cpoly, const uint32_t* __restrict__ zetas) {
  __shared__ __align__(16) uint32_t tiles[16 * kPolyWords];
  const OctetCtx o = octet_ctx(tiles);
  const size_t base = ((size_t)blockIdx.x * 4 + o.warp) * 4;
  if (base >= nact) return;
  const bool active = base + o.oct < nact;
  const size_t op = act[active ? base + o.oct : nact - 1];
  uint32_t r[32];
  gload_S(cpoly + op * N, o.v, r);
  LaneTw t;
  load_lane_tw_fwd(t, zetas, o.v);
  ntt_octet(r, o.tile, o.v, t);
  __syncwarp();
  gstore_C_via_tile(cpoly + op * N, o.tile, o.v, r, active);
}

// InvNTT(c-hat . x-hat) on an octet: returns S layout
__device__ __forceinline__ void c_times(uint32_t (&r)[32], const uint32_t* __restrict__ chat,
                                        const uint32_t* __restrict__ xhat, const OctetCtx& o, const volatile uint2* iz) {
  uint4 x[8], z[8];
  gload_I(chat, o.v, x);
  gload_I_ro(xhat, o.v, z);
#pragma unroll
  for (int c = 0; c < 8; c++) {
    r[4 * c] = mont_mul(x[c].x, z[c].x);
    r[4 * c + 1] = mont_mul(x[c].y, z[c].y);
    r[4 * c + 2] = mont_mul(x[c].z, z[c].z);
    r[4 * c + 3] = mont_mul(x[c].w, z[c].w);
  }
  i_to_c(r, o.tile, o.v);
  invntt_octet_smem(r, o.tile, o.v, iz);
}

// makeHint (rounding.go:56-67)
template <class P>
__device__ __forceinline__ uint32_t make_hint(uint32_t z0, uint32_t r1) {
  constexpr uint32_t GAMMA2 = P::GAMMA2;
  return (z0 <= GAMMA2 || z0 > Q - GAMMA2 || (z0 == Q - GAMMA2 && r1 == 0)) ? 0u : 1u;
}

// The three norm checks + hint (dilithium.go:407-464).  Any failed check rejects the attempt and nothing of a rejected
// attempt is ever output, so the checks may run in any order; they run as three launches, cheapest filter first, each
// over the compacted list of ops that survived the previous one (81 % of the attempts of ML-DSA-65 never reach the
// last stage).  A unit of work is one (op, polynomial) pair on one octet; the units of a list are dealt to the octets
// of a persistent grid with no padding between ops.
//   stage 0: r0 = w0 - c s2, kept in place of w0 for stage 2           K units per op of the active list
//   stage 1: z = y + c s1, packed into the signature staging buffer     L units per op of list1
//   stage 2: c t0 and the hints                                         K units per op of list2
// An op moves to the next list when its last unit passes (per-op counter); passing stage 1 clears flags[op], which
// the challenge kernel set, and stage 2 sets it again on a failure, so finalize accepts exactly the ops with flags == 0.
template <class P, int STAGE>
__global__ void __launch_bounds__(128) response_kernel(const uint32_t* __restrict__ list, const uint32_t* __restrict__ count_dev,
                                                       size_t count_host, int key_shared, const uint32_t* __restrict__ sh,
                                                       const uint32_t* __restrict__ cpoly, const uint32_t* __restrict__ y,
                                                       uint32_t* __restrict__ w0, const uint8_t* __restrict__ w1u,
                                                       uint8_t* __restrict__ zbuf, uint32_t* __restrict__ hintbits,
                                                       uint32_t* __restrict__ flags, uint32_t* __restrict__ hintcnt,
                                                       uint32_t* __restrict__ pass, uint32_t* __restrict__ next_list,
                                                       uint32_t* __restrict__ next_count, const uint32_t* __restrict__ owner,
                                                       const uint32_t* __restrict__ zetas) {
  MLDSA_USE(P);
  __shared__ __align__(16) uint32_t tiles[16 * kPolyWords];
  __shared__ __align__(8) uint2 izs[256];
  stage_inv_pairs(izs, zetas);
  __syncthreads();
  const volatile uint2* ti = izs;
  const OctetCtx o = octet_ctx(tiles);
  const unsigned octmask = 0xffu << (8 * o.oct);
  constexpr int ITEMS = STAGE == 1 ? L : K;
  const size_t total = (count_dev ? (size_t)*count_dev : count_host) * ITEMS;
  for (size_t base = ((size_t)blockIdx.x * 4 + o.warp) * 4; base < total; base += (size_t)gridDim.x * 16) {
    const bool active = base + o.oct < total;
    const size_t u = active ? base + o.oct : total - 1;
    const size_t op = list[u / ITEMS];
    const int item = (int)(u % ITEMS);
    const uint32_t* keyp = sh + (key_shared ? 0 : (size_t)owner[op]) * (NKEYPOLY * N);
    const uint32_t* chat = cpoly + op * N;
    uint32_t r[32];
    bool reject = false;
    if constexpr (STAGE == 0) {
      const int i = item;
      uint32_t* w0p = w0 + (op * K + i) * N;
      uint2 aw[16];  // w0[i], requested before the product and the inverse transform instead of after them
#pragma unroll
      for (int s = 0; s < 16; s++) aw[s] = *reinterpret_cast<const uint2*>(w0p + 16 * s + 2 * o.v);
      c_times(r, chat, keyp + (L + i) * N, o, ti);  // c s2[i]
#pragma unroll
      for (int s = 0; s < 16; s++) {
        const uint2 a = aw[s];
        r[2 * s] = modq(a.x + (2 * Q - r[2 * s]));  // w0 - c s2, Normalize
        r[2 * s + 1] = modq(a.y + (2 * Q - r[2 * s + 1]));
        reject |= exceeds1(r[2 * s], GAMMA2 - BETA) | exceeds1(r[2 * s + 1], GAMMA2 - BETA);
        if (active) *reinterpret_cast<uint2*>(w0p + 16 * s + 2 * o.v) = make_uint2(r[2 * s], r[2 * s + 1]);
      }
    } else if constexpr (STAGE == 1) {
      const int j = item;
      const uint32_t* yp = y + (op * L + j) * N;
      uint2 aw[16];  // y[j], requested before the product and the inverse transform
#pragma unroll
      for (int s = 0; s < 16; s++) aw[s] = __ldg(reinterpret_cast<const uint2*>(yp + 16 * s + 2 * o.v));
      c_times(r, chat, keyp + j * N, o, ti);  // c s1[j]
#pragma unroll
      for (int s = 0; s < 16; s++) {
        const uint2 a = aw[s];
        r[2 * s] = modq(r[2 * s] + a.x);
        r[2 * s + 1] = modq(r[2 * s + 1] + a.y);
        reject |= exceeds1(r[2 * s], GAMMA1 - BETA) | exceeds1(r[2 * s + 1], GAMMA1 - BETA);
      }
      // PolyPackLeGamma1 (internal/pack.go:236-252): 32 coefficients -> 20 aligned words in the staging
      // buffer; finalize copies them into the (3309-byte strided) signature only if the attempt is accepted
      s_to_c(r, o.tile, o.v);
      uint32_t* zw = reinterpret_cast<uint32_t*>(zbuf + (op * L + j) * (size_t)POLY_Z) + ZBITS * o.v;
      uint64_t accb = 0;
      int bits = 0, ow = 0;
#pragma unroll
      for (int c = 0; c < 32; c++) {
        uint32_t p = GAMMA1 - r[c];
        p += (uint32_t)((int32_t)p >> 31) & Q;
        accb |= (uint64_t)(p & ((1u << ZBITS) - 1)) << bits;
        bits += ZBITS;
        if (bits >= 32) {
          if (active) zw[ow] = (uint32_t)accb;
          ow++;
          accb >>= 32;
          bits -= 32;
        }
      }
    } else {
      const int i = item;
      // the 8 hint words of row i belong to this octet alone; the exchanges inside c_times order these stores
      // before the atomicOr of the other lanes
      if (active) hintbits[8 * K * op + 8 * i + o.v] = 0;
      c_times(r, chat, keyp + (L + K + i) * N, o, ti);  // c t0[i]
      const uint32_t* r0p = w0 + (op * K + i) * N;        // w0 - c s2 from stage 0
      const uint8_t* w1b = w1u + (op * K + i) * SignW1<P>::stride;
      uint32_t pop = 0;
#pragma unroll
      for (int s = 0; s < 16; s++) {
        const uint32_t t0 = le2q_modq(r[2 * s]), t1 = le2q_modq(r[2 * s + 1]);
        reject |= exceeds1(t0, GAMMA2) | exceeds1(t1, GAMMA2);
        const uint2 r0 = *reinterpret_cast<const uint2*>(r0p + 16 * s + 2 * o.v);
        uint32_t w1a, w1c;
        SignW1<P>::load(w1b, s, o.v, w1a, w1c);
        const uint32_t h0 = make_hint<P>(le2q_modq(r0.x + t0), w1a);
        const uint32_t h1 = make_hint<P>(le2q_modq(r0.y + t1), w1c);
        const uint32_t bits = h0 | (h1 << 1);
        pop += h0 + h1;
        if (bits && active) atomicOr(hintbits + 8 * K * op + 8 * i + (s >> 1), bits << (16 * (s & 1) + 2 * o.v));
      }
      if (pop && active) atomicAdd(hintcnt + op, pop);
    }
    reject = __any_sync(octmask, reject);
    if (active && o.v == 0) {
      if constexpr (STAGE == 2) {
        if (reject) atomicOr(flags + op, 1u);
      } else if (!reject) {
        if (atomicAdd(pass + 2 * op, 1u) == (uint32_t)(ITEMS - 1)) {  // last unit of this op: all of them passed
          if constexpr (STAGE == 1) flags[op] = 0;
          next_list[atomicAdd(next_count, 1u)] = (uint32_t)op;
        }
      }
    }
  }
}

// The slot list of a round: T attempts per active op; attempt 0 runs in the op's own slot, attempt t >= 1 in the
// slot of a finished op.  One thread per (op, t).
__global__ void spec_expand_kernel(const uint32_t* __restrict__ act, size_t nact, int T, const uint32_t* __restrict__ done,
                                   uint32_t* __restrict__ slots, uint32_t* __restrict__ owner, uint32_t* __restrict__ tofs) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nact * T) return;
  const size_t p = i / T;
  const int t = (int)(i % T);
  const uint32_t op = act[p];
  const uint32_t slot = t == 0 ? op : done[p * (T - 1) + (t - 1)];
  slots[i] = slot;
  owner[slot] = op;
  tofs[slot] = (uint32_t)t;
}

// accept / reject (dilithium.go:369-377,459-469), phase 1: every slot whose attempt passed all checks bids for its
// op with (t << 24 | slot); the lowest t wins, i.e. the first passing attempt in the reference's order.
template <class P>
__global__ void finalize_bid_kernel(const uint32_t* __restrict__ slots, size_t nslots, const uint32_t* __restrict__ flags,
                                    const uint32_t* __restrict__ hintcnt, const uint32_t* __restrict__ owner,
                                    const uint32_t* __restrict__ tofs, const uint32_t* __restrict__ attempt,
                                    uint32_t* __restrict__ best) {
  MLDSA_USE(P);
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nslots) return;
  const uint32_t slot = slots[i], own = owner[slot], t = tofs[slot];
  // "attempt >= 576" (dilithium.go:372-377): attempts past the cap are never accepted
  if (flags[slot] == 0 && hintcnt[slot] <= OMEGA && attempt[own] + t + 1 < (uint32_t)MAX_ATTEMPTS)
    atomicMin(best + own, (t << 24) | slot);
}

// phase 2, one warp per active op: accepted -> c~, z and hints of the winning slot into the signature, the op id
// joins the free-slot list; rejected -> T more attempts are spent and the op joins the next active list.
template <class P>
__global__ void __launch_bounds__(128) finalize_kernel(const uint32_t* __restrict__ act, size_t nact, int T,
                                                       const uint64_t* __restrict__ ctilde,
                                                       const uint8_t* __restrict__ zbuf,
                                                       const uint32_t* __restrict__ hintbits, uint32_t* __restrict__ best,
                                                       uint32_t* __restrict__ attempt, uint8_t* __restrict__ sig,
                                                       uint8_t* __restrict__ status, uint32_t* __restrict__ next,
                                                       uint32_t* __restrict__ next_count, uint32_t* __restrict__ done,
                                                       uint32_t* __restrict__ done_count,
                                                       unsigned long long* __restrict__ total_attempts) {
  MLDSA_USE(P);
  const size_t s = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (s >= nact) return;
  const size_t op = act[s];
  uint8_t* sg = sig + op * (size_t)SIG_BYTES;
  const uint32_t b = best[op];
  __syncwarp();
  if (lane == 0) best[op] = 0xffffffffu;
  if (b != 0xffffffffu) {
    const size_t slot = b & 0xffffffu;
    const uint8_t* ct = reinterpret_cast<const uint8_t*>(ctilde + (CTILDE / 8) * slot);
    for (int i = lane; i < CTILDE; i += 32) sg[i] = ct[i];
    // z: word-aligned staging rows into a signature that starts at an arbitrary byte (SIG_BYTES is odd): bytes up to
    // the first aligned destination word, then aligned words assembled from two source words, then the tail bytes
    const uint8_t* zs = zbuf + slot * (size_t)(L * POLY_Z);
    const uint32_t* zw = reinterpret_cast<const uint32_t*>(zs);
    uint8_t* zd = sg + CTILDE;
    constexpr int ZB = L * POLY_Z;
    const int head = (int)((4 - (reinterpret_cast<uintptr_t>(zd) & 3)) & 3);
    if (lane < head) zd[lane] = zs[lane];
    uint32_t* dw = reinterpret_cast<uint32_t*>(zd + head);
    const int nw = (ZB - head) >> 2;
    // head == 0: the shift is 0 and word j + 1 of the last iteration would lie past the row
    for (int j = lane; j < nw; j += 32) dw[j] = __funnelshift_r(zw[j], head ? zw[j + 1] : 0u, 8 * head);
    for (int i = head + 4 * nw + lane; i < ZB; i += 32) zd[i] = zs[i];
    if (lane == 0) {
      uint8_t* hb = sg + CTILDE + L * POLY_Z;  // PackHint (internal/pack.go:77-95)
      int off = 0;
      for (int i = 0; i < K; i++) {
        for (int w = 0; w < 8; w++) {
          uint32_t m = hintbits[8 * K * slot + 8 * i + w];
          while (m) {
            const int bit = __ffs(m) - 1;
            hb[off++] = (uint8_t)(32 * w + bit);
            m &= m - 1;
          }
        }
        hb[OMEGA + i] = (uint8_t)off;
      }
      for (; off < OMEGA; off++) hb[off] = 0;
      if (status) status[op] = 0;
      atomicAdd(total_attempts, (unsigned long long)(attempt[op] + (b >> 24) + 1));
      done[atomicAdd(done_count, 1u)] = (uint32_t)op;
    }
  } else {
    const uint32_t at = attempt[op] + T;
    __syncwarp();
    if (at + 1 >= (uint32_t)MAX_ATTEMPTS) {  // every attempt below the cap has been tried: give up, flag the op
      for (int i = lane; i < SIG_BYTES; i += 32) sg[i] = 0;
      if (lane == 0) {
        if (status) status[op] = 1;
        atomicAdd(total_attempts, (unsigned long long)(MAX_ATTEMPTS - 1));
        done[atomicAdd(done_count, 1u)] = (uint32_t)op;
      }
    } else if (lane == 0) {
      next[atomicAdd(next_count, 1u)] = (uint32_t)op;
    }
    if (lane == 0) attempt[op] = at;
  }
}

__global__ void iota_kernel(uint32_t* a, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = (uint32_t)i;
}

// ================================================================== Verify (SURVEY.md 8(f) row 3)
// internal/dilithium.go:273-332.  pk = rho (32) || t1 (6 x 320); sig = c~ (48) || z (5 x 640) || hints (61).

// tr = H(pk), mu = H(tr || M'), c = SampleInBall(c~), hint unpacking with the validity rules of
// UnpackHint (internal/pack.go:113-140).  One thread per op.
template <class P>
__global__ void __launch_bounds__(128) verify_prep_kernel(const uint8_t* __restrict__ pk, size_t pk_stride,
                                                          const uint8_t* __restrict__ msgs,
                                                          const uint64_t* __restrict__ msg_off,
                                                          const uint8_t* __restrict__ ctxstr, int ctxlen, int internal,
                                                          const uint8_t* __restrict__ sig, size_t n,
                                                          uint64_t* __restrict__ mu, uint32_t* __restrict__ cpoly,
                                                          uint32_t* __restrict__ hintbits, uint32_t* __restrict__ flags) {
  MLDSA_USE(P);
  const size_t op = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (op >= n) return;
  const uint8_t* pkp = pk + op * pk_stride;
  const uint8_t* sg = sig + op * (size_t)SIG_BYTES;
  uint64_t a[25];
  keccak::zero(a);
  {  // tr = SHAKE256(pk, 64) (dilithium.go:122-125)
    constexpr int PW = PK_BYTES / 8, FULL = PW / 17, REM = PW % 17;
    const uint64_t* pw = reinterpret_cast<const uint64_t*>(pkp);
#pragma unroll 1
    for (int b = 0; b < FULL; b++) {
#pragma unroll
      for (int w = 0; w < 17; w++) a[w] ^= __ldg(pw + 17 * b + w);
      keccak::f1600(a);
    }
#pragma unroll
    for (int w = 0; w < REM; w++) a[w] ^= __ldg(pw + 17 * FULL + w);
    a[REM] ^= 0x1f;
    a[16] ^= 0x8000000000000000ull;
    keccak::f1600(a);
  }
  ByteSponge sp;
  sp.init();
  for (int i = 0; i < TR; i++) sp.put((uint8_t)(a[i >> 3] >> (8 * (i & 7))));
  if (!internal && P::NIST) {
    sp.put(0);
    sp.put((uint8_t)ctxlen);
    for (int i = 0; i < ctxlen; i++) sp.put(ctxstr[i]);
  }
  for (uint64_t i = msg_off[op]; i < msg_off[op + 1]; i++) sp.put(msgs[i]);
  sp.finish();
#pragma unroll
  for (int i = 0; i < 8; i++) mu[8 * op + i] = sp.a[i];
  // c = SampleInBall(sig.c)
  keccak::zero(a);
  for (int i = 0; i < CTILDE; i++) a[i >> 3] |= (uint64_t)sg[i] << (8 * (i & 7));
  a[CTILDE / 8] = 0x1f;
  a[16] = 0x8000000000000000ull;
  keccak::f1600(a);
  uint64_t buf[17];
#pragma unroll
  for (int i = 0; i < 17; i++) buf[i] = a[i];
  uint64_t signs = buf[0];
  int off = 8;
  uint32_t* c = cpoly + op * N;
  for (int i = 0; i < N; i += 4) *reinterpret_cast<uint4*>(c + i) = make_uint4(0, 0, 0, 0);
  for (int i = N - TAU; i < N; i++) {
    uint32_t b;
    for (;;) {
      if (off >= 136) {
        keccak::f1600(a);
#pragma unroll
        for (int q = 0; q < 17; q++) buf[q] = a[q];
        off = 0;
      }
      b = (uint32_t)(buf[off >> 3] >> (8 * (off & 7))) & 0xff;
      off++;
      if (b <= (uint32_t)i) break;
    }
    c[i] = c[b];
    c[b] = (signs & 1) ? Q - 1 : 1;
    signs >>= 1;
  }
  // UnpackHint
  uint32_t* hb = hintbits + 8 * K * op;
  for (int i = 0; i < 8 * K; i++) hb[i] = 0;
  const uint8_t* hp = sg + CTILDE + L * POLY_Z;
  bool ok = true;
  int prev = 0;
  for (int i = 0; i < K && ok; i++) {
    const int sop = hp[OMEGA + i];
    if (sop < prev || sop > OMEGA) {
      ok = false;
      break;
    }
    for (int j = prev; j < sop; j++) {
      if (j > prev && hp[j] <= hp[j - 1]) {
        ok = false;
        break;
      }
      hb[8 * i + (hp[j] >> 5)] |= 1u << (hp[j] & 31);
    }
    prev = sop;
  }
  for (int j = prev; j < OMEGA && ok; j++)
    if (hp[j] != 0) ok = false;
  flags[op] = ok ? 0u : 1u;
}

// zh[j] = NTT(UnpackLeGamma1(sig.z[j])), reject if z exceeds gamma1 - beta (dilithium.go:87-90): octet per (op, j)
template <class P>
__global__ void __launch_bounds__(128) verify_z_kernel(const uint8_t* __restrict__ sig, size_t n, uint32_t* __restrict__ zh,
                                                       uint32_t* __restrict__ flags, const uint32_t* __restrict__ zetas) {
  MLDSA_USE(P);
  __shared__ __align__(16) uint32_t tiles[16 * kPolyWords];
  const OctetCtx o = octet_ctx(tiles);
  const unsigned octmask = 0xffu << (8 * o.oct);
  const size_t total = n * L, base = ((size_t)blockIdx.x * 4 + o.warp) * 4;
  if (base >= total) return;
  const bool active = base + o.oct < total;
  const size_t u = active ? base + o.oct : total - 1;
  const size_t op = u % n;
  const int j = (int)(u / n);
  const uint8_t* zb = sig + op * (size_t)SIG_BYTES + CTILDE + POLY_Z * j + 4 * ZBITS * o.v;  // unaligned: byte loads
  uint32_t zw[ZBITS + 1];
#pragma unroll
  for (int q = 0; q < ZBITS; q++)
    zw[q] = (uint32_t)zb[4 * q] | ((uint32_t)zb[4 * q + 1] << 8) | ((uint32_t)zb[4 * q + 2] << 16) | ((uint32_t)zb[4 * q + 3] << 24);
  zw[ZBITS] = 0;
  uint32_t r[32];
  bool reject = false;
#pragma unroll
  for (int q = 0; q < 32; q++) {  // PolyUnpackLeGamma1 (internal/pack.go:146-203)
    uint32_t c = GAMMA1 - field32<ZBITS>(zw, q);
    c += (uint32_t)((int32_t)c >> 31) & Q;
    reject |= exceeds1(c, GAMMA1 - BETA);
    r[q] = c;
  }
  c_to_s(r, o.tile, o.v);
  LaneTw t;
  load_lane_tw_fwd(t, zetas, o.v);
  ntt_octet(r, o.tile, o.v, t);
  gstore_C_via_tile(zh + (op * L + j) * N, o.tile, o.v, r, active);
  reject = __any_sync(octmask, reject);
  if (reject && active && o.v == 0) atomicOr(flags + op, 1u);
}

// w1' = UseHint(InvNTT(A z - c t1 2^d), h), packed (dilithium.go:297-316, rounding.go:98-135): octet per (op, i)
template <class P>
__global__ void __launch_bounds__(128) verify_w_kernel(const uint8_t* __restrict__ pk, size_t pk_stride, int key_shared,
                                                       const uint32_t* __restrict__ A, const uint32_t* __restrict__ zh,
                                                       const uint32_t* __restrict__ cpoly,
                                                       const uint32_t* __restrict__ hintbits, size_t n,
                                                       uint8_t* __restrict__ w1u, const uint32_t* __restrict__ zetas) {
  MLDSA_USE(P);
  __shared__ __align__(16) uint32_t tiles[16 * kPolyWords];
  __shared__ __align__(8) uint2 izs[256];
  stage_inv_pairs(izs, zetas);
  __syncthreads();
  const OctetCtx o = octet_ctx(tiles);
  const size_t total = n * K, base = ((size_t)blockIdx.x * 4 + o.warp) * 4;
  if (base >= total) return;
  const bool active = base + o.oct < total;
  const size_t u = active ? base + o.oct : total - 1;
  const size_t op = u % n;
  const int i = (int)(u / n);
  // t1[i] * 2^d, NTT  (dilithium.go:299-300); t1: 10-bit fields, 32 coefficients = 40 bytes = 10 words
  uint32_t r[32];
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(pk + op * pk_stride + 32 + POLY_T1 * i + 40 * o.v);
    uint32_t w[11];
#pragma unroll
    for (int q = 0; q < 10; q++) w[q] = __ldg(src + q);
    w[10] = 0;
#pragma unroll
    for (int q = 0; q < 32; q++) {
      const int bit = 10 * q, wi = bit >> 5, sh = bit & 31;
      uint32_t f = w[wi] >> sh;
      if (sh > 22) f |= w[wi + 1] << (32 - sh);
      r[q] = (f & 0x3ff) << 13;
    }
  }
  c_to_s(r, o.tile, o.v);
  {
    LaneTw t;
    load_lane_tw_fwd(t, zetas, o.v);
    ntt_octet(r, o.tile, o.v, t);
  }
  // Az[i] - c-hat * that, ReduceLe2Q (C layout)
  const uint32_t* Ai = A + ((key_shared ? 0 : op) * (K * L) + i * L) * N;
  const uint4* cp = reinterpret_cast<const uint4*>(cpoly + op * N + 32 * o.v);
#pragma unroll
  for (int c = 0; c < 8; c++) {
    const uint4 ch = cp[c];
    r[4 * c] = 2 * Q - mont_mul(r[4 * c], ch.x);
    r[4 * c + 1] = 2 * Q - mont_mul(r[4 * c + 1], ch.y);
    r[4 * c + 2] = 2 * Q - mont_mul(r[4 * c + 2], ch.z);
    r[4 * c + 3] = 2 * Q - mont_mul(r[4 * c + 3], ch.w);
  }
#pragma unroll 1
  for (int j = 0; j < L; j++) {
    const uint4* ap = reinterpret_cast<const uint4*>(Ai + j * N + 32 * o.v);
    const uint4* zp = reinterpret_cast<const uint4*>(zh + (op * L + j) * N + 32 * o.v);
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const uint4 x = __ldg(ap + c), z = zp[c];
      r[4 * c] += mont_mul(x.x, z.x);
      r[4 * c + 1] += mont_mul(x.y, z.y);
      r[4 * c + 2] += mont_mul(x.z, z.z);
      r[4 * c + 3] += mont_mul(x.w, z.w);
    }
  }
#pragma unroll
  for (int c = 0; c < 32; c++) r[c] = reduce_le2q(r[c]);
  invntt_octet_smem(r, o.tile, o.v, izs);  // -> S layout
  uint8_t* w1b = w1u + (op * K + i) * 256;
  const uint32_t* hb = hintbits + 8 * K * op + 8 * i;
#pragma unroll
  for (int s = 0; s < 16; s++) {
    const uint32_t hbits = (hb[s >> 1] >> (16 * (s & 1) + 2 * o.v)) & 3;
    uint32_t q[2], h[2];
    decompose<P>(le2q_modq(r[2 * s]), q[0], h[0]);
    decompose<P>(le2q_modq(r[2 * s + 1]), q[1], h[1]);
#pragma unroll
    for (int e = 0; e < 2; e++) {  // PolyUseHint (rounding.go:98-135)
      if (!((hbits >> e) & 1)) continue;
      if constexpr (P::GAMMA2 == 261888) {
        h[e] = (q[e] > Q) ? ((h[e] + 1) & 15) : ((h[e] - 1) & 15);
      } else {
        if (q[e] > Q)
          h[e] = (h[e] == 43) ? 0 : h[e] + 1;
        else
          h[e] = (h[e] == 0) ? 43 : h[e] - 1;
      }
    }
    if (active) *reinterpret_cast<uint16_t*>(w1b + 16 * s + 2 * o.v) = (uint16_t)(h[0] | (h[1] << 8));
  }
}

// ok = valid && (c~ == H(mu || w1')) (dilithium.go:318-331): thread per op
template <class P>
__global__ void __launch_bounds__(128) verify_final_kernel(const uint8_t* __restrict__ sig, const uint64_t* __restrict__ mu,
                                                           const uint8_t* __restrict__ w1u,
                                                           const uint32_t* __restrict__ flags, size_t n,
                                                           uint8_t* __restrict__ okout) {
  MLDSA_USE(P);
  const size_t op = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (op >= n) return;
  uint64_t a[25];
  keccak::zero(a);
  constexpr int WORDS = 8 + K * POLY_W1 / 8, FULL = WORDS / 17, REM = WORDS % 17;
  const uint8_t* w1o = w1u + op * (K * 256);
#pragma unroll 1
  for (int b = 0; b < FULL; b++) {
#pragma unroll
    for (int w = 0; w < 17; w++) {
      const int k = 17 * b + w;
      a[w] ^= (k < 8) ? mu[8 * op + k] : w1_word<P>(w1o, k - 8);
    }
    keccak::f1600(a);
  }
#pragma unroll
  for (int w = 0; w < REM; w++) a[w] ^= w1_word<P>(w1o, 17 * FULL + w - 8);
  a[REM] ^= 0x1f;
  a[16] ^= 0x8000000000000000ull;
  keccak::f1600(a);
  const uint8_t* sg = sig + op * (size_t)SIG_BYTES;
  bool same = true;
  for (int i = 0; i < CTILDE; i++) same &= sg[i] == (uint8_t)(a[i >> 3] >> (8 * (i & 7)));
  okout[op] = (same && flags[op] == 0) ? 1 : 0;
}

template <class P>
static int verify_device(const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                         const uint8_t* ctxstr, int ctxlen, const uint8_t* sig, uint8_t* okout, size_t n, int internal,
                         cudaStream_t st, int slot) {
  MLDSA_USE(P);
  Dev& c = ctx();
  const bool shared = pk_stride == 0;
  const size_t nkeys = shared ? 1 : n;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t oA = take(nkeys * K * L * 1024), oMu = take(n * 64), oZh = take(n * L * 1024), oC = take(n * 1024),
               oHb = take(n * 8 * K * 4), oFl = take(n * 4), oW1 = take(n * K * 256), oAct = take(n * 4);
  void* base = nullptr;
  int rc = ensure_work(slot, off, &base);
  if (rc) return rc;
  char* b = (char*)base;
  uint32_t* A = (uint32_t*)(b + oA);
  uint64_t* mu = (uint64_t*)(b + oMu);
  uint32_t* zh = (uint32_t*)(b + oZh);
  uint32_t* cp = (uint32_t*)(b + oC);
  uint32_t* hb = (uint32_t*)(b + oHb);
  uint32_t* fl = (uint32_t*)(b + oFl);
  uint8_t* w1p = (uint8_t*)(b + oW1);
  uint32_t* act = (uint32_t*)(b + oAct);
  const uint32_t* zetas = (const uint32_t*)c.dil_tw;
  if (int arc = ensure_smem_attr((const void*)expand_a_kernel<P>, kExpThreads * kExpRow * 4)) return arc;
  auto blocks = [](size_t units, size_t per) { return (unsigned)((units + per - 1) / per); };
  {
    KernelScope ks(KID_MLDSA_EXPAND, st);  // ExpandA(rho): rho is the first 32 bytes of pk
    expand_a_kernel<P><<<blocks(nkeys * K * L, kExpThreads), kExpThreads, kExpThreads * kExpRow * 4, st>>>(pk, pk_stride,
                                                                                                        nkeys, A);
  }
  {
    KernelScope ks(KID_MLDSA_MU, st);
    verify_prep_kernel<P><<<blocks(n, 128), 128, 0, st>>>(pk, pk_stride, msgs, msg_off, ctxstr, ctxlen, internal, sig, n, mu,
                                                       cp, hb, fl);
  }
  {
    KernelScope ks(KID_MLDSA_W, st);
    verify_z_kernel<P><<<blocks(n * L, 16), 128, 0, st>>>(sig, n, zh, fl, zetas);
  }
  {
    KernelScope ks(KID_MLDSA_COMPACT, st);
    iota_kernel<<<blocks(n, 256), 256, 0, st>>>(act, n);
  }
  {
    KernelScope ks(KID_MLDSA_RESPONSE, st);
    cntt_kernel<<<blocks(n, 16), 128, 0, st>>>(act, n, cp, zetas);
  }
  {
    KernelScope ks(KID_MLDSA_W, st);
    verify_w_kernel<P><<<blocks(n * K, 16), 128, 0, st>>>(pk, pk_stride, shared ? 1 : 0, A, zh, cp, hb, n, w1p, zetas);
  }
  {
    KernelScope ks(KID_MLDSA_CHALLENGE, st);
    verify_final_kernel<P><<<blocks(n, 128), 128, 0, st>>>(sig, mu, w1p, fl, n, okout);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// ================================================================== KeyGen (SURVEY.md 8(f) row 2)
// NewKeyFromSeed, internal/dilithium.go:181-241 (+ computeT0andT1 :253-267).
// (rho, rho', key) = SHAKE256(seed || K || L, 128); thread per op
template <class P>
__global__ void __launch_bounds__(128) kg_seed_kernel(const uint8_t* __restrict__ seed, size_t n, uint8_t* __restrict__ pk,
                                                      uint8_t* __restrict__ sk, uint64_t* __restrict__ sseed) {
  MLDSA_USE(P);
  const size_t op = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (op >= n) return;
  const uint64_t* sd = reinterpret_cast<const uint64_t*>(seed + 32 * op);
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll
  for (int i = 0; i < 4; i++) a[i] = sd[i];
  a[4] = P::NIST ? ((uint64_t)K | ((uint64_t)L << 8) | (0x1full << 16)) : 0x1full;  // dilithium.go:191-193
  a[16] = 0x8000000000000000ull;
  keccak::f1600(a);
  uint64_t* pkw = reinterpret_cast<uint64_t*>(pk + op * (size_t)PK_BYTES);
  uint64_t* skw = reinterpret_cast<uint64_t*>(sk + op * (size_t)SK_BYTES);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    pkw[i] = a[i];       // rho
    skw[i] = a[i];
    skw[4 + i] = a[12 + i];  // key = eSeed[96:128]
  }
#pragma unroll
  for (int i = 0; i < 8; i++) sseed[8 * op + i] = a[4 + i];  // rho' = eSeed[32:96]
}

// One SHAKE256 stream of PolyDeriveUniformLeqEta (sample.go:129-181): `a` holds the absorbed, padded block
// seed || nonce; row[i] = t_i, the accepted nibble (reduced mod 5 for eta = 2), i.e. eta - coefficient.
template <int ETA>
__device__ __forceinline__ void leqeta_stream(uint64_t (&a)[25], uint32_t* row) {
  int ctr = 0;
  do {
    keccak::f1600(a);
#pragma unroll
    for (int w = 0; w < 17; w++) {
      const uint64_t x = a[w];
#pragma unroll
      for (int q = 0; q < 16; q++) {
        uint32_t t = (uint32_t)(x >> (4 * q)) & 15;
        bool ok;
        if constexpr (ETA == 2) {  // accept t <= 14, reduce mod 5 (sample.go:144-156)
          ok = t <= 14;
          t -= ((205 * t) >> 10) * 5;
        } else {
          ok = t <= 2 * ETA;
        }
        row[ctr] = t;  // eta - coefficient; Q + eta - t is formed on the way out
        ctr += (ok && ctr < N);
      }
    }
  } while (ctr < N);
}

// s1, s2 = PolyDeriveUniformLeqEta (sample.go:129-181, eta = 4): thread per (op, poly); the accepted nibbles
// are at once the PackLeqEta image (internal/pack.go:13-20), so the packed key is written here too.
template <class P>
__global__ void __launch_bounds__(kExpThreads) kg_eta_kernel(const uint64_t* __restrict__ sseed, size_t n,
                                                             uint32_t* __restrict__ spoly, uint8_t* __restrict__ sk) {
  MLDSA_USE(P);
  extern __shared__ __align__(16) uint32_t rows[];
  const size_t s0 = (size_t)blockIdx.x * blockDim.x, total = n * (L + K);
  const size_t s = s0 + threadIdx.x;
  const size_t sc = s < total ? s : total - 1;
  const size_t op = sc % n;
  const int p = (int)(sc / n);
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll
  for (int w = 0; w < 8; w++) a[w] = sseed[8 * op + w];
  a[8] = (uint64_t)p | (0x1full << 16);  // nonce = p (s1: 0..L-1, s2: L..L+K-1), little endian 16 bit
  a[16] = 0x8000000000000000ull;
  leqeta_stream<ETA>(a, rows + threadIdx.x * kExpRow);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int q = warp; q < kExpThreads; q += kExpThreads / 32) {
    const size_t sp = s0 + q;
    if (sp >= total) break;
    const size_t qop = sp % n;
    const int qp = (int)(sp / n);
    uint32_t* dst = spoly + (qop * (L + K) + qp) * N;
    uint8_t* pb = sk + qop * (size_t)SK_BYTES + OFF_S1 + POLY_ETA * qp;
    // each lane owns coefficients 8*lane .. 8*lane+7: 8 values -> 4 bytes (eta = 4) or 3 bytes (eta = 2)
    uint32_t t[8];
#pragma unroll
    for (int e = 0; e < 8; e++) t[e] = rows[q * kExpRow + 8 * lane + e];
    *reinterpret_cast<uint4*>(dst + 8 * lane) = make_uint4(Q + ETA - t[0], Q + ETA - t[1], Q + ETA - t[2], Q + ETA - t[3]);
    *reinterpret_cast<uint4*>(dst + 8 * lane + 4) = make_uint4(Q + ETA - t[4], Q + ETA - t[5], Q + ETA - t[6], Q + ETA - t[7]);
    if constexpr (ETA == 4) {
#pragma unroll
      for (int e = 0; e < 4; e++) pb[4 * lane + e] = (uint8_t)(t[2 * e] | (t[2 * e + 1] << 4));
    } else {
      uint32_t bits = 0;
#pragma unroll
      for (int e = 0; e < 8; e++) bits |= t[e] << (3 * e);
      pb[3 * lane] = (uint8_t)bits;
      pb[3 * lane + 1] = (uint8_t)(bits >> 8);
      pb[3 * lane + 2] = (uint8_t)(bits >> 16);
    }
  }
}

// s1h = NTT(s1): octet per (op, j)
template <class P>
__global__ void __launch_bounds__(128) kg_s1ntt_kernel(const uint32_t* __restrict__ spoly, size_t n, uint32_t* __restrict__ s1h,
                                                       const uint32_t* __restrict__ zetas) {
  MLDSA_USE(P);
  __shared__ __align__(16) uint32_t tiles[16 * kPolyWords];
  const OctetCtx o = octet_ctx(tiles);
  const size_t total = n * L, base = ((size_t)blockIdx.x * 4 + o.warp) * 4;
  if (base >= total) return;
  const bool active = base + o.oct < total;
  const size_t u = active ? base + o.oct : total - 1;
  const size_t op = u % n;
  const int j = (int)(u / n);
  uint32_t r[32];
  gload_S(spoly + (op * (L + K) + j) * N, o.v, r);
  LaneTw t;
  load_lane_tw_fwd(t, zetas, o.v);
  ntt_octet(r, o.tile, o.v, t);
  gstore_C_via_tile(s1h + (op * L + j) * N, o.tile, o.v, r, active);
}

// t = Normalize(InvNTT(ReduceLe2Q(A[i] . s1h)) + s2[i]); Power2Round; PackT1 -> pk, PackT0 -> sk: octet per (op, i)
template <class P>
__global__ void __launch_bounds__(128) kg_t_kernel(const uint32_t* __restrict__ A, const uint32_t* __restrict__ s1h,
                                                   const uint32_t* __restrict__ spoly, size_t n, uint8_t* __restrict__ pk,
                                                   uint8_t* __restrict__ sk, const uint32_t* __restrict__ zetas) {
  MLDSA_USE(P);
  __shared__ __align__(16) uint32_t tiles[16 * kPolyWords];
  const OctetCtx o = octet_ctx(tiles);
  const size_t total = n * K, base = ((size_t)blockIdx.x * 4 + o.warp) * 4;
  if (base >= total) return;
  const bool active = base + o.oct < total;
  const size_t u = active ? base + o.oct : total - 1;
  const size_t op = u % n;
  const int i = (int)(u / n);
  const uint32_t* Ai = A + (op * (K * L) + i * L) * N;
  uint32_t r[32];
#pragma unroll
  for (int c = 0; c < 32; c++) r[c] = 0;
#pragma unroll 1
  for (int j = 0; j < L; j++) {
    const uint4* ap = reinterpret_cast<const uint4*>(Ai + j * N + 32 * o.v);
    const uint4* sp = reinterpret_cast<const uint4*>(s1h + (op * L + j) * N + 32 * o.v);
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const uint4 x = __ldg(ap + c), z = sp[c];
      r[4 * c] += mont_mul(x.x, z.x);
      r[4 * c + 1] += mont_mul(x.y, z.y);
      r[4 * c + 2] += mont_mul(x.z, z.z);
      r[4 * c + 3] += mont_mul(x.w, z.w);
    }
  }
#pragma unroll
  for (int c = 0; c < 32; c++) r[c] = reduce_le2q(r[c]);
  LaneTw t;
  load_lane_tw_inv(t, zetas, o.v);
  invntt_octet(r, o.tile, o.v, t);  // S layout
  const uint32_t* s2 = spoly + (op * (L + K) + L + i) * N;
#pragma unroll
  for (int s = 0; s < 16; s++) {
    const uint2 e = *reinterpret_cast<const uint2*>(s2 + 16 * s + 2 * o.v);
    r[2 * s] = modq(r[2 * s] + e.x);
    r[2 * s + 1] = modq(r[2 * s + 1] + e.y);
  }
  s_to_c(r, o.tile, o.v);
  // Power2Round (field.go:35-49), PackT1 (pack.go:88-100): 10 words, PackT0 (pack.go:23-54): 13 words
  uint64_t acc1 = 0, acc0 = 0;
  int b1 = 0, b0 = 0, o1 = 0, o0 = 0;
  uint32_t* d1 = reinterpret_cast<uint32_t*>(pk + op * (size_t)PK_BYTES + 32 + POLY_T1 * i) + 10 * o.v;
  uint32_t* d0 = reinterpret_cast<uint32_t*>(sk + op * (size_t)SK_BYTES + OFF_T0 + 416 * i) + 13 * o.v;
#pragma unroll
  for (int c = 0; c < 32; c++) {
    const uint32_t a = r[c];
    uint32_t a0 = a & 0x1fff;
    a0 -= (1u << 12) + 1;
    a0 += (uint32_t)((int32_t)a0 >> 31) & (1u << 13);
    a0 -= (1u << 12) - 1;
    const uint32_t a1 = (a - a0) >> 13;
    acc1 |= (uint64_t)(a1 & 0x3ff) << b1;
    b1 += 10;
    if (b1 >= 32) {
      if (active) d1[o1] = (uint32_t)acc1;
      o1++;
      acc1 >>= 32;
      b1 -= 32;
    }
    acc0 |= (uint64_t)(((1u << 12) - a0) & 0x1fff) << b0;  // Q + 2^12 - (Q + a0)
    b0 += 13;
    if (b0 >= 32) {
      if (active) d0[o0] = (uint32_t)acc0;
      o0++;
      acc0 >>= 32;
      b0 -= 32;
    }
  }
}

// tr = SHAKE256(pk, 64) -> sk[64:128] (dilithium.go:233-236): thread per op
template <class P>
__global__ void __launch_bounds__(128) kg_tr_kernel(const uint8_t* __restrict__ pk, size_t n, uint8_t* __restrict__ sk) {
  MLDSA_USE(P);
  const size_t op = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (op >= n) return;
  const uint64_t* pw = reinterpret_cast<const uint64_t*>(pk + op * (size_t)PK_BYTES);
  uint64_t a[25];
  keccak::zero(a);
  constexpr int PW = PK_BYTES / 8, FULL = PW / 17, REM = PW % 17;
#pragma unroll 1
  for (int b = 0; b < FULL; b++) {
#pragma unroll
    for (int w = 0; w < 17; w++) a[w] ^= pw[17 * b + w];
    keccak::f1600(a);
  }
#pragma unroll
  for (int w = 0; w < REM; w++) a[w] ^= pw[17 * FULL + w];
  a[REM] ^= 0x1f;
  a[16] ^= 0x8000000000000000ull;
  keccak::f1600(a);
  uint64_t* tr = reinterpret_cast<uint64_t*>(sk + op * (size_t)SK_BYTES + OFF_TR);
#pragma unroll
  for (int i = 0; i < TR / 8; i++) tr[i] = a[i];
}

template <class P>
static int keygen_device(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n, cudaStream_t st, int slot) {
  MLDSA_USE(P);
  Dev& c = ctx();
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t oA = take(n * K * L * 1024), oSs = take(n * 64), oSp = take(n * (L + K) * 1024), oSh = take(n * L * 1024);
  void* base = nullptr;
  int rc = ensure_work(slot, off, &base);
  if (rc) return rc;
  char* b = (char*)base;
  uint32_t* A = (uint32_t*)(b + oA);
  uint64_t* sseed = (uint64_t*)(b + oSs);
  uint32_t* spoly = (uint32_t*)(b + oSp);
  uint32_t* s1h = (uint32_t*)(b + oSh);
  const uint32_t* zetas = (const uint32_t*)c.dil_tw;
  if (int arc = ensure_smem_attr((const void*)expand_a_kernel<P>, kExpThreads * kExpRow * 4)) return arc;
  if (int arc = ensure_smem_attr((const void*)kg_eta_kernel<P>, kExpThreads * kExpRow * 4)) return arc;
  auto blocks = [](size_t units, size_t per) { return (unsigned)((units + per - 1) / per); };
  {
    KernelScope ks(KID_MLDSA_MU, st);
    kg_seed_kernel<P><<<blocks(n, 128), 128, 0, st>>>(seeds, n, pk, sk, sseed);
  }
  {
    KernelScope ks(KID_MLDSA_MASK, st);
    kg_eta_kernel<P><<<blocks(n * (L + K), kExpThreads), kExpThreads, kExpThreads * kExpRow * 4, st>>>(sseed, n, spoly, sk);
  }
  {
    KernelScope ks(KID_MLDSA_EXPAND, st);
    expand_a_kernel<P><<<blocks(n * K * L, kExpThreads), kExpThreads, kExpThreads * kExpRow * 4, st>>>(pk, PK_BYTES, n, A);
  }
  {
    KernelScope ks(KID_MLDSA_W, st);
    kg_s1ntt_kernel<P><<<blocks(n * L, 16), 128, 0, st>>>(spoly, n, s1h, zetas);
  }
  {
    KernelScope ks(KID_MLDSA_W, st);
    kg_t_kernel<P><<<blocks(n * K, 16), 128, 0, st>>>(A, s1h, spoly, n, pk, sk, zetas);
  }
  {
    KernelScope ks(KID_MLDSA_CHALLENGE, st);
    kg_tr_kernel<P><<<blocks(n, 128), 128, 0, st>>>(pk, n, sk);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------ host side
template <class P>
static int sign_device(const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                       const uint8_t* ctxstr, int ctxlen, const uint8_t* rnd, uint8_t* sig, uint8_t* status, size_t n,
                       int internal, cudaStream_t st, int slot, uint64_t* attempts_out, volatile uint32_t* h_count) {
  // h_count: 8 bytes of pinned host memory for the per-round counter (owned by the caller: the host-pointer path
  // keeps per-op status bytes in the same pinned block)
  MLDSA_USE(P);
  Dev& c = ctx();
  const bool shared = sk_stride == 0;
  const size_t nkeys = shared ? 1 : n;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t oA = take(nkeys * K * L * 1024), oS = take(nkeys * NKEYPOLY * 1024), oMu = take(n * 64),
               oRh = take(n * 64), oY = take(n * L * 1024), oYh = take(n * L * 1024), oW0 = take(n * K * 1024),
               oW1 = take(n * K * SignW1<P>::stride), oCm = take(n * 64), oZ = take(n * L * POLY_Z), oC = take(n * 1024), oCt = take(n * CTILDE), oHb = take(n * 8 * K * 4),
               oFl = take(n * 4), oHc = take(n * 4), oAt = take(n * 4), oA0 = take(n * 4), oA1 = take(n * 4),
               oPs = take(n * 8), oL1 = take(n * 4), oL2 = take(n * 4), oOw = take(n * 4), oTo = take(n * 4),
               oBe = take(n * 4), oDn = take(n * 4), oSl = take(n * 4), oCnt = take(32);
  void* base = nullptr;
  int rc = ensure_work(slot, off, &base);
  if (rc) return rc;
  char* b = (char*)base;
  Work w;
  w.A = (uint32_t*)(b + oA);
  w.sh = (uint32_t*)(b + oS);
  w.mu = (uint64_t*)(b + oMu);
  w.rhop = (uint64_t*)(b + oRh);
  w.y = (uint32_t*)(b + oY);
  w.yh = (uint32_t*)(b + oYh);
  w.w0 = (uint32_t*)(b + oW0);
  w.w1u = (uint8_t*)(b + oW1);
  w.cmask = (uint32_t*)(b + oCm);
  w.zbuf = (uint8_t*)(b + oZ);
  w.c = (uint32_t*)(b + oC);
  w.ctilde = (uint64_t*)(b + oCt);
  w.hintbits = (uint32_t*)(b + oHb);
  w.flags = (uint32_t*)(b + oFl);
  w.hintcnt = (uint32_t*)(b + oHc);
  w.attempt = (uint32_t*)(b + oAt);
  w.act[0] = (uint32_t*)(b + oA0);
  w.act[1] = (uint32_t*)(b + oA1);
  w.count = (uint32_t*)(b + oCnt);
  w.pass = (uint32_t*)(b + oPs);
  w.list1 = (uint32_t*)(b + oL1);
  w.list2 = (uint32_t*)(b + oL2);
  w.owner = (uint32_t*)(b + oOw);
  w.tofs = (uint32_t*)(b + oTo);
  w.best = (uint32_t*)(b + oBe);
  w.done = (uint32_t*)(b + oDn);
  w.slots = (uint32_t*)(b + oSl);
  const uint32_t* zetas = (const uint32_t*)c.dil_tw;
  constexpr int kChSmem = ChLayout<P>::smem;

  if (int arc = ensure_smem_attr((const void*)expand_a_kernel<P>, kExpThreads * kExpRow * 4)) return arc;
  if (kChSmem) if (int arc = ensure_smem_attr((const void*)challenge_kernel<P>, kChSmem)) return arc;
  if (int arc = ensure_smem_attr((const void*)w_kernel<P>, WSm::bytes)) return arc;
  auto blocks = [](size_t units, size_t per) { return (unsigned)((units + per - 1) / per); };
  {
    KernelScope ks(KID_MLDSA_EXPAND, st);
    expand_a_kernel<P><<<blocks(nkeys * K * L, kExpThreads), kExpThreads, kExpThreads * kExpRow * 4, st>>>(sk, sk_stride,
                                                                                                        nkeys, w.A);
  }
  {
    KernelScope ks(KID_MLDSA_EXPAND, st);
    expand_s_kernel<P><<<blocks(nkeys * NKEYPOLY, 16), 128, 0, st>>>(sk, sk_stride, nkeys, w.sh, zetas);
  }
  {
    KernelScope ks(KID_MLDSA_MU, st);
    mu_kernel<P><<<blocks(n, 128), 128, 0, st>>>(sk, sk_stride, msgs, msg_off, ctxstr, ctxlen, internal, rnd, n, w.mu, w.rhop,
                                              w.attempt, w.act[0], w.owner, w.tofs);
  }
  CB200_CUDA(cudaGetLastError());

  size_t nact = n;
  int cur = 0;
  uint64_t total_attempts = 0;
  CB200_CUDA(cudaMemsetAsync(w.count, 0, 32, st));
  CB200_CUDA(cudaMemsetAsync(w.best, 0xff, n * 4, st));
  constexpr int kMaxSpec = 8;
  auto pgrid = [&](size_t units, int per_sm) {
    return (unsigned)std::min<size_t>((units + 15) / 16, (size_t)c.sm_count * per_sm);
  };
  for (int round = 0; nact > 0; round++) {
    if (round >= MAX_ATTEMPTS) break;
    // attempts per op this round: as many as there are free slots (ids of finished ops) to run them in
    const int T = (int)std::min<size_t>(kMaxSpec, 1 + (n - nact) / nact);
    const size_t ns = nact * T;
    const uint32_t* act = w.act[cur];
    const uint32_t* sl = w.slots;
    CB200_CUDA(cudaMemsetAsync(w.count + (cur ^ 1), 0, 4, st));
    CB200_CUDA(cudaMemsetAsync(w.count + 2, 0, 8, st));
    {
      KernelScope ks(KID_MLDSA_COMPACT, st);
      spec_expand_kernel<<<blocks(ns, 256), 256, 0, st>>>(act, nact, T, w.done, w.slots, w.owner, w.tofs);
    }
    {
      KernelScope ks(KID_MLDSA_MASK, st);
      mask_kernel<P><<<blocks(ns * L, 128), 128, 0, st>>>(sl, ns, w.rhop, w.attempt, w.owner, w.tofs, w.y);
    }
    {
      KernelScope ks(KID_MLDSA_W, st);
      yntt_kernel<P><<<blocks(ns * L, 16), 128, 0, st>>>(sl, ns, w.y, w.yh, zetas);
    }
    {
      KernelScope ks(KID_MLDSA_W, st);
      w_kernel<P><<<pgrid(ns * K, kWCtas), 128, WSm::bytes, st>>>(sl, ns, shared ? 1 : 0, w.A, w.yh, w.w0, w.w1u, w.owner, zetas);
    }
    {
      KernelScope ks(KID_MLDSA_CHALLENGE, st);
      challenge_kernel<P><<<blocks(ns, kChThreads), kChThreads, kChSmem, st>>>(sl, ns, w.mu, w.w1u, w.ctilde, w.cmask, w.flags,
                                                                               w.hintcnt, w.pass, w.owner);
    }
    {
      KernelScope ks(KID_MLDSA_RESPONSE, st);
      cntt_mask_kernel<<<blocks(ns, 16), 128, 0, st>>>(sl, ns, w.cmask, w.c, zetas);
    }
    {
      KernelScope ks(KID_MLDSA_RESPONSE, st);
      count_launch(2);  // three launches in this scope
      response_kernel<P, 0><<<pgrid(ns * K, 8), 128, 0, st>>>(sl, nullptr, ns, shared ? 1 : 0, w.sh, w.c, w.y, w.w0, w.w1u,
                                                              w.zbuf, w.hintbits, w.flags, w.hintcnt, w.pass, w.list1,
                                                              w.count + 2, w.owner, zetas);
      response_kernel<P, 1><<<pgrid(ns * L, 8), 128, 0, st>>>(w.list1, w.count + 2, 0, shared ? 1 : 0, w.sh, w.c, w.y, w.w0,
                                                              w.w1u, w.zbuf, w.hintbits, w.flags, w.hintcnt, w.pass + 1,
                                                              w.list2, w.count + 3, w.owner, zetas);
      response_kernel<P, 2><<<pgrid(ns * K, 8), 128, 0, st>>>(w.list2, w.count + 3, 0, shared ? 1 : 0, w.sh, w.c, w.y, w.w0,
                                                              w.w1u, w.zbuf, w.hintbits, w.flags, w.hintcnt, nullptr, nullptr,
                                                              nullptr, w.owner, zetas);
    }
    {
      KernelScope ks(KID_MLDSA_COMPACT, st);
      count_launch(1);  // two launches in this scope
      finalize_bid_kernel<P><<<blocks(ns, 256), 256, 0, st>>>(sl, ns, w.flags, w.hintcnt, w.owner, w.tofs, w.attempt, w.best);
      finalize_kernel<P><<<blocks(nact * 32, 128), 128, 0, st>>>(
          act, nact, T, w.ctilde, w.zbuf, w.hintbits, w.best, w.attempt, sig, status, w.act[cur ^ 1], w.count + (cur ^ 1),
          w.done, w.count + 4, reinterpret_cast<unsigned long long*>(w.count + 6));
    }
    CB200_CUDA(cudaMemcpyAsync((void*)h_count, w.count + (cur ^ 1), 4, cudaMemcpyDeviceToHost, st));
    CB200_CUDA(cudaStreamSynchronize(st));
    nact = *h_count;
    cur ^= 1;
  }
  if (attempts_out) {
    CB200_CUDA(cudaMemcpyAsync((void*)h_count, w.count + 6, 8, cudaMemcpyDeviceToHost, st));
    CB200_CUDA(cudaStreamSynchronize(st));
    total_attempts = *reinterpret_cast<volatile uint64_t*>(h_count);
  }
  CB200_CUDA(cudaGetLastError());
  if (attempts_out) *attempts_out = total_attempts;
  return 0;
}

// ------------------------------------------------------------------ the samplers on their own (thread per polynomial)
// seed bytes at an arbitrary address -> the first `words` lanes of a zeroed state
__device__ __forceinline__ void absorb_seed(uint64_t (&a)[25], const uint8_t* seed, int words) {
  keccak::zero(a);
#pragma unroll
  for (int w = 0; w < 8; w++) {
    if (w >= words) break;
    uint64_t v = 0;
#pragma unroll
    for (int b = 0; b < 8; b++) v |= (uint64_t)seed[8 * w + b] << (8 * b);
    a[w] = v;
  }
}
// rows of kExpRow words -> polynomials (one warp per row, coalesced)
__device__ __forceinline__ void rows_out(const uint32_t* rows, size_t s0, size_t n, uint32_t* __restrict__ polys, uint32_t base,
                                         bool negate) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int p = warp; p < kExpThreads; p += kExpThreads / 32) {
    if (s0 + p >= n) break;
    uint32_t* dst = polys + (s0 + p) * N;
#pragma unroll
    for (int w = 0; w < 8; w++) {
      const uint32_t t = rows[p * kExpRow + 32 * w + lane];
      dst[32 * w + lane] = negate ? base - t : t;
    }
  }
}
__global__ void __launch_bounds__(kExpThreads) derive_uniform_kernel(const uint8_t* __restrict__ seeds, size_t seed_stride,
                                                                     const uint16_t* __restrict__ nonces, size_t n,
                                                                     uint32_t* __restrict__ polys) {
  extern __shared__ __align__(16) uint32_t rows[];
  const size_t s0 = (size_t)blockIdx.x * blockDim.x, s = s0 + threadIdx.x, sc = s < n ? s : n - 1;
  uint64_t a[25];
  absorb_seed(a, seeds + sc * seed_stride, 4);
  a[4] = (uint64_t)nonces[sc] | (0x1full << 16);
  a[20] = 0x8000000000000000ull;
  uniform_stream(a, rows + threadIdx.x * kExpRow);
  __syncthreads();
  rows_out(rows, s0, n, polys, 0, false);
}
template <int ETA>
__global__ void __launch_bounds__(kExpThreads) derive_leqeta_kernel(const uint8_t* __restrict__ seeds, size_t seed_stride,
                                                                    const uint16_t* __restrict__ nonces, size_t n,
                                                                    uint32_t* __restrict__ polys) {
  extern __shared__ __align__(16) uint32_t rows[];
  const size_t s0 = (size_t)blockIdx.x * blockDim.x, s = s0 + threadIdx.x, sc = s < n ? s : n - 1;
  uint64_t a[25];
  absorb_seed(a, seeds + sc * seed_stride, 8);
  a[8] = (uint64_t)nonces[sc] | (0x1full << 16);
  a[16] = 0x8000000000000000ull;
  leqeta_stream<ETA>(a, rows + threadIdx.x * kExpRow);
  __syncthreads();
  rows_out(rows, s0, n, polys, Q + ETA, true);  // p[i] = Q + eta - t (sample.go:158,171)
}
template <class P>
__global__ void __launch_bounds__(128) derive_legamma1_kernel(const uint8_t* __restrict__ seeds, size_t seed_stride,
                                                              const uint16_t* __restrict__ nonces, size_t n,
                                                              uint32_t* __restrict__ polys) {
  const size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  uint64_t a[25];
  absorb_seed(a, seeds + s * seed_stride, 8);
  a[8] = (uint64_t)nonces[s] | (0x1full << 16);
  a[16] = 0x8000000000000000ull;
  legamma1_poly<P>(a, polys + s * N);
}
template <class P>
__global__ void __launch_bounds__(64) derive_ball_kernel(const uint8_t* __restrict__ seeds, size_t seed_stride, size_t n,
                                                         uint32_t* __restrict__ polys) {
  const size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  constexpr int CTW = P::CTILDE / 8;
  uint64_t a[25], ct[CTW], nz[4], ng[4];
  absorb_seed(a, seeds + s * seed_stride, CTW);
#pragma unroll
  for (int i = 0; i < CTW; i++) ct[i] = a[i];
  sample_in_ball<P>(ct, a, nz, ng);
  uint32_t* dst = polys + s * N;
#pragma unroll 1
  for (int q = 0; q < 4; q++)
    for (int b = 0; b < 64; b++) dst[64 * q + b] = ((nz[q] >> b) & 1) ? (((ng[q] >> b) & 1) ? Q - 1 : 1u) : 0u;
}

}  // namespace mldsa
}  // namespace cb200

using namespace cb200;

namespace {

struct ModeSizes {
  size_t pk, sk, sig;
};
bool mode_sizes(int mode, ModeSizes* m) {
  switch (mode) {
    case 44: *m = {1312, 2560, 2420}; return true;
    case 65: *m = {1952, 4032, 3309}; return true;
    case 87: *m = {2592, 4896, 4627}; return true;
    case 2: *m = {1312, 2528, 2420}; return true;  // round-3 Dilithium2/3/5 (sign/dilithium/mode*/internal)
    case 3: *m = {1952, 4000, 3293}; return true;
    case 5: *m = {2592, 4864, 4595}; return true;
  }
  return false;
}

template <class... A>
int dispatch_sign(int mode, A... a) {
  switch (mode) {
    case 44: return mldsa::sign_device<mldsa::Params<44>>(a...);
    case 65: return mldsa::sign_device<mldsa::Params<65>>(a...);
    case 87: return mldsa::sign_device<mldsa::Params<87>>(a...);
    case 2: return mldsa::sign_device<mldsa::Params<2>>(a...);
    case 3: return mldsa::sign_device<mldsa::Params<3>>(a...);
    default: return mldsa::sign_device<mldsa::Params<5>>(a...);
  }
}
template <class... A>
int dispatch_verify(int mode, A... a) {
  switch (mode) {
    case 44: return mldsa::verify_device<mldsa::Params<44>>(a...);
    case 65: return mldsa::verify_device<mldsa::Params<65>>(a...);
    case 87: return mldsa::verify_device<mldsa::Params<87>>(a...);
    case 2: return mldsa::verify_device<mldsa::Params<2>>(a...);
    case 3: return mldsa::verify_device<mldsa::Params<3>>(a...);
    default: return mldsa::verify_device<mldsa::Params<5>>(a...);
  }
}
template <class... A>
int dispatch_keygen(int mode, A... a) {
  switch (mode) {
    case 44: return mldsa::keygen_device<mldsa::Params<44>>(a...);
    case 65: return mldsa::keygen_device<mldsa::Params<65>>(a...);
    case 87: return mldsa::keygen_device<mldsa::Params<87>>(a...);
    case 2: return mldsa::keygen_device<mldsa::Params<2>>(a...);
    case 3: return mldsa::keygen_device<mldsa::Params<3>>(a...);
    default: return mldsa::keygen_device<mldsa::Params<5>>(a...);
  }
}

}  // namespace

extern "C" {

size_t cb200_mldsa_public_key_size(int mode) {
  ModeSizes m;
  return mode_sizes(mode, &m) ? m.pk : 0;
}
size_t cb200_mldsa_private_key_size(int mode) {
  ModeSizes m;
  return mode_sizes(mode, &m) ? m.sk : 0;
}
size_t cb200_mldsa_signature_size(int mode) {
  ModeSizes m;
  return mode_sizes(mode, &m) ? m.sig : 0;
}

int cb200_mldsa_sign(int mode, const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                     const uint8_t* context, size_t ctxlen, const uint8_t* rnd, uint8_t* sig, uint8_t* status, size_t n,
                     int flags, uint64_t* attempts) {
  int rc = require_ready();
  if (rc) return rc;
  ModeSizes ms;
  if (!mode_sizes(mode, &ms)) {
    set_error("cb200_mldsa_sign: mode must be 44, 65, 87 (ML-DSA) or 2, 3, 5 (round-3 Dilithium), got %d", mode);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  if (mode < 10 && ctxlen) {  // sign.ErrContextNotSupported (sign/dilithium/mode3/dilithium.go:227-229)
    set_error("cb200_mldsa_sign: round-3 Dilithium takes no context string");
    return CB200_ERR_ARG;
  }
  if (!sk || !msgs || !msg_off || !sig || ctxlen > 255 || (ctxlen && !context) || (sk_stride != 0 && sk_stride < ms.sk)) {
    set_error("cb200_mldsa_sign: bad argument");  // len(ctx) > 255 is sign.ErrContextTooLong in the Go shim
    return CB200_ERR_ARG;
  }
  const int internal = flags & CB200_SIGN_INTERNAL;
  Batch b{"cb200_mldsa_sign", n, sig, 0, 0,
          {{sk, ms.sk, sk_stride, kIn}, {sig, ms.sig, ms.sig, kOut}, {status, 1, 1, kStatus}, {rnd, 32, 32, kIn}},
          {{!aligned({sk, msg_off}, {sk_stride}, 16), "%s: device sk and sk_stride must be 16-byte aligned"},
           // the attempt bid of the finalize step packs (attempt << 24 | slot)
           {n >= (1u << 24), "%s: a device-pointer batch is limited to 2^24 - 1 signatures per call (got %zu)"}},
          msgs, msg_off, context, ctxlen};
  // host pointers: one contiguous range of the batch per GPU; on each GPU chunks of 2^16 signatures go through the three
  // staging slots.  The rejection loop of a chunk keeps the host busy (one counter read per round), so the input of
  // chunk i+1 is put in flight before chunk i starts and the signatures of chunk i travel back while chunk i+1 runs.
  std::atomic<uint64_t> all_attempts{0};
  std::atomic<size_t> all_bad{0};
  b.host = [&]() -> int {
  int rc = for_each_shard(n, 1u << 12, [&](size_t sh_first, size_t sh_n) -> int {
  Dev& c = ctx();
  int rc = 0;
  constexpr size_t kChunk = 1u << 16;
  const size_t nchunks = (sh_n + kChunk - 1) / kChunk, cmax = sh_n < kChunk ? sh_n : kChunk;
  size_t max_msg = 0;
  for (size_t first = sh_first; first < sh_first + sh_n; first += kChunk) {
    const size_t cnt = sh_first + sh_n - first < kChunk ? sh_first + sh_n - first : kChunk;
    max_msg = std::max<size_t>(max_msg, (size_t)(msg_off[first + cnt] - msg_off[first]));
  }
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t oSk = take((sk_stride ? cmax : 1) * ms.sk), oMsg = take(max_msg + 8), oOff = take((cmax + 1) * 8),
               oRnd = take(cmax * 32), oSig = take(cmax * ms.sig), oSt = take(cmax), oCtx = take(256);
  const int nslots = nchunks < 3 ? (int)nchunks : 3;
  for (int sl = 0; sl < nslots; sl++) {
    rc = ensure_scratch(sl, off);
    if (rc) return rc;
  }
  void* pin = nullptr;
  rc = ensure_pinned(sh_n + 64, &pin);
  if (rc) return rc;
  uint8_t* hs = (uint8_t*)pin;
  volatile uint32_t* h_count = (volatile uint32_t*)((char*)pin + ((sh_n + 15) & ~(size_t)15));
  std::vector<std::vector<uint64_t>> rebased(nchunks);  // message offsets relative to the chunk; alive until the final sync
  auto issue_h2d = [&](size_t ci) -> int {
    const size_t first = sh_first + ci * kChunk, cnt = sh_first + sh_n - first < kChunk ? sh_first + sh_n - first : kChunk;
    const int sl = (int)(ci % 3);
    cudaStream_t st = c.pipe[sl];
    char* d = (char*)c.scratch[sl];
    if (sk_stride == 0)
      CB200_CUDA(cudaMemcpyAsync(d + oSk, sk, ms.sk, cudaMemcpyHostToDevice, st));
    else if (sk_stride == ms.sk)
      CB200_CUDA(cudaMemcpyAsync(d + oSk, sk + first * ms.sk, cnt * ms.sk, cudaMemcpyHostToDevice, st));
    else
      CB200_CUDA(cudaMemcpy2DAsync(d + oSk, ms.sk, sk + first * sk_stride, sk_stride, ms.sk, cnt, cudaMemcpyHostToDevice, st));
    const uint64_t m0 = msg_off[first], mb = msg_off[first + cnt] - m0;
    if (mb) CB200_CUDA(cudaMemcpyAsync(d + oMsg, msgs + m0, mb, cudaMemcpyHostToDevice, st));
    std::vector<uint64_t>& ro = rebased[ci];
    ro.resize(cnt + 1);
    for (size_t i = 0; i <= cnt; i++) ro[i] = msg_off[first + i] - m0;
    CB200_CUDA(cudaMemcpyAsync(d + oOff, ro.data(), (cnt + 1) * 8, cudaMemcpyHostToDevice, st));
    if (rnd) CB200_CUDA(cudaMemcpyAsync(d + oRnd, rnd + 32 * first, cnt * 32, cudaMemcpyHostToDevice, st));
    if (ctxlen) CB200_CUDA(cudaMemcpyAsync(d + oCtx, context, ctxlen, cudaMemcpyHostToDevice, st));
    return 0;
  };
  uint64_t total_attempts = 0;
  rc = issue_h2d(0);
  for (size_t ci = 0; ci < nchunks && rc == 0; ci++) {
    const size_t first = sh_first + ci * kChunk, cnt = sh_first + sh_n - first < kChunk ? sh_first + sh_n - first : kChunk;
    const int sl = (int)(ci % 3);
    cudaStream_t st = c.pipe[sl];
    char* d = (char*)c.scratch[sl];
    if (ci + 1 < nchunks) {
      rc = issue_h2d(ci + 1);
      if (rc) break;
    }
    uint64_t att = 0;
    rc = dispatch_sign(mode, (const uint8_t*)d + oSk, sk_stride ? ms.sk : (size_t)0, (const uint8_t*)d + oMsg,
                       (const uint64_t*)(d + oOff), ctxlen ? (const uint8_t*)d + oCtx : (const uint8_t*)nullptr, (int)ctxlen,
                       rnd ? (const uint8_t*)d + oRnd : (const uint8_t*)nullptr, (uint8_t*)d + oSig, (uint8_t*)d + oSt, cnt,
                       internal, st, sl, attempts ? &att : (uint64_t*)nullptr, h_count);
    if (rc) break;
    total_attempts += att;
    CB200_CUDA(cudaMemcpyAsync(sig + first * ms.sig, d + oSig, cnt * ms.sig, cudaMemcpyDeviceToHost, st));
    CB200_CUDA(cudaMemcpyAsync(hs + (first - sh_first), d + oSt, cnt, cudaMemcpyDeviceToHost, st));
  }
  for (int sl = 0; sl < 3; sl++) CB200_CUDA(cudaStreamSynchronize(c.pipe[sl]));
  if (rc) return rc;
  all_attempts += total_attempts;
  size_t nbad = 0;
  for (size_t i = 0; i < sh_n; i++) nbad += hs[i] != 0;
  all_bad += nbad;
  if (status) memcpy(status + sh_first, hs, sh_n);
  return 0;
  });
  if (rc) return rc;
  if (attempts) *attempts = all_attempts.load();
  return 0;
  };
  rc = run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return dispatch_sign(mode, r[0].p, r[0].stride, r.msgs, r.msg_off, r.ctx, (int)ctxlen, r[3].p, r[1].p, r[2].p, cnt,
                         internal, st, slot, attempts, (volatile uint32_t*)wset(slot).pin);
  });
  if (rc) return rc;
  return sign_attempts_result("cb200_mldsa_sign", all_bad.load(), n);
}

int cb200_mldsa_verify(int mode, const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                       const uint8_t* context, size_t ctxlen, const uint8_t* sig, uint8_t* ok, size_t n, int flags) {
  int rc = require_ready();
  if (rc) return rc;
  ModeSizes ms;
  if (!mode_sizes(mode, &ms)) {
    set_error("cb200_mldsa_verify: mode must be 44, 65, 87 (ML-DSA) or 2, 3, 5 (round-3 Dilithium), got %d", mode);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  if (mode < 10 && ctxlen) {
    set_error("cb200_mldsa_verify: round-3 Dilithium takes no context string");
    return CB200_ERR_ARG;
  }
  if (!pk || !msgs || !msg_off || !sig || !ok || ctxlen > 255 || (ctxlen && !context) ||
      (pk_stride != 0 && pk_stride < ms.pk)) {
    set_error("cb200_mldsa_verify: bad argument");
    return CB200_ERR_ARG;
  }
  const int internal = flags & CB200_SIGN_INTERNAL;
  // host pointers: one contiguous range per GPU, each in chunks of 2^15 signatures on the first staging slot
  Batch b{"cb200_mldsa_verify", n, ok, 1u << 15, 1u << 12,
          {{pk, ms.pk, pk_stride, kIn}, {sig, ms.sig, ms.sig, kIn}, {ok, 1, 1, kOut}},
          {{!aligned({pk, msg_off}, {pk_stride}, 16), "%s: device pk and pk_stride must be 16-byte aligned"}},
          msgs, msg_off, context, ctxlen};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return dispatch_verify(mode, (const uint8_t*)r[0].p, r[0].stride, (const uint8_t*)r.msgs, r.msg_off, r.ctx, (int)ctxlen,
                           (const uint8_t*)r[1].p, r[2].p, cnt, internal, st, slot);
  });
}

int cb200_mldsa_keygen(int mode, const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  ModeSizes ms;
  if (!mode_sizes(mode, &ms)) {
    set_error("cb200_mldsa_keygen: mode must be 44, 65, 87 (ML-DSA) or 2, 3, 5 (round-3 Dilithium), got %d", mode);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  if (!seeds || !pk || !sk) {
    set_error("cb200_mldsa_keygen: null pointer");
    return CB200_ERR_ARG;
  }
  Batch b{"cb200_mldsa_keygen", n, pk, 1u << 14, 1u << 12, {{seeds, 32, 32, kIn}, {pk, ms.pk, ms.pk, kOut}, {sk, ms.sk, ms.sk, kOut}},
          {{!aligned({seeds, pk, sk}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    return dispatch_keygen(mode, (const uint8_t*)r[0].p, r[1].p, r[2].p, cnt, st, slot);
  });
}

/* ML-DSA-65 entry points under their original names */
int cb200_mldsa65_sign(const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                       const uint8_t* context, size_t ctxlen, const uint8_t* rnd, uint8_t* sig, uint8_t* status, size_t n,
                       int flags, uint64_t* attempts) {
  return cb200_mldsa_sign(65, sk, sk_stride, msgs, msg_off, context, ctxlen, rnd, sig, status, n, flags, attempts);
}
int cb200_mldsa65_verify(const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
                         const uint8_t* context, size_t ctxlen, const uint8_t* sig, uint8_t* ok, size_t n, int flags) {
  return cb200_mldsa_verify(65, pk, pk_stride, msgs, msg_off, context, ctxlen, sig, ok, n, flags);
}
int cb200_mldsa65_keygen(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  return cb200_mldsa_keygen(65, seeds, pk, sk, n);
}
size_t cb200_mldsa65_signature_size(void) { return 3309; }
size_t cb200_mldsa65_public_key_size(void) { return 1952; }
size_t cb200_mldsa65_private_key_size(void) { return 4032; }

/* ---- the samplers as entry points of their own (sign/mldsa/mldsa{44,65,87}/internal/sample.go) ---- */
static int sampler_entry(const char* fn, int kind, int mode, uint32_t* polys, const uint8_t* seeds, size_t seed_stride,
                         size_t seed_len, const uint16_t* nonces, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (mode != 44 && mode != 65 && mode != 87) {
    set_error("%s: mode must be 44, 65 or 87, got %d", fn, mode);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  if (!polys || !seeds || (kind != 3 && !nonces) || (seed_stride != 0 && seed_stride < seed_len)) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  auto launch = [&](const uint8_t* sd, size_t stride, const uint16_t* nn, uint32_t* out, size_t cnt, cudaStream_t st) -> int {
    using namespace mldsa;
    KernelScope ks(KID_SAMPLER, st);
    const unsigned g64 = (unsigned)((cnt + kExpThreads - 1) / kExpThreads), g128 = (unsigned)((cnt + 127) / 128);
    constexpr int smem = kExpThreads * kExpRow * 4;
    if (kind == 0) {
      if (int arc = ensure_smem_attr((const void*)derive_uniform_kernel, smem)) return arc;
      derive_uniform_kernel<<<g64, kExpThreads, smem, st>>>(sd, stride, nn, cnt, out);
    } else if (kind == 1) {
      if (mode == 65) {
        if (int arc = ensure_smem_attr((const void*)derive_leqeta_kernel<4>, smem)) return arc;
        derive_leqeta_kernel<4><<<g64, kExpThreads, smem, st>>>(sd, stride, nn, cnt, out);
      } else {
        if (int arc = ensure_smem_attr((const void*)derive_leqeta_kernel<2>, smem)) return arc;
        derive_leqeta_kernel<2><<<g64, kExpThreads, smem, st>>>(sd, stride, nn, cnt, out);
      }
    } else if (kind == 2) {
      if (mode == 44)
        derive_legamma1_kernel<Params<44>><<<g128, 128, 0, st>>>(sd, stride, nn, cnt, out);
      else
        derive_legamma1_kernel<Params<65>><<<g128, 128, 0, st>>>(sd, stride, nn, cnt, out);  // 87: the same gamma1
    } else {
      if (mode == 44)
        derive_ball_kernel<Params<44>><<<g64, 64, 0, st>>>(sd, stride, cnt, out);
      else if (mode == 65)
        derive_ball_kernel<Params<65>><<<g64, 64, 0, st>>>(sd, stride, cnt, out);
      else
        derive_ball_kernel<Params<87>><<<g64, 64, 0, st>>>(sd, stride, cnt, out);
    }
    CB200_CUDA(cudaGetLastError());
    return 0;
  };
  Batch b{fn, n, polys, 1u << 15, 1u << 13,
          {{seeds, seed_len, seed_stride, kIn}, {polys, 1024, 1024, kOut}, {nonces, 2, 2, kIn}},
          {{!aligned({polys}, {}, 16) || !aligned({nonces}, {}, 2), "%s: device polynomials must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch(r[0].p, r[0].stride, (const uint16_t*)r[2].p, (uint32_t*)r[1].p, cnt, st);
  });
}
int cb200_dil_derive_uniform(uint32_t* polys, const uint8_t* seeds, size_t seed_stride, const uint16_t* nonces, size_t n) {
  return sampler_entry("cb200_dil_derive_uniform", 0, 65, polys, seeds, seed_stride, 32, nonces, n);
}
int cb200_dil_derive_leq_eta(int mode, uint32_t* polys, const uint8_t* seeds, size_t seed_stride, const uint16_t* nonces,
                             size_t n) {
  return sampler_entry("cb200_dil_derive_leq_eta", 1, mode, polys, seeds, seed_stride, 64, nonces, n);
}
int cb200_dil_derive_le_gamma1(int mode, uint32_t* polys, const uint8_t* seeds, size_t seed_stride, const uint16_t* nonces,
                               size_t n) {
  return sampler_entry("cb200_dil_derive_le_gamma1", 2, mode, polys, seeds, seed_stride, 64, nonces, n);
}
int cb200_dil_derive_ball(int mode, uint32_t* polys, const uint8_t* seeds, size_t seed_stride, size_t n) {
  const size_t len = mode == 44 ? 32 : mode == 65 ? 48 : 64;
  return sampler_entry("cb200_dil_derive_ball", 3, mode, polys, seeds, seed_stride, len, nullptr, n);
}

}  // extern "C"

// device-level entry points for the composite signatures of eddsa.cu (mldsa_internal.h); defined after the C entry
// points so that the flows are instantiated in the same order as before
namespace cb200 {
namespace mldsa {

int dev_keygen(int mode, const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n, cudaStream_t st, int slot) {
  return dispatch_keygen(mode, seeds, pk, sk, n, st, slot);
}
int dev_sign(int mode, const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off, uint8_t* sig,
             uint8_t* status, size_t n, cudaStream_t st, int slot, volatile uint32_t* h_count) {
  return dispatch_sign(mode, sk, sk_stride, msgs, msg_off, (const uint8_t*)nullptr, 0, (const uint8_t*)nullptr, sig, status, n,
                       0, st, slot, (uint64_t*)nullptr, h_count);
}
int dev_verify(int mode, const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
               const uint8_t* sig, uint8_t* ok, size_t n, cudaStream_t st, int slot) {
  return dispatch_verify(mode, pk, pk_stride, msgs, msg_off, (const uint8_t*)nullptr, 0, sig, ok, n, 0, st, slot);
}

}  // namespace mldsa
}  // namespace cb200
