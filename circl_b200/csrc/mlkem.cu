// circl_b200/csrc/mlkem.cu -- batched ML-KEM-768 / ML-KEM-1024 Encapsulate on sm_90a.
//
// Replaces, per operation and bit-exactly:
//   scheme.UnmarshalBinaryPublicKey   kem/mlkem/mlkem768/kyber.go:390-396 -> :247-263
//     cpapke.UnpackMLKEM              pke/kyber/kyber768/internal/cpapke.go:45-63 (modulus check, aT.Derive)
//     Mat.Derive / DeriveUniform      internal/mat.go:13-29, common/sample.go:192-236 (SHAKE128 rejection)
//   (*PublicKey).EncapsulateTo        kem/mlkem/mlkem768/kyber.go:103-137  (G = SHA3-512(m || H(ek)))
//     (*PublicKey).EncryptTo          internal/cpapke.go:137-181
//     DeriveNoise2                    common/sample.go:67-95 (SHAKE256 PRF + CBD_2)
//     CompressTo                      common/poly.go:248-328
//
// Pipeline (all intermediates stay on the device; sub-batches of kSub ops alternate between two streams, and A^T is
// the only intermediate of a sub-batch in memory -- 36 MiB at 8192 ops, K = 3):
//   1. hash_kernel    one thread per op/key: h = SHA3-256(ek), (K', r) = SHA3-512(m || h)
//   2. sample_kernel  one thread per Keccak stream: K*K SHAKE128 matrix streams per key, staged a block at a time
//                     and written by each warp itself (uniform_block)
//   3. encrypt_dp_kernel one octet (8 lanes) per op: the 2K+1 SHAKE256 noise streams (lane p: nonces p, p + 8),
//                     NTT(r), A^T o r, t o r, InvNTT, +e, compress
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "../../include/circl_b200.h"
#include "context.h"
#include "flow_internal.h"
#include "mlkem_internal.h"
#include "keccak.cuh"
#include "kyber.cuh"

namespace cb200 {
namespace mlkem {

using kyber::N;
using kyber::Q;

template <int K>
struct Params {
  static constexpr int k = K;
  static constexpr int du = (K == 4) ? 11 : 10;
  static constexpr int dv = (K == 4) ? 5 : 4;
  static constexpr int ek_bytes = 384 * K + 32;
  static constexpr int ct_bytes = 32 * (du * K + dv);
  static constexpr int eta1 = (K == 2) ? 3 : 2;  // pke/kyber/kyber{512,768,1024}/internal/params.go
  static constexpr int n_noise = 2 * K + 1;      // r[0..K) (eta1), e1[0..K), e2 (eta2 = 2)
};

// ------------------------------------------------------------------ 1. hashes
// h = SHA3-256(ek) (kyber.go:258-260).  One thread per key; ek is 8-byte aligned.
template <int K>
__device__ __forceinline__ void sha3_256_ek(const uint8_t* ek, uint64_t (&h)[4]) {
  constexpr int words = Params<K>::ek_bytes / 8;  // 148 / 196
  constexpr int full = words / 17, rem = words % 17;
  uint64_t a[25];
  keccak::zero(a);
  const uint8_t* p = ek;
#pragma unroll 1
  for (int b = 0; b < full; b++) {
#pragma unroll
    for (int w = 0; w < 17; w++) a[w] ^= keccak::ld64(p + 8 * w);
    keccak::f1600(a);
    p += 136;
  }
#pragma unroll
  for (int w = 0; w < rem; w++) a[w] ^= keccak::ld64(p + 8 * w);
  a[rem] ^= 0x06;
  a[16] ^= 0x8000000000000000ull;
  keccak::f1600(a);
#pragma unroll
  for (int i = 0; i < 4; i++) h[i] = a[i];
}

template <int K>
__global__ void __launch_bounds__(128) hash_ek_kernel(const uint8_t* __restrict__ ek, size_t ek_stride, size_t nkeys,
                                                      uint64_t* __restrict__ hout) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nkeys) return;
  uint64_t h[4];
  sha3_256_ek<K>(ek + i * ek_stride, h);
#pragma unroll
  for (int j = 0; j < 4; j++) hout[4 * i + j] = h[j];
}

// (K', r) = SHA3-512(m || h)  (kyber.go:126-131); ss = K' (kyber.go:136)
__global__ void __launch_bounds__(128) g_kernel(const uint8_t* __restrict__ m, const uint8_t* __restrict__ h,
                                                size_t h_stride, size_t n, uint8_t* __restrict__ ss,
                                                uint64_t* __restrict__ r_out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t a[25];
  keccak::zero(a);
  const uint64_t* hp = reinterpret_cast<const uint64_t*>(h + i * h_stride);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    a[j] = reinterpret_cast<const uint64_t*>(m + 32 * i)[j];
    a[4 + j] = hp[j];
  }
  a[8] = 0x8000000000000006ull;  // rate 72: pad bytes 64 (0x06) and 71 (0x80) share lane 8
  keccak::f1600(a);
  uint64_t* so = reinterpret_cast<uint64_t*>(ss + 32 * i);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    so[j] = a[j];
    r_out[4 * i + j] = a[4 + j];
  }
}

// ------------------------------------------------------------------ 2. samplers
// 12-bit rejection sampling of one 168-byte SHAKE128 block (sample.go:203-233): 112 candidates, field f at bit 12 f
// of the block (d1 = low, d2 = high 12 bits of each 3-byte group, in that order).  `wp` is the 32-bit shared-memory
// address of the next free int16 of this thread's staging: every candidate is stored there (clamped to `end`, the
// entry of coefficient 256, once 256 are in) and only the advance is predicated -- per candidate a shift/mask pair, a
// min, a compare, one STS and one predicated add, all on 32-bit registers.  Returns the new address (>= end when full).
template <bool CHECKED>
__device__ __forceinline__ uint32_t reject_block(const uint64_t (&a)[25], uint32_t wp, uint32_t end) {
#pragma unroll
  for (int f = 0; f < 112; f++) {
    const int bit = 12 * f, wi = bit >> 5, sh = bit & 31;
    const uint32_t lo = (uint32_t)(a[wi >> 1] >> (32 * (wi & 1)));
    uint32_t d;
    if (sh + 12 <= 32) {
      d = (lo >> sh) & 0xfff;
    } else {
      const uint32_t hi = (uint32_t)(a[(wi + 1) >> 1] >> (32 * ((wi + 1) & 1)));
      d = __funnelshift_r(lo, hi, sh) & 0xfff;
    }
    // the first two blocks hold 224 candidates: they cannot run past coefficient 256, so only later blocks clamp
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(CHECKED ? min(wp, end) : wp), "h"((uint16_t)d) : "memory");
    wp += (d < (uint32_t)Q) ? 2u : 0u;
  }
  return wp;
}

// CBD_2 of 128 bytes (sample.go:80-93), written as 256 packed int16 (kyber::cbd2_words: eight coefficients per word)
__device__ __forceinline__ void cbd2_store(const uint64_t (&a)[25], int16_t* __restrict__ dst) {
  uint4* out = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int i = 0; i < 16; i++) {
    uint32_t lo[4], hi[4];
    kyber::cbd2_words((uint32_t)a[i], lo);
    kyber::cbd2_words((uint32_t)(a[i] >> 32), hi);
    out[2 * i] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    out[2 * i + 1] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  }
}

// sub-batch size.  A sub-batch leaves only A^T in memory (4.5 KiB / op for K=3, 8 KiB for K=4), so two 4096-op
// sub-batches in flight fit the 50 MB L2 and two of 8192 do not; 8192 still measured faster (ML-KEM-768, 2^20 per-op
// keys, H100 80GB HBM3 SXM at 700 W: 19.9 ms per step against 20.9 at 4096), as it halves the launches and the tail
// waves, sample_fix_kernel's most of all (1.8 against 3.5 ms per step).  With the noise still in memory (8 KiB / op)
// 4096 had been the faster (H100 SXM at 400 W: 24.7 ms per step at 4096, 25.5 at 8192, 30.0 at 2048).  Per sub-batch
// of 8192 ops (K = 3) sample_kernel runs 576 CTAs on 792 resident slots (6 per SM) and encrypt_dp_kernel 1024 on 924.
constexpr size_t kSub = 8192;
// The matrix sampler's staging (uniform_block): per thread 15 chunks of 8 int16 -- up to 7 coefficients carried from
// the last block, the 112 candidates of this one and the clamp slot -- 240 B, so 30,720 B per 128-thread CTA and
// registers, not shared memory, set its residency: 80 per thread, 6 CTAs per SM (it had been 3, by a 66,048-byte row
// per CTA; at 72 registers ptxas spills).
constexpr int kStageChunks = 15;
constexpr int kSampleThreads = 128;
constexpr int kSampleMinBlocks = 6;
constexpr int kSampleSmem = kSampleThreads * kStageChunks * 16;

// CBD_3 of 192 bytes (sample.go:31-62): 6-byte windows, 8 coefficients each; w = 24 squeezed words
__device__ __forceinline__ void cbd3_store(const uint64_t (&w)[24], int16_t* __restrict__ dst) {
  uint4* out = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int g = 0; g < 8; g++) {  // 3 words -> 4 windows -> 32 coefficients
    const uint64_t w0 = w[3 * g], w1 = w[3 * g + 1], w2 = w[3 * g + 2];
    uint64_t t[4];
    t[0] = w0;
    t[1] = (w0 >> 48) | (w1 << 16);
    t[2] = (w1 >> 32) | (w2 << 32);
    t[3] = w2 >> 16;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const uint64_t x = t[q];
      uint64_t d = x & 0x249249249249ull;
      d += (x >> 1) & 0x249249249249ull;
      d += (x >> 2) & 0x249249249249ull;
      uint32_t c[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int c0 = (int)((d >> (12 * j)) & 7) - (int)((d >> (12 * j + 3)) & 7);
        const int c1 = (int)((d >> (12 * j + 6)) & 7) - (int)((d >> (12 * j + 9)) & 7);
        c[j] = ((uint32_t)c0 & 0xffffu) | ((uint32_t)c1 << 16);
      }
      out[4 * g + q] = make_uint4(c[0], c[1], c[2], c[3]);
    }
  }
}

// One SHAKE128 block of the 32 streams of a warp (sample.go:203-233), warp-collective.  `wst` is the warp's staging
// (32 x kStageChunks chunks of 16 B, lane l's at l * kStageChunks); this lane's polynomial is the 32 chunks from
// out[poly]; `cnt` is the number of coefficients it holds so far.  Returns the new count, clamped to 256 (CHECKED; the
// first two blocks hold at most 224 candidates and need no clamp).  Staging entry e stands for coefficient base + e,
// base = cnt rounded down to a multiple of 8, so the entries [0, cnt - base) are the ones carried over from the last
// block and every chunk of the staging is a 16-byte chunk of the polynomial:
//   1. permute; parse the 112 candidates into the thread's staging from entry cnt - base on (reject_block);
//   2. the warp writes the chunks [base / 8, ceil(cnt' / 8)) of every stream (at most 15), two streams per pass --
//      lanes 0-15 stream 2q, lanes 16-31 stream 2q + 1 -- with one 16-byte load and store per lane: 16 passes of one
//      shuffle (the stream's first chunk and chunk count, packed), unpacking, a compare, LDS.128 and STG.128;
//   3. the thread moves its last, partial chunk to the front of its staging for the next block.
// A partial chunk is written with whatever follows the last coefficient in the staging and rewritten whole by the
// next block's pass (or, for a stream sample_kernel hands off, from position cnt' on by sample_fix_kernel).
// Threads past the end of the batch (`live` false) take part and write nothing.  poly must stay below 2^23 - 1, so
// that (32 poly + 32) << 4 fits the 32-bit job word.
template <bool CHECKED>
__device__ __forceinline__ uint32_t uniform_block(uint64_t (&a)[25], uint4* wst, int lane, uint4* __restrict__ out,
                                                  uint32_t poly, uint32_t cnt, bool live) {
  keccak::f1600(a);
  uint4* own = wst + lane * kStageChunks;
  const uint32_t base = cnt & ~7u, s0 = smem_u32(own), end = s0 + 2 * (N - base);
  const uint32_t wp = reject_block<CHECKED>(a, s0 + 2 * (cnt - base), end);
  cnt = base + ((min(wp, end) - s0) >> 1);
  // first chunk to write << 4 | chunk count (<= 15)
  const uint32_t job = live ? ((32 * poly + base / 8) << 4) | ((cnt - base + 7) >> 3) : 0;
  __syncwarp();
  const int half = lane >> 4, c = lane & 15;
  const uint4* rd = wst + half * kStageChunks + c;
#pragma unroll 4
  for (int q = 0; q < 16; q++) {
    const uint32_t jp = __shfl_sync(0xffffffffu, job, 2 * q + half);
    if (c < (int)(jp & 15)) out[(jp >> 4) + c] = rd[2 * q * kStageChunks];
  }
  __syncwarp();
  if (cnt < N) own[0] = own[(cnt - base) >> 3];
  return cnt;
}

// One SHAKE128 stream of DeriveUniform (sample.go:192-236) per lane of a warp: `a` holds the absorbed, padded first
// block; the 256 accepted coefficients go to out[poly] (uniform_block).  The warp squeezes blocks until all its streams
// are full.
__device__ __forceinline__ void uniform_stream(uint64_t (&a)[25], uint4* wst, int lane, uint4* out, uint32_t poly,
                                               bool live) {
  uint32_t cnt = 0;
#pragma unroll 1
  for (int b = 0; b < 2; b++) cnt = uniform_block<false>(a, wst, lane, out, poly, cnt, live);
  do {
    cnt = uniform_block<true>(a, wst, lane, out, poly, cnt, live);
  } while (__any_sync(0xffffffffu, cnt < N));
}
// The same with exactly three blocks -- what 99 % of the streams need (SURVEY.md 8(a)) -- so that all lanes of a warp
// finish together; returns the number of coefficients accepted, the first that many of which are in the polynomial.
// A stream that is short of 256 is handed, with its sponge state, to sample_fix_kernel: a warp no longer squeezes a
// fourth block for all 32 lanes because one of them needs it (27 % of the warps did).
__device__ __forceinline__ uint32_t uniform_stream3(uint64_t (&a)[25], uint4* wst, int lane, uint4* out, uint32_t poly,
                                                    bool live) {
  uint32_t cnt = 0;
#pragma unroll 1
  for (int b = 0; b < 2; b++) cnt = uniform_block<false>(a, wst, lane, out, poly, cnt, live);
  return uniform_block<true>(a, wst, lane, out, poly, cnt, live);
}
struct Pending {  // one unfinished SHAKE128 stream
  uint32_t stream, count;
  uint64_t a[25];
};
struct FixList {  // in front of the Pending array (64 bytes)
  unsigned int n, done, pad[14];
};

// One SHAKE256 PRF stream of DeriveNoise (sample.go:31-95): `a` holds the absorbed, padded block seed || nonce
template <int ETA>
__device__ __forceinline__ void noise_stream(uint64_t (&a)[25], int16_t* __restrict__ dst) {
  keccak::f1600(a);
  if constexpr (ETA == 3) {
    uint64_t w[24];
#pragma unroll
    for (int q = 0; q < 17; q++) w[q] = a[q];
    keccak::f1600(a);
#pragma unroll
    for (int q = 0; q < 7; q++) w[17 + q] = a[q];
    cbd3_store(w, dst);
  } else {
    cbd2_store(a, dst);
  }
}

// One thread per matrix stream, s = (i*K + j) * nkeys + key -> A^T[key][i][j] = XOF(rho, i, j).  (The noise is made
// by the K-PKE kernels themselves, octet_prf.)
template <int K>
__global__ void __launch_bounds__(kSampleThreads, kSampleMinBlocks) sample_kernel(const uint8_t* __restrict__ rho0, size_t ek_stride,
                                                                size_t nkeys, int16_t* __restrict__ A, int transpose,
                                                                FixList* __restrict__ fix) {
  // rho0 + key*ek_stride is rho of that key; transpose = 1 derives A^T (encryption), 0 derives A (key
  // generation, mat.go:13-29)
  // Each warp stages its 32 streams a block at a time and writes them to A itself (uniform_block): no CTA barrier.
  extern __shared__ __align__(16) uint4 stage[];
  const int lane = threadIdx.x & 31, wbase = threadIdx.x & ~31;
  const size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = nkeys * K * K;
  if (s - lane >= total) return;  // a warp with no stream of the batch
  uint64_t a[25];
  keccak::zero(a);
  const bool live = s < total;
  const size_t sc = live ? s : total - 1;
  const size_t key = sc % nkeys;
  const int ij = (int)(sc / nkeys), i = ij / K, j = ij % K;
  const uint8_t* rho = rho0 + key * ek_stride;
#pragma unroll
  for (int w = 0; w < 4; w++) a[w] = keccak::ld64(rho + 8 * w);
  // m[i][j] = XOF(rho, x, y) with (x, y) = (i, j) if transpose else (j, i)
  a[4] = (uint64_t)(transpose ? i : j) | ((uint64_t)(transpose ? j : i) << 8) | (0x1full << 16);
  a[20] = 0x8000000000000000ull;                               // rate 168
  const uint32_t got = uniform_stream3(a, stage + wbase * kStageChunks, lane, reinterpret_cast<uint4*>(A),
                                       (uint32_t)(key * K * K + ij), live);
  if (live && got < N) {  // ~1 % of the streams: finished by sample_fix_kernel from this state
    Pending* list = reinterpret_cast<Pending*>(fix + 1);
    Pending& e = list[atomicAdd(&fix->n, 1u)];
    e.stream = (uint32_t)s;
    e.count = got;
#pragma unroll
    for (int w = 0; w < 25; w++) e.a[w] = a[w];
  }
}

// ------------------------------------------------------------------ 3. K-PKE.Encrypt
// Compress_q(x, d) for x in [0, q)  (poly.go:262-328)
template <int D>
__device__ __forceinline__ uint32_t compress1(uint32_t x) {
  const uint32_t v = (x << D) + Q / 2;
  if constexpr (D <= 5)
    return ((v * 315u) >> 20) & ((1u << D) - 1);
  else
    return (__umulhi(v, 20642679u) >> 4) & ((1u << D) - 1);
}

// 32 normalised coefficients (high-half registers, C layout) -> D words of ciphertext
template <int D>
__device__ __forceinline__ void compress_store_C(const int32_t (&r)[32], uint32_t* __restrict__ dst) {
  uint64_t acc = 0;
  int bits = 0, o = 0;
#pragma unroll
  for (int i = 0; i < 32; i++) {
    acc |= (uint64_t)compress1<D>((uint32_t)r[i] >> 16) << bits;
    bits += D;
    if (bits >= 32) {
      dst[o++] = (uint32_t)acc;
      acc >>= 32;
      bits -= 32;
    }
  }
}

// 12-bit unpack of 32 coefficients (48 bytes, 16-byte aligned) into high-half registers
// (poly.go:123-129); returns nonzero if any coefficient is >= q (cpapke.go:45-55).
__device__ __forceinline__ uint32_t unpack12_C(const uint8_t* __restrict__ src, int32_t (&r)[32]) {
  const uint4* p = reinterpret_cast<const uint4*>(src);
  uint32_t w[12];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    uint4 q4 = __ldg(p + i);
    w[4 * i] = q4.x;
    w[4 * i + 1] = q4.y;
    w[4 * i + 2] = q4.z;
    w[4 * i + 3] = q4.w;
  }
  uint32_t bad = 0;
#pragma unroll
  for (int g = 0; g < 4; g++) {  // 3 words -> 8 coefficients
    const uint32_t a = w[3 * g], b = w[3 * g + 1], c = w[3 * g + 2];
    uint32_t t[8];
    t[0] = a & 0xfff;
    t[1] = (a >> 12) & 0xfff;
    t[2] = ((a >> 24) | (b << 8)) & 0xfff;
    t[3] = (b >> 4) & 0xfff;
    t[4] = (b >> 16) & 0xfff;
    t[5] = ((b >> 28) | (c << 4)) & 0xfff;
    t[6] = (c >> 8) & 0xfff;
    t[7] = c >> 20;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      bad |= (t[j] >= (uint32_t)Q);
      r[8 * g + j] = (int32_t)(t[j] << 16);
    }
  }
  return bad;
}


// The streams sample_kernel left short of 256 coefficients: thread per stream, squeeze on from the saved state and
// append to the polynomial in A (2-byte global stores; about 1 % of the streams, one or two dozen coefficients each).
template <int K>
__global__ void __launch_bounds__(64) sample_fix_kernel(FixList* __restrict__ fix, size_t nkeys, int16_t* __restrict__ A) {
  __shared__ uint64_t sq[64][21];
  const Pending* list = reinterpret_cast<const Pending*>(fix + 1);
  const unsigned int total = fix->n;
  for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    uint64_t a[25];
#pragma unroll
    for (int w = 0; w < 25; w++) a[w] = list[i].a[w];
    const size_t sp = list[i].stream;
    int16_t* dst = A + ((sp % nkeys) * K * K + sp / nkeys) * N;
    int cnt = (int)list[i].count;
    uint8_t* blk = reinterpret_cast<uint8_t*>(sq[threadIdx.x]);
    while (cnt < N) {
      keccak::f1600(a);
#pragma unroll
      for (int w = 0; w < 21; w++) sq[threadIdx.x][w] = a[w];
#pragma unroll 1
      for (int f = 0; f < 112 && cnt < N; f++) {  // sample.go:203-233: 12-bit candidates, low half of each 3 bytes first
        const int byte = (3 * f) >> 1;
        uint32_t d = (uint32_t)blk[byte] | ((uint32_t)blk[byte + 1] << 8);
        d = ((f & 1) ? d >> 4 : d) & 0xfff;
        if (d < (uint32_t)Q) dst[cnt++] = (int16_t)d;
      }
    }
  }
  // the last CTA to finish empties the list for the next launch on this lane
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&fix->done, 1u) == gridDim.x - 1) {
      fix->n = 0;
      fix->done = 0;
    }
  }
}

// sample_kernel + sample_fix_kernel on stream `ls`; `lane` picks the unfinished-stream list of the work set
template <int K>
static int launch_sample(int slot, int lane, cudaStream_t ls, const uint8_t* rho0, size_t ek_stride, size_t nkeys,
                         int16_t* A, int transpose) {
  if (nkeys == 0) return 0;
  static_assert(kSub * 16 < (1u << 23) - 1, "uniform_block: polynomial index too large");  // nkeys <= kSub
  if (int arc = ensure_smem_attr((const void*)sample_kernel<K>, kSampleSmem)) return arc;
  const size_t streams = nkeys * K * K;
  void* fix = nullptr;
  if (int frc = ensure_fix(slot, lane, sizeof(FixList) + streams * sizeof(Pending), ls, &fix)) return frc;
  {
    KernelScope ks(KID_MLKEM_SAMPLE, ls);
    sample_kernel<K><<<(unsigned)((streams + kSampleThreads - 1) / kSampleThreads), kSampleThreads, kSampleSmem, ls>>>(
        rho0, ek_stride, nkeys, A, transpose, (FixList*)fix);
  }
  {
    KernelScope ks(KID_MLKEM_SAMPLE_FIX, ls);
    const unsigned grid = (unsigned)std::min<size_t>(64, (streams / 64 + 63) / 64 + 1);  // ~1 % of the streams, 64 per CTA
    sample_fix_kernel<K><<<grid, 64, 0, ls>>>((FixList*)fix, nkeys, A);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------ 3. K-PKE.Encrypt (cpapke.go:137-181), one octet per op
// u = InvNTT(A^T o NTT(r)) + e1, v = InvNTT(t o NTT(r)) + e2 + Decompress(m), ct = Compress(u) || Compress(v).  What leaves
// the kernel is Compress(Normalize(.)), so only residues mod q matter inside it, not the reference's Montgomery
// representatives, and the matrix-vector products are done differently from MulHat:
//
//   * A^T and t-hat are used as they lie in memory: one 32-bit word = one degree-2 block (a0 | a1 << 16), plain
//     residues in [0, 4096);
//   * r-hat is prepared once per op as byte-split operands in shared memory, two words per block:
//       W0 = [b0.lo, z b1.lo, b0.hi, z b1.hi]    W1 = [b1.lo, b0.lo, b1.hi, b0.hi]    (z = +-zeta of the block)
//     (low bytes unsigned, high bytes signed), so that the two outputs of the block over all K columns,
//       p0 = sum a0 b0 + a1 (z b1),   p1 = sum a0 b1 + a1 b0                         (poly.go:63-100 without the R^-1)
//     are 4 IDP.2A (16-bit x 8-bit dot products with accumulate) per column and block, with no unpacking of A at all --
//     against 5 Montgomery products, i.e. ~50 instructions, in the reference's formulation;
//   * one Montgomery reduction per output coefficient then yields p R^-1 mod q, the residue MulHat would have
//     produced; the constant of the inverse transform (ntt.go:187-192: x 1441 = R^2 / 128, Montgomery) is folded into
//     the operands instead -- they carry r-hat R / 128 = 512 r-hat -- which costs a multiplication per coefficient of
//     r-hat once instead of one per coefficient of every output row and doubles as their reduction.
//
// Bounds: |b| < q after the Montgomery multiplication, |z b1| < q, a < 4096 (a < q unless the key is not canonical): a
// 32-bit sum p of 2 K products is below 8 . 4096 . q < 2^27, and |montReduce(p)| <= |p| / 2^16 + q / 2 <= q, which is the
// input bound of the inverse transform's lazy-Barrett schedule (ntt.go:145-150).
constexpr int kOpPad = 16;  // words between the operand areas of two ops: half-warps (two octets) hit disjoint banks
// behind the operands: the lanes' words of e2 (4 each), which encrypt_dp_kernel keeps here until its last row -- in
// registers they would push the K = 3 kernel past the 128 it may use at 7 CTAs per SM
constexpr int kE2Words = 32;
template <int K, int THREADS>
struct EncSmem {
  static constexpr int op_words = K * 128 * 2 + kE2Words + kOpPad;
  static constexpr int words = (THREADS / 8) * op_words + (THREADS / 8) * kyber::kPolyWords + 256;
  static constexpr int bytes = words * 4;
};

__device__ __forceinline__ uint32_t dp2a_lo_uu(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("dp2a.lo.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ int32_t dp2a_hi_us(uint32_t a, uint32_t b, int32_t c) {
  int32_t d;
  asm("dp2a.hi.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
// montReduce(p) of a 32-bit signed p (field.go:4-32) as a plain sign-extended value
__device__ __forceinline__ int32_t mont_red_lo(int32_t p) {
  const int32_t m = (int32_t)((uint32_t)p * (kyber::QINV << 16)) >> 16;
  return (p - m * Q) >> 16;
}
// hi32(a * b) as a wide multiplication (IMAD.WIDE.U32) rather than the IMAD.HI.U32 __umulhi compiles to; the issue rates
// of the two are what scripts/ubench_pipes.cu measures
__device__ __forceinline__ uint32_t umulhi_wide(uint32_t a, uint32_t b) {
  uint32_t hi;
  asm("{ .reg .b64 t; mul.wide.u32 t, %1, %2; mov.b64 {_, %0}, t; }" : "=r"(hi) : "r"(a), "r"(b));
  return hi;
}
// Compress_q(x, d) (poly.go:248-328) from ANY representative x of the residue with |x| < 2^15, low-format register:
// round(x 2^d / q) mod 2^d does not change when a multiple of q is added to x, so x + 10 q in [0, 2^16) is compressed
// directly -- floor((x' 2^d + 1664) / q) as a 32 x 32 -> 64 multiplication by ceil(2^40 / q), exact below 2^28 -- and the
// Normalize of cpapke.go:176-177 needs no instruction of its own.  Checked exhaustively against the reference's two
// constant pairs for every 16-bit x' and d in {4, 5, 10, 11} (tests/test_compress_identity.py).
template <int D>
__device__ __forceinline__ uint32_t compress_any(int32_t x) {
  const uint32_t v = ((uint32_t)(x + 10 * Q) << D) + Q / 2;
  return (umulhi_wide(v, 330282857u) >> 8) & ((1u << D) - 1);
}
template <int D>
__device__ __forceinline__ void compress_any_store_C(const int32_t (&r)[32], uint32_t* __restrict__ dst) {
  uint64_t acc = 0;
  int bits = 0, o = 0;
#pragma unroll
  for (int i = 0; i < 32; i++) {
    acc |= (uint64_t)compress_any<D>(r[i]) << bits;
    bits += D;
    if (bits >= 32) {
      dst[o++] = (uint32_t)acc;
      acc >>= 32;
      bits -= 32;
    }
  }
}

// 32 normalised coefficients (C layout, plain values in [0, q)) -> 12 words (poly.go:106-116)
__device__ __forceinline__ void pack12_C_lo(const int32_t (&r)[32], uint32_t (&w)[12]) {
#pragma unroll
  for (int g = 0; g < 4; g++) {
    uint32_t t[8];
#pragma unroll
    for (int j = 0; j < 8; j++) t[j] = (uint32_t)r[8 * g + j];
    w[3 * g] = t[0] | (t[1] << 12) | (t[2] << 24);
    w[3 * g + 1] = (t[2] >> 8) | (t[3] << 4) | (t[4] << 16) | (t[5] << 28);
    w[3 * g + 2] = (t[5] >> 4) | (t[6] << 8) | (t[7] << 20);
  }
}
// Normalize (field.go:45-74) of a low-format register holding any int16 value: csubq(barrettReduce(x))
__device__ __forceinline__ int32_t normalize_lo(int32_t x) {
  x = kyber::barrett_lo(x) - Q;
  return x + ((x >> 31) & Q);
}

// 24 bytes (8-byte aligned) of a 12-bit packed polynomial -> 16 coefficients as 8 packed pairs (poly.go:123-129);
// returns nonzero if any coefficient is >= q (cpapke.go:45-55)
__device__ __forceinline__ uint32_t unpack12_half(const uint32_t (&w)[8], uint32_t (&aw)[8]) {
  uint32_t bad = 0;
#pragma unroll
  for (int g = 0; g < 2; g++) {  // 3 words -> 8 coefficients -> 4 pairs
    const uint32_t a = w[3 * g], b = w[3 * g + 1], c = w[3 * g + 2];
    uint32_t t[8];
    t[0] = a & 0xfff;
    t[1] = (a >> 12) & 0xfff;
    t[2] = ((a >> 24) | (b << 8)) & 0xfff;
    t[3] = (b >> 4) & 0xfff;
    t[4] = (b >> 16) & 0xfff;
    t[5] = ((b >> 28) | (c << 4)) & 0xfff;
    t[6] = (c >> 8) & 0xfff;
    t[7] = c >> 20;
#pragma unroll
    for (int j = 0; j < 8; j++) bad |= (t[j] >= (uint32_t)Q);
#pragma unroll
    for (int j = 0; j < 4; j++) aw[4 * g + j] = t[2 * j] | (t[2 * j + 1] << 16);
  }
  return bad;
}

// What the three IDP.2A kernels (encrypt_dp_kernel, decrypt_dp_kernel, keygen_dp_kernel) share: the octet of a lane
// with its slices of dynamic shared memory, the byte-split operands and the accumulation of one half-row.
//
// The octet set-up: dynamic shared memory holds the operand areas of the THREADS / 8 octets, their transposition tiles
// and the 128 twiddle pairs, which are staged here (hence the __syncthreads: every thread of the CTA builds one).  base is
// the first op of this warp; a kernel returns when base >= n and asks for active(n) / op(n) only after that.
template <int K, int THREADS>
struct Octet {
  uint2* ops;  // this lane's column of the octet's operands, [j][block][lane]
  uint32_t* tile;
  const volatile kyber::TwLow* tabl;
  int oct, v;
  unsigned mask;
  size_t base;
  __device__ __forceinline__ explicit Octet(const kyber::TwPair* __restrict__ tw) {
    using S = EncSmem<K, THREADS>;
    constexpr int OCTS = THREADS / 8;
    extern __shared__ __align__(16) uint32_t enc_smem[];
    uint32_t* tiles = enc_smem + OCTS * S::op_words;
    kyber::TwPair* tws = reinterpret_cast<kyber::TwPair*>(tiles + OCTS * kyber::kPolyWords);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    oct = lane >> 3;
    v = lane & 7;
    mask = 0xffu << (8 * oct);
    tile = tiles + (warp * 4 + oct) * kyber::kPolyWords;
    ops = reinterpret_cast<uint2*>(enc_smem + (size_t)(warp * 4 + oct) * S::op_words) + v;
    for (int i = threadIdx.x; i < 128; i += THREADS) tws[i] = tw[128 + i];  // {zp, kk} pairs in tw_slot order
    __syncthreads();
    tabl = reinterpret_cast<const volatile kyber::TwLow*>(tws);
    base = ((size_t)blockIdx.x * (THREADS / 32) + warp) * 4;
  }
  __device__ __forceinline__ bool active(size_t n) const { return base + oct < n; }
  // this octet's op, clamped to n - 1 so that an inactive octet still reads valid memory
  __device__ __forceinline__ size_t op(size_t n) const { return active(n) ? base + oct : n - 1; }
  // the octet's whole operand area (op_words words)
  __device__ __forceinline__ uint32_t* area() const { return reinterpret_cast<uint32_t*>(ops - v); }
};

// The noise of one op, made by its octet (K-PKE.KeyGen / Encrypt: DeriveNoise, sample.go:31-95).  Lane p runs the PRF
// streams p, p + 8, ... < S -- SHAKE256(seed || p), the first E1 of them squeezed to 64 ETA1 bytes, the others to 128
// (eta = 2) -- and stages the output in the octet's operand area, which is free until the first store_operands:
// stream j at word prf_offset(j), 34 / 50 words apart so that the 64-bit stores of the lanes fall in different banks.
// After a __syncwarp each lane gathers its words of every stream with kyber::noise_select; the polynomials never
// exist in global memory.
template <int ETA1, int E1>
__host__ __device__ constexpr int prf_offset(int j) {
  return j < E1 ? j * (ETA1 == 3 ? 50 : 34) : E1 * (ETA1 == 3 ? 50 : 34) + (j - E1) * 34;
}
template <int K, int THREADS, int S, int E1, int ETA1>
__device__ __forceinline__ void octet_prf(uint32_t* area, const uint64_t* __restrict__ seed, int v) {
  static_assert(prf_offset<ETA1, E1>(S) <= EncSmem<K, THREADS>::op_words, "PRF output must fit in the operand area");
#pragma unroll 1
  for (int p = v; p < S; p += 8) {
    uint64_t a[25];
    keccak::zero(a);
#pragma unroll
    for (int w = 0; w < 4; w++) a[w] = __ldg(seed + w);
    a[4] = (uint64_t)p | (0x1full << 8);
    a[16] = 0x8000000000000000ull;  // rate 136
    keccak::f1600(a);
    uint64_t* dst = reinterpret_cast<uint64_t*>(area + prf_offset<ETA1, E1>(p));
    if (ETA1 == 3 && p < E1) {
#pragma unroll
      for (int q = 0; q < 17; q++) dst[q] = a[q];
      keccak::f1600(a);
#pragma unroll
      for (int q = 0; q < 7; q++) dst[17 + q] = a[q];
    } else {
#pragma unroll
      for (int q = 0; q < 16; q++) dst[q] = a[q];
    }
  }
}

// The byte-split operands W0, W1 of column j from a transformed polynomial (this lane's 32 coefficients, C layout), each
// coefficient first multiplied by the constant of the Shoup pair (zp, kk).  Quad q of the lane has zeta = Zetas[64 + 8 v + q]:
// +zeta for its first block, -zeta for its second.
__device__ __forceinline__ void store_operands(uint2* ops, int j, const int32_t (&r)[32], const volatile kyber::TwLow* tabl,
                                               int v, int32_t zp, int32_t kk) {
  using namespace kyber;
#pragma unroll
  for (int q = 0; q < 8; q++) {
    const TwLow z = twl_at(tabl, 64 + 8 * q + v);
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int blk = 2 * q + h;
      const int32_t b0 = mont_mul_lo(r[2 * blk], zp, kk), b1 = mont_mul_lo(r[2 * blk + 1], zp, kk);
      int32_t zb1 = mont_mul_lo(b1, z.zp, z.kk);
      if (h) zb1 = -zb1;
      // bytes 0 (low, unsigned) and 1 (high, signed) of the registers
      ops[(j * 16 + blk) * 8] = make_uint2(__byte_perm((uint32_t)b0, (uint32_t)zb1, 0x5140),
                                           __byte_perm((uint32_t)b1, (uint32_t)b0, 0x5140));
    }
  }
}

// The outputs p0, p1 of eight blocks (one half-row), summed over the columns: per column and block four IDP.2A, the
// products with the low (unsigned) and the high (signed) operand bytes kept apart until the reduction.
struct DotAcc {
  int32_t p0l[8], p0h[8], p1l[8], p1h[8];
  __device__ __forceinline__ DotAcc() {
#pragma unroll
    for (int c = 0; c < 8; c++) p0l[c] = p0h[c] = p1l[c] = p1h[c] = 0;
  }
  // one column: the eight packed words aw against the operands oj of the same eight blocks
  __device__ __forceinline__ void add(const uint32_t (&aw)[8], const uint2* oj) {
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const uint2 w = oj[c * 8];
      p0l[c] = (int32_t)dp2a_lo_uu(aw[c], w.x, (uint32_t)p0l[c]);
      p0h[c] = dp2a_hi_us(aw[c], w.x, p0h[c]);
      p1l[c] = (int32_t)dp2a_lo_uu(aw[c], w.y, (uint32_t)p1l[c]);
      p1h[c] = dp2a_hi_us(aw[c], w.y, p1h[c]);
    }
  }
  // montReduce of the two outputs of block c
  __device__ __forceinline__ int32_t p0(int c) const { return mont_red_lo(p0l[c] + p0h[c] * 256); }
  __device__ __forceinline__ int32_t p1(int c) const { return mont_red_lo(p1l[c] + p1h[c] * 256); }
  // the eight blocks are coefficients r[OFF .. OFF + 16)
  template <int OFF>
  __device__ __forceinline__ void reduce_into(int32_t (&r)[32]) const {
#pragma unroll
    for (int c = 0; c < 8; c++) {
      r[OFF + 2 * c] = p0(c);
      r[OFF + 2 * c + 1] = p1(c);
    }
  }
};

// THREADS / 8 operations per CTA.  Small CTAs (64 threads, 8 operations, ~31 KB of shared memory for K = 3) keep 7 CTAs
// = 14 warps per SM resident; every global load is issued one step before its data is used (register double buffers),
// because a warp walks 19 dependent load -> compute phases per operation and L2 latency, not the instruction count,
// was what bounded the first version (ncu: long_scoreboard 1.3 per issue at 12-16 warps per SM).
template <int K, int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) encrypt_dp_kernel(
    const uint8_t* __restrict__ ek, size_t ek_stride, const int16_t* __restrict__ A, int a_shared,
    const uint64_t* __restrict__ rseed, const uint8_t* __restrict__ m, size_t n, uint8_t* __restrict__ ct,
    uint8_t* __restrict__ ss, uint8_t* __restrict__ status, const kyber::TwPair* __restrict__ tw, int lenient) {
  // lenient = 1: re-encryption inside Decapsulate (PublicKey.Unpack, cpapke.go:58-63: no modulus check; the
  // Normalize of t-hat is immaterial here because only residues are used).  rseed: the PRF seed r, 4 words per op.
  using P = Params<K>;
  using namespace kyber;
  // every transform of this kernel runs on low-format registers (kyber.cuh): its inputs are bounded by construction
  // (|noise| <= 3, |montReduce(.)| <= q), far inside the range where no int16 of the reference would wrap
  const Octet<K, THREADS> o(tw);
  if (o.base >= n) return;
  const int v = o.v;
  const size_t op = o.op(n);
  const uint8_t* ekp = ek + op * ek_stride;
  const uint32_t* Ap = reinterpret_cast<const uint32_t*>(A) + (a_shared ? 0 : op * K * K * (N / 2));
  uint8_t* ctp = ct + op * P::ct_bytes;

  // r[0..K) (eta1), e1[0..K), e2 (eta2 = 2) from PRF(r, 0 .. 2K) (cpapke.go:145-159): the lane's words of each, those
  // of e1 kept in registers until their row (eb[0] is always the next one), those of e2 behind the operands
  int32_t r[32];
  uint32_t eb[K][4];
  uint4* const e2s = reinterpret_cast<uint4*>(o.area() + 2 * 128 * K) + v;
  {
    uint32_t* const area = o.area();
    octet_prf<K, THREADS, P::n_noise, K, P::eta1>(area, rseed + 4 * op, v);
    __syncwarp();
    uint32_t rb[K][kNoiseWords<P::eta1>], e2[4];
#pragma unroll
    for (int j = 0; j < K; j++) {
      noise_select<P::eta1>(area + prf_offset<P::eta1, K>(j), v, rb[j]);
      noise_select<2>(area + prf_offset<P::eta1, K>(K + j), v, eb[j]);
    }
    noise_select<2>(area + prf_offset<P::eta1, K>(2 * K), v, e2);
    *e2s = make_uint4(e2[0], e2[1], e2[2], e2[3]);
    __syncwarp();  // the operands overwrite the staged PRF output

    // operands of rh = NTT(r) x 512  (cpapke.go:142-144; the reduction is the multiplication)
#pragma unroll 1
    for (int j = 0; j < K; j++) {
      noise_cbd<P::eta1>(rb[0], r);
#pragma unroll
      for (int q = 0; q + 1 < K; q++)
#pragma unroll
        for (int w = 0; w < kNoiseWords<P::eta1>; w++) rb[q][w] = rb[q + 1][w];
      fwd_pass_S_lo(r);
      store_S_lo(o.tile, v, r);
      __syncwarp();
      load_C_lo(o.tile, v, r);
      fwd_pass_C_lo_smem(r, o.tabl, v);
      __syncwarp();
      // x 512 = R / 128: the Montgomery product by 512 R mod q = 1441, i.e. the pair (kScaleZp, kScaleKk) of the
      // inverse transform (|in| <= 7 q, |out| < q)
      store_operands(o.ops, j, r, o.tabl, v, kScaleZp, kScaleKk);
    }
  }
  __syncwarp();

  // u[i] = InvNTT(A^T[i] . rh) + e1[i]; v = InvNTT(t . rh) + e2 + m.  A row is accumulated in two halves of eight
  // blocks (32 accumulators).
  auto fetch = [&](int i, int h, int j, uint32_t (&raw)[8]) {
    if (i < K) {
      const uint4* p = reinterpret_cast<const uint4*>(Ap + (i * K + j) * (N / 2) + 16 * v + 8 * h);
      const uint4 x = __ldg(p), y = __ldg(p + 1);
      raw[0] = x.x, raw[1] = x.y, raw[2] = x.z, raw[3] = x.w, raw[4] = y.x, raw[5] = y.y, raw[6] = y.z, raw[7] = y.w;
    } else {  // row K: t-hat from the encapsulation key, PolyDotHat(&v, &pk.th, &rh) (cpapke.go:167)
      const uint2* p = reinterpret_cast<const uint2*>(ekp + 384 * j + 48 * v + 24 * h);
      const uint2 x = __ldg(p), y = __ldg(p + 1), z = __ldg(p + 2);
      raw[0] = x.x, raw[1] = x.y, raw[2] = y.x, raw[3] = y.y, raw[4] = z.x, raw[5] = z.y;
    }
  };
  // raw[j]: the eight words of column j of the half-row that comes next; refilled for the half-row after it as soon as they
  // have been consumed, i.e. every load is K steps (~250 instructions of this warp) ahead of its use
  uint32_t bad = 0;
  uint32_t raw[K][8];
#pragma unroll
  for (int j = 0; j < K; j++) fetch(0, 0, j, raw[j]);
#pragma unroll 1
  for (int i = 0; i <= K; i++) {
#pragma unroll 1
    for (int h = 0; h < 2; h++) {
      DotAcc acc;
      const int ni = h ? i + 1 : i, nh = h ^ 1;  // the half-row after this one
#pragma unroll
      for (int j = 0; j < K; j++) {
        uint32_t aw[8];
        if (i < K) {
#pragma unroll
          for (int c = 0; c < 8; c++) aw[c] = raw[j][c];
        } else {
          const uint32_t b = unpack12_half(raw[j], aw);
          if (!lenient) bad |= b;
        }
        if (ni <= K) fetch(ni, nh, j, raw[j]);
        acc.add(aw, o.ops + (size_t)(j * 16 + 8 * h) * 8);
      }
      if (h == 0)
        acc.reduce_into<0>(r);
      else
        acc.reduce_into<16>(r);
    }
    inv_pass_C_lo(r, o.tabl, v);
    store_C_lo(o.tile, v, r);
    __syncwarp();
    load_S_lo(o.tile, v, r);
    inv_pass_S_lo<false>(r, v);
    __syncwarp();
    // before the constant the reference bounds the values by 9 q (ntt.go:187-190), so adding e (<= 2) and the message
    // term (1665) stays inside the int16 range the packed tile below carries
    {  // + e1[i] / + e2 (+ Decompress_q(m, 1)), S layout
      const uint32_t* mw = reinterpret_cast<const uint32_t*>(m + 32 * op);
      uint32_t ew[4];
      if (i < K) {
#pragma unroll
        for (int w = 0; w < 4; w++) ew[w] = eb[0][w];
      } else {
        const uint4 t = *e2s;
        ew[0] = t.x, ew[1] = t.y, ew[2] = t.z, ew[3] = t.w;
      }
#pragma unroll
      for (int k = 0; k < 4; k++) {
        uint32_t ep[4];
        noise_pairs<2>(ew, k, ep);
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int s = 4 * k + q;
          int32_t e0, e1;
          unpack2_lo(ep[q], e0, e1);
          r[2 * s] += e0;
          r[2 * s + 1] += e1;
          if (i == K) {  // DecompressMessage, poly.go:134-147: coefficient idx = 16 s + 2 v + b <- bit idx of m
            const uint32_t word = __ldg(mw + (s >> 1));
            const uint32_t bits = (word >> (16 * (s & 1) + 2 * v)) & 3;
            r[2 * s] += (bits & 1) ? (Q + 1) / 2 : 0;
            r[2 * s + 1] += (bits & 2) ? (Q + 1) / 2 : 0;
          }
        }
      }
#pragma unroll
      for (int q = 0; q + 1 < K; q++)
#pragma unroll
        for (int w = 0; w < 4; w++) eb[q][w] = eb[q + 1][w];
    }
    store_S_lo(o.tile, v, r);  // Normalize (cpapke.go:176-177) is absorbed by compress_any
    __syncwarp();
    load_C_lo(o.tile, v, r);
    __syncwarp();
    bad = __any_sync(o.mask, bad) ? 1u : 0u;  // after row K this holds the modulus check of the whole key
    if (o.active(n)) {
      if (i < K)
        compress_any_store_C<P::du>(r, reinterpret_cast<uint32_t*>(ctp + i * 32 * P::du) + v * P::du);
      else if (!bad)
        compress_any_store_C<P::dv>(r, reinterpret_cast<uint32_t*>(ctp + K * 32 * P::du) + v * P::dv);
    }
  }
  // kem.ErrPubKey (cpapke.go:48-54): no output for a non-canonical key
  if (o.active(n)) {
    if (bad) {
      uint32_t* c32 = reinterpret_cast<uint32_t*>(ctp);
      for (int w = v; w < P::ct_bytes / 4; w += 8) c32[w] = 0;
      if (ss) reinterpret_cast<uint32_t*>(ss + 32 * op)[v] = 0;
    }
    if (status && v == 0 && !lenient) status[op] = (uint8_t)bad;
  }
}

// The launch of the three IDP.2A kernels (encrypt_dp_kernel, decrypt_dp_kernel, keygen_dp_kernel) over n ops, all
// timed under KID_MLKEM_ENCRYPT.  7 CTAs of 64 threads per SM (K = 4: 6, its operands and registers are larger); H100
// has the register file and shared memory per SM these were sized for.
constexpr int kDpThreads = 64;
template <int K>
constexpr int kDpMinBlocks = K == 4 ? 6 : 7;
template <int K, typename... P, typename... A>
static int launch_dp(void (*kernel)(P...), size_t n, cudaStream_t st, A... args) {
  constexpr int bytes = EncSmem<K, kDpThreads>::bytes, per_cta = kDpThreads / 8;
  if (int arc = ensure_smem_attr((const void*)kernel, bytes)) return arc;
  KernelScope ks(KID_MLKEM_ENCRYPT, st);
  kernel<<<(unsigned)((n + per_cta - 1) / per_cta), kDpThreads, bytes, st>>>(args...);
  return 0;
}

// Sub-batches of sub_batch(n) ops alternate between the two lanes of the work set, forked from the caller's stream and
// joined back to it with events: the tail wave of one sub-batch's kernels overlaps the next sub-batch instead of idling
// SMs.  launch(first, cnt, lane, stream) enqueues one sub-batch; a nonzero result ends the loop and is returned.
static size_t sub_batch(size_t n) { return n < kSub ? n : kSub; }
template <typename F>
static int for_sub_batches(WorkSet& ws, size_t n, cudaStream_t st, F&& launch) {
  const size_t sub = sub_batch(n);
  CB200_CUDA(cudaEventRecord(ws.ev_fork, st));
  for (int l = 0; l < 2; l++) CB200_CUDA(cudaStreamWaitEvent(ws.lane[l], ws.ev_fork, 0));
  int l = 0;
  for (size_t first = 0; first < n; first += sub, l ^= 1) {
    // per-kernel event timing (cb200_profile_enable) wants true, non-overlapped durations: stay on one stream
    cudaStream_t ls = profiling_on() ? st : ws.lane[l];
    const size_t cnt = (n - first < sub) ? n - first : sub;
    if (int rc = launch(first, cnt, l, ls)) return rc;
  }
  for (int l = 0; l < 2; l++) {
    CB200_CUDA(cudaEventRecord(ws.ev_join[l], ws.lane[l]));
    CB200_CUDA(cudaStreamWaitEvent(st, ws.ev_join[l], 0));
  }
  return 0;
}

// (K', r) = G(m || h), ct = K-PKE.Encrypt(ek, m, r) with the lenient key parse, per-op keys: the re-encryption of
// ML-KEM and round-3 Kyber Decapsulate, and the body of round-3 Kyber Encapsulate.  base + o_A[l] is the matrix buffer
// of lane l.
template <int K>
static int encrypt_lenient(const uint8_t* ek, size_t ek_stride, const uint8_t* h, size_t h_stride, const uint8_t* m,
                           uint8_t* ct, uint8_t* kbar, uint64_t* r, char* base, const size_t (&o_A)[2], size_t n,
                           cudaStream_t st, int slot) {
  using P = Params<K>;
  {
    KernelScope ks(KID_MLKEM_G, st);
    g_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(m, h, h_stride, n, kbar, r);
  }
  const kyber::TwPair* tw = (const kyber::TwPair*)ctx().kyber_tw;
  return for_sub_batches(wset(slot), n, st, [&](size_t first, size_t cnt, int l, cudaStream_t ls) {
    int16_t* A = (int16_t*)(base + o_A[l]);
    if (int src = launch_sample<K>(slot, l, ls, ek + 384 * K + first * ek_stride, ek_stride, cnt, A, 1)) return src;
    return launch_dp<K>(encrypt_dp_kernel<K, kDpThreads, kDpMinBlocks<K>>, cnt, ls, ek + first * ek_stride, ek_stride, A, 0,
                        (const uint64_t*)(r + 4 * first), m + 32 * first, cnt, ct + first * P::ct_bytes, nullptr, nullptr,
                        tw, 1);
  });
}


// ------------------------------------------------------------------ 4. Decapsulate
// Decompress_q(x, d) (poly.go:170-243) of 32 coefficients (C layout) from D words
template <int D, bool LOW = false>
__device__ __forceinline__ void decompress_C(const uint32_t* __restrict__ src, int32_t (&r)[32]) {
  uint32_t w[D + 1];
#pragma unroll
  for (int i = 0; i < D; i++) w[i] = __ldg(src + i);
  w[D] = 0;
#pragma unroll
  for (int i = 0; i < 32; i++) {
    const int bit = D * i, wi = bit >> 5, sh = bit & 31;
    uint32_t t = w[wi] >> sh;
    if (sh + D > 32) t |= w[wi + 1] << (32 - sh);
    t &= (1u << D) - 1;
    const uint32_t x = ((1u << (D - 1)) + t * (uint32_t)Q) >> D;
    r[i] = (int32_t)(LOW ? x : x << 16);
  }
}

// K-PKE.Decrypt (cpapke.go:113-130): m' = CompressMessage(v - InvNTT(s-hat . NTT(u))); one octet per op.
// The message bits only depend on residues, so the kernel has the shape of the last row of encrypt_dp_kernel: the packed
// 12-bit words of s-hat in dk are the 16-bit side of IDP.2A products (any 12-bit value will do: PrivateKey.Unpack's
// Normalize, cpapke.go:32-36, does not change a residue), NTT(u[j]) x 512 are the byte-split operands, one Montgomery
// reduction per coefficient feeds the inverse transform without its final constant; all transforms on low-format
// registers (|Decompress(.)| < q).
template <int K, int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) decrypt_dp_kernel(const uint8_t* __restrict__ dk, size_t dk_stride,
                                                                   const uint8_t* __restrict__ ct, size_t n,
                                                                   uint8_t* __restrict__ mprime,
                                                                   const kyber::TwPair* __restrict__ tw) {
  using P = Params<K>;
  using namespace kyber;
  const Octet<K, THREADS> o(tw);
  if (o.base >= n) return;
  const int v = o.v;
  const size_t op = o.op(n);
  const uint8_t* dkp = dk + op * dk_stride;
  const uint8_t* ctp = ct + op * P::ct_bytes;
  int32_t r[32];
#pragma unroll 1
  for (int j = 0; j < K; j++) {  // operands of u-hat[j] = NTT(Decompress(u[j])) x 512
    decompress_C<P::du, true>(reinterpret_cast<const uint32_t*>(ctp + j * 32 * P::du) + v * P::du, r);
    store_C_lo(o.tile, v, r);
    __syncwarp();
    load_S_lo(o.tile, v, r);
    __syncwarp();
    fwd_pass_S_lo(r);
    store_S_lo(o.tile, v, r);
    __syncwarp();
    load_C_lo(o.tile, v, r);
    fwd_pass_C_lo_smem(r, o.tabl, v);
    __syncwarp();
    store_operands(o.ops, j, r, o.tabl, v, kScaleZp, kScaleKk);
  }
  __syncwarp();
  // PolyDotHat(&m, &sk.sh, &u) (cpapke.go:121): one row over the K columns, in two halves of eight blocks
#pragma unroll 1
  for (int h = 0; h < 2; h++) {
    DotAcc acc;
#pragma unroll
    for (int j = 0; j < K; j++) {
      const uint2* p = reinterpret_cast<const uint2*>(dkp + 384 * j + 48 * v + 24 * h);
      const uint2 x = __ldg(p), y = __ldg(p + 1), zz = __ldg(p + 2);
      uint32_t raw[8] = {x.x, x.y, y.x, y.y, zz.x, zz.y, 0, 0}, aw[8];
      unpack12_half(raw, aw);
      acc.add(aw, o.ops + (size_t)(j * 16 + 8 * h) * 8);
    }
    if (h == 0)
      acc.reduce_into<0>(r);
    else
      acc.reduce_into<16>(r);
  }
  inv_pass_C_lo(r, o.tabl, v);
  store_C_lo(o.tile, v, r);
  __syncwarp();
  load_S_lo(o.tile, v, r);
  __syncwarp();
  inv_pass_S_lo<false>(r, v);
  // v polynomial: decompress in C layout, bring to S layout
  int32_t vv[32];
  decompress_C<P::dv, true>(reinterpret_cast<const uint32_t*>(ctp + K * 32 * P::du) + v * P::dv, vv);
  store_C_lo(o.tile, v, vv);
  __syncwarp();
  load_S_lo(o.tile, v, vv);
  __syncwarp();
  // m = Normalize(v - m); CompressMessageTo (poly.go:150-166); coefficient 16 s + 2 v + b -> bit of m'
  uint32_t words[8];
#pragma unroll
  for (int w = 0; w < 8; w++) words[w] = 0;
#pragma unroll
  for (int s = 0; s < 16; s++) {
#pragma unroll
    for (int b = 0; b < 2; b++) {
      const int32_t d = normalize_lo(vv[2 * s + b] - r[2 * s + b]);
      int32_t x = 1664 - d;
      x = (x >> 31) ^ x;
      x -= 832;
      const uint32_t bit = (uint32_t)x >> 31;
      words[s >> 1] |= bit << (16 * (s & 1) + 2 * v + b);
    }
  }
#pragma unroll
  for (int w = 0; w < 8; w++) {
    uint32_t x = words[w];
    x |= __shfl_xor_sync(o.mask, x, 1);
    x |= __shfl_xor_sync(o.mask, x, 2);
    x |= __shfl_xor_sync(o.mask, x, 4);
    words[w] = x;
  }
  if (o.active(n)) {
    uint32_t mine = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) mine = (v == w) ? words[w] : mine;
    reinterpret_cast<uint32_t*>(mprime + 32 * op)[v] = mine;
  }
}

// Implicit rejection (kyber.go:168-183): ss = (ct == ct2) ? K' : SHAKE256(z || ct)[:32]; also checks
// H(ek) against the copy stored in dk (kem.ErrPrivKey, kyber.go:226-228).  One thread per op.
template <int K>
__global__ void __launch_bounds__(128) select_kernel(const uint8_t* __restrict__ dk, size_t dk_stride,
                                                     const uint8_t* __restrict__ ct, const uint8_t* __restrict__ ct2,
                                                     const uint8_t* __restrict__ kbar, const uint64_t* __restrict__ hcalc,
                                                     size_t n, uint8_t* __restrict__ ss, uint8_t* __restrict__ status) {
  using P = Params<K>;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t* z = reinterpret_cast<const uint64_t*>(dk + i * dk_stride + 384 * K + P::ek_bytes + 32);
  const uint64_t* hst = reinterpret_cast<const uint64_t*>(dk + i * dk_stride + 384 * K + P::ek_bytes);
  const uint64_t* c1 = reinterpret_cast<const uint64_t*>(ct + i * P::ct_bytes);
  const uint64_t* c2 = reinterpret_cast<const uint64_t*>(ct2 + i * P::ct_bytes);
  constexpr int ctw = P::ct_bytes / 8, words = 4 + ctw, full = words / 17, rem = words % 17;
  uint64_t a[25];
  keccak::zero(a);
  uint64_t diff = 0;
  int k = 0;
#pragma unroll 1
  for (int b = 0; b < full; b++) {
#pragma unroll
    for (int w = 0; w < 17; w++, k++) {
      uint64_t x;
      if (k < 4) {
        x = z[k];
      } else {
        x = c1[k - 4];
        diff |= x ^ c2[k - 4];
      }
      a[w] ^= x;
    }
    keccak::f1600(a);
  }
#pragma unroll
  for (int w = 0; w < rem; w++, k++) {
    const uint64_t x = c1[k - 4];
    diff |= x ^ c2[k - 4];
    a[w] ^= x;
  }
  a[rem] ^= 0x1f;
  a[16] ^= 0x8000000000000000ull;
  keccak::f1600(a);
  const bool hbad = (hst[0] ^ hcalc[4 * i]) | (hst[1] ^ hcalc[4 * i + 1]) | (hst[2] ^ hcalc[4 * i + 2]) |
                    (hst[3] ^ hcalc[4 * i + 3]);
  const uint64_t* kb = reinterpret_cast<const uint64_t*>(kbar + 32 * i);
  uint64_t* so = reinterpret_cast<uint64_t*>(ss + 32 * i);
#pragma unroll
  for (int j = 0; j < 4; j++) so[j] = hbad ? 0 : (diff == 0 ? kb[j] : a[j]);
  if (status) status[i] = hbad ? 2 : 0;
}

template <int K>
static int decaps_device(const uint8_t* dk, size_t dk_stride, const uint8_t* ct, uint8_t* ss, uint8_t* status, size_t n,
                         cudaStream_t st, int slot) {
  using P = Params<K>;
  Dev& c = ctx();
  const size_t sub = sub_batch(n);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t o_h = take(n * 32), o_r = take(n * 32), o_m = take(n * 32), o_k = take(n * 32),
               o_ct2 = take(n * (size_t)P::ct_bytes);
  size_t o_A[2];
  for (int q = 0; q < 2; q++) o_A[q] = take(sub * K * K * 512);
  void* base = nullptr;
  int rc = ensure_work(slot, off, &base);
  if (rc) return rc;
  char* b = (char*)base;
  uint64_t* h = (uint64_t*)(b + o_h);
  uint64_t* r = (uint64_t*)(b + o_r);
  uint8_t* mprime = (uint8_t*)(b + o_m);
  uint8_t* kbar = (uint8_t*)(b + o_k);
  uint8_t* ct2 = (uint8_t*)(b + o_ct2);
  const uint8_t* ek = dk + 384 * K;  // dk = sk || ek || H(ek) || z (kyber.go:187-201)
  if (int arc = ensure_smem_attr((const void*)sample_kernel<K>, kSampleSmem)) return arc;
  const kyber::TwPair* tw = (const kyber::TwPair*)c.kyber_tw;
  if (int drc = launch_dp<K>(decrypt_dp_kernel<K, kDpThreads, kDpMinBlocks<K>>, n, st, dk, dk_stride, ct, n, mprime, tw))
    return drc;
  {
    KernelScope ks(KID_MLKEM_HASH_EK, st);
    hash_ek_kernel<K><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(ek, dk_stride, n, h);
  }
  // (K', r') = G(m' || h) with the h stored in dk (kyber.go:160-164), ct' = K-PKE.Encrypt(ek, m', r')
  rc = encrypt_lenient<K>(ek, dk_stride, dk + 384 * K + P::ek_bytes, dk_stride, mprime, ct2, kbar, r, b, o_A, n, st, slot);
  if (rc) return rc;
  {
    KernelScope ks(KID_MLKEM_G, st);
    select_kernel<K><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(dk, dk_stride, ct, ct2, kbar, h, n, ss, status);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}


// ------------------------------------------------------------------ 5. KeyGen (SURVEY.md 8(f) row 2)
// (rho, sigma) = SHA3-512(d || byte(K))  (pke/kyber/kyber768/kyber.go:77-86, cpapke.go:72-79); one thread per op.
// Writes rho||sigma (8 words) to rs, rho into ek/dk, z into dk.
template <int K>
__global__ void __launch_bounds__(128) keygen_seed_kernel(const uint8_t* __restrict__ seed, size_t n,
                                                          uint64_t* __restrict__ rs, uint8_t* __restrict__ ek,
                                                          uint8_t* __restrict__ dk, int mlkem) {
  using P = Params<K>;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t* sd = reinterpret_cast<const uint64_t*>(seed + 64 * i);
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll
  for (int j = 0; j < 4; j++) a[j] = sd[j];
  a[4] = mlkem ? ((uint64_t)K | (0x06ull << 8)) : 0x06ull;  // round-3 Kyber hashes the bare 32-byte seed
  a[8] = 0x8000000000000000ull;                               // SHA3-512, rate 72
  keccak::f1600(a);
  uint64_t* ekr = reinterpret_cast<uint64_t*>(ek + i * P::ek_bytes + 384 * K);
  uint64_t* dkr = reinterpret_cast<uint64_t*>(dk + i * (768 * K + 96) + 384 * K + 384 * K);
  uint64_t* dkz = reinterpret_cast<uint64_t*>(dk + i * (768 * K + 96) + 384 * K + P::ek_bytes + 32);
#pragma unroll
  for (int j = 0; j < 8; j++) rs[8 * i + j] = a[j];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    ekr[j] = a[j];
    dkr[j] = a[j];
    dkz[j] = sd[4 + j];  // z = seed[32:64] (kem/mlkem/mlkem768/kyber.go:66-67)
  }
}

// 32 normalised coefficients (C layout, high-half registers) -> 12 words (poly.go:106-116)
__device__ __forceinline__ void pack12_C(const int32_t (&r)[32], uint32_t (&w)[12]) {
#pragma unroll
  for (int g = 0; g < 4; g++) {
    uint32_t t[8];
#pragma unroll
    for (int j = 0; j < 8; j++) t[j] = (uint32_t)r[8 * g + j] >> 16;
    w[3 * g] = t[0] | (t[1] << 12) | (t[2] << 24);
    w[3 * g + 1] = (t[2] >> 8) | (t[3] << 4) | (t[4] << 16) | (t[5] << 28);
    w[3 * g + 2] = (t[5] >> 4) | (t[6] << 8) | (t[7] << 20);
  }
}

// K-PKE.KeyGen arithmetic (cpapke.go:83-105): s-hat = Normalize(NTT(s)), e-hat = NTT(e),
// t-hat[i] = Normalize(ToMont(A[i] . s-hat) + e-hat[i]); packs s-hat into dk and t-hat into ek and dk.  Octet per op.
// What leaves the kernel is Normalize(.), so -- as in encrypt_dp_kernel -- only residues matter inside it and the same two
// devices apply: the matrix-vector product runs as IDP.2A dot products of the packed words of A with byte-split
// operands made once per op from s-hat, here carrying s-hat R (one Montgomery multiplication by R^2 = 1353, which is the
// reference's ToMont moved onto the operand: montReduce(sum a . s-hat R) = sum a . s-hat), and every transform runs on
// low-format registers (inputs |c| <= 3).
template <int K, int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) keygen_dp_kernel(const int16_t* __restrict__ A,
                                                                  const uint64_t* __restrict__ rs, size_t n,
                                                                  uint8_t* __restrict__ ek, uint8_t* __restrict__ dk,
                                                                  const kyber::TwPair* __restrict__ tw) {
  using P = Params<K>;
  using namespace kyber;
  // R^2 mod q = 1353 (field.go:35-39) as a Shoup pair: zp = R mod q = 2285 - q
  constexpr int32_t kR2Zp = 2285 - Q, kR2Kk = (kR2Zp * 65536 - 1353) / Q;
  static_assert(kR2Zp * 65536 - 1353 == kR2Kk * Q, "ToMont constant");
  const Octet<K, THREADS> o(tw);
  if (o.base >= n) return;
  const int v = o.v;
  const size_t op = o.op(n);
  const uint32_t* Ap = reinterpret_cast<const uint32_t*>(A) + op * K * K * (N / 2);
  uint8_t* ekp = ek + op * P::ek_bytes;
  uint8_t* dkp = dk + op * (768 * K + 96);

  // s[0..K), e[0..K) (both eta1) from PRF(sigma, 0 .. 2K) (cpapke.go:81-94), sigma = rs[8 op + 4 ..): the lane's words of
  // each, the e-words kept until their row (eb[0] is always the next one)
  constexpr int NW = kNoiseWords<P::eta1>;
  int32_t r[32];
  uint32_t eb[K][NW];
  {  // s-hat[j]: packed into dk (normalised) and turned into the operands of the products
    uint32_t* const area = o.area();
    octet_prf<K, THREADS, 2 * K, 2 * K, P::eta1>(area, rs + 8 * op + 4, v);
    __syncwarp();
    uint32_t sb[K][NW];
#pragma unroll
    for (int j = 0; j < K; j++) {
      noise_select<P::eta1>(area + prf_offset<P::eta1, 2 * K>(j), v, sb[j]);
      noise_select<P::eta1>(area + prf_offset<P::eta1, 2 * K>(K + j), v, eb[j]);
    }
    __syncwarp();  // the operands overwrite the staged PRF output
#pragma unroll 1
    for (int j = 0; j < K; j++) {
      noise_cbd<P::eta1>(sb[0], r);
#pragma unroll
      for (int q = 0; q + 1 < K; q++)
#pragma unroll
        for (int w = 0; w < NW; w++) sb[q][w] = sb[q + 1][w];
      fwd_pass_S_lo(r);
      store_S_lo(o.tile, v, r);
      __syncwarp();
      load_C_lo(o.tile, v, r);
      fwd_pass_C_lo_smem(r, o.tabl, v);
      __syncwarp();
      store_operands(o.ops, j, r, o.tabl, v, kR2Zp, kR2Kk);
#pragma unroll
      for (int c = 0; c < 32; c++) r[c] = normalize_lo(r[c]);
      uint32_t pw[12];
      pack12_C_lo(r, pw);
      if (o.active(n)) {
        uint32_t* dst = reinterpret_cast<uint32_t*>(dkp + 384 * j) + 12 * v;
#pragma unroll
        for (int w = 0; w < 12; w++) dst[w] = pw[w];
      }
    }
  }
  __syncwarp();

  // t-hat[i] = Normalize(A[i] . s-hat + e-hat[i]); a row is accumulated in two halves of eight blocks, every load of A
  // issued K steps before its use (as in encrypt_dp_kernel)
  auto fetch = [&](int i, int h, int j, uint32_t (&raw)[8]) {
    const uint4* p = reinterpret_cast<const uint4*>(Ap + (i * K + j) * (N / 2) + 16 * v + 8 * h);
    const uint4 x = __ldg(p), y = __ldg(p + 1);
    raw[0] = x.x, raw[1] = x.y, raw[2] = x.z, raw[3] = x.w, raw[4] = y.x, raw[5] = y.y, raw[6] = y.z, raw[7] = y.w;
  };
  uint32_t raw[K][8];
#pragma unroll
  for (int j = 0; j < K; j++) fetch(0, 0, j, raw[j]);
#pragma unroll 1
  for (int i = 0; i < K; i++) {
    noise_cbd<P::eta1>(eb[0], r);  // e-hat[i] = NTT(e[i])
#pragma unroll
    for (int q = 0; q + 1 < K; q++)
#pragma unroll
      for (int w = 0; w < NW; w++) eb[q][w] = eb[q + 1][w];
    fwd_pass_S_lo(r);
    store_S_lo(o.tile, v, r);
    __syncwarp();
    load_C_lo(o.tile, v, r);
    fwd_pass_C_lo_smem(r, o.tabl, v);
    __syncwarp();
#pragma unroll 1
    for (int h = 0; h < 2; h++) {
      DotAcc acc;
      const int ni = h ? i + 1 : i, nh = h ^ 1;  // the half-row after this one
#pragma unroll
      for (int j = 0; j < K; j++) {
        uint32_t aw[8];
#pragma unroll
        for (int c = 0; c < 8; c++) aw[c] = raw[j][c];
        if (ni < K) fetch(ni, nh, j, raw[j]);
        acc.add(aw, o.ops + (size_t)(j * 16 + 8 * h) * 8);
      }
      if (h == 0) {
#pragma unroll
        for (int c = 0; c < 8; c++) {
          r[2 * c] = normalize_lo(acc.p0(c) + r[2 * c]);
          r[2 * c + 1] = normalize_lo(acc.p1(c) + r[2 * c + 1]);
        }
      } else {
#pragma unroll
        for (int c = 0; c < 8; c++) {
          r[16 + 2 * c] = normalize_lo(acc.p0(c) + r[16 + 2 * c]);
          r[16 + 2 * c + 1] = normalize_lo(acc.p1(c) + r[16 + 2 * c + 1]);
        }
      }
    }
    uint32_t pw[12];
    pack12_C_lo(r, pw);
    if (o.active(n)) {
      uint32_t* d1 = reinterpret_cast<uint32_t*>(ekp + 384 * i) + 12 * v;
      uint32_t* d2 = reinterpret_cast<uint32_t*>(dkp + 384 * K + 384 * i) + 12 * v;
#pragma unroll
      for (int w = 0; w < 12; w++) {
        d1[w] = pw[w];
        d2[w] = pw[w];
      }
    }
  }
}

template <int K>
static int keygen_device(const uint8_t* seeds, uint8_t* ek, uint8_t* dk, size_t n, cudaStream_t st, int slot,
                         int mlkem = 1) {
  using P = Params<K>;
  Dev& c = ctx();
  const size_t sub = sub_batch(n);
  constexpr size_t dksz = 768 * K + 96;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t o_rs = take(n * 64), o_h = take(n * 32);
  size_t o_A[2];
  for (int q = 0; q < 2; q++) o_A[q] = take(sub * K * K * 512);
  void* base = nullptr;
  int rc = ensure_work(slot, off, &base);
  if (rc) return rc;
  char* b = (char*)base;
  uint64_t* rs = (uint64_t*)(b + o_rs);
  uint64_t* h = (uint64_t*)(b + o_h);
  if (int arc = ensure_smem_attr((const void*)sample_kernel<K>, kSampleSmem)) return arc;
  {
    KernelScope ks(KID_MLKEM_G, st);
    keygen_seed_kernel<K><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(seeds, n, rs, ek, dk, mlkem);
  }
  const kyber::TwPair* tw = (const kyber::TwPair*)c.kyber_tw;
  rc = for_sub_batches(wset(slot), n, st, [&](size_t first, size_t cnt, int l, cudaStream_t ls) {
    int16_t* A = (int16_t*)(b + o_A[l]);
    // A (not transposed) from rho = rs[0..4); the kernel derives s and e from sigma = rs[4..8)
    if (int src = launch_sample<K>(slot, l, ls, (const uint8_t*)(rs + 8 * first), 64, cnt, A, 0)) return src;
    return launch_dp<K>(keygen_dp_kernel<K, kDpThreads, kDpMinBlocks<K>>, cnt, ls, A, (const uint64_t*)(rs + 8 * first), cnt,
                        ek + first * P::ek_bytes, dk + first * dksz, tw);
  });
  if (rc) return rc;
  {  // H(ek) into dk (kyber.go:69-75)
    KernelScope ks(KID_MLKEM_HASH_EK, st);
    hash_ek_kernel<K><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(ek, P::ek_bytes, n, h);
  }
  CB200_CUDA(cudaMemcpy2DAsync(dk + 384 * K + P::ek_bytes, dksz, h, 32, 32, n, cudaMemcpyDeviceToDevice, st));
  CB200_CUDA(cudaGetLastError());
  return 0;
}


// ------------------------------------------------------------------ 6. round-3 Kyber KEM (SURVEY.md 8(f) row 4)
// kem/kyber/kyber768/kyber.go:98-198: same K-PKE; m = H(seed) ("hash of shame"), ss = KDF(K || H(ct)),
// implicit rejection replaces K by z.  Thread per op.
__global__ void __launch_bounds__(128) r3_m_kernel(const uint8_t* __restrict__ seeds, size_t n, uint8_t* __restrict__ m) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll
  for (int j = 0; j < 4; j++) a[j] = reinterpret_cast<const uint64_t*>(seeds + 32 * i)[j];
  a[4] = 0x06;
  a[16] = 0x8000000000000000ull;  // SHA3-256, rate 136
  keccak::f1600(a);
#pragma unroll
  for (int j = 0; j < 4; j++) reinterpret_cast<uint64_t*>(m + 32 * i)[j] = a[j];
}

// ss = SHAKE256(Kbar' || SHA3-256(ct), 32) with Kbar' = Kbar, or z when ct2 is given and differs from ct
template <int K>
__global__ void __launch_bounds__(128) r3_kdf_kernel(const uint8_t* __restrict__ ct, const uint8_t* __restrict__ ct2,
                                                     const uint8_t* __restrict__ kbar, const uint8_t* __restrict__ z,
                                                     size_t z_stride, size_t n, uint8_t* __restrict__ ss) {
  using P = Params<K>;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t* c1 = reinterpret_cast<const uint64_t*>(ct + i * P::ct_bytes);
  const uint64_t* c2 = ct2 ? reinterpret_cast<const uint64_t*>(ct2 + i * P::ct_bytes) : nullptr;
  constexpr int words = P::ct_bytes / 8, full = words / 17, rem = words % 17;
  uint64_t a[25];
  keccak::zero(a);
  uint64_t diff = 0;
#pragma unroll 1
  for (int b = 0; b < full; b++) {
#pragma unroll
    for (int w = 0; w < 17; w++) {
      const uint64_t x = c1[17 * b + w];
      if (c2) diff |= x ^ c2[17 * b + w];
      a[w] ^= x;
    }
    keccak::f1600(a);
  }
#pragma unroll
  for (int w = 0; w < rem; w++) {
    const uint64_t x = c1[17 * full + w];
    if (c2) diff |= x ^ c2[17 * full + w];
    a[w] ^= x;
  }
  a[rem] ^= 0x06;
  a[16] ^= 0x8000000000000000ull;
  keccak::f1600(a);
  uint64_t hc[4];
#pragma unroll
  for (int j = 0; j < 4; j++) hc[j] = a[j];
  const uint64_t* kb = (diff != 0) ? reinterpret_cast<const uint64_t*>(z + i * z_stride)
                                   : reinterpret_cast<const uint64_t*>(kbar + 32 * i);
  keccak::zero(a);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    a[j] = kb[j];
    a[4 + j] = hc[j];
  }
  a[8] = 0x1f;
  a[16] = 0x8000000000000000ull;  // SHAKE256
  keccak::f1600(a);
#pragma unroll
  for (int j = 0; j < 4; j++) reinterpret_cast<uint64_t*>(ss + 32 * i)[j] = a[j];
}

// mode 0: encaps (in = seeds, key = ek), mode 1: decaps (in = ct, key = dk); per-op keys
template <int K>
static int r3_device(int decaps, const uint8_t* key, size_t key_stride, const uint8_t* in, uint8_t* ct_out, uint8_t* ss, size_t n,
                     cudaStream_t st, int slot) {
  using P = Params<K>;
  Dev& c = ctx();
  const size_t sub = sub_batch(n);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t o_h = take(n * 32), o_r = take(n * 32), o_m = take(n * 32), o_k = take(n * 32),
               o_ct2 = take(decaps ? n * (size_t)P::ct_bytes : 0);
  size_t o_A[2];
  for (int q = 0; q < 2; q++) o_A[q] = take(sub * K * K * 512);
  void* basev = nullptr;
  int rc = ensure_work(slot, off, &basev);
  if (rc) return rc;
  char* b = (char*)basev;
  uint64_t* h = (uint64_t*)(b + o_h);
  uint64_t* r = (uint64_t*)(b + o_r);
  uint8_t* m = (uint8_t*)(b + o_m);
  uint8_t* kbar = (uint8_t*)(b + o_k);
  if (int arc = ensure_smem_attr((const void*)sample_kernel<K>, kSampleSmem)) return arc;
  const kyber::TwPair* tw = (const kyber::TwPair*)c.kyber_tw;
  if (!decaps) {
    {
      KernelScope ks(KID_MLKEM_G, st);
      r3_m_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(in, n, m);
    }
    {
      KernelScope ks(KID_MLKEM_HASH_EK, st);
      hash_ek_kernel<K><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(key, key_stride, n, h);
    }
    rc = encrypt_lenient<K>(key, key_stride, (const uint8_t*)h, 32, m, ct_out, kbar, r, b, o_A, n, st, slot);
    if (rc) return rc;
    KernelScope ks(KID_MLKEM_G, st);
    r3_kdf_kernel<K><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(ct_out, nullptr, kbar, nullptr, 0, n, ss);
  } else {
    uint8_t* ct2 = (uint8_t*)(b + o_ct2);
    const uint8_t* ek = key + 384 * K;
    if (int drc = launch_dp<K>(decrypt_dp_kernel<K, kDpThreads, kDpMinBlocks<K>>, n, st, key, key_stride, in, n, m, tw))
      return drc;
    rc = encrypt_lenient<K>(ek, key_stride, key + 384 * K + P::ek_bytes, key_stride, m, ct2, kbar, r, b, o_A, n, st, slot);
    if (rc) return rc;
    KernelScope ks(KID_MLKEM_G, st);
    r3_kdf_kernel<K><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(in, ct2, kbar, key + 384 * K + P::ek_bytes + 32, key_stride,
                                                                  n, ss);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------ host side
// push_ct / push_ss (optional): where the rows of this call belong in a gather destination -- rank 0's buffer mapped
// through CUDA IPC, or local memory.  Every sub-batch is copied there as soon as its encrypt kernel has run, by the copy
// engines on the work set's copy stream, while the next sub-batches compute: the result gather of SURVEY.md 8(e)
// overlapped inside the flow, with no SM taken from the (ALU-saturated) kernels.
template <int K>
static int encaps_device(const uint8_t* ek, size_t ek_stride, const uint8_t* seeds, uint8_t* ct, uint8_t* ss,
                         uint8_t* status, size_t n, cudaStream_t st, int slot, uint8_t* push_ct = nullptr,
                         uint8_t* push_ss = nullptr) {
  using P = Params<K>;
  Dev& c = ctx();
  WorkSet& ws = wset(slot);
  const bool shared = (ek_stride == 0);
  const size_t nkeys = shared ? 1 : n;
  const size_t sub = sub_batch(n);
  const size_t subkeys = shared ? 1 : sub;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += (bytes + 255) & ~(size_t)255;
    return o;
  };
  const size_t o_h = take(nkeys * 32), o_r = take(n * 32);
  size_t o_A[2];
  o_A[0] = take(subkeys * K * K * 512);
  o_A[1] = shared ? o_A[0] : take(subkeys * K * K * 512);
  void* base = nullptr;
  int rc = ensure_work(slot, off, &base);
  if (rc) return rc;
  uint64_t* h = (uint64_t*)((char*)base + o_h);
  uint64_t* r = (uint64_t*)((char*)base + o_r);

  if (int arc = ensure_smem_attr((const void*)sample_kernel<K>, kSampleSmem)) return arc;
  {
    KernelScope ks(KID_MLKEM_HASH_EK, st);
    hash_ek_kernel<K><<<(unsigned)((nkeys + 127) / 128), 128, 0, st>>>(ek, ek_stride, nkeys, h);
  }
  {
    KernelScope ks(KID_MLKEM_G, st);
    g_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(seeds, (const uint8_t*)h, shared ? 0 : 32, n, ss, r);
  }
  // one key: A^T is derived once, before the sub-batches fork, and a sub-batch is then a single kernel
  if (shared)
    if (int src = launch_sample<K>(slot, 0, st, ek + 384 * K, 0, 1, (int16_t*)((char*)base + o_A[0]), 1)) return src;
  const kyber::TwPair* tw = (const kyber::TwPair*)c.kyber_tw;
  rc = for_sub_batches(ws, n, st, [&](size_t first, size_t cnt, int l, cudaStream_t ls) {
    int16_t* A = (int16_t*)((char*)base + o_A[l]);
    if (!shared)
      if (int src = launch_sample<K>(slot, l, ls, ek + 384 * K + first * ek_stride, ek_stride, cnt, A, 1)) return src;
    if (int erc = launch_dp<K>(encrypt_dp_kernel<K, kDpThreads, kDpMinBlocks<K>>, cnt, ls,
                               ek + (shared ? 0 : first * ek_stride), ek_stride, A, shared ? 1 : 0,
                               (const uint64_t*)(r + 4 * first), seeds + 32 * first, cnt, ct + first * P::ct_bytes,
                               ss + 32 * first, status ? status + first : nullptr, tw, 0))
      return erc;
    if (push_ct || push_ss) {
      CB200_CUDA(cudaEventRecord(ws.ev_copy, ls));
      CB200_CUDA(cudaStreamWaitEvent(ws.copy, ws.ev_copy, 0));
      if (push_ct)
        CB200_CUDA(cudaMemcpyAsync(push_ct + first * P::ct_bytes, ct + first * P::ct_bytes, cnt * (size_t)P::ct_bytes,
                                   cudaMemcpyDefault, ws.copy));
      if (push_ss) CB200_CUDA(cudaMemcpyAsync(push_ss + 32 * first, ss + 32 * first, cnt * 32, cudaMemcpyDefault, ws.copy));
    }
    return 0;
  });
  if (rc) return rc;
  if (push_ct || push_ss) {  // the caller's stream covers the pushes too
    CB200_CUDA(cudaEventRecord(ws.ev_copy, ws.copy));
    CB200_CUDA(cudaStreamWaitEvent(st, ws.ev_copy, 0));
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

static int encaps_any(int k, const uint8_t* ek, size_t ek_stride, const uint8_t* seeds, uint8_t* ct, uint8_t* ss,
                      uint8_t* status, size_t n, cudaStream_t st, int slot, uint8_t* push_ct = nullptr,
                      uint8_t* push_ss = nullptr) {
  return k == 2   ? encaps_device<2>(ek, ek_stride, seeds, ct, ss, status, n, st, slot, push_ct, push_ss)
         : k == 3 ? encaps_device<3>(ek, ek_stride, seeds, ct, ss, status, n, st, slot, push_ct, push_ss)
                  : encaps_device<4>(ek, ek_stride, seeds, ct, ss, status, n, st, slot, push_ct, push_ss);
}

// ------------------------------------------------------------------ 7. the sampler and serialisation surface on its own
// (*Poly).DeriveUniform (sample.go:192-236) for n independent (seed, x, y): the stream of sample_kernel
__global__ void __launch_bounds__(kSampleThreads) derive_uniform_kernel(const uint8_t* __restrict__ seeds,
                                                                        size_t seed_stride,
                                                                        const uint8_t* __restrict__ xy, size_t n,
                                                                        int16_t* __restrict__ polys) {
  extern __shared__ __align__(16) uint4 stage[];
  const int lane = threadIdx.x & 31, wbase = threadIdx.x & ~31;
  const size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x, sc = s < n ? s : n - 1;
  if (s - lane >= n) return;  // a warp with no stream of the batch
  const uint8_t* seed = seeds + sc * seed_stride;
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll
  for (int w = 0; w < 4; w++) {
    uint64_t v = 0;
#pragma unroll
    for (int b = 0; b < 8; b++) v |= (uint64_t)seed[8 * w + b] << (8 * b);
    a[w] = v;
  }
  a[4] = (uint64_t)xy[2 * sc] | ((uint64_t)xy[2 * sc + 1] << 8) | (0x1full << 16);
  a[20] = 0x8000000000000000ull;
  // polynomials relative to the warp's first, so the chunk indices stay small whatever n is
  uniform_stream(a, stage + wbase * kStageChunks, lane, reinterpret_cast<uint4*>(polys + (s - lane) * N),
                 (uint32_t)(sc - (s - lane)), s < n);
}
// (*Poly).DeriveNoise (sample.go:31-95) for n independent (seed, nonce), thread per polynomial (the K-PKE kernels
// sample theirs per octet, octet_prf)
template <int ETA>
__global__ void __launch_bounds__(128) derive_noise_kernel(const uint8_t* __restrict__ seeds, size_t seed_stride,
                                                           const uint8_t* __restrict__ nonces, size_t n,
                                                           int16_t* __restrict__ polys) {
  const size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const uint8_t* seed = seeds + s * seed_stride;
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll
  for (int w = 0; w < 4; w++) {
    uint64_t v = 0;
#pragma unroll
    for (int b = 0; b < 8; b++) v |= (uint64_t)seed[8 * w + b] << (8 * b);
    a[w] = v;
  }
  a[4] = (uint64_t)nonces[s] | (0x1full << 8);
  a[16] = 0x8000000000000000ull;
  noise_stream<ETA>(a, polys + s * N);
}

// Pack / Unpack / CompressTo / Decompress / CompressMessageTo / DecompressMessage (poly.go:106-328): octet per
// polynomial on the C layout, the same lane code the fused kernels use.  OP 0 = pack, 1 = unpack, 2 = compress, 3 = decompress.
template <int OP, int D>
__global__ void __launch_bounds__(128) codec_kernel(const void* __restrict__ in, void* __restrict__ out, size_t n) {
  using namespace kyber;
  const int lane = threadIdx.x & 31, v = lane & 7;
  const size_t p = (size_t)blockIdx.x * 16 + (threadIdx.x >> 3);
  if (p >= n) return;
  constexpr int bytes = (D == 12) ? 384 : 32 * D;
  int32_t r[32];
  if (OP == 0 || OP == 2) {
    gload_C(reinterpret_cast<const uint32_t*>(in) + p * (N / 2), v, r);
    uint32_t* dst = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(out) + p * bytes);
    if (OP == 0) {
      uint32_t w[12];
      pack12_C(r, w);
#pragma unroll
      for (int i = 0; i < 12; i++) dst[12 * v + i] = w[i];
    } else if (D == 1) {  // CompressMessageTo, poly.go:150-166: bit i of m <- coefficient i = 32 v + i
      uint32_t word = 0;
#pragma unroll
      for (int i = 0; i < 32; i++) {
        int32_t x = (1664 << 16) - r[i];
        x = (x >> 31) ^ x;
        x &= 0xffff0000;
        x -= (832 << 16);
        word |= ((uint32_t)x >> 31) << i;
      }
      dst[v] = word;
    } else {
      compress_store_C<(D == 12 || D == 1) ? 4 : D>(r, dst + v * D);
    }
  } else {
    const uint8_t* src = reinterpret_cast<const uint8_t*>(in) + p * bytes;
    if (OP == 1) {
      unpack12_C(src + 48 * v, r);
    } else if (D == 1) {  // DecompressMessage, poly.go:134-147
      const uint32_t word = reinterpret_cast<const uint32_t*>(src)[v];
#pragma unroll
      for (int i = 0; i < 32; i++) r[i] = ((word >> i) & 1) ? ((Q + 1) / 2) << 16 : 0;
    } else {
      decompress_C<(D == 12 || D == 1) ? 4 : D>(reinterpret_cast<const uint32_t*>(src) + v * D, r);
    }
    gstore_C(reinterpret_cast<uint32_t*>(out) + p * (N / 2), v, r);
  }
}
template <int OP>
static int launch_codec(int d, const void* in, void* out, size_t n, cudaStream_t st) {
  KernelScope ks(KID_KYBER_EW, st);
  const unsigned grid = (unsigned)((n + 15) / 16);
  switch (d) {
    case 1: codec_kernel<OP, 1><<<grid, 128, 0, st>>>(in, out, n); break;
    case 4: codec_kernel<OP, 4><<<grid, 128, 0, st>>>(in, out, n); break;
    case 5: codec_kernel<OP, 5><<<grid, 128, 0, st>>>(in, out, n); break;
    case 10: codec_kernel<OP, 10><<<grid, 128, 0, st>>>(in, out, n); break;
    case 11: codec_kernel<OP, 11><<<grid, 128, 0, st>>>(in, out, n); break;
    default: codec_kernel<OP, 12><<<grid, 128, 0, st>>>(in, out, n); break;
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}
int launch_kyber_codec(int op, int d, const void* in, void* out, size_t n, cudaStream_t st) {
  switch (op) {
    case 0: return launch_codec<0>(12, in, out, n, st);
    case 1: return launch_codec<1>(12, in, out, n, st);
    case 2: return launch_codec<2>(d, in, out, n, st);
    default: return launch_codec<3>(d, in, out, n, st);
  }
}
int launch_derive_uniform(const uint8_t* seeds, size_t seed_stride, const uint8_t* xy, int16_t* polys, size_t n,
                          cudaStream_t st) {
  if (int arc = ensure_smem_attr((const void*)derive_uniform_kernel, kSampleSmem)) return arc;
  KernelScope ks(KID_SAMPLER, st);
  derive_uniform_kernel<<<(unsigned)((n + kSampleThreads - 1) / kSampleThreads), kSampleThreads, kSampleSmem, st>>>(
      seeds, seed_stride, xy, n, polys);
  CB200_CUDA(cudaGetLastError());
  return 0;
}
int launch_derive_noise(int eta, const uint8_t* seeds, size_t seed_stride, const uint8_t* nonces, int16_t* polys, size_t n,
                        cudaStream_t st) {
  KernelScope ks(KID_SAMPLER, st);
  if (eta == 3)
    derive_noise_kernel<3><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(seeds, seed_stride, nonces, n, polys);
  else
    derive_noise_kernel<2><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(seeds, seed_stride, nonces, n, polys);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// dst[i] = src for i < n: one packed key made per-op for the flows that index keys by operation
__global__ void __launch_bounds__(256) replicate_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int words,
                                                        size_t n) {
  const size_t total = n * (size_t)words;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
    dst[i] = __ldg(src + (i % words));
}
int replicate_rows(const uint8_t* src, uint8_t* dst, size_t width, size_t n, cudaStream_t st) {
  KernelScope ks(KID_HYBRID_GLUE, st);
  const size_t total = n * (width / 16);
  replicate_kernel<<<(unsigned)std::min<size_t>((total + 255) / 256, (size_t)ctx().sm_count * 8), 256, 0, st>>>(
      (const uint4*)src, (uint4*)dst, (int)(width / 16), n);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// ---- entry points for hybrid.cu (mlkem_internal.h)
int dev_keygen(int k, int mlkem, const uint8_t* seeds, uint8_t* ek, uint8_t* dk, size_t n, cudaStream_t st, int slot) {
  return k == 2   ? keygen_device<2>(seeds, ek, dk, n, st, slot, mlkem)
         : k == 3 ? keygen_device<3>(seeds, ek, dk, n, st, slot, mlkem)
                  : keygen_device<4>(seeds, ek, dk, n, st, slot, mlkem);
}
int dev_encaps(int k, int mlkem, const uint8_t* ek, size_t ek_stride, const uint8_t* seeds, uint8_t* ct, uint8_t* ss,
               uint8_t* status, size_t n, cudaStream_t st, int slot) {
  if (mlkem) return encaps_any(k, ek, ek_stride, seeds, ct, ss, status, n, st, slot);
  return k == 2   ? r3_device<2>(0, ek, ek_stride, seeds, ct, ss, n, st, slot)
         : k == 3 ? r3_device<3>(0, ek, ek_stride, seeds, ct, ss, n, st, slot)
                  : r3_device<4>(0, ek, ek_stride, seeds, ct, ss, n, st, slot);
}
int dev_decaps(int k, int mlkem, const uint8_t* dk, size_t dk_stride, const uint8_t* ct, uint8_t* ss, uint8_t* status, size_t n,
               cudaStream_t st, int slot) {
  if (mlkem)
    return k == 2   ? decaps_device<2>(dk, dk_stride, ct, ss, status, n, st, slot)
           : k == 3 ? decaps_device<3>(dk, dk_stride, ct, ss, status, n, st, slot)
                    : decaps_device<4>(dk, dk_stride, ct, ss, status, n, st, slot);
  return k == 2   ? r3_device<2>(1, dk, dk_stride, ct, nullptr, ss, n, st, slot)
         : k == 3 ? r3_device<3>(1, dk, dk_stride, ct, nullptr, ss, n, st, slot)
                  : r3_device<4>(1, dk, dk_stride, ct, nullptr, ss, n, st, slot);
}

}  // namespace mlkem
}  // namespace cb200

using namespace cb200;

namespace {

// Error text of a batch whose per-op status bytes had bits set (host-pointer calls)
int status_error(const char* fn, size_t bit0, size_t bit1, size_t n) {
  if (bit0) {
    set_error("%s: %zu of %zu encapsulation keys are not canonical (kem.ErrPubKey)", fn, bit0, n);
    return CB200_ERR_PUBKEY;
  }
  if (bit1) {
    set_error("%s: H(ek) stored in %zu of %zu private keys does not match (kem.ErrPrivKey)", fn, bit1, n);
    return CB200_ERR_PRIVKEY;
  }
  return 0;
}

}  // namespace

extern "C" {

static int keygen_entry(const char* fn, int mlkem_flag, int k, const uint8_t* seeds, uint8_t* ek, uint8_t* dk, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (k < 2 || k > 4) {
    set_error("%s: k must be 2, 3 or 4 (ML-KEM-512/768/1024 or Kyber512/768/1024), got %d", fn, k);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  if (!seeds || !ek || !dk) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  const size_t eksz = cb200_mlkem_public_key_size(k), dksz = 768u * k + 96;
  Batch b{fn, n, ek, 1u << 15, 1u << 13, {{seeds, 64, 64, kIn}, {ek, eksz, eksz, kOut}, {dk, dksz, dksz, kOut}},
          {{!aligned({seeds, ek, dk}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return mlkem::dev_keygen(k, mlkem_flag, r[0].p, r[1].p, r[2].p, cnt, st, slot);
  });
}

int cb200_mlkem_keygen(int k, const uint8_t* seeds, uint8_t* ek, uint8_t* dk, size_t n) {
  return keygen_entry("cb200_mlkem_keygen", 1, k, seeds, ek, dk, n);
}

// ---- round-3 Kyber512/768/1024 KEM (kem/kyber): same sizes as ML-KEM-512/768/1024
int cb200_kyber_kem_keygen(int k, const uint8_t* seeds, uint8_t* ek, uint8_t* dk, size_t n) {
  return keygen_entry("cb200_kyber_kem_keygen", 0, k, seeds, ek, dk, n);
}

static int kyber_kem_run(int decaps, int k, const uint8_t* key, size_t key_stride, const uint8_t* in, uint8_t* ct, uint8_t* ss,
                         size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  const char* fn = decaps ? "cb200_kyber_kem_decaps" : "cb200_kyber_kem_encaps";
  if (k < 2 || k > 4) {
    set_error("%s: k must be 2, 3 or 4 (Kyber512/768/1024), got %d", fn, k);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const size_t keysz = decaps ? 768u * k + 96 : cb200_mlkem_public_key_size(k), ctsz = cb200_mlkem_ciphertext_size(k);
  if (!key || !in || !ss || (!decaps && !ct) || (key_stride != 0 && key_stride < keysz)) {
    set_error("%s: bad argument", fn);
    return CB200_ERR_ARG;
  }
  const size_t insz = decaps ? ctsz : (size_t)32;
  Batch b{fn, n, ss, 1u << 15, 1u << 13,
          {{key, keysz, key_stride, kIn}, {in, insz, insz, kIn}, {ss, 32, 32, kOut}, {ct, ctsz, ctsz, kOut}},
          {{!aligned({key, in, ct, ss}, {key_stride}, 16), "%s: device buffers and the key stride must be 16-byte aligned"},
           {key_stride == 0 && decaps, "%s: a shared dk needs host pointers (the device path expects one dk per op)"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return k == 2   ? mlkem::r3_device<2>(decaps, r[0].p, r[0].stride, r[1].p, r[3].p, r[2].p, cnt, st, slot)
           : k == 3 ? mlkem::r3_device<3>(decaps, r[0].p, r[0].stride, r[1].p, r[3].p, r[2].p, cnt, st, slot)
                    : mlkem::r3_device<4>(decaps, r[0].p, r[0].stride, r[1].p, r[3].p, r[2].p, cnt, st, slot);
  });
}
int cb200_kyber_kem_encaps(int k, const uint8_t* ek, size_t ek_stride, const uint8_t* seeds, uint8_t* ct, uint8_t* ss,
                           size_t n) {
  return kyber_kem_run(0, k, ek, ek_stride, seeds, ct, ss, n);
}
int cb200_kyber_kem_decaps(int k, const uint8_t* dk, size_t dk_stride, const uint8_t* ct, uint8_t* ss, size_t n) {
  return kyber_kem_run(1, k, dk, dk_stride, ct, nullptr, ss, n);
}

size_t cb200_mlkem_private_key_size(int k) { return (k >= 2 && k <= 4) ? 768u * k + 96 : 0; }

int cb200_mlkem_decaps(int k, const uint8_t* dk, size_t dk_stride, const uint8_t* ct, uint8_t* ss, uint8_t* status,
                       size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (k < 2 || k > 4) {
    set_error("cb200_mlkem_decaps: k must be 2, 3 or 4 (ML-KEM-512/768/1024), got %d", k);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const size_t dksz = cb200_mlkem_private_key_size(k), ctsz = cb200_mlkem_ciphertext_size(k);
  if (!dk || !ct || !ss || (dk_stride != 0 && dk_stride < dksz)) {
    set_error("cb200_mlkem_decaps: bad argument");
    return CB200_ERR_ARG;
  }
  // a shared dk is replicated per op on the device inside each staged chunk (the decapsulation pipeline is per-op)
  Batch b{"cb200_mlkem_decaps", n, ss, 1u << 15, 1u << 13,
          {{dk, dksz, dk_stride, kIn}, {ct, ctsz, ctsz, kIn}, {ss, 32, 32, kOut}, {status, 1, 1, kStatus},
           {nullptr, dk_stride ? 0 : dksz, dksz, kScratch}},  // per-op replicas of a shared dk (host path only)
          {{!aligned({dk, ct, ss}, {dk_stride}, 16), "%s: device buffers and dk_stride must be 16-byte aligned"},
           {dk_stride == 0, "%s: a shared dk needs host pointers (device path expects one dk per op)"}}};
  Counts c;
  rc = run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    const uint8_t* keys = r[0].p;
    size_t stride = r[0].stride;
    if (r[4].p) {
      int e = mlkem::replicate_rows(r[0].p, r[4].p, dksz, cnt, st);
      if (e) return e;
      keys = r[4].p;
      stride = dksz;
    }
    return mlkem::dev_decaps(k, 1, keys, stride, r[1].p, r[2].p, r[3].p, cnt, st, slot);
  }, &c);
  if (rc) return rc;
  return status_error("cb200_mlkem_decaps", 0, c.bit1, n);
}

size_t cb200_mlkem_public_key_size(int k) { return (k >= 2 && k <= 4) ? 384u * k + 32 : 0; }
size_t cb200_mlkem_ciphertext_size(int k) { return k == 3 ? 1088 : k == 4 ? 1568 : k == 2 ? 768 : 0; }

static int mlkem_encaps_entry(int k, const uint8_t* ek, size_t ek_stride, const uint8_t* seeds, uint8_t* ct, uint8_t* ss,
                              uint8_t* status, size_t n, uint8_t* push_ct, uint8_t* push_ss);
int cb200_mlkem_encaps(int k, const uint8_t* ek, size_t ek_stride, const uint8_t* seeds, uint8_t* ct, uint8_t* ss,
                       uint8_t* status, size_t n) {
  return mlkem_encaps_entry(k, ek, ek_stride, seeds, ct, ss, status, n, nullptr, nullptr);
}
int cb200_mlkem_encaps_push(int k, const uint8_t* ek, size_t ek_stride, const uint8_t* seeds, uint8_t* ct, uint8_t* ss,
                            uint8_t* status, size_t n, uint8_t* push_ct, uint8_t* push_ss) {
  if (!is_device_ptr(ct)) {
    set_error("cb200_mlkem_encaps_push: device pointers only (host-pointer calls already end in the caller's buffers)");
    return CB200_ERR_ARG;
  }
  return mlkem_encaps_entry(k, ek, ek_stride, seeds, ct, ss, status, n, push_ct, push_ss);
}
static int mlkem_encaps_entry(int k, const uint8_t* ek, size_t ek_stride, const uint8_t* seeds, uint8_t* ct, uint8_t* ss,
                              uint8_t* status, size_t n, uint8_t* push_ct, uint8_t* push_ss) {
  int rc = require_ready();
  if (rc) return rc;
  if (k < 2 || k > 4) {
    set_error("cb200_mlkem_encaps: k must be 2, 3 or 4 (ML-KEM-512/768/1024), got %d", k);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const size_t eksz = cb200_mlkem_public_key_size(k), ctsz = cb200_mlkem_ciphertext_size(k);
  if (!ek || !seeds || !ct || !ss || (ek_stride != 0 && ek_stride < eksz)) {
    set_error("cb200_mlkem_encaps: bad argument");
    return CB200_ERR_ARG;
  }
  // host pointers: one contiguous index range per GPU, each staged through HBM in chunks on three streams
  // (H2D | kernels | D2H overlap); the per-op status always comes back (it carries kem.ErrPubKey).  With device
  // pointers the caller reads status asynchronously.
  Batch b{"cb200_mlkem_encaps", n, ct, 1u << 16, 1u << 13,
          {{ek, eksz, ek_stride, kIn}, {seeds, 32, 32, kIn}, {ct, ctsz, ctsz, kOut}, {ss, 32, 32, kOut}, {status, 1, 1, kStatus}},
          {{!aligned({ek, seeds, ct, ss}, {ek_stride}, 16), "%s: device buffers and ek_stride must be 16-byte aligned"}}};
  Counts c;
  rc = run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) {
    return mlkem::encaps_any(k, r[0].p, r[0].stride, r[1].p, r[2].p, r[3].p, r[4].p, cnt, st, slot, push_ct, push_ss);
  }, &c);
  if (rc) return rc;
  return status_error("cb200_mlkem_encaps", c.bit0, 0, n);
}

int cb200_kyber_derive_uniform(int16_t* polys, const uint8_t* seeds, size_t seed_stride, const uint8_t* xy, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!polys || !seeds || !xy || (seed_stride != 0 && seed_stride < 32)) {
    set_error("cb200_kyber_derive_uniform: bad argument");
    return CB200_ERR_ARG;
  }
  Batch b{"cb200_kyber_derive_uniform", n, polys, 1u << 16, 1u << 14,
          {{seeds, 32, seed_stride, kIn}, {xy, 2, 2, kIn}, {polys, 512, 512, kOut}},
          {{!aligned({polys}, {}, 16), "%s: device polynomials must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return mlkem::launch_derive_uniform(r[0].p, r[0].stride, r[1].p, (int16_t*)r[2].p, cnt, st);
  });
}

int cb200_kyber_derive_noise(int16_t* polys, int eta, const uint8_t* seeds, size_t seed_stride, const uint8_t* nonces,
                             size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (eta != 2 && eta != 3) {
    set_error("cb200_kyber_derive_noise: eta must be 2 or 3, got %d", eta);  // sample.go:19-28 panics likewise
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  if (!polys || !seeds || !nonces || (seed_stride != 0 && seed_stride < 32)) {
    set_error("cb200_kyber_derive_noise: bad argument");
    return CB200_ERR_ARG;
  }
  Batch b{"cb200_kyber_derive_noise", n, polys, 1u << 16, 1u << 14,
          {{seeds, 32, seed_stride, kIn}, {nonces, 1, 1, kIn}, {polys, 512, 512, kOut}},
          {{!aligned({polys}, {}, 16), "%s: device polynomials must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return mlkem::launch_derive_noise(eta, r[0].p, r[0].stride, r[1].p, (int16_t*)r[2].p, cnt, st);
  });
}

// op 0 pack, 1 unpack, 2 compress, 3 decompress; polys is the int16 side, bytes the packed side
static int codec_entry(const char* fn, int op, int d, const void* in, void* out, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (op >= 2 && d != 1 && d != 4 && d != 5 && d != 10 && d != 11) {
    set_error("%s: d must be 1, 4, 5, 10 or 11, got %d", fn, d);  // poly.go:176,258 panic on other sizes
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  if (!in || !out) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  const size_t bytes = op < 2 ? 384 : 32 * (size_t)d;
  const size_t in_unit = (op == 0 || op == 2) ? 512 : bytes, out_unit = (op == 0 || op == 2) ? bytes : 512;
  Batch b{fn, n, out, 1u << 17, 1u << 15, {{in, in_unit, in_unit, kIn}, {out, out_unit, out_unit, kOut}},
          {{!aligned({in, out}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return mlkem::launch_kyber_codec(op, d, r[0].p, r[1].p, cnt, st);
  });
}
int cb200_kyber_pack(uint8_t* out, const int16_t* polys, size_t n) { return codec_entry("cb200_kyber_pack", 0, 12, polys, out, n); }
int cb200_kyber_unpack(int16_t* polys, const uint8_t* in, size_t n) { return codec_entry("cb200_kyber_unpack", 1, 12, in, polys, n); }
int cb200_kyber_compress(uint8_t* out, const int16_t* polys, int d, size_t n) {
  return codec_entry("cb200_kyber_compress", 2, d, polys, out, n);
}
int cb200_kyber_decompress(int16_t* polys, const uint8_t* in, int d, size_t n) {
  return codec_entry("cb200_kyber_decompress", 3, d, in, polys, n);
}

}  // extern "C"
