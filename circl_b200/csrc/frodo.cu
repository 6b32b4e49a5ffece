// FrodoKEM-640-SHAKE (kem/frodo/frodo640shake) batched on the device:
//   frodo.go:84-135    newKeyFromSeed        -> frodo_keygen_seed_kernel, frodo_keygen_a_kernel, frodo_hash_kernel
//   frodo.go:160-240   EncapsulateTo         -> frodo_hash_kernel (H(pk)), frodo_se_kernel (G2, S'/E'/E''),
//                                             S'A + E' (below), frodo_tail_kernel (C), frodo_hash_kernel (F)
//   frodo.go:247-329   DecapsulateTo         -> frodo_decode_kernel (mu'), then as EncapsulateTo, with the compare and
//                                             the masked selection of k' or s in the product kernels and the tail
// S'A + E' has two paths:
//   * per-op keys: A is expanded and consumed on chip (frodo_sa_kernel, one CTA per op), never written to memory;
//   * one key for the batch (stride 0): A is expanded once per call into the work area (frodo_expand_a_kernel) and
//     S'A runs for the whole batch as one int8 tensor-core GEMM (frodo_gemm_kernel, mma.sync m16n8k32 s8 x u8).
// Every sum is exact mod 2^16, so the order of summation does not matter and both paths give the same bytes.
// Profiling classes: KID_FRODO for every kernel but the GEMM, KID_FRODO_GEMM for the GEMM.
#include <cstring>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "frodo.cuh"
#include "keccak.cuh"

namespace cb200 {
namespace frodo {

// Per-op work row (bytes): the sampled stream as int8 (KeyGen: S^T | E; Encaps/Decaps: S' | E' | E''), k (then the
// selected k' or s), mu', the compare flag and H(pk).  Every sampled value is in [-12, 12].
constexpr int kStream = 2 * kN * kNbar + kNbar * kNbar;  // 10304
constexpr int kOffSp = 0, kOffEp = kN * kNbar, kOffEpp = 2 * kN * kNbar;
constexpr int kOffK = kStream, kOffMu = kOffK + 16, kOffFlag = kOffMu + 16, kOffHpk = kOffFlag + 16;
constexpr size_t kWork = kOffHpk + 16;  // 10368 bytes per op
// the shared-key path: A^T as two byte planes (lo, hi) of 640 x 640, once per call
constexpr size_t kPlane = (size_t)kN * kN;
constexpr size_t kShared = 2 * kPlane;
// operations per device sub-batch: bounds the work area of a device-pointer call to kChunk * kWork bytes
constexpr size_t kChunk = 1u << 13;
// operations per staged chunk of a host-pointer call: at most 29.6 KB of rows per op (Decaps: sk, ct, ss), so about
// 121 MB of staging per pipeline slot, the size of the existing entry points' chunks
constexpr size_t kHostChunk = 1u << 12;

using keccak::f1600;

__device__ __forceinline__ uint64_t ld64(const uint8_t* p) { return *reinterpret_cast<const uint64_t*>(p); }

// SHAKE128 absorbing one short message given as 64-bit lanes (nbytes <= 160), with the 0x1F / 0x80 padding
__device__ __forceinline__ void pad_shake128(uint64_t (&a)[25], int nbytes) {
  a[nbytes >> 3] ^= (uint64_t)0x1F << (8 * (nbytes & 7));
  a[20] ^= (uint64_t)0x80 << 56;
}

// state of SHAKE128(byte || 16-byte seed), the seed given as two little-endian lanes
__device__ __forceinline__ void absorb_prefixed(uint64_t (&a)[25], uint8_t prefix, uint64_t w0, uint64_t w1) {
  keccak::zero(a);
  a[0] = prefix | (w0 << 8);
  a[1] = (w0 >> 56) | (w1 << 8);
  a[2] = w1 >> 56;
  pad_shake128(a, 17);
}

// Squeezes `ncoef` (a multiple of 4) coefficients from an absorbed sponge, samples them and stores them as int8 to a
// 4-byte aligned row: the stream is read exactly as the reference's byte stream of little-endian uint16.
__device__ void squeeze_sample_s8(uint64_t (&a)[25], uint8_t* out, int ncoef) {
  uint32_t* o = reinterpret_cast<uint32_t*>(out);
#pragma unroll 1
  for (int b = 0; b * kPerBlock < ncoef; b++) {
    f1600(a);
#pragma unroll
    for (int l = 0; l < 21; l++) {
      if (b * kPerBlock + 4 * l < ncoef) {
        uint32_t w = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) w |= (uint32_t)(sample((uint16_t)(a[l] >> (16 * q))) & 0xFF) << (8 * q);
        o[b * 21 + l] = w;
      }
    }
  }
}

// State of A's row i: SHAKE128(uint16_le(i) || seedA) (matrix_shake.go:13-19).  s0..s2 are the seed's lanes shifted
// by the two index bytes, computed once by the caller.
__device__ __forceinline__ void absorb_row(uint64_t (&a)[25], int i, uint64_t s0, uint64_t s1, uint64_t s2) {
  keccak::zero(a);
  a[0] = (uint64_t)i | s0;
  a[1] = s1;
  a[2] = s2;
  pad_shake128(a, 18);
}
__device__ __forceinline__ void seed_lanes(const uint8_t* seedA, uint64_t* s0, uint64_t* s1, uint64_t* s2) {
  const uint64_t w0 = ld64(seedA), w1 = ld64(seedA + 8);
  *s0 = w0 << 16;
  *s1 = (w0 >> 48) | (w1 << 16);
  *s2 = w1 >> 48;
}

// ------------------------------------------------------------------ thread-per-op sponge kernels
// KeyGen's seeds (frodo.go:97-118): seedA = SHAKE128(z)[:16] to pk and sk, s to sk, and SHAKE128(0x5F || seedSE)
// sampled into S^T | E (int8) in the work row.  seed = s || seedSE || z.
__global__ void __launch_bounds__(128) frodo_keygen_seed_kernel(const uint8_t* __restrict__ seeds, uint8_t* __restrict__ pk,
                                                                uint8_t* __restrict__ sk, uint8_t* __restrict__ W, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* seed = seeds + i * kSeed;
  uint8_t* p = pk + i * kPk;
  uint8_t* s = sk + i * kSk;
  uint64_t a[25];
  keccak::zero(a);
  a[0] = ld64(seed + 32);
  a[1] = ld64(seed + 40);
  pad_shake128(a, 16);
  f1600(a);
  // pk, sk and the seeds are 8-byte aligned (their sizes are multiples of 8)
  reinterpret_cast<uint64_t*>(p)[0] = a[0];
  reinterpret_cast<uint64_t*>(p)[1] = a[1];
  reinterpret_cast<uint64_t*>(s + kSkPk)[0] = a[0];
  reinterpret_cast<uint64_t*>(s + kSkPk)[1] = a[1];
  reinterpret_cast<uint64_t*>(s)[0] = ld64(seed);
  reinterpret_cast<uint64_t*>(s)[1] = ld64(seed + 8);
  absorb_prefixed(a, 0x5F, ld64(seed + 16), ld64(seed + 24));
  squeeze_sample_s8(a, W + i * kWork, 2 * kN * kNbar);
}

// out[i] = SHAKE128(m[i][0:L] || t[i][0:16] (if T)) [0:16]: H(pk) (L = 9616) and F(ct || k) (L = 9720, T).  Rows are
// 8-byte aligned; a stride of 0 reads one row for the whole batch.
template <int L, bool T>
__global__ void __launch_bounds__(128) frodo_hash_kernel(const uint8_t* __restrict__ m, size_t ms,
                                                         const uint8_t* __restrict__ t, size_t ts,
                                                         uint8_t* __restrict__ out, size_t os, size_t n) {
  constexpr int kWords = L / 8 + (T ? 2 : 0), kBytes = 8 * kWords;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* row = m + i * ms;
  const uint8_t* tail = T ? t + i * ts : nullptr;
  uint64_t a[25];
  keccak::zero(a);
#pragma unroll 1
  for (int b = 0; b * 21 < kWords; b++) {
#pragma unroll
    for (int l = 0; l < 21; l++) {
      const int w = b * 21 + l;
      if (w < L / 8)
        a[l] ^= ld64(row + 8 * w);
      else if (T && w < kWords)
        a[l] ^= ld64(tail + 8 * (w - L / 8));
    }
    if ((b + 1) * 21 <= kWords) f1600(a);  // a full block; the last, partial one is padded below
  }
  // kBytes % 168 != 0 for both messages (9616 and 9736), so the padding falls in the block absorbed last
  static_assert(kBytes % 168 != 0, "padding block");
  a[(kBytes % 168) >> 3] ^= (uint64_t)0x1F << (8 * (kBytes & 7));
  a[20] ^= (uint64_t)0x80 << 56;
  f1600(a);
  reinterpret_cast<uint64_t*>(out + i * os)[0] = a[0];
  reinterpret_cast<uint64_t*>(out + i * os)[1] = a[1];
}

// Encaps / Decaps (frodo.go:204-220, 283-298): seedSE || k = SHAKE128(hpk || mu) (k to the work row), then
// SHAKE128(0x96 || seedSE) sampled into S' | E' | E'' (int8).  Clears the compare flag.
__global__ void __launch_bounds__(128) frodo_se_kernel(const uint8_t* __restrict__ hpk, size_t hs,
                                                       const uint8_t* __restrict__ mu, size_t mus,
                                                       uint8_t* __restrict__ W, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t* w = W + i * kWork;
  uint64_t a[25];
  keccak::zero(a);
  a[0] = ld64(hpk + i * hs);
  a[1] = ld64(hpk + i * hs + 8);
  a[2] = ld64(mu + i * mus);
  a[3] = ld64(mu + i * mus + 8);
  pad_shake128(a, 32);
  f1600(a);
  const uint64_t se0 = a[0], se1 = a[1];
  reinterpret_cast<uint64_t*>(w + kOffK)[0] = a[2];
  reinterpret_cast<uint64_t*>(w + kOffK)[1] = a[3];
  reinterpret_cast<uint32_t*>(w + kOffFlag)[0] = 0;
  absorb_prefixed(a, 0x96, se0, se1);
  squeeze_sample_s8(a, w, kStream);
}

// ------------------------------------------------------------------ KeyGen: B = A S + E, row-local
// One CTA of 128 threads per (op, 128 rows).  The thread that squeezes row i accumulates its 8 outputs against S held
// in shared memory as [j][k] (mulAddASPlusE, matrix_shake.go:29-41); the 8 outputs pack to pk[16 + 15 i].  The CTA
// of the first rows also writes S^T to the private key as little-endian uint16.
__global__ void __launch_bounds__(128) frodo_keygen_a_kernel(uint8_t* __restrict__ pk, uint8_t* __restrict__ sk,
                                                             const uint8_t* __restrict__ W) {
  __shared__ __align__(16) int16_t S[kN][kNbar];
  const size_t op = blockIdx.y;
  const uint8_t* w = W + op * kWork;
  uint8_t* p = pk + op * kPk;
  uint8_t* s = sk + op * kSk;
  for (int idx = threadIdx.x; idx < kN * kNbar; idx += blockDim.x) {
    const int16_t v = (int8_t)w[kOffSp + idx];  // S^T[k][j], idx = k 640 + j
    S[idx % kN][idx / kN] = v;
    if (blockIdx.x == 0) reinterpret_cast<uint16_t*>(s + kSkS)[idx] = (uint16_t)v;
  }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // 5 x 128 = 640 rows
  uint64_t s0, s1, s2;
  seed_lanes(p, &s0, &s1, &s2);  // seedA was written by frodo_keygen_seed_kernel
  uint64_t a[25];
  absorb_row(a, i, s0, s1, s2);
  uint32_t acc[kNbar] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll 1
  for (int b = 0; b < kRowBlocks; b++) {
    f1600(a);
#pragma unroll
    for (int l = 0; l < 21; l++) {
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int j = b * kPerBlock + 4 * l + q;
        if (j < kN) {
          const uint32_t x = (uint16_t)(a[l] >> (16 * q));
          const uint4 sv = *reinterpret_cast<const uint4*>(S[j]);
          acc[0] += x * (uint32_t)(int32_t)(int16_t)(sv.x & 0xFFFF);
          acc[1] += x * (uint32_t)(int32_t)(int16_t)(sv.x >> 16);
          acc[2] += x * (uint32_t)(int32_t)(int16_t)(sv.y & 0xFFFF);
          acc[3] += x * (uint32_t)(int32_t)(int16_t)(sv.y >> 16);
          acc[4] += x * (uint32_t)(int32_t)(int16_t)(sv.z & 0xFFFF);
          acc[5] += x * (uint32_t)(int32_t)(int16_t)(sv.z >> 16);
          acc[6] += x * (uint32_t)(int32_t)(int16_t)(sv.w & 0xFFFF);
          acc[7] += x * (uint32_t)(int32_t)(int16_t)(sv.w >> 16);
        }
      }
    }
  }
  uint16_t v[8];
#pragma unroll
  for (int k = 0; k < kNbar; k++) v[k] = (uint16_t)(acc[k] + (uint32_t)(int32_t)(int8_t)w[kOffEp + i * kNbar + k]);
  uint8_t g[15];
  pack8(g, v);
#pragma unroll
  for (int b = 0; b < 15; b++) {
    p[16 + 15 * i + b] = g[b];
    s[kSkPk + 16 + 15 * i + b] = g[b];
  }
}

// ------------------------------------------------------------------ B' = S' A + E', per-op keys
// Encaps packs B' into ct[0:9600]; Decaps compares it with the ciphertext's B' and sets the op's flag.  Both take the
// packed 8 x 640 matrix as rows k of 1200 bytes, 15 bytes per 8 coefficients.
template <bool DEC>
__device__ __forceinline__ void emit_bp_group(uint8_t* ct, int k, int grp, const uint16_t (&v)[8], uint32_t* diff) {
  uint8_t* g = ct + k * (kN * kLogQ / 8) + 15 * grp;
  if (!DEC) {
    uint8_t b[15];
    pack8(b, v);
#pragma unroll
    for (int t = 0; t < 15; t++) g[t] = b[t];
  } else {
    uint16_t c[8];
    unpack8(c, g);
#pragma unroll
    for (int t = 0; t < 8; t++) *diff |= (uint32_t)((v[t] & kQMask) ^ c[t]);
  }
}

// One CTA of 128 threads per op.  Each pass, 128 threads squeeze one block (84 coefficients) of 128 rows j into
// shared memory; threads 0..83 then fold the staged block into the 8 x 640 accumulator, item (column pair, k quad).
// mulAddSAPlusE (matrix_shake.go:43-55): B'[k][i] = E'[k][i] + sum_j S'[k][j] A[j][i].
constexpr int kSaThreads = 128;
template <bool DEC>
__global__ void __launch_bounds__(kSaThreads) frodo_sa_kernel(const uint8_t* __restrict__ seedA, size_t ss_,
                                                              uint8_t* __restrict__ ct, const uint8_t* __restrict__ W) {
  __shared__ __align__(16) uint64_t stage[kSaThreads][21];  // 21.5 KB
  __shared__ __align__(16) uint16_t acc[kNbar][kN];         // 10 KB
  __shared__ __align__(16) int8_t spT[kN][kNbar];           // 5 KB: S'^T
  const size_t op = blockIdx.x;
  const int tid = threadIdx.x;
  const uint8_t* w = W + op * kWork;
  uint8_t* c = ct + op * kCt;
  for (int idx = tid; idx < kN * kNbar; idx += kSaThreads) {
    spT[idx % kN][idx / kN] = (int8_t)w[kOffSp + idx];
    acc[idx / kN][idx % kN] = (uint16_t)(int16_t)(int8_t)w[kOffEp + idx];
  }
  uint64_t s0, s1, s2;
  seed_lanes(seedA + op * ss_, &s0, &s1, &s2);
  __syncthreads();
  const int c2 = tid % 42, kq = tid / 42;  // fold item of threads 0..83
#pragma unroll 1
  for (int g = 0; g < kN / kSaThreads; g++) {
    uint64_t a[25];
    absorb_row(a, g * kSaThreads + tid, s0, s1, s2);
#pragma unroll 1
    for (int b = 0; b < kRowBlocks; b++) {
      f1600(a);
#pragma unroll
      for (int l = 0; l < 21; l++) stage[tid][l] = a[l];
      __syncthreads();
      const int col = b * kPerBlock + 2 * c2;
      if (tid < 84 && col < kN) {
        uint32_t s[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // s[2 q + h]: k = 4 kq + q, column col + h
#pragma unroll 4
        for (int t = 0; t < kSaThreads; t++) {
          const uint32_t x = reinterpret_cast<const uint32_t*>(stage[t])[c2];
          const uint32_t sv = *reinterpret_cast<const uint32_t*>(&spT[g * kSaThreads + t][4 * kq]);
          const uint32_t x0 = x & 0xFFFF, x1 = x >> 16;
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const uint32_t sq = (uint32_t)(int32_t)(int8_t)(sv >> (8 * q));
            s[2 * q] += x0 * sq;
            s[2 * q + 1] += x1 * sq;
          }
        }
#pragma unroll
        for (int q = 0; q < 4; q++) {
          acc[4 * kq + q][col] += (uint16_t)s[2 * q];
          acc[4 * kq + q][col + 1] += (uint16_t)s[2 * q + 1];
        }
      }
      __syncthreads();
    }
  }
  uint32_t diff = 0;
  for (int it = tid; it < kNbar * (kN / 8); it += kSaThreads) {
    const int k = it / (kN / 8), grp = it % (kN / 8);
    uint16_t v[8];
#pragma unroll
    for (int t = 0; t < 8; t++) v[t] = acc[k][8 * grp + t];
    emit_bp_group<DEC>(c, k, grp, v, &diff);
  }
  if (DEC) {
    const int any = __syncthreads_or(diff != 0);
    if (tid == 0) atomicOr(reinterpret_cast<uint32_t*>(const_cast<uint8_t*>(w) + kOffFlag), (uint32_t)any);
  }
}

// ------------------------------------------------------------------ B' = S' A + E', one key for the batch
// A^T as two byte planes: lo[i][j] = A[j][i] & 0xFF, hi[i][j] = A[j][i] >> 8, so that A = lo + 256 hi.  Thread j
// squeezes row j; a warp writes 32 consecutive bytes of each plane row.
__global__ void __launch_bounds__(128) frodo_expand_a_kernel(const uint8_t* __restrict__ seedA, uint8_t* __restrict__ AT) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t s0, s1, s2;
  seed_lanes(seedA, &s0, &s1, &s2);
  uint64_t a[25];
  absorb_row(a, j, s0, s1, s2);
#pragma unroll 1
  for (int b = 0; b < kRowBlocks; b++) {
    f1600(a);
#pragma unroll
    for (int l = 0; l < 21; l++)
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int i = b * kPerBlock + 4 * l + q;
        if (i < kN) {
          const uint16_t x = (uint16_t)(a[l] >> (16 * q));
          AT[(size_t)i * kN + j] = (uint8_t)x;
          AT[kPlane + (size_t)i * kN + j] = (uint8_t)(x >> 8);
        }
      }
  }
}

// S' A for the batch as one GEMM on the int8 tensor cores: M = 8 n rows (op, k) of S', K = 640, N = 640.
//   S' A = S' lo + 256 (S' hi)  (mod 2^16),  with lo, hi the byte planes of A.
// S' is freshly sampled in [-12, 12] by frodo_se_kernel, so it is exact as the s8 operand; lo and hi are u8.  Each
// int32 sum is exact: |sum| <= 640 * 255 * 12 < 2^21.  (The secret key S of Decaps' B' S comes from caller bytes and
// may hold any 16-bit value: that product stays on the CUDA cores, frodo_decode_kernel.)
// CTA tile 64 x 64, K in stages of 64, four warps of 32 x 32 (2 m16 x 4 n8 tiles x 2 planes), mma.sync m16n8k32.
constexpr int kGm = 64, kGn = 64, kGk = 64, kGpad = 80;  // row pitch 80 bytes: conflict-free 32-bit fragment loads
__device__ __forceinline__ void mma_s8u8(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <bool DEC>
__global__ void __launch_bounds__(128) frodo_gemm_kernel(const uint8_t* __restrict__ W, const uint8_t* __restrict__ AT,
                                                         uint8_t* __restrict__ ct, size_t n) {
  __shared__ __align__(16) uint8_t As[kGm][kGpad];
  __shared__ __align__(16) uint8_t Bs[2][kGn][kGpad];
  __shared__ __align__(16) uint16_t Cs[kGm][kGn + 8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  const int g = lane >> 2, t = lane & 3;
  const size_t m0 = (size_t)blockIdx.y * kGm;
  const int n0 = blockIdx.x * kGn;
  const size_t M = 8 * n;
  int acc[2][2][4][4];  // [plane][m tile][n tile][fragment]
#pragma unroll
  for (int p = 0; p < 2; p++)
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
      for (int ni = 0; ni < 4; ni++)
#pragma unroll
        for (int r = 0; r < 4; r++) acc[p][mi][ni][r] = 0;
#pragma unroll 1
  for (int k0 = 0; k0 < kN; k0 += kGk) {
    // S' rows m = 8 op + k live at W + op * kWork + k * 640 (16-byte aligned)
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const int e = tid + 128 * r, row = e >> 2, seg = e & 3;
      const size_t m = m0 + row;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (m < M) v = *reinterpret_cast<const uint4*>(W + (m >> 3) * kWork + kOffSp + (m & 7) * kN + k0 + 16 * seg);
      *reinterpret_cast<uint4*>(&As[row][16 * seg]) = v;
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int e = tid + 128 * r, p = e >> 8, row = (e >> 2) & 63, seg = e & 3;
      *reinterpret_cast<uint4*>(&Bs[p][row][16 * seg]) =
          *reinterpret_cast<const uint4*>(AT + p * kPlane + (size_t)(n0 + row) * kN + k0 + 16 * seg);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGk; kk += 32) {
      uint32_t af[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; mi++) {
        const int r0 = wm + 16 * mi + g;
        af[mi][0] = *reinterpret_cast<const uint32_t*>(&As[r0][kk + 4 * t]);
        af[mi][1] = *reinterpret_cast<const uint32_t*>(&As[r0 + 8][kk + 4 * t]);
        af[mi][2] = *reinterpret_cast<const uint32_t*>(&As[r0][kk + 16 + 4 * t]);
        af[mi][3] = *reinterpret_cast<const uint32_t*>(&As[r0 + 8][kk + 16 + 4 * t]);
      }
#pragma unroll
      for (int p = 0; p < 2; p++)
#pragma unroll
        for (int ni = 0; ni < 4; ni++) {
          const int c0 = wn + 8 * ni + g;
          const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&Bs[p][c0][kk + 4 * t]);
          const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&Bs[p][c0][kk + 16 + 4 * t]);
#pragma unroll
          for (int mi = 0; mi < 2; mi++) mma_s8u8(acc[p][mi][ni], af[mi], b0, b1);
        }
    }
    __syncthreads();
  }
  // B'[m][i] = lo + 256 hi + E'[m][i] (mod 2^16) into the tile
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int ni = 0; ni < 4; ni++)
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int row = wm + 16 * mi + g + 8 * (r >> 1), col = wn + 8 * ni + 2 * t + (r & 1);
        const size_t m = m0 + row;
        uint32_t e = 0;
        if (m < M) e = (uint32_t)(int32_t)(int8_t)W[(m >> 3) * kWork + kOffEp + (m & 7) * kN + n0 + col];
        Cs[row][col] = (uint16_t)((uint32_t)acc[0][mi][ni][r] + ((uint32_t)acc[1][mi][ni][r] << 8) + e);
      }
  __syncthreads();
  // thread -> (row tid / 2, four 8-column groups); the 16 lanes of one op's 8 rows combine their compare bits
  const int row = tid >> 1;
  const size_t m = m0 + row;
  uint32_t diff = 0;
  if (m < M) {
    uint8_t* c = ct + (m >> 3) * kCt;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int grp = 4 * (tid & 1) + q;
      uint16_t v[8];
#pragma unroll
      for (int x = 0; x < 8; x++) v[x] = Cs[row][8 * grp + x];
      emit_bp_group<DEC>(c, (int)(m & 7), n0 / 8 + grp, v, &diff);
    }
  }
  if (DEC) {
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) diff |= __shfl_xor_sync(0xffffffffu, diff, o);
    if ((lane & 15) == 0 && m < M) atomicOr(reinterpret_cast<uint32_t*>(const_cast<uint8_t*>(W) + (m >> 3) * kWork + kOffFlag),
                                            nonzero_bit(diff));
  }
}

// ------------------------------------------------------------------ the 8 x 8 tail and Decaps' message
// V = S' B + E'' (mulAddSBPlusE, util.go:117-131), C = V + Encode(mu).  Encaps packs C into ct[9600:9720]; Decaps
// compares it with the ciphertext's C, adds the B' flag and selects k' or s into the work row (frodo.go:321-323).
// One CTA of 64 threads per op, thread (k, l); B is unpacked into shared memory from the public key (stride 0: one).
// S' rows are padded to 644 bytes: a warp reads rows k = 0..3 at one j, which a 640-byte pitch (0 mod 128) would put
// in one bank.
constexpr int kSpPitch = kN + 4;
template <bool DEC>
__global__ void __launch_bounds__(64) frodo_tail_kernel(const uint8_t* __restrict__ B, size_t bs, const uint8_t* __restrict__ mu,
                                                        size_t mus, const uint8_t* __restrict__ sfail, size_t sfs,
                                                        uint8_t* __restrict__ ct, uint8_t* __restrict__ W) {
  __shared__ __align__(16) uint16_t Bm[kN][kNbar];
  __shared__ __align__(16) int8_t Sp[kNbar][kSpPitch];
  __shared__ uint16_t Cm[kNbar * kNbar];
  const size_t op = blockIdx.x;
  const int tid = threadIdx.x, k = tid >> 3, l = tid & 7;
  uint8_t* w = W + op * kWork;
  const uint8_t* b = B + op * bs;
  for (int j = tid; j < kN; j += 64) {
    uint16_t v[8];
    unpack8(v, b + 15 * j);
#pragma unroll
    for (int x = 0; x < 8; x++) Bm[j][x] = v[x];
  }
  for (int q = tid; q < kN * kNbar / 4; q += 64)
    reinterpret_cast<uint32_t*>(&Sp[q / (kN / 4)][0])[q % (kN / 4)] = reinterpret_cast<const uint32_t*>(w + kOffSp)[q];
  __syncthreads();
  uint32_t v = (uint32_t)(int32_t)(int8_t)w[kOffEpp + tid];
#pragma unroll 8
  for (int j = 0; j < kN; j++) v += (uint32_t)(int32_t)Sp[k][j] * Bm[j][l];
  const uint8_t* m = DEC ? w + kOffMu : mu + op * mus;
  const uint16_t cv = (uint16_t)((v + encode_coef(m, tid)) & kQMask);
  uint8_t* c = ct + op * kCt + kBpBytes;
  if (!DEC) {
    Cm[tid] = cv;
    __syncthreads();
    if (tid < kNbar) {
      uint16_t r[8];
#pragma unroll
      for (int x = 0; x < 8; x++) r[x] = Cm[8 * tid + x];
      uint8_t g[15];
      pack8(g, r);
#pragma unroll
      for (int x = 0; x < 15; x++) c[15 * tid + x] = g[x];
    }
  } else {
    uint16_t r[8];
    unpack8(r, c + 15 * k);
    uint16_t mine = 0;
#pragma unroll
    for (int x = 0; x < 8; x++) mine |= (uint16_t)(x == l ? r[x] : 0);
    const int any = __syncthreads_or((cv ^ mine) != 0);
    const uint8_t mask = select_mask(reinterpret_cast<const uint32_t*>(w + kOffFlag)[0] | (uint32_t)any);
    if (tid < 16) {
      const uint8_t kp = w[kOffK + tid], s = sfail[op * sfs + tid];
      w[kOffK + tid] = (uint8_t)(kp ^ (mask & (kp ^ s)));
    }
  }
}

// Decaps' W = C - B' S and mu' = Decode(W) (frodo.go:276-281, util.go:133-143).  S comes from the private key and may
// hold any 16-bit value.  One CTA of 64 threads per op, thread (i, j); rows padded to avoid bank conflicts.
constexpr int kPitch = kN + 8;
__global__ void __launch_bounds__(64) frodo_decode_kernel(const uint8_t* __restrict__ sk, size_t sks,
                                                          const uint8_t* __restrict__ ct, uint8_t* __restrict__ W) {
  __shared__ __align__(16) uint16_t Bp[kNbar][kPitch];
  __shared__ __align__(16) uint16_t St[kNbar][kPitch];
  __shared__ uint8_t bits[kNbar * kNbar];
  const size_t op = blockIdx.x;
  const int tid = threadIdx.x, i = tid >> 3, j = tid & 7;
  const uint8_t* c = ct + op * kCt;
  const uint8_t* s = sk + op * sks + kSkS;
  for (int q = tid; q < kNbar * kN / 8; q += 64) {
    const int r = q / (kN / 8), grp = q % (kN / 8);
    uint16_t v[8];
    unpack8(v, c + 15 * q);
#pragma unroll
    for (int x = 0; x < 8; x++) Bp[r][8 * grp + x] = v[x];
    const uint64_t sv0 = ld64(s + 16 * q), sv1 = ld64(s + 16 * q + 8);  // S^T row r, columns 8 grp .. 8 grp + 7
#pragma unroll
    for (int x = 0; x < 4; x++) {
      St[r][8 * grp + x] = (uint16_t)(sv0 >> (16 * x));
      St[r][8 * grp + 4 + x] = (uint16_t)(sv1 >> (16 * x));
    }
  }
  __syncthreads();
  uint32_t v = 0;
#pragma unroll 8
  for (int k = 0; k < kN; k++) v += (uint32_t)Bp[i][k] * St[j][k];
  uint16_t cc[8];
  unpack8(cc, c + kBpBytes + 15 * i);
  uint16_t ci = 0;
#pragma unroll
  for (int x = 0; x < 8; x++) ci |= (uint16_t)(x == j ? cc[x] : 0);
  bits[tid] = (uint8_t)decode_coef((uint16_t)(ci - v));
  __syncthreads();
  if (tid < 16) {
    uint8_t* mu = W + op * kWork + kOffMu;
    mu[tid] = (uint8_t)(bits[4 * tid] | (bits[4 * tid + 1] << 2) | (bits[4 * tid + 2] << 4) | (bits[4 * tid + 3] << 6));
  }
}

// ------------------------------------------------------------------ host side
static inline unsigned blocks(size_t units, size_t per) { return (unsigned)((units + per - 1) / per); }

struct Area {
  uint8_t* W;   // kWork bytes per op of the sub-batch
  uint8_t* AT;  // kShared bytes (the shared-key path)
};
static int area(int slot, size_t cnt, bool shared, Area* a) {
  Arena A;
  const size_t rows = std::min(cnt, kChunk) * kWork;
  int rc = arena(slot, rows + (shared ? kShared : 0), &A);
  if (rc) return rc;
  a->W = A.take(rows);
  a->AT = shared ? A.take(kShared) : nullptr;
  return 0;
}

static int keygen_flow(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n, cudaStream_t st, int slot) {
  Area a;
  int rc = area(slot, n, false, &a);
  if (rc) return rc;
  for (size_t f = 0; f < n; f += kChunk) {
    const size_t c = std::min(kChunk, n - f);
    {
      KernelScope ks(KID_FRODO, st);
      frodo_keygen_seed_kernel<<<blocks(c, 128), 128, 0, st>>>(seeds + f * kSeed, pk + f * kPk, sk + f * kSk, a.W, c);
    }
    {
      KernelScope ks(KID_FRODO, st);
      frodo_keygen_a_kernel<<<dim3(kN / 128, (unsigned)c), 128, 0, st>>>(pk + f * kPk, sk + f * kSk, a.W);
    }
    KernelScope ks(KID_FRODO, st);
    frodo_hash_kernel<kPk, false><<<blocks(c, 128), 128, 0, st>>>(pk + f * kPk, kPk, nullptr, 0, sk + f * kSk + kSkHpk, kSk, c);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// B' = S' A + E' of a sub-batch: on chip per op, or (AT != null) the GEMM over A^T expanded once per call
template <bool DEC>
static void sa(const uint8_t* seedA, size_t ss_, uint8_t* ct, const Area& a, size_t c, cudaStream_t st) {
  if (!a.AT) {
    KernelScope ks(KID_FRODO, st);
    frodo_sa_kernel<DEC><<<(unsigned)c, kSaThreads, 0, st>>>(seedA, ss_, ct, a.W);
  } else {
    KernelScope ks(KID_FRODO_GEMM, st);
    frodo_gemm_kernel<DEC><<<dim3(kN / kGn, blocks(8 * c, kGm)), 128, 0, st>>>(a.W, a.AT, ct, c);
  }
}
// H(pk) of c public keys into the hpk field of the work rows
static void hpk(const uint8_t* pk, size_t pks, uint8_t* W, size_t c, cudaStream_t st) {
  KernelScope ks(KID_FRODO, st);
  frodo_hash_kernel<kPk, false><<<blocks(c, 128), 128, 0, st>>>(pk, pks, nullptr, 0, W + kOffHpk, kWork, c);
}
// ss = F(ct || k) with k the work rows' k field (frodo.go:235-239, 325-328)
static void kdf(const uint8_t* ct, const uint8_t* W, uint8_t* ss, size_t c, cudaStream_t st) {
  KernelScope ks(KID_FRODO, st);
  frodo_hash_kernel<kCt, true><<<blocks(c, 128), 128, 0, st>>>(ct, kCt, W + kOffK, kWork, ss, kSs, c);
}
static void expand_a(const uint8_t* seedA, const Area& a, cudaStream_t st) {
  KernelScope ks(KID_FRODO, st);
  frodo_expand_a_kernel<<<kN / 128, 128, 0, st>>>(seedA, a.AT);
}

static int encaps_flow(const uint8_t* pk, size_t pks, const uint8_t* seeds, uint8_t* ct, uint8_t* ss, size_t n,
                       cudaStream_t st, int slot) {
  Area a;
  int rc = area(slot, n, pks == 0, &a);
  if (rc) return rc;
  if (!pks) {  // A and H(pk) of the shared key, once per call (H(pk) into the hpk field of work row 0)
    expand_a(pk, a, st);
    hpk(pk, 0, a.W, 1, st);
  }
  for (size_t f = 0; f < n; f += kChunk) {
    const size_t c = std::min(kChunk, n - f);
    const uint8_t* p = pk + f * pks;
    uint8_t* cf = ct + f * kCt;
    if (pks) hpk(p, pks, a.W, c, st);
    {
      KernelScope ks(KID_FRODO, st);
      frodo_se_kernel<<<blocks(c, 128), 128, 0, st>>>(a.W + kOffHpk, pks ? kWork : 0, seeds + f * kEseed, kEseed, a.W, c);
    }
    sa<false>(p, pks, cf, a, c, st);
    {
      KernelScope ks(KID_FRODO, st);
      frodo_tail_kernel<false><<<(unsigned)c, 64, 0, st>>>(p + 16, pks, seeds + f * kEseed, kEseed, nullptr, 0, cf, a.W);
    }
    kdf(cf, a.W, ss + f * kSs, c, st);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

static int decaps_flow(const uint8_t* sk, size_t sks, const uint8_t* ct, uint8_t* ss, size_t n, cudaStream_t st,
                       int slot) {
  Area a;
  int rc = area(slot, n, sks == 0, &a);
  if (rc) return rc;
  if (!sks) expand_a(sk + kSkPk, a, st);
  for (size_t f = 0; f < n; f += kChunk) {
    const size_t c = std::min(kChunk, n - f);
    const uint8_t* s = sk + f * sks;
    uint8_t* cf = const_cast<uint8_t*>(ct) + f * kCt;  // read only: DEC kernels compare, they do not write
    {
      KernelScope ks(KID_FRODO, st);
      frodo_decode_kernel<<<(unsigned)c, 64, 0, st>>>(s, sks, cf, a.W);
    }
    {
      KernelScope ks(KID_FRODO, st);
      frodo_se_kernel<<<blocks(c, 128), 128, 0, st>>>(s + kSkHpk, sks, a.W + kOffMu, kWork, a.W, c);
    }
    sa<true>(s + kSkPk, sks, cf, a, c, st);
    {
      KernelScope ks(KID_FRODO, st);
      frodo_tail_kernel<true><<<(unsigned)c, 64, 0, st>>>(s + kSkPk + 16, sks, nullptr, 0, s, sks, cf, a.W);
    }
    kdf(cf, a.W, ss + f * kSs, c, st);
  }
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// Device pointers and strides: 8-byte aligned.  A contiguous batch of ciphertexts (9720-byte rows) is 8- but not
// 16-byte aligned, so every kernel reads ct with at most 8-byte accesses.
static const char* kAlign = "%s: device buffers and strides must be 8-byte aligned";
static bool bad_stride(size_t s, size_t unit) { return s != 0 && s < unit; }

}  // namespace frodo
}  // namespace cb200

using namespace cb200;
using namespace cb200::frodo;

extern "C" {

size_t cb200_frodo640shake_public_key_size(void) { return kPk; }
size_t cb200_frodo640shake_private_key_size(void) { return kSk; }
size_t cb200_frodo640shake_ciphertext_size(void) { return kCt; }
size_t cb200_frodo640shake_shared_key_size(void) { return kSs; }
size_t cb200_frodo640shake_seed_size(void) { return kSeed; }
size_t cb200_frodo640shake_encapsulation_seed_size(void) { return kEseed; }

int cb200_frodo640shake_keygen(const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!seeds || !pk || !sk) {
    set_error("cb200_frodo640shake_keygen: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_frodo640shake_keygen", n, pk, kHostChunk, 1u << 12,
          {{seeds, kSeed, kSeed, kIn}, {pk, kPk, kPk, kOut}, {sk, kSk, kSk, kOut}},
          {{!aligned({seeds, pk, sk}, {}, 8), kAlign}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    return keygen_flow(r[0].p, r[1].p, r[2].p, cnt, st, slot);
  });
}

int cb200_frodo640shake_encaps(const uint8_t* pk, size_t pk_stride, const uint8_t* seeds, uint8_t* ct, uint8_t* ss,
                               size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!pk || !seeds || !ct || !ss || bad_stride(pk_stride, kPk)) {
    set_error("cb200_frodo640shake_encaps: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_frodo640shake_encaps", n, ct, kHostChunk, 1u << 12,
          {{pk, kPk, pk_stride, kIn}, {seeds, kEseed, kEseed, kIn}, {ct, kCt, kCt, kOut}, {ss, kSs, kSs, kOut}},
          {{!aligned({pk, seeds, ct, ss}, {pk_stride}, 8), kAlign}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    return encaps_flow(r[0].p, r[0].stride, r[1].p, r[2].p, r[3].p, cnt, st, slot);
  });
}

int cb200_frodo640shake_decaps(const uint8_t* sk, size_t sk_stride, const uint8_t* ct, uint8_t* ss, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!sk || !ct || !ss || bad_stride(sk_stride, kSk)) {
    set_error("cb200_frodo640shake_decaps: bad argument");
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  Batch b{"cb200_frodo640shake_decaps", n, ss, kHostChunk, 1u << 12,
          {{sk, kSk, sk_stride, kIn}, {ct, kCt, kCt, kIn}, {ss, kSs, kSs, kOut}},
          {{!aligned({sk, ct, ss}, {sk_stride}, 8), kAlign}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    return decaps_flow(r[0].p, r[0].stride, r[1].p, r[2].p, cnt, st, slot);
  });
}

}  // extern "C"
