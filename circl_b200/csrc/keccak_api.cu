// circl_b200/csrc/keccak_api.cu -- the permutation and the one-shot sponges as batch entry points of their own.
//
//   cb200_keccak_f1600  <- (*StateX4).Permute      simd/keccakf1600/f1600x.go:115-121 (asm f1600x4_amd64.s:9)
//                          KeccakF1600             internal/sha3/keccakf.go:12
//   cb200_sha3          <- Sum256 / Sum512 / ShakeSum128 / ShakeSum256   internal/sha3/hashes.go:21-60, shake.go:56-110
//
// The reference interleaves 4 states in AVX2 lanes; here 32 states ride the 32 lanes of a warp, 25 lanes of 64 bits
// per thread in registers (keccak.cuh).  A CTA moves its 128 states between HBM and registers through shared memory so
// that global accesses are whole 128-byte lines (a state is 200 bytes: thread-private rows would touch 7 sectors each).
#include "../../include/circl_b200.h"
#include "context.h"
#include "flow_internal.h"
#include "keccak.cuh"

namespace cb200 {
namespace keccakapi {

constexpr int kThreads = 128;
constexpr int kRow = 25;  // 64-bit words per state; 25 is odd, so thread-private rows are bank-conflict free

__global__ void __launch_bounds__(kThreads) f1600_kernel(uint64_t* __restrict__ states, size_t n, int first_round) {
  __shared__ uint64_t tile[kThreads * kRow];
  const size_t s0 = (size_t)blockIdx.x * kThreads;
  const size_t here = n - s0 < (size_t)kThreads ? n - s0 : (size_t)kThreads;
  const size_t words = here * kRow;
  uint64_t* g = states + s0 * kRow;
  for (size_t i = threadIdx.x; i < words; i += kThreads) tile[i] = g[i];
  __syncthreads();
  if (threadIdx.x < here) {
    uint64_t a[25];
#pragma unroll
    for (int i = 0; i < 25; i++) a[i] = tile[threadIdx.x * kRow + i];
    keccak::f1600(a, first_round);
#pragma unroll
    for (int i = 0; i < 25; i++) tile[threadIdx.x * kRow + i] = a[i];
  }
  __syncthreads();
  for (size_t i = threadIdx.x; i < words; i += kThreads) g[i] = tile[i];
}

// up to 8 little-endian bytes from an arbitrary address
__device__ __forceinline__ uint64_t load_le(const uint8_t* p, int nbytes) {
  if (nbytes >= 8 && ((uintptr_t)p & 7) == 0) return *reinterpret_cast<const uint64_t*>(p);
  uint64_t v = 0;
  for (int i = 0; i < nbytes && i < 8; i++) v |= (uint64_t)p[i] << (8 * i);
  return v;
}

// thread per message; RW = rate in 64-bit words (21: SHAKE128, 17: SHAKE256 / SHA3-256, 9: SHA3-512)
template <int RW>
__global__ void __launch_bounds__(kThreads) sponge_kernel(const uint8_t* __restrict__ in, size_t in_stride, size_t inlen,
                                                          uint8_t* __restrict__ out, size_t outlen, size_t n, uint8_t ds) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* p = in + i * in_stride;
  uint64_t a[25];
  keccak::zero(a);
  size_t left = inlen;
  while (left >= (size_t)RW * 8) {  // internal/sha3/sha3.go:128-160 (Write)
#pragma unroll
    for (int w = 0; w < RW; w++) a[w] ^= load_le(p + 8 * w, 8);
    keccak::f1600(a);
    p += RW * 8;
    left -= RW * 8;
  }
  // last block: the remaining bytes, the domain separator and the final bit of pad10*1 (sha3.go:103-126)
#pragma unroll
  for (int w = 0; w < RW; w++) {
    const long rem = (long)left - 8 * w;
    uint64_t v = 0;
    if (rem > 0) v = load_le(p + 8 * w, rem >= 8 ? 8 : (int)rem);
    if (rem >= 0 && rem < 8) v ^= (uint64_t)ds << (8 * rem);
    if (w == RW - 1) v ^= 0x8000000000000000ull;
    a[w] ^= v;
  }
  keccak::f1600(a);
  uint8_t* o = out + i * outlen;
  size_t done = 0;
  for (;;) {  // sha3.go:163-190 (Read)
#pragma unroll
    for (int w = 0; w < RW; w++) {
      const uint64_t v = a[w];
      for (int b = 0; b < 8; b++)
        if (done + 8 * w + b < outlen) o[done + 8 * w + b] = (uint8_t)(v >> (8 * b));
    }
    done += RW * 8;
    if (done >= outlen) break;
    keccak::f1600(a);
  }
}

static int launch_f1600(uint64_t* d, size_t n, int turbo, cudaStream_t st) {
  KernelScope ks(KID_KECCAK, st);
  f1600_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, st>>>(d, n, turbo ? 12 : 0);
  CB200_CUDA(cudaGetLastError());
  return 0;
}
static int launch_sponge(int rw, const uint8_t* in, size_t in_stride, size_t inlen, uint8_t* out, size_t outlen, size_t n,
                         uint8_t ds, cudaStream_t st) {
  KernelScope ks(KID_KECCAK, st);
  const unsigned grid = (unsigned)((n + kThreads - 1) / kThreads);
  if (rw == 21)
    sponge_kernel<21><<<grid, kThreads, 0, st>>>(in, in_stride, inlen, out, outlen, n, ds);
  else if (rw == 17)
    sponge_kernel<17><<<grid, kThreads, 0, st>>>(in, in_stride, inlen, out, outlen, n, ds);
  else
    sponge_kernel<9><<<grid, kThreads, 0, st>>>(in, in_stride, inlen, out, outlen, n, ds);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace keccakapi
}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_keccak_f1600(uint64_t* states, size_t n, int turbo) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!states) {
    set_error("cb200_keccak_f1600: null pointer");
    return CB200_ERR_ARG;
  }
  Batch b{"cb200_keccak_f1600", n, states, 1u << 18, 1u << 16, {{states, 200, 200, kInOut}},
          {{!aligned({states}, {}, 8), "%s: device states must be 8-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return keccakapi::launch_f1600((uint64_t*)r[0].p, cnt, turbo, st);
  });
}

int cb200_sha3(int bits, const uint8_t* in, size_t in_stride, size_t inlen, uint8_t* out, size_t outlen, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  int rw = 0;
  uint8_t ds = 0;
  switch (bits) {
    case 128: rw = 21; ds = 0x1f; break;   // shake.go:56
    case 256: rw = 17; ds = 0x1f; break;   // shake.go:74
    case -256: rw = 17; ds = 0x06; break;  // hashes.go:21
    case -512: rw = 9; ds = 0x06; break;   // hashes.go:35
    default:
      set_error("cb200_sha3: bits must be 128, 256 (SHAKE) or -256, -512 (SHA3), got %d", bits);
      return CB200_ERR_ARG;
  }
  if ((bits == -256 && outlen != 32) || (bits == -512 && outlen != 64) || outlen == 0) {
    set_error("cb200_sha3: output length %zu does not fit the function", outlen);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  if (!out || (!in && inlen) || (in_stride != 0 && in_stride < inlen)) {
    set_error("cb200_sha3: bad argument");
    return CB200_ERR_ARG;
  }
  // an empty input is never read: its rows are a device area only (unit 1 keeps the staged image non-empty)
  Batch b{"cb200_sha3", n, out, 1u << 16, 1u << 14,
          {{in, inlen ? inlen : 1, in_stride, inlen ? kIn : kScratch}, {out, outlen, outlen, kOut}}, {}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return keccakapi::launch_sponge(rw, r[0].p, r[0].stride, inlen, r[1].p, outlen, cnt, ds, st);
  });
}

}  // extern "C"
