// Helpers shared by the flows that compose the lattice flows with a curve (hybrid.cu, eddsa.cu, ed448.cu), and the
// host side of the signature entry points that take variable-length messages (eddsa.cu, ed448.cu).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <functional>
#include <initializer_list>
#include <vector>

#include "common.cuh"
#include "context.h"

namespace cb200 {

// bump allocator over the level-1 work area of a slot (level 0 belongs to the lattice flows the caller runs)
struct Arena {
  char* base = nullptr;
  size_t off = 0;
  uint8_t* take(size_t bytes) {
    uint8_t* p = (uint8_t*)(base + off);
    off += (bytes + 255) & ~(size_t)255;
    return p;
  }
};
inline int arena(int slot, size_t bytes, Arena* a) {
  void* p = nullptr;
  int rc = ensure_work(kLevel1 + slot, bytes + 4096, &p);
  if (rc) return rc;
  a->base = (char*)p;
  a->off = 0;
  return 0;
}

// 2D device-to-device copy on the call's stream: n rows of `width` bytes
inline int copy2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t n, cudaStream_t st) {
  CB200_CUDA(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, n, cudaMemcpyDeviceToDevice, st));
  return 0;
}

namespace sigio {
// host-pointer calls with variable-length messages: one contiguous range per GPU, staged in chunks through
// scratch slot 0 (flows run with slot 0).  rows[j]: fixed-width per-op buffers (shared = one row for the batch).
struct Row {
  const uint8_t* in;
  uint8_t* out;
  size_t unit;
  size_t host_stride;  // 0 = dense
  bool shared;
};
using MsgBody = std::function<int(uint8_t** d, const uint8_t* msgs, const uint64_t* off, size_t cnt, cudaStream_t st)>;
inline int run_msgs(size_t n, const std::vector<Row>& rows, const uint8_t* msgs, const uint64_t* msg_off, const MsgBody& body) {
  return for_each_shard(n, 1u << 12, [&](size_t f0, size_t sn) -> int {
    Dev& c = ctx();
    cudaStream_t st = c.pipe[0];
    constexpr size_t kChunk = 1u << 15;
    std::vector<uint64_t> ro;
    for (size_t first = f0; first < f0 + sn; first += kChunk) {
      const size_t cnt = std::min(kChunk, f0 + sn - first);
      const uint64_t m0 = msg_off[first];
      const size_t mb = (size_t)(msg_off[first + cnt] - m0);
      size_t off = 0;
      auto take = [&](size_t bytes) {
        size_t o = off;
        off += (bytes + 255) & ~(size_t)255;
        return o;
      };
      std::vector<size_t> ro_off(rows.size());
      for (size_t j = 0; j < rows.size(); j++) ro_off[j] = take(rows[j].shared ? rows[j].unit : cnt * rows[j].unit);
      const size_t oMsg = take(mb + 8), oOff = take((cnt + 1) * 8);
      int rc = ensure_scratch(0, off);
      if (rc) return rc;
      char* d = (char*)c.scratch[0];
      std::vector<uint8_t*> dp(rows.size());
      for (size_t j = 0; j < rows.size(); j++) {
        const Row& r = rows[j];
        dp[j] = (uint8_t*)d + ro_off[j];
        if (!r.in) continue;
        const size_t hs = r.host_stride ? r.host_stride : r.unit;
        if (r.shared)
          CB200_CUDA(cudaMemcpyAsync(dp[j], r.in, r.unit, cudaMemcpyHostToDevice, st));
        else if (hs == r.unit)
          CB200_CUDA(cudaMemcpyAsync(dp[j], r.in + first * hs, cnt * r.unit, cudaMemcpyHostToDevice, st));
        else
          CB200_CUDA(cudaMemcpy2DAsync(dp[j], r.unit, r.in + first * hs, hs, r.unit, cnt, cudaMemcpyHostToDevice, st));
      }
      if (mb) CB200_CUDA(cudaMemcpyAsync(d + oMsg, msgs + m0, mb, cudaMemcpyHostToDevice, st));
      ro.resize(cnt + 1);
      for (size_t i = 0; i <= cnt; i++) ro[i] = msg_off[first + i] - m0;
      CB200_CUDA(cudaMemcpyAsync(d + oOff, ro.data(), (cnt + 1) * 8, cudaMemcpyHostToDevice, st));
      rc = body(dp.data(), (const uint8_t*)d + oMsg, (const uint64_t*)(d + oOff), cnt, st);
      if (rc) return rc;
      for (size_t j = 0; j < rows.size(); j++)
        if (rows[j].out) CB200_CUDA(cudaMemcpyAsync(rows[j].out + first * rows[j].unit, dp[j], cnt * rows[j].unit,
                                                    cudaMemcpyDeviceToHost, st));
      CB200_CUDA(cudaStreamSynchronize(st));  // `ro` and the scratch are reused by the next chunk
    }
    return 0;
  });
}

inline bool same_side(std::initializer_list<const void*> ps, bool* dev) {
  bool first = true;
  for (const void* p : ps) {
    if (!p) continue;
    const bool d = is_device_ptr(p);
    if (first) {
      *dev = d;
      first = false;
    } else if (d != *dev) {
      return false;
    }
  }
  return true;
}
inline bool aligned(std::initializer_list<const void*> ps, std::initializer_list<size_t> strides, uintptr_t a) {
  uintptr_t acc = 0;
  for (const void* p : ps) acc |= (uintptr_t)p;
  for (size_t v : strides) acc |= v;
  return (acc & (a - 1)) == 0;
}

}  // namespace sigio

namespace hybrid {
// out[i] = SHAKE256(in[i] (inlen <= 64 bytes), outlen <= 128 bytes), thread per row (hybrid.cu shake_kernel); inlen and
// outlen multiples of 8, rows 4-byte aligned.
void shake256_rows(const uint8_t* in, size_t in_stride, int inlen, uint8_t* out, size_t out_stride, int outlen, size_t n,
                   cudaStream_t st);
}  // namespace hybrid
}  // namespace cb200
