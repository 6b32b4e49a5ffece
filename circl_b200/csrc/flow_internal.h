// Helpers shared by the flows that compose the lattice flows with a curve (hybrid.cu, eddsa.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

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

namespace hybrid {
// out[i] = SHAKE256(in[i] (inlen <= 64 bytes), outlen <= 128 bytes), thread per row (hybrid.cu shake_kernel); inlen and
// outlen multiples of 8, rows 4-byte aligned.
void shake256_rows(const uint8_t* in, size_t in_stride, int inlen, uint8_t* out, size_t out_stride, int outlen, size_t n,
                   cudaStream_t st);
}  // namespace hybrid
}  // namespace cb200
