// Device-level entry points of the ML-DSA / round-3 Dilithium flows (mldsa.cu) for the composite signatures in
// eddsa.cu.  All pointers are device pointers; `mode` is 44, 65, 87 (ML-DSA) or 2, 3, 5 (round-3 Dilithium); `slot`
// is the work-area slot (0..3 staging pipeline, kDevSlot device-pointer calls) and the flows use its level-0 area.
// Keys and signatures are contiguous rows of the mode's sizes; key pointers and strides are 16-byte aligned, msg_off
// too, and msgs carries 8 bytes of read padding.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

namespace cb200 {
namespace mldsa {

int dev_keygen(int mode, const uint8_t* seeds, uint8_t* pk, uint8_t* sk, size_t n, cudaStream_t st, int slot);
// deterministic signing of the message as given (round-3 SignTo; no context string); status[i] = 1 where the
// 576-attempt cap was hit.  h_count: 8 bytes of pinned host memory for the per-round counter of the rejection loop.
int dev_sign(int mode, const uint8_t* sk, size_t sk_stride, const uint8_t* msgs, const uint64_t* msg_off, uint8_t* sig,
             uint8_t* status, size_t n, cudaStream_t st, int slot, volatile uint32_t* h_count);
int dev_verify(int mode, const uint8_t* pk, size_t pk_stride, const uint8_t* msgs, const uint64_t* msg_off,
               const uint8_t* sig, uint8_t* ok, size_t n, cudaStream_t st, int slot);

}  // namespace mldsa
}  // namespace cb200
