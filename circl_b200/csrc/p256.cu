// P-256 ECDH as Go's crypto/ecdh.P256() computes it for the reference's DHKEM(P-256) (hpke/shortkem.go), batched on the
// device, thread per op:
//   ecdh.PrivateKey.PublicKey               KeyGen  -> p256_base_kernel (fixed-base table built here at cb200_init)
//   NewPublicKey + ecdh.PrivateKey.ECDH     Shared  -> p256_kernel
// Both validate what they read (NewPrivateKey / NewPublicKey rules) and write a per-op status.  The curve code is
// p256.cuh; the DHKEM flows around it are hpke.cu's, which reach it through p256_rows.
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "p256.cuh"

namespace cb200 {

int init_p256_table(Dev& c) {  // device c.device is current
  std::vector<uint32_t> t(p256::kTableWords);
  p256::build_base_table(t.data());
  if (c.p256_table) cudaFree(c.p256_table);
  CB200_CUDA(cudaMalloc(&c.p256_table, t.size() * sizeof(uint32_t)));
  CB200_CUDA(cudaMemcpy(c.p256_table, t.data(), t.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  return 0;
}

namespace p256k {

// out[i] = 0x04 || X || Y of [k_i]G; status[i] |= 2 where k_i is not in [1, n - 1] (its row is then all zero)
__global__ void __launch_bounds__(128) p256_base_kernel(const uint8_t* __restrict__ scalars, size_t s_stride,
                                                        uint8_t* __restrict__ out, size_t o_stride,
                                                        uint8_t* __restrict__ status, const uint32_t* __restrict__ table,
                                                        size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t st = p256::keygen(out + i * o_stride, scalars + i * s_stride, table);
  if (status && st) status[i] |= (uint8_t)st;
}

// out[i] = X of [k_i]P_i; status[i] |= 1 where P_i is not a valid public key, 2 where k_i is not a valid private key
__global__ void __launch_bounds__(128) p256_kernel(const uint8_t* __restrict__ scalars, size_t s_stride,
                                                   const uint8_t* __restrict__ points, size_t p_stride,
                                                   uint8_t* __restrict__ out, size_t o_stride, uint8_t* __restrict__ status,
                                                   size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t st = p256::shared(out + i * o_stride, scalars + i * s_stride, points + i * p_stride);
  if (status && st) status[i] |= (uint8_t)st;
}

static inline unsigned blocks(size_t units, size_t per) { return (unsigned)((units + per - 1) / per); }

}  // namespace p256k

namespace hybrid {
void p256_rows(const uint8_t* k, size_t ks_, const uint8_t* p, size_t ps, uint8_t* o, size_t os, uint8_t* status, size_t n,
               cudaStream_t st) {
  KernelScope ks(KID_P256, st);
  if (p)
    p256k::p256_kernel<<<p256k::blocks(n, 128), 128, 0, st>>>(k, ks_, p, ps, o, os, status, n);
  else
    p256k::p256_base_kernel<<<p256k::blocks(n, 128), 128, 0, st>>>(k, ks_, o, os, status,
                                                                   (const uint32_t*)ctx().p256_table, n);
}
}  // namespace hybrid

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_p256(const uint8_t* scalars, const uint8_t* points, uint8_t* out, uint8_t* status, size_t n) {
  const char* fn = "cb200_p256";
  int rc = require_ready();
  if (rc) return rc;
  if (!scalars || !out) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const size_t ow = points ? 32 : 65;
  Batch b{fn, n, out, 1u << 16, 1u << 13, {{scalars, 32, 32, kIn}, {out, ow, ow, kOut}, {status, 1, 1, kStatus},
                                           {points, 65, 65, kIn}}, {}};
  Counts c;
  rc = run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) -> int {
    if (r[2].p) CB200_CUDA(cudaMemsetAsync(r[2].p, 0, cnt, st));
    hybrid::p256_rows(r[0].p, 32, r[3].p, 65, r[1].p, ow, r[2].p, cnt, st);
    CB200_CUDA(cudaGetLastError());
    return 0;
  }, &c);
  if (rc) return rc;
  if (c.bit1) {
    set_error("%s: %zu of %zu scalars are not in [1, n - 1] (ecdh: invalid private key)", fn, c.bit1, n);
    return CB200_ERR_PRIVKEY;
  }
  if (c.bit0) {
    set_error("%s: %zu of %zu points are not valid uncompressed P-256 points (ecdh: invalid public key)", fn, c.bit0, n);
    return CB200_ERR_PUBKEY;
  }
  return 0;
}

}  // extern "C"
