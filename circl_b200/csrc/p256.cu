// P-256, P-384 and P-521 ECDH as Go's crypto/ecdh computes it for the reference's NIST DHKEMs (hpke/shortkem.go),
// batched on the device, thread per op:
//   ecdh.PrivateKey.PublicKey               KeyGen  -> p256_base_kernel / p384_base_kernel / p521_base_kernel
//                                                      (fixed-base tables built here at cb200_init)
//   NewPublicKey + ecdh.PrivateKey.ECDH     Shared  -> p256_kernel / p384_kernel / p521_kernel
// All validate what they read (NewPrivateKey / NewPublicKey rules) and write a per-op status.  The curve code is
// nistp.cuh with the curve types of p256.cuh, p384.cuh and p521.cuh; the DHKEM flows around it are hpke.cu's, which
// reach it through p256_rows / p384_rows / p521_rows.
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "p256.cuh"
#include "p384.cuh"
#include "p521.cuh"

namespace cb200 {

template <class C>
static int init_table(void*& slot) {
  std::vector<uint32_t> t(nistp::kTableWords<C>);
  nistp::build_base_table<C>(t.data());
  if (slot) cudaFree(slot);
  slot = nullptr;
  CB200_CUDA(cudaMalloc(&slot, t.size() * sizeof(uint32_t)));
  CB200_CUDA(cudaMemcpy(slot, t.data(), t.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  return 0;
}
int init_nistp_tables(Dev& c) {  // device c.device is current
  int rc = init_table<nistp::P256>(c.p256_table);
  if (!rc) rc = init_table<nistp::P384>(c.p384_table);
  if (!rc) rc = init_table<nistp::P521>(c.p521_table);
  return rc;
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

// The same two operations on P-384 and P-521
#define CB200_NISTP_KERNELS(name, C)                                                                                   \
  __global__ void __launch_bounds__(128)                                                                               \
      name##_base_kernel(const uint8_t* __restrict__ scalars, size_t s_stride, uint8_t* __restrict__ out,              \
                         size_t o_stride, uint8_t* __restrict__ status, const uint32_t* __restrict__ table, size_t n) { \
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;                                                    \
    if (i >= n) return;                                                                                                \
    const uint32_t st = nistp::keygen<C>(out + i * o_stride, scalars + i * s_stride, table);                           \
    if (status && st) status[i] |= (uint8_t)st;                                                                        \
  }                                                                                                                    \
  __global__ void __launch_bounds__(128)                                                                               \
      name##_kernel(const uint8_t* __restrict__ scalars, size_t s_stride, const uint8_t* __restrict__ points,          \
                    size_t p_stride, uint8_t* __restrict__ out, size_t o_stride, uint8_t* __restrict__ status,         \
                    size_t n) {                                                                                        \
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;                                                    \
    if (i >= n) return;                                                                                                \
    const uint32_t st = nistp::shared<C>(out + i * o_stride, scalars + i * s_stride, points + i * p_stride);           \
    if (status && st) status[i] |= (uint8_t)st;                                                                        \
  }
CB200_NISTP_KERNELS(p384, nistp::P384)
CB200_NISTP_KERNELS(p521, nistp::P521)
#undef CB200_NISTP_KERNELS

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
void p384_rows(const uint8_t* k, size_t ks_, const uint8_t* p, size_t ps, uint8_t* o, size_t os, uint8_t* status, size_t n,
               cudaStream_t st) {
  KernelScope ks(KID_P384, st);
  if (p)
    p256k::p384_kernel<<<p256k::blocks(n, 128), 128, 0, st>>>(k, ks_, p, ps, o, os, status, n);
  else
    p256k::p384_base_kernel<<<p256k::blocks(n, 128), 128, 0, st>>>(k, ks_, o, os, status,
                                                                   (const uint32_t*)ctx().p384_table, n);
}
void p521_rows(const uint8_t* k, size_t ks_, const uint8_t* p, size_t ps, uint8_t* o, size_t os, uint8_t* status, size_t n,
               cudaStream_t st) {
  KernelScope ks(KID_P521, st);
  if (p)
    p256k::p521_kernel<<<p256k::blocks(n, 128), 128, 0, st>>>(k, ks_, p, ps, o, os, status, n);
  else
    p256k::p521_base_kernel<<<p256k::blocks(n, 128), 128, 0, st>>>(k, ks_, o, os, status,
                                                                   (const uint32_t*)ctx().p521_table, n);
}
}  // namespace hybrid

// cb200_p256 / cb200_p384 / cb200_p521 on rows of B-byte scalars and 1 + 2B-byte points
using Rows_fn = void (*)(const uint8_t*, size_t, const uint8_t*, size_t, uint8_t*, size_t, uint8_t*, size_t, cudaStream_t);
static int ecdh_entry(const char* fn, const char* curve, size_t B, Rows_fn rows, const uint8_t* scalars,
                      const uint8_t* points, uint8_t* out, uint8_t* status, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (!scalars || !out) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  if (n == 0) return 0;
  const size_t pw = 1 + 2 * B, ow = points ? B : pw;
  Batch b{fn, n, out, 1u << 16, 1u << 13, {{scalars, B, B, kIn}, {out, ow, ow, kOut}, {status, 1, 1, kStatus},
                                           {points, pw, pw, kIn}}, {}};
  Counts c;
  rc = run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) -> int {
    if (r[2].p) CB200_CUDA(cudaMemsetAsync(r[2].p, 0, cnt, st));
    rows(r[0].p, B, r[3].p, pw, r[1].p, ow, r[2].p, cnt, st);
    CB200_CUDA(cudaGetLastError());
    return 0;
  }, &c);
  if (rc) return rc;
  if (c.bit1) {
    set_error("%s: %zu of %zu scalars are not in [1, n - 1] (ecdh: invalid private key)", fn, c.bit1, n);
    return CB200_ERR_PRIVKEY;
  }
  if (c.bit0) {
    set_error("%s: %zu of %zu points are not valid uncompressed %s points (ecdh: invalid public key)", fn, c.bit0, n,
              curve);
    return CB200_ERR_PUBKEY;
  }
  return 0;
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_p256(const uint8_t* scalars, const uint8_t* points, uint8_t* out, uint8_t* status, size_t n) {
  return ecdh_entry("cb200_p256", "P-256", 32, hybrid::p256_rows, scalars, points, out, status, n);
}
int cb200_p384(const uint8_t* scalars, const uint8_t* points, uint8_t* out, uint8_t* status, size_t n) {
  return ecdh_entry("cb200_p384", "P-384", 48, hybrid::p384_rows, scalars, points, out, status, n);
}
int cb200_p521(const uint8_t* scalars, const uint8_t* points, uint8_t* out, uint8_t* status, size_t n) {
  return ecdh_entry("cb200_p521", "P-521", 66, hybrid::p521_rows, scalars, points, out, status, n);
}

}  // extern "C"
