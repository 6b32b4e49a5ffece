// circl_b200/csrc/tables.cu -- device tables built at cb200_init time.
#include "common.cuh"
#include "context.h"
#include "dilithium.cuh"
#include "x25519.cuh"

#include <vector>

namespace cb200 {
int init_extra_tables(Dev& c) {  // device c.device is current
  uint32_t tw[dil::kTwWords];
  dil_fill_twiddles(tw);
  if (c.dil_tw) cudaFree(c.dil_tw);
  CB200_CUDA(cudaMalloc(&c.dil_tw, sizeof tw));
  CB200_CUDA(cudaMemcpy(c.dil_tw, tw, sizeof tw, cudaMemcpyHostToDevice));
  // fixed-base table of X25519 KeyGen: 256 affine multiples of the base point, computed here with the same limb
  // code the kernels use (x25519.cuh is host/device code)
  std::vector<int32_t> xt(x25519::kBaseTableWords);
  x25519::build_base_table(xt.data());
  if (c.x25519_table) cudaFree(c.x25519_table);
  CB200_CUDA(cudaMalloc(&c.x25519_table, xt.size() * sizeof(int32_t)));
  CB200_CUDA(cudaMemcpy(c.x25519_table, xt.data(), xt.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
  // fixed-base tables of Ed448 (ed448.cu) and P-256 / P-384 / P-521 (p256.cu)
  int rc = init_ed448_table(c);
  if (rc) return rc;
  return init_nistp_tables(c);
}
}  // namespace cb200
