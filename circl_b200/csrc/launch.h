// circl_b200/csrc/launch.h -- internal launcher prototypes (device pointers, explicit stream).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace cb200 {

void set_error(const char* fmt, ...);

// kyber_kernels.cu
int launch_kyber_ntt(int16_t* d_polys, size_t n, int inverse, const void* tw, cudaStream_t st);
int launch_kyber_dot(int16_t* d_out, const int16_t* d_a, const int16_t* d_b, int k, size_t n, const void* tw,
                     cudaStream_t st);
int launch_kyber_poly_op(int op, int16_t* d_out, const int16_t* d_a, const int16_t* d_b, size_t n, cudaStream_t st);
void kyber_fill_twiddles(int32_t* out);

}  // namespace cb200

namespace cb200 {
// dil_kernels.cu
int launch_dil_ntt(uint32_t* d_polys, size_t n, int inverse, const void* tw, cudaStream_t st);
int launch_dil_dot(uint32_t* out, const uint32_t* a, const uint32_t* b, int k, size_t n, cudaStream_t st);
int launch_dil_poly_op(int op, uint32_t* out, const uint32_t* a, const uint32_t* b, size_t n, cudaStream_t st);
int launch_dil_exceeds(const uint32_t* a, uint32_t bound, size_t n, uint8_t* flags, cudaStream_t st);
int launch_dil_power2round(uint32_t* a0q, uint32_t* a1, const uint32_t* a, size_t n, cudaStream_t st);
int launch_dil_pack_le16(uint8_t* out, const uint32_t* a, size_t n, cudaStream_t st);
void dil_fill_twiddles(uint32_t* out);
// tables.cu: twiddle tables other than Kyber's (ML-DSA) and the X25519 base table; called once per GPU at init
struct Dev;
int init_extra_tables(Dev& d);
int init_ed448_table(Dev& d);  // ed448.cu
int init_nistp_tables(Dev& d);  // p256.cu: P-256, P-384 and P-521
}  // namespace cb200
