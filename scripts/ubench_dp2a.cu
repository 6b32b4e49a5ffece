// Is IDP.2A (dp2a: 16-bit x 8-bit pairs, accumulate) as fast as IMAD on sm_90a?  Decides the inner product of the
// fused K-PKE encrypt kernel (csrc/mlkem.cu, matvec on packed coefficient pairs).
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a scripts/ubench_dp2a.cu -o ubench_dp2a && ./ubench_dp2a
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// multiprocessors of device 0: the grids below put the same number of CTAs on every SM
static int sms() {
  static int n = 0;
  if (!n) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0);
  return n;
}

#define ITERS 4096
template <int MODE>
__global__ void k(uint32_t* out, uint32_t seed) {
  uint32_t a[16];
#pragma unroll
  for (int i = 0; i < 16; i++) a[i] = seed + threadIdx.x * 16 + i;
  uint32_t w = seed * 2654435761u, b = seed ^ 0x01020304u;
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int i = 0; i < 16; i++) {
      if (MODE == 0) asm volatile("dp2a.lo.u32.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(w), "r"(b));
      if (MODE == 1) asm volatile("dp2a.hi.u32.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(w), "r"(b));
      if (MODE == 2) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(w), "r"(b));
      if (MODE == 3) asm volatile("dp4a.u32.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(w), "r"(b));
      if (MODE == 4) asm volatile("prmt.b32 %0, %0, %1, 0x5140;" : "+r"(a[i]) : "r"(w));
      if (MODE == 5) {  // dp2a + lop3 on other registers: do the pipes overlap?
        asm volatile("dp2a.lo.u32.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(w), "r"(b));
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[(i + 8) & 15]) : "r"(w), "r"(b));
      }
    }
    w += a[0];
  }
  uint32_t s = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) s ^= a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int MODE>
void run(const char* name, int ops) {
  uint32_t* d;
  cudaMalloc(&d, sms() * 1024 * 4);
  for (int warps = 8; warps <= 32; warps *= 2) {
    k<MODE><<<sms(), warps * 32>>>(d, 12345);
    cudaDeviceSynchronize();
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    cudaEventRecord(a);
    k<MODE><<<sms(), warps * 32>>>(d, 12345);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    double warp_instr = (double)ITERS * 16 * ops * warps;
    double cycles = ms * 1e-3 * 1.965e9;
    printf("%-22s warps/SM=%2d  %.3f ms  warp-instr/clk/SMSP = %.3f\n", name, warps, ms, warp_instr / cycles / 4);
  }
  cudaFree(d);
}
int main() {
  run<0>("dp2a.lo", 1);
  run<1>("dp2a.hi", 1);
  run<2>("mad.lo", 1);
  run<3>("dp4a", 1);
  run<4>("prmt", 1);
  run<5>("dp2a.lo + lop3", 2);
  return 0;
}
