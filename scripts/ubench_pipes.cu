// Pipe-throughput microbenchmark for the integer ops the NTT butterflies use (sm_90a).
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a scripts/ubench_pipes.cu -o ubench_pipes && ./ubench_pipes
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdint.h>

// multiprocessors of device 0: the grids below put the same number of CTAs on every SM
static int sms() {
  static int n = 0;
  if (!n) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0);
  return n;
}

#define ITERS 4096
template <int MODE>
__global__ void k(int32_t* out, int32_t seed) {
  int32_t a[8];
#pragma unroll
  for (int i = 0; i < 8; i++) a[i] = seed + threadIdx.x * 8 + i;
  int32_t z = seed | 1, q = -3329;
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      if (MODE == 0) asm volatile("mad.lo.s32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(z), "r"(q));
      if (MODE == 1) asm volatile("mad.hi.s32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(z), "r"(q));
      if (MODE == 2) asm volatile("shr.s32 %0, %0, 1;" : "+r"(a[i]));
      if (MODE == 3) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(z), "r"(q));
      if (MODE == 4) {  // 1 mad.lo + 1 shift (different registers -> dual pipe)
        asm volatile("mad.lo.s32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(z), "r"(q));
        asm volatile("shr.s32 %0, %0, 1;" : "+r"(a[(i + 4) & 7]));
      }
      if (MODE == 5) {  // 1 mad.hi + 1 add
        asm volatile("mad.hi.s32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(z), "r"(q));
        asm volatile("add.s32 %0, %0, %1;" : "+r"(a[(i + 4) & 7]) : "r"(q));
      }
      if (MODE == 6) asm volatile("mad.lo.s32 %0, %0, 2571, %1;" : "+r"(a[i]) : "r"(q));       // immediate multiplier
      if (MODE == 7) asm volatile("mad.hi.s32 %0, %0, 168493056, %1;" : "+r"(a[i]) : "r"(q));  // immediate multiplier
      if (MODE == 8) asm volatile("add.s32 %0, %0, %1;" : "+r"(a[i]) : "r"(q));
      if (MODE == 9) {  // butterfly A: 3 mad.lo + 2 shr + 2 add
        int32_t c, m, p, t;
        asm volatile("shr.s32 %0, %1, 16;" : "=r"(c) : "r"(a[i]));
        asm volatile("mul.lo.s32 %0, %1, 2571;" : "=r"(p) : "r"(c));
        asm volatile("mul.lo.s32 %0, %1, 0x7b0b0000;" : "=r"(m) : "r"(c));
        asm volatile("shr.s32 %0, %0, 16;" : "+r"(m));
        asm volatile("mad.lo.s32 %0, %1, -3329, %2;" : "=r"(t) : "r"(m), "r"(p));
        asm volatile("add.s32 %0, %0, %1;" : "+r"(a[i]) : "r"(t));
        asm volatile("sub.s32 %0, %0, %1;" : "+r"(a[(i + 1) & 7]) : "r"(t));
      }
      if (MODE == 11) {  // mad.wide.u32 with 64-bit accumulate (IMAD.WIDE.U32): the X25519 / Dilithium product
        uint64_t acc = ((uint64_t)(uint32_t)a[(i + 1) & 7] << 32) | (uint32_t)a[i];
        asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc) : "r"(z), "r"(q));
        a[i] = (int32_t)acc;
        a[(i + 1) & 7] = (int32_t)(acc >> 32);
      }
      if (MODE == 12) {  // mad.wide.u32 + lop3 on other registers
        uint64_t acc = ((uint64_t)(uint32_t)a[(i + 1) & 7] << 32) | (uint32_t)a[i];
        asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc) : "r"(z), "r"(q));
        a[i] = (int32_t)acc;
        a[(i + 1) & 7] = (int32_t)(acc >> 32);
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[(i + 4) & 7]) : "r"(z), "r"(q));
      }
      if (MODE == 10) {  // butterfly B: 1 mul.lo + 2 mad.hi + 2 add
        int32_t m, h, t;
        asm volatile("mul.lo.s32 %0, %1, 31499;" : "=r"(m) : "r"(a[i]));
        asm volatile("mul.hi.s32 %0, %1, 168493056;" : "=r"(h) : "r"(a[i]));
        asm volatile("mad.hi.s32 %0, %1, -218169344, %2;" : "=r"(t) : "r"(m), "r"(h));
        asm volatile("add.s32 %0, %0, %1;" : "+r"(a[i]) : "r"(t));
        asm volatile("sub.s32 %0, %0, %1;" : "+r"(a[(i + 1) & 7]) : "r"(t));
      }
    }
  }
  int32_t s = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) s ^= a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int MODE>
void run(const char* name, int ops_per_inner) {
  int32_t* d;
  cudaMalloc(&d, sms() * 8 * 256 * 4);
  for (int warps = 4; warps <= 32; warps *= 2) {
    // one CTA per SM with `warps` warps -> warps/4 per SMSP
    k<MODE><<<sms(), warps * 32>>>(d, 12345);
    cudaDeviceSynchronize();
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a);
    k<MODE><<<sms(), warps * 32>>>(d, 12345);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    double warp_instr = (double)ITERS * 8 * ops_per_inner * warps;   // per SM
    // assume ~1.9 GHz if clock rate query fails
    int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    double cycles = ms * 1e-3 * khz * 1e3;
    printf("%-28s warps/SM=%2d  %.3f ms  warp-instr/cycle/SM = %.2f (per SMSP %.2f) [clk attr %d kHz]\n", name, warps, ms,
           warp_instr / cycles, warp_instr / cycles / 4, khz);
  }
  cudaFree(d);
}

int main() {
  run<0>("mad.lo (IMAD)", 1);
  run<1>("mad.hi (IMAD.HI)", 1);
  run<6>("mad.lo imm", 1);
  run<7>("mad.hi imm", 1);
  run<2>("shr (SHF)", 1);
  run<3>("lop3", 1);
  run<8>("add (IADD3)", 1);
  run<4>("mad.lo + shr", 2);
  run<5>("mad.hi + add", 2);
  run<9>("butterfly A (3 IMAD,2 SHF,2 ADD)", 7);
  run<10>("butterfly B (1 IMAD,2 IMAD.HI,2 ADD)", 5);
  run<11>("mad.wide.u32 (IMAD.WIDE)", 1);
  run<12>("mad.wide.u32 + lop3", 2);
  return 0;
}
