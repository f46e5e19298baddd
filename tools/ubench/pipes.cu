// pipes.cu — issue-rate micro-benchmark for the instruction kinds the cull / raster kernels are made of (sm_90a).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a --fmad=false -O3 -o pipes pipes.cu ; run on an H100.
// Prints warp-instructions / clk / SM for each kind with 8 independent chains per thread (ILP) and 32 warps / SM.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#define DI __device__ __forceinline__
DI float rcpa(float a) { float r; asm volatile("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r; }

constexpr int ITERS = 4096;
constexpr int CH = 8;

template <int KIND>
__global__ void __launch_bounds__(256) k(float* out, float seed, long long* clk) {
  float x[CH], y = seed * 1.0001f, z = seed * 0.5f;
  uint32_t n[CH];
#pragma unroll
  for (int i = 0; i < CH; i++) { x[i] = seed + i + threadIdx.x; n[i] = threadIdx.x + i; }
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int i = 0; i < CH; i++) {
      if (KIND == 0) x[i] = __fadd_rn(x[i], y);
      if (KIND == 1) x[i] = __fmul_rn(x[i], y);
      if (KIND == 2) x[i] = __fmaf_rn(x[i], y, z);
      if (KIND == 6) x[i] = fminf(x[i], y);
      if (KIND == 8) x[i] = rcpa(x[i]);
      if (KIND == 9) n[i] = (n[i] ^ (n[i] >> 3)) + 0x9E3779B9u;           // LOP3/SHF + IADD
      if (KIND == 10) { x[i] = __fadd_rn(x[i], y); n[i] = n[i] * 3u + 7u; } // FADD + IMAD
      if (KIND == 11) { x[i] = __fadd_rn(x[i], y); n[i] = (n[i] + 77u) ^ 5u; } // FADD + IADD/LOP (alu)
      if (KIND == 13) x[i] = __fdiv_rn(x[i], y);
      if (KIND == 14) x[i] = __fsqrt_rn(x[i]);
    }
  }
  long long t1 = clock64();
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < CH; i++) { acc += x[i] + (float)n[i]; }
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
  if (threadIdx.x == 0 && blockIdx.x == 0) *clk = t1 - t0;
}

template <int KIND>
void run(const char* name, float ops_per_iter) {
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  float* out; long long* clk; cudaMalloc(&out, sizeof(float) * sms * 4 * 256); cudaMalloc(&clk, 8);
  k<KIND><<<sms * 4, 256>>>(out, 1.5f, clk); cudaDeviceSynchronize();
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  cudaEventRecord(a); k<KIND><<<sms * 4, 256>>>(out, 1.5f, clk); cudaEventRecord(b); cudaDeviceSynchronize();
  float ms; cudaEventElapsedTime(&ms, a, b);
  long long c; cudaMemcpy(&c, clk, 8, cudaMemcpyDeviceToHost);
  // per SM: 32 warps x ITERS x CH x ops ; cycles = c
  const double winst = 32.0 * ITERS * CH * ops_per_iter;
  printf("%-28s %8.3f ms  %10lld clk  %6.3f warp-inst/clk/SM (%.3f /SMSP)\n", name, ms, c, winst / c, winst / c / 4);
  cudaFree(out); cudaFree(clk);
}

int main() {
  run<0>("FADD", 1); run<1>("FMUL", 1); run<2>("FFMA", 1);
  run<6>("FMNMX", 1); run<8>("MUFU.RCP", 1); run<9>("LOP/SHF+IADD (2 ops)", 2);
  run<10>("FADD+IMAD (2 ops)", 2); run<11>("FADD+IADD+LOP (3 ops)", 3);
  run<13>("fdiv_rn (1 call)", 1); run<14>("fsqrt_rn (1 call)", 1);
  return 0;
}
