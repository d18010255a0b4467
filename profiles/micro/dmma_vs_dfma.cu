// Micro-benchmark: fp64 tensor-core MMA (mma.sync.m8n8k4.f64, SASS DMMA) against the fp64 FMA
// pipe on H100: (1) DFMA only, (2) DMMA only, (3) both interleaved.  If time(3) ~ max(1, 2) the two
// run on different pipes and the tap sums of the expansion kernel (2 x taps of its ~38 fp64
// instructions per point) can move to the tensor pipe.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o dmma_vs_dfma dmma_vs_dfma.cu
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma(double &c0, double &c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__global__ void __launch_bounds__(128) k(int mode, int iters, double *out) {
  const int t = threadIdx.x;
  double f[16], c[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) { f[i] = t + i; c[i] = i; }
  const double a = 1.0 + 1e-9 * t, b = 1.0 - 1e-9 * t;
  for (int it = 0; it < iters; ++it) {
    if (mode & 1) {
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int i = 0; i < 16; ++i) f[i] = fma(f[i], a, b);      // 64 DFMA per thread
    }
    if (mode & 2) {
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int i = 0; i < 16; i += 2) dmma(c[i], c[i + 1], a, b);  // 16 DMMA per warp = 16 x 256 FMA
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += f[i] + c[i];
  out[blockIdx.x * blockDim.x + t] = s;
}
int main() {
  double *out;
  cudaMalloc(&out, sizeof(double) * 132 * 16 * 128);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int iters = 4000, ctas = 132 * 4;
  for (int mode = 1; mode <= 3; ++mode) {
    k<<<ctas, 128>>>(mode, 10, out);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    k<<<ctas, 128>>>(mode, iters, out);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    const double warps = ctas * 4.0;
    const double dfma = (mode & 1) ? warps * 32 * 64.0 * iters : 0;   // thread-FMAs
    const double dm = (mode & 2) ? warps * 16.0 * 256 * iters : 0;    // FMAs inside the MMAs
    printf("mode %d (%s): %.3f ms  DFMA %.2f TFLOP/s  DMMA %.2f TFLOP/s\n", mode,
           mode == 1 ? "DFMA" : mode == 2 ? "DMMA" : "both", ms, 2 * dfma / ms / 1e9, 2 * dm / ms / 1e9);
  }
  return 0;
}
