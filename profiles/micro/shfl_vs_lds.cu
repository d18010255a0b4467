// Micro-benchmark: do warp shuffles and shared-memory accesses share one pipe on H100?
// (a) LDS.128+STS.128 only, (b) SHFL only, (c) both interleaved.  If time(c) ~ max(a, b) the
// paths are independent and an FFT exchange can be split between them.
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(int mode, int iters, double2 *out) {
  extern __shared__ double2 sm[];
  const int t = threadIdx.x;
  double2 v = make_double2(t, t + 1.0), w = make_double2(1.0, 2.0);
  sm[t] = v;
  __syncthreads();
  for (int i = 0; i < iters; ++i) {
    if (mode & 1) {
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        sm[(t + 32 * r) & 1023] = v;
        v = sm[(t + 32 * r + 64) & 1023];
        v.x += 1.0;
      }
    }
    if (mode & 2) {
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        w.x = __shfl_xor_sync(0xffffffffu, w.x, 1 + (r & 15));
        w.y = __shfl_xor_sync(0xffffffffu, w.y, 2 + (r & 7));
      }
    }
  }
  out[blockIdx.x * blockDim.x + t] = make_double2(v.x + w.x, v.y + w.y);
}
int main() {
  double2 *out;
  cudaMalloc(&out, sizeof(double2) * 132 * 8 * 256);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int mode = 1; mode <= 3; ++mode) {
    k<<<132 * 4, 256, 1024 * 16>>>(mode, 10, out);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    k<<<132 * 4, 256, 1024 * 16>>>(mode, 2000, out);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    // per iteration per warp: mode1: 8 STS.128 + 8 LDS.128; mode2: 64 SHFL.32 (16 x 2 x 64-bit)
    printf("mode %d (%s): %.3f ms\n", mode, mode == 1 ? "LDS+STS" : mode == 2 ? "SHFL" : "both", ms);
  }
  return 0;
}
