// Micro-benchmark: streaming bandwidth of the H100 memory system as a function of the working
// set (L2-resident vs DRAM), for the access mixes of the two-kernel transform path:
//   read-only, write-only, copy (read + write), and "read a small L2-resident buffer while
//   streaming writes to a large one" (the second kernel with its intermediate kept in L2).
// Build:  nvcc -O3 -gencode arch=compute_90a,code=sm_90a l2_bw.cu -o l2_bw
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__global__ void k_read(const double2 *__restrict__ a, size_t n, double2 *sink) {
  double2 acc = make_double2(0, 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    double2 v = a[i];
    acc.x += v.x; acc.y += v.y;
  }
  if (acc.x == 1.2345e300) sink[0] = acc;
}
__global__ void k_write(double2 *__restrict__ a, size_t n, int streaming) {
  const double2 v = make_double2(1.0, 2.0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (streaming) __stcs(&a[i], v); else a[i] = v;
  }
}
__global__ void k_copy(const double2 *__restrict__ a, double2 *__restrict__ b, size_t n, int streaming) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    double2 v = a[i];
    if (streaming) __stcs(&b[i], v); else b[i] = v;
  }
}
// read src (nsrc elements, cycled) and stream-write dst (ndst elements): ndst/nsrc passes over src
__global__ void k_mix(const double2 *__restrict__ src, size_t nsrc, double2 *__restrict__ dst, size_t ndst) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < ndst; i += (size_t)gridDim.x * blockDim.x) {
    double2 v = src[i % nsrc];
    __stcs(&dst[i], v);
  }
}

template <class F> float timeit(F f, int reps) {
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  f();
  CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(e0));
  for (int i = 0; i < reps; ++i) f();
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  return ms / reps;
}

int main() {
  const size_t big = (size_t)1 << 30;   // bytes
  double2 *A, *B, *sink;
  CK(cudaMalloc(&A, big)); CK(cudaMalloc(&B, big)); CK(cudaMalloc(&sink, 64));
  CK(cudaMemset(A, 1, big)); CK(cudaMemset(B, 1, big));
  const int grid = 132 * 8, block = 256;
  const size_t sizes_mb[] = {4, 8, 16, 24, 32, 48, 64, 96, 128, 256, 1024};
  printf("working set MB | read GB/s | write GB/s | write.cs GB/s | copy(r+w) GB/s | copy.cs GB/s\n");
  for (size_t mb : sizes_mb) {
    const size_t n = (mb << 20) / sizeof(double2);
    const int reps = mb <= 128 ? 50 : 10;
    const float tr = timeit([&] { k_read<<<grid, block>>>(A, n, sink); }, reps);
    const float tw = timeit([&] { k_write<<<grid, block>>>(A, n, 0); }, reps);
    const float tws = timeit([&] { k_write<<<grid, block>>>(A, n, 1); }, reps);
    const size_t nh = n / 2;   // copy: half the working set each
    const float tc = timeit([&] { k_copy<<<grid, block>>>(A, A + nh, nh, 0); }, reps);
    const float tcs = timeit([&] { k_copy<<<grid, block>>>(A, A + nh, nh, 1); }, reps);
    const double bytes = (double)n * sizeof(double2);
    printf("%6zu | %8.0f | %8.0f | %8.0f | %8.0f | %8.0f\n", mb, bytes / tr / 1e6, bytes / tw / 1e6,
           bytes / tws / 1e6, bytes / tc / 1e6, bytes / tcs / 1e6);
  }
  printf("mix: read an L2-resident source while streaming 1 GB of writes (GB/s counted on the WRITES)\n");
  const size_t src_mb[] = {8, 16, 32, 64, 1024};
  for (size_t mb : src_mb) {
    const size_t ns = (mb << 20) / sizeof(double2), nd = big / sizeof(double2);
    const float t = timeit([&] { k_mix<<<grid, block>>>(A, ns, B, nd); }, 10);
    printf("src %4zu MB: %8.0f GB/s written (+ the same read)\n", mb, (double)big / t / 1e6);
  }
  return 0;
}
