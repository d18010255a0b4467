// Micro-benchmark: the power test's count pass (PowerCountBody without selection bits) against the
// alternative of comparing with a stored |W_obs|^2.  Per scale-point of a unit:
//   A (as the engine does): read W_i and W_obs (complex), form both powers, read + write the uint32
//     counter: 2 x 16 + 8 = 40 B in fp64, 2 x 8 + 8 = 24 B in fp32;
//   B: read W_i and a stored double P_obs, read + write the counter: 16 + 8 + 8 = 32 B in fp64, and
//     8 + 8 + 8 = 24 B in fp32 (a double P_obs is as large as an fp32 W_obs).
// B also holds 8 B per point more on the device while the power is resident.  Both kernels have the
// engine's launch shape (128 threads, one per column, grid (columns / 128, rows)) and its loads
// (streaming, __ldcs) and power arithmetic (__dmul_rn / __dadd_rn); the counts of the two variants
// are checked equal.  Sizes: config 4 (145 x 2^18) and config 2 (256 x 2^20).  Median of --reps
// timed launches per variant, the variants alternating, with the card's name and clocks printed.
// Build:  nvcc -O3 -gencode arch=compute_90a,code=sm_90a power_count_ab.cu -o /tmp/power_count_ab
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

template <typename C> __device__ __forceinline__ double pw(const C &v) {
  return __dadd_rn(__dmul_rn((double)v.x, (double)v.x), __dmul_rn((double)v.y, (double)v.y));
}

template <typename C>
__global__ void __launch_bounds__(128) k_obs(const C *W, const C *obs, unsigned *cnt, long long n) {
  const long long c = (long long)blockIdx.x * 128 + threadIdx.x;
  if (c >= n) return;
  const size_t o = (size_t)blockIdx.y * n + c;
  const double P = pw(__ldcs(&W[o]));
  if (!isfinite(P) || P >= pw(__ldcs(&obs[o]))) cnt[o] += 1u;
}

template <typename C>
__global__ void __launch_bounds__(128) k_stored(const C *W, const double *Pobs, unsigned *cnt, long long n) {
  const long long c = (long long)blockIdx.x * 128 + threadIdx.x;
  if (c >= n) return;
  const size_t o = (size_t)blockIdx.y * n + c;
  const double P = pw(__ldcs(&W[o]));
  if (!isfinite(P) || P >= __ldcs(&Pobs[o])) cnt[o] += 1u;
}

template <typename C> __global__ void k_fill(C *a, size_t m, unsigned seed) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (size_t)gridDim.x * blockDim.x) {
    unsigned h = (unsigned)i * 2654435761u ^ seed;
    h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
    a[i].x = (h & 0xFFFF) / 65536.0f - 0.5f;
    a[i].y = (h >> 16) / 65536.0f - 0.5f;
  }
}
template <typename C> __global__ void k_pow(const C *a, double *p, size_t m) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (size_t)gridDim.x * blockDim.x)
    p[i] = pw(a[i]);
}

template <typename C>
void run(const char *name, int S, long long n, int reps) {
  const size_t m = (size_t)S * n;
  C *W, *obs;
  double *P;
  unsigned *ka, *kb;
  CK(cudaMalloc(&W, m * sizeof(C)));
  CK(cudaMalloc(&obs, m * sizeof(C)));
  CK(cudaMalloc(&P, m * sizeof(double)));
  CK(cudaMalloc(&ka, m * 4));
  CK(cudaMalloc(&kb, m * 4));
  k_fill<<<1024, 256>>>(W, m, 1u);
  k_fill<<<1024, 256>>>(obs, m, 2u);
  k_pow<<<1024, 256>>>(obs, P, m);
  CK(cudaMemset(ka, 0, m * 4));
  CK(cudaMemset(kb, 0, m * 4));
  const dim3 grid((unsigned)((n + 127) / 128), (unsigned)S);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  std::vector<float> ta, tb;
  for (int r = 0; r < reps + 2; ++r) {   // two warm-up rounds
    float t;
    CK(cudaEventRecord(e0));
    k_obs<C><<<grid, 128>>>(W, obs, ka, n);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&t, e0, e1));
    if (r >= 2) ta.push_back(t);
    CK(cudaEventRecord(e0));
    k_stored<C><<<grid, 128>>>(W, P, kb, n);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&t, e0, e1));
    if (r >= 2) tb.push_back(t);
  }
  CK(cudaGetLastError());
  std::vector<unsigned> ha(m), hb(m);
  CK(cudaMemcpy(ha.data(), ka, m * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hb.data(), kb, m * 4, cudaMemcpyDeviceToHost));
  const bool same = ha == hb;
  std::sort(ta.begin(), ta.end());
  std::sort(tb.begin(), tb.end());
  const double bA = (double)m * (2 * sizeof(C) + 8), bB = (double)m * (sizeof(C) + 16);
  const double mA = ta[ta.size() / 2], mB = tb[tb.size() / 2];
  printf("%-22s A (W_obs): %.3f ms (%.3f-%.3f) %.2f TB/s | B (stored P_obs): %.3f ms (%.3f-%.3f) %.2f TB/s | "
         "B/A %.3f | counts equal: %s\n", name, mA, ta.front(), ta.back(), bA / mA / 1e9, mB, tb.front(), tb.back(),
         bB / mB / 1e9, mB / mA, same ? "yes" : "NO");
  for (void *p : {(void *)W, (void *)obs, (void *)P, (void *)ka, (void *)kb}) CK(cudaFree(p));
  CK(cudaEventDestroy(e0));
  CK(cudaEventDestroy(e1));
}

int main(int argc, char **argv) {
  const int reps = argc > 1 ? atoi(argv[1]) : 20;
  cudaDeviceProp p;
  CK(cudaGetDeviceProperties(&p, 0));
  printf("device: %s, %d SMs, reps %d\n", p.name, p.multiProcessorCount, reps);
  run<double2>("config 4 fp64 145x2^18", 145, 1ll << 18, reps);
  run<float2>("config 4 fp32 145x2^18", 145, 1ll << 18, reps);
  run<double2>("config 2 fp64 256x2^20", 256, 1ll << 20, reps);
  return 0;
}
