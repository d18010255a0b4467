// Micro-benchmark: streaming bandwidth of the H100 memory system as a function of the working
// set (L2-resident vs DRAM), for the access mixes of the two-kernel transform path:
//   read-only, write-only, copy (read + write), and "read a small L2-resident buffer while
//   streaming writes to a large one" (the second kernel with its intermediate kept in L2).
// Then the write roof of the fp64 expansion kernel's store patterns on a 4 GiB buffer: coalesced
// st.global.cs, two 16-byte stores per lane 32 bytes apart (as is and with lane pairs exchanged), and
// shared-memory staging written by cp.async.bulk in 1 KiB and 128 B runs.  H100 SXM at 400 W (GB/s):
//   coalesced 3190-3200 | pair 1543-1549 | pair exchanged 3224-3233 | bulk 1 KiB 3157-3169 | bulk 128 B 2942-2948
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

// ---- write patterns of the fp64 expansion kernel (ExpandMmaBody), each warp owning 1 KiB chunks ----
// pair16: two 16-byte streaming stores per lane, lanes 32 bytes apart (the MMA C fragment stored as is):
//         every 32-byte sector is half-written by one instruction and half by the next
// xchg16: the same two stores after lanes q and q^1 swap one value: each instruction writes whole sectors
__global__ void k_write_pair16(double2 *__restrict__ a, size_t nchunk, int xchg) {
  const int lane = threadIdx.x & 31;
  const size_t w0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((size_t)gridDim.x * blockDim.x) >> 5;
  const double2 v = make_double2(1.0, 2.0);
  for (size_t c = w0; c < nchunk; c += nw) {
    double2 *p = a + c * 64 + 2 * lane;
    if (xchg) {
      const int odd = lane & 1;
      __stcs(p - odd, v);       // even lane: its x0; odd lane: its partner's x1
      __stcs(p + 2 - odd, v);   // even lane: its partner's x0; odd lane: its x1
    } else {
      __stcs(p, v);
      __stcs(p + 1, v);
    }
  }
}
// bulk: the warp stages its 1 KiB chunk in shared memory (ring of 4 slots per warp) and one lane writes
// it with cp.async.bulk (L2 evict-first hint) as 1024 / RUN runs of RUN bytes
template <int RUN> __global__ void k_write_bulk(double2 *__restrict__ a, size_t nchunk) {
  __shared__ __align__(128) double2 ring[4][4][64];   // [warp][slot][1 KiB]
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t w0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((size_t)gridDim.x * blockDim.x) >> 5;
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  int slot = 0;
  for (size_t c = w0; c < nchunk; c += nw) {
    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 3;" ::: "memory");
    __syncwarp();
    double2 *s = ring[wid][slot];
    s[2 * lane] = make_double2(1.0, 2.0);
    s[2 * lane + 1] = make_double2(1.0, 2.0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
    if (lane == 0) {
      for (int r = 0; r < 1024 / RUN; ++r) {
        const unsigned sa = (unsigned)__cvta_generic_to_shared((char *)s + r * RUN);
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                     ::"l"((char *)(a + c * 64) + r * RUN), "r"(sa), "n"(RUN), "l"(pol) : "memory");
      }
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    slot = (slot + 1) & 3;
  }
  if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
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
  CK(cudaFree(A)); CK(cudaFree(B));
  // write roof of the expansion kernel's store patterns: a 4 GiB buffer (~ W of config 2), 128-thread CTAs
  const size_t huge = (size_t)4 << 30, nchunk = huge / 1024;
  double2 *H;
  CK(cudaMalloc(&H, huge));
  CK(cudaMemset(H, 1, huge));
  const size_t nh = huge / sizeof(double2);
  const int g128 = 132 * 16;
  printf("write patterns, 4 GiB buffer (GB/s):\n");
  for (int rep = 0; rep < 3; ++rep) {
    const float ta = timeit([&] { k_write<<<g128, 128>>>(H, nh, 1); }, 5);
    const float tb = timeit([&] { k_write_pair16<<<g128, 128>>>(H, nchunk, 0); }, 5);
    const float td = timeit([&] { k_write_pair16<<<g128, 128>>>(H, nchunk, 1); }, 5);
    const float tc1 = timeit([&] { k_write_bulk<1024><<<g128, 128>>>(H, nchunk); }, 5);
    const float tc2 = timeit([&] { k_write_bulk<128><<<g128, 128>>>(H, nchunk); }, 5);
    CK(cudaGetLastError());
    printf("  (a) coalesced st.cs %6.0f | (b) pair16 st.cs %6.0f | (b') pair16 exchanged %6.0f | "
           "(c) bulk 1 KiB %6.0f | (c) bulk 128 B %6.0f\n", huge / ta / 1e6, huge / tb / 1e6, huge / td / 1e6,
           huge / tc1 / 1e6, huge / tc2 / 1e6);
  }
  CK(cudaFree(H));
  return 0;
}
