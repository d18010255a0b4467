// H100-native CWT engine: host planning, kernel launches and the C ABI of
// include/cwt_b200.h.  Device code is in kernels.cuh / fft_tile.cuh / cplx.cuh.
//
// Build (sm_90a):    nvcc -std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a
//                         -Xcompiler -fPIC -shared engine.cu -o libcwtb200.so
// Build (CPU emulation of the kernels, TESTS ONLY, never shipped/loaded by the package):
//                    nvcc -std=c++17 -O2 -DCWTB_HOST_EMU ... -o libcwtb200_emu.so
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <type_traits>
#include <vector>

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <initializer_list>

#include "../../include/cwt_b200.h"
#include "kernels.cuh"

using namespace cwtb;

// threads per CTA of a kernel body: Body::NTB if it declares one (tile kernels: per precision),
// else the global NT
template <class B, class = void> struct BodyNT { static constexpr int value = NT; };
template <class B> struct BodyNT<B, std::void_t<decltype(B::NTB)>> { static constexpr int value = B::NTB; };


// ======================================================================================
// runtime abstraction
// ======================================================================================
// Everything the host code asks of the CUDA runtime goes through these wrappers, so that the
// emulation build runs the same host control flow.  There, streams and events are plain handles:
// every launch runs to completion in the order it is issued, which satisfies every wait, so
// recording, waiting and synchronising do nothing and no time elapses.
#ifdef CWTB_HOST_EMU
typedef int rt_stream;
typedef int rt_event;
static inline int rt_malloc(void **p, size_t n) { *p = malloc(n ? n : 1); return *p ? 0 : 1; }
static inline int rt_free(void *p) { free(p); return 0; }
static inline int rt_host_alloc(void **p, size_t n) { *p = malloc(n ? n : 1); return *p ? 0 : 1; }
static inline int rt_host_free(void *p) { free(p); return 0; }
static inline int rt_h2d(void *d, const void *s, size_t n, rt_stream) { memcpy(d, s, n); return 0; }
static inline int rt_d2h(void *d, const void *s, size_t n, rt_stream) { memcpy(d, s, n); return 0; }
static inline int rt_memset(void *d, int v, size_t n, rt_stream) { memset(d, v, n); return 0; }
static inline int rt_sync(rt_stream) { return 0; }
static inline const char *rt_errstr(int) { return "emulation error"; }
static inline int rt_event_create(rt_event *e) { *e = 0; return 0; }
static inline int rt_event_create_sync(rt_event *e) { *e = 0; return 0; }
static inline int rt_event_destroy(rt_event) { return 0; }
static inline int rt_record(rt_event, rt_stream) { return 0; }
static inline int rt_wait(rt_stream, rt_event) { return 0; }
static inline int rt_event_sync(rt_event) { return 0; }
static inline int rt_elapsed_ms(float *ms, rt_event, rt_event) { *ms = 0; return 0; }
static inline int rt_stream_create(rt_stream *s) { *s = 0; return 0; }
static inline int rt_stream_create_highest(std::initializer_list<rt_stream *> ss) {
  for (rt_stream *s : ss) *s = 0;
  return 0;
}
static inline int rt_stream_destroy(rt_stream) { return 0; }
static inline int rt_set_device(int) { return 0; }
static inline int rt_device_count(int *n) { *n = 1; return 0; }
static inline int rt_sm_count(int *, int) { return 0; }   // keeps the caller's value
#else
typedef cudaStream_t rt_stream;
typedef cudaEvent_t rt_event;
static inline int rt_malloc(void **p, size_t n) { return (int)cudaMalloc(p, n ? n : 1); }
static inline int rt_free(void *p) { return (int)cudaFree(p); }
static inline int rt_host_alloc(void **p, size_t n) { return (int)cudaHostAlloc(p, n ? n : 1, cudaHostAllocDefault); }
static inline int rt_host_free(void *p) { return (int)cudaFreeHost(p); }
static inline int rt_h2d(void *d, const void *s, size_t n, rt_stream st) {
  return (int)cudaMemcpyAsync(d, s, n, cudaMemcpyHostToDevice, st);
}
static inline int rt_d2h(void *d, const void *s, size_t n, rt_stream st) {
  return (int)cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToHost, st);
}
static inline int rt_memset(void *d, int v, size_t n, rt_stream st) { return (int)cudaMemsetAsync(d, v, n, st); }
static inline int rt_sync(rt_stream st) { return (int)cudaStreamSynchronize(st); }
static inline const char *rt_errstr(int e) { return cudaGetErrorString((cudaError_t)e); }
static inline int rt_event_create(rt_event *e) { return (int)cudaEventCreate(e); }
static inline int rt_event_create_sync(rt_event *e) { return (int)cudaEventCreateWithFlags(e, cudaEventDisableTiming); }
static inline int rt_event_destroy(rt_event e) { return (int)cudaEventDestroy(e); }
static inline int rt_record(rt_event e, rt_stream st) { return (int)cudaEventRecord(e, st); }
static inline int rt_wait(rt_stream st, rt_event e) { return (int)cudaStreamWaitEvent(st, e, 0); }
static inline int rt_event_sync(rt_event e) { return (int)cudaEventSynchronize(e); }
static inline int rt_elapsed_ms(float *ms, rt_event e0, rt_event e1) { return (int)cudaEventElapsedTime(ms, e0, e1); }
static inline int rt_stream_create(rt_stream *s) { return (int)cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); }
// streams of the device's highest priority; every one is created, the first error is returned
static inline int rt_stream_create_highest(std::initializer_list<rt_stream *> ss) {
  int lo = 0, hi = 0;   // numerically lower = higher priority
  int e = (int)cudaDeviceGetStreamPriorityRange(&lo, &hi);
  for (rt_stream *s : ss) {
    const int r = (int)cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, hi);
    if (!e) e = r;
  }
  return e;
}
static inline int rt_stream_destroy(rt_stream st) { return (int)cudaStreamDestroy(st); }
static inline int rt_set_device(int d) { return (int)cudaSetDevice(d); }
static inline int rt_device_count(int *n) { return (int)cudaGetDeviceCount(n); }
static inline int rt_sm_count(int *n, int d) { return (int)cudaDeviceGetAttribute(n, cudaDevAttrMultiProcessorCount, d); }

template <class B, class = void> struct BodyMinB { static constexpr int value = CWTB_MINB; };
template <class B> struct BodyMinB<B, std::void_t<decltype(B::MINB)>> { static constexpr int value = B::MINB; };

template <class Body, int PH>
__device__ __forceinline__ void run_phases(const typename Body::Args &a, void *sm) {
  Body::template phase<PH>(a, (int)blockIdx.x, (int)blockIdx.y, (int)threadIdx.x, sm);
  if constexpr (PH + 1 < Body::NPHASE) {
    __syncthreads();
    run_phases<Body, PH + 1>(a, sm);
  }
}
template <class Body>
__global__ void __launch_bounds__(BodyNT<Body>::value, BodyMinB<Body>::value) k_run(const __grid_constant__ typename Body::Args a) {
  extern __shared__ __align__(16) unsigned char smraw[];
  run_phases<Body, 0>(a, smraw);
}
// persistent kernel of a body with run_tiles(): `total` work items of which `gm` per row
template <class Body>
__global__ void __launch_bounds__(Body::NTB, Body::MINB) k_persist(const __grid_constant__ typename Body::Args a,
                                                                   unsigned gm, unsigned total) {
  extern __shared__ __align__(16) unsigned char smraw[];
  Body::run_tiles(a, gm, total, (typename Body::V *)smraw);
}
#endif

// ======================================================================================
// context
// ======================================================================================
struct Buf {
  void *p = nullptr;
  size_t bytes = 0;
};

// longest pruned length K' that one kernel transforms (up to 2^10 SingleBody, above DirectBody);
// longer ones run through the two-kernel path
constexpr int DIRECT_MAX_LOG2 = 13;

struct ClassRun {   // scales sharing one execution plan
  int log2K;        // exact path: pruned length K' = 1 << log2K
  int first, count; // range in the sorted descriptor array
  int expand = 0;   // 1: band-limited expansion path (coarse transform + interpolation)
  int log2Nc = 0;   // expansion: coarse grid length
  int taps = 0;     // expansion: interpolation taps
  long long woff = 0;   // expansion: offset of the class's weight table
  int os = 0;           // overlap-save group + 1 (0: another path)
};

// The clusters of a map, in table order (Q descending, ties by the flat index of the first point):
// Q = sum of q_j over the points, the point count, and the box [row0, row1) x [col0, col1)
struct ClusterTable {
  std::vector<unsigned long long> Q, pts;
  std::vector<long long> box;   // [clusters][4]
};

// A product that one call writes to a device buffer of its own and that later calls read in place
// (cwtb_wct_resident, cwtb_xwt_resident).  serial is bumped before every write and on release.
// The resident transform has the same record (cwtb_ctx::wt) without a buffer: W stays scratch.
struct ResidentSlot {
  Buf buf;
  int S = 0;                     // rows resident (0: none)
  long long n0 = 0;
  int prec = 0;
  long long serial = 0;
  // the coherence slots: surrogate exceedance counts of the resident fields, uint32 [S][n0] per
  // measure (cwtb_coherence*_surrogate_counts), and the units they hold (-1: none readable)
  Buf counts;
  long long units = -1;
  int null = CWTB_NULL_PHASE;    // the coherence slots: the null of the units counted (cwtb_null)
  // the coherence slots: the observed clusters of the last cwtb_coherence*_cluster_test, the label
  // image int32 [S][n0] (0: no cluster, c + 1: row c of the table) and the table, valid with
  // `clusters`
  Buf labels;
  ClusterTable table;
  bool clusters = false;
};

// A call that writes a slot invalidates it first, so that one failing part-way leaves none resident
// (and no counts or clusters of an earlier product readable)
static void slot_begin(ResidentSlot &s) {
  ++s.serial;
  s.S = 0;
  s.n0 = 0;
  s.units = -1;
  s.clusters = false;
  s.table = ClusterTable{};
}

// overlap-save plan of one input scale (os_plan): group + 1 (0: not overlap-save), kept taps
// [t1 - M + 1, t1] of its impulse response, offset of its H in the context's H buffer
struct OsRow { int grp = 0, t1 = 0, M = 0; long long hoff = 0; };

struct Job {
  bool valid = false;
  int precision = 0;       // CWTB_F64 / CWTB_F32
  long long n0 = 0;
  unsigned N = 0;
  int log2N = 0;
  int S = 0;          // scales per channel
  int nbatch = 1;     // channels transformed together (rows = nbatch * S)
  double dt = 0;
  Fam fam{};
  std::vector<ScaleDesc> descs;   // sorted by class
  std::vector<ClassRun> classes;
  std::vector<int> plan_log2K;    // per input scale
  std::vector<double> scales;     // per input scale (= output row)
  size_t b_single = 0;            // elements of the band buffer used by single-kernel scales
  size_t coarse_elems = 0;        // elements of the coarse buffers used by the expansion rows
  int sig_is_f32 = 0;
  bool exact = false;             // un-padded mode: N = n0 (not a power of two), Bluestein transforms
  std::vector<OsGroup> os_groups; // overlap-save groups (uploaded to cwtb_ctx::osgrp)
};

struct BluePlan {   // chirp tables of one transform length (device memory, owned by the context)
  unsigned n = 0, L = 0;
  double2 *wm = nullptr;                 // e^{-i pi k^2 / n}, k < n
  double2 *bf[2] = {nullptr, nullptr};   // FFT_L of the chirp filter for sign -1 / +1
};

struct NTabDev {
  double2 *hi = nullptr, *lo = nullptr;
  int h = 0;
};

struct cwtb_ctx {
  int device = 0;
  rt_stream stream{};
  rt_stream aux_stream{};        // single-kernel classes run here, concurrently with the two-kernel chains
  rt_stream prio_stream{};       // highest-priority stream: the coarse transforms in front of the expansion
                                 // kernels (coarse lengths above 1024) -- its CTAs are dispatched before the
                                 // pending CTAs of the big launches on the other streams
  rt_stream prio_short{};        // the same priority: the coarse transforms of lengths up to 1024
  int prio_mode = 1;             // CWTB_PRIO: 0 = no priority stream, 1 = coarse chain, 2 = coarse chain and
                                 // the expansion kernels
  rt_stream chain_streams[3]{};  // two-kernel classes rotate over the engine's stream and these (own Z
                                 // and band-chunk region per chain)
  int n_chains = 2;              // chains in use, 1..4 (CWTB_CHAINS)
  rt_stream cur{};               // stream the launcher uses right now
  int pad_pow2 = 1;              // 1: transform length = next power of two (reference default,
                                 // helpers.py:27-30); 0: the signal's own length (pyfftw policy,
                                 // helpers.py:15-19) -- cwtb_set_padding
  int coh_precision = 0;         // arithmetic of xwt / wct / wct_mc: CWTB_F64 or CWTB_F32
                                 // (cwtb_set_coherence_precision)
  std::map<unsigned, BluePlan> blue;
  rt_stream copy_streams[2]{};   // device->host copies that overlap the kernels or each other
  std::string err;
  double band_eps = 1e-16;
  double band_eps32 = 1e-9;      // fp32 engine: pruning threshold matched to the arithmetic (fp32
                                 // rounding is 6e-8; the dropped terms stay two orders below it)
  double expand_eps = 5e-13;     // fp64 engine: bound on the aliasing error of the expansion path
                                 // (0: path off, every scale through the exact pruned transforms)
  double expand_eps32 = 2e-7;    // fp32 engine
  int expand_mma = 1;            // fp64 expansion kernels with DMMA tap sums (CWTB_EXPAND_MMA=0: scalar kernel)
  int dense_margin = 2;          // pruned lengths within this many octaves of Np run as dense scales
                                 // (CWTB_DENSE_MARGIN)
  int expand_min_log2R = 0;      // log2 of the smallest Np / Nc (CWTB_EXPAND_MIN_R); 0: by kernel, see build_job
  int os_on = 1;                 // overlap-save rows (OsBody; CWTB_OS=0: off)
  Buf osH, osgrp;                // overlap-save: DFT_L of the truncated impulse responses, group table
  void *comm = nullptr;          // ncclComm_t of cwtb_comm_init (one rank per context)
  int comm_world = 1, comm_rank = 0;
  Buf comm_send, comm_recv;      // device staging of the host-buffer collectives
  int group = 0;   // rows per two-kernel chunk; 0 = as many as fit in group_bytes of Z (CWTB_GROUP)
  size_t group_bytes = (size_t)512 << 20;
  int num_sms = 132;
  int pf_dist = 132;   // PassB: L2 prefetch distance in tiles, one per SM of an H100 (CWTB_PF_DIST)
  int pf_rows_a = 32, pf_rows_b = 32;   // the same for the batched row transforms (CWTB_PF_ROWS_A / _B)
  int pf_dist_a = 132;  // PassA (band): L2 prefetch distance in tiles (CWTB_PF_DIST_A)
  size_t batch_bytes = (size_t)4 << 30;   // coefficients per chunk of cwtb_cwt_batch
  double2 *tw64 = nullptr;
  float2 *tw32 = nullptr;
  std::map<unsigned, NTabDev> ntabs;
  Buf filt;                      // caller-supplied time-smoothing responses [S][N] (cwtb_set_smooth_filter)
  int filt_rows = 0;
  long long filt_n = 0;
  double morse_ga = 3.0;         // shape parameter of CWTB_MORSE (cwtb_set_morse_ga)
  Buf Zx, Cout, wtab;            // expansion path: intermediate of the coarse transforms, coarse samples,
                                 // interpolation weight tables
  std::map<std::array<long long, 3>, long long> wtab_index;   // (log2R, taps, round(beta*1e6)) -> offset
  std::vector<double> wtab_host; // host mirror of wtab (tables are appended, never moved)
  size_t wtab_uploaded = 0;      // elements already on the device
  size_t wtab_max_bytes = (size_t)256 << 20;   // CWTB_WTAB_MB: host mirror size above which the cache starts over
  Buf sig, sig2, sig3, spec, Z, Zc[3], Y, B, W, W2, W3, descs, table, scratch, C, A12, F, aux, rowd, win, mask, hist, noise, wide, blueA, blueX, blueY, pspec, prot;
  // cluster tests: the selection bitmask, its per-row arguments (thr, lo, hi, q), the chunk and row
  // tables of the labeller, its run tables (sized from the run count of each map), the units' maxima
  Buf cl_bits, cl_rows, cl_hdr, cl_runs, cl_qmax;
  Buf arc;                       // AR(1) surrogates: the CTAs' (g^L, b) pairs and carry-ins (Ar1Args::blk)
  Job job;
  // what the resident plan (job + uploaded descriptors) was built from: a call with the same
  // geometry and settings reuses it (planning + descriptor upload: ~0.3 ms for 256 scales, several ms
  // for the 8192 rows of a batch chunk)
  struct PlanKey {
    long long n0 = -1;
    double dt = 0, param = 0, band_eps = 0, band_eps32 = 0, expand_eps = 0, expand_eps32 = 0;
    double ga = 0;                 // Morse's shape parameter (0 for the other families)
    int S = 0, family = 0, precision = 0, nbatch = 0, pad = 0;
    std::vector<double> scales;
    bool operator==(const PlanKey &o) const {
      return n0 == o.n0 && dt == o.dt && param == o.param && ga == o.ga && band_eps == o.band_eps && band_eps32 == o.band_eps32 &&
             expand_eps == o.expand_eps && expand_eps32 == o.expand_eps32 && S == o.S && family == o.family &&
             precision == o.precision && nbatch == o.nbatch && pad == o.pad && scales == o.scales;
    }
  } plan_key;
  int plan_reuse = 1;            // CWTB_PLAN_REUSE=0: plan every call
  // cwtb_cwt_batch pipeline: two page-locked staging buffers and two device input buffers so that the
  // host copy and the H2D of chunk k+1 overlap the kernels of chunk k; per-row power of every chunk is
  // accumulated on the device and read back once
  void *stage_host[2] = {nullptr, nullptr};
  size_t stage_bytes = 0;
  Buf stage_dev[2], batch_power;
  int batch_pipeline = 1;        // CWTB_BATCH_PIPELINE=0: one synchronous chunk after the other
  double *angle_host = nullptr;  // cwtb_wct: host destination of the phase angle, copied on a copy stream
                                 // as soon as it exists (before the smoothing transforms), not after them
  // resident coherence (cwtb_wct_resident): WCT [S][n0], aWCT at coh_angle_offset(S*n0), double.
  // Only cwtb_wct_resident writes this slot, so it outlives any other call.
  ResidentSlot coh;
  // resident cross spectrum (cwtb_xwt_resident): W12 [S][n0] of precision prec.
  // cwtb_xwt_resident hands its transform's W over by swapping the two buffers, so W12 is never
  // copied and the old cross buffer becomes the next transform's W.  Nothing else writes it.
  ResidentSlot cross;
  // resident partial and multiple coherence (cwtb_wct3_resident): RP2 [S][n0], the partial phase at
  // coh_angle_offset(S*n0), RM2 at twice that offset, double.  Only cwtb_wct3_resident writes it.
  ResidentSlot coh3;
  // resident wavelet power (cwtb_power_resident): its transform's W [S][n0] of precision prec, handed
  // over by swapping buffers as cwtb_xwt_resident does, with the power tests' counts and clusters.
  // Only cwtb_power_resident writes it.
  ResidentSlot pw;
  // resident transform: rows = scales x channels of the complete W in the scratch buffer W, of
  // precision prec.  prepare opens it (serial: cwtb_job_serial); only a transform entry point that
  // completes fills it (w_fill), so while it is filled `job` is the plan it was filled from.
  ResidentSlot wt;
  const void *job_dsig = nullptr;  // device signal of the last cwt_dev call (not owned)
  double last_ms = 0;
  int launches = 0;
  std::set<const void *> configured;
  // per-launch event profiling (cwtb_profile_last)
  bool profiling = false;        // also puts a transform's kernels on one stream (run_job): per-kernel times
                                 // are not blurred by overlap
  const char *prof_tag = "";     // prefix of the kernel names recorded while profiling: "fwd:" (forward
                                 // transform of the signal), "coarse:" (coarse-grid transforms of the
                                 // expansion path), "data:" / "phase:" (spectra of the data and generation of
                                 // their phase-randomised surrogates); W-writing launches carry no tag
  struct ProfRec { std::string name; unsigned gx, gy; int ev; };
  std::vector<ProfRec> prof;
  std::vector<rt_event> prof_events;
  std::set<void *> pinned, devallocs;
  rt_event e0{}, e1{};
  rt_event ev_fork{}, ev_join{}, ev_joinc[3]{}, ev_coarse{}, ev_coarse_short{};
  rt_event ev_h2d[2]{}, ev_used[2]{};
  rt_event ev_angle{};
};

static int fail(cwtb_ctx *c, int code, const std::string &msg) {
  if (c) c->err = msg;
  return code;
}
#define RT(call)                                                                             \
  do {                                                                                       \
    int e_ = (call);                                                                         \
    if (e_ != 0) return fail(c, CWTB_ERR_CUDA, std::string(#call) + ": " + rt_errstr(e_));   \
  } while (0)

static int ensure(cwtb_ctx *c, Buf &b, size_t bytes) {
  if (b.bytes >= bytes && b.p) return 0;
  if (b.p) rt_free(b.p);
  b.p = nullptr;
  b.bytes = 0;
  if (rt_malloc(&b.p, bytes) != 0) return fail(c, CWTB_ERR_NOMEM, "device allocation failed");
  b.bytes = bytes;
  return 0;
}

// ======================================================================================
// launcher
// ======================================================================================
#ifdef CWTB_HOST_EMU
template <class Body, int PH>
static void emu_phases(const typename Body::Args &a, int bx, int by, void *sm) {
  for (int tid = 0; tid < BodyNT<Body>::value; ++tid) Body::template phase<PH>(a, bx, by, tid, sm);
  if constexpr (PH + 1 < Body::NPHASE) emu_phases<Body, PH + 1>(a, bx, by, sm);
}
#endif

// "... [with Body = cwtb::PassBBody<double, 1>]"  ->  "PassBBody<double, 1>"
static std::string body_name(const char *pretty) {
  std::string s(pretty);
  size_t i = s.find("Body = ");
  if (i == std::string::npos) return s;
  s = s.substr(i + 7);
  size_t j = s.find_first_of(";]");
  if (j != std::string::npos) s = s.substr(0, j);
  if (s.rfind("cwtb::", 0) == 0) s = s.substr(6);
  return s;
}

constexpr unsigned MAX_ROWS = 65535;   // gridDim.y: rows of one launch

// What every launch of Body shares: an empty grid launches nothing, at most MAX_ROWS rows,
// and while profiling the launch is recorded under the body's name between an event pair.
// `dispatch()` launches on c->cur and returns 0 or an error.
template <class Body, class Dispatch>
static int launch_rec(cwtb_ctx *c, unsigned gx, unsigned gy, Dispatch &&dispatch) {
  if (gx == 0 || gy == 0) return 0;
  if (gy > MAX_ROWS) return fail(c, CWTB_ERR_ARG, "too many rows in one launch");
  int ev = -1;
  if (c->profiling) {
    ev = (int)c->prof.size() * 2;
    while ((int)c->prof_events.size() < ev + 2) {
      rt_event e;
      RT(rt_event_create(&e));
      c->prof_events.push_back(e);
    }
    c->prof.push_back({std::string(c->prof_tag) + body_name(__PRETTY_FUNCTION__), gx, gy, ev});
    RT(rt_record(c->prof_events[ev], c->cur));
  }
  int e = dispatch();
  if (e) return e;
  if (ev >= 0) RT(rt_record(c->prof_events[ev + 1], c->cur));
  c->launches++;
  return 0;
}

template <class Body>
static int launch(cwtb_ctx *c, unsigned gx, unsigned gy, const typename Body::Args &a) {
  return launch_rec<Body>(c, gx, gy, [&]() -> int {
#ifdef CWTB_HOST_EMU
    std::vector<unsigned char> smv(Body::SMEM + 64);
    unsigned char *sm = smv.data();
    sm += (16 - ((unsigned long long)sm & 15)) & 15;   // 16-byte aligned base, like the device's
    for (unsigned by = 0; by < gy; ++by)
      for (unsigned bx = 0; bx < gx; ++bx) emu_phases<Body, 0>(a, (int)bx, (int)by, sm);
    if (emu_bulk_copy_faults() != 0) {
      emu_bulk_copy_faults() = 0;
      return fail(c, CWTB_ERR_CUDA, "emulation: bulk-async copy with a misaligned address or size");
    }
#else
    const void *fn = (const void *)k_run<Body>;
    if (Body::SMEM > 48 * 1024 && !c->configured.count(fn)) {
      RT(cudaFuncSetAttribute(k_run<Body>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Body::SMEM));
      c->configured.insert(fn);
    }
    k_run<Body><<<dim3(gx, gy), BodyNT<Body>::value, Body::SMEM, c->cur>>>(a);
    RT(cudaGetLastError());
#endif
    return 0;
  });
}

// ======================================================================================
// tables
// ======================================================================================
static int make_table(cwtb_ctx *c, double2 *o64, float2 *o32, unsigned count, double step) {
  TabArgs a{o64, o32, count, step};
  return launch<TabBody>(c, (count + NT - 1) / NT, 1, a);
}

static int init_tables(cwtb_ctx *c) {
  RT(rt_malloc((void **)&c->tw64, sizeof(double2) * TW_TOTAL));
  RT(rt_malloc((void **)&c->tw32, sizeof(float2) * TW_TOTAL));
  PassTwArgs a{c->tw64, c->tw32};
  return launch<PassTwBody>(c, (TW_TOTAL + NT - 1) / NT, 1, a);
}

static int get_ntab(cwtb_ctx *c, unsigned N, int log2N, NTab *out) {
  auto it = c->ntabs.find(N);
  if (it == c->ntabs.end()) {
    NTabDev t;
    t.h = (log2N + 1) / 2;
    unsigned nlo = 1u << t.h, nhi = N >> t.h;
    if (nhi == 0) nhi = 1;
    RT(rt_malloc((void **)&t.lo, sizeof(double2) * nlo));
    RT(rt_malloc((void **)&t.hi, sizeof(double2) * nhi));
    int e = make_table(c, t.lo, nullptr, nlo, 1.0 / (double)N);
    if (e) return e;
    e = make_table(c, t.hi, nullptr, nhi, (double)nlo / (double)N);
    if (e) return e;
    it = c->ntabs.emplace(N, t).first;
  }
  out->hi = it->second.hi;
  out->lo = it->second.lo;
  out->h = it->second.h;
  out->lomask = (1u << it->second.h) - 1;
  out->nmask = N - 1;
  return 0;
}

// ======================================================================================
// planning (host): band of each scale -> pruned length K'
// ======================================================================================
static int ilog2(unsigned long long v) {
  int l = 0;
  while ((1ull << l) < v) ++l;
  return l;
}

// largest f (beyond the maximum of g) with  m*ln f - a(f) = target
static double solve_upper(double m, bool gaussian, double target, double fstart) {
  auto g = [&](double f) { return m * std::log(f) - (gaussian ? 0.5 * f * f : f); };
  double lo = fstart, hi = fstart + 1;
  while (g(hi) > target && hi < 1e7) hi *= 2;
  for (int it = 0; it < 200; ++it) {
    double mid = 0.5 * (lo + hi);
    if (g(mid) > target) lo = mid; else hi = mid;
  }
  return hi;
}

// frequency-domain support [flo, fhi] (in f = s*w) where |psi_ft| >= eps * max|psi_ft|
// (ga: Morse's shape parameter, unused by the other families)
static void family_band(int family, double param, double ga, double eps, double *flo, double *fhi, bool *pos_only) {
  const double LN_MIN = -745.2;  // exp() underflows to exactly 0 below this
  const double lneps = eps > 0 ? std::log(eps) : 0;
  *pos_only = false;
  if (family == CWTB_MORSE) {
    // the peak-relative exponent g(u) = be u - (be/ga) expm1(ga u), u = ln(f / f_p), rises to 0 at
    // u = 0 and falls on both sides; its two roots of g = target by bisection in u.  (The value
    // itself carries the constant psi_ft(f_p) = O(1), so the exact-mode floor applies to g as is.)
    const double be = param, bg = be / ga;
    const double target = eps > 0 ? lneps : LN_MIN;
    auto g = [&](double u) { return be * u - bg * std::expm1(ga * u); };
    double lo = (target - bg) / be, hi = 0;    // g(u) <= be u + be/ga: g(lo) <= target
    for (int it = 0; it < 200; ++it) {
      const double mid = 0.5 * (lo + hi);
      if (g(mid) < target) lo = mid; else hi = mid;
    }
    const double ulo = lo;
    lo = 0; hi = 1;
    while (g(hi) > target) hi *= 2;               // expm1 overflows to inf: g = -inf ends it
    for (int it = 0; it < 200; ++it) {
      const double mid = 0.5 * (lo + hi);
      if (g(mid) > target) lo = mid; else hi = mid;
    }
    const double lnfp = std::log(bg) / ga;
    *flo = std::exp(ulo + lnfp);
    *fhi = std::exp(hi + lnfp);
    *pos_only = true;
  } else if (family == CWTB_MORLET) {
    double xc = std::sqrt(-2.0 * (eps > 0 ? lneps : LN_MIN));
    *flo = param - xc;
    *fhi = param + xc;
  } else if (family == CWTB_PAUL) {
    double m = param;
    double target = eps > 0 ? lneps + (m * std::log(m) - m) : LN_MIN;
    *flo = 0;
    *fhi = solve_upper(m, false, target, m);
    *pos_only = true;
  } else {  // DOG
    double m = param;
    double mx = m > 0 ? 0.5 * m * std::log(m) - 0.5 * m : 0.0;
    double target = eps > 0 ? lneps + mx : LN_MIN;
    double fc = solve_upper(m, true, target, std::sqrt(m > 0 ? m : 1.0));
    *flo = -fc;
    *fhi = fc;
  }
}

// ---- band-limited expansion path: Kaiser-Bessel kernel, alias bound, weight tables ------------
// phi(x) = I0(beta sqrt(1 - (2x/w)^2)) / I0(beta) on |x| <= w/2; its transform is
// phi^(xi) = w / I0(beta) * sinh(z)/z, z = sqrt(beta^2 - (pi w xi)^2)  (sin(z)/z beyond the cut-off).
static double kb_hat_shape(double xi, int w, double beta) {   // phi^(xi) * I0(beta) / w
  const double x = M_PI * w * xi;
  const double z2 = beta * beta - x * x;
  const double z = std::sqrt(std::fabs(z2));
  if (z < 1e-8) return 1.0;
  return z2 > 0 ? std::sinh(z) / z : std::sin(z) / z;
}
// max over |xi| <= xi_b of sum_{l != 0} |phi^(xi + l)| / |phi^(xi)|, beta = pi w (1 - xi_b): the
// relative aliasing error of the expansion for a band of half-width xi_b * Nc bins
static double kb_alias_bound(double xi_b, int w) {
  const double beta = M_PI * w * (1.0 - xi_b);
  double worst = 0;
  for (int i = 0; i <= 64; ++i) {
    const double xi = xi_b * i / 64.0;
    double num = 0;
    for (int l = 1; l <= 4; ++l) num += std::fabs(kb_hat_shape(xi + l, w, beta)) + std::fabs(kb_hat_shape(xi - l, w, beta));
    worst = std::max(worst, num / std::fabs(kb_hat_shape(xi, w, beta)));
  }
  return worst;
}
// Buckets of the relative band half-width xi = (band half-width) / Nc and the tap counts tried for
// them.  Beyond xi = 1/4 (coarse grid less than 2x oversampled) the kernel needs 16..20 taps for
// the fp64 tolerance: affordable only where the tap sums run on the tensor cores (ExpandMmaBody),
// `max_taps` says how far the caller may go (16 for the scalar kernels).  The buckets stop at 11/32:
// the coarse spectrum is the band product divided by phi^(xi), and phi^(0) / phi^(xi_b) -- the factor by
// which the rounding noise of the coarse transform can exceed the signal when the energy of the band
// sits at its edge -- is 9 at xi_b = 1/4 (16 taps), 450 at 11/32 (20 taps), 1e4 at 3/8 (24 taps) and
// 1e9 at 7/16 (32 taps; measured on the emulation: 4e-9 error for a Paul scale whose peak is
// off-centre).  450 x 1e-16 stays below the alias tolerance for every signal.
static const double kExpandXi[] = {1.0 / 16, 3.0 / 32, 1.0 / 8, 5.0 / 32, 3.0 / 16, 7.0 / 32, 1.0 / 4,
                                   9.0 / 32, 5.0 / 16, 11.0 / 32};
static const int kExpandBuckets = 10;
static const int kExpandTaps64[] = {10, 12, 14, 16, 20};
static const int kExpandTaps32[] = {6, 8, 10};

// smallest tap count whose alias bound at the bucket of `xi` is <= eps; 0 if none.  *xi_b: bucket.
static int expand_taps(double xi, double eps, bool f32, int max_taps, double *xi_b) {
  // (bucket, taps) -> bound; shared by every context of the process (one per GPU, possibly driven from
  // different host threads)
  static std::map<std::pair<int, int>, double> cache;
  static std::mutex cache_mutex;
  std::lock_guard<std::mutex> cache_lock(cache_mutex);
  int b = -1;
  for (int i = 0; i < kExpandBuckets; ++i)
    if (xi <= kExpandXi[i] * (1 + 1e-12)) { b = i; break; }
  if (b < 0) return 0;
  *xi_b = kExpandXi[b];
  const int *taps = f32 ? kExpandTaps32 : kExpandTaps64;
  const int ntaps = f32 ? 3 : 5;
  for (int i = 0; i < ntaps && taps[i] <= max_taps; ++i) {
    auto key = std::make_pair(b, taps[i]);
    auto it = cache.find(key);
    if (it == cache.end()) it = cache.emplace(key, kb_alias_bound(kExpandXi[b], taps[i])).first;
    if (it->second <= eps) return taps[i];
  }
  return 0;
}

// Dynamic-range check of a candidate (coarse length, taps) beyond xi_b = 1/4: the coarse spectrum is
// the band product divided by phi^(xi); the rounding noise of the coarse transform, relative to the
// largest coarse component, comes back multiplied by up to phi^(0).  Returns
// max_k |psi^(k)| / max|psi^| * phi^(0) / phi^(xi_k) over the band: ~1 when the response peaks at the
// band centre (Morlet, DOG), large when it peaks near an edge (Paul: one-sided band, peak at f = m).
static double expand_gain(const Fam &fam, double s, long long klo, long long khi, long long kc, int log2Nc,
                          int w, double beta) {
  const double Nc = (double)(1ll << log2Nc);
  double peak_amp = 0, worst = 0;
  const double at_centre = beta / std::sinh(beta);
  for (int pass = 0; pass < 2; ++pass)
    for (int i = 0; i <= 256; ++i) {
      const long long k = klo + (long long)std::llround((double)(khi - klo) * i / 256.0);
      const double amp = std::fabs(amp_eval(fam, s, (int)k));
      const double x = M_PI * w * ((double)(k - kc) / Nc);
      const double z = std::sqrt(std::max(beta * beta - x * x, 1e-30));
      const double inv_phi = z / std::sinh(z);          // 1 / phi^ up to a constant
      if (pass == 0) {
        if (amp > peak_amp) peak_amp = amp;
      } else if (peak_amp > 0) {
        worst = std::max(worst, (amp / peak_amp) * (inv_phi / at_centre));
      }
    }
  return worst;
}

// weight table of one class: h[t][rho] = phi(rho / R - (t - (w/2 - 1))), t < w, rho < R (doubles,
// appended to the context's host mirror; uploaded by upload_descs when it grew)
static long long expand_weights(cwtb_ctx *c, std::vector<double> &host, int log2R, int w, double beta) {
  const std::array<long long, 3> key{log2R, w, (long long)std::llround(beta * 1e6)};
  auto it = c->wtab_index.find(key);
  if (it != c->wtab_index.end()) return it->second;
  const long long off = (long long)host.size();
  const int R = 1 << log2R;
  host.resize(host.size() + (size_t)w * R);
  const double i0b = std::cyl_bessel_i(0.0, beta);
  for (int t = 0; t < w; ++t)
    for (int rho = 0; rho < R; ++rho) {
      const double x = (double)rho / R - (double)(t - (w / 2 - 1));
      const double a = 1.0 - (2.0 * x / w) * (2.0 * x / w);
      host[off + (size_t)t * R + rho] = a >= 0 ? std::cyl_bessel_i(0.0, beta * std::sqrt(a)) / i0b : 0.0;
    }
  c->wtab_index.emplace(key, off);
  return off;
}

static int build_job(cwtb_ctx *c, Job &job, long long n0, double dt, const double *scales, int S,
                     int family, double param, int precision, bool have_table, int nbatch = 1,
                     const std::vector<OsRow> *os = nullptr) {
  if (n0 < 1 || S < 1 || !(dt > 0)) return fail(c, CWTB_ERR_ARG, "bad n0 / n_scales / dt");
  if (family < 0 || family > 4) return fail(c, CWTB_ERR_ARG, "unknown wavelet family");
  if (family == CWTB_TABLE && !have_table) return fail(c, CWTB_ERR_ARG, "CWTB_TABLE needs a table");
  if ((family == CWTB_PAUL || family == CWTB_DOG) && (param != std::floor(param) || param < 1 || param > 64))
    return fail(c, CWTB_ERR_ARG, "Paul/DOG order must be an integer in [1, 64]");
  const double ga = c->morse_ga;
  if (family == CWTB_MORSE && !(param >= 1 && param <= 256 && ga >= 1 && ga <= 12))
    return fail(c, CWTB_ERR_ARG, "Morse needs 1 <= be <= 256 and 1 <= ga <= 12");
  if (n0 > (1ll << 28)) return fail(c, CWTB_ERR_UNSUPPORTED, "signal longer than 2^28");
  job = Job();
  job.precision = precision;
  job.n0 = n0;
  job.log2N = ilog2((unsigned long long)n0);   // pycwt/helpers.py:27-30
  job.N = 1u << job.log2N;
  if (!c->pad_pow2 && (n0 & (n0 - 1)) != 0) {
    // un-padded mode (helpers.py:15-19): transform length = n0; a power-of-two n0 is the
    // padded case anyway
    if (precision != CWTB_F64) return fail(c, CWTB_ERR_UNSUPPORTED, "un-padded transforms run in fp64");
    if (nbatch != 1) return fail(c, CWTB_ERR_UNSUPPORTED, "batched transforms need the padded mode");
    if (n0 > (1ll << 24)) return fail(c, CWTB_ERR_UNSUPPORTED, "un-padded transform longer than 2^24");
    job.exact = true;
    job.N = (unsigned)n0;
  }
  job.S = S;
  job.nbatch = nbatch;
  job.dt = dt;
  const unsigned N = job.N;
  Fam &fam = job.fam;
  fam.family = family;
  fam.m = (int)param;
  fam.f0 = param;
  fam.unit = 0;
  fam.dw = 1.0 / ((double)N * dt);
  fam.table = nullptr;
  fam.tpitch = N;
  fam.be = fam.ga = fam.lnfp = fam.bg = 0;
  double fconst = 1.0;
  if (family == CWTB_MORLET) fconst = std::pow(M_PI, -0.25);
  else if (family == CWTB_PAUL) {
    int m = (int)param;
    double fact = 1;
    for (int i = 2; i < 2 * m; ++i) fact *= i;  // prod(range(2, 2m)) = (2m-1)!
    fconst = std::pow(2.0, m) / std::sqrt(m * fact);
  } else if (family == CWTB_DOG) {
    int m = (int)param;
    fconst = 1.0 / std::sqrt(std::tgamma(m + 0.5));
    // conj(-(1j**m)):  m%4: 0 -> -1, 1 -> +i, 2 -> +1, 3 -> -i
    static const int unit_of[4] = {2, 1, 0, 3};
    fam.unit = unit_of[m & 3];
  } else if (family == CWTB_MORSE) {
    const double be = param;
    fam.be = be;
    fam.ga = ga;
    fam.bg = be / ga;
    fam.lnfp = std::log(fam.bg) / ga;
    // psi_ft(f_p) = A f_p^be exp(-f_p^ga), A = sqrt(ga 2^r / Gamma(r)), r = (2be+1)/ga, in logs (both
    // factors overflow for large be, their product is O(1))
    const double r = (2 * be + 1) / ga;
    fconst = std::exp(0.5 * (std::log(ga) + r * std::log(2.0) - std::lgamma(r)) + be * fam.lnfp - fam.bg);
  }
  // ftfreqs[1]; for Np == 2 numpy's fftfreq(2)[1] is -0.5/dt, so the reference's
  // normalisation sqrt(s*w1*Np) is NaN there -- reproduced.
  const double w1 = 6.283185307179586 * ((N == 2 ? -1.0 : 1.0) * fam.dw);
  double flo = 0, fhi = 0;
  bool pos_only = false;
  // eps = 0 (exact mode) applies to both engines
  const double beps = (precision == CWTB_F32 && c->band_eps > 0) ? std::max(c->band_eps, c->band_eps32) : c->band_eps;
  if (family != CWTB_TABLE) family_band(family, param, ga, beps, &flo, &fhi, &pos_only);

  std::vector<ScaleDesc> ds(S);
  job.plan_log2K.assign(S, 0);
  job.scales.assign(scales, scales + S);
  const long long half = (long long)N / 2;
  for (int j = 0; j < S; ++j) {
    ScaleDesc &d = ds[j];
    const double s = scales[j];
    d.s = s;
    d.row = j;
    d.trow = j;
    d.chan = 0;
    d.pad_ = 0;
    d.boff = 0;
    const double norm = std::sqrt(s * w1 * (double)N);  // wavelet.py:103
    d.amp = (family == CWTB_TABLE ? 1.0 : norm * fconst) / (double)N;
    long long klo = -half, khi = ((long long)N - 1) / 2;   // numpy fftfreq's signed bins, any N
    if (family != CWTB_TABLE && s > 0 && std::isfinite(s)) {
      const double cc = (double)N * dt / (6.283185307179586 * s);
      double a = std::ceil(flo * cc) - 1, b = std::floor(fhi * cc) + 1;
      if (a > (double)klo) klo = (long long)a;
      if (b < (double)khi) khi = (long long)b;
      if (pos_only && klo < 1) klo = 1;
    }
    if (N == 1) { klo = 0; khi = 0; }
    if (khi < klo) { klo = 1; khi = 0; }  // empty band: every B is zero
    d.k_lo = (int)klo;
    d.k_hi = (int)khi;
    // window [lo, lo + K') must contain k = 0 (see DESIGN.md "pruned transform")
    long long lo = std::min<long long>(klo, 0), hi = std::max<long long>(khi, 0);
    if (khi < klo) { lo = 0; hi = 0; }
    int lk = std::max(5, ilog2((unsigned long long)(hi - lo + 1)));
    if (lk > DIRECT_MAX_LOG2) {  // two-kernel path: negative part must be a multiple of K2
      lo = -((-lo + K2C - 1) / K2C) * K2C;
      lk = std::max(DIRECT_MAX_LOG2 + 1, ilog2((unsigned long long)(hi - lo + 1)));
    }
    if (lk > 20) lk = job.log2N;   // pruned lengths above 2^20 are not built: treat as dense
    const bool band_limited = lk < job.log2N;   // (before the promotion below: such a scale may still expand)
    // a pruned length of 2^18 or more within `dense_margin` octaves of the full one saves nothing
    // over the dense kernel pair (first kernels of 256 / 512 points cost what the 1024-point dense
    // one does once the band-product launch is counted): treat as dense (CWTB_DENSE_MARGIN)
    if (lk >= 18 && lk < job.log2N && job.log2N - lk <= c->dense_margin && job.log2N <= 20) lk = job.log2N;
    if (lk >= job.log2N) {  // dense
      lk = job.log2N;
      d.rsplit = (int)half;
      if (N == 1) d.rsplit = 1;
    } else {
      d.rsplit = (int)((1ll << lk) + lo);  // lo <= 0
    }
    d.log2K = lk;
    job.plan_log2K[j] = job.exact ? -1 : ((N < 32) ? 0 : lk);
    // ---- band-limited expansion instead of the pruned transforms (kernels.cuh: ExpandBody) ----
    d.ip_log2Nc = 0; d.ip_kc = 0; d.ip_w = 0; d.os_grp = 0; d.ip_coff = 0; d.ip_woff = 0;
    d.ip_beta = 0; d.ip_dc = 0;
    const double xeps = precision == CWTB_F64 ? c->expand_eps : c->expand_eps32;
    if (xeps > 0 && !job.exact && family != CWTB_TABLE && khi >= klo && job.log2N >= 9 && band_limited) {
      const long long kc = (klo + khi) / 2 - (((klo + khi) % 2 != 0 && (klo + khi) < 0) ? 1 : 0);   // floor
      const long long hw = std::max(khi - kc, kc - klo);
      // the tensor-core kernel (fp64, Np >= 4096, every row expanding by 8 or more) makes 20 taps
      // affordable: coarse grids down to 32/11 of the band half-width instead of 4x
#ifdef CWTB_HOST_EMU
      const bool mma = false;
      const int max_taps = precision == CWTB_F64 ? 20 : 10;   // the emulated scalar kernel has every tap count
#else
      const bool mma = precision == CWTB_F64 && c->expand_mma && job.log2N >= 12;
      const int max_taps = mma ? 20 : (precision == CWTB_F64 ? 16 : 10);
#endif
      const long long need = max_taps > 16 ? (32 * hw + 10) / 11 : 4 * hw;
      int lmin = std::max(6, ilog2((unsigned long long)std::max<long long>(need, 1)));
      lmin = std::max(lmin, job.log2N - 14);          // weight tables of at most 2^14 phases
      double best = 1e300;
      // smallest expansion factor: 4 for the tensor-core kernel, 8 for the scalar one.  With R = 4 config 2
      // expands 16 more rows (an exact dense row costs more than an expansion row plus its two-kernel
      // coarse transform of Np/4 points): 2.866 against 2.925 ms per step on H100 at 400 W, spread 0.012 ms.
      // The scalar kernel's trade-off at R = 4 has not been measured on H100.
      const int min_log2R = c->expand_min_log2R ? c->expand_min_log2R : (mma ? 2 : 3);
      // (coarse grids of at most 2^20 points: their transforms run as one 1024-point pass pair, CoarseABody)
      for (int l = lmin; l <= lmin + 2 && l <= 20 && job.log2N - l >= min_log2R; ++l) {
        double xi_b = 0;
        int w = expand_taps((double)hw / (double)(1ll << l), xeps, precision != CWTB_F64, max_taps, &xi_b);
        if (!w) continue;
        if (mma) w = (w + 3) / 4 * 4;   // the tensor-core kernel pads to DMMA steps of four taps anyway: 10 -> 12 and
                                        // 14 -> 16 cost nothing, lower the alias error and merge two launches
        if (xi_b > 0.25 && expand_gain(fam, s, klo, khi, kc, l, w, M_PI * w * (1.0 - xi_b)) > 64.0) continue;
        // cost model (us at Np = 2^20): the expansion kernel + the coarse transform.  Scalar kernel: its
        // fp64 work; tensor-core kernel: the W store until the DMMA steps of four taps exceed it
        const int ksteps = job.log2N - l == 2 ? (w + 4) / 4 : (w + 3) / 4;   // R = 4 needs one more tap column
        const double xcost = mma ? std::max(2.72, 0.83 * ksteps) : 0.06 * (2 * w + 8);
        const double cost = xcost + (mma ? 18.0 : 12.0) * (double)(1ll << l) / (double)N;
        if (cost < best) {
          best = cost;
          d.ip_log2Nc = l; d.ip_kc = (int)kc; d.ip_w = w;
          d.ip_beta = M_PI * w * (1.0 - xi_b);
          d.ip_dc = std::cyl_bessel_i(0.0, d.ip_beta) / w;
        }
      }
      if (d.ip_log2Nc) {
        d.ip_woff = expand_weights(c, c->wtab_host, job.log2N - d.ip_log2Nc, d.ip_w, d.ip_beta);
        job.plan_log2K[j] = -d.ip_log2Nc;
      }
    }
    if (os && (*os)[j].grp) {   // overlap-save (os_plan): replaces whatever was chosen above
      d.ip_log2Nc = 0; d.ip_kc = 0; d.ip_w = 0; d.ip_woff = 0; d.ip_beta = 0; d.ip_dc = 0;
      d.os_grp = (*os)[j].grp;
      job.plan_log2K[j] = CWTB_PLAN_OS;
    }
  }
  // one descriptor per (channel, scale) row; rows of channel ch are ch*S .. ch*S+S-1
  if (nbatch > 1) {
    int ngrp = 0;   // overlap-save groups are per channel (one signal per launch block)
    for (int j = 0; j < S; ++j) ngrp = std::max(ngrp, ds[j].os_grp);
    ds.resize((size_t)S * nbatch);
    for (int ch = 1; ch < nbatch; ++ch)
      for (int j = 0; j < S; ++j) {
        ScaleDesc d = ds[j];
        d.chan = ch;
        d.row = ch * S + j;
        if (d.os_grp) d.os_grp += ch * ngrp;
        ds[(size_t)ch * S + j] = d;
      }
  }
  const int R = S * nbatch;
  // sort by class (descending K': small scales first), stable
  std::vector<int> order(R);
  for (int j = 0; j < R; ++j) order[j] = j;
  // exact classes first (two-kernel, then single-kernel: descending K'), expansion classes last
  // (descending coarse length, then taps / weight table)
  auto sort_key = [&](const ScaleDesc &d) -> long long {
    if (d.os_grp) return (1ll << 41) - d.os_grp;   // overlap-save groups first, in group order
    if (!d.ip_log2Nc) return (1ll << 40) + d.log2K;
    return ((long long)(64 - d.ip_w) << 32) + ((long long)d.ip_log2Nc << 24) - (d.ip_woff & 0xffffff);
  };
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return sort_key(ds[a]) > sort_key(ds[b]); });
  job.descs.resize(R);
  size_t boff = 0, coff = 0;
  for (int i = 0; i < R; ++i) {
    job.descs[i] = ds[order[i]];
    ScaleDesc &d = job.descs[i];
    bool same = !job.classes.empty();
    if (same) {
      const ClassRun &b = job.classes.back();
      same = d.os_grp ? b.os == d.os_grp
           : d.ip_log2Nc ? (b.expand && b.log2Nc == d.ip_log2Nc && b.taps == d.ip_w && b.woff == d.ip_woff)
                         : (!b.expand && !b.os && b.log2K == d.log2K);
    }
    if (!same) {
      ClassRun cl{d.log2K, i, 0};
      if (d.ip_log2Nc) { cl.expand = 1; cl.log2Nc = d.ip_log2Nc; cl.taps = d.ip_w; cl.woff = d.ip_woff; }
      cl.os = d.os_grp;
      job.classes.push_back(cl);
    }
    job.classes.back().count++;
    if (d.os_grp) {
      if (job.classes.back().count == 1) {
        const OsRow &o = (*os)[d.row % S];
        job.os_groups.push_back(OsGroup{i, 0, o.t1, OsBody<4>::L - o.M + 1, o.hoff});
      }
      job.os_groups.back().count++;
    } else if (d.ip_log2Nc) {
      d.ip_coff = (long long)coff;
      coff += (size_t)1 << d.ip_log2Nc;
    } else if (d.log2K <= 10 || (d.log2K <= DIRECT_MAX_LOG2 && d.log2K < job.log2N)) {  // single-kernel scale
      d.boff = (long long)boff;
      boff += (size_t)1 << d.log2K;
    }
  }
  job.b_single = boff;
  job.coarse_elems = coff;
  job.valid = true;
  return 0;
}

// ======================================================================================
// execution
// ======================================================================================
template <typename T> struct Tw;
template <> struct Tw<double> { static const double2 *get(cwtb_ctx *c) { return c->tw64; } };
template <> struct Tw<float> { static const float2 *get(cwtb_ctx *c) { return c->tw32; } };

// batched FFT over matrix rows, any power-of-two n >= 2; in/out on device.
// real_in: input rows are T (zero-padded from n_in to n); else cx<T>.
template <typename T, int SIGN>
static int fft_rows(cwtb_ctx *c, const void *in, int real_in, long long in_pitch, long long n_in,
                    cx<T> *out, long long out_pitch, unsigned n, int nrows, long long nout = -1,
                    const double *grow = nullptr, double post = 1.0);

template <typename T, int SIGN, int K>
static int fft_rows_small(cwtb_ctx *c, const RowsArgs<T> &a) {
  constexpr int P = Lay<T, K>::P;
  return launch<RowsBody<T, K, SIGN>>(c, (a.nrows + P - 1) / P, 1, a);
}

template <typename T, int SIGN, int K1, int MODE>
static int launch_passA(cwtb_ctx *c, const PassAArgs<T> &a, int ny) {
  using B = PassABody<T, K1, MODE, SIGN>;
  const unsigned M = a.N / ((unsigned)K1 * a.K2);
  return launch<B>(c, M * (a.K2 / B::T2), ny, a);
}

template <typename T, int SIGN, int MODE>
static int dispatch_passA(cwtb_ctx *c, int log2K1, const PassAArgs<T> &a, int ny) {
  switch (log2K1) {
    case 1: return launch_passA<T, SIGN, 2, MODE>(c, a, ny);
    case 2: return launch_passA<T, SIGN, 4, MODE>(c, a, ny);
    case 3: return launch_passA<T, SIGN, 8, MODE>(c, a, ny);
    case 4: return launch_passA<T, SIGN, 16, MODE>(c, a, ny);
    case 5: return launch_passA<T, SIGN, 32, MODE>(c, a, ny);
    case 6: return launch_passA<T, SIGN, 64, MODE>(c, a, ny);
    case 7: return launch_passA<T, SIGN, 128, MODE>(c, a, ny);
    case 8: return launch_passA<T, SIGN, 256, MODE>(c, a, ny);
    case 9: return launch_passA<T, SIGN, 512, MODE>(c, a, ny);
    case 10: return launch_passA<T, SIGN, 1024, MODE>(c, a, ny);
  }
  return fail(c, CWTB_ERR_UNSUPPORTED, "transform longer than 2^20 per row is not supported yet");
}

// Z bytes per launch pair of two_kernel_rows: launches of >= 8 waves beat keeping the
// intermediate in L2 (50 MB on H100)
constexpr size_t ROWS_CHUNK_BYTES = (size_t)256 << 20;

// Rows of length n (1024 < n <= 2^20) through PassA<REAL|CPLX> + PassB, in chunks that fit the
// Z buffer.  Input row g becomes sub-transform g % ileave of output row out_row0 + g / ileave
// (ileave = 1: plain rows).  Output rows are renamed through descs[first + outer].row if given.
template <typename T, int SIGN>
static int two_kernel_rows(cwtb_ctx *c, const void *in, int real_in, long long in_pitch, long long n_in,
                           cx<T> *out, long long out_pitch, unsigned n, int nrows, long long nout,
                           const double *grow, double post, int ileave, const ScaleDesc *descs, int first,
                           int out_row0, int epi) {
  const int l2 = ilog2(n);
  NTab nt;
  int e = get_ntab(c, n, l2, &nt);
  if (e) return e;
  // rows per chunk: the intermediate of a chunk is at most ROWS_CHUNK_BYTES
  const int chunk = std::max(1, std::min(nrows, (int)std::max<size_t>(1, ROWS_CHUNK_BYTES / ((size_t)n * sizeof(cx<T>)))));
  Buf &Zt = c->Z;
  if ((e = ensure(c, Zt, (size_t)chunk * n * sizeof(cx<T>)))) return e;
  for (int r0 = 0; r0 < nrows; r0 += chunk) {
    const int nr = std::min(chunk, nrows - r0);
    PassAArgs<T> a{};
    a.in = in; a.Z = (cx<T> *)Zt.p; a.tw = Tw<T>::get(c); a.nt = nt;
    a.in_pitch = in_pitch; a.n_in = n_in; a.N = n; a.first = 0; a.K2 = K2C;
    a.row0 = (ileave > 1 ? 0 : out_row0) + r0;   // interleaved input rows are numbered from 0
    a.pf_dist = c->pf_rows_a;
    e = real_in ? dispatch_passA<T, SIGN, MODE_REAL>(c, l2 - 10, a, nr)
                : dispatch_passA<T, SIGN, MODE_CPLX>(c, l2 - 10, a, nr);
    if (e) return e;
    PassBArgs<T> b{};
    b.Z = (const cx<T> *)Zt.p; b.out = out; b.tw = Tw<T>::get(c); b.descs = descs;
    b.pitch = out_pitch; b.nout = nout; b.N = n; b.first = first;
    b.epi = grow ? EPI_GAUSS : epi; b.grow = grow; b.post = post;
    b.pf_dist = c->pf_rows_b; b.ny = nr; b.ileave = ileave;
    if (ileave > 1) { b.row0 = out_row0; b.by0 = r0; } else { b.row0 = out_row0 + r0; b.by0 = 0; }
    e = launch<PassBBody<T, SIGN>>(c, (n / K2C + Lay<T, K2C>::P - 1) / Lay<T, K2C>::P, nr, b);
    if (e) return e;
  }
  return 0;
}

template <typename T, int SIGN>
static int fft_rows(cwtb_ctx *c, const void *in, int real_in, long long in_pitch, long long n_in,
                    cx<T> *out, long long out_pitch, unsigned n, int nrows, long long nout,
                    const double *grow, double post) {
  const int l2 = ilog2(n);
  if (nout < 0) nout = n;
  if (n <= 1024) {
    RowsArgs<T> a;
    a.in = in; a.out = out; a.tw = Tw<T>::get(c); a.grow = grow;
    a.in_pitch = in_pitch; a.out_pitch = out_pitch; a.n_in = n_in; a.nout = nout;
    a.post = post; a.nrows = nrows; a.real_in = real_in; a.n = (int)n;
    switch (l2) {
      case 1: return fft_rows_small<T, SIGN, 2>(c, a);
      case 2: return fft_rows_small<T, SIGN, 4>(c, a);
      case 3: return fft_rows_small<T, SIGN, 8>(c, a);
      case 4: return fft_rows_small<T, SIGN, 16>(c, a);
      case 5: return fft_rows_small<T, SIGN, 32>(c, a);
      case 6: return fft_rows_small<T, SIGN, 64>(c, a);
      case 7: return fft_rows_small<T, SIGN, 128>(c, a);
      case 8: return fft_rows_small<T, SIGN, 256>(c, a);
      case 9: return fft_rows_small<T, SIGN, 512>(c, a);
      case 10: return fft_rows_small<T, SIGN, 1024>(c, a);
    }
    return fail(c, CWTB_ERR_ARG, "fft_rows: bad length");
  }
  if (n <= (1u << 20))
    return two_kernel_rows<T, SIGN>(c, in, real_in, in_pitch, n_in, out, out_pitch, n, nrows, nout, grow, post,
                                    1, nullptr, 0, 0, EPI_STORE);
  // ---- Np > 2^20: three levels.  A pre-pass (PassA with K1 = K0 = n / 2^20 and rows of 2^20)
  // turns each row into K0 twiddled sequences y_c[j]; output bin K0*q + c is bin q of the
  // 2^20-point transform of y_c, computed by the two-kernel path with interleaved stores.
  const int l0 = l2 - 20;
  const unsigned K0 = 1u << l0, Nsub = 1u << 20;
  NTab nt;
  int e = get_ntab(c, n, l2, &nt);
  if (e) return e;
  const int chunk = std::max(1, std::min(nrows, (int)std::max<size_t>(1, ((size_t)512 << 20) / ((size_t)n * sizeof(cx<T>)))));
  if ((e = ensure(c, c->Y, (size_t)chunk * n * sizeof(cx<T>)))) return e;
  for (int r0 = 0; r0 < nrows; r0 += chunk) {
    const int nr = std::min(chunk, nrows - r0);
    PassAArgs<T> a{};
    a.in = in; a.Z = (cx<T> *)c->Y.p; a.tw = Tw<T>::get(c); a.nt = nt;
    a.in_pitch = in_pitch; a.n_in = n_in; a.N = n; a.first = 0; a.row0 = r0; a.K2 = Nsub;
    e = real_in ? dispatch_passA<T, SIGN, MODE_REAL>(c, l0, a, nr)
                : dispatch_passA<T, SIGN, MODE_CPLX>(c, l0, a, nr);
    if (e) return e;
    if ((e = two_kernel_rows<T, SIGN>(c, c->Y.p, 0, Nsub, Nsub, out, out_pitch, Nsub, nr * (int)K0, nout, grow, post,
                                      (int)K0, nullptr, 0, r0, EPI_STORE)))
      return e;
  }
  return 0;
}


// ======================================================================================
// un-padded mode (pycwt/helpers.py:15-19, the reference's pyfftw branch): transforms at the
// signal's own length n through Bluestein's chirp-z algorithm on the power-of-two kernels.
// A compatibility path: ~2 transforms of length >= 2n per scale and no band pruning.
// ======================================================================================
static int get_blue(cwtb_ctx *c, unsigned n, const BluePlan **out) {
  auto it = c->blue.find(n);
  if (it == c->blue.end()) {
    // keep at most a few lengths resident
    if (c->blue.size() >= 4) {
      for (auto &kv : c->blue) { rt_free(kv.second.wm); rt_free(kv.second.bf[0]); rt_free(kv.second.bf[1]); }
      c->blue.clear();
    }
    BluePlan pl;
    pl.n = n;
    pl.L = 1u << ilog2(2ull * n - 1);
    RT(rt_malloc((void **)&pl.wm, sizeof(double2) * n));
    BlueChirpArgs ca{pl.wm, n};
    int e = launch<BlueChirpBody>(c, (n + NT - 1) / NT, 1, ca);
    if (e) return e;
    if ((e = ensure(c, c->blueX, (size_t)pl.L * sizeof(double2)))) return e;
    for (int si = 0; si < 2; ++si) {
      RT(rt_malloc((void **)&pl.bf[si], sizeof(double2) * pl.L));
      BlueFilterArgs fa{pl.wm, (double2 *)c->blueX.p, n, pl.L, si ? +1 : -1};
      if ((e = launch<BlueFilterBody>(c, (pl.L + NT - 1) / NT, 1, fa))) return e;
      if ((e = fft_rows<double, -1>(c, c->blueX.p, 0, pl.L, pl.L, pl.bf[si], pl.L, pl.L, 1, -1, nullptr, 1.0))) return e;
    }
    it = c->blue.emplace(n, pl).first;
  }
  *out = &it->second;
  return 0;
}

// rows of the convolution buffers a chunk may use (two buffers of L complex per row), and at most
// MAX_ROWS: every launch of a chunk has one row per chunk row
static int blue_chunk_rows(unsigned L, int nrows) {
  const size_t per_row = (size_t)L * sizeof(double2);
  return (int)std::max<size_t>(1, std::min<size_t>({(size_t)nrows, ((size_t)1 << 30) / per_row, (size_t)MAX_ROWS}));
}

// convolution core: blueA rows (pitch n) already hold a = x * w_s; result rows y in blueY
static int blue_convolve(cwtb_ctx *c, const BluePlan &pl, int nr, int sign) {
  int e;
  if ((e = fft_rows<double, -1>(c, c->blueA.p, 0, pl.n, pl.n, (double2 *)c->blueX.p, pl.L, pl.L, nr, -1, nullptr, 1.0)))
    return e;
  BlueMulArgs ma{(double2 *)c->blueX.p, pl.bf[sign > 0 ? 1 : 0], pl.L};
  if ((e = launch<BlueMulBody>(c, (pl.L + NT - 1) / NT, nr, ma))) return e;
  return fft_rows<double, +1>(c, c->blueX.p, 0, pl.L, pl.L, (double2 *)c->blueY.p, pl.L, pl.L, nr, -1, nullptr, 1.0);
}

// out[r][k] = scale * sum_j in[r][j] e^{sign 2 pi i jk/n}, k < nout, for rows of any length n >= 2
static int blue_rows(cwtb_ctx *c, const void *in, int real_in, long long in_pitch, double2 *out,
                     long long out_pitch, unsigned n, int nrows, int sign, double scale, long long nout) {
  const BluePlan *pl;
  int e = get_blue(c, n, &pl);
  if (e) return e;
  const int chunk = blue_chunk_rows(pl->L, nrows);
  if ((e = ensure(c, c->blueA, (size_t)chunk * n * sizeof(double2)))) return e;
  if ((e = ensure(c, c->blueX, (size_t)chunk * pl->L * sizeof(double2)))) return e;
  if ((e = ensure(c, c->blueY, (size_t)chunk * pl->L * sizeof(double2)))) return e;
  const size_t isz = real_in ? sizeof(double) : sizeof(double2);
  for (int r0 = 0; r0 < nrows; r0 += chunk) {
    const int nr = std::min(chunk, nrows - r0);
    BluePreArgs pa{(const char *)in + (size_t)r0 * in_pitch * isz, (double2 *)c->blueA.p, pl->wm,
                   in_pitch, (long long)n, n, real_in, sign};
    if ((e = launch<BluePreBody>(c, (n + NT - 1) / NT, nr, pa))) return e;
    if ((e = blue_convolve(c, *pl, nr, sign))) return e;
    BluePostArgs po{(const double2 *)c->blueY.p, out, pl->wm, nullptr, out_pitch, nout,
                    scale / (double)pl->L, pl->L, 0, r0, sign, EPI_STORE};
    if ((e = launch<BluePostBody>(c, (unsigned)((nout + NT - 1) / NT), nr, po))) return e;
  }
  return 0;
}

// every kernel of one un-padded transform (fp64): spectrum at length n0, then for chunks of scales
// product + inverse transform at length n0
static int run_job_exact(cwtb_ctx *c, const Job &job, const double *dsig, double2 *Wout, int epi) {
  const unsigned n = job.N;
  const int S = job.S;
  int e;
  if (job.nbatch != 1) return fail(c, CWTB_ERR_UNSUPPORTED, "batched transforms need the padded mode");
  if ((e = ensure(c, c->spec, (size_t)n * sizeof(double2)))) return e;
  if (!Wout) {
    if ((e = ensure(c, c->W, (size_t)S * job.n0 * sizeof(double2)))) return e;
    Wout = (double2 *)c->W.p;
  }
  if ((e = blue_rows(c, dsig, 1, n, (double2 *)c->spec.p, n, n, 1, -1, 1.0, n))) return e;
  const BluePlan *pl;
  if ((e = get_blue(c, n, &pl))) return e;
  Fam fam = job.fam;
  if (fam.family == CWTB_TABLE) fam.table = (const double2 *)c->table.p;
  const int chunk = blue_chunk_rows(pl->L, S);
  if ((e = ensure(c, c->blueA, (size_t)chunk * n * sizeof(double2)))) return e;
  if ((e = ensure(c, c->blueX, (size_t)chunk * pl->L * sizeof(double2)))) return e;
  if ((e = ensure(c, c->blueY, (size_t)chunk * pl->L * sizeof(double2)))) return e;
  const ScaleDesc *ddesc = (const ScaleDesc *)c->descs.p;
  for (int r0 = 0; r0 < S; r0 += chunk) {
    const int nr = std::min(chunk, S - r0);
    BlueProdArgs pa{ddesc, (const double2 *)c->spec.p, (double2 *)c->blueA.p, pl->wm, fam, (long long)n, n, r0};
    if ((e = launch<BlueProdBody>(c, (n + NT - 1) / NT, nr, pa))) return e;
    if ((e = blue_convolve(c, *pl, nr, +1))) return e;
    // descriptor amplitudes already carry the 1/n of the inverse transform
    BluePostArgs po{(const double2 *)c->blueY.p, Wout, pl->wm, ddesc, job.n0, job.n0,
                    1.0 / (double)pl->L, pl->L, r0, 0, +1, epi};
    if ((e = launch<BluePostBody>(c, (unsigned)((job.n0 + NT - 1) / NT), nr, po))) return e;
  }
  return 0;
}

template <typename T, int K>
static int launch_single(cwtb_ctx *c, const SingleArgs<T> &a, int count) {
  constexpr int P = Lay<T, K>::P;
  const unsigned M = a.N / K;
  return launch<SingleBody<T, K>>(c, (M + P - 1) / P, count, a);
}

// rows (scale x channel) per chunk of the two-kernel path: the Z intermediate of a chunk is
// rows * Np elements
static int chunk_rows(const cwtb_ctx *c, unsigned N, size_t elem_bytes) {
  if (c->group > 0) return c->group;
  size_t g = c->group_bytes / ((size_t)N * elem_bytes);
  return (int)std::max<size_t>(1, std::min<size_t>(g, 32768));
}

static bool class_single(const Job &job, const ClassRun &cl) {
  return !cl.expand && !cl.os && (cl.log2K <= 10 || (cl.log2K <= DIRECT_MAX_LOG2 && cl.log2K < job.log2N));
}
static bool class_two_kernel(const Job &job, const ClassRun &cl) {
  return !cl.expand && !cl.os && !class_single(job, cl);
}

// Which band-chunk region / Z buffer / stream a two-kernel class uses: its position among the
// two-kernel classes modulo the number of chains (dense classes included, they only use Z).
static int job_chain_region(const cwtb_ctx *c, const Job &job, const ClassRun &cl) {
  int idx = 0;
  for (const ClassRun &o : job.classes) {
    if (&o == &cl) break;
    if (class_two_kernel(job, o)) ++idx;
  }
  return idx % std::max(1, c->n_chains);
}

// elements of one band-chunk region: the largest chunk of band products of any two-kernel class
static size_t band_chunk_elems(const Job &job, int G) {
  size_t bchunk = 0;
  for (const ClassRun &cl : job.classes)
    if (class_two_kernel(job, cl) && cl.log2K < job.log2N)
      bchunk = std::max(bchunk, (size_t)std::min(G, cl.count) << cl.log2K);
  return bchunk;
}

#ifndef CWTB_HOST_EMU
// one CTA per resident slot (occupancy x SMs), each looping over the rows x gm tiles of the launch
template <class Body>
static int launch_persistent(cwtb_ctx *c, unsigned gm, unsigned rows, const typename Body::Args &a) {
  auto kern = k_persist<Body>;
  const void *fn = (const void *)kern;
  if (!c->configured.count(fn)) {
    RT(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Body::SMEM));
    c->configured.insert(fn);
  }
  int occ = 0;
  RT(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, Body::NTB, Body::SMEM));
  if (occ < 1) return fail(c, CWTB_ERR_CUDA, "persistent kernel does not fit on an SM");
  const unsigned long long total = (unsigned long long)gm * rows;
  if (total > 0xffffffffull) return fail(c, CWTB_ERR_ARG, "too many tiles in one launch");
  const unsigned grid = (unsigned)std::min<unsigned long long>(total, (unsigned long long)occ * c->num_sms);
  return launch_rec<Body>(c, grid, rows, [&]() -> int {
    kern<<<grid, Body::NTB, Body::SMEM, c->cur>>>(a, gm, (unsigned)total);
    RT(cudaGetLastError());
    return 0;
  });
}
#endif

// One ragged launch of Body (CoarseRowsBody / CoarseABody / CoarseBBody) over the given segments:
// a single launch unless there are more than CSEG_MAX of them
template <class Body, typename T>
static int launch_coarse(cwtb_ctx *c, CoarseArgs<T> a, const std::vector<CoarseSeg> &segs) {
  for (size_t s0 = 0; s0 < segs.size(); s0 += CSEG_MAX) {
    a.nseg = (int)std::min<size_t>(CSEG_MAX, segs.size() - s0);
    unsigned ctas = 0;
    for (int i = 0; i < a.nseg; ++i) {
      a.seg[i] = segs[s0 + i];
      a.seg[i].cta0 = (int)ctas;
      ctas += (unsigned)Body::ctas(a.seg[i].log2Nc, a.seg[i].count);
    }
    int e = launch<Body>(c, ctas, 1, a);
    if (e) return e;
  }
  return 0;
}

template <typename T, int TAPS>
static int launch_expand_t(cwtb_ctx *c, const ExpandArgs<T> &a, int rows, int min_log2Nc) {
  using B = ExpandBody<T, TAPS>;
  // tiles per row: (R / RB) * ceil(Nc / MT) with RB = min(R, NT), MT = (NT / RB) * L -- equal to
  // N / (NT * L) for every coarse length with Nc >= MT; rows with a shorter coarse grid use the
  // first tiles of the launch only
  const unsigned gx = std::max<unsigned>(1, a.N / (unsigned)(B::NT * B::L));
#ifndef CWTB_HOST_EMU
  // fp64: tap sums on the tensor cores (kernels.cuh: ExpandMmaBody) whenever every row expands by 8 or more
  if constexpr (std::is_same<T, double>::value) {
    static_assert(ExpandMmaBody<TAPS>::OUT_PER_CTA == 4096, "the planner assumes the tensor-core kernel from Np = 2^12");
    if (c->expand_mma && a.N >= (unsigned)ExpandMmaBody<TAPS>::OUT_PER_CTA) {
      // tiles per row: N / (32 L); a row whose coarse grid is shorter than one run (Nc < L, R > 32) needs
      // one tile per 32 phases instead
      const unsigned gm = a.N / (32u * std::min<unsigned>(ExpandMmaBody<TAPS>::L, 1u << min_log2Nc));
      if (a.epi == EPI_MULCONJ) return launch_persistent<ExpandMmaBody<TAPS, EPI_MULCONJ>>(c, gm, rows, a);
      return launch_persistent<ExpandMmaBody<TAPS>>(c, gm, rows, a);
    }
  }
  if constexpr (TAPS > 16) {
    return fail(c, CWTB_ERR_STATE, "expansion: tap counts above 16 exist on the tensor-core kernel only");
  } else
#endif
  {
    if (a.epi == EPI_MULCONJ) return launch<ExpandBody<T, TAPS, EPI_MULCONJ>>(c, gx, rows, a);
    return launch<B>(c, gx, rows, a);
  }
}
template <typename T>
static int launch_expand(cwtb_ctx *c, int taps, const ExpandArgs<T> &a, int rows, int min_log2Nc) {
  if constexpr (std::is_same<T, double>::value) {
    switch (taps) {
      case 10: return launch_expand_t<T, 10>(c, a, rows, min_log2Nc);
      case 12: return launch_expand_t<T, 12>(c, a, rows, min_log2Nc);
      case 14: return launch_expand_t<T, 14>(c, a, rows, min_log2Nc);
      case 16: return launch_expand_t<T, 16>(c, a, rows, min_log2Nc);
      case 20: return launch_expand_t<T, 20>(c, a, rows, min_log2Nc);
    }
  } else {
    switch (taps) {
      case 6: return launch_expand_t<T, 6>(c, a, rows, min_log2Nc);
      case 8: return launch_expand_t<T, 8>(c, a, rows, min_log2Nc);
      case 10: return launch_expand_t<T, 10>(c, a, rows, min_log2Nc);
    }
  }
  return fail(c, CWTB_ERR_STATE, "expansion: unsupported tap count");
}

// all kernels of one transform: forward FFT of the (device, type T) signal, then every scale
template <typename T>
static int run_job(cwtb_ctx *c, const Job &job, const T *dsig, cx<T> *Wout = nullptr, int epi = EPI_STORE) {
  using V = cx<T>;
  if (job.exact) {
    if constexpr (std::is_same<T, double>::value) return run_job_exact(c, job, dsig, Wout, epi);
    else return fail(c, CWTB_ERR_UNSUPPORTED, "un-padded transforms run in fp64");
  }
  const unsigned N = job.N;
  const int S = job.S * job.nbatch;   // rows: one per (channel, scale)
  int e;
  // whatever path leaves this function (also an error in the middle of the fork), the launcher
  // is back on the engine's stream afterwards
  struct CurGuard { cwtb_ctx *c; ~CurGuard() { c->cur = c->stream; c->prof_tag = ""; } } cur_guard{c};
  if ((e = ensure(c, c->spec, (size_t)job.nbatch * N * sizeof(V)))) return e;
  if (!Wout) {
    if ((e = ensure(c, c->W, (size_t)S * job.n0 * sizeof(V)))) return e;
    Wout = (V *)c->W.p;
  }
  V *spec = (V *)c->spec.p;
  V *W = Wout;
  const ScaleDesc *ddesc = (const ScaleDesc *)c->descs.p;
  Fam fam = job.fam;
  if (fam.family == CWTB_TABLE) fam.table = (const double2 *)c->table.p;

  // ---- forward transform of the zero-padded signal (wavelet.py:91) ----
  if (N < 32) {
    if (job.nbatch != 1) return fail(c, CWTB_ERR_UNSUPPORTED, "batched transform needs n0 > 16");
    TinyFwdArgs<T> fa{dsig, spec, job.n0, N};
    if ((e = launch<TinyFwdBody<T>>(c, 1, 1, fa))) return e;
    TinyArgs<T> ta{ddesc, spec, W, fam, job.n0, N, 0, epi};
    return launch<TinyBody<T>>(c, (unsigned)((job.n0 + NT - 1) / NT), S, ta);
  }
  c->prof_tag = "fwd:";
  e = fft_rows<T, -1>(c, dsig, 1, job.n0, job.n0, spec, N, N, job.nbatch);
  c->prof_tag = "";
  if (e) return e;

  NTab nt;
  if ((e = get_ntab(c, N, job.log2N, &nt))) return e;
  const int G = chunk_rows(c, N, sizeof(V));
  const size_t bchunk = band_chunk_elems(job, G);   // two regions: one per chain stream
  if ((e = ensure(c, c->B, (job.b_single + (size_t)std::max(1, c->n_chains) * bchunk) * sizeof(V)))) return e;
  V *Bbuf = (V *)c->B.p;

  // band products of every single-kernel scale in one launch (their descriptors are contiguous
  // in the class-sorted array; blocks beyond a scale's K' exit immediately)
  {
    int first = -1, maxlk = 0, nrows = 0;
    for (const ClassRun &cl : job.classes)
      if (class_single(job, cl)) {
        if (first < 0) first = cl.first;
        maxlk = std::max(maxlk, cl.log2K);
        nrows += cl.count;
      }
    if (first >= 0) {
      BandArgs<T> ba{ddesc, spec, Bbuf, fam, N, first};
      const unsigned Kmax = 1u << maxlk;
      const unsigned gx = (Kmax + NT * BandBody<T>::PER - 1) / (NT * BandBody<T>::PER);
      if ((e = fam.family == CWTB_MORSE ? launch<BandBodyMorse<T>>(c, gx, nrows, ba) : launch<BandBody<T>>(c, gx, nrows, ba)))
        return e;
    }
  }
  // The single-kernel classes (independent of the two-kernel chains: different W rows, read-only
  // band products) run on a second stream so that their CTAs fill the tails of the chains.  While
  // profiling, every launch stays on the engine's stream.
  const bool split = !c->profiling;
  if (split) {
    RT(rt_record(c->ev_fork, c->stream));
    RT(rt_wait(c->aux_stream, c->ev_fork));
    for (int k = 1; k < c->n_chains; ++k) RT(rt_wait(c->chain_streams[k - 1], c->ev_fork));
  }
  // ---- expansion classes (kernels.cuh: ExpandBody): the coarse transforms of every expansion row
  // form their coarse spectra while they fill their tiles, in one launch for the coarse lengths up
  // to 1024 and one launch pair for the longer ones; then one expansion launch per tap count.
  if (job.coarse_elems) {
    const bool prio = split && c->prio_mode > 0;
    // the coarse launches go to high-priority streams: queued behind the big launches of the other
    // streams they would only advance in those launches' tails.  Short and long coarse lengths run
    // side by side; an expansion launch waits only for the lengths it reads.
    if (prio) {
      RT(rt_wait(c->prio_stream, c->ev_fork));
      RT(rt_wait(c->prio_short, c->ev_fork));
    }
    if (split) c->cur = prio ? c->prio_stream : c->aux_stream;
    if ((e = ensure(c, c->Cout, job.coarse_elems * sizeof(V)))) return e;
    // segments: consecutive expansion rows of one coarse length (their coarse rows are contiguous)
    std::vector<CoarseSeg> short_segs, long_segs;
    size_t zx_elems = 0;
    for (size_t ci = 0; ci < job.classes.size(); ++ci) {
      const ClassRun &cl = job.classes[ci];
      if (!cl.expand) continue;
      if (cl.log2Nc < 6 || cl.log2Nc > 20)   // the lengths CoarseRowsBody / CoarseABody have tiles for
        return fail(c, CWTB_ERR_STATE, "expansion: coarse length outside 2^6 .. 2^20");
      std::vector<CoarseSeg> &v = cl.log2Nc <= 10 ? short_segs : long_segs;
      if (ci > 0 && job.classes[ci - 1].expand && job.classes[ci - 1].log2Nc == cl.log2Nc) v.back().count += cl.count;
      else v.push_back(CoarseSeg{cl.first, cl.count, cl.log2Nc, 0});
      if (cl.log2Nc > 10)   // Z rows sit at the rows' offsets in C
        zx_elems = std::max(zx_elems, (size_t)job.descs[cl.first].ip_coff + ((size_t)cl.count << cl.log2Nc));
    }
    CoarseArgs<T> ca{};
    ca.descs = ddesc; ca.spec = spec; ca.C = (V *)c->Cout.p; ca.tw = Tw<T>::get(c); ca.fam = fam; ca.Nx = N;
    ca.pf_dist = c->pf_rows_b;
    c->prof_tag = "coarse:";
    if (!long_segs.empty()) {
      if ((e = ensure(c, c->Zx, zx_elems * sizeof(V)))) return e;
      ca.Z = (V *)c->Zx.p;
      for (const CoarseSeg &g : long_segs)
        if ((e = get_ntab(c, 1u << g.log2Nc, g.log2Nc, &ca.nt[g.log2Nc - 10]))) return e;
      if ((e = launch_coarse<CoarseABody<T>>(c, ca, long_segs))) return e;
      if ((e = launch_coarse<CoarseBBody<T>>(c, ca, long_segs))) return e;
    }
    if (!short_segs.empty()) {
      if (prio) c->cur = c->prio_short;
      if ((e = launch_coarse<CoarseRowsBody<T>>(c, ca, short_segs))) return e;
    }
    c->prof_tag = "";
    if (prio) {
      RT(rt_record(c->ev_coarse_short, c->prio_short));
      RT(rt_record(c->ev_coarse, c->prio_stream));
      c->cur = c->prio_mode == 1 ? c->aux_stream : c->prio_stream;   // 1: expansion kernels at ordinary priority
      RT(rt_wait(c->cur, c->ev_coarse_short));
    }
    // one expansion launch per tap count (classes are sorted by taps first): those that read only
    // coarse lengths up to 1024 first, the others behind the long coarse transforms
    for (int pass = 0; pass < 2 && !e; ++pass) {
      if (pass == 1 && prio && c->prio_mode == 1) RT(rt_wait(c->cur, c->ev_coarse));
      for (size_t ci = 0; ci < job.classes.size() && !e; ++ci) {
        const ClassRun &cl = job.classes[ci];
        if (!cl.expand || (ci > 0 && job.classes[ci - 1].expand && job.classes[ci - 1].taps == cl.taps)) continue;
        int rows = 0, minl = 30, maxl = 0;
        for (size_t cj = ci; cj < job.classes.size() && job.classes[cj].expand && job.classes[cj].taps == cl.taps; ++cj) {
          rows += job.classes[cj].count;
          minl = std::min(minl, job.classes[cj].log2Nc);
          maxl = std::max(maxl, job.classes[cj].log2Nc);
        }
        if ((maxl > 10) != (pass == 1)) continue;
        ExpandArgs<T> ea{ddesc, (const V *)c->Cout.p, (const double *)c->wtab.p, W, nt, job.n0, N, cl.first, epi,
                         job.log2N};
        e = launch_expand<T>(c, cl.taps, ea, rows, minl);
      }
    }
    if (prio && !e) {   // later work of the second stream and the join follow the coarse chain
      if (c->prio_mode == 2) RT(rt_record(c->ev_coarse, c->prio_stream));
      RT(rt_wait(c->aux_stream, c->ev_coarse));
    }
    c->cur = c->stream;
    if (e) return e;
  }
  // ---- overlap-save groups (kernels.cuh: OsBody): one launch on the stream of the first chain ----
  if (!job.os_groups.empty()) {
    if constexpr (std::is_same<T, double>::value) {
      unsigned gx = 0;
      for (const OsGroup &g : job.os_groups)
        gx = std::max<unsigned>(gx, (unsigned)((job.n0 + (long long)g.hop * OsBody<4>::P - 1) /
                                               ((long long)g.hop * OsBody<4>::P)));
      OsArgs oa{ddesc, (const OsGroup *)c->osgrp.p, dsig, (const double2 *)c->osH.p, W, Tw<T>::get(c),
                job.n0, N, epi};
      if ((e = launch<OsBody<4>>(c, gx, (unsigned)job.os_groups.size(), oa))) return e;
    } else {
      return fail(c, CWTB_ERR_STATE, "overlap-save rows run in fp64 only");
    }
  }
  for (int pass = 0; pass < 2; ++pass)
  for (const ClassRun &cl : job.classes) {
    if (cl.expand || cl.os) continue;
    const unsigned K = 1u << cl.log2K;
    const bool single = class_single(job, cl);
    if (single != (pass == 0)) continue;   // pass 0: single-kernel classes, pass 1: two-kernel chains
    if (single) {
      if (split) c->cur = c->aux_stream;
      // ---- single kernel: pruned K'-point transforms from the band products ----
      SingleArgs<T> sa{ddesc, Bbuf, W, Tw<T>::get(c), nt, job.n0, N, cl.first, epi};
      switch (cl.log2K) {
        case 5: e = launch_single<T, 32>(c, sa, cl.count); break;
        case 6: e = launch_single<T, 64>(c, sa, cl.count); break;
        case 7: e = launch_single<T, 128>(c, sa, cl.count); break;
        case 8: e = launch_single<T, 256>(c, sa, cl.count); break;
        case 9: e = launch_single<T, 512>(c, sa, cl.count); break;
        case 10: e = launch_single<T, 1024>(c, sa, cl.count); break;
        case 11: e = launch<DirectBody<T, 2>>(c, (N / K2C + Lay<T, K2C>::P - 1) / Lay<T, K2C>::P, cl.count, sa); break;
        case 12: e = launch<DirectBody<T, 4>>(c, (N / K2C + Lay<T, K2C>::P - 1) / Lay<T, K2C>::P, cl.count, sa); break;
        case 13: e = launch<DirectBody<T, 8>>(c, (N / K2C + Lay<T, K2C>::P - 1) / Lay<T, K2C>::P, cl.count, sa); break;
        default: e = fail(c, CWTB_ERR_STATE, "bad single-kernel class");
      }
      c->cur = c->stream;
      if (e) return e;
      continue;
    }
    // ---- two kernels through Z ----
    const bool dense = (cl.log2K == job.log2N);
    if (dense && job.log2N > 20) {
      // ---- Np > 2^20: pre-pass (K0-point transforms over rows of 2^20, response generated
      // in-kernel) into Y, then the K0 interleaved 2^20-point transforms of every scale ----
      const int l0 = job.log2N - 20;
      const unsigned Nsub = 1u << 20;
      const int gy = std::max<int>(1, (int)std::min<size_t>((size_t)cl.count, ((size_t)512 << 20) / ((size_t)N * sizeof(V))));
      if ((e = ensure(c, c->Y, (size_t)gy * N * sizeof(V)))) return e;
      for (int g0 = 0; g0 < cl.count; g0 += gy) {
        const int ng = std::min(gy, cl.count - g0);
        PassAArgs<T> a{};
        a.descs = ddesc; a.spec = spec; a.Bbuf = Bbuf; a.Z = (V *)c->Y.p; a.tw = Tw<T>::get(c);
        a.fam = fam; a.nt = nt; a.N = N; a.first = cl.first + g0; a.row0 = 0;
        a.pf_dist = 0; a.K2 = Nsub;
        if ((e = dispatch_passA<T, +1, MODE_DENSE>(c, l0, a, ng))) return e;
        if ((e = two_kernel_rows<T, +1>(c, c->Y.p, 0, Nsub, Nsub, W, job.n0, Nsub, ng << l0, job.n0, nullptr, 1.0,
                                         1 << l0, ddesc, cl.first + g0, 0, epi)))
          return e;
      }
      continue;
    }
    // successive two-kernel classes rotate over the chains, each with its own stream, Z buffer
    // and band-chunk region (descriptor offsets already point into the right region)
    const int chain = split ? job_chain_region(c, job, cl) : 0;
    Buf &Zb = chain > 0 ? c->Zc[chain - 1] : c->Z;
    if ((e = ensure(c, Zb, (size_t)G * N * sizeof(V)))) return e;
    c->cur = chain > 0 ? c->chain_streams[chain - 1] : c->stream;
    for (int g0 = 0; g0 < cl.count; g0 += G) {
      const int ng = std::min(G, cl.count - g0);
      PassAArgs<T> a{};
      a.descs = ddesc; a.spec = spec; a.Bbuf = Bbuf; a.Z = (V *)Zb.p; a.tw = Tw<T>::get(c);
      a.fam = fam; a.nt = nt; a.N = N; a.first = cl.first + g0; a.row0 = 0;
      // band scales: second pass of 512 points (full 128-byte output runs, conflict-free tile);
      // dense scales keep 1024 so that K1 = N/K2 <= 1024
      // (fp32: the 512-point tile has an odd row pitch, its rows would not be 16-byte aligned)
      constexpr bool k512_ok = (Lay<T, 512, true>::PITCH * sizeof(V)) % 16 == 0;
      // 512 pays up to K' = 2^16 (measured per class: first kernel + second kernel per row)
      const int l2k = (dense || cl.log2K > 16 || !k512_ok) ? 10 : 9;
      a.pf_dist = c->pf_dist_a; a.K2 = 1u << l2k;
      PassBArgs<T> b{};
      b.Z = (const V *)Zb.p; b.out = W; b.tw = Tw<T>::get(c); b.descs = ddesc;
      b.pitch = job.n0; b.nout = job.n0; b.N = N; b.first = cl.first + g0; b.row0 = 0;
      b.epi = epi; b.grow = nullptr; b.post = 1.0;
      b.pf_dist = c->pf_dist; b.ny = ng;
      if (!dense) {
        BandArgs<T> ba{ddesc, spec, Bbuf, fam, N, cl.first + g0};
        const unsigned gx = (K + NT * BandBody<T>::PER - 1) / (NT * BandBody<T>::PER);
        if ((e = fam.family == CWTB_MORSE ? launch<BandBodyMorse<T>>(c, gx, ng, ba) : launch<BandBody<T>>(c, gx, ng, ba)))
          return e;
      }
      e = dense ? dispatch_passA<T, +1, MODE_DENSE>(c, cl.log2K - l2k, a, ng)
                : dispatch_passA<T, +1, MODE_BAND>(c, cl.log2K - l2k, a, ng);
      if (e) return e;
      if constexpr (k512_ok) {
        if (l2k == 9)
          e = launch<PassBBody<T, +1, 512>>(c, (N / 512 + Lay<T, 512>::P - 1) / Lay<T, 512>::P, ng, b);
      }
      if (l2k != 9)
        e = launch<PassBBody<T, +1>>(c, (N / K2C + Lay<T, K2C>::P - 1) / Lay<T, K2C>::P, ng, b);
      if (e) return e;
    }
    c->cur = c->stream;
  }
  if (split) {   // join: later work on the main stream sees every row of W
    RT(rt_record(c->ev_join, c->aux_stream));
    RT(rt_wait(c->stream, c->ev_join));
    for (int k = 1; k < c->n_chains; ++k) {
      RT(rt_record(c->ev_joinc[k - 1], c->chain_streams[k - 1]));
      RT(rt_wait(c->stream, c->ev_joinc[k - 1]));
    }
  }
  return 0;
}

// band-buffer offsets of the two-kernel scales depend on the chunk position; set them here
static void assign_chunk_offsets(cwtb_ctx *c, Job &job) {
  const int G = chunk_rows(c, job.N, job.precision == CWTB_F64 ? sizeof(double2) : sizeof(float2));
  const size_t bchunk = band_chunk_elems(job, G);
  for (const ClassRun &cl : job.classes) {
    if (!class_two_kernel(job, cl) || cl.log2K == job.log2N) continue;
    const size_t region = (size_t)job_chain_region(c, job, cl) * bchunk;
    for (int i = 0; i < cl.count; ++i)
      job.descs[cl.first + i].boff =
          (long long)(job.b_single + region + (size_t)(i % G) * ((size_t)1 << cl.log2K));
  }
}

static int upload_descs(cwtb_ctx *c, Job &job) {
  assign_chunk_offsets(c, job);
  if (c->wtab_host.size() > c->wtab_uploaded) {   // new expansion weight tables (appended)
    const size_t bytes = c->wtab_host.size() * sizeof(double);
    if (c->wtab.bytes < bytes) {
      RT(rt_sync(c->stream));
      int e2 = ensure(c, c->wtab, std::max(bytes, (size_t)2 * c->wtab.bytes));
      if (e2) return e2;
      c->wtab_uploaded = 0;   // a new allocation: everything again
    }
    RT(rt_h2d((char *)c->wtab.p + c->wtab_uploaded * sizeof(double), c->wtab_host.data() + c->wtab_uploaded,
              (c->wtab_host.size() - c->wtab_uploaded) * sizeof(double), c->stream));
    c->wtab_uploaded = c->wtab_host.size();
  }
  int e = ensure(c, c->descs, job.descs.size() * sizeof(ScaleDesc));
  if (e) return e;
  RT(rt_h2d(c->descs.p, job.descs.data(), job.descs.size() * sizeof(ScaleDesc), c->stream));
  RT(rt_sync(c->stream));  // job.descs is pageable host memory
  return 0;
}

// Device time of a kernel sequence on the engine's stream: time_begin in front of it, time_stop
// behind it, time_read once the stream has been synchronised past the stop.  time_end stops, waits
// and reads; a caller whose copies overlap the sequence's tail reads only after they are synchronised.
static int time_begin(cwtb_ctx *c) {
  RT(rt_record(c->e0, c->stream));
  return 0;
}
static int time_stop(cwtb_ctx *c) {
  RT(rt_record(c->e1, c->stream));
  return 0;
}
static int time_read(cwtb_ctx *c, double *ms) {
  float f = 0;
  RT(rt_elapsed_ms(&f, c->e0, c->e1));
  *ms = f;
  return 0;
}
static int time_end(cwtb_ctx *c, double *ms) {
  int e = time_stop(c);
  if (e) return e;
  RT(rt_event_sync(c->e1));
  return time_read(c, ms);
}

// The record of the resident transform, filled from the plan by a transform entry point once W is
// complete.  A read that the entry point makes afterwards and that fails empties it again (w_kept):
// a call that fails leaves no transform resident.
static void w_fill(cwtb_ctx *c) {
  c->wt.S = c->job.S * c->job.nbatch;
  c->wt.n0 = c->job.n0;
  c->wt.prec = c->job.precision;
}
static int w_kept(cwtb_ctx *c, int e) {
  if (e) c->wt.S = 0;
  return e;
}

// iters runs of the plan on the device signal dsig; W is complete, and resident, afterwards
static int timed_run(cwtb_ctx *c, const void *dsig, int iters, double *ms_out) {
  const Job &job = c->job;
  c->launches = 0;
  int e = time_begin(c);
  if (e) return e;
  for (int it = 0; it < iters; ++it) {
    e = job.precision == CWTB_F64 ? run_job<double>(c, job, (const double *)dsig)
                                  : run_job<float>(c, job, (const float *)dsig);
    if (e) return e;
  }
  double ms = 0;
  if ((e = time_end(c, &ms))) return e;
  if (ms_out) *ms_out = ms / iters;
  c->launches /= std::max(1, iters);
  w_fill(c);
  return 0;
}

// ---- conversions ---------------------------------------------------------------------
template <typename TI, typename TO> struct CvtArgs { const TI *in; TO *out; long long n; };
template <typename TI, typename TO> struct CvtBody {
  using Args = CvtArgs<TI, TO>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    long long i = (long long)bx * NT + tid;
    if (i < a.n) a.out[i] = (TO)a.in[i];
  }
};

// ======================================================================================
// C ABI
// ======================================================================================
extern "C" {

const char *cwtb_version(void) {
#ifdef CWTB_HOST_EMU
  return "cwt_b200 0.1 (host emulation build - tests only)";
#else
  return "cwt_b200 0.1 (sm_90a)";
#endif
}

int cwtb_device_count(void) {
  int n = 0;
  if (rt_device_count(&n) != 0) return 0;
  return n;
}

int cwtb_create(int device, cwtb_ctx **out) {
  if (!out) return CWTB_ERR_ARG;
  *out = nullptr;
  cwtb_ctx *c = new cwtb_ctx();
  c->device = device;
  if (rt_set_device(device) != 0) { delete c; return CWTB_ERR_CUDA; }
  if (rt_stream_create(&c->stream) != 0) { delete c; return CWTB_ERR_CUDA; }
  rt_event_create(&c->e0);
  rt_event_create(&c->e1);
  for (auto &st : c->copy_streams) rt_stream_create(&st);
  rt_stream_create(&c->aux_stream);
  rt_stream_create_highest({&c->prio_stream, &c->prio_short});
  rt_event_create_sync(&c->ev_angle);
  rt_event_create_sync(&c->ev_coarse);
  rt_event_create_sync(&c->ev_coarse_short);
  for (auto &ev : c->ev_h2d) rt_event_create_sync(&ev);
  for (auto &ev : c->ev_used) rt_event_create_sync(&ev);
  if (const char *g = getenv("CWTB_BATCH_PIPELINE")) c->batch_pipeline = atoi(g) != 0;
  if (const char *g = getenv("CWTB_PRIO")) c->prio_mode = std::min(2, std::max(0, atoi(g)));
  for (auto &st : c->chain_streams) rt_stream_create(&st);
  for (auto &ev : c->ev_joinc) rt_event_create_sync(&ev);
  rt_event_create_sync(&c->ev_fork);
  rt_event_create_sync(&c->ev_join);
  c->cur = c->stream;
  if (const char *g = getenv("CWTB_GROUP")) c->group = std::max(0, atoi(g));
  if (const char *g = getenv("CWTB_GROUP_MB")) c->group_bytes = (size_t)std::max(1, atoi(g)) << 20;
  if (const char *g = getenv("CWTB_BAND_EPS")) c->band_eps = atof(g);
  if (const char *g = getenv("CWTB_BAND_EPS32")) c->band_eps32 = atof(g);
  if (const char *g = getenv("CWTB_EXPAND_EPS")) c->expand_eps = std::max(0.0, atof(g));
  if (const char *g = getenv("CWTB_EXPAND_EPS32")) c->expand_eps32 = std::max(0.0, atof(g));
  if (const char *g = getenv("CWTB_EXPAND_MIN_R")) c->expand_min_log2R = std::min(14, std::max(2, atoi(g)));
  if (const char *g = getenv("CWTB_EXPAND_MMA")) c->expand_mma = atoi(g) != 0;
  if (const char *g = getenv("CWTB_OS")) c->os_on = atoi(g) != 0;
  if (const char *g = getenv("CWTB_WTAB_MB")) c->wtab_max_bytes = (size_t)std::max(0, atoi(g)) << 20;
  if (const char *g = getenv("CWTB_PLAN_REUSE")) c->plan_reuse = atoi(g) != 0;
  if (const char *g = getenv("CWTB_DENSE_MARGIN")) c->dense_margin = std::max(0, atoi(g));
  if (const char *g = getenv("CWTB_PF_DIST")) c->pf_dist = std::max(0, atoi(g));
  if (const char *g = getenv("CWTB_CHAINS")) c->n_chains = std::min(4, std::max(1, atoi(g)));
  if (const char *g = getenv("CWTB_FFT_PAD")) c->pad_pow2 = atoi(g) != 0;
  if (const char *g = getenv("CWTB_PF_ROWS_A")) c->pf_rows_a = std::max(0, atoi(g));
  if (const char *g = getenv("CWTB_PF_ROWS_B")) c->pf_rows_b = std::max(0, atoi(g));
  if (const char *g = getenv("CWTB_PF_DIST_A")) c->pf_dist_a = std::max(0, atoi(g));
  if (const char *g = getenv("CWTB_BATCH_MB")) c->batch_bytes = (size_t)std::max(1, atoi(g)) << 20;
  rt_sm_count(&c->num_sms, device);
  int e = init_tables(c);
  if (e == 0) e = rt_sync(c->stream) ? CWTB_ERR_CUDA : 0;
  if (e) { delete c; return e; }
  *out = c;
  return CWTB_OK;
}

void cwtb_destroy(cwtb_ctx *c) {
  if (!c) return;
  rt_set_device(c->device);
  rt_sync(c->stream);
  cwtb_comm_destroy(c);
  for (Buf *b : {&c->osH, &c->osgrp, &c->stage_dev[0], &c->stage_dev[1], &c->batch_power, &c->filt, &c->comm_send, &c->comm_recv, &c->Zx, &c->Cout, &c->wtab, &c->sig, &c->sig2, &c->sig3, &c->spec, &c->Z, &c->Zc[0], &c->Zc[1], &c->Zc[2], &c->Y, &c->B, &c->W, &c->W2, &c->W3, &c->descs, &c->table, &c->scratch,
                 &c->C, &c->A12, &c->F, &c->aux, &c->rowd, &c->win, &c->mask, &c->hist, &c->noise, &c->wide, &c->blueA, &c->blueX, &c->blueY, &c->pspec, &c->prot, &c->coh.buf, &c->cross.buf, &c->coh3.buf, &c->coh.counts, &c->coh3.counts, &c->coh.labels, &c->coh3.labels, &c->pw.buf, &c->pw.counts, &c->pw.labels, &c->cross.counts, &c->cross.labels, &c->arc, &c->cl_bits, &c->cl_rows, &c->cl_hdr, &c->cl_runs, &c->cl_qmax})
    if (b->p) rt_free(b->p);
  for (auto &kv : c->ntabs) { rt_free(kv.second.hi); rt_free(kv.second.lo); }
  for (auto &kv : c->blue) { rt_free(kv.second.wm); rt_free(kv.second.bf[0]); rt_free(kv.second.bf[1]); }
  if (c->tw64) rt_free(c->tw64);
  if (c->tw32) rt_free(c->tw32);
  for (void *p : c->pinned) rt_host_free(p);
  for (void *p : c->devallocs) rt_free(p);
  rt_event_destroy(c->e0);
  rt_event_destroy(c->e1);
  rt_stream_destroy(c->stream);
  for (auto &st : c->copy_streams) rt_stream_destroy(st);
  rt_stream_destroy(c->aux_stream);
  rt_stream_destroy(c->prio_stream);
  rt_stream_destroy(c->prio_short);
  rt_event_destroy(c->ev_angle);
  rt_event_destroy(c->ev_coarse);
  rt_event_destroy(c->ev_coarse_short);
  for (auto &ev : c->ev_h2d) rt_event_destroy(ev);
  for (auto &ev : c->ev_used) rt_event_destroy(ev);
  for (void *p : c->stage_host) if (p) rt_host_free(p);
  for (auto &st : c->chain_streams) rt_stream_destroy(st);
  for (auto &ev : c->ev_joinc) rt_event_destroy(ev);
  rt_event_destroy(c->ev_fork);
  rt_event_destroy(c->ev_join);
  delete c;
}

const char *cwtb_last_error(cwtb_ctx *c) { return c ? c->err.c_str() : "null context"; }

int cwtb_set_band_eps(cwtb_ctx *c, double eps) {
  if (!c || !(eps >= 0) || eps >= 1e-6) return fail(c, CWTB_ERR_ARG, "band eps must be in [0, 1e-6)");
  c->band_eps = eps;
  return 0;
}

int cwtb_set_expand_eps(cwtb_ctx *c, double eps64, double eps32) {
  if (!c || !(eps64 >= 0) || !(eps32 >= 0) || eps64 > 1e-6 || eps32 > 1e-3)
    return fail(c, CWTB_ERR_ARG, "expansion tolerance must be in [0, 1e-6] (fp64) / [0, 1e-3] (fp32)");
  c->expand_eps = eps64;
  c->expand_eps32 = eps32;
  return 0;
}

int cwtb_host_alloc(cwtb_ctx *c, size_t bytes, void **out) {
  if (!c || !out) return CWTB_ERR_ARG;
  if (rt_host_alloc(out, bytes) != 0) return fail(c, CWTB_ERR_NOMEM, "pinned allocation failed");
  c->pinned.insert(*out);
  return 0;
}
int cwtb_host_free(cwtb_ctx *c, void *p) {
  if (!c || !c->pinned.count(p)) return CWTB_ERR_ARG;
  c->pinned.erase(p);
  rt_host_free(p);
  return 0;
}
int cwtb_dev_alloc(cwtb_ctx *c, size_t bytes, void **out) {
  if (!c || !out) return CWTB_ERR_ARG;
  if (rt_malloc(out, bytes) != 0) return fail(c, CWTB_ERR_NOMEM, "device allocation failed");
  c->devallocs.insert(*out);
  return 0;
}
int cwtb_dev_free(cwtb_ctx *c, void *p) {
  if (!c || !c->devallocs.count(p)) return CWTB_ERR_ARG;
  c->devallocs.erase(p);
  rt_free(p);
  return 0;
}
int cwtb_memcpy_h2d(cwtb_ctx *c, void *dst, const void *src, size_t bytes) {
  RT(rt_h2d(dst, src, bytes, c->stream));
  RT(rt_sync(c->stream));
  return 0;
}
int cwtb_memcpy_d2h(cwtb_ctx *c, void *dst, const void *src, size_t bytes) {
  RT(rt_d2h(dst, src, bytes, c->stream));
  RT(rt_sync(c->stream));
  return 0;
}
int cwtb_sync(cwtb_ctx *c) {
  RT(rt_sync(c->stream));
  return 0;
}

// ---- overlap-save planning (kernels.cuh: OsBody) ----------------------------------------------
// Cost model, us per row of 2^20 outputs on H100 (see DESIGN.md §4): the overlap-save kernel at
// hop = L scaled by L / hop, against the two-kernel pair the row would otherwise take.  Measured at
// config 2 (H100 80GB HBM3, 700 W) with the register-resident tile core: OsBody<4> 0.245 ms for rows
// j = 20..47 (83..263 taps, L / hop 1.09..1.35), 8.75 us per row; the dense pair 11.7 + 11.8 us per
// row.  Rows that expand by R = 4 are not candidates: their expansion kernel (7.3-7.8 us per row with
// 16-20 taps, plus a share of the coarse transform) costs less than the overlap-save kernel even at
// hop = L.
static const double kOsUs = 7.0;
static const double kTwoKernelUs = 23.5;   // dense first + second kernel (PassABody<1024> + PassBBody<1024>)

struct DevTmp {   // device scratch of the planner, freed on every path out
  void *p = nullptr;
  ~DevTmp() { if (p) rt_free(p); }
};

// Rows that would run the two-kernel exact path, fp64 and padded, whose band [k_lo, k_hi] stays
// clear of Nyquist: their impulse response h_j = IDFT(norm conj psi^) decays like the wavelet in
// time.  h_j is computed by the exact path on a unit impulse (x^ = 1, into W, which the call
// overwrites anyway), truncated to the shortest window [t1 - M + 1, t1] around t = 0 that keeps all
// of its l1 mass but band_eps, not counting taps at the rounding noise of that computation (at most
// max(2 * the largest tap beyond L of t = 0, 8 ulp of max|h_j|)), and taken as
// H_j = DFT_L(h_j mod L) / L.  A row whose h_j has a tap above 128 ulp of max|h_j| beyond L of t = 0
// (a band cut at Nyquist, Paul's one-sided spectrum) or needs M > L/2 keeps its path, as does a row
// the cost model prices higher.  Accepted rows are grouped by M, up to four to a group.
// Plan-time cost: one exact transform of the candidate rows and a few host round trips, once per
// geometry (CWTB_PLAN_REUSE keeps it out of repeated calls).
static int os_plan(cwtb_ctx *c, const Job &job, double dt, int family, double param, std::vector<OsRow> &os) {
  constexpr int L = OsBody<4>::L, GR = 4;
  // a window of M taps (M <= L/2: hop >= L/2 + 1) against the two-kernel pair the row leaves
  auto os_cheaper = [](int M) { return M <= L / 2 && kOsUs * L / (double)(L - M + 1) < kTwoKernelUs; };
  os.assign(job.S, OsRow());
  const unsigned N = job.N;
  if (!c->os_on || job.precision != CWTB_F64 || job.exact || family == CWTB_TABLE ||
      !(c->band_eps > 0) || !(c->expand_eps > 0) || N < 2u * L)
    return 0;
  const long long half = (long long)N / 2;
  std::vector<int> cand;      // input scales
  std::vector<double> cs;
  for (const ScaleDesc &d : job.descs) {
    if (d.chan != 0 || d.k_hi < d.k_lo || d.k_lo <= -half || d.k_hi >= ((long long)N - 1) / 2) continue;
    if (d.ip_log2Nc || (d.log2K <= 10 || (d.log2K <= DIRECT_MAX_LOG2 && d.log2K < job.log2N))) continue;
    cand.push_back(d.row);
    cs.push_back(d.s);
  }
  if (cand.empty()) return 0;
  const int nc = (int)cand.size();
  // impulse responses: the exact path (expansion off) on x = delta, n0 = Np, into W in chunks of
  // as many rows of Np as the call's own W holds (at least one), so that W grows by less than one row
  const size_t wcap = (size_t)job.S * job.nbatch * job.n0;
  const int chunk = (int)std::max<size_t>(1, wcap / N);
  int e = ensure(c, c->W, std::max<size_t>((size_t)chunk * N, wcap) * sizeof(double2));
  if (e) return e;
  double2 *h = (double2 *)c->W.p;
  DevTmp dimp, part;
  if (rt_malloc(&dimp.p, (size_t)N * sizeof(double))) return fail(c, CWTB_ERR_NOMEM, "device allocation failed");
  {
    std::vector<double> delta(N, 0.0);
    delta[0] = 1.0;
    RT(rt_h2d(dimp.p, delta.data(), (size_t)N * sizeof(double), c->stream));
    RT(rt_sync(c->stream));
  }
  const int nblk = 64;
  if (rt_malloc(&part.p, (size_t)chunk * nblk * sizeof(double))) return fail(c, CWTB_ERR_NOMEM, "device allocation failed");
  std::vector<double> farmax(nc, 0.0);            // largest tap beyond L of t = 0 (device)
  std::vector<double2> win((size_t)nc * 2 * L);   // the taps within L: h[t], t = -L .. L-1 (host)
  for (int r0 = 0; r0 < nc; r0 += chunk) {
    const int nr = std::min(chunk, nc - r0);
    Job imp;
    const double xeps = c->expand_eps;
    c->expand_eps = 0;
    e = build_job(c, imp, (long long)N, dt, cs.data() + r0, nr, family, param, CWTB_F64, false, 1);
    c->expand_eps = xeps;
    if (e) return e;
    if ((e = upload_descs(c, imp))) return e;
    if ((e = run_job<double>(c, imp, (const double *)dimp.p, h, EPI_STORE))) return e;
    if (N > 2u * L) {
      AbsMaxArgs aa{h, (double *)part.p, (long long)N, (long long)L, (long long)N - L, nblk};
      if ((e = launch<AbsMaxBody>(c, nblk, nr, aa))) return e;
      std::vector<double> ph((size_t)nr * nblk);
      RT(rt_d2h(ph.data(), part.p, ph.size() * sizeof(double), c->stream));
      RT(rt_sync(c->stream));
      for (int r = 0; r < nr; ++r)
        for (int b = 0; b < nblk; ++b) farmax[r0 + r] = std::max(farmax[r0 + r], ph[(size_t)r * nblk + b]);
    }
    for (int r = 0; r < nr; ++r) {
      RT(rt_d2h(&win[(size_t)(r0 + r) * 2 * L], h + (size_t)r * N + (N - L), L * sizeof(double2), c->stream));
      RT(rt_d2h(&win[(size_t)(r0 + r) * 2 * L + L], h + (size_t)r * N, L * sizeof(double2), c->stream));
    }
    RT(rt_sync(c->stream));
  }
  // truncation
  struct Acc { int r, t0, t1; };
  std::vector<Acc> acc;
  std::vector<double> m(2 * L), pre(2 * L + 1);
  for (int r = 0; r < nc; ++r) {
    const double2 *w = &win[(size_t)r * 2 * L];
    double mx = farmax[r];
    for (int i = 0; i < 2 * L; ++i) mx = std::max(mx, std::max(std::fabs(w[i].x), std::fabs(w[i].y)));
    const double ulp = 2.220446049250313e-16 * mx;
    if (!(mx > 0) || farmax[r] > 128 * ulp) continue;
    // beyond L the response is rounding noise of its own computation: taps within L count from
    // twice that level up (8 ulp where the far region is empty)
    const double floor_ = std::max(2 * farmax[r], 8 * ulp);
    double l1 = 0;
    pre[0] = 0;
    for (int i = 0; i < 2 * L; ++i) {
      const double a = std::hypot(w[i].x, w[i].y);
      l1 += a;
      m[i] = std::max(std::fabs(w[i].x), std::fabs(w[i].y)) > floor_ ? a : 0.0;
      pre[i + 1] = pre[i] + m[i];
    }
    const double tol = c->band_eps * l1;
    int t0 = 1, t1 = 0;
    for (int M = 1; M <= L / 2 && t0 > t1; ++M)
      for (int a = -(M - 1); a <= 0; ++a) {   // window [a, a + M - 1] contains t = 0
        if (pre[2 * L] - (pre[a + M + L] - pre[a + L]) <= tol) { t0 = a; t1 = a + M - 1; break; }
      }
    if (t0 > t1) continue;
    if (!os_cheaper(t1 - t0 + 1)) continue;
    acc.push_back({r, t0, t1});
  }
  if (acc.empty()) return 0;
  // groups of up to GR rows of similar M; a group runs at the hop of the union of its rows' windows,
  // so a row joins the group only while the cost model still prices that hop below the row's path.
  // Within a group, rows in input order (the order of the class-sorted descriptors) so that H of
  // group row i sits at hoff + i*L.
  std::stable_sort(acc.begin(), acc.end(), [](const Acc &a, const Acc &b) { return a.t1 - a.t0 < b.t1 - b.t0; });
  const int na = (int)acc.size();
  std::vector<double2> hl((size_t)na * L, make_double2(0.0, 0.0));
  long long slot = 0;
  for (int g0 = 0, g1 = 0, grp = 1; g0 < na; g0 = g1, ++grp) {
    int t0 = acc[g0].t0, t1 = acc[g0].t1;
    for (g1 = g0 + 1; g1 < na && g1 - g0 < GR; ++g1) {
      const int u0 = std::min(t0, acc[g1].t0), u1 = std::max(t1, acc[g1].t1);
      if (!os_cheaper(u1 - u0 + 1)) break;
      t0 = u0; t1 = u1;
    }
    std::sort(acc.begin() + g0, acc.begin() + g1, [&](const Acc &a, const Acc &b) { return cand[a.r] < cand[b.r]; });
    for (int i = g0; i < g1; ++i) {
      OsRow &o = os[cand[acc[i].r]];
      o.grp = grp; o.t1 = t1; o.M = t1 - t0 + 1; o.hoff = (slot - (i - g0)) * L;
      const double2 *w = &win[(size_t)acc[i].r * 2 * L];
      for (int t = acc[i].t0; t <= acc[i].t1; ++t)
        hl[(size_t)slot * L + ((t + L) % L)] = make_double2(w[t + L].x / L, w[t + L].y / L);
      ++slot;
    }
  }
  if ((e = ensure(c, c->osH, (size_t)na * L * sizeof(double2)))) return e;
  DevTmp dh;
  if (rt_malloc(&dh.p, (size_t)na * L * sizeof(double2))) return fail(c, CWTB_ERR_NOMEM, "device allocation failed");
  RT(rt_h2d(dh.p, hl.data(), hl.size() * sizeof(double2), c->stream));
  if ((e = fft_rows<double, -1>(c, dh.p, 0, L, L, (double2 *)c->osH.p, L, L, na))) return e;
  RT(rt_sync(c->stream));
  return 0;
}

static int prepare(cwtb_ctx *c, long long n0, double dt, const double *scales, int S, int family,
                   double param, int precision, const void *table, int nbatch = 1) {
  if (!c) return CWTB_ERR_ARG;
  if (precision != CWTB_F64 && precision != CWTB_F32) return fail(c, CWTB_ERR_ARG, "bad precision");
  if (!scales) return fail(c, CWTB_ERR_ARG, "null scales");
  RT(rt_set_device(c->device));
  if (nbatch < 1 || (long long)nbatch * S > 60000)
    return fail(c, CWTB_ERR_ARG, "batch too large for one launch: n_chan * n_scales must be at most 60000");
  // whatever transform was resident is about to be replaced, and the re-runs of cwtb_bench_last /
  // cwtb_profile_last wait for a signal of the new plan
  slot_begin(c->wt);
  c->job_dsig = nullptr;
  cwtb_ctx::PlanKey key;
  key.n0 = n0; key.dt = dt; key.param = param; key.band_eps = c->band_eps; key.band_eps32 = c->band_eps32;
  key.expand_eps = c->expand_eps; key.expand_eps32 = c->expand_eps32; key.S = S; key.family = family;
  key.ga = family == CWTB_MORSE ? c->morse_ga : 0;
  key.precision = precision; key.nbatch = nbatch; key.pad = c->pad_pow2;
  key.scales.assign(scales, scales + std::max(S, 0));
  if (c->plan_reuse && family != CWTB_TABLE && c->job.valid && key == c->plan_key) return 0;
  c->plan_key = cwtb_ctx::PlanKey();   // invalid until the new plan is complete
  // expansion weight tables are cached across calls; start over if many transform geometries have
  // piled up more than CWTB_WTAB_MB of them.  Only here, before any planning of this call: the
  // tables a plan appends must stay until upload_descs has uploaded them (os_plan plans a second job
  // in between).
  if (c->wtab_host.size() * sizeof(double) > c->wtab_max_bytes) {
    c->wtab_host.clear();
    c->wtab_index.clear();
    c->wtab_uploaded = 0;
  }
  int e = build_job(c, c->job, n0, dt, scales, S, family, param, precision, table != nullptr, nbatch);
  if (e) return e;
  std::vector<OsRow> os;
  if ((e = os_plan(c, c->job, dt, family, param, os))) return e;
  if (std::any_of(os.begin(), os.end(), [](const OsRow &o) { return o.grp != 0; })) {
    if ((e = build_job(c, c->job, n0, dt, scales, S, family, param, precision, table != nullptr, nbatch, &os))) return e;
    const Job &job = c->job;
    if ((e = ensure(c, c->osgrp, job.os_groups.size() * sizeof(OsGroup)))) return e;
    RT(rt_h2d(c->osgrp.p, job.os_groups.data(), job.os_groups.size() * sizeof(OsGroup), c->stream));
  }
  if (family == CWTB_TABLE) {
    size_t bytes = (size_t)S * c->job.N * sizeof(double2);
    if ((e = ensure(c, c->table, bytes))) return e;
    RT(rt_h2d(c->table.p, table, bytes, c->stream));
  }
  if ((e = upload_descs(c, c->job))) return e;
  if (family != CWTB_TABLE) c->plan_key = std::move(key);
  return 0;
}

int cwtb_cwt_dev(cwtb_ctx *c, const void *d_signal, int signal_is_f32, int64_t n0, double dt,
                 const double *scales, int n_scales, int family, double param, int precision) {
  if (!c || !d_signal) return fail(c, CWTB_ERR_ARG, "null argument");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, "use cwtb_cwt for CWTB_TABLE");
  int e = prepare(c, n0, dt, scales, n_scales, family, param, precision, nullptr);
  if (e) return e;
  const void *dsig = d_signal;
  const bool want_f32 = (precision == CWTB_F32);
  if ((signal_is_f32 != 0) != want_f32) {  // convert to the engine's real type
    if ((e = ensure(c, c->sig, (size_t)n0 * (want_f32 ? 4 : 8)))) return e;
    unsigned gx = (unsigned)((n0 + NT - 1) / NT);
    if (want_f32) {
      CvtArgs<double, float> a{(const double *)d_signal, (float *)c->sig.p, n0};
      e = launch<CvtBody<double, float>>(c, gx, 1, a);
    } else {
      CvtArgs<float, double> a{(const float *)d_signal, (double *)c->sig.p, n0};
      e = launch<CvtBody<float, double>>(c, gx, 1, a);
    }
    if (e) return e;
    dsig = c->sig.p;
  }
  c->job_dsig = dsig;
  c->job.sig_is_f32 = want_f32;
  return timed_run(c, dsig, 1, &c->last_ms);
}

int cwtb_cwt(cwtb_ctx *c, const void *signal, int signal_is_f32, int64_t n0, double dt,
             const double *scales, int n_scales, int family, double param, int precision,
             const void *table) {
  if (!c || !signal) return fail(c, CWTB_ERR_ARG, "null argument");
  int e = prepare(c, n0, dt, scales, n_scales, family, param, precision, table);
  if (e) return e;
  const bool want_f32 = (precision == CWTB_F32);
  const size_t esz = want_f32 ? 4 : 8;
  if ((e = ensure(c, c->sig, (size_t)n0 * esz))) return e;
  if ((signal_is_f32 != 0) == want_f32) {
    RT(rt_h2d(c->sig.p, signal, (size_t)n0 * esz, c->stream));
    RT(rt_sync(c->stream));
  } else {
    std::vector<unsigned char> tmp((size_t)n0 * esz);
    if (want_f32) for (int64_t i = 0; i < n0; ++i) ((float *)tmp.data())[i] = (float)((const double *)signal)[i];
    else for (int64_t i = 0; i < n0; ++i) ((double *)tmp.data())[i] = (double)((const float *)signal)[i];
    RT(rt_h2d(c->sig.p, tmp.data(), (size_t)n0 * esz, c->stream));
    RT(rt_sync(c->stream));
  }
  c->job_dsig = c->sig.p;
  c->job.sig_is_f32 = want_f32;
  return timed_run(c, c->sig.p, 1, &c->last_ms);
}

int cwtb_bench_last(cwtb_ctx *c, int iters, double *ms_out) {
  if (!c || !c->job.valid || !c->job_dsig) return fail(c, CWTB_ERR_STATE, "no transform to re-run");
  if (iters < 1) return fail(c, CWTB_ERR_ARG, "iters < 1");
  return timed_run(c, c->job_dsig, iters, ms_out);
}

static bool w_resident(const cwtb_ctx *c) { return c->wt.S > 0; }

double cwtb_last_kernel_ms(cwtb_ctx *c) { return c ? c->last_ms : -1; }
int cwtb_last_launch_count(cwtb_ctx *c) { return c ? c->launches : -1; }
int64_t cwtb_padded_length(cwtb_ctx *c) { return (c && c->job.valid) ? (int64_t)c->job.N : -1; }
int64_t cwtb_job_serial(cwtb_ctx *c) { return c ? c->wt.serial : -1; }
void *cwtb_w_device_ptr(cwtb_ctx *c) { return (c && w_resident(c)) ? c->W.p : nullptr; }

int cwtb_last_plan(cwtb_ctx *c, int *out, int n) {
  if (!c || !c->job.valid || !out) return CWTB_ERR_ARG;
  int m = std::min<int>(n, (int)c->job.plan_log2K.size());
  for (int i = 0; i < m; ++i) out[i] = c->job.plan_log2K[i];
  return m;
}

// Host copy of `cnt` coefficients from element `first` of a device complex field of precision
// `prec`: complex128, or complex64 for an fp32 field with out_f64 == 0.
static int field_to_host(cwtb_ctx *c, const void *field, int prec, size_t first, size_t cnt, void *out,
                         int out_f64) {
  if (prec == CWTB_F64) {
    RT(rt_d2h(out, (const double2 *)field + first, cnt * sizeof(double2), c->stream));
    RT(rt_sync(c->stream));
  } else if (!out_f64) {
    RT(rt_d2h(out, (const float2 *)field + first, cnt * sizeof(float2), c->stream));
    RT(rt_sync(c->stream));
  } else {
    // complex64 on the device, complex128 for the caller: widen on the device in chunks and
    // copy each chunk out while the next one is converted (two staging halves, two streams).
    // 16 B per element over PCIe beats an 8 B copy plus a host-side conversion pass.
    const float2 *src = (const float2 *)field + first;
    const size_t chunk = std::min<size_t>(cnt, (size_t)8 << 20);   // elements per staging half
    int e;
    if ((e = ensure(c, c->wide, 2 * chunk * sizeof(double2)))) return e;
    RT(rt_sync(c->stream));   // kernels done
    int half = 0;
    for (size_t off = 0; off < cnt; off += chunk, half ^= 1) {
      const size_t m = std::min(chunk, cnt - off);
      double2 *stage = (double2 *)c->wide.p + (size_t)half * chunk;
      WidenArgs wa{src + off, stage, (long long)m};
      c->cur = c->copy_streams[half];
      e = launch<WidenBody>(c, (unsigned)((m + 4 * NT - 1) / (4 * NT)), 1, wa);
      c->cur = c->stream;
      if (e) return e;
      RT(rt_d2h((double2 *)out + off, stage, m * sizeof(double2), c->copy_streams[half]));
    }
    RT(rt_sync(c->copy_streams[0]));
    RT(rt_sync(c->copy_streams[1]));
  }
  return 0;
}

int cwtb_get_w(cwtb_ctx *c, void *out, int out_f64, int row0, int nrows) {
  if (!c || !w_resident(c) || !out) return fail(c, CWTB_ERR_STATE, "no transform resident");
  const ResidentSlot &w = c->wt;
  if (row0 < 0 || nrows < 0 || row0 + nrows > w.S) return fail(c, CWTB_ERR_ARG, "row range");
  return field_to_host(c, c->W.p, w.prec, (size_t)row0 * w.n0, (size_t)nrows * w.n0, out, out_f64);
}

int cwtb_get_signal_fft(cwtb_ctx *c, void *out) {
  if (!c || !c->job.valid || !out) return fail(c, CWTB_ERR_STATE, "no transform resident");
  const Job &job = c->job;
  const size_t cnt = job.N / 2 > 0 ? job.N / 2 - 1 : 0;
  if (cnt == 0) return 0;
  const double sc = 1.0 / std::sqrt((double)job.N);
  double *o = (double *)out;
  if (job.precision == CWTB_F64) {
    // scaled on the device (the host loop cost as much as the 8 MB copy at N = 2^20)
    int e = ensure(c, c->aux, cnt * sizeof(double2));
    if (e) return e;
    ScaleCopyArgs sa{(const double *)((const double2 *)c->spec.p + 1), (double *)c->aux.p, (long long)(2 * cnt), sc};
    if ((e = launch<ScaleCopyBody>(c, (unsigned)((2 * cnt + NT - 1) / NT), 1, sa))) return e;
    RT(rt_d2h(out, c->aux.p, cnt * sizeof(double2), c->stream));
    RT(rt_sync(c->stream));
  } else {
    std::vector<float> tmp(cnt * 2);
    RT(rt_d2h(tmp.data(), (const float2 *)c->spec.p + 1, cnt * sizeof(float2), c->stream));
    RT(rt_sync(c->stream));
    for (size_t i = 0; i < cnt * 2; ++i) o[i] = (double)tmp[i] * sc;
  }
  return 0;
}

int cwtb_fft_c2c(cwtb_ctx *c, const void *in, void *out, int64_t n, int batch, int sign, int precision) {
  if (!c || !in || !out || n < 2 || batch < 1 || (sign != 1 && sign != -1))
    return fail(c, CWTB_ERR_ARG, "fft_c2c: bad argument");
  if (precision != CWTB_F64 && precision != CWTB_F32) return fail(c, CWTB_ERR_ARG, "bad precision");
  if (n > (1ll << 26)) return fail(c, CWTB_ERR_UNSUPPORTED, "fft_c2c: n > 2^26");
  const bool pow2 = (n & (n - 1)) == 0;
  if (!pow2 && precision != CWTB_F64) return fail(c, CWTB_ERR_UNSUPPORTED, "fft_c2c: lengths other than 2^k run in fp64");
  if (!pow2 && n > (1ll << 24)) return fail(c, CWTB_ERR_UNSUPPORTED, "fft_c2c: non power-of-two n > 2^24");
  RT(rt_set_device(c->device));
  const size_t cnt = (size_t)n * batch;
  const size_t esz = precision == CWTB_F64 ? sizeof(double2) : sizeof(float2);
  int e;
  // context-owned staging buffers (released with the context, also on error paths)
  if ((e = ensure(c, c->C, cnt * esz))) return e;
  if ((e = ensure(c, c->A12, cnt * esz))) return e;
  void *din = c->C.p, *dout = c->A12.p;
  if (!pow2) {   // any length: Bluestein on the power-of-two kernels
    RT(rt_h2d(din, in, cnt * esz, c->stream));
    if ((e = blue_rows(c, din, 0, n, (double2 *)dout, n, (unsigned)n, batch, sign, 1.0, n))) return e;
    RT(rt_d2h(out, dout, cnt * esz, c->stream));
    RT(rt_sync(c->stream));
    return 0;
  }
  if (precision == CWTB_F64) {
    RT(rt_h2d(din, in, cnt * esz, c->stream));
    e = sign < 0 ? fft_rows<double, -1>(c, din, 0, n, n, (double2 *)dout, n, (unsigned)n, batch)
                 : fft_rows<double, +1>(c, din, 0, n, n, (double2 *)dout, n, (unsigned)n, batch);
    if (e) return e;
    RT(rt_d2h(out, dout, cnt * esz, c->stream));
    RT(rt_sync(c->stream));
    return 0;
  }
  std::vector<float> tmp(cnt * 2);
  const double *src = (const double *)in;
  for (size_t i = 0; i < cnt * 2; ++i) tmp[i] = (float)src[i];
  RT(rt_h2d(din, tmp.data(), cnt * esz, c->stream));
  RT(rt_sync(c->stream));
  e = sign < 0 ? fft_rows<float, -1>(c, din, 0, n, n, (float2 *)dout, n, (unsigned)n, batch)
               : fft_rows<float, +1>(c, din, 0, n, n, (float2 *)dout, n, (unsigned)n, batch);
  if (e) return e;
  RT(rt_d2h(tmp.data(), dout, cnt * esz, c->stream));
  RT(rt_sync(c->stream));
  double *o = (double *)out;
  for (size_t i = 0; i < cnt * 2; ++i) o[i] = (double)tmp[i];
  return 0;
}

}  // extern "C"

extern "C" {

// ---- helpers for the post-processing entry points ---------------------------------------
static int upload_doubles(cwtb_ctx *c, Buf &b, const std::vector<double> &v) {
  int e = ensure(c, b, v.size() * sizeof(double));
  if (e) return e;
  RT(rt_h2d(b.p, v.data(), v.size() * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

static int upload_signal_f64(cwtb_ctx *c, Buf &b, const double *y, long long n0) {
  int e = ensure(c, b, (size_t)n0 * sizeof(double));
  if (e) return e;
  RT(rt_h2d(b.p, y, (size_t)n0 * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

// boxcar with half-weight end taps, normalised (helpers.py:176-191), followed by one unit tap
// (the one-tap window of wct_core's path for boxcars longer than 64 taps)
static int upload_window(cwtb_ctx *c, int K) {
  if (K < 1) return fail(c, CWTB_ERR_ARG, "boxcar length must be >= 1");
  std::vector<double> w(K, 1.0);
  w[0] = 0.5;
  w[K - 1] = 0.5;   // K == 1: single tap 0.5, normalised to 1
  double sum = 0;
  for (double v : w) sum += v;
  for (double &v : w) v /= sum;
  w.push_back(1.0);
  return upload_doubles(c, c->win, w);
}

extern "C++" {   // templates of the coherence pipeline, one instantiation per engine type
// Morlet.smooth, time part (mothers.py:83-93), in place on X[S][n0] (complex, engine type T, device):
// forward transform of the zero-padded rows with the Gaussian folded into its output pass,
// inverse transform trimmed to n0.
template <typename T>
static int smooth_time(cwtb_ctx *c, cx<T> *X, int S, long long n0, unsigned N, const double *d_g) {
  int e = ensure(c, c->F, (size_t)S * N * sizeof(cx<T>));
  if (e) return e;
  cx<T> *F = (cx<T> *)c->F.p;
  if (N < 2) return 0;  // single sample: filter is exp(0) = 1
  const bool table = c->filt_rows > 0;     // caller-supplied responses instead of Morlet's Gaussian
  if (table && (c->filt_rows != S || c->filt_n != (long long)N))
    return fail(c, CWTB_ERR_STATE, "smoothing filter table does not match the rows / transform length of this call");
  if ((N & (N - 1)) != 0) {
    // un-padded mode: circular filter at the rows' own length (N == n0), Bluestein transforms
    if constexpr (sizeof(T) == 8) {
      if ((e = blue_rows(c, X, 0, n0, F, N, N, S, -1, 1.0, N))) return e;
      if (table) {
        FilterMulArgs<T> fa{F, (const double *)c->filt.p, (long long)N, N, 1.0 / (double)N};
        if ((e = launch<FilterMulBody<T>>(c, (N + NT - 1) / NT, S, fa))) return e;
      } else {
        BlueGaussArgs ga{F, d_g, (long long)N, N, 1.0 / (double)N};
        if ((e = launch<BlueGaussBody>(c, (N + NT - 1) / NT, S, ga))) return e;
      }
      return blue_rows(c, F, 0, N, X, n0, N, S, +1, 1.0, n0);
    } else {
      return fail(c, CWTB_ERR_UNSUPPORTED, "un-padded transforms run in fp64");
    }
  }
  if (table) {
    if ((e = fft_rows<T, -1>(c, X, 0, n0, n0, F, N, N, S, N))) return e;
    FilterMulArgs<T> fa{F, (const double *)c->filt.p, (long long)N, N, 1.0 / (double)N};
    if ((e = launch<FilterMulBody<T>>(c, (N + NT - 1) / NT, S, fa))) return e;
  } else if ((e = fft_rows<T, -1>(c, X, 0, n0, n0, F, N, N, S, N, d_g, 1.0 / (double)N))) {
    return e;
  }
  return fft_rows<T, +1>(c, F, 0, N, N, X, n0, N, S, n0);
}

// two transforms + coherence pipeline in the engine type T; outputs are device pointers (any may
// be null) and double for every T
template <typename T>
static int wct_core(cwtb_ctx *c, const Job &job, const T *dsig1, const T *dsig2, int K,
                    double *dWCT, double *daWCT, const unsigned char *dmask, int maxscale, int nbins,
                    unsigned long long *dhist, const double *dobs = nullptr, unsigned *dcnt = nullptr,
                    const SelArgs *sel = nullptr) {
  using V = cx<T>;
  const int S = job.S;
  const long long n0 = job.n0;
  const size_t cnt = (size_t)S * n0;
  int e;
  if ((e = ensure(c, c->W, cnt * sizeof(V)))) return e;
  if ((e = ensure(c, c->W2, cnt * sizeof(V)))) return e;
  if ((e = ensure(c, c->C, cnt * sizeof(V)))) return e;
  if ((e = ensure(c, c->A12, cnt * sizeof(V)))) return e;
  if ((e = run_job<T>(c, job, dsig1, (V *)c->W.p, EPI_STORE))) return e;
  if ((e = run_job<T>(c, job, dsig2, (V *)c->W2.p, EPI_STORE))) return e;
  const double *d_scale = (const double *)c->rowd.p;      // [S] scales, then [S] g
  const double *d_g = d_scale + S;
  WctPrepArgs<T> pa{(const V *)c->W.p, (const V *)c->W2.p, d_scale, (V *)c->C.p, (V *)c->A12.p, daWCT, n0};
  const unsigned gx = (unsigned)((n0 + NT - 1) / NT);
  if ((e = launch<WctPrepBody<T>>(c, gx, S, pa))) return e;
  if (c->angle_host && daWCT) {   // the angle is final here: its 8 B per point cross PCIe under the smoothing
    RT(rt_record(c->ev_angle, c->stream));
    RT(rt_wait(c->copy_streams[0], c->ev_angle));
    RT(rt_d2h(c->angle_host, daWCT, cnt * sizeof(double), c->copy_streams[0]));
  }
  if ((e = smooth_time<T>(c, (V *)c->C.p, S, n0, job.N, d_g))) return e;
  if ((e = smooth_time<T>(c, (V *)c->A12.p, S, n0, job.N, d_g))) return e;
  const int rows_out = dWCT || dcnt || sel ? S : maxscale;   // counting or selection bits: every row
  if (rows_out <= 0) return 0;
  WctFinalArgs<T> fa{(const V *)c->C.p, (const V *)c->A12.p, (const double *)c->win.p, dWCT,
                     dmask, dhist, n0, S, K, maxscale, nbins, dobs, dcnt, sel ? *sel : SelArgs{}};
  if (K > 64) {
    // longer than the fused kernel stages: the scale boxcar of both fields into W and W2 (dead
    // since WctPrepBody), then the ratio through the fused kernel with the unit tap at win + K
    BoxcarArgs<T> b1{fa.C, (V *)c->W.p, fa.win, n0, S, K}, b2{fa.A12, (V *)c->W2.p, fa.win, n0, S, K};
    if ((e = launch<BoxcarBody<T>>(c, gx, rows_out, b1))) return e;
    if ((e = launch<BoxcarBody<T>>(c, gx, rows_out, b2))) return e;
    fa.C = (const V *)c->W.p;
    fa.A12 = (const V *)c->W2.p;
    fa.win += K;
    fa.K = 1;
  }
  using F16 = WctFinalBody<T, 16>;
  const unsigned fx = (unsigned)((n0 + F16::CW - 1) / F16::CW), fy = (unsigned)((rows_out + F16::RS - 1) / F16::RS);
  if (sel)
    return K <= 16 ? launch<WctFinalBody<T, 16, true>>(c, fx, fy, fa) : launch<WctFinalBody<T, 64, true>>(c, fx, fy, fa);
  return K <= 16 ? launch<F16>(c, fx, fy, fa) : launch<WctFinalBody<T, 64>>(c, fx, fy, fa);
}

// the launch of Wct3FinalBody: F16 for boxcars of up to 16 taps, else F64K
template <class F16, class F64K>
static int wct3_final(cwtb_ctx *c, const typename F16::Args &fa, int K, long long n0, int rows_out) {
  if (K <= 16)
    return launch<F16>(c, (unsigned)((n0 + F16::CW - 1) / F16::CW), (unsigned)((rows_out + F16::RS - 1) / F16::RS), fa);
  return launch<F64K>(c, (unsigned)((n0 + F64K::CW - 1) / F64K::CW), (unsigned)((rows_out + F64K::RS - 1) / F64K::RS), fa);
}

// three transforms + partial / multiple coherence in the engine type T; outputs are device
// pointers (any may be null) and double for every T, dPP the partial phase.  With every output null
// (Monte-Carlo mode) only the rows below maxscale are finished, into the histograms dhP / dhM
// (either may be null); with counters (cP / cM, against the observed oP / oM) or selection bits
// (sel) every row is finished.
// Device memory per scale-point: the three transforms W, W2, W3 (the crosses are written over
// them), the two auto fields C, A12 and the smoothing buffer F.
template <typename T>
static int wct3_core(cwtb_ctx *c, const Job &job, const T *dy, const T *dx1, const T *dx2, int K,
                     double *dRP2, double *dRM2, const unsigned char *dmask = nullptr, int maxscale = 0,
                     int nbins = 0, unsigned long long *dhP = nullptr, unsigned long long *dhM = nullptr,
                     double *dPP = nullptr, const double *oP = nullptr, const double *oM = nullptr,
                     unsigned *cP = nullptr, unsigned *cM = nullptr, const SelArgs *sel = nullptr) {
  using V = cx<T>;
  const int S = job.S;
  const long long n0 = job.n0;
  const size_t cnt = (size_t)S * n0;
  int e;
  for (Buf *b : {&c->W, &c->W2, &c->W3, &c->C, &c->A12})
    if ((e = ensure(c, *b, cnt * sizeof(V)))) return e;
  if ((e = run_job<T>(c, job, dy, (V *)c->W.p, EPI_STORE))) return e;
  if ((e = run_job<T>(c, job, dx1, (V *)c->W2.p, EPI_STORE))) return e;
  if ((e = run_job<T>(c, job, dx2, (V *)c->W3.p, EPI_STORE))) return e;
  const double *d_scale = (const double *)c->rowd.p;      // [S] scales, then [S] g
  const double *d_g = d_scale + S;
  V *f[5] = {(V *)c->C.p, (V *)c->A12.p, (V *)c->W.p, (V *)c->W2.p, (V *)c->W3.p};
  Wct3PrepArgs<T> pa{f[2], f[3], f[4], d_scale, f[0], f[1], f[2], f[3], f[4], n0};
  const unsigned gx = (unsigned)((n0 + NT - 1) / NT);
  if ((e = launch<Wct3PrepBody<T>>(c, gx, S, pa))) return e;
  for (V *x : f)
    if ((e = smooth_time<T>(c, x, S, n0, job.N, d_g))) return e;
  const int rows_out = dRP2 || dRM2 || dPP || cP || cM || sel ? S : maxscale;
  if (rows_out <= 0) return 0;
  const double *win = (const double *)c->win.p;
  if (K > 64) {
    // longer than the fused kernel stages: the scale boxcar of each field into the buffer the
    // previous field left (the first into F, free after the smoothing), then the fused kernel
    // with the unit tap at win + K
    V *dst = (V *)c->F.p;
    for (V *&x : f) {
      BoxcarArgs<T> b{x, dst, win, n0, S, K};
      if ((e = launch<BoxcarBody<T>>(c, gx, rows_out, b))) return e;
      std::swap(x, dst);
    }
    win += K;
    K = 1;
  }
  Wct3FinalArgs<T> fa{f[0], f[1], f[2], f[3], f[4], win, dRP2, dRM2, dPP, dmask, dhP, dhM, n0, S, K, maxscale, nbins,
                      oP, oM, cP, cM, sel ? *sel : SelArgs{}};
  if (sel) return wct3_final<Wct3FinalBody<T, 16, 32, 16, true>, Wct3FinalBody<T, 64, 64, 8, true>>(c, fa, K, n0, rows_out);
  return wct3_final<Wct3FinalBody<T, 16, 32, 16>, Wct3FinalBody<T, 64, 64, 8>>(c, fa, K, n0, rows_out);
}

// the engine precision of T, and host series (double) as device series of type T: the fp32
// coherence converts on the device, so that its inputs are the fp64 inputs rounded
template <typename T> constexpr int prec_of() { return sizeof(T) == 8 ? CWTB_F64 : CWTB_F32; }

static int to_f32(cwtb_ctx *c, const double *in, float *out, long long n) {
  CvtArgs<double, float> a{in, out, n};
  return launch<CvtBody<double, float>>(c, (unsigned)((n + NT - 1) / NT), 1, a);
}

template <typename T> static int upload_series(cwtb_ctx *c, Buf &b, const double *y, long long n0) {
  if constexpr (sizeof(T) == 8) {
    return upload_signal_f64(c, b, y, n0);
  } else {
    int e = upload_signal_f64(c, c->scratch, y, n0);
    if (e) return e;
    if ((e = ensure(c, b, (size_t)n0 * sizeof(float)))) return e;
    return to_f32(c, (const double *)c->scratch.p, (float *)b.p, n0);
  }
}
}  // extern "C++"

static int upload_row_tables(cwtb_ctx *c, const Job &job) {
  std::vector<double> v(2 * (size_t)job.S);
  for (int j = 0; j < job.S; ++j) {
    v[j] = job.scales[j];
    const double snorm = job.scales[j] / job.dt;
    v[job.S + j] = -0.5 * (snorm * snorm);
  }
  return upload_doubles(c, c->rowd, v);
}

// rows of W written by the single-kernel classes (the chain on aux_stream): true and *r0 set if
// they are exactly the rows [r0, S) -- the case for any ascending scale array
static bool single_kernel_rows(const cwtb_ctx *c, const Job &job, int *r0) {
  const int S = job.S;
  int lo = S, cnt = 0;
  for (const ClassRun &cl : job.classes) {
    if (!(cl.expand || class_single(job, cl))) continue;
    for (int i = cl.first; i < cl.first + cl.count; ++i) {
      lo = std::min(lo, job.descs[i].row);
      ++cnt;
    }
  }
  if (cnt == 0 || cnt == S || lo != S - cnt) return false;
  *r0 = lo;
  return true;
}

int cwtb_cwt_to_host(cwtb_ctx *c, const void *signal, int signal_is_f32, int64_t n0, double dt,
                     const double *scales, int n_scales, int family, double param, int precision,
                     void *out, int out_f64) {
  if (!c || !signal || !out) return fail(c, CWTB_ERR_ARG, "null argument");
  // fp64, analytic family, forked streams: the device->host copy of the rows the single-kernel
  // chain produced starts as soon as that chain is done, while the two-kernel chains still run
  if (precision == CWTB_F64 && family != CWTB_TABLE && !c->profiling) {
    int e = prepare(c, n0, dt, scales, n_scales, family, param, precision, nullptr);
    if (e) return e;
    const Job &job = c->job;
    int r0 = 0;
    if (!job.exact && job.N >= 32 && job.nbatch == 1 && single_kernel_rows(c, job, &r0)) {
      if ((e = ensure(c, c->sig, (size_t)n0 * sizeof(double)))) return e;
      if (signal_is_f32) {
        std::vector<double> tmp((size_t)n0);
        for (int64_t i = 0; i < n0; ++i) tmp[i] = (double)((const float *)signal)[i];
        RT(rt_h2d(c->sig.p, tmp.data(), (size_t)n0 * sizeof(double), c->stream));
        RT(rt_sync(c->stream));
      } else {
        RT(rt_h2d(c->sig.p, signal, (size_t)n0 * sizeof(double), c->stream));
      }
      c->job_dsig = c->sig.p;
      c->job.sig_is_f32 = 0;
      c->launches = 0;
      if ((e = time_begin(c))) return e;
      if ((e = run_job<double>(c, job, (const double *)c->sig.p))) return e;
      if ((e = time_stop(c))) return e;
      const size_t rowb = (size_t)n0 * sizeof(double2);
      const char *W = (const char *)c->W.p;
      RT(rt_wait(c->copy_streams[0], c->ev_join));   // single-kernel chain done
      RT(rt_d2h((char *)out + (size_t)r0 * rowb, W + (size_t)r0 * rowb, (size_t)(n_scales - r0) * rowb, c->copy_streams[0]));
      RT(rt_d2h(out, W, (size_t)r0 * rowb, c->stream));               // after every chain has joined
      RT(rt_sync(c->copy_streams[0]));
      RT(rt_sync(c->stream));
      if ((e = time_read(c, &c->last_ms))) return e;
      w_fill(c);
      return 0;
    }
    // not eligible: fall through to the plain sequence (prepare runs again, cheap)
  }
  int e = cwtb_cwt(c, signal, signal_is_f32, n0, dt, scales, n_scales, family, param, precision, nullptr);
  if (e) return e;
  return w_kept(c, cwtb_get_w(c, out, out_f64, 0, n_scales));
}

// rows per block of the column reductions: enough blocks to fill the machine, few enough that the
// atomics stay negligible
static int reduction_rows_per_block(int rows) { return rows <= 32 ? rows : 32; }

int cwtb_icwt_sum(cwtb_ctx *c, double *out) {
  if (!c || !w_resident(c) || !out) return fail(c, CWTB_ERR_STATE, "no transform resident");
  const Job &job = c->job;
  if (job.nbatch != 1) return fail(c, CWTB_ERR_UNSUPPORTED, "icwt of a batched transform: fetch rows per channel");
  std::vector<double> rs(job.S);
  for (int j = 0; j < job.S; ++j) rs[j] = 1.0 / std::sqrt(job.scales[j]);
  int e = upload_doubles(c, c->rowd, rs);
  if (e) return e;
  if ((e = ensure(c, c->aux, (size_t)job.n0 * sizeof(double)))) return e;
  const unsigned gx = (unsigned)((job.n0 + NT - 1) / NT);
  const int rpb = reduction_rows_per_block(job.S);
  const unsigned gy = (unsigned)((job.S + rpb - 1) / rpb);
  if (gy > 1) RT(rt_memset(c->aux.p, 0, (size_t)job.n0 * sizeof(double), c->stream));
  if (job.precision == CWTB_F64) {
    IcwtArgs<double> a{(const double2 *)c->W.p, (const double *)c->rowd.p, (double *)c->aux.p, job.n0, job.n0, job.S, 0, rpb};
    e = launch<IcwtBody<double>>(c, gx, gy, a);
  } else {
    IcwtArgs<float> a{(const float2 *)c->W.p, (const double *)c->rowd.p, (double *)c->aux.p, job.n0, job.n0, job.S, 0, rpb};
    e = launch<IcwtBody<float>>(c, gx, gy, a);
  }
  if (e) return e;
  RT(rt_d2h(out, c->aux.p, (size_t)job.n0 * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

int cwtb_icwt_sum_host(cwtb_ctx *c, const void *W, const double *scales, int n_scales, int64_t n, double *out) {
  if (!c || !W || !scales || !out || n_scales < 1 || n < 1) return fail(c, CWTB_ERR_ARG, "icwt: bad argument");
  std::vector<double> rs(n_scales);
  for (int j = 0; j < n_scales; ++j) rs[j] = 1.0 / std::sqrt(scales[j]);
  int e = upload_doubles(c, c->rowd, rs);
  if (e) return e;
  if ((e = ensure(c, c->aux, (size_t)n * sizeof(double)))) return e;
  const int chunk = (int)std::max<long long>(1, std::min<long long>(n_scales, (256ll << 20) / (n * 16)));
  if ((e = ensure(c, c->scratch, (size_t)chunk * n * sizeof(double2)))) return e;
  const unsigned gx = (unsigned)((n + NT - 1) / NT);
  for (int r0 = 0; r0 < n_scales; r0 += chunk) {
    const int nr = std::min(chunk, n_scales - r0);
    RT(rt_h2d(c->scratch.p, (const double2 *)W + (size_t)r0 * n, (size_t)nr * n * sizeof(double2), c->stream));
    IcwtArgs<double> a{(const double2 *)c->scratch.p, (const double *)c->rowd.p + r0, (double *)c->aux.p, n, n, nr, r0 > 0, nr};
    if ((e = launch<IcwtBody<double>>(c, gx, 1, a))) return e;
    RT(rt_sync(c->stream));
  }
  RT(rt_d2h(out, c->aux.p, (size_t)n * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

static int power_common(cwtb_ctx *c, double *power_out, double *mean_out, const double *row_scale,
                        const int64_t *lo, const int64_t *hi) {
  if (!c || !w_resident(c)) return fail(c, CWTB_ERR_STATE, "no transform resident");
  const Job &job = c->job;
  const int R = job.S * job.nbatch;
  const size_t cnt = (size_t)R * job.n0;
  // aux: [row sums R][row factors R][lo R][hi R][power cnt]
  int e = ensure(c, c->aux, (power_out ? cnt : 0) * sizeof(double) + (size_t)4 * R * sizeof(double));
  if (e) return e;
  double *dsum = (double *)c->aux.p;
  double *dmul = dsum + R;
  long long *dlo = (long long *)(dmul + R), *dhi = dlo + R;
  double *dpow = power_out ? (double *)(dhi + R) : nullptr;
  RT(rt_memset(dsum, 0, (size_t)R * sizeof(double), c->stream));
  if (row_scale) RT(rt_h2d(dmul, row_scale, (size_t)R * sizeof(double), c->stream));
  std::vector<long long> rng;
  if (lo && hi) {
    rng.resize(2 * (size_t)R);
    for (int j = 0; j < R; ++j) {
      rng[j] = std::max<long long>(0, lo[j]);
      rng[R + j] = std::min<long long>(job.n0, hi[j]);
    }
    RT(rt_h2d(dlo, rng.data(), rng.size() * sizeof(long long), c->stream));
  }
  const unsigned gx = (unsigned)((job.n0 + PowerBody<double>::PER * NT - 1) / (PowerBody<double>::PER * NT));
  if (job.precision == CWTB_F64) {
    PowerArgs<double> a{(const double2 *)c->W.p, dpow, dsum, job.n0, row_scale ? dmul : nullptr,
                        rng.empty() ? nullptr : dlo, rng.empty() ? nullptr : dhi};
    e = launch<PowerBody<double>>(c, gx, R, a);
  } else {
    PowerArgs<float> a{(const float2 *)c->W.p, dpow, dsum, job.n0, row_scale ? dmul : nullptr,
                       rng.empty() ? nullptr : dlo, rng.empty() ? nullptr : dhi};
    e = launch<PowerBody<float>>(c, gx, R, a);
  }
  if (e) return e;
  if (power_out) RT(rt_d2h(power_out, dpow, cnt * sizeof(double), c->stream));
  if (mean_out) RT(rt_d2h(mean_out, dsum, (size_t)R * sizeof(double), c->stream));
  RT(rt_sync(c->stream));   // also covers the pageable host sources above
  if (mean_out)
    for (int j = 0; j < R; ++j) {
      const long long cntj = rng.empty() ? (long long)job.n0 : rng[R + j] - rng[j];
      mean_out[j] = cntj > 0 ? mean_out[j] / (double)cntj : std::nan("");
    }
  return 0;
}
int cwtb_get_power(cwtb_ctx *c, double *out) { return power_common(c, out, nullptr, nullptr, nullptr, nullptr); }
int cwtb_global_power(cwtb_ctx *c, double *out) { return power_common(c, nullptr, out, nullptr, nullptr, nullptr); }
int cwtb_get_power_scaled(cwtb_ctx *c, const double *row_scale, double *out) {
  if (!out) return fail(c, CWTB_ERR_ARG, "null argument");
  return power_common(c, out, nullptr, row_scale, nullptr, nullptr);
}
int cwtb_global_power_ranges(cwtb_ctx *c, const int64_t *lo, const int64_t *hi, double *out) {
  if (!lo || !hi || !out) return fail(c, CWTB_ERR_ARG, "null argument");
  return power_common(c, nullptr, out, nullptr, lo, hi);
}

// scale-averaged power of the S x n0 complex field W of precision prec (cwtb_scale_avg_power)
static int scale_avg_power_run(cwtb_ctx *c, const void *W, int prec, int S, long long n0, const double *weights,
                               double *out) {
  if (!weights || !out) return fail(c, CWTB_ERR_ARG, "null argument");
  // [weights S doubles][selected rows S ints]: rows with a zero weight are not read at all
  std::vector<double> w(weights, weights + S);
  std::vector<int> sel;
  for (int j = 0; j < S; ++j)
    if (w[j] != 0.0) sel.push_back(j);
  const int nsel = (int)sel.size();
  w.resize((size_t)S + ((size_t)S + 1) / 2);
  if (nsel) memcpy(w.data() + S, sel.data(), sizeof(int) * nsel);
  int e = upload_doubles(c, c->rowd, w);
  if (e) return e;
  if ((e = ensure(c, c->aux, (size_t)n0 * sizeof(double)))) return e;
  const unsigned gx = (unsigned)((n0 + NT - 1) / NT);
  const int spb = nsel <= 32 ? std::max(nsel, 1) : 32;
  const unsigned gy = (unsigned)std::max(1, (nsel + spb - 1) / spb);
  if (gy > 1) RT(rt_memset(c->aux.p, 0, (size_t)n0 * sizeof(double), c->stream));
  const int *dsel = (const int *)((const double *)c->rowd.p + S);
  if (prec == CWTB_F64) {
    ScaleAvgArgs<double> a{(const double2 *)W, (const double *)c->rowd.p, (double *)c->aux.p, n0, S, dsel, nsel, spb};
    e = launch<ScaleAvgBody<double>>(c, gx, gy, a);
  } else {
    ScaleAvgArgs<float> a{(const float2 *)W, (const double *)c->rowd.p, (double *)c->aux.p, n0, S, dsel, nsel, spb};
    e = launch<ScaleAvgBody<float>>(c, gx, gy, a);
  }
  if (e) return e;
  RT(rt_d2h(out, c->aux.p, (size_t)n0 * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

int cwtb_scale_avg_power(cwtb_ctx *c, const double *weights, double *out) {
  if (!c || !w_resident(c)) return fail(c, CWTB_ERR_STATE, "no transform resident");
  const Job &job = c->job;
  if (job.nbatch != 1) return fail(c, CWTB_ERR_UNSUPPORTED, "scale average of a batched transform: fetch rows per channel");
  return scale_avg_power_run(c, c->W.p, job.precision, job.S, job.n0, weights, out);
}

// W12 in W; the plan is a job of type T afterwards: cwtb_get_w widens an fp32 W12 on the device
extern "C++" {
template <typename T>
static int xwt_run(cwtb_ctx *c, const double *y1, const double *y2, int64_t n0, double dt, const double *scales,
                   int n_scales, int family, double param) {
  int e = prepare(c, n0, dt, scales, n_scales, family, param, prec_of<T>(), nullptr);
  if (e) return e;
  if ((e = upload_series<T>(c, c->sig, y1, n0))) return e;
  if ((e = upload_series<T>(c, c->sig2, y2, n0))) return e;
  c->launches = 0;
  if ((e = time_begin(c))) return e;
  if ((e = run_job<T>(c, c->job, (const T *)c->sig.p, nullptr, EPI_STORE))) return e;
  if ((e = run_job<T>(c, c->job, (const T *)c->sig2.p, nullptr, EPI_MULCONJ))) return e;
  if ((e = time_end(c, &c->last_ms))) return e;
  c->job_dsig = nullptr;
  RT(rt_sync(c->stream));
  return 0;
}
}  // extern "C++"

int cwtb_xwt(cwtb_ctx *c, const double *y1, const double *y2, int64_t n0, double dt, const double *scales,
             int n_scales, int family, double param, void *W12_out) {
  if (!c || !y1 || !y2) return fail(c, CWTB_ERR_ARG, "null argument");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, "xwt needs an analytic wavelet family");
  int e = c->coh_precision == CWTB_F32 ? xwt_run<float>(c, y1, y2, n0, dt, scales, n_scales, family, param)
                                       : xwt_run<double>(c, y1, y2, n0, dt, scales, n_scales, family, param);
  if (e) return e;
  w_fill(c);   // W12 is the resident transform
  return W12_out ? w_kept(c, cwtb_get_w(c, W12_out, 1, 0, n_scales)) : 0;
}

// ---- resident products and the reading calls ------------------------------------------------
static int slot_release(cwtb_ctx *c, ResidentSlot &s) {
  slot_begin(s);
  if (s.buf.p || s.counts.p || s.labels.p) {
    RT(rt_set_device(c->device));
    RT(rt_sync(c->stream));
    for (Buf *b : {&s.buf, &s.counts, &s.labels}) {
      if (b->p) rt_free(b->p);
      *b = Buf{};
    }
  }
  return 0;
}

int cwtb_xwt_resident(cwtb_ctx *c, const double *y1, const double *y2, int64_t n0, double dt,
                      const double *scales, int n_scales, int family, double param) {
  if (!c || !y1 || !y2) return fail(c, CWTB_ERR_ARG, "null argument");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, "xwt needs an analytic wavelet family");
  slot_begin(c->cross);
  int e = c->coh_precision == CWTB_F32 ? xwt_run<float>(c, y1, y2, n0, dt, scales, n_scales, family, param)
                                       : xwt_run<double>(c, y1, y2, n0, dt, scales, n_scales, family, param);
  if (e) return e;
  // W12 is the transform's W: take the buffer over.  No kernel or plan keeps W's address (every
  // run takes it afresh from c->W), so the old cross buffer can serve as the next W.
  std::swap(c->W, c->cross.buf);
  c->cross.S = n_scales;
  c->cross.n0 = n0;
  c->cross.prec = c->job.precision;
  return 0;
}

int64_t cwtb_cross_serial(cwtb_ctx *c) { return c ? c->cross.serial : -1; }
int cwtb_cross_release(cwtb_ctx *c) { return c ? slot_release(c, c->cross) : CWTB_ERR_ARG; }

// W of one series in W: what cwtb_cwt runs on it in the engine type T (the series rounded on the
// device for fp32, as cwtb_cwt rounds it on the host)
extern "C++" {
template <typename T>
static int power_run(cwtb_ctx *c, const double *y, int64_t n0, double dt, const double *scales, int n_scales,
                     int family, double param) {
  int e = prepare(c, n0, dt, scales, n_scales, family, param, prec_of<T>(), nullptr);
  if (e) return e;
  if ((e = upload_series<T>(c, c->sig, y, n0))) return e;
  c->launches = 0;
  if ((e = time_begin(c))) return e;
  if ((e = run_job<T>(c, c->job, (const T *)c->sig.p, nullptr, EPI_STORE))) return e;
  if ((e = time_end(c, &c->last_ms))) return e;
  c->job_dsig = nullptr;
  RT(rt_sync(c->stream));
  return 0;
}
}  // extern "C++"

int cwtb_power_resident(cwtb_ctx *c, const double *y, int64_t n0, double dt, const double *scales, int n_scales,
                        int family, double param) {
  if (!c || !y) return fail(c, CWTB_ERR_ARG, "null argument");
  slot_begin(c->pw);
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, "power_resident needs an analytic wavelet family");
  int e = c->coh_precision == CWTB_F32 ? power_run<float>(c, y, n0, dt, scales, n_scales, family, param)
                                       : power_run<double>(c, y, n0, dt, scales, n_scales, family, param);
  if (e) return e;
  std::swap(c->W, c->pw.buf);   // as cwtb_xwt_resident: the transform's W becomes the slot's buffer
  c->pw.S = n_scales;
  c->pw.n0 = n0;
  c->pw.prec = c->job.precision;
  return 0;
}

int64_t cwtb_power_serial(cwtb_ctx *c) { return c ? c->pw.serial : -1; }
int cwtb_power_release(cwtb_ctx *c) { return c ? slot_release(c, c->pw) : CWTB_ERR_ARG; }

int cwtb_power_scale_avg(cwtb_ctx *c, const double *weights, double *out) {
  if (!c) return CWTB_ERR_ARG;
  const ResidentSlot &s = c->pw;
  if (s.S <= 0 || !s.buf.p) return fail(c, CWTB_ERR_STATE, "no power resident");
  RT(rt_set_device(c->device));
  return scale_avg_power_run(c, s.buf.p, s.prec, s.S, s.n0, weights, out);
}

// WCT and aWCT of a coherence share one device buffer; aWCT starts on a 256-byte boundary, so that
// a flat index has the same alignment in both fields (the 16-byte loads of RowStatsBody<CohView>)
static size_t coh_angle_offset(size_t cnt) { return (cnt + 31) & ~(size_t)31; }

// A resident field of the reading calls: a cwtb_field (the transform's W, the cross spectrum or the
// kept W of the power),
// or a double field under an id of its own: the coherence (WCT with aWCT), the partial coherence
// (RP2 with its phase) or the multiple coherence (RM2, no phase)
static constexpr int FIELD_COH = -1, FIELD_COH3_P = -2, FIELD_COH3_M = -3;
static bool double_field(int field) { return field < 0; }
struct FieldRef {
  int field;
  const void *p;
  int prec, S;      // prec: the complex field's element type (the double fields are double)
  long long n0;
  size_t angle;     // coherence / partial coherence: the phase's offset from the value, in doubles
  // a double field read with its surrogate exceedance counts (count_ref): the counts, the units M
  // they hold and the row stats' cut k <= kmax; cnt null: the field alone
  const unsigned *cnt = nullptr;
  long long m = 0, kmax = 0;
  bool power = false;   // a complex field's window as its power P (CxPowerView)
  // a complex field's row stats over the points of one cluster (CxLabelView): the label image of
  // its last cluster test and the label to select; lab null: every point
  const int *lab = nullptr;
  int want = 0;
};

static int field_ref(cwtb_ctx *c, int field, FieldRef &f) {
  if (!c) return CWTB_ERR_ARG;
  if (field == CWTB_FIELD_W) {
    const ResidentSlot &s = c->wt;
    if (s.S <= 0) return fail(c, CWTB_ERR_STATE, "no transform resident");
    if (c->job.nbatch != 1) return fail(c, CWTB_ERR_UNSUPPORTED, "field of a batched transform: fetch rows per channel");
    f = FieldRef{field, c->W.p, s.prec, s.S, s.n0, 0};
  } else if (field == CWTB_FIELD_CROSS || field == CWTB_FIELD_POWER || field == FIELD_COH) {
    const bool coh = field == FIELD_COH;
    const ResidentSlot &s = coh ? c->coh : field == CWTB_FIELD_POWER ? c->pw : c->cross;
    if (s.S <= 0 || !s.buf.p)
      return fail(c, CWTB_ERR_STATE, coh ? "no coherence resident"
                                     : field == CWTB_FIELD_POWER ? "no power resident" : "no cross spectrum resident");
    f = FieldRef{field, s.buf.p, s.prec, s.S, s.n0, coh ? coh_angle_offset((size_t)s.S * s.n0) : 0};
  } else {   // FIELD_COH3_P / _M: RP2, phase, RM2 at 0, off, 2 off
    const ResidentSlot &s = c->coh3;
    if (s.S <= 0 || !s.buf.p) return fail(c, CWTB_ERR_STATE, "no partial / multiple coherence resident");
    const size_t off = coh_angle_offset((size_t)s.S * s.n0);
    const bool part = field == FIELD_COH3_P;
    f = FieldRef{field, (const double *)s.buf.p + (part ? 0 : 2 * off), s.prec, s.S, s.n0, part ? off : 0};
  }
  RT(rt_set_device(c->device));
  return 0;
}

// The counts of a tested field f (field_ref of FIELD_COH, FIELD_COH3_P, FIELD_COH3_M,
// CWTB_FIELD_POWER or CWTB_FIELD_CROSS) added to it, with the row stats' cut kmax
static int count_ref(cwtb_ctx *c, long long kmax, FieldRef &f) {
  const ResidentSlot &s = f.field == FIELD_COH          ? c->coh
                        : f.field == CWTB_FIELD_POWER   ? c->pw
                        : f.field == CWTB_FIELD_CROSS   ? c->cross : c->coh3;
  if (s.units < 0 || !s.counts.p) return fail(c, CWTB_ERR_STATE, "no surrogate counts resident for this product");
  f.cnt = (const unsigned *)s.counts.p + (f.field == FIELD_COH3_M ? coh_angle_offset((size_t)s.S * s.n0) : 0);
  f.m = s.units;
  f.kmax = kmax;
  return 0;
}

// the field of a cwtb_field_* call
static int cx_field_ref(cwtb_ctx *c, int field, FieldRef &f) {
  if (c && field != CWTB_FIELD_W && field != CWTB_FIELD_CROSS && field != CWTB_FIELD_POWER)
    return fail(c, CWTB_ERR_ARG, "unknown field");
  return field_ref(c, field, f);
}

extern "C++" {
// fn(view) with the kernel view of a resident field (kernels.cuh)
template <typename Fn>
static int with_view(const FieldRef &f, int want_phase, Fn &&fn) {
  if (f.field == FIELD_COH || f.field == FIELD_COH3_P) {
    const double *w = (const double *)f.p;
    return fn(CohView{w, w + f.angle, want_phase});
  }
  if (f.field == FIELD_COH3_M) return fn(CohMagView{(const double *)f.p, nullptr, 0});
  if (f.prec == CWTB_F64) return fn(CxView<double>{(const cx<double> *)f.p});
  return fn(CxView<float>{(const cx<float> *)f.p});
}

// fn(view) with the counting view of a field that carries counts (count_ref)
template <typename Fn>
static int with_count_view(const FieldRef &f, int want_phase, Fn &&fn) {
  if (!double_field(f.field)) {   // the power
    if (f.prec == CWTB_F64) return fn(CxCountView<double>{(const cx<double> *)f.p, f.cnt, f.kmax, f.m});
    return fn(CxCountView<float>{(const cx<float> *)f.p, f.cnt, f.kmax, f.m});
  }
  const double *w = (const double *)f.p;
  if (f.field == FIELD_COH3_M) return fn(CohCountViewT<false>{w, nullptr, f.cnt, f.kmax, f.m, 0});
  return fn(CohCountViewT<true>{w, w + f.angle, f.cnt, f.kmax, f.m, want_phase});
}

// the reads of the window and the row stats: with_view's view, or the counting view of a field
// that carries counts
template <typename Fn>
static int with_read_view(const FieldRef &f, int want_phase, Fn &&fn) {
  return f.cnt ? with_count_view(f, want_phase, fn) : with_view(f, want_phase, fn);
}

// Strided sub-grid into out0 / out1: a double field's value / phase (nothing asked for: nothing to
// do; a field without a phase takes out1 == null), a field with counts its p-values into out0, a
// complex field read as power its P into out0 (double), or a complex field as complex128 into out0
static int window_run(cwtb_ctx *c, const FieldRef &f, int row0, int nrows, int row_step, int64_t col0,
                      int64_t ncols, int64_t col_step, void *out0, void *out1) {
  const int S = f.S;
  const long long n0 = f.n0;
  const bool coh = double_field(f.field);
  if (nrows < 0 || ncols < 0 || row_step < 1 || col_step < 1)
    return fail(c, CWTB_ERR_ARG, "window: negative count or step < 1");
  if (nrows == 0 || ncols == 0 || (!out0 && !out1)) return 0;
  if (row0 < 0 || row0 >= S || (long long)(nrows - 1) > (long long)(S - 1 - row0) / row_step ||
      col0 < 0 || col0 >= n0 || (ncols - 1) > (n0 - 1 - col0) / col_step)
    return fail(c, CWTB_ERR_ARG, "window outside the resident field");
  if (!f.cnt && !f.power && row_step == 1 && col_step == 1 && col0 == 0 && ncols == n0) {   // whole rows: plain copies
    const size_t off = (size_t)row0 * n0, cnt = (size_t)nrows * n0;
    if (!coh) return field_to_host(c, f.p, f.prec, off, cnt, out0, 1);
    const double *dW = (const double *)f.p;
    if (out0) RT(rt_d2h(out0, dW + off, cnt * sizeof(double), c->stream));
    if (out1) RT(rt_d2h(out1, dW + f.angle + off, cnt * sizeof(double), c->stream));
    RT(rt_sync(c->stream));
    return 0;
  }
  const size_t m = (size_t)nrows * ncols;
  int e = ensure(c, c->aux, m * sizeof(double2));
  if (e) return e;
  double *o0 = (double *)c->aux.p, *o1 = o0 + m;   // a complex128 output takes both halves
  auto run = [&](auto v) {
    WindowArgs<decltype(v)> a{v, out0 ? o0 : nullptr, out1 ? o1 : nullptr, n0, row0, row_step, col0, col_step, ncols};
    return launch<WindowBody<decltype(v)>>(c, (unsigned)((ncols + NT - 1) / NT), (unsigned)nrows, a);
  };
  if (!f.power) e = with_read_view(f, 0, run);
  else if (f.prec == CWTB_F64) e = run(CxPowerView<double>{(const cx<double> *)f.p});
  else e = run(CxPowerView<float>{(const cx<float> *)f.p});
  if (e) return e;
  const size_t bytes = m * (coh || f.cnt || f.power ? sizeof(double) : sizeof(double2));
  if (out0) RT(rt_d2h(out0, o0, bytes, c->stream));
  if (out1) RT(rt_d2h(out1, o1, bytes, c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

// The view's K sums per row over the columns [lo_j, hi_j) (every column where lo / hi is null)
static int row_stats_run(cwtb_ctx *c, const FieldRef &f, const int64_t *lo, const int64_t *hi,
                         const double *thr, int want_phase, double *out) {
  if (!out) return fail(c, CWTB_ERR_ARG, "null argument");
  const int S = f.S;
  const long long n0 = f.n0;
  std::vector<long long> h(3 * (size_t)S);
  for (int j = 0; j < S; ++j) {
    h[j] = lo ? lo[j] : 0;
    h[S + j] = hi ? hi[j] : n0;
    if (h[j] < 0 || h[S + j] > n0 || h[j] > h[S + j])
      return fail(c, CWTB_ERR_ARG, "row_stats: column range outside [0, n0) or lo > hi");
  }
  if (thr) memcpy(h.data() + 2 * (size_t)S, thr, (size_t)S * sizeof(double));
  auto run = [&](auto v) {
    using B = RowStatsBody<decltype(v)>;
    constexpr int K = B::K;
    const int nchunk = (int)((n0 + B::CHUNK - 1) / B::CHUNK);
    // aux: [lo S][hi S][thr S][partials S*nchunk*K][sums S*K], 8 bytes each
    const size_t npart = (size_t)S * nchunk * K;
    int e = ensure(c, c->aux, (3 * (size_t)S + npart + K * (size_t)S) * sizeof(double));
    if (e) return e;
    long long *dlo = (long long *)c->aux.p, *dhi = dlo + S;
    double *dthr = (double *)(dhi + S), *dpart = dthr + S, *dsum = dpart + npart;
    RT(rt_h2d(dlo, h.data(), h.size() * sizeof(long long), c->stream));
    typename B::Args a{v, dlo, dhi, thr ? dthr : nullptr, dpart, n0, nchunk};
    if ((e = launch<B>(c, (unsigned)nchunk, (unsigned)S, a))) return e;
    RowSumArgs r{dpart, dsum, S, nchunk};
    if ((e = launch<RowSumBody<K>>(c, (unsigned)((K * S + NT - 1) / NT), 1, r))) return e;
    RT(rt_d2h(out, dsum, (size_t)S * K * sizeof(double), c->stream));
    RT(rt_sync(c->stream));
    return 0;
  };
  if (!f.lab) return with_read_view(f, want_phase, run);
  if (f.prec == CWTB_F64) return run(CxLabelView<double>{(const cx<double> *)f.p, f.lab, f.want});
  return run(CxLabelView<float>{(const cx<float> *)f.p, f.lab, f.want});
}

// The view's NA weighted sums per column over the rows with a non-zero weight
static int scale_avg_run(cwtb_ctx *c, const FieldRef &f, const double *weights, void *out) {
  if (!weights || !out) return fail(c, CWTB_ERR_ARG, "null argument");
  const int S = f.S;
  const long long n0 = f.n0;
  // aux: [weights S doubles][selected rows S ints][out NA*n0 doubles, 16-byte aligned]: rows with
  // a zero weight are not read
  std::vector<double> w(weights, weights + S);
  std::vector<int> sel;
  for (int j = 0; j < S; ++j)
    if (w[j] != 0.0) sel.push_back(j);
  const int nsel = (int)sel.size();
  const size_t head = ((size_t)S + ((size_t)S + 1) / 2 + 1) & ~(size_t)1;
  w.resize(head);
  if (nsel) memcpy(w.data() + S, sel.data(), sizeof(int) * nsel);
  return with_view(f, 0, [&](auto v) {
    using B = SelScaleAvgBody<decltype(v)>;
    const size_t nout = decltype(v)::NA * (size_t)n0;
    int e = ensure(c, c->aux, (head + nout) * sizeof(double));
    if (e) return e;
    double *dw = (double *)c->aux.p, *dout = dw + head;
    RT(rt_h2d(dw, w.data(), head * sizeof(double), c->stream));
    typename B::Args a{v, dw, (const int *)(dw + S), nsel, dout, n0};
    if ((e = launch<B>(c, (unsigned)((n0 + NT - 1) / NT), 1, a))) return e;
    RT(rt_d2h(out, dout, nout * sizeof(double), c->stream));
    RT(rt_sync(c->stream));
    return 0;
  });
}

// The reconstruction's sum out[n] = sum_j weights[j] Re F[j, n] of a complex field (cwtb_*_reconstruct)
// over the columns [lo_j, hi_j), where thr is null or P > thr[j], and, for a field with counts
// (count_ref), where P is finite and k <= kmax, or, with `mark` (n_mark bytes over the labels of
// f.lab), where mark[label] != 0.  Rows with a zero weight or an empty range are not read; a
// column without a selected point is 0.
static int reconstruct_run(cwtb_ctx *c, const FieldRef &f, const double *weights, const int64_t *lo,
                           const int64_t *hi, const double *thr, const unsigned char *mark, size_t n_mark,
                           double *out) {
  if (!weights || !lo || !hi || !out) return fail(c, CWTB_ERR_ARG, "null argument");
  const int S = f.S;
  const long long n0 = f.n0;
  std::vector<int> sel;
  for (int j = 0; j < S; ++j) {
    if (lo[j] < 0 || hi[j] > n0 || lo[j] > hi[j])
      return fail(c, CWTB_ERR_ARG, "reconstruct: column range outside [0, n0) or lo > hi");
    if (weights[j] != 0.0 && lo[j] < hi[j]) sel.push_back(j);
  }
  const int nsel = (int)sel.size();
  // aux, 8-byte words: [weights S][lo S][hi S][thr S][selected rows, S ints][mark bytes][out n0]
  const size_t wsel = ((size_t)S + 1) / 2, wmark = (n_mark + 7) / 8;
  const size_t head = 4 * (size_t)S + wsel + wmark;
  std::vector<double> h(head, 0.0);
  memcpy(h.data(), weights, (size_t)S * sizeof(double));
  memcpy(h.data() + S, lo, (size_t)S * sizeof(int64_t));
  memcpy(h.data() + 2 * (size_t)S, hi, (size_t)S * sizeof(int64_t));
  if (thr) memcpy(h.data() + 3 * (size_t)S, thr, (size_t)S * sizeof(double));
  if (nsel) memcpy(h.data() + 4 * (size_t)S, sel.data(), (size_t)nsel * sizeof(int));
  if (n_mark) memcpy(h.data() + 4 * (size_t)S + wsel, mark, n_mark);
  int e = ensure(c, c->aux, (head + (size_t)n0) * sizeof(double));
  if (e) return e;
  double *dh = (double *)c->aux.p, *dout = dh + head;
  RT(rt_h2d(dh, h.data(), head * sizeof(double), c->stream));
  const long long *dlo = (const long long *)(dh + S), *dhi = dlo + S;
  const int *dsel = (const int *)(dh + 4 * (size_t)S);
  const unsigned char *dmark = (const unsigned char *)(dh + 4 * (size_t)S + wsel);
  auto run = [&](auto v) {
    using B = SelScaleAvgBody<decltype(v)>;
    typename B::Args a{v, dh, dsel, nsel, dout, n0, dlo, dhi, thr ? dh + 3 * (size_t)S : nullptr};
    int e2 = launch<B>(c, (unsigned)((n0 + NT - 1) / NT), 1, a);
    if (e2) return e2;
    RT(rt_d2h(out, dout, (size_t)n0 * sizeof(double), c->stream));
    RT(rt_sync(c->stream));
    return 0;
  };
  if (f.prec == CWTB_F64) {
    const cx<double> *F = (const cx<double> *)f.p;
    if (mark) return run(CxReView<double, RE_LABEL>{F, nullptr, 0, f.lab, dmark});
    if (f.cnt) return run(CxReView<double, RE_COUNT>{F, f.cnt, f.kmax});
    return run(CxReView<double, RE_ALL>{F});
  }
  const cx<float> *F = (const cx<float> *)f.p;
  if (mark) return run(CxReView<float, RE_LABEL>{F, nullptr, 0, f.lab, dmark});
  if (f.cnt) return run(CxReView<float, RE_COUNT>{F, f.cnt, f.kmax});
  return run(CxReView<float, RE_ALL>{F});
}

// Histogram [M + 1] of the counts of a field with counts over the columns [lo_j, hi_j) of every
// row, of the points whose value is finite
static int count_hist_run(cwtb_ctx *c, const FieldRef &f, const int64_t *lo, const int64_t *hi, int64_t nbins,
                          int64_t *out) {
  if (!lo || !hi || !out) return fail(c, CWTB_ERR_ARG, "null argument");
  if (nbins != f.m + 1) return fail(c, CWTB_ERR_ARG, "count_hist: the histogram has M + 1 bins (M: the units counted)");
  const int S = f.S;
  const long long n0 = f.n0;
  std::vector<long long> h(2 * (size_t)S);
  long long span = 0;
  for (int j = 0; j < S; ++j) {
    h[j] = lo[j];
    h[S + j] = hi[j];
    if (lo[j] < 0 || hi[j] > n0 || lo[j] > hi[j])
      return fail(c, CWTB_ERR_ARG, "count_hist: column range outside [0, n0) or lo > hi");
    span = std::max(span, (long long)(hi[j] - lo[j]));
  }
  // aux: [lo S][hi S][hist nbins], 8 bytes each
  int e = ensure(c, c->aux, (2 * (size_t)S + (size_t)nbins) * sizeof(long long));
  if (e) return e;
  long long *dlo = (long long *)c->aux.p, *dhi = dlo + S;
  unsigned long long *dh = (unsigned long long *)(dhi + S);
  RT(rt_h2d(dlo, h.data(), h.size() * sizeof(long long), c->stream));
  RT(rt_memset(dh, 0, (size_t)nbins * sizeof(long long), c->stream));
  e = with_count_view(f, 0, [&](auto v) {
    CountHistArgs<decltype(v)> a{v, dlo, dhi, dh, n0, nbins};
    using Sh = CountHistBody<decltype(v), true>;
    const unsigned gx = (unsigned)((span + Sh::CHUNK - 1) / Sh::CHUNK);
    return nbins <= Sh::SMEM_BINS ? launch<Sh>(c, gx, (unsigned)S, a)
                                  : launch<CountHistBody<decltype(v), false>>(c, gx, (unsigned)S, a);
  });
  if (e) return e;
  RT(rt_d2h(out, dh, (size_t)nbins * sizeof(long long), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}
}  // extern "C++"

int cwtb_field_get(cwtb_ctx *c, int field, int row0, int nrows, void *out) {
  FieldRef f;
  int e = cx_field_ref(c, field, f);
  if (e) return e;
  if (!out) return fail(c, CWTB_ERR_ARG, "null argument");
  if (row0 < 0 || nrows < 0 || row0 > f.S - nrows) return fail(c, CWTB_ERR_ARG, "row range");
  return field_to_host(c, f.p, f.prec, (size_t)row0 * f.n0, (size_t)nrows * f.n0, out, 1);
}

int cwtb_field_window(cwtb_ctx *c, int field, int row0, int nrows, int row_step, int64_t col0,
                      int64_t ncols, int64_t col_step, void *out) {
  FieldRef f;
  int e = cx_field_ref(c, field, f);
  if (e) return e;
  if (!out && nrows > 0 && ncols > 0) return fail(c, CWTB_ERR_ARG, "null argument");
  return window_run(c, f, row0, nrows, row_step, col0, ncols, col_step, out, nullptr);
}

int cwtb_field_row_stats(cwtb_ctx *c, int field, const int64_t *lo, const int64_t *hi, const double *thr,
                         double *out) {
  FieldRef f;
  int e = cx_field_ref(c, field, f);
  return e ? e : row_stats_run(c, f, lo, hi, thr, 0, out);
}

int cwtb_field_reconstruct(cwtb_ctx *c, int field, const double *weights, const int64_t *lo, const int64_t *hi,
                           const double *thr, double *out) {
  if (c && field == CWTB_FIELD_CROSS)
    return fail(c, CWTB_ERR_ARG, "reconstruct: the cross spectrum has no inverse transform");
  FieldRef f;
  int e = cx_field_ref(c, field, f);
  return e ? e : reconstruct_run(c, f, weights, lo, hi, thr, nullptr, 0, out);
}

int cwtb_cross_scale_avg(cwtb_ctx *c, const double *weights, void *out) {
  FieldRef f;
  int e = field_ref(c, CWTB_FIELD_CROSS, f);
  return e ? e : scale_avg_run(c, f, weights, out);
}

// Coherence of two series in the engine type T into the device buffer `dst` (WCT, then aWCT at
// coh_angle_offset), grown as needed.  `angle_host`: host destination of an early angle copy (see
// wct_core), or null.
extern "C++" {
template <typename T>
static int wct_run(cwtb_ctx *c, const double *y1, const double *y2, int64_t n0, double dt,
                   const double *scales, int n_scales, int family, double param, int boxcar_len,
                   Buf &dst, bool want_angle, double *angle_host) {
  int e = prepare(c, n0, dt, scales, n_scales, family, param, prec_of<T>(), nullptr);
  if (e) return e;
  if ((e = upload_series<T>(c, c->sig, y1, n0))) return e;
  if ((e = upload_series<T>(c, c->sig2, y2, n0))) return e;
  if ((e = upload_window(c, boxcar_len))) return e;
  if ((e = upload_row_tables(c, c->job))) return e;
  const size_t cnt = (size_t)n_scales * n0;
  if ((e = ensure(c, dst, (coh_angle_offset(cnt) + cnt) * sizeof(double)))) return e;
  double *dW = (double *)dst.p, *dA = dW + coh_angle_offset(cnt);
  c->launches = 0;
  if ((e = time_begin(c))) return e;
  c->angle_host = angle_host;
  e = wct_core<T>(c, c->job, (const T *)c->sig.p, (const T *)c->sig2.p, boxcar_len, dW,
                  want_angle ? dA : nullptr, nullptr, 0, 0, nullptr);
  c->angle_host = nullptr;
  if (e) return e;
  if ((e = time_end(c, &c->last_ms))) return e;
  c->job_dsig = nullptr;
  return 0;
}
}  // extern "C++"

static int wct_dispatch(cwtb_ctx *c, const double *y1, const double *y2, int64_t n0, double dt,
                        const double *scales, int n_scales, int family, double param, int boxcar_len,
                        Buf &dst, bool want_angle, double *angle_host) {
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, "wct needs an analytic wavelet family");
  return c->coh_precision == CWTB_F32
             ? wct_run<float>(c, y1, y2, n0, dt, scales, n_scales, family, param, boxcar_len, dst, want_angle, angle_host)
             : wct_run<double>(c, y1, y2, n0, dt, scales, n_scales, family, param, boxcar_len, dst, want_angle, angle_host);
}

int cwtb_wct(cwtb_ctx *c, const double *y1, const double *y2, int64_t n0, double dt, double dj,
             const double *scales, int n_scales, int family, double param, int boxcar_len,
             double *WCT_out, double *aWCT_out) {
  (void)dj;
  if (!c || !y1 || !y2) return fail(c, CWTB_ERR_ARG, "null argument");
  int e = wct_dispatch(c, y1, y2, n0, dt, scales, n_scales, family, param, boxcar_len, c->aux,
                       aWCT_out != nullptr, aWCT_out);
  if (e) return e;
  const size_t cnt = (size_t)n_scales * n0;
  const double *dW = (const double *)c->aux.p;
  if (WCT_out) RT(rt_d2h(WCT_out, dW, cnt * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  if (aWCT_out) RT(rt_sync(c->copy_streams[0]));
  return 0;
}

// ---- partial and multiple coherence of three series ------------------------------------------
extern "C++" {
template <typename T>
static int wct3_run(cwtb_ctx *c, const double *y, const double *x1, const double *x2, int64_t n0, double dt,
                    const double *scales, int n_scales, int family, double param, int boxcar_len,
                    double *dRP2, double *dRM2, double *dPP = nullptr) {
  int e = prepare(c, n0, dt, scales, n_scales, family, param, prec_of<T>(), nullptr);
  if (e) return e;
  if ((e = upload_series<T>(c, c->sig, y, n0))) return e;
  if ((e = upload_series<T>(c, c->sig2, x1, n0))) return e;
  if ((e = upload_series<T>(c, c->sig3, x2, n0))) return e;
  if ((e = upload_window(c, boxcar_len))) return e;
  if ((e = upload_row_tables(c, c->job))) return e;
  c->launches = 0;
  if ((e = time_begin(c))) return e;
  e = wct3_core<T>(c, c->job, (const T *)c->sig.p, (const T *)c->sig2.p, (const T *)c->sig3.p,
                   boxcar_len, dRP2, dRM2, nullptr, 0, 0, nullptr, nullptr, dPP);
  if (e) return e;
  if ((e = time_end(c, &c->last_ms))) return e;
  c->job_dsig = nullptr;
  return 0;
}
}  // extern "C++"

int cwtb_wct3(cwtb_ctx *c, const double *y, const double *x1, const double *x2, int64_t n0, double dt,
              double dj, const double *scales, int n_scales, int family, double param, int boxcar_len,
              double *RP2_out, double *RM2_out) {
  (void)dj;
  if (!c || !y || !x1 || !x2) return fail(c, CWTB_ERR_ARG, "null argument");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, "wct3 needs an analytic wavelet family");
  if (n0 < 1 || n_scales < 1) return fail(c, CWTB_ERR_ARG, "bad n0 / n_scales");
  const size_t cnt = (size_t)n_scales * n0;
  // outputs in aux: RP2, then RM2
  int e = ensure(c, c->aux, 2 * cnt * sizeof(double));
  if (e) return e;
  double *dRP2 = RP2_out ? (double *)c->aux.p : nullptr, *dRM2 = RM2_out ? (double *)c->aux.p + cnt : nullptr;
  e = c->coh_precision == CWTB_F32
          ? wct3_run<float>(c, y, x1, x2, n0, dt, scales, n_scales, family, param, boxcar_len, dRP2, dRM2)
          : wct3_run<double>(c, y, x1, x2, n0, dt, scales, n_scales, family, param, boxcar_len, dRP2, dRM2);
  if (e) return e;
  if (RP2_out) RT(rt_d2h(RP2_out, dRP2, cnt * sizeof(double), c->stream));
  if (RM2_out) RT(rt_d2h(RM2_out, dRM2, cnt * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

// ---- resident coherence ---------------------------------------------------------------------
int cwtb_wct_resident(cwtb_ctx *c, const double *y1, const double *y2, int64_t n0, double dt, double dj,
                      const double *scales, int n_scales, int family, double param, int boxcar_len) {
  (void)dj;
  if (!c || !y1 || !y2) return fail(c, CWTB_ERR_ARG, "null argument");
  slot_begin(c->coh);
  int e = wct_dispatch(c, y1, y2, n0, dt, scales, n_scales, family, param, boxcar_len, c->coh.buf, true, nullptr);
  if (e) return e;
  RT(rt_sync(c->stream));
  c->coh.S = n_scales;
  c->coh.n0 = n0;
  c->coh.prec = CWTB_F64;
  return 0;
}

int64_t cwtb_coherence_serial(cwtb_ctx *c) { return c ? c->coh.serial : -1; }
int cwtb_coherence_release(cwtb_ctx *c) { return c ? slot_release(c, c->coh) : CWTB_ERR_ARG; }

int cwtb_coherence_window(cwtb_ctx *c, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                          int64_t col_step, double *WCT_out, double *aWCT_out) {
  FieldRef f;
  int e = field_ref(c, FIELD_COH, f);
  return e ? e : window_run(c, f, row0, nrows, row_step, col0, ncols, col_step, WCT_out, aWCT_out);
}

int cwtb_coherence_row_stats(cwtb_ctx *c, const int64_t *lo, const int64_t *hi, const double *thr,
                             int want_phase, double *out) {
  FieldRef f;
  int e = field_ref(c, FIELD_COH, f);
  return e ? e : row_stats_run(c, f, lo, hi, thr, want_phase != 0, out);
}

int cwtb_coherence_scale_avg(cwtb_ctx *c, const double *weights, double *out) {
  FieldRef f;
  int e = field_ref(c, FIELD_COH, f);
  return e ? e : scale_avg_run(c, f, weights, out);
}

// ---- resident partial and multiple coherence ---------------------------------------------------
int cwtb_wct3_resident(cwtb_ctx *c, const double *y, const double *x1, const double *x2, int64_t n0, double dt,
                       double dj, const double *scales, int n_scales, int family, double param, int boxcar_len) {
  (void)dj;
  if (!c || !y || !x1 || !x2) return fail(c, CWTB_ERR_ARG, "null argument");
  slot_begin(c->coh3);
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, "wct3 needs an analytic wavelet family");
  if (n0 < 1 || n_scales < 1) return fail(c, CWTB_ERR_ARG, "bad n0 / n_scales");
  const size_t cnt = (size_t)n_scales * n0, off = coh_angle_offset(cnt);
  RT(rt_set_device(c->device));
  int e = ensure(c, c->coh3.buf, (2 * off + cnt) * sizeof(double));
  if (e) return e;
  double *d = (double *)c->coh3.buf.p;
  e = c->coh_precision == CWTB_F32
          ? wct3_run<float>(c, y, x1, x2, n0, dt, scales, n_scales, family, param, boxcar_len, d, d + 2 * off, d + off)
          : wct3_run<double>(c, y, x1, x2, n0, dt, scales, n_scales, family, param, boxcar_len, d, d + 2 * off, d + off);
  if (e) return e;
  RT(rt_sync(c->stream));
  c->coh3.S = n_scales;
  c->coh3.n0 = n0;
  c->coh3.prec = CWTB_F64;
  return 0;
}

int64_t cwtb_coherence3_serial(cwtb_ctx *c) { return c ? c->coh3.serial : -1; }
int cwtb_coherence3_release(cwtb_ctx *c) { return c ? slot_release(c, c->coh3) : CWTB_ERR_ARG; }

// the field of a cwtb_coherence3_* call; the multiple coherence has no phase
static int coh3_ref(cwtb_ctx *c, int measure, bool want_phase, FieldRef &f) {
  if (!c) return CWTB_ERR_ARG;
  if (measure != CWTB_MEASURE_PARTIAL && measure != CWTB_MEASURE_MULTIPLE)
    return fail(c, CWTB_ERR_ARG, "unknown measure");
  if (want_phase && measure == CWTB_MEASURE_MULTIPLE)
    return fail(c, CWTB_ERR_ARG, "the multiple coherence has no phase");
  return field_ref(c, measure == CWTB_MEASURE_PARTIAL ? FIELD_COH3_P : FIELD_COH3_M, f);
}

int cwtb_coherence3_window(cwtb_ctx *c, int measure, int row0, int nrows, int row_step, int64_t col0,
                           int64_t ncols, int64_t col_step, double *R_out, double *phase_out) {
  FieldRef f;
  int e = coh3_ref(c, measure, phase_out != nullptr, f);
  return e ? e : window_run(c, f, row0, nrows, row_step, col0, ncols, col_step, R_out, phase_out);
}

int cwtb_coherence3_row_stats(cwtb_ctx *c, int measure, const int64_t *lo, const int64_t *hi, const double *thr,
                              int want_phase, double *out) {
  FieldRef f;
  int e = coh3_ref(c, measure, want_phase != 0, f);
  return e ? e : row_stats_run(c, f, lo, hi, thr, want_phase != 0, out);
}

int cwtb_coherence3_scale_avg(cwtb_ctx *c, int measure, const double *weights, double *out) {
  FieldRef f;
  int e = coh3_ref(c, measure, false, f);
  return e ? e : scale_avg_run(c, f, weights, out);
}

// ---- point-wise tests against surrogates: reading the counts ----------------------------------
int cwtb_coherence_pvalue_window(cwtb_ctx *c, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                                 int64_t col_step, double *p_out) {
  FieldRef f;
  int e = field_ref(c, FIELD_COH, f);
  if (e || (e = count_ref(c, 0, f))) return e;
  if (!p_out && nrows > 0 && ncols > 0) return fail(c, CWTB_ERR_ARG, "null argument");
  return window_run(c, f, row0, nrows, row_step, col0, ncols, col_step, p_out, nullptr);
}

int cwtb_coherence_pvalue_row_stats(cwtb_ctx *c, const int64_t *lo, const int64_t *hi, const double *thr,
                                    int64_t kmax, int want_phase, double *out) {
  FieldRef f;
  int e = field_ref(c, FIELD_COH, f);
  if (e || (e = count_ref(c, kmax, f))) return e;
  return row_stats_run(c, f, lo, hi, thr, want_phase != 0, out);
}

int cwtb_coherence_count_hist(cwtb_ctx *c, const int64_t *lo, const int64_t *hi, int64_t nbins, int64_t *out) {
  FieldRef f;
  int e = field_ref(c, FIELD_COH, f);
  if (e || (e = count_ref(c, 0, f))) return e;
  return count_hist_run(c, f, lo, hi, nbins, out);
}

int cwtb_coherence3_pvalue_window(cwtb_ctx *c, int measure, int row0, int nrows, int row_step, int64_t col0,
                                  int64_t ncols, int64_t col_step, double *p_out) {
  FieldRef f;
  int e = coh3_ref(c, measure, false, f);
  if (e || (e = count_ref(c, 0, f))) return e;
  if (!p_out && nrows > 0 && ncols > 0) return fail(c, CWTB_ERR_ARG, "null argument");
  return window_run(c, f, row0, nrows, row_step, col0, ncols, col_step, p_out, nullptr);
}

int cwtb_coherence3_pvalue_row_stats(cwtb_ctx *c, int measure, const int64_t *lo, const int64_t *hi,
                                     const double *thr, int64_t kmax, int want_phase, double *out) {
  FieldRef f;
  int e = coh3_ref(c, measure, want_phase != 0, f);
  if (e || (e = count_ref(c, kmax, f))) return e;
  return row_stats_run(c, f, lo, hi, thr, want_phase != 0, out);
}

int cwtb_coherence3_count_hist(cwtb_ctx *c, int measure, const int64_t *lo, const int64_t *hi, int64_t nbins,
                               int64_t *out) {
  FieldRef f;
  int e = coh3_ref(c, measure, false, f);
  if (e || (e = count_ref(c, 0, f))) return e;
  return count_hist_run(c, f, lo, hi, nbins, out);
}

int cwtb_resident_shape(cwtb_ctx *c, int product, int *rows, int64_t *n0, int *precision) {
  if (!c) return CWTB_ERR_ARG;
  const ResidentSlot *s = product == CWTB_PRODUCT_W           ? &c->wt
                        : product == CWTB_PRODUCT_CROSS       ? &c->cross
                        : product == CWTB_PRODUCT_COHERENCE   ? &c->coh
                        : product == CWTB_PRODUCT_COHERENCE3  ? &c->coh3
                        : product == CWTB_PRODUCT_POWER       ? &c->pw : nullptr;
  if (!s) return fail(c, CWTB_ERR_ARG, "unknown product");
  const bool on = s->S > 0;
  if (rows) *rows = on ? s->S : 0;
  if (n0) *n0 = on ? s->n0 : 0;
  if (precision) *precision = on ? s->prec : CWTB_F64;
  return 0;
}

int cwtb_set_coherence_precision(cwtb_ctx *c, int precision) {
  if (!c) return CWTB_ERR_ARG;
  if (precision != CWTB_F64 && precision != CWTB_F32) return fail(c, CWTB_ERR_ARG, "bad precision");
  c->coh_precision = precision;
  return 0;
}

int cwtb_set_morse_ga(cwtb_ctx *c, double ga) {
  if (!c) return CWTB_ERR_ARG;
  if (!(ga >= 1 && ga <= 12)) return fail(c, CWTB_ERR_ARG, "Morse ga must be in [1, 12]");
  c->morse_ga = ga;
  return 0;
}

int cwtb_set_smooth_filter(cwtb_ctx *c, const double *table, int n_rows, int64_t n) {
  if (!c) return CWTB_ERR_ARG;
  if (!table || n_rows <= 0 || n <= 0) {   // back to Morlet's Gaussian (mothers.py:83-91)
    c->filt_rows = 0;
    c->filt_n = 0;
    return 0;
  }
  RT(rt_set_device(c->device));
  const size_t bytes = (size_t)n_rows * (size_t)n * sizeof(double);
  int e = ensure(c, c->filt, bytes);
  if (e) return e;
  RT(rt_h2d(c->filt.p, table, bytes, c->stream));
  RT(rt_sync(c->stream));
  c->filt_rows = n_rows;
  c->filt_n = n;
  return 0;
}

int cwtb_set_padding(cwtb_ctx *c, int pad_to_pow2) {
  if (!c) return CWTB_ERR_ARG;
  c->pad_pow2 = pad_to_pow2 != 0;
  return 0;
}

int cwtb_smooth(cwtb_ctx *c, const void *in, int is_complex, int n_scales, int64_t n, double dt,
                const double *scales, int boxcar_len, void *out) {
  if (!c || !in || !out || !scales || n_scales < 1 || n < 1 || !(dt > 0))
    return fail(c, CWTB_ERR_ARG, "smooth: bad argument");
  if (n > (1ll << 26)) return fail(c, CWTB_ERR_UNSUPPORTED, "smooth: rows longer than 2^26");
  if (n_scales > (int)MAX_ROWS) return fail(c, CWTB_ERR_ARG, "smooth: more than 65535 scales in one call");
  RT(rt_set_device(c->device));
  const int S = n_scales;
  const size_t cnt = (size_t)S * n;
  if (!c->pad_pow2 && n > (1ll << 24)) return fail(c, CWTB_ERR_UNSUPPORTED, "smooth: un-padded rows longer than 2^24");
  const unsigned N = c->pad_pow2 ? 1u << ilog2((unsigned long long)n) : (unsigned)n;   // helpers.py:15-30
  int e = upload_window(c, boxcar_len);
  if (e) return e;
  std::vector<double> g(2 * (size_t)S);
  for (int j = 0; j < S; ++j) { g[j] = scales[j]; double sn = scales[j] / dt; g[S + j] = -0.5 * (sn * sn); }
  if ((e = upload_doubles(c, c->rowd, g))) return e;
  if ((e = ensure(c, c->C, cnt * sizeof(double2)))) return e;
  if ((e = ensure(c, c->A12, cnt * sizeof(double2)))) return e;
  double2 *X = (double2 *)c->C.p, *Y = (double2 *)c->A12.p;
  if (is_complex) {
    RT(rt_h2d(X, in, cnt * sizeof(double2), c->stream));
  } else {
    RT(rt_h2d(Y, in, cnt * sizeof(double), c->stream));   // stage the reals in Y, widen into X
    R2CArgs ra{(const double *)Y, X, (long long)cnt};
    if ((e = launch<R2CBody>(c, (unsigned)((cnt + NT - 1) / NT), 1, ra))) return e;
  }
  if ((e = smooth_time<double>(c, X, S, n, N, (const double *)c->rowd.p + S))) return e;
  BoxcarArgs<double> ba{X, Y, (const double *)c->win.p, n, S, boxcar_len};
  if ((e = launch<BoxcarBody<double>>(c, (unsigned)((n + NT - 1) / NT), S, ba))) return e;
  if (is_complex) {
    RT(rt_d2h(out, Y, cnt * sizeof(double2), c->stream));
    RT(rt_sync(c->stream));
  } else {
    std::vector<double2> tmp(cnt);
    RT(rt_d2h(tmp.data(), Y, cnt * sizeof(double2), c->stream));
    RT(rt_sync(c->stream));
    double *o = (double *)out;
    for (size_t i = 0; i < cnt; ++i) o[i] = tmp[i].x;   // .real, mothers.py:95-96
  }
  return 0;
}

// ---- cluster labelling ---------------------------------------------------------------------------
extern "C++" {
// Labels the selection bitmask c->cl_bits [S][ceil(n0 / 32)] with the per-row weights dq (device,
// [S]) through ClusterCountBody .. ClusterMaxBody: the largest cluster sum goes to *dqmax (device,
// zeroed by the caller).  With `tab`, also the table of every cluster and the label image dlabels
// [S][n0].  The run count is read back to size the run tables: one synchronisation per map.
static int label_bits(cwtb_ctx *c, int S, long long n0, const unsigned long long *dq, unsigned long long *dqmax,
                      ClusterTable *tab, int *dlabels) {
  using CB = ClusterCountBody;
  ClusterArgs a{};
  a.bits = (const unsigned *)c->cl_bits.p;
  a.n = n0;
  a.words = (n0 + 31) / 32;
  a.rows = S;
  a.cpr = (int)((a.words + CB::CHW - 1) / CB::CHW);
  a.q = dq;
  a.qmax = dqmax;
  const size_t nch = (size_t)S * a.cpr;
  int e = ensure(c, c->cl_hdr, (2 * nch + S + 3) * sizeof(unsigned));
  if (e) return e;
  a.chunk = (unsigned *)c->cl_hdr.p;
  a.chunk_end = a.chunk + nch;
  a.rowbeg = a.chunk_end + nch;
  a.total = a.rowbeg + S + 1;
  if ((e = launch<CB>(c, (unsigned)a.cpr, (unsigned)S, a))) return e;
  if ((e = launch<ClusterScanBody>(c, 1, 1, a))) return e;
  unsigned tot[2];
  RT(rt_d2h(tot, a.total, sizeof tot, c->stream));
  RT(rt_sync(c->stream));
  if (tot[0] != tot[1]) return fail(c, CWTB_ERR_STATE, "cluster labelling: the runs' starts and ends differ");
  const size_t R = tot[0];
  a.runs = tot[0];
  // 8-byte sums first: qsum [R] (and pts [R]); then start, end, parent [R] (and rmax, cmin, cmax,
  // cid [R]) of 4 bytes
  // grown with half again as much room, so that the units of a Monte-Carlo run, whose run counts
  // scatter around one value, rarely free and allocate inside the loop
  const size_t per = tab ? 2 * 8 + 7 * 4 : 8 + 3 * 4, need = std::max<size_t>(R, 1) * per;
  if (c->cl_runs.bytes < need && (e = ensure(c, c->cl_runs, need + need / 2))) return e;
  unsigned long long *q64 = (unsigned long long *)c->cl_runs.p;
  unsigned *u32 = (unsigned *)(q64 + (tab ? 2 : 1) * R);
  a.qsum = q64;
  a.start = u32;
  a.end = u32 + R;
  a.parent = u32 + 2 * R;
  if (tab) a.st = ClusterStats{q64 + R, u32 + 3 * R, u32 + 4 * R, u32 + 5 * R};
  const unsigned gr = (unsigned)((R + NT - 1) / NT);
  if ((e = launch<ClusterExtractBody>(c, (unsigned)a.cpr, (unsigned)S, a))) return e;
  if ((e = launch<ClusterUnionBody>(c, gr, 1, a))) return e;
  if ((e = launch<ClusterSumBody>(c, gr, 1, a))) return e;
  if ((e = launch<ClusterMaxBody>(c, gr, 1, a))) return e;
  if (!tab) return 0;
  // the table: the roots (parent[k] == k) in table order
  std::vector<unsigned long long> hq(R), hpts(R);
  std::vector<unsigned> hu(6 * R);
  if (R) {
    RT(rt_d2h(hq.data(), a.qsum, R * 8, c->stream));
    RT(rt_d2h(hpts.data(), a.st.pts, R * 8, c->stream));
    RT(rt_d2h(hu.data(), u32, 6 * R * 4, c->stream));
    RT(rt_sync(c->stream));
  }
  const unsigned *hs = hu.data(), *hp = hs + 2 * R, *hrm = hs + 3 * R, *hc0 = hs + 4 * R, *hc1 = hs + 5 * R;
  std::vector<unsigned> roots;
  for (size_t k = 0; k < R; ++k)
    if (hp[k] == (unsigned)k) roots.push_back((unsigned)k);
  std::sort(roots.begin(), roots.end(), [&](unsigned x, unsigned y) {
    return hq[x] != hq[y] ? hq[x] > hq[y] : hs[x] < hs[y];
  });
  ClusterTable t;
  std::vector<int> cid(std::max<size_t>(R, 1), 0);
  for (size_t i = 0; i < roots.size(); ++i) {
    const unsigned r = roots[i];
    cid[r] = (int)i + 1;
    t.Q.push_back(hq[r]);
    t.pts.push_back(hpts[r]);
    for (long long v : {(long long)(hs[r] / (unsigned long long)n0), (long long)hrm[r] + 1, (long long)hc0[r], (long long)hc1[r]})
      t.box.push_back(v);
  }
  int *dcid = (int *)(u32 + 6 * R);
  if (R) RT(rt_h2d(dcid, cid.data(), R * sizeof(int), c->stream));
  ClusterPaintArgs pa{a, dcid, dlabels};
  if ((e = launch<ClusterPaintBody>(c, (unsigned)((n0 + NT - 1) / NT), (unsigned)S, pa))) return e;
  RT(rt_sync(c->stream));
  *tab = std::move(t);
  return 0;
}
}  // extern "C++"

// common part of the Monte-Carlo entry points, for surrogate units of nser = 2 series (coherence,
// one histogram) or 3 (partial and multiple coherence, hist[0] and hist[1], either may be null):
// `noise` host surrogates [n_units][nser][n0]; or a null `tn` drawn on the device from (seed,
// unit0 + i) (test_null: phase-randomised surrogates of the data whose spectra are in c->pspec, or
// AR(1) series with held rows); or neither -> white noise drawn on the device from (seed,
// unit0 + i); coherence in the engine type T
struct PhaseSrc { int group[3]; };
struct Ar1Src { double g, m, sigma; };
// The null of a test of nser series: AR(1) units, series s with its own parameters ar[s] under the
// series tag s, or phase-randomised units of the series (their spectra in c->pspec, series s in
// phase group ph.group[s]).  An AR(1) series with held[s] is not drawn: every unit has the data's
// row s of `series` there (host doubles, read once per call; the coherence tests only).
struct TestNull {
  int kind, nser;
  Ar1Src ar[3];
  PhaseSrc ph;
  int held[3];
  const double *series;
};

extern "C++" {
template <typename T>
static int ar1_units(cwtb_ctx *c, const Ar1Src &ar, unsigned long long seed, long long unit0, int nb, int64_t n0,
                     T *out, int nser, unsigned stag);
}  // extern "C++"
// the exceedance counters of a counting run (cwtb_coherence*_surrogate_counts) and the observed
// fields they compare against, per measure: the coherence in [0]; the partial and the multiple
// coherence in [0] and [1] (either counter may be null)
// A cluster test (cwtb_coherence*_cluster_test) adds the selection bits of every unit's map (sel),
// labelled after the unit's final launch with the per-row weights q; the unit's largest cluster sum
// goes to qmax[unit - unit0].
struct CountDst {
  const double *obs[2];
  unsigned *cnt[2];
  SelArgs sel;
  const unsigned long long *q;
  unsigned long long *qmax;
};

extern "C++" {
// nb surrogate units of the data spectra c->pspec [nser][n0] into out [nb][nser][n0]: rotation,
// inverse transform at length n0 (in place: every row transform reads its chunk of rows into a
// work buffer before it stores them) and real part.  c->prot holds nb * nser * n0 double2.
template <typename T>
static int phase_units(cwtb_ctx *c, const PhaseSrc &ph, int nser, unsigned long long seed, long long unit0, int nb,
                       int64_t n0, T *out) {
  const int rows = nser * nb;
  double2 *R = (double2 *)c->prot.p;
  struct Tag { cwtb_ctx *c; ~Tag() { c->prof_tag = ""; } } tag{c};
  c->prof_tag = "phase:";                 // profiles tell the generator's row transforms from the pipeline's
  PhaseRotArgs ra{(const double2 *)c->pspec.p, R, seed, unit0, (long long)n0, nser, {ph.group[0], ph.group[1], ph.group[2]}};
  int e = launch<PhaseRotBody>(c, (unsigned)((n0 / 2 + 1 + NT - 1) / NT), (unsigned)rows, ra);
  if (e) return e;
  e = (n0 & (n0 - 1)) ? blue_rows(c, R, 0, n0, R, n0, (unsigned)n0, rows, +1, 1.0, n0)
                      : fft_rows<double, +1>(c, R, 0, n0, n0, R, n0, (unsigned)n0, rows);
  if (e) return e;
  const long long cnt = (long long)rows * n0;
  RealPartArgs<T> pa{R, out, cnt, 1.0 / (double)n0};
  return launch<RealPartBody<T>>(c, (unsigned)((cnt + NT - 1) / NT), 1, pa);
}

template <typename T>
static int mc_run(cwtb_ctx *c, int nser, const double *noise, const TestNull *tn, unsigned long long seed, long long unit0,
                  int n_units, int64_t n0, double dt, const double *scales, int n_scales, int family,
                  double param, int boxcar_len, const uint8_t *mask, int maxscale, int nbins,
                  int64_t *const hist[2], const CountDst *cd = nullptr) {
  int e = prepare(c, n0, dt, scales, n_scales, family, param, prec_of<T>(), nullptr);
  if (e) return e;
  if ((e = upload_window(c, boxcar_len))) return e;
  if ((e = upload_row_tables(c, c->job))) return e;
  const bool phase = tn && tn->kind == CWTB_NULL_PHASE, ar1 = tn && tn->kind == CWTB_NULL_AR1;
  // AR(1): the held rows in the engine type, where wct3_run keeps x1 and x2 (row 0 is always
  // drawn); the drawn rows of a unit are consecutive, row r at slot[r]
  Buf *const held_buf[3] = {&c->sig, &c->sig2, &c->sig3};
  int ndraw = nser, slot[3] = {0, 1, 2};
  if (ar1) {
    ndraw = 0;
    for (int r = 0; r < nser; ++r) {
      slot[r] = ndraw;
      if (!tn->held[r]) ++ndraw;
      else if ((e = upload_series<T>(c, *held_buf[r], tn->series + (size_t)r * n0, n0))) return e;
    }
  }
  const size_t cnt = (size_t)n_scales * n0;
  if ((e = ensure(c, c->mask, cnt))) return e;
  RT(rt_h2d(c->mask.p, mask, cnt, c->stream));
  const int nh = nser == 2 ? 1 : 2;                 // histograms: one per measure
  const size_t hb = (size_t)n_scales * nbins * sizeof(unsigned long long);
  if ((e = ensure(c, c->hist, nh * hb))) return e;
  RT(rt_memset(c->hist.p, 0, nh * hb, c->stream));
  unsigned long long *dh[2] = {nullptr, nullptr};
  for (int k = 0; k < nh; ++k)
    if (hist[k]) dh[k] = (unsigned long long *)c->hist.p + (size_t)k * n_scales * nbins;
  // surrogates of at most `batch` units are resident at a time
  // (host surrogates stay double on the device; an fp32 run rounds one unit at a time into sig)
  const size_t usz = (size_t)ndraw * n0;            // samples drawn per unit
  // (the rotated spectra of a batch of phase-randomised units take 16 B per sample, AR(1) units
  // sizeof(T); a batch drawn on the device is one launch of ndraw rows per unit)
  const size_t resident = phase ? sizeof(double2) : ar1 ? sizeof(T) : sizeof(double);
  const int batch = noise ? n_units
                          : (int)std::max<size_t>(1, std::min<size_t>({(size_t)n_units, ((size_t)256 << 20) / (usz * resident),
                                                                       (size_t)(MAX_ROWS / ndraw)}));
  const size_t nsz = noise ? sizeof(double) : sizeof(T);
  if ((e = ensure(c, c->noise, (size_t)std::max(batch, 1) * usz * nsz))) return e;
  if (phase && (e = ensure(c, c->prot, (size_t)std::max(batch, 1) * usz * sizeof(double2)))) return e;
  if (noise) RT(rt_h2d(c->noise.p, noise, (size_t)n_units * usz * sizeof(double), c->stream));
  if (noise && sizeof(T) != 8 && (e = ensure(c, c->sig, usz * sizeof(T)))) return e;
  RT(rt_sync(c->stream));
  c->launches = 0;
  if ((e = time_begin(c))) return e;
  for (int i0 = 0; i0 < n_units; i0 += batch) {
    const int nb = std::min(batch, n_units - i0);
    if (phase) {
      if ((e = phase_units<T>(c, tn->ph, nser, seed, unit0 + i0, nb, n0, (T *)c->noise.p))) return e;
    } else if (ar1) {
      for (int r = 0; r < nser; ++r)
        if (!tn->held[r] && (e = ar1_units<T>(c, tn->ar[r], seed, unit0 + i0, nb, n0, (T *)c->noise.p + (size_t)slot[r] * n0,
                                              ndraw, (unsigned)r)))
          return e;
    } else if (!noise) {
      NoiseArgs<T> na{(T *)c->noise.p, seed, unit0 + i0, (long long)n0, nb, nser};
      if ((e = launch<NoiseBody<T>>(c, (unsigned)(((n0 + 1) / 2 + NT - 1) / NT), (unsigned)(nser * nb), na))) return e;
    }
    for (int i = 0; i < nb; ++i) {
      const T *a;
      if constexpr (sizeof(T) == 8) {
        a = (const T *)c->noise.p + (size_t)i * usz;
      } else if (noise) {
        if ((e = to_f32(c, (const double *)c->noise.p + (size_t)i * usz, (float *)c->sig.p, (long long)usz))) return e;
        a = (const T *)c->sig.p;
      } else {
        a = (const T *)c->noise.p + (size_t)i * usz;
      }
      const T *u[3];
      for (int r = 0; r < nser; ++r) u[r] = ar1 && tn->held[r] ? (const T *)held_buf[r]->p : a + (size_t)slot[r] * n0;
      const unsigned char *dmask = (const unsigned char *)c->mask.p;
      // The counters are read and written without atomics by the final kernel of every unit.  That
      // kernel runs on c->stream (run_job forks its transforms onto other streams but joins them
      // back and leaves c->cur = c->stream; the smoothing and final launches follow on it), so the
      // final launches of successive units and batches are ordered and never overlap.
      // The selection bits are written the same way, and labelled on c->stream before the next
      // unit's final launch writes them again.
      const CountDst k = cd ? *cd : CountDst{};
      const SelArgs *sel = k.sel.bits ? &k.sel : nullptr;
      e = nser == 2 ? wct_core<T>(c, c->job, u[0], u[1], boxcar_len, nullptr, nullptr, dmask, maxscale, nbins, dh[0],
                                  k.obs[0], k.cnt[0], sel)
                    : wct3_core<T>(c, c->job, u[0], u[1], u[2], boxcar_len, nullptr, nullptr, dmask, maxscale,
                                   nbins, dh[0], dh[1], nullptr, k.obs[0], k.obs[1], k.cnt[0], k.cnt[1], sel);
      if (e) return e;
      if (sel && (e = label_bits(c, n_scales, n0, k.q, k.qmax + i0 + i, nullptr, nullptr))) return e;
    }
  }
  if ((e = time_end(c, &c->last_ms))) return e;
  c->job_dsig = nullptr;
  std::vector<unsigned long long> h((size_t)n_scales * nbins);
  for (int k = 0; k < nh; ++k) {
    if (!hist[k]) continue;
    RT(rt_d2h(h.data(), dh[k], hb, c->stream));
    RT(rt_sync(c->stream));
    for (size_t i = 0; i < h.size(); ++i) hist[k][i] += (int64_t)h[i];
  }
  return 0;
}
}  // extern "C++"

static int mc_core(cwtb_ctx *c, int nser, const double *noise, const TestNull *tn, unsigned long long seed,
                   long long unit0, int n_units, int64_t n0, double dt, const double *scales, int n_scales, int family,
                   double param, int boxcar_len, const uint8_t *mask, int maxscale, int nbins,
                   int64_t *const hist[2], const CountDst *cd = nullptr) {
  if (!c || !mask || !(hist[0] || hist[1]) || n_units < 0 || nbins < 1 || maxscale < 0 || maxscale > n_scales)
    return fail(c, CWTB_ERR_ARG, nser == 2 ? "wct_mc: bad argument" : "wct3_mc: bad argument");
  if (family == CWTB_TABLE)
    return fail(c, CWTB_ERR_UNSUPPORTED, nser == 2 ? "wct_mc needs an analytic wavelet family"
                                                   : "wct3_mc needs an analytic wavelet family");
  return c->coh_precision == CWTB_F32
             ? mc_run<float>(c, nser, noise, tn, seed, unit0, n_units, n0, dt, scales, n_scales, family, param,
                             boxcar_len, mask, maxscale, nbins, hist, cd)
             : mc_run<double>(c, nser, noise, tn, seed, unit0, n_units, n0, dt, scales, n_scales, family, param,
                              boxcar_len, mask, maxscale, nbins, hist, cd);
}

int cwtb_wct_mc(cwtb_ctx *c, const double *noise, int n_pairs, int64_t n0, double dt, double dj,
                const double *scales, int n_scales, int family, double param, int boxcar_len,
                const uint8_t *mask, int maxscale, int nbins, int64_t *hist) {
  (void)dj;
  if (!noise) return fail(c, CWTB_ERR_ARG, "wct_mc: null surrogates");
  int64_t *const h[2] = {hist, nullptr};
  return mc_core(c, 2, noise, nullptr, 0, 0, n_pairs, n0, dt, scales, n_scales, family, param, boxcar_len, mask,
                 maxscale, nbins, h);
}

int cwtb_wct_mc_seeded(cwtb_ctx *c, uint64_t seed, int64_t first_pair, int n_pairs, int64_t n0, double dt,
                       const double *scales, int n_scales, int family, double param, int boxcar_len,
                       const uint8_t *mask, int maxscale, int nbins, int64_t *hist) {
  int64_t *const h[2] = {hist, nullptr};
  return mc_core(c, 2, nullptr, nullptr, seed, first_pair, n_pairs, n0, dt, scales, n_scales, family, param, boxcar_len,
                 mask, maxscale, nbins, h);
}

int cwtb_wct3_mc(cwtb_ctx *c, const double *noise, int n_triples, int64_t n0, double dt, const double *scales,
                 int n_scales, int family, double param, int boxcar_len, const uint8_t *mask, int maxscale,
                 int nbins, int64_t *hist_partial, int64_t *hist_multiple) {
  if (!noise) return fail(c, CWTB_ERR_ARG, "wct3_mc: null surrogates");
  int64_t *const h[2] = {hist_partial, hist_multiple};
  return mc_core(c, 3, noise, nullptr, 0, 0, n_triples, n0, dt, scales, n_scales, family, param, boxcar_len, mask,
                 maxscale, nbins, h);
}

int cwtb_wct3_mc_seeded(cwtb_ctx *c, uint64_t seed, int64_t first_triple, int n_triples, int64_t n0, double dt,
                        const double *scales, int n_scales, int family, double param, int boxcar_len,
                        const uint8_t *mask, int maxscale, int nbins, int64_t *hist_partial,
                        int64_t *hist_multiple) {
  int64_t *const h[2] = {hist_partial, hist_multiple};
  return mc_core(c, 3, nullptr, nullptr, seed, first_triple, n_triples, n0, dt, scales, n_scales, family, param,
                 boxcar_len, mask, maxscale, nbins, h);
}

// test hooks: the surrogates of the seeded mode, [n_units][nser][n0] to the host, drawn in launches
// of at most MAX_ROWS / nser units like mc_run's
static int mc_surrogates(cwtb_ctx *c, int nser, uint64_t seed, int64_t unit0, int n_units, int64_t n0, double *out) {
  if (!c || !out || n_units < 1 || n0 < 1) return fail(c, CWTB_ERR_ARG, "mc_surrogates: bad argument");
  const size_t usz = (size_t)nser * n0, bytes = (size_t)n_units * usz * sizeof(double);
  int e = ensure(c, c->noise, bytes);
  if (e) return e;
  const int batch = (int)(MAX_ROWS / nser);
  for (int i0 = 0; i0 < n_units; i0 += batch) {
    const int nb = std::min(batch, n_units - i0);
    NoiseArgs<double> na{(double *)c->noise.p + (size_t)i0 * usz, seed, unit0 + i0, (long long)n0, nb, nser};
    if ((e = launch<NoiseBody<double>>(c, (unsigned)(((n0 + 1) / 2 + NT - 1) / NT), (unsigned)(nser * nb), na))) return e;
  }
  RT(rt_d2h(out, c->noise.p, bytes, c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

int cwtb_mc_surrogates(cwtb_ctx *c, uint64_t seed, int64_t first_pair, int n_pairs, int64_t n0, double *out) {
  return mc_surrogates(c, 2, seed, first_pair, n_pairs, n0, out);
}

int cwtb_mc_surrogates3(cwtb_ctx *c, uint64_t seed, int64_t first_triple, int n_triples, int64_t n0, double *out) {
  return mc_surrogates(c, 3, seed, first_triple, n_triples, n0, out);
}

// ---- phase-randomised surrogates of the data (PhaseRotBody) -----------------------------------
// argument checks shared by the two entry points, then the spectra of the nser series at their own
// length into c->pspec (fp64; the reals are staged in c->prot)
static int phase_spectra(cwtb_ctx *c, const char *name, const double *series, int nser, const int *group,
                         int64_t first_unit, int n_units, int64_t n0, PhaseSrc *ph) {
  const std::string nm(name);
  if (!c || !series || !group || nser < 1 || nser > 3 || n0 < 4 || n_units < 0 || first_unit < 0 ||
      first_unit > (1ll << 61) - n_units)
    return fail(c, CWTB_ERR_ARG, nm + ": bad argument");
  for (int r = 0; r < nser; ++r) {
    if (group[r] < 0) return fail(c, CWTB_ERR_ARG, nm + ": negative phase group");
    ph->group[r] = group[r];
  }
  const bool pow2 = (n0 & (n0 - 1)) == 0;
  if (n0 > (pow2 ? 1ll << 26 : 1ll << 24))
    return fail(c, CWTB_ERR_UNSUPPORTED, nm + ": series longer than 2^26 (2^24 if the length is not 2^k)");
  RT(rt_set_device(c->device));
  const size_t cnt = (size_t)nser * n0;
  int e;
  if ((e = ensure(c, c->pspec, cnt * sizeof(double2)))) return e;
  if ((e = ensure(c, c->prot, cnt * sizeof(double)))) return e;
  RT(rt_h2d(c->prot.p, series, cnt * sizeof(double), c->stream));
  c->prof_tag = "data:";
  e = pow2 ? fft_rows<double, -1>(c, c->prot.p, 1, n0, n0, (double2 *)c->pspec.p, n0, (unsigned)n0, nser)
           : blue_rows(c, c->prot.p, 1, n0, (double2 *)c->pspec.p, n0, (unsigned)n0, nser, -1, 1.0, n0);
  c->prof_tag = "";
  if (e) return e;
  RT(rt_sync(c->stream));   // `series` is the caller's again
  return 0;
}

static int test_null(cwtb_ctx *c, const std::string &nm, const double *series, int nser, int null, const int *group,
                     const double *g, const double *m, const double *sigma, const int *held, int64_t first_unit,
                     int n_units, int64_t n0, TestNull &tn);

static int wct_mc_null(cwtb_ctx *c, const std::string &nm, const double *series, int nser, int null,
                       const int *group, const double *g, const double *m, const double *sigma, const int *held,
                       uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                       int n_scales, int family, double param, int boxcar_len, const uint8_t *mask, int maxscale,
                       int nbins, int64_t *hist_a, int64_t *hist_b) {
  if (nser == 2 && hist_b) return fail(c, CWTB_ERR_ARG, nm + ": two series have one histogram");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, nm + " needs an analytic wavelet family");
  if (!mask || !(hist_a || hist_b) || (nser != 2 && nser != 3)) return fail(c, CWTB_ERR_ARG, nm + ": bad argument");
  TestNull tn;
  int e = test_null(c, nm, series, nser, null, group, g, m, sigma, held, first_unit, n_units, n0, tn);
  if (e) return e;
  int64_t *const h[2] = {hist_a, hist_b};
  return mc_core(c, nser, nullptr, &tn, seed, first_unit, n_units, n0, dt, scales, n_scales, family, param,
                 boxcar_len, mask, maxscale, nbins, h);
}

int cwtb_wct_mc_phase(cwtb_ctx *c, const double *series, int nser, const int *group, uint64_t seed,
                      int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                      int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                      int maxscale, int nbins, int64_t *hist_a, int64_t *hist_b) {
  return wct_mc_null(c, "wct_mc_phase", series, nser, CWTB_NULL_PHASE, group, nullptr, nullptr, nullptr, nullptr,
                     seed, first_unit, n_units, n0, dt, scales, n_scales, family, param, boxcar_len, mask, maxscale,
                     nbins, hist_a, hist_b);
}

int cwtb_wct_mc_null(cwtb_ctx *c, const double *series, int nser, int null, const int *group, const double *g,
                     const double *m, const double *sigma, const int *held, uint64_t seed, int64_t first_unit,
                     int n_units, int64_t n0, double dt, const double *scales, int n_scales, int family,
                     double param, int boxcar_len, const uint8_t *mask, int maxscale, int nbins, int64_t *hist_a,
                     int64_t *hist_b) {
  return wct_mc_null(c, "wct_mc_null", series, nser, null, group, g, m, sigma, held, seed, first_unit, n_units, n0,
                     dt, scales, n_scales, family, param, boxcar_len, mask, maxscale, nbins, hist_a, hist_b);
}

int cwtb_mc_phase_surrogates(cwtb_ctx *c, const double *series, int nser, const int *group, uint64_t seed,
                             int64_t first_unit, int n_units, int64_t n0, double *out) {
  if (!out || n_units < 1 || (nser != 2 && nser != 3)) return fail(c, CWTB_ERR_ARG, "mc_phase_surrogates: bad argument");
  PhaseSrc ph{};
  int e = phase_spectra(c, "mc_phase_surrogates", series, nser, group, first_unit, n_units, n0, &ph);
  if (e) return e;
  const size_t usz = (size_t)nser * n0, cnt = (size_t)n_units * usz;
  const int batch = (int)(MAX_ROWS / nser);   // units per launch, like mc_run's
  if ((e = ensure(c, c->noise, cnt * sizeof(double)))) return e;
  if ((e = ensure(c, c->prot, (size_t)std::min(batch, n_units) * usz * sizeof(double2)))) return e;
  for (int i0 = 0; i0 < n_units; i0 += batch) {
    const int nb = std::min(batch, n_units - i0);
    if ((e = phase_units<double>(c, ph, nser, seed, first_unit + i0, nb, n0, (double *)c->noise.p + (size_t)i0 * usz)))
      return e;
  }
  RT(rt_d2h(out, c->noise.p, cnt * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

// ---- point-wise tests against surrogates: counting -------------------------------------------
// The units' exceedance counts of the resident coherence (nser 2) or partial and multiple
// coherence (nser 3) added to the slot's counters, with the histograms of cwtb_wct_mc_phase
static int surrogate_counts(cwtb_ctx *c, int nser, const double *series, int null, const int *group,
                            const double *g, const double *m, const double *sigma, const int *held, uint64_t seed,
                            int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                            int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                            int maxscale, int nbins, int64_t *hist_a, int64_t *hist_b, int64_t serial, int reset) {
  if (!c) return CWTB_ERR_ARG;
  const std::string nm = nser == 2 ? "coherence_surrogate_counts" : "coherence3_surrogate_counts";
  ResidentSlot &s = nser == 2 ? c->coh : c->coh3;
  if (s.S <= 0 || !s.buf.p || serial != s.serial)
    return fail(c, CWTB_ERR_STATE, nm + ": the serial is not that of the resident product");
  if (n_scales != s.S || n0 != s.n0)
    return fail(c, CWTB_ERR_STATE, nm + ": scales or length differ from the resident product's");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, nm + " needs an analytic wavelet family");
  if (!mask || !(hist_a || hist_b)) return fail(c, CWTB_ERR_ARG, nm + ": bad argument");
  const long long base = reset || s.units < 0 ? 0 : s.units;
  if (n_units < 0 || n_units > 0xFFFFFFFFll - base)
    return fail(c, CWTB_ERR_ARG, nm + ": more units than a 32-bit counter holds");
  TestNull tn;
  int e = test_null(c, nm, series, nser, null, group, g, m, sigma, held, first_unit, n_units, n0, tn);
  if (e) return e;
  if (base > 0 && null != s.null)
    return fail(c, CWTB_ERR_STATE, nm + ": the counts hold the units of another null: reset them first");
  const size_t cnt = (size_t)s.S * s.n0, off = coh_angle_offset(cnt);
  if ((e = ensure(c, s.counts, (nser == 2 ? cnt : off + cnt) * sizeof(unsigned)))) return e;
  s.units = -1;   // nothing readable until this call completes
  if (base == 0) RT(rt_memset(s.counts.p, 0, s.counts.bytes, c->stream));
  const double *obs = (const double *)s.buf.p;   // WCT; RP2 at 0 and RM2 at 2 off
  unsigned *k = (unsigned *)s.counts.p;           // one field; RP2's at 0 and RM2's at off
  const CountDst cd = nser == 2 ? CountDst{{obs, nullptr}, {k, nullptr}} : CountDst{{obs, obs + 2 * off}, {k, k + off}};
  int64_t *const h[2] = {hist_a, hist_b};
  if ((e = mc_core(c, nser, nullptr, &tn, seed, first_unit, n_units, n0, dt, scales, n_scales, family, param,
                   boxcar_len, mask, maxscale, nbins, h, &cd)))
    return e;
  s.units = base + n_units;
  s.null = null;
  return 0;
}

int cwtb_coherence_surrogate_counts(cwtb_ctx *c, const double *series, const int *group, uint64_t seed,
                                    int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                    int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                    int maxscale, int nbins, int64_t *hist, int64_t serial, int reset) {
  return surrogate_counts(c, 2, series, CWTB_NULL_PHASE, group, nullptr, nullptr, nullptr, nullptr, seed, first_unit,
                          n_units, n0, dt, scales, n_scales, family, param, boxcar_len, mask, maxscale, nbins, hist,
                          nullptr, serial, reset);
}

int cwtb_coherence3_surrogate_counts(cwtb_ctx *c, const double *series, const int *group, uint64_t seed,
                                     int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                     int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                     int maxscale, int nbins, int64_t *hist_partial, int64_t *hist_multiple,
                                     int64_t serial, int reset) {
  return surrogate_counts(c, 3, series, CWTB_NULL_PHASE, group, nullptr, nullptr, nullptr, nullptr, seed, first_unit,
                          n_units, n0, dt, scales, n_scales, family, param, boxcar_len, mask, maxscale, nbins,
                          hist_partial, hist_multiple, serial, reset);
}

int cwtb_coherence_surrogate_counts_null(cwtb_ctx *c, const double *series, int null, const int *group,
                                         const double *g, const double *m, const double *sigma, const int *held,
                                         uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double dt,
                                         const double *scales, int n_scales, int family, double param,
                                         int boxcar_len, const uint8_t *mask, int maxscale, int nbins, int64_t *hist,
                                         int64_t serial, int reset) {
  return surrogate_counts(c, 2, series, null, group, g, m, sigma, held, seed, first_unit, n_units, n0, dt, scales,
                          n_scales, family, param, boxcar_len, mask, maxscale, nbins, hist, nullptr, serial, reset);
}

int cwtb_coherence3_surrogate_counts_null(cwtb_ctx *c, const double *series, int null, const int *group,
                                          const double *g, const double *m, const double *sigma, const int *held,
                                          uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double dt,
                                          const double *scales, int n_scales, int family, double param,
                                          int boxcar_len, const uint8_t *mask, int maxscale, int nbins,
                                          int64_t *hist_partial, int64_t *hist_multiple, int64_t serial, int reset) {
  return surrogate_counts(c, 3, series, null, group, g, m, sigma, held, seed, first_unit, n_units, n0, dt, scales,
                          n_scales, family, param, boxcar_len, mask, maxscale, nbins, hist_partial, hist_multiple,
                          serial, reset);
}

// ---- cluster tests against surrogates ----------------------------------------------------------
// The per-row arguments of a cluster test into c->cl_rows: thr [S] double, lo, hi [S] int64, q [S]
// uint64 (thr, lo, hi null: the test hook, which needs q alone)
static int cluster_rows(cwtb_ctx *c, const std::string &nm, int S, long long n0, const double *thr, const int64_t *lo,
                        const int64_t *hi, const uint64_t *q, SelArgs &sel, const unsigned long long *&dq) {
  if (!q || (!thr && (lo || hi)) || (thr && (!lo || !hi))) return fail(c, CWTB_ERR_ARG, nm + ": null argument");
  for (int j = 0; j < S; ++j) {
    if (q[j] > (1ull << 32)) return fail(c, CWTB_ERR_ARG, nm + ": a weight q above 2^32");
    if (lo && (lo[j] < 0 || hi[j] > n0 || lo[j] > hi[j]))
      return fail(c, CWTB_ERR_ARG, nm + ": column range outside [0, n0) or lo > hi");
  }
  int e = ensure(c, c->cl_rows, (size_t)S * 32);
  if (e) return e;
  double *dthr = (double *)c->cl_rows.p;
  long long *dlo = (long long *)(dthr + S), *dhi = dlo + S;
  unsigned long long *dq64 = (unsigned long long *)(dhi + S);
  if (thr) {
    RT(rt_h2d(dthr, thr, (size_t)S * 8, c->stream));
    RT(rt_h2d(dlo, lo, (size_t)S * 8, c->stream));
    RT(rt_h2d(dhi, hi, (size_t)S * 8, c->stream));
  }
  RT(rt_h2d(dq64, q, (size_t)S * 8, c->stream));
  const long long words = (n0 + 31) / 32;
  if ((e = ensure(c, c->cl_bits, (size_t)S * words * sizeof(unsigned)))) return e;
  sel = SelArgs{(unsigned *)c->cl_bits.p, dthr, dlo, dhi, words, 0};
  dq = dq64;
  return 0;
}

// a map of S x n0 points labels with 32-bit flat indices, and its sums of q <= 2^32 fit 64 bits
static int cluster_shape(cwtb_ctx *c, const std::string &nm, long long S, long long n0) {
  if (S < 1 || n0 < 1) return fail(c, CWTB_ERR_ARG, nm + ": bad n_scales / n0");
  if ((unsigned long long)S * (unsigned long long)n0 >= (1ull << 32))
    return fail(c, CWTB_ERR_UNSUPPORTED, nm + ": n_scales * n0 must stay below 2^32");
  if (S > (long long)MAX_ROWS) return fail(c, CWTB_ERR_ARG, nm + ": more than 65535 scales");
  return 0;
}

static int cluster_test(cwtb_ctx *c, int nser, const double *series, int null, const int *group, const double *g,
                        const double *m, const double *sigma, const int *held, uint64_t seed,
                        int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales, int n_scales,
                        int family, double param, int boxcar_len, const uint8_t *mask, int maxscale, int nbins,
                        int64_t *hist_a, int64_t *hist_b, int64_t serial, const double *thr, const int64_t *lo,
                        const int64_t *hi, const uint64_t *q, int measure, uint64_t *qmax_out) {
  if (!c) return CWTB_ERR_ARG;
  const std::string nm = nser == 2 ? "coherence_cluster_test" : "coherence3_cluster_test";
  ResidentSlot &s = nser == 2 ? c->coh : c->coh3;
  s.clusters = false;   // nothing readable until this call completes
  s.table = ClusterTable{};
  if (s.S <= 0 || !s.buf.p || serial != s.serial)
    return fail(c, CWTB_ERR_STATE, nm + ": the serial is not that of the resident product");
  if (n_scales != s.S || n0 != s.n0)
    return fail(c, CWTB_ERR_STATE, nm + ": scales or length differ from the resident product's");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, nm + " needs an analytic wavelet family");
  if (!mask || !(hist_a || hist_b) || !thr || (n_units > 0 && !qmax_out))
    return fail(c, CWTB_ERR_ARG, nm + ": bad argument");
  int e = cluster_shape(c, nm, n_scales, n0);
  if (e) return e;
  FieldRef f;
  if ((e = nser == 2 ? field_ref(c, FIELD_COH, f) : coh3_ref(c, measure, false, f))) return e;
  TestNull tn;
  if ((e = test_null(c, nm, series, nser, null, group, g, m, sigma, held, first_unit, n_units, n0, tn))) return e;
  SelArgs sel;
  const unsigned long long *dq;
  if ((e = cluster_rows(c, nm, n_scales, n0, thr, lo, hi, q, sel, dq))) return e;
  sel.measure = measure == CWTB_MEASURE_MULTIPLE ? 1 : 0;
  if ((e = ensure(c, c->cl_qmax, (size_t)(n_units + 1) * sizeof(unsigned long long)))) return e;
  if ((e = ensure(c, s.labels, (size_t)n_scales * n0 * sizeof(int)))) return e;
  unsigned long long *dqmax = (unsigned long long *)c->cl_qmax.p;
  RT(rt_memset(dqmax, 0, (size_t)(n_units + 1) * sizeof(unsigned long long), c->stream));
  // the observed map: its bits through the field layer, then the same labelling as the units'
  ThreshBitsArgs ta{(const double *)f.p, sel, n0};
  if ((e = launch<ThreshBitsBody>(c, (unsigned)((n0 + NT - 1) / NT), (unsigned)n_scales, ta))) return e;
  ClusterTable tab;
  if ((e = label_bits(c, n_scales, n0, dq, dqmax + n_units, &tab, (int *)s.labels.p))) return e;
  // the units: the final kernels write whole chunks of columns, so the bits past the last column
  // stay as zeroed here
  RT(rt_memset(sel.bits, 0, (size_t)n_scales * sel.words * sizeof(unsigned), c->stream));
  CountDst cd{};
  cd.sel = sel;
  cd.q = dq;
  cd.qmax = dqmax;
  int64_t *const h[2] = {hist_a, hist_b};
  if ((e = mc_core(c, nser, nullptr, &tn, seed, first_unit, n_units, n0, dt, scales, n_scales, family, param,
                   boxcar_len, mask, maxscale, nbins, h, &cd)))
    return e;
  if (n_units > 0) RT(rt_d2h(qmax_out, dqmax, (size_t)n_units * sizeof(unsigned long long), c->stream));
  RT(rt_sync(c->stream));
  s.table = std::move(tab);
  s.clusters = true;
  return 0;
}

int cwtb_coherence_cluster_test(cwtb_ctx *c, const double *series, const int *group, uint64_t seed,
                                int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                int maxscale, int nbins, int64_t *hist, int64_t serial, const double *thr,
                                const int64_t *lo, const int64_t *hi, const uint64_t *q, uint64_t *qmax_out) {
  return cluster_test(c, 2, series, CWTB_NULL_PHASE, group, nullptr, nullptr, nullptr, nullptr, seed, first_unit,
                      n_units, n0, dt, scales, n_scales, family, param, boxcar_len, mask, maxscale, nbins, hist,
                      nullptr, serial, thr, lo, hi, q, 0, qmax_out);
}

int cwtb_coherence3_cluster_test(cwtb_ctx *c, const double *series, const int *group, uint64_t seed,
                                 int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                 int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                 int maxscale, int nbins, int64_t *hist_partial, int64_t *hist_multiple,
                                 int64_t serial, const double *thr, const int64_t *lo, const int64_t *hi,
                                 const uint64_t *q, int measure, uint64_t *qmax_out) {
  return cluster_test(c, 3, series, CWTB_NULL_PHASE, group, nullptr, nullptr, nullptr, nullptr, seed, first_unit,
                      n_units, n0, dt, scales, n_scales, family, param, boxcar_len, mask, maxscale, nbins,
                      hist_partial, hist_multiple, serial, thr, lo, hi, q, measure, qmax_out);
}

int cwtb_coherence_cluster_test_null(cwtb_ctx *c, const double *series, int null, const int *group, const double *g,
                                     const double *m, const double *sigma, const int *held, uint64_t seed,
                                     int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                     int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                     int maxscale, int nbins, int64_t *hist, int64_t serial, const double *thr,
                                     const int64_t *lo, const int64_t *hi, const uint64_t *q, uint64_t *qmax_out) {
  return cluster_test(c, 2, series, null, group, g, m, sigma, held, seed, first_unit, n_units, n0, dt, scales,
                      n_scales, family, param, boxcar_len, mask, maxscale, nbins, hist, nullptr, serial, thr, lo, hi,
                      q, 0, qmax_out);
}

int cwtb_coherence3_cluster_test_null(cwtb_ctx *c, const double *series, int null, const int *group, const double *g,
                                      const double *m, const double *sigma, const int *held, uint64_t seed,
                                      int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                      int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                      int maxscale, int nbins, int64_t *hist_partial, int64_t *hist_multiple,
                                      int64_t serial, const double *thr, const int64_t *lo, const int64_t *hi,
                                      const uint64_t *q, int measure, uint64_t *qmax_out) {
  return cluster_test(c, 3, series, null, group, g, m, sigma, held, seed, first_unit, n_units, n0, dt, scales,
                      n_scales, family, param, boxcar_len, mask, maxscale, nbins, hist_partial, hist_multiple, serial,
                      thr, lo, hi, q, measure, qmax_out);
}

// the first min(cap, count) rows of a table
static int table_out(cwtb_ctx *c, const ClusterTable &t, int64_t cap, int64_t *count, uint64_t *Q, int64_t *points,
                     int64_t *box) {
  if (!count || cap < 0) return fail(c, CWTB_ERR_ARG, "cluster table: bad argument");
  const size_t m = std::min<size_t>((size_t)cap, t.Q.size());
  if (m && (!Q || !points || !box)) return fail(c, CWTB_ERR_ARG, "cluster table: null argument");
  *count = (int64_t)t.Q.size();
  for (size_t i = 0; i < m; ++i) {
    Q[i] = t.Q[i];
    points[i] = (int64_t)t.pts[i];
  }
  if (m) memcpy(box, t.box.data(), m * 4 * sizeof(int64_t));
  return 0;
}

static int clusters_of(cwtb_ctx *c, ResidentSlot &s, const char *what) {
  if (!c) return CWTB_ERR_ARG;
  if (s.S <= 0 || !s.buf.p) return fail(c, CWTB_ERR_STATE, std::string("no ") + what + " resident");
  if (!s.clusters) return fail(c, CWTB_ERR_STATE, "no cluster test has run for this product");
  RT(rt_set_device(c->device));
  return 0;
}

int cwtb_coherence_cluster_table(cwtb_ctx *c, int64_t cap, int64_t *count, uint64_t *Q, int64_t *points,
                                 int64_t *box) {
  int e = c ? clusters_of(c, c->coh, "coherence") : CWTB_ERR_ARG;
  return e ? e : table_out(c, c->coh.table, cap, count, Q, points, box);
}

int cwtb_coherence3_cluster_table(cwtb_ctx *c, int64_t cap, int64_t *count, uint64_t *Q, int64_t *points,
                                  int64_t *box) {
  int e = c ? clusters_of(c, c->coh3, "partial / multiple coherence") : CWTB_ERR_ARG;
  return e ? e : table_out(c, c->coh3.table, cap, count, Q, points, box);
}

// labels[row0 + r row_step][col0 + k col_step] into out [nrows][ncols], with window_run's checks
static int labels_window(cwtb_ctx *c, const ResidentSlot &s, int row0, int nrows, int row_step, int64_t col0,
                         int64_t ncols, int64_t col_step, int32_t *out) {
  const int S = s.S;
  const long long n0 = s.n0;
  if (nrows < 0 || ncols < 0 || row_step < 1 || col_step < 1) return fail(c, CWTB_ERR_ARG, "bad window");
  if (nrows == 0 || ncols == 0) return 0;
  if (!out) return fail(c, CWTB_ERR_ARG, "null argument");
  if (row0 < 0 || row0 >= S || (long long)(nrows - 1) > (long long)(S - 1 - row0) / row_step ||
      col0 < 0 || col0 >= n0 || (ncols - 1) > (n0 - 1 - col0) / col_step)
    return fail(c, CWTB_ERR_ARG, "window outside the resident field");
  const size_t m = (size_t)nrows * ncols;
  int e = ensure(c, c->aux, m * sizeof(int));
  if (e) return e;
  LabelWindowArgs a{(const int *)s.labels.p, (int *)c->aux.p, n0, row0, row_step, col0, col_step, ncols};
  if ((e = launch<LabelWindowBody>(c, (unsigned)((ncols + NT - 1) / NT), (unsigned)nrows, a))) return e;
  RT(rt_d2h(out, c->aux.p, m * sizeof(int), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

int cwtb_coherence_cluster_labels(cwtb_ctx *c, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                                  int64_t col_step, int32_t *out) {
  int e = c ? clusters_of(c, c->coh, "coherence") : CWTB_ERR_ARG;
  return e ? e : labels_window(c, c->coh, row0, nrows, row_step, col0, ncols, col_step, out);
}

int cwtb_coherence3_cluster_labels(cwtb_ctx *c, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                                   int64_t col_step, int32_t *out) {
  int e = c ? clusters_of(c, c->coh3, "partial / multiple coherence") : CWTB_ERR_ARG;
  return e ? e : labels_window(c, c->coh3, row0, nrows, row_step, col0, ncols, col_step, out);
}

int cwtb_cluster_label_bits(cwtb_ctx *c, const uint32_t *bits, int n_scales, int64_t n0, const uint64_t *q,
                            int64_t cap, int64_t *count, uint64_t *Q, int64_t *points, int64_t *box,
                            int32_t *labels, uint64_t *qmax) {
  if (!c) return CWTB_ERR_ARG;
  const std::string nm = "cluster_label_bits";
  int e = cluster_shape(c, nm, n_scales, n0);
  if (e) return e;
  if (!bits || !qmax || !count) return fail(c, CWTB_ERR_ARG, nm + ": null argument");
  const long long words = (n0 + 31) / 32;
  if (n0 % 32)
    for (int j = 0; j < n_scales; ++j)
      if (bits[(size_t)j * words + words - 1] >> (n0 % 32))
        return fail(c, CWTB_ERR_ARG, nm + ": bits set past the last column");
  RT(rt_set_device(c->device));
  SelArgs sel;
  const unsigned long long *dq;
  if ((e = cluster_rows(c, nm, n_scales, n0, nullptr, nullptr, nullptr, q, sel, dq))) return e;
  RT(rt_h2d(sel.bits, bits, (size_t)n_scales * words * sizeof(unsigned), c->stream));
  if ((e = ensure(c, c->cl_qmax, sizeof(unsigned long long)))) return e;
  if ((e = ensure(c, c->scratch, (size_t)n_scales * n0 * sizeof(int)))) return e;
  RT(rt_memset(c->cl_qmax.p, 0, sizeof(unsigned long long), c->stream));
  ClusterTable t;
  if ((e = label_bits(c, n_scales, n0, dq, (unsigned long long *)c->cl_qmax.p, &t, (int *)c->scratch.p))) return e;
  RT(rt_d2h(qmax, c->cl_qmax.p, sizeof(unsigned long long), c->stream));
  if (labels) RT(rt_d2h(labels, c->scratch.p, (size_t)n_scales * n0 * sizeof(int), c->stream));
  RT(rt_sync(c->stream));
  return table_out(c, t, cap, count, Q, points, box);
}

// ---- AR(1) red-noise surrogates (Ar1BlockBody, Ar1CarryBody, Ar1WriteBody) ------------------------
static int ar1_check(cwtb_ctx *c, const std::string &nm, const Ar1Src &ar) {
  if (!std::isfinite(ar.g) || !(std::fabs(ar.g) < 1.0) || !std::isfinite(ar.m) || !std::isfinite(ar.sigma))
    return fail(c, CWTB_ERR_ARG, nm + ": the AR(1) parameters must be finite, with |g| < 1");
  return 0;
}

extern "C++" {
// nb AR(1) units from unit0 of the series tag `stag` into out [nb][nser][n0] (nb <= MAX_ROWS; out
// points at the series' first row); c->arc holds the CTAs' carries
template <typename T>
static int ar1_units(cwtb_ctx *c, const Ar1Src &ar, unsigned long long seed, long long unit0, int nb, int64_t n0,
                     T *out, int nser, unsigned stag) {
  const long long per = (long long)NT * AR1_CH;   // samples per CTA
  const int nblk = (int)((n0 + per - 1) / per);
  int e = ensure(c, c->arc, (size_t)nb * nblk * 2 * sizeof(double));
  if (e) return e;
  struct Tag { cwtb_ctx *c; ~Tag() { c->prof_tag = ""; } } tag{c};
  c->prof_tag = "ar1:";
  Ar1Args<T> a{out, (double *)c->arc.p, seed, unit0, (long long)n0, ar.g, std::sqrt((1.0 - ar.g) * (1.0 + ar.g)),
               ar.m, ar.sigma, nblk, nb, nser, stag};
  if ((e = launch<Ar1BlockBody<T>>(c, (unsigned)nblk, (unsigned)nb, a))) return e;
  Ar1CarryArgs ca{(double *)c->arc.p, nblk, nb};
  if ((e = launch<Ar1CarryBody>(c, (unsigned)((nb + NT - 1) / NT), 1, ca))) return e;
  return launch<Ar1WriteBody<T>>(c, (unsigned)nblk, (unsigned)nb, a);
}
}  // extern "C++"

int cwtb_mc_ar1_surrogates(cwtb_ctx *c, double g, double m, double sigma, uint64_t seed, int64_t first_unit,
                           int n_units, int64_t n0, double *out) {
  if (!c) return CWTB_ERR_ARG;
  const std::string nm = "mc_ar1_surrogates";
  if (!out || n_units < 1 || n0 < 1 || first_unit < 0 || first_unit > (1ll << 61) - n_units)
    return fail(c, CWTB_ERR_ARG, nm + ": bad argument");
  const Ar1Src ar{g, m, sigma};
  int e = ar1_check(c, nm, ar);
  if (e) return e;
  RT(rt_set_device(c->device));
  const size_t cnt = (size_t)n_units * n0;
  if ((e = ensure(c, c->noise, cnt * sizeof(double)))) return e;
  for (int i0 = 0; i0 < n_units; i0 += (int)MAX_ROWS) {
    const int nb = std::min((int)MAX_ROWS, n_units - i0);
    if ((e = ar1_units<double>(c, ar, seed, first_unit + i0, nb, n0, (double *)c->noise.p + (size_t)i0 * n0, 1, 0)))
      return e;
  }
  RT(rt_d2h(out, c->noise.p, cnt * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

// ---- the nulls of the tests against surrogates ---------------------------------------------------
// The null of a test of nser series (TestNull): phase-randomised units in the phase groups `group`,
// or AR(1) units with the parameters g, m, sigma [nser] and, where held (may be null: none) is 1, the
// data's row of `series` in every unit.  Only the coherence tests hold rows: x1 and x2 of the
// partial and multiple coherence (y, and the series of a pair, are always drawn).
static int test_null(cwtb_ctx *c, const std::string &nm, const double *series, int nser, int null, const int *group,
                     const double *g, const double *m, const double *sigma, const int *held, int64_t first_unit,
                     int n_units, int64_t n0, TestNull &tn) {
  tn = TestNull{null, nser, {}, PhaseSrc{}, {0, 0, 0}, nullptr};
  if (null == CWTB_NULL_PHASE) return phase_spectra(c, nm.c_str(), series, nser, group, first_unit, n_units, n0, &tn.ph);
  if (null != CWTB_NULL_AR1) return fail(c, CWTB_ERR_ARG, nm + ": unknown null");
  if (!g || !m || !sigma || nser < 1 || nser > 3 || n_units < 0 || first_unit < 0 ||
      first_unit > (1ll << 61) - n_units)
    return fail(c, CWTB_ERR_ARG, nm + ": bad argument");
  for (int r = 0; r < nser; ++r) {
    tn.held[r] = held ? held[r] : 0;
    if (tn.held[r] != 0 && (tn.held[r] != 1 || r == 0 || nser != 3))
      return fail(c, CWTB_ERR_ARG, nm + ": only x1 and x2 of three series can be held at the data");
    if (tn.held[r]) {
      if (!series) return fail(c, CWTB_ERR_ARG, nm + ": held series without data");
      continue;
    }
    tn.ar[r] = Ar1Src{g[r], m[r], sigma[r]};
    int e = ar1_check(c, nm, tn.ar[r]);
    if (e) return e;
  }
  tn.series = series;
  RT(rt_set_device(c->device));
  return 0;
}

// ---- tests of the resident power and cross spectrum against surrogates -----------------------
// Their nulls draw every series (the power: 1, the cross spectrum: 2): AR(1) units, or phase-
// randomised units of the series in phase group s: independent phases
static const int PHASE_GROUPS[2] = {0, 1};

// the checks of a test against the resident product of slot s
static int test_slot(cwtb_ctx *c, const ResidentSlot &s, const std::string &nm, int64_t serial, int n_scales,
                     int64_t n0, int family) {
  if (s.S <= 0 || !s.buf.p || serial != s.serial)
    return fail(c, CWTB_ERR_STATE, nm + ": the serial is not that of the resident product");
  if (n_scales != s.S || n0 != s.n0)
    return fail(c, CWTB_ERR_STATE, nm + ": scales or length differ from the resident product's");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, nm + " needs an analytic wavelet family");
  return 0;
}

extern "C++" {
// PowerCountBody over the S x n0 field W: counts against obs into cnt (may be null), selection bits
// (sel may be null)
template <typename T>
static int power_compare(cwtb_ctx *c, const void *W, const void *obs, unsigned *cnt, const SelArgs *sel, int S,
                         int64_t n0) {
  PowerCountArgs<T> a{(const cx<T> *)W, (const cx<T> *)obs, cnt, sel ? *sel : SelArgs{}, (long long)n0};
  const unsigned gx = (unsigned)((n0 + NT - 1) / NT);
  return sel ? launch<PowerCountBody<T, true>>(c, gx, (unsigned)S, a)
             : launch<PowerCountBody<T, false>>(c, gx, (unsigned)S, a);
}

// The units [unit0, unit0 + n_units) of the null, drawn as batches [nb][nser][n0]: each transformed
// with the resident product's plan, one unit at a time, W in c->W, exactly as one cwtb_cwt of it (one
// series) or one cwtb_xwt of its two series (W1 stored, W1 conj(W2) in the second transform's
// epilogue), and compared with the resident field obs: counts into cnt, or selection bits (sel)
// labelled right away, the unit's largest cluster into dqmax[i]
template <typename T>
static int test_units(cwtb_ctx *c, const TestNull &tn, const void *obs, unsigned long long seed, long long unit0,
                      int n_units, int64_t n0, double dt, const double *scales, int S, int family, double param,
                      unsigned *cnt, const SelArgs *sel, const unsigned long long *dq, unsigned long long *dqmax) {
  int e = prepare(c, n0, dt, scales, S, family, param, prec_of<T>(), nullptr);
  if (e) return e;
  const bool phase = tn.kind == CWTB_NULL_PHASE;
  const int nser = tn.nser;
  // the units of one draw: the rotated spectra of phase-randomised units take 16 B per sample
  const size_t per = (size_t)nser * n0 * (phase ? sizeof(double2) : sizeof(T));
  const int batch = (int)std::max<size_t>(
      1, std::min<size_t>({(size_t)n_units, ((size_t)256 << 20) / per, (size_t)MAX_ROWS / nser}));
  if ((e = ensure(c, c->noise, (size_t)batch * nser * n0 * sizeof(T)))) return e;
  if (phase && (e = ensure(c, c->prot, (size_t)batch * nser * n0 * sizeof(double2)))) return e;
  c->launches = 0;
  if ((e = time_begin(c))) return e;
  for (int i0 = 0; i0 < n_units; i0 += batch) {
    const int nb = std::min(batch, n_units - i0);
    T *x = (T *)c->noise.p;
    if (phase) {
      if ((e = phase_units<T>(c, tn.ph, nser, seed, unit0 + i0, nb, n0, x))) return e;
    } else {
      for (int r = 0; r < nser; ++r)
        if ((e = ar1_units<T>(c, tn.ar[r], seed, unit0 + i0, nb, n0, x + (size_t)r * n0, nser, (unsigned)r)))
          return e;
    }
    for (int i = 0; i < nb; ++i) {
      // run_job joins its streams back into c->stream, where the comparisons of successive units
      // follow each other: the counters and the selection bits have one writer at a time
      const T *u = x + (size_t)i * nser * n0;
      if ((e = run_job<T>(c, c->job, u, nullptr, EPI_STORE))) return e;
      if (nser == 2 && (e = run_job<T>(c, c->job, u + n0, nullptr, EPI_MULCONJ))) return e;
      if ((e = power_compare<T>(c, c->W.p, obs, cnt, sel, S, n0))) return e;
      if (sel && (e = label_bits(c, S, n0, dq, dqmax + i0 + i, nullptr, nullptr))) return e;
    }
  }
  if ((e = time_end(c, &c->last_ms))) return e;
  c->job_dsig = nullptr;
  return 0;
}
}  // extern "C++"

// cwtb_power_surrogate_counts / cwtb_cross_surrogate_counts on slot s, a field of nser series
static int test_counts(cwtb_ctx *c, const char *name, ResidentSlot &s, int nser, const double *series, int null,
                       const double *g, const double *m, const double *sigma, uint64_t seed, int64_t first_unit,
                       int n_units, int64_t n0, double dt, const double *scales, int n_scales, int family,
                       double param, int64_t serial, int reset) {
  if (!c) return CWTB_ERR_ARG;
  const std::string nm = name;
  int e = test_slot(c, s, nm, serial, n_scales, n0, family);
  if (e) return e;
  const long long base = reset || s.units < 0 ? 0 : s.units;
  if (n_units < 0 || n_units > 0xFFFFFFFFll - base)
    return fail(c, CWTB_ERR_ARG, nm + ": more units than a 32-bit counter holds");
  TestNull tn;
  if ((e = test_null(c, nm, series, nser, null, PHASE_GROUPS, g, m, sigma, nullptr, first_unit, n_units, n0, tn))) return e;
  if ((e = ensure(c, s.counts, (size_t)s.S * s.n0 * sizeof(unsigned)))) return e;
  s.units = -1;   // nothing readable until this call completes
  if (base == 0) RT(rt_memset(s.counts.p, 0, s.counts.bytes, c->stream));
  e = s.prec == CWTB_F32 ? test_units<float>(c, tn, s.buf.p, seed, first_unit, n_units, n0, dt, scales, n_scales,
                                             family, param, (unsigned *)s.counts.p, nullptr, nullptr, nullptr)
                         : test_units<double>(c, tn, s.buf.p, seed, first_unit, n_units, n0, dt, scales, n_scales,
                                              family, param, (unsigned *)s.counts.p, nullptr, nullptr, nullptr);
  if (e) return e;
  RT(rt_sync(c->stream));
  s.units = base + n_units;
  return 0;
}

// cwtb_power_cluster_test / cwtb_cross_cluster_test on slot s, a field of nser series
static int test_clusters(cwtb_ctx *c, const char *name, ResidentSlot &s, int nser, const double *series, int null,
                         const double *g, const double *m, const double *sigma, uint64_t seed, int64_t first_unit,
                         int n_units, int64_t n0, double dt, const double *scales, int n_scales, int family,
                         double param, int64_t serial, const double *thr, const int64_t *lo, const int64_t *hi,
                         const uint64_t *q, uint64_t *qmax_out) {
  if (!c) return CWTB_ERR_ARG;
  const std::string nm = name;
  s.clusters = false;   // nothing readable until this call completes
  s.table = ClusterTable{};
  int e = test_slot(c, s, nm, serial, n_scales, n0, family);
  if (e) return e;
  if (!thr || n_units < 0 || (n_units > 0 && !qmax_out)) return fail(c, CWTB_ERR_ARG, nm + ": bad argument");
  if ((e = cluster_shape(c, nm, n_scales, n0))) return e;
  TestNull tn;
  if ((e = test_null(c, nm, series, nser, null, PHASE_GROUPS, g, m, sigma, nullptr, first_unit, n_units, n0, tn))) return e;
  SelArgs sel;
  const unsigned long long *dq;
  if ((e = cluster_rows(c, nm, n_scales, n0, thr, lo, hi, q, sel, dq))) return e;
  if ((e = ensure(c, c->cl_qmax, (size_t)(n_units + 1) * sizeof(unsigned long long)))) return e;
  if ((e = ensure(c, s.labels, (size_t)n_scales * n0 * sizeof(int)))) return e;
  unsigned long long *dqmax = (unsigned long long *)c->cl_qmax.p;
  RT(rt_memset(dqmax, 0, (size_t)(n_units + 1) * sizeof(unsigned long long), c->stream));
  // the observed map: the comparison kernel's bits of the resident field, labelled as the units' are
  // (every launch writes whole words: no bit past the last column is ever set)
  e = s.prec == CWTB_F32 ? power_compare<float>(c, s.buf.p, nullptr, nullptr, &sel, n_scales, n0)
                         : power_compare<double>(c, s.buf.p, nullptr, nullptr, &sel, n_scales, n0);
  if (e) return e;
  ClusterTable tab;
  if ((e = label_bits(c, n_scales, n0, dq, dqmax + n_units, &tab, (int *)s.labels.p))) return e;
  e = s.prec == CWTB_F32 ? test_units<float>(c, tn, s.buf.p, seed, first_unit, n_units, n0, dt, scales, n_scales,
                                             family, param, nullptr, &sel, dq, dqmax)
                         : test_units<double>(c, tn, s.buf.p, seed, first_unit, n_units, n0, dt, scales, n_scales,
                                              family, param, nullptr, &sel, dq, dqmax);
  if (e) return e;
  if (n_units > 0) RT(rt_d2h(qmax_out, dqmax, (size_t)n_units * sizeof(unsigned long long), c->stream));
  RT(rt_sync(c->stream));
  s.table = std::move(tab);
  s.clusters = true;
  return 0;
}

int cwtb_power_surrogate_counts(cwtb_ctx *c, const double *series, int null, double g, double m, double sigma,
                                uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double dt,
                                const double *scales, int n_scales, int family, double param, int64_t serial,
                                int reset) {
  return c ? test_counts(c, "power_surrogate_counts", c->pw, 1, series, null, &g, &m, &sigma, seed, first_unit,
                         n_units, n0, dt, scales, n_scales, family, param, serial, reset)
           : CWTB_ERR_ARG;
}

int cwtb_power_cluster_test(cwtb_ctx *c, const double *series, int null, double g, double m, double sigma,
                            uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double dt,
                            const double *scales, int n_scales, int family, double param, int64_t serial,
                            const double *thr, const int64_t *lo, const int64_t *hi, const uint64_t *q,
                            uint64_t *qmax_out) {
  return c ? test_clusters(c, "power_cluster_test", c->pw, 1, series, null, &g, &m, &sigma, seed, first_unit,
                           n_units, n0, dt, scales, n_scales, family, param, serial, thr, lo, hi, q, qmax_out)
           : CWTB_ERR_ARG;
}

int cwtb_power_window(cwtb_ctx *c, int row0, int nrows, int row_step, int64_t col0, int64_t ncols, int64_t col_step,
                      double *out) {
  FieldRef f;
  int e = field_ref(c, CWTB_FIELD_POWER, f);
  if (e) return e;
  if (!out && nrows > 0 && ncols > 0) return fail(c, CWTB_ERR_ARG, "null argument");
  f.power = true;
  return window_run(c, f, row0, nrows, row_step, col0, ncols, col_step, out, nullptr);
}

int cwtb_power_pvalue_window(cwtb_ctx *c, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                             int64_t col_step, double *p_out) {
  FieldRef f;
  int e = field_ref(c, CWTB_FIELD_POWER, f);
  if (e || (e = count_ref(c, 0, f))) return e;
  if (!p_out && nrows > 0 && ncols > 0) return fail(c, CWTB_ERR_ARG, "null argument");
  return window_run(c, f, row0, nrows, row_step, col0, ncols, col_step, p_out, nullptr);
}

int cwtb_power_pvalue_row_stats(cwtb_ctx *c, const int64_t *lo, const int64_t *hi, const double *thr, int64_t kmax,
                                double *out) {
  FieldRef f;
  int e = field_ref(c, CWTB_FIELD_POWER, f);
  if (e || (e = count_ref(c, kmax, f))) return e;
  return row_stats_run(c, f, lo, hi, thr, 0, out);
}

int cwtb_power_count_hist(cwtb_ctx *c, const int64_t *lo, const int64_t *hi, int64_t nbins, int64_t *out) {
  FieldRef f;
  int e = field_ref(c, CWTB_FIELD_POWER, f);
  if (e || (e = count_ref(c, 0, f))) return e;
  return count_hist_run(c, f, lo, hi, nbins, out);
}

int cwtb_power_cluster_table(cwtb_ctx *c, int64_t cap, int64_t *count, uint64_t *Q, int64_t *points, int64_t *box) {
  int e = c ? clusters_of(c, c->pw, "power") : CWTB_ERR_ARG;
  return e ? e : table_out(c, c->pw.table, cap, count, Q, points, box);
}

int cwtb_power_cluster_labels(cwtb_ctx *c, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                              int64_t col_step, int32_t *out) {
  int e = c ? clusters_of(c, c->pw, "power") : CWTB_ERR_ARG;
  return e ? e : labels_window(c, c->pw, row0, nrows, row_step, col0, ncols, col_step, out);
}

int cwtb_power_pvalue_reconstruct(cwtb_ctx *c, const double *weights, const int64_t *lo, const int64_t *hi,
                                  const double *thr, int64_t kmax, double *out) {
  FieldRef f;
  int e = field_ref(c, CWTB_FIELD_POWER, f);
  if (e || (e = count_ref(c, kmax, f))) return e;
  return reconstruct_run(c, f, weights, lo, hi, thr, nullptr, 0, out);
}

int cwtb_power_cluster_reconstruct(cwtb_ctx *c, const double *weights, const int64_t *lo, const int64_t *hi,
                                   const int64_t *clusters, int64_t n_clusters, double *out) {
  int e = c ? clusters_of(c, c->pw, "power") : CWTB_ERR_ARG;
  if (e) return e;
  if (n_clusters < 0 || (n_clusters > 0 && !clusters)) return fail(c, CWTB_ERR_ARG, "null argument");
  // mark[label]: label c + 1 is row c of the table, label 0 is off the clusters
  const size_t nt = c->pw.table.Q.size();
  std::vector<unsigned char> mark(nt + 1, 0);
  for (int64_t i = 0; i < n_clusters; ++i) {
    if (clusters[i] < 0 || clusters[i] >= (int64_t)nt)
      return fail(c, CWTB_ERR_ARG, "power_cluster_reconstruct: no such cluster in the last cluster test");
    mark[(size_t)clusters[i] + 1] = 1;
  }
  FieldRef f;
  if ((e = field_ref(c, CWTB_FIELD_POWER, f))) return e;
  f.lab = (const int *)c->pw.labels.p;
  return reconstruct_run(c, f, weights, lo, hi, nullptr, mark.data(), mark.size(), out);
}

// ---- tests of the resident cross spectrum against surrogate pairs ---------------------------------
// the AR(1) units of nser series, series s under the tag s, out [n_units][nser][n0]
static int mc_ar1_units(cwtb_ctx *c, const std::string &nm, int nser, const double *g, const double *m,
                        const double *sigma, uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double *out) {
  if (!c) return CWTB_ERR_ARG;
  if (!out || n_units < 1 || n0 < 1) return fail(c, CWTB_ERR_ARG, nm + ": bad argument");
  TestNull tn;
  int e = test_null(c, nm, nullptr, nser, CWTB_NULL_AR1, nullptr, g, m, sigma, nullptr, first_unit, n_units, n0, tn);
  if (e) return e;
  const size_t cnt = (size_t)n_units * nser * n0;
  if ((e = ensure(c, c->noise, cnt * sizeof(double)))) return e;
  for (int i0 = 0; i0 < n_units; i0 += (int)MAX_ROWS) {
    const int nb = std::min((int)MAX_ROWS, n_units - i0);
    double *x = (double *)c->noise.p + (size_t)i0 * nser * n0;
    for (int r = 0; r < nser; ++r)
      if ((e = ar1_units<double>(c, tn.ar[r], seed, first_unit + i0, nb, n0, x + (size_t)r * n0, nser, (unsigned)r)))
        return e;
  }
  RT(rt_d2h(out, c->noise.p, cnt * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

int cwtb_mc_ar1_pair_surrogates(cwtb_ctx *c, const double *g, const double *m, const double *sigma, uint64_t seed,
                                int64_t first_unit, int n_units, int64_t n0, double *out) {
  return mc_ar1_units(c, "mc_ar1_pair_surrogates", 2, g, m, sigma, seed, first_unit, n_units, n0, out);
}

int cwtb_mc_ar1_series_surrogates(cwtb_ctx *c, int nser, const double *g, const double *m, const double *sigma,
                                  uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double *out) {
  if (c && (nser < 1 || nser > 3)) return fail(c, CWTB_ERR_ARG, "mc_ar1_series_surrogates: nser must be 1, 2 or 3");
  return mc_ar1_units(c, "mc_ar1_series_surrogates", nser, g, m, sigma, seed, first_unit, n_units, n0, out);
}

int cwtb_cross_surrogate_counts(cwtb_ctx *c, const double *series, int null, const double *g, const double *m,
                                const double *sigma, uint64_t seed, int64_t first_unit, int n_units, int64_t n0,
                                double dt, const double *scales, int n_scales, int family, double param,
                                int64_t serial, int reset) {
  return c ? test_counts(c, "cross_surrogate_counts", c->cross, 2, series, null, g, m, sigma, seed, first_unit,
                         n_units, n0, dt, scales, n_scales, family, param, serial, reset)
           : CWTB_ERR_ARG;
}

int cwtb_cross_cluster_test(cwtb_ctx *c, const double *series, int null, const double *g, const double *m,
                            const double *sigma, uint64_t seed, int64_t first_unit, int n_units, int64_t n0,
                            double dt, const double *scales, int n_scales, int family, double param, int64_t serial,
                            const double *thr, const int64_t *lo, const int64_t *hi, const uint64_t *q,
                            uint64_t *qmax_out) {
  return c ? test_clusters(c, "cross_cluster_test", c->cross, 2, series, null, g, m, sigma, seed, first_unit,
                           n_units, n0, dt, scales, n_scales, family, param, serial, thr, lo, hi, q, qmax_out)
           : CWTB_ERR_ARG;
}

int cwtb_cross_pvalue_window(cwtb_ctx *c, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                             int64_t col_step, double *p_out) {
  FieldRef f;
  int e = field_ref(c, CWTB_FIELD_CROSS, f);
  if (e || (e = count_ref(c, 0, f))) return e;
  if (!p_out && nrows > 0 && ncols > 0) return fail(c, CWTB_ERR_ARG, "null argument");
  return window_run(c, f, row0, nrows, row_step, col0, ncols, col_step, p_out, nullptr);
}

int cwtb_cross_pvalue_row_stats(cwtb_ctx *c, const int64_t *lo, const int64_t *hi, const double *thr, int64_t kmax,
                                double *out) {
  FieldRef f;
  int e = field_ref(c, CWTB_FIELD_CROSS, f);
  if (e || (e = count_ref(c, kmax, f))) return e;
  return row_stats_run(c, f, lo, hi, thr, 0, out);
}

int cwtb_cross_count_hist(cwtb_ctx *c, const int64_t *lo, const int64_t *hi, int64_t nbins, int64_t *out) {
  FieldRef f;
  int e = field_ref(c, CWTB_FIELD_CROSS, f);
  if (e || (e = count_ref(c, 0, f))) return e;
  return count_hist_run(c, f, lo, hi, nbins, out);
}

int cwtb_cross_cluster_table(cwtb_ctx *c, int64_t cap, int64_t *count, uint64_t *Q, int64_t *points, int64_t *box) {
  int e = c ? clusters_of(c, c->cross, "cross spectrum") : CWTB_ERR_ARG;
  return e ? e : table_out(c, c->cross.table, cap, count, Q, points, box);
}

int cwtb_cross_cluster_labels(cwtb_ctx *c, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                              int64_t col_step, int32_t *out) {
  int e = c ? clusters_of(c, c->cross, "cross spectrum") : CWTB_ERR_ARG;
  return e ? e : labels_window(c, c->cross, row0, nrows, row_step, col0, ncols, col_step, out);
}

int cwtb_cross_cluster_row_stats(cwtb_ctx *c, int64_t cluster, const int64_t *lo, const int64_t *hi, double *out) {
  int e = c ? clusters_of(c, c->cross, "cross spectrum") : CWTB_ERR_ARG;
  if (e) return e;
  if (cluster < 0 || cluster >= (int64_t)c->cross.table.Q.size())
    return fail(c, CWTB_ERR_ARG, "cross_cluster_row_stats: no such cluster in the last cluster test");
  FieldRef f;
  if ((e = field_ref(c, CWTB_FIELD_CROSS, f))) return e;
  f.lab = (const int *)c->cross.labels.p;
  f.want = (int)cluster + 1;
  return row_stats_run(c, f, lo, hi, nullptr, 0, out);
}

// One pass of the last cwtb_cwt_dev transform with a CUDA event pair around every launch.
// Writes one line per kernel type: "name,launches,total_ms,rows" (rows = sum of gridDim.y, i.e.
// scale rows processed) into `out`.  Returns the number of bytes written (<= cap-1) or < 0.
static int profile_report(cwtb_ctx *c, char *out, size_t cap) {
  RT(rt_sync(c->stream));
  std::map<std::string, std::array<double, 3>> agg;
  std::vector<std::string> order;
  for (auto &r : c->prof) {
    float ms = 0;
    RT(rt_elapsed_ms(&ms, c->prof_events[r.ev], c->prof_events[r.ev + 1]));
    if (!agg.count(r.name)) order.push_back(r.name);
    auto &a = agg[r.name];
    a[0] += 1; a[1] += ms; a[2] += r.gy;
  }
  std::string txt;
  char line[512];
  for (auto &n : order) {
    auto &a = agg[n];
    snprintf(line, sizeof line, "%s|%d|%.6f|%d\n", n.c_str(), (int)a[0], a[1], (int)a[2]);
    txt += line;
  }
  size_t m = std::min(cap - 1, txt.size());
  memcpy(out, txt.data(), m);
  out[m] = 0;
  return (int)m;
}

int cwtb_profile_last(cwtb_ctx *c, char *out, size_t cap) {
  if (!c || !c->job.valid || !c->job_dsig || !out || cap < 2) return fail(c, CWTB_ERR_STATE, "no transform to profile");
  c->prof.clear();
  c->profiling = true;
  int e = timed_run(c, c->job_dsig, 1, nullptr);
  c->profiling = false;
  if (e) return e;
  return profile_report(c, out, cap);
}

// Profile ANY sequence of calls (xwt, wct, wct_mc, smooth ...): between begin and end every kernel
// launch is bracketed by an event pair and the independent chains run on one stream.
int cwtb_profile_begin(cwtb_ctx *c) {
  if (!c) return CWTB_ERR_ARG;
  c->prof.clear();
  c->profiling = true;
  return 0;
}
int cwtb_profile_end(cwtb_ctx *c, char *out, size_t cap) {
  if (!c || !out || cap < 2) return CWTB_ERR_ARG;
  if (!c->profiling) return fail(c, CWTB_ERR_STATE, "profile_end without profile_begin");
  c->profiling = false;
  return profile_report(c, out, cap);
}

// Batched transform of independent channels: chunks of channels share every kernel launch
// (one descriptor row per (channel, scale)).  X: host [n_chan][n0].
// Per-row sums of |W|^2 of the resident chunk into dsum (device, R doubles, zeroed by the caller), on
// the engine's stream, no synchronisation.
static int launch_row_power(cwtb_ctx *c, double *dsum) {
  const Job &job = c->job;
  const int R = job.S * job.nbatch;
  const unsigned gx = (unsigned)((job.n0 + PowerBody<double>::PER * NT - 1) / (PowerBody<double>::PER * NT));
  if (job.precision == CWTB_F64) {
    PowerArgs<double> a{(const double2 *)c->W.p, nullptr, dsum, job.n0, nullptr, nullptr, nullptr};
    return launch<PowerBody<double>>(c, gx, R, a);
  }
  PowerArgs<float> a{(const float2 *)c->W.p, nullptr, dsum, job.n0, nullptr, nullptr, nullptr};
  return launch<PowerBody<float>>(c, gx, R, a);
}

// Spectra-only batch: chunk k+1 is copied into page-locked memory and sent to the device while the
// kernels of chunk k run; nothing synchronises until the per-row power of all chunks is read back.
static int cwt_batch_pipelined(cwtb_ctx *c, const void *X, int x_is_f32, int n_chan, int64_t n0, double dt,
                               const double *scales, int n_scales, int family, double param, int precision,
                               double *power_out, int nb) {
  const bool f32 = (precision == CWTB_F32);
  const size_t esz_in = x_is_f32 ? 4 : 8, esz = f32 ? 4 : 8;
  const size_t chunk_bytes = (size_t)nb * n0 * esz;
  int e;
  if (c->stage_bytes < chunk_bytes) {
    RT(rt_sync(c->stream));
    for (auto &p : c->stage_host) {
      if (p) RT(rt_host_free(p));
      p = nullptr;
      RT(rt_host_alloc(&p, chunk_bytes));
    }
    c->stage_bytes = chunk_bytes;
  }
  for (auto &b : c->stage_dev)
    if ((e = ensure(c, b, chunk_bytes))) return e;
  if ((e = ensure(c, c->batch_power, (size_t)n_chan * n_scales * sizeof(double)))) return e;
  double *dpow = (double *)c->batch_power.p;
  rt_stream copy = c->copy_streams[0];
  RT(rt_memset(dpow, 0, (size_t)n_chan * n_scales * sizeof(double), c->stream));
  c->launches = 0;
  int k = 0;
  for (int ch0 = 0; ch0 < n_chan; ch0 += nb, ++k) {
    const int nc = std::min(nb, n_chan - ch0), slot = k & 1;
    // (re-plans only when the chunk geometry changes: first and a shorter last chunk)
    if ((e = prepare(c, n0, dt, scales, n_scales, family, param, precision, nullptr, nc))) return e;
    if (k == 0 && (e = time_begin(c))) return e;   // behind the first plan's synchronisation
    const char *src = (const char *)X + (size_t)ch0 * n0 * esz_in;
    const size_t cnt = (size_t)nc * n0;
    const void *from = src;
    if ((x_is_f32 != 0) != f32) {   // conversion: through the page-locked staging buffer
      if (k >= 2) RT(rt_event_sync(c->ev_h2d[slot]));   // the staging buffer is free again
      if (f32) for (size_t i = 0; i < cnt; ++i) ((float *)c->stage_host[slot])[i] = (float)((const double *)src)[i];
      else for (size_t i = 0; i < cnt; ++i) ((double *)c->stage_host[slot])[i] = (double)((const float *)src)[i];
      from = c->stage_host[slot];
    }
    // (input of the engine's type: straight from the caller's pageable array -- the driver's own staged
    // copy is faster than a host memcpy into page-locked memory plus a DMA, and while it blocks this
    // thread the kernels of the previous chunk keep running)
    if (k >= 2) RT(rt_wait(copy, c->ev_used[slot]));   // chunk k-2 has consumed this device buffer
    RT(rt_h2d(c->stage_dev[slot].p, from, cnt * esz, copy));
    RT(rt_record(c->ev_h2d[slot], copy));
    RT(rt_wait(c->stream, c->ev_h2d[slot]));
    c->job_dsig = c->stage_dev[slot].p;
    c->job.sig_is_f32 = f32;
    e = f32 ? run_job<float>(c, c->job, (const float *)c->stage_dev[slot].p)
            : run_job<double>(c, c->job, (const double *)c->stage_dev[slot].p);
    if (e) return e;
    if ((e = launch_row_power(c, dpow + (size_t)ch0 * n_scales))) return e;
    RT(rt_record(c->ev_used[slot], c->stream));
  }
  if ((e = time_stop(c))) return e;
  RT(rt_d2h(power_out, dpow, (size_t)n_chan * n_scales * sizeof(double), c->stream));
  RT(rt_sync(c->stream));
  RT(rt_sync(copy));
  if ((e = time_read(c, &c->last_ms))) return e;
  for (size_t i = 0; i < (size_t)n_chan * n_scales; ++i) power_out[i] /= (double)n0;
  w_fill(c);   // the last chunk
  return 0;
}

int cwtb_cwt_batch(cwtb_ctx *c, const void *X, int x_is_f32, int n_chan, int64_t n0, double dt,
                   const double *scales, int n_scales, int family, double param, int precision,
                   double *power_out, void *W_out) {
  if (!c || !X || n_chan < 1 || n0 < 1 || n_scales < 1) return fail(c, CWTB_ERR_ARG, "cwt_batch: bad argument");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, "cwt_batch needs an analytic wavelet family");
  const bool f32 = (precision == CWTB_F32);
  const size_t esz_in = x_is_f32 ? 4 : 8, esz = f32 ? 4 : 8;
  const size_t wrow = (f32 ? 8 : 16) * (size_t)n0;
  // channels per chunk: coefficients of a chunk <= batch_bytes, rows <= 32768
  size_t per_chan = wrow * n_scales;
  int nb = (int)std::max<size_t>(1, std::min<size_t>(c->batch_bytes / std::max<size_t>(per_chan, 1), 32768 / n_scales));
  nb = std::max(1, std::min(nb, n_chan));
  if (c->batch_pipeline && power_out && !W_out && (c->pad_pow2 || (n0 & (n0 - 1)) == 0))
    return cwt_batch_pipelined(c, X, x_is_f32, n_chan, n0, dt, scales, n_scales, family, param, precision, power_out, nb);
  std::vector<unsigned char> conv;
  for (int ch0 = 0; ch0 < n_chan; ch0 += nb) {
    const int nc = std::min(nb, n_chan - ch0);
    int e = prepare(c, n0, dt, scales, n_scales, family, param, precision, nullptr, nc);
    if (e) return e;
    if ((e = ensure(c, c->sig, (size_t)nc * n0 * esz))) return e;
    const char *src = (const char *)X + (size_t)ch0 * n0 * esz_in;
    if ((x_is_f32 != 0) == f32) {
      RT(rt_h2d(c->sig.p, src, (size_t)nc * n0 * esz, c->stream));
    } else {
      conv.resize((size_t)nc * n0 * esz);
      const size_t cnt = (size_t)nc * n0;
      if (f32) for (size_t i = 0; i < cnt; ++i) ((float *)conv.data())[i] = (float)((const double *)src)[i];
      else for (size_t i = 0; i < cnt; ++i) ((double *)conv.data())[i] = (double)((const float *)src)[i];
      RT(rt_h2d(c->sig.p, conv.data(), conv.size(), c->stream));
    }
    RT(rt_sync(c->stream));
    c->job_dsig = c->sig.p;
    c->job.sig_is_f32 = f32;
    if ((e = timed_run(c, c->sig.p, 1, &c->last_ms))) return e;
    if (power_out && (e = cwtb_global_power(c, power_out + (size_t)ch0 * n_scales))) return w_kept(c, e);
    if (W_out && (e = cwtb_get_w(c, (char *)W_out + (size_t)ch0 * per_chan, 0, 0, nc * n_scales))) return w_kept(c, e);
  }
  return 0;
}

// Device-resident batched transform for benchmarks: d_X [n_chan][n0] of the engine's real
// type; all channels in one chunk (rows = n_chan * n_scales <= 60000).  W stays on the device
// (cwtb_w_device_ptr), per-row mean power is optionally copied to power_out.
int cwtb_cwt_batch_dev(cwtb_ctx *c, const void *d_X, int n_chan, int64_t n0, double dt, const double *scales,
                       int n_scales, int family, double param, int precision, double *power_out) {
  if (!c || !d_X || n_chan < 1) return fail(c, CWTB_ERR_ARG, "cwt_batch_dev: bad argument");
  if (family == CWTB_TABLE) return fail(c, CWTB_ERR_UNSUPPORTED, "cwt_batch needs an analytic wavelet family");
  int e = prepare(c, n0, dt, scales, n_scales, family, param, precision, nullptr, n_chan);
  if (e) return e;
  c->job_dsig = d_X;
  c->job.sig_is_f32 = (precision == CWTB_F32);
  if ((e = timed_run(c, d_X, 1, &c->last_ms))) return e;
  return power_out ? w_kept(c, cwtb_global_power(c, power_out)) : 0;
}


// ======================================================================================
// Multi-GPU collectives (SURVEY 8b vii / 8e): one context per GPU and process, an NCCL
// communicator owned by the context.  NCCL is bound at run time (dlopen of libnccl.so.2), so the
// library has no link-time dependency and single-GPU users never touch it.  The data path of the
// transform needs no collective (channels / scales / surrogate pairs are independent); what
// crosses NVLink are the REDUCED products: per-row spectra (all-gather), Monte-Carlo histograms
// (all-reduce), timings (max).  Buffers are host arrays staged through context-owned device
// memory: sizes are O(channels x scales), a few MB.
// ======================================================================================
namespace {
typedef struct { char internal[128]; } nccl_uid;
struct NcclApi {
  void *h = nullptr;
  int (*GetUniqueId)(nccl_uid *) = nullptr;
  int (*CommInitRank)(void **, int, nccl_uid, int) = nullptr;
  int (*CommDestroy)(void *) = nullptr;
  int (*AllGather)(const void *, void *, size_t, int, void *, rt_stream) = nullptr;
  int (*AllReduce)(const void *, void *, size_t, int, int, void *, rt_stream) = nullptr;
  int (*Broadcast)(const void *, void *, size_t, int, int, void *, rt_stream) = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
  bool ok = false;
};
NcclApi &nccl_api() {
  static NcclApi a;
  static std::mutex m;   // contexts of several host threads may bind NCCL at the same time
  std::lock_guard<std::mutex> lock(m);
  if (a.h) return a;
#ifndef CWTB_HOST_EMU   // the emulation binds nothing: it has no device buffers to hand NCCL
  for (const char *name : {"libnccl.so.2", "libnccl.so"}) {
    a.h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
    if (a.h) break;
  }
#endif
  if (!a.h) return a;
  a.GetUniqueId = (int (*)(nccl_uid *))dlsym(a.h, "ncclGetUniqueId");
  a.CommInitRank = (int (*)(void **, int, nccl_uid, int))dlsym(a.h, "ncclCommInitRank");
  a.CommDestroy = (int (*)(void *))dlsym(a.h, "ncclCommDestroy");
  a.AllGather = (int (*)(const void *, void *, size_t, int, void *, rt_stream))dlsym(a.h, "ncclAllGather");
  a.AllReduce = (int (*)(const void *, void *, size_t, int, int, void *, rt_stream))dlsym(a.h, "ncclAllReduce");
  a.Broadcast = (int (*)(const void *, void *, size_t, int, int, void *, rt_stream))dlsym(a.h, "ncclBroadcast");
  a.GetErrorString = (const char *(*)(int))dlsym(a.h, "ncclGetErrorString");
  a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.AllGather && a.AllReduce && a.Broadcast;
  return a;
}
enum { NCCL_CHAR = 0, NCCL_INT64 = 4, NCCL_FLOAT64 = 8, NCCL_SUM = 0, NCCL_MAX = 2 };
}  // namespace
#define NCCLCHK(call)                                                                               \
  do {                                                                                              \
    int r_ = (call);                                                                                \
    if (r_ != 0)                                                                                    \
      return fail(c, CWTB_ERR_COMM, std::string(#call) + ": " +                                     \
                                        (nccl_api().GetErrorString ? nccl_api().GetErrorString(r_) : "NCCL error")); \
  } while (0)

int cwtb_comm_unique_id(void *id128) {
  if (!id128) return CWTB_ERR_ARG;
  NcclApi &a = nccl_api();
  if (!a.ok) return CWTB_ERR_COMM;
  return a.GetUniqueId((nccl_uid *)id128) == 0 ? 0 : CWTB_ERR_COMM;
}

int cwtb_comm_init(cwtb_ctx *c, int world, int rank, const void *id128) {
  if (!c || !id128 || world < 1 || rank < 0 || rank >= world) return fail(c, CWTB_ERR_ARG, "comm_init: bad argument");
  cwtb_comm_destroy(c);
  c->comm_world = world;
  c->comm_rank = rank;
  if (world == 1) return 0;
  NcclApi &a = nccl_api();
  if (!a.ok) return fail(c, CWTB_ERR_COMM, "libnccl.so.2 could not be loaded");
  RT(rt_set_device(c->device));
  nccl_uid id;
  memcpy(&id, id128, sizeof id);
  NCCLCHK(a.CommInitRank(&c->comm, world, id, rank));
  return 0;
}

int cwtb_comm_destroy(cwtb_ctx *c) {
  if (!c) return CWTB_ERR_ARG;
  if (c->comm) {
    rt_set_device(c->device);
    rt_sync(c->stream);
    nccl_api().CommDestroy(c->comm);
    c->comm = nullptr;
  }
  c->comm_world = 1;
  c->comm_rank = 0;
  return 0;
}

int cwtb_comm_world(cwtb_ctx *c) { return c ? c->comm_world : -1; }
int cwtb_comm_rank(cwtb_ctx *c) { return c ? c->comm_rank : -1; }

// recv[r * bytes .. (r+1) * bytes) = rank r's send, for every rank (host buffers)
int cwtb_comm_allgather(cwtb_ctx *c, const void *send, void *recv, size_t bytes) {
  if (!c || !send || !recv) return fail(c, CWTB_ERR_ARG, "allgather: null argument");
  if (c->comm_world == 1) { memmove(recv, send, bytes); return 0; }
  if (!c->comm) return fail(c, CWTB_ERR_COMM, "no communicator");
  int e;
  RT(rt_set_device(c->device));
  if ((e = ensure(c, c->comm_send, bytes))) return e;
  if ((e = ensure(c, c->comm_recv, bytes * c->comm_world))) return e;
  RT(rt_h2d(c->comm_send.p, send, bytes, c->stream));
  NCCLCHK(nccl_api().AllGather(c->comm_send.p, c->comm_recv.p, bytes, NCCL_CHAR, c->comm, c->stream));
  RT(rt_d2h(recv, c->comm_recv.p, bytes * c->comm_world, c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

static int comm_allreduce(cwtb_ctx *c, void *buf, size_t count, int dtype, int op) {
  if (!c || !buf) return fail(c, CWTB_ERR_ARG, "allreduce: null argument");
  if (c->comm_world == 1) return 0;
  if (!c->comm) return fail(c, CWTB_ERR_COMM, "no communicator");
  int e;
  RT(rt_set_device(c->device));
  if ((e = ensure(c, c->comm_send, count * 8))) return e;
  RT(rt_h2d(c->comm_send.p, buf, count * 8, c->stream));
  NCCLCHK(nccl_api().AllReduce(c->comm_send.p, c->comm_send.p, count, dtype, op, c->comm, c->stream));
  RT(rt_d2h(buf, c->comm_send.p, count * 8, c->stream));
  RT(rt_sync(c->stream));
  return 0;
}
int cwtb_comm_allreduce_sum_i64(cwtb_ctx *c, int64_t *buf, size_t count) {
  return comm_allreduce(c, buf, count, NCCL_INT64, NCCL_SUM);
}
int cwtb_comm_allreduce_max_f64(cwtb_ctx *c, double *buf, size_t count) {
  return comm_allreduce(c, buf, count, NCCL_FLOAT64, NCCL_MAX);
}
int cwtb_comm_broadcast(cwtb_ctx *c, void *buf, size_t bytes, int root) {
  if (!c || !buf || root < 0 || root >= c->comm_world) return fail(c, CWTB_ERR_ARG, "broadcast: bad argument");
  if (c->comm_world == 1) return 0;
  if (!c->comm) return fail(c, CWTB_ERR_COMM, "no communicator");
  int e;
  RT(rt_set_device(c->device));
  if ((e = ensure(c, c->comm_send, bytes))) return e;
  if (c->comm_rank == root) RT(rt_h2d(c->comm_send.p, buf, bytes, c->stream));
  NCCLCHK(nccl_api().Broadcast(c->comm_send.p, c->comm_send.p, bytes, NCCL_CHAR, root, c->comm, c->stream));
  RT(rt_d2h(buf, c->comm_send.p, bytes, c->stream));
  RT(rt_sync(c->stream));
  return 0;
}

}  // extern "C"
