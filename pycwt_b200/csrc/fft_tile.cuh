// Batched K-point FFT on a [P][K] tile: the compute core shared by every kernel
// of the engine.
//
// One CTA (NT threads) owns a tile of P independent K-point transforms
// (P * K = TILE elements).  The transform is an in-place decimation-in-frequency
// mixed-radix FFT with radices (R1, R2, R3) taken from Plan<K>:
//
//   * every pass but the last:  lanes run over the position inside the transform,
//     each thread LOOPS over the batch index b with the pass twiddles held in
//     registers (loaded once per thread, reused for all its b);
//   * the last pass is twiddle-free and its lanes run over b, so that the results
//     leave the CTA straight from registers as P*sizeof(complex)-byte contiguous
//     segments (b is the contiguous index in global memory for every output
//     layout the engine uses);
//   * between passes the tile lives in shared memory; a thread reads and writes
//     the same positions in a pass (in-place), so only one barrier per pass.
//
// After the passes, output index q of a transform is  q = c1 + R1*(c2 + R2*c3)
// where c_i is the output digit of pass i (digit reversal is absorbed by the
// final global store).
//
// All functions take the thread id as an argument and are __host__ __device__:
// tests emulate a CTA on the CPU by looping over tid phase by phase.
#pragma once
#include "cplx.cuh"

namespace cwtb {

#ifndef CWTB_NT
#define CWTB_NT 128       // threads per CTA of the fp64 tile kernels and of every element-wise kernel
#endif
#ifndef CWTB_NT_F32
#define CWTB_NT_F32 256   // threads per CTA of the fp32 tile kernels (measured +10..18 % over 128)
#endif
#ifndef CWTB_TILE_F64
#define CWTB_TILE_F64 4096
#endif
#ifndef CWTB_TILE_F32
#define CWTB_TILE_F32 8192
#endif
#ifndef CWTB_MINB
#define CWTB_MINB 1
#endif
#ifndef CWTB_UNROLL_B
#define CWTB_UNROLL_B 1
#endif
#define CWTB_STR_(x) #x
#define CWTB_STR(x) CWTB_STR_(x)
#define CWTB_PRAGMA_UNROLL_B _Pragma(CWTB_STR(unroll CWTB_UNROLL_B))
#ifndef CWTB_PASSA_BATCH
#define CWTB_PASSA_BATCH 8     // spectrum loads in flight per thread while a dense first-kernel tile is filled
#endif
#ifndef CWTB_UNROLL_A
#define CWTB_UNROLL_A 4        // loads in flight per thread while a band / row tile of the first kernel is filled
#endif
#define CWTB_PRAGMA_UNROLL_A _Pragma(CWTB_STR(unroll CWTB_UNROLL_A))
constexpr int NT = CWTB_NT;  // threads per CTA
// Pass twiddle tables: for a pass of radix R on sub-transforms of length L the factor
// w_L^{j c} (c = 1..R-1, j < L/R) is stored at  tw[tw_offset(L) + (c-1)*(L/R) + j], i.e. lanes
// (consecutive j) read consecutive entries.  Each L has one radix in the plans below.
#ifndef CWTB_PLAN1024_R32
#define CWTB_PLAN1024_R32 0
#endif
#ifndef CWTB_PLAN256_3PASS
#define CWTB_PLAN256_3PASS 1
#endif
HD constexpr int tw_radix(int L) {
  return L == 32 ? 4 : (L == 256 ? (CWTB_PLAN256_3PASS ? 4 : 16) : ((L == 1024 && CWTB_PLAN1024_R32) ? 32 : 8));
}
HD constexpr int tw_count(int L) { return (tw_radix(L) - 1) * (L / tw_radix(L)); }
HD constexpr int tw_offset(int L) {
  return L == 32 ? 0 : (L == 64 ? tw_count(32) : tw_offset(L / 2) + tw_count(L / 2));
}
constexpr int TW_TOTAL = tw_offset(1024) + tw_count(1024);
constexpr int K2C = 1024;   // length of the second-pass transform (two-kernel scales)

template <typename T> struct TileCfg {
  static constexpr int TILE = sizeof(T) == 8 ? CWTB_TILE_F64 : CWTB_TILE_F32;  // elements per CTA
  static constexpr int NT = sizeof(T) == 8 ? CWTB_NT : CWTB_NT_F32;            // threads per CTA
  static constexpr int Q = 128 / (2 * (int)sizeof(T));       // lanes per smem conflict domain
};

template <int K> struct Plan;
#define CWTB_PLAN(K_, A_, B_, C_)                                                   \
  template <> struct Plan<K_> {                                                     \
    static constexpr int R1 = A_, R2 = B_, R3 = C_;                                 \
    static constexpr int NP = (B_ == 1) ? 1 : ((C_ == 1) ? 2 : 3);                  \
    static constexpr int RL = (NP == 1) ? A_ : ((NP == 2) ? B_ : C_); /* last */    \
    HD static int qlow(int g) {                                                     \
      return NP == 3 ? (g / B_) + A_ * (g % B_) : (NP == 2 ? g : 0);                \
    }                                                                               \
  };
CWTB_PLAN(2, 2, 1, 1)
CWTB_PLAN(4, 4, 1, 1)
CWTB_PLAN(8, 8, 1, 1)
CWTB_PLAN(16, 16, 1, 1)
CWTB_PLAN(32, 4, 8, 1)
CWTB_PLAN(64, 8, 8, 1)
CWTB_PLAN(128, 8, 16, 1)
#if CWTB_PLAN256_3PASS
CWTB_PLAN(256, 4, 8, 8)
#else
CWTB_PLAN(256, 16, 16, 1)
#endif
CWTB_PLAN(512, 8, 8, 8)
#if CWTB_PLAN1024_R32
CWTB_PLAN(1024, 32, 32, 1)
#else
CWTB_PLAN(1024, 8, 8, 16)
#endif
#undef CWTB_PLAN

// Shared-memory layout of the tile: [b][pos] with a row pitch chosen so that both
// access patterns (lanes over pos, lanes over b) are bank-conflict free.
template <typename T, int K, bool ROWS = false> struct Lay {
  static constexpr int TILE = TileCfg<T>::TILE;
  static constexpr int P = TILE / K;
  static constexpr int Q = TileCfg<T>::Q;
  // For P < Q one pad element is inserted after every 16 positions (pos + pos/16), which shifts
  // the second position of a quarter-warp onto the free bank groups -> conflict-free in every
  // pass.  ROWS = true marks tiles whose rows are filled by bulk-async (TMA) copies: with the
  // skew a row arrives as K/16 copies of 16 elements (CHUNKED); that needs 16-byte aligned
  // chunk starts, i.e. 16-byte elements (fp64) -- fp32 row tiles stay unskewed (one contiguous
  // copy per row, 2-way conflict on the last pass's reads when P = Q/2).
#ifndef CWTB_ROWS_SKEW
#define CWTB_ROWS_SKEW 0
#endif
  static constexpr bool SKEW = (P < Q) && (!ROWS || (CWTB_ROWS_SKEW && sizeof(T) == 8));
  static constexpr bool CHUNKED = ROWS && SKEW;
  static constexpr int KS = SKEW ? K + K / 16 : K;
  static constexpr int PITCH = (P < Q) ? (KS - (KS % Q) + 2 + ((KS % Q) > 2 ? Q : 0)) : K + 1;
  static constexpr int ELEMS = P * PITCH;
  static constexpr size_t TILE_BYTES = (size_t)ELEMS * 2 * sizeof(T);
  static constexpr size_t BYTES = (Plan<K>::NP == 1) ? 0 : TILE_BYTES;
  HD static int phys(int b, int pos) { return b * PITCH + pos + (SKEW ? (pos >> 4) : 0); }
};

// ---- bulk asynchronous copy (TMA, cp.async.bulk) global -> shared with an mbarrier --------
// One thread arms the barrier with the expected byte count and issues the copies; every
// thread then waits on the barrier's phase.  Host emulation: plain memcpy, wait is a no-op.
HD void warp_sync() {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  __syncwarp();
#endif
}

#ifdef CWTB_HOST_EMU
inline long long &emu_bulk_copy_faults() {   // misaligned bulk copies seen by the emulation
  static long long n = 0;
  return n;
}
#endif

struct TileBarrier {
  unsigned long long *bar;  // 8-byte slot in shared memory
  HD void init_and_expect(unsigned bytes) const {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
    const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(a) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(a), "r"(bytes) : "memory");
#else
    (void)bytes;
#endif
  }
  // dst (shared) and src (global) 16-byte aligned, bytes a multiple of 16
  HD void copy(void *dst, const void *src, unsigned bytes) const {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
    const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(d), "l"(src), "r"(bytes), "r"(a) : "memory");
#else
    // the hardware requirement, checked where no GPU is present: the emulation's shared
    // memory base is 16-byte aligned, so offsets are what is being tested
#ifdef CWTB_HOST_EMU
    if ((((unsigned long long)dst | (unsigned long long)src | bytes) & 15ull) != 0) ++emu_bulk_copy_faults();
#endif
    const char *s_ = (const char *)src;
    char *d_ = (char *)dst;
    for (unsigned i = 0; i < bytes; ++i) d_[i] = s_[i];
#endif
  }
  // fire-and-forget prefetch of a global range into L2 (no barrier involved)
  HD static void prefetch_l2(const void *src, unsigned bytes) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
#else
    (void)src; (void)bytes;
#endif
  }
  HD void inval() const {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
    const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
    asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(a) : "memory");
#endif
  }
  HD void wait(unsigned parity) const {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
    const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
    unsigned done = 0;
    while (!done) {
      asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                   "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(a), "r"(parity) : "memory");
    }
#else
    (void)parity;
#endif
  }
};

// Ampere-style asynchronous copy global -> shared of one element (8 or 16 bytes) that bypasses the
// register file: a thread can have its whole share of a tile in flight at once instead of
// compiler-sized batches of loads followed by stores.  Off by default for the first kernel of the band
// scales: the element-wise LDGSTS scatter costs more than the extra loads in flight gain, against
// batches of four LDG.128 + STS.128 (CWTB_PASSA_ASYNC=1 builds it in).  cp_async_wait() makes the thread's own
// copies visible to itself; the CTA barrier that follows publishes them.  Host emulation: plain copy.
#ifndef CWTB_PASSA_ASYNC
#define CWTB_PASSA_ASYNC 0
#endif
template <typename V> HD void cp_async(V *dst, const V *src) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  static_assert(sizeof(V) == 16 || sizeof(V) == 8, "cp_async: 8- or 16-byte elements");
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  if constexpr (sizeof(V) == 16)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src) : "memory");
  else
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(src) : "memory");
#else
  *dst = *src;
#endif
}
HD void cp_async_wait() {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  asm volatile("cp.async.wait_all;" ::: "memory");
#endif
}

template <typename V> HD V ldg(const V *p) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  return __ldg(p);
#else
  return *p;
#endif
}

// streaming (evict-first) store for results that are never re-read by the engine
template <typename V> HD void st_stream(V *p, V v) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  __stcs(p, v);
#else
  *p = v;
#endif
}

// e^{2 pi i e / N} from a two-level table (N a power of two): hi[e >> h] * lo[e & mask].
struct NTab {
  const double2 *hi;
  const double2 *lo;
  int h;
  unsigned lomask;
  unsigned nmask;  // N - 1
};
HD double2 nroot(const NTab &t, unsigned e) {
  e &= t.nmask;
  return cmul(ldg(&t.hi[e >> t.h]), ldg(&t.lo[e & t.lomask]));
}
template <typename T> HD cx<T> nroot_t(const NTab &t, unsigned e) {
  double2 w = nroot(t, e);
  return mk<T>((T)w.x, (T)w.y);
}

// ---- loaders for the first pass (template on radix R) -------------------------
// Interface:  begin(base, stride, bstart, bstep);  load(b, x[R])
//   the R inputs of the butterfly sit at positions base + i*stride.

template <typename T, int K, bool ROWS = false> struct SmemLoader {
  using V = cx<T>;
  const V *sm;
  int base, stride;
  HD void begin(int base_, int stride_, int, int) { base = base_; stride = stride_; }
  template <int R> HD void load(int b, V (&x)[R]) const {
#pragma unroll
    for (int i = 0; i < R; ++i) x[i] = sm[Lay<T, K, ROWS>::phys(b, base + i * stride)];
  }
};

// shared-memory tile whose rows still need the first-kernel twist
//   e^{2 pi i k1 p / (K1 M)} = e^{2 pi i (k1 p K2) / N},  k1 = pos - K [pos*K2 >= rsplit],
// applied while loading: the R factors of a thread do not depend on b, so they live in registers
// (one per-lane table lookup, the rest by multiplying with warp-uniform steps).
template <typename T, int K, int R> struct SmemTwistLoader {
  using V = cx<T>;
  const V *sm;
  NTab nt;
  int rsplit_row;   // first row (pos) whose residues are >= rsplit  (rsplit is a multiple of K2)
  unsigned pk2;     // p * K2
  int base, stride;
  V tw[R];
  HD void begin(int base_, int stride_, int, int) {
    base = base_; stride = stride_;
    V e = nroot_t<T>(nt, (unsigned)base * pk2);
    const V se = nroot_t<T>(nt, (unsigned)stride * pk2);
    const V ne = nroot_t<T>(nt, (unsigned)(-K) * pk2);
#pragma unroll
    for (int i = 0; i < R; ++i) {
      tw[i] = (base + i * stride >= rsplit_row) ? cmul(e, ne) : e;
      e = cmul(e, se);
    }
  }
  HD void load(int b, V (&x)[R]) const {
#pragma unroll
    for (int i = 0; i < R; ++i) x[i] = cmul(sm[Lay<T, K>::phys(b, base + i * stride)], tw[i]);
  }
};

// rows of a [rows][K] global array (second-pass kernel: Z[u][r2])
template <typename T, int K> struct RowLoader {
  using V = cx<T>;
  const V *src;   // already offset to row u0
  int nvalid;     // rows available from u0
  int base, stride;
  HD void begin(int base_, int stride_, int, int) { base = base_; stride = stride_; }
  template <int R> HD void load(int b, V (&x)[R]) const {
    if (b < nvalid) {
      const V *row = src + (size_t)b * K + base;
#pragma unroll
      for (int i = 0; i < R; ++i) x[i] = row[i * stride];
    } else {
#pragma unroll
      for (int i = 0; i < R; ++i) x[i] = mk<T>(0, 0);
    }
  }
};

// pruned-band generator: a_p[r] = B[r] * e^{2 pi i k p / N}, p = p0 + b, advanced by
// recurrence over b (a <- a * delta, delta = e^{2 pi i k bstep / N}).
template <typename T, int K, int R> struct GenLoader {
  using V = cx<T>;
  static constexpr int P = Lay<T, K>::P;
  static constexpr int I = K / R;
  static constexpr int NT = TileCfg<T>::NT;
  static constexpr int GROUPS = (I >= NT) ? 1 : NT / I;
  static constexpr bool ONE_SHOT = (P / GROUPS <= 1);   // one batch index per thread: no recurrence
  const V *B;      // K entries, residue order
  NTab nt;
  int rsplit;      // r >= rsplit  ->  k = r - K
  unsigned p0;
  V a[ONE_SHOT ? 1 : R], d[ONE_SHOT ? 1 : R];
  int base, stride;
  unsigned pp;
  // Phase factors e^{2 pi i k_i p / N} (p = the thread's first index) and the per-step
  // multipliers e^{2 pi i k_i bstep / N} for the R residues r_i = base + i*stride, signed bins
  // k_i = r_i - K [r_i >= rsplit].  Only the i = 0 factors need a per-lane table lookup; the
  // others follow by multiplying with warp-uniform steps (broadcast loads), which keeps the
  // scattered 16-byte gathers off the LSU pipe.
  HD void begin(int base_, int stride_, int bstart, int bstep) {
    base = base_; stride = stride_;
    pp = p0 + (unsigned)bstart;
    if (ONE_SHOT) return;
    V e = nroot_t<T>(nt, (unsigned)base * pp);
    V de = nroot_t<T>(nt, (unsigned)base * (unsigned)bstep);
    const V se = nroot_t<T>(nt, (unsigned)stride * pp);
    const V sd = nroot_t<T>(nt, (unsigned)stride * (unsigned)bstep);
    const V ne = nroot_t<T>(nt, (unsigned)(-K) * pp);
    const V nd = nroot_t<T>(nt, (unsigned)(-K) * (unsigned)bstep);
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const int r = base + i * stride;
      const bool neg = r >= rsplit;
      d[ONE_SHOT ? 0 : i] = neg ? cmul(de, nd) : de;
      a[ONE_SHOT ? 0 : i] = cmul(ldg(&B[r]), neg ? cmul(e, ne) : e);
      e = cmul(e, se);
      de = cmul(de, sd);
    }
  }
  HD void load(int, V (&x)[R]) {
    if (ONE_SHOT) {
      V e = nroot_t<T>(nt, (unsigned)base * pp);
      const V se = nroot_t<T>(nt, (unsigned)stride * pp);
      const V ne = nroot_t<T>(nt, (unsigned)(-K) * pp);
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const int r = base + i * stride;
        x[i] = cmul(ldg(&B[r]), (r >= rsplit) ? cmul(e, ne) : e);
        e = cmul(e, se);
      }
      return;
    }
#pragma unroll
    for (int i = 0; i < R; ++i) { x[i] = a[ONE_SHOT ? 0 : i]; a[ONE_SHOT ? 0 : i] = cmul(a[ONE_SHOT ? 0 : i], d[ONE_SHOT ? 0 : i]); }
  }
};

// ---- passes --------------------------------------------------------------------
// One non-final pass on sub-transforms of length L (K/L of them per row).
template <typename T, int K, int L, int R, int SIGN, class Loader, bool ROWS = false>
HD void pass_mid(cx<T> *sm, const cx<T> *__restrict__ tw, Loader &ld, int tid) {
  using V = cx<T>;
  using LY = Lay<T, K, ROWS>;
  constexpr int NT = TileCfg<T>::NT;
  constexpr int Ln = L / R, I = K / R, P = LY::P;
  constexpr int LANES = (I >= NT) ? NT : I;
  constexpr int GROUPS = NT / LANES;
  const int tp0 = tid % LANES, bg = tid / LANES;
  for (int tp = tp0; tp < I; tp += LANES) {
    const int g = tp / Ln, j = tp % Ln;
    V twv[R];
#pragma unroll
    static_assert(tw_radix(L) == R, "pass twiddle table was built for another radix");
    for (int c = 1; c < R; ++c) {
      V w = ldg(&tw[tw_offset(L) + (c - 1) * Ln + j]);
      if (SIGN < 0) w.y = -w.y;
      twv[c] = w;
    }
    ld.begin(g * L + j, Ln, bg, GROUPS);
    CWTB_PRAGMA_UNROLL_B
    for (int b = bg; b < P; b += GROUPS) {
      V x[R];
      ld.load(b, x);
      dftR<R, SIGN, T>(x);
#pragma unroll
      for (int c = 1; c < R; ++c) x[c] = cmul(x[c], twv[c]);
#pragma unroll
      for (int c = 0; c < R; ++c) sm[LY::phys(b, g * L + c * Ln + j)] = x[c];
    }
  }
}

// Final pass: radix R = Plan<K>::RL on K/R sub-transforms per row, lanes over b.
// Storer interface: store(b, qlow, qstride, x[R])  with output index q = qlow + c*qstride.
template <typename T, int K, int SIGN, class Storer, bool ROWS = false>
HD void pass_last(const cx<T> *sm, Storer &st, int tid) {
  using V = cx<T>;
  using LY = Lay<T, K, ROWS>;
  constexpr int NT = TileCfg<T>::NT;
  constexpr int R = Plan<K>::RL, G = K / R, P = LY::P;
  for (int idx = tid; idx < G * P; idx += NT) {
    const int b = idx % P, g = idx / P;
    V x[R];
#pragma unroll
    for (int i = 0; i < R; ++i) x[i] = sm[LY::phys(b, g * R + i)];
    dftR<R, SIGN, T>(x);
    st.store(b, Plan<K>::qlow(g), G, x);
  }
}

// Runs passes [first .. last) of the plan that go through shared memory.
// phase 0: first pass (with the caller's loader); phase 1: second pass (3-pass plans);
// final phase: pass_last.  Returns nothing; the caller inserts barriers between phases.
template <typename T, int K> struct TilePhases {
  static constexpr int NP = Plan<K>::NP;  // number of phases of the multi-pass core
};

template <typename T, int K, int SIGN, class Loader, bool ROWS = false>
HD void tile_first(cx<T> *sm, const cx<T> *tw, Loader &ld, int tid) {
  pass_mid<T, K, K, Plan<K>::R1, SIGN, Loader, ROWS>(sm, tw, ld, tid);
}
template <typename T, int K, int SIGN, bool ROWS = false>
HD void tile_second(cx<T> *sm, const cx<T> *tw, int tid) {  // only for 3-pass plans
  SmemLoader<T, K, ROWS> ld;
  ld.sm = sm;
  pass_mid<T, K, K / Plan<K>::R1, Plan<K>::R2, SIGN, SmemLoader<T, K, ROWS>, ROWS>(sm, tw, ld, tid);
}

}  // namespace cwtb
