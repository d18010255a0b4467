// Kernel bodies of the CWT engine.  Every kernel is a `Body` struct with
//   Args, NPHASE, SMEM (bytes), and  template<int PH> phase(args, bx, by, tid, smem)
// Phases are separated by a CTA barrier.  The generic __global__ wrapper lives in
// engine.cu; tests/emu runs the same phases sequentially on the CPU.
#pragma once
#include <math.h>
#include "fft_tile.cuh"

namespace cwtb {

// ---- per-scale descriptor (host-planned, read by the kernels) -------------------
struct ScaleDesc {
  double s;        // scale s_j
  double amp;      // sqrt(s*w1*Np) * family constant / Np
  int row;         // output row of W (after NaN-row removal, done by the host)
  int k_lo, k_hi;  // signed band limits (inclusive) outside which psi_ft is treated as 0
  int log2K;       // pruned transform length K' = 1 << log2K  (K' == Np: dense)
  int rsplit;      // residue r >= rsplit  <->  signed bin k = r - K'
  int trow;        // row in the caller's psi_ft table (CWTB_TABLE family)
  int chan;        // channel of a batched transform: spectrum at spec + chan*Np
  int pad_;
  long long boff;  // offset of this scale's band product B[] in the band buffer
  // ---- band-limited expansion path (ip_log2Nc > 0; see ExpandBody) ----
  int ip_log2Nc;   // coarse grid length Nc = 1 << ip_log2Nc  (0: exact pruned-transform path)
  int ip_kc;       // centre bin of the band (signed): the coarse grid holds the band shifted to 0
  int ip_w;        // taps of the interpolation kernel
  int os_grp;      // overlap-save group + 1 (OsBody; 0: another path)
  long long ip_coff;   // offset of this row's Nc coarse samples in the coarse buffers
  long long ip_woff;   // offset of the [taps][R] weight table of this row's class
  double ip_beta;      // Kaiser-Bessel shape parameter
  double ip_dc;        // I0(beta) / taps: 1 / (transform of the kernel) = ip_dc * z / sinh(z)
};

struct Fam {
  int family;      // 0 Morlet, 1 Paul, 2 DOG, 3 table, 4 Morse
  int m;           // order (Paul, DOG)
  int unit;        // multiply by i^unit  (conj(-(1j**m)) for DOG)
  int pad_;
  double f0;       // Morlet wavenumber
  double dw;       // 1 / (Np * dt)   (numpy fftfreq's `val`)
  const double2 *table;  // [S][Np] complex128: sqrt(s*w1*Np)*conj(psi_ft)  (family 3)
  long long tpitch;
  // Morse (family 4): psi_ft(f) / psi_ft(f_p) = exp(be u - (be/ga) expm1(ga u)), u = ln(f / f_p),
  // f_p = (be/ga)^(1/ga) the peak; the family constant psi_ft(f_p) is folded into ScaleDesc::amp
  double be, ga;
  double lnfp;     // ln f_p
  double bg;       // be / ga  (= f_p^ga)
};

HD double ipow(double f, int m) {
  double r = 1.0, b = f;
  int e = m < 0 ? -m : m;
  while (e) { if (e & 1) r *= b; b *= b; e >>= 1; }
  return m < 0 ? 1.0 / r : r;
}

// |conj(psi_ft(s*w_k))| without the family constant; pycwt/mothers.py:26-28,118-122,170-173.
// w_k is formed as numpy does: 2*pi * (k * (1/(Np*dt))).
// (MORSE = false: the Morse branch is compiled out, for kernels that never see a Morse row; see BandBody)
template <bool MORSE = true> HD double amp_eval(const Fam &fp, double s, int k) {
  const double w = 6.283185307179586 * ((double)k * fp.dw);
  const double f = s * w;
  if (fp.family == 0) {
    const double d = f - fp.f0;
    return exp(-0.5 * d * d);
  } else if (fp.family == 1) {
    return f > 0.0 ? ipow(f, fp.m) * exp(-f) : 0.0;
  } else if (MORSE && fp.family == 4) {
    // peak-relative log form: no power of f is formed, so a large be never gives inf * 0
    if (!(f > 0.0)) return 0.0;
    const double u = log(f) - fp.lnfp;
    return exp(fp.be * u - fp.bg * expm1(fp.ga * u));
  } else {
    return ipow(f, fp.m) * exp(-0.5 * f * f);
  }
}

// the same in the engine's arithmetic: the fp32 engine forms f = s*w in double (w spans 2^18 bins)
// and evaluates the power and the exponential in float (the caller keeps orders above 8 in double:
// their powers overflow float).  fp64 instructions run at half the fp32 rate on H100: one double exp per band product
// would make the band-product launches and the generating first kernel fp64-pipe bound in the fp32 engine.
template <typename T, bool MORSE = true> HD T amp_eval_t(const Fam &fp, double s, int k) {
  if constexpr (sizeof(T) == 8) {
    return amp_eval<MORSE>(fp, s, k);
  } else {
    const double w = 6.283185307179586 * ((double)k * fp.dw);
    const double f = s * w;
    if (fp.family == 0) {
      const float d = (float)(f - fp.f0);
      return expf(-0.5f * d * d);
    }
    const float ff = (float)f;
    float r = 1.0f, b = ff;
    for (int e = fp.m; e; e >>= 1) { if (e & 1) r *= b; b *= b; }
    if (fp.family == 1) return ff > 0.0f ? r * expf(-ff) : 0.0f;
    return r * expf(-0.5f * ff * ff);
  }
}

template <typename T> HD cx<T> rot_unit(cx<T> v, int unit) {
  switch (unit & 3) {
    case 1: return mk<T>(-v.y, v.x);
    case 2: return mk<T>(-v.x, -v.y);
    case 3: return mk<T>(v.y, -v.x);
    default: return v;
  }
}

// value of x^[bin] * conj(psi_ft)(s, k) * norm / Np  for one scale
template <typename T, bool MORSE = true>
HD cx<T> band_value(const Fam &fp, const ScaleDesc &d, const cx<T> *spec, unsigned bin, int k, unsigned N) {
  cx<T> v = ldg(&spec[(size_t)d.chan * N + bin]);
  if (fp.family == 3) {
    double2 t = ldg(&fp.table[(size_t)d.trow * fp.tpitch + bin]);
    cx<T> tt = mk<T>((T)(t.x * d.amp), (T)(t.y * d.amp));
    return cmul(v, tt);
  }
  // (Paul / DOG orders above 8: value and normalisation only combine to a float-range number in
  // double.  Morse too is evaluated in double in the fp32 engine: a float evaluation of its exponent
  // (logf, expm1f, expf) inlined here raised the fp32 dense first kernel PassABody<float, 16> from 78 to
  // 88 registers and made config 3 measurably slower for Paul and DOG; the double one reuses the code
  // the orders above 8 already take.)
  const T a = (sizeof(T) == 8 || (MORSE && fp.family == 4) || (fp.family != 0 && fp.m > 8))
                  ? (T)(amp_eval<MORSE>(fp, d.s, k) * d.amp)
                  : (T)(amp_eval_t<T, MORSE>(fp, d.s, k) * (T)d.amp);
  return rot_unit<T>(cscale(v, a), fp.unit);
}

// ---- storers -------------------------------------------------------------------
// final output: out[row][u + q*U], u = u0 + b, trimmed to n < nout.
// Epilogues fused into the store:
//   EPI_STORE      out = x
//   EPI_MULCONJ    out = out * conj(x)          (cross-wavelet: second transform of xwt)
//   EPI_GAUSS      out = x * exp(g * k_n^2) * post, k_n = 2 pi fftfreq(nfreq)[n]
//                  (time-smoothing filter of Morlet.smooth applied to a forward transform)
enum { EPI_STORE = 0, EPI_MULCONJ = 1, EPI_GAUSS = 2 };
template <typename T> struct Epilogue {
  int mode;
  double g;        // EPI_GAUSS: -0.5 * (s/dt)^2 of this row
  double invn;     // 1 / nfreq
  double post;     // extra real factor (1/npad of the following inverse transform)
  long long nfreq;
  HD cx<T> apply(cx<T> x, cx<T> old, long long n) const {
    if (mode == EPI_MULCONJ) return cmul(old, cconj(x));
    if (mode == EPI_GAUSS) {
      const long long qs = n < nfreq / 2 ? n : n - nfreq;   // numpy fftfreq ordering
      const double k = 6.283185307179586 * ((double)qs * invn);
      if constexpr (sizeof(T) == 8) {
        const T f = (T)(exp(g * (k * k)) * post);
        return cscale(x, f);
      } else {
        // argument in double (k spans the whole transform), exponential in float: one double
        // transcendental per element would make the fp32 smoothing transforms fp64-pipe bound
        const T f = expf((float)(g * (k * k))) * (float)post;
        return cscale(x, f);
      }
    }
    return x;
  }
};
template <typename T> struct OutStorer {
  using V = cx<T>;
  V *row;          // out + row*pitch
  long long nout;  // keep final index < nout
  int u0, U;
  Epilogue<T> epi;
  int ostride = 1, ooff = 0;   // final index = n*ostride + ooff (interleaved sub-transforms, Np > 2^20)
  template <int R> HD void store(int b, int ql, int qs, V (&x)[R]) const {
    const int u = u0 + b;
    if (u >= U) return;
    size_t step = (size_t)qs * (size_t)U;
    size_t n = (size_t)u + (size_t)ql * (size_t)U;
    if (ostride != 1) { n = n * (size_t)ostride + (size_t)ooff; step *= (size_t)ostride; }
    if (epi.mode == EPI_STORE && (long long)(n + (R - 1) * step) < nout) {
      // common case: every output of this butterfly is kept -> pointer walk, no per-element test
      V *p = row + n;
#pragma unroll
      for (int c = 0; c < R; ++c) { st_stream(p, x[c]); p += step; }
      return;
    }
#pragma unroll
    for (int c = 0; c < R; ++c, n += step) {
      if ((long long)n < nout) {
        if (epi.mode == EPI_STORE) st_stream(&row[n], x[c]);
        else row[n] = epi.apply(x[c], epi.mode == EPI_MULCONJ ? row[n] : x[c], (long long)n);
      }
    }
  }
};

// first-kernel output: Z[(p + q*M)*K2 + r2] = x_q * e^{SIGN 2 pi i r2 (p+qM)/N}
template <typename T, int SIGN> struct ZStorer {
  using V = cx<T>;
  V *Z;
  NTab nt;
  int p, M, r20, bmax;
  unsigned K2 = K2C;   // row length of Z
  int cached_b = -1;   // the step factor depends on b only: looked up once per thread
  V cached_st;
  template <int R> HD void store(int b, int ql, int qs, V (&x)[R]) {
    if (b >= bmax) return;
    const unsigned r2 = (unsigned)(r20 + b);
    const unsigned u = (unsigned)(p + ql * M);
    const unsigned du = (unsigned)(qs * M);
    V t = nroot_t<T>(nt, r2 * u);
    if (b != cached_b) {
      cached_st = nroot_t<T>(nt, r2 * du);
      if (SIGN < 0) cached_st.y = -cached_st.y;
      cached_b = b;
    }
    const V st = cached_st;
    if (SIGN < 0) t.y = -t.y;
    V *dst = Z + (size_t)u * K2 + r2;
#pragma unroll
    for (int c = 0; c < R; ++c) {
      dst[(size_t)c * du * K2] = cmul(x[c], t);
      t = cmul(t, st);
    }
  }
};

// ---- Body: single-kernel pruned inverse transform (K' <= 1024) -------------------
template <typename T> struct SingleArgs {
  const ScaleDesc *descs;  // device
  const cx<T> *Bbuf;       // band products
  cx<T> *W;                // [rows][n0]
  const cx<T> *tw;         // pass twiddle tables (fft_tile.cuh: tw_offset)
  NTab nt;
  long long n0;
  unsigned N;
  int first;               // descs[first + blockIdx.y]
  int epi;                 // EPI_STORE / EPI_MULCONJ
};

template <typename T, int K> struct SingleBody {
  static constexpr int NTB = TileCfg<T>::NT;   // threads per CTA of this kernel
  static constexpr int NT = NTB;
  using V = cx<T>;
  using Args = SingleArgs<T>;
  using LY = Lay<T, K>;
  static constexpr int NP = Plan<K>::NP;
  static_assert(NP >= 2, "single-kernel path needs a multi-pass plan");
  static constexpr int NPHASE = NP;
  static constexpr size_t SMEM = LY::BYTES;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    V *sm = (V *)smraw;
    const ScaleDesc d = a.descs[a.first + by];
    const int M = (int)(a.N / K);
    const int p0 = bx * LY::P;
    if constexpr (PH == 0) {
      GenLoader<T, K, Plan<K>::R1> ld;
      ld.B = a.Bbuf + d.boff;
      ld.nt = a.nt;
      ld.rsplit = d.rsplit;
      ld.p0 = (unsigned)p0;
      tile_first<T, K, +1>(sm, a.tw, ld, tid);
    } else if constexpr (PH == 1 && NP == 3) {
      tile_second<T, K, +1>(sm, a.tw, tid);
    } else {
      OutStorer<T> st;
      st.row = a.W + (size_t)d.row * a.n0;
      st.nout = a.n0;
      st.u0 = p0;
      st.U = M;
      st.epi.mode = a.epi;
      pass_last<T, K, +1>(sm, st, tid);
    }
  }
};


// ---- Body: K' = K1*1024 with small K1 (2, 4, 8) in ONE kernel -------------------------------
// The K1-point transform over r1 is evaluated as a direct sum while the tile is filled, so the
// Z round trip of the two-kernel path disappears:
//   in[u][r2] = e^{2 pi i r2 u / N} * sum_{r1 < K1} B[r1*1024 + r2] * w_u^{k1},  w_u = e^{2 pi i u / U},
//   W[u + q2*U] = sum_{r2} in[u][r2] e^{2 pi i r2 q2 / 1024}
// (k1 = r1 - K1 [r >= rsplit] is the signed row of residue r; no alignment of the window needed).
template <typename T, int K1> struct DirectBody {
  static constexpr int NTB = TileCfg<T>::NT;   // threads per CTA of this kernel
  static constexpr int NT = NTB;
  using V = cx<T>;
  using Args = SingleArgs<T>;
  static constexpr int K = K2C;
  using LY = Lay<T, K>;
  static constexpr int NP = Plan<K>::NP;
  static constexpr int P = LY::P;
  static constexpr int NPHASE = 2 + NP;
  static constexpr int NW = 2 * K1 * P;   // w_u^{k1} for k1 = r1 and r1 - K1, per b
  static constexpr size_t SMEM = LY::TILE_BYTES + NW * sizeof(V);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    V *sm = (V *)smraw;
    V *wt = (V *)((char *)smraw + LY::TILE_BYTES);   // [b][2][K1]
    const ScaleDesc d = a.descs[a.first + by];
    const int U = (int)(a.N / K);
    const int u0 = bx * P;
    if constexpr (PH == 0) {
      for (int i = tid; i < NW; i += NT) {
        const int b = i / (2 * K1), s = (i / K1) & 1, r1 = i % K1;
        const int k1 = r1 - (s ? K1 : 0);
        wt[i] = nroot_t<T>(a.nt, (unsigned)k1 * (unsigned)(u0 + b) * (unsigned)K);
      }
    } else if constexpr (PH == 1) {
      const V *B = a.Bbuf + d.boff;
      // Positions r2 = tid + NT*it are handled IB at a time: the K1*IB band values stay in
      // registers while the K1 weights of each batch index b are read from shared memory once
      // (they depend on (b, r1) only, except on the single row r1s that the signed-bin split
      // cuts, where the sign is chosen per position).
      constexpr int NIT = K / NT;
      constexpr int IB = (8 / K1) < 1 ? 1 : ((8 / K1) < NIT ? (8 / K1) : NIT);
      const int r1s = d.rsplit / K, r2s = d.rsplit % K;   // residues >= rsplit are "negative"
      V e = nroot_t<T>(a.nt, (unsigned)tid * (unsigned)u0);    // e^{2 pi i r2 u0 / N}
      const V se = nroot_t<T>(a.nt, (unsigned)NT * (unsigned)u0);
      V dr = nroot_t<T>(a.nt, (unsigned)tid);                  // e^{2 pi i r2 / N}
      const V sdr = nroot_t<T>(a.nt, (unsigned)NT);
      if constexpr (K1 >= 8) {
        // many terms per position: one position at a time, weights straight from shared memory
        for (int it = 0; it < NIT; ++it) {
          const int r2 = tid + NT * it;
          V bv[K1];
          bool neg[K1];
#pragma unroll
          for (int r1 = 0; r1 < K1; ++r1) {
            bv[r1] = ldg(&B[r1 * K + r2]);
            neg[r1] = (r1 * K + r2) >= d.rsplit;
          }
          V t = e;
#pragma unroll
          for (int b = 0; b < P; ++b) {
            V acc = mk<T>(0, 0);
#pragma unroll
            for (int r1 = 0; r1 < K1; ++r1)
              acc = cadd(acc, cmul(bv[r1], wt[(b * 2 + (neg[r1] ? 1 : 0)) * K1 + r1]));
            sm[LY::phys(b, r2)] = cmul(acc, t);
            t = cmul(t, dr);
          }
          e = cmul(e, se);
          dr = cmul(dr, sdr);
        }
      } else
      for (int it0 = 0; it0 < NIT; it0 += IB) {
        V bv[IB][K1], t[IB], dd[IB];
#pragma unroll
        for (int q = 0; q < IB; ++q) {
          const int r2 = tid + NT * (it0 + q);
#pragma unroll
          for (int r1 = 0; r1 < K1; ++r1) bv[q][r1] = ldg(&B[r1 * K + r2]);
          t[q] = e;
          dd[q] = dr;
          e = cmul(e, se);
          dr = cmul(dr, sdr);
        }
#pragma unroll
        for (int b = 0; b < P; ++b) {
          V acc[IB];
#pragma unroll
          for (int q = 0; q < IB; ++q) acc[q] = mk<T>(0, 0);
#pragma unroll
          for (int r1 = 0; r1 < K1; ++r1) {
            if (r1 != r1s) {   // warp-uniform: one weight for the whole row
              const V w = wt[(b * 2 + (r1 > r1s ? 1 : 0)) * K1 + r1];
#pragma unroll
              for (int q = 0; q < IB; ++q) acc[q] = cadd(acc[q], cmul(bv[q][r1], w));
            } else {
              const V wp = wt[(b * 2 + 0) * K1 + r1], wn = wt[(b * 2 + 1) * K1 + r1];
#pragma unroll
              for (int q = 0; q < IB; ++q) {
                const bool neg = (tid + NT * (it0 + q)) >= r2s;
                acc[q] = cadd(acc[q], cmul(bv[q][r1], neg ? wn : wp));
              }
            }
          }
#pragma unroll
          for (int q = 0; q < IB; ++q) {
            sm[LY::phys(b, tid + NT * (it0 + q))] = cmul(acc[q], t[q]);
            t[q] = cmul(t[q], dd[q]);
          }
        }
      }
    } else if constexpr (PH == 2) {
      SmemLoader<T, K> ld;
      ld.sm = sm;
      tile_first<T, K, +1>(sm, a.tw, ld, tid);
    } else if constexpr (PH == 3 && NP == 3) {
      tile_second<T, K, +1>(sm, a.tw, tid);
    } else {
      OutStorer<T> st;
      st.row = a.W + (size_t)d.row * a.n0;
      st.nout = a.n0;
      st.u0 = u0;
      st.U = U;
      st.epi.mode = a.epi;
      pass_last<T, K, +1>(sm, st, tid);
    }
  }
};

// ---- Body: second kernel of the two-kernel path: K2 = 1024 or 512 over r2, rows of Z -------
template <typename T> struct PassBArgs {
  const cx<T> *Z;          // [ny][U][K2]
  cx<T> *out;              // [rows][pitch]
  const cx<T> *tw;
  const ScaleDesc *descs;  // may be null: output row = blockIdx.y + row0
  const double *grow;      // EPI_GAUSS: per-row coefficient g
  long long pitch, nout;
  double post;
  unsigned N;
  int first, row0;
  int epi;
  int pf_dist;             // L2 prefetch distance in tiles (0 = off)
  int ny;                  // gridDim.y of this launch (rows)
  int by0;                 // global index of this launch's first Z row (interleave bookkeeping)
  int ileave;              // > 1: Z row `by` is sub-transform by % ileave of output row by / ileave
                           // (final index n*ileave + by % ileave): three-level path, Np > 2^20
};

// K2 = 1024 leaves P = TILE/K2 = Q/2 transforms per tile (64-byte output runs, 2-way bank
// conflict on the last pass of the unskewed row layout); K2 = 512 has P = Q: 128-byte output
// runs, conflict-free.  The pruned (band) scales use 512, the dense ones need 1024 (K1 <= 1024).
// REG: fp64 K2 = 1024 runs the register-resident core (fft_tile.cuh: x32_first / x32_last) with the
// exchange in place in the row tile; the coarse transforms of the expansion rows (CoarseBBody) keep
// the three-pass core.
template <typename T, int SIGN, int K2 = K2C, bool REG = (sizeof(T) == 8 && K2 == X32::K)> struct PassBBody {
  static constexpr int NTB = TileCfg<T>::NT;   // threads per CTA of this kernel
  static constexpr int NT = NTB;
  using V = cx<T>;
  using Args = PassBArgs<T>;
  static constexpr int K = K2;
  using LY = Lay<T, K, true>;   // rows are filled by bulk-async copies: no skew
  static constexpr int NP = Plan<K>::NP;
  // phase 0: one thread issues the bulk-async (TMA) copies of the tile's rows -- the rows
  // Z[u0 .. u0+P) are contiguous in global memory -- then the FFT passes run from shared memory
  static constexpr int NPHASE = REG ? 3 : NP + 1;
  static constexpr size_t SMEM = LY::TILE_BYTES + 16;
  // bulk-async copies need 16-byte aligned shared-memory destinations: every row start
  static constexpr bool ROWS_ALIGNED = (LY::PITCH * sizeof(V)) % 16 == 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    static_assert(ROWS_ALIGNED, "PassB: tile rows must start on 16-byte boundaries");
    // rows run last-to-first: the first kernel wrote the last rows of Z most recently, they are
    // the ones still resident in L2
    const int ey = by;                   // position in execution order
    by = a.ny - 1 - ey;
    V *sm = (V *)smraw;
    const int U = (int)(a.N / K);
    const int u0 = bx * LY::P;
    TileBarrier tb;
    tb.bar = (unsigned long long *)((char *)smraw + LY::TILE_BYTES);
    if constexpr (PH == 0) {
      const int nvalid = (U - u0) < LY::P ? (U - u0) : LY::P;
      const V *src = a.Z + (size_t)by * a.N + (size_t)u0 * K;
      if (tid == 0) {
        // one thread arms the barrier and issues one bulk copy per row
        tb.init_and_expect((unsigned)(nvalid * K * sizeof(V)));
        for (int b = 0; b < nvalid; ++b)
          tb.copy(sm + LY::phys(b, 0), src + (size_t)b * K, (unsigned)(K * sizeof(V)));
      }
      // warm L2 with the tile a CTA `pf_dist` blocks ahead will load (same row of the grid,
      // or the next row when this one is exhausted): its TMA copies then hit L2
      if (tid == 0 && a.pf_dist > 0) {
        long long t = (long long)bx + a.pf_dist;
        int pe = ey;
        const int tiles = (U + LY::P - 1) / LY::P;
        while (t >= tiles && pe + 1 < a.ny) { t -= tiles; ++pe; }
        const int py = a.ny - 1 - pe;
        if (t < tiles && t * LY::P + LY::P <= U)
          TileBarrier::prefetch_l2(a.Z + (size_t)py * a.N + (size_t)t * LY::P * K,
                                   (unsigned)(LY::P * K * sizeof(V)));
      }
      for (int b = nvalid; b < LY::P; ++b)
        for (int i = tid; i < K; i += NT) sm[LY::phys(b, i)] = mk<T>(0, 0);
    } else if constexpr (PH == 1) {
      tb.wait(0);
      SmemLoader<T, K, true> ld;
      ld.sm = sm;
      if constexpr (REG)
        x32_first<SIGN, X32_WARP, X32InTile<true>>(sm, a.tw, ld, tid);
      else
        tile_first<T, K, SIGN, SmemLoader<T, K, true>, true>(sm, a.tw, ld, tid);
    } else if constexpr (PH == 2 && NP == 3 && !REG) {
      tile_second<T, K, SIGN, true>(sm, a.tw, tid);
    } else {
      const int il = a.ileave > 1 ? a.ileave : 1;
      const int outer = (a.by0 + by) / il;
      const int row = a.descs ? a.descs[a.first + outer].row : a.row0 + outer;
      OutStorer<T> st;
      st.row = a.out + (size_t)row * a.pitch;
      st.nout = a.nout;
      st.u0 = u0;
      st.U = U;
      st.ostride = il;
      st.ooff = (a.by0 + by) % il;
      st.epi.mode = a.epi;
      if (a.epi == EPI_GAUSS) {
        st.epi.g = a.grow[row];
        st.epi.invn = 1.0 / ((double)a.N * il);
        st.epi.post = a.post;
        st.epi.nfreq = (long long)a.N * il;
      }
      if constexpr (REG)
        x32_last<SIGN, X32_BMAJOR, X32InTile<true>>(sm, st, tid);
      else
        pass_last<T, K, SIGN, OutStorer<T>, true>(sm, st, tid);
      if (tid == 0) tb.inval();   // every thread passed wait() at least one barrier ago
    }
  }
};

// ---- Body: overlap-save rows (fp64, short impulse response) ---------------------------------
// Row j of W is the circular convolution of the signal with h_j = IDFT(norm conj psi^) (what the
// exact path gives for x^ = 1); the planner keeps its taps t in [t1 - M + 1, t1] (engine.cu: os_plan).
// A CTA owns P consecutive blocks of hop = L - M + 1 outputs for a group of up to G rows sharing
// (t1, M):
//   y_b[i] = x[(n_b - t1 + i) mod Np] (0 past n0),  n_b = (bx*P + b) * hop,
//   W[n_b + i - t1] = IDFT_L(DFT_L(y_b) * H_j)[i]  for t1 <= i < t1 + hop,  H_j = DFT_L(h_j mod L) / L.
// The forward transform of the real blocks is taken once and kept in shared memory as its
// non-negative half (X[L - k] = conj X[k]); each row of the group multiplies it by H_j while the
// inverse transform is loaded, and stores its hop valid outputs contiguously.
struct OsGroup {
  int first, count;  // descriptors first .. first + count (one class of the sorted array)
  int t1, hop;
  long long hoff;    // H of the group's first row; the others follow, L entries each
};
struct OsArgs {
  const ScaleDesc *descs;
  const OsGroup *groups;
  const double *sig;   // real signals, n0 samples per channel (ScaleDesc::chan)
  const double2 *H;
  double2 *W;
  const double2 *tw;
  long long n0;
  unsigned N;
  int epi;             // EPI_STORE / EPI_MULCONJ
};

template <int L, int R> struct OsSigLoader {
  const double *x;
  long long start, n0;   // start: n_0 - t1 of the tile's first block
  unsigned nmask;
  int hop, base, stride;
  HD void begin(int base_, int stride_, int, int) { base = base_; stride = stride_; }
  HD void load(int b, double2 (&v)[R]) const {
    const long long s = start + (long long)b * hop + base;
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const long long n = (s + (long long)i * stride) & (long long)nmask;   // circular modulo Np
      v[i] = make_double2(n < n0 ? ldg(&x[n]) : 0.0, 0.0);
    }
  }
};
template <int L> struct OsHalfStorer {
  double2 *xs;   // [P][L/2 + 1]
  template <int R> HD void store(int b, int ql, int qs, double2 (&x)[R]) const {
#pragma unroll
    for (int c = 0; c < R; ++c) {
      const int q = ql + c * qs;
      if (q <= L / 2) xs[b * (L / 2 + 1) + q] = x[c];
    }
  }
};
template <int L, int R> struct OsSpecLoader {
  const double2 *xs, *H;
  int base, stride;
  double2 hv[R];
  HD void begin(int base_, int stride_, int, int) {
    base = base_; stride = stride_;
#pragma unroll
    for (int i = 0; i < R; ++i) hv[i] = ldg(&H[base + i * stride]);
  }
  HD void load(int b, double2 (&v)[R]) const {
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const int q = base + i * stride;
      const double2 y = q <= L / 2 ? xs[b * (L / 2 + 1) + q] : cconj(xs[b * (L / 2 + 1) + L - q]);
      v[i] = cmul(y, hv[i]);
    }
  }
};
struct OsStorer {
  double2 *row;
  long long nb0, n0;   // W index of tile position i of block b: nb0 + b*hop + i
  int t1, hop, epi;
  template <int R> HD void store(int b, int ql, int qs, double2 (&x)[R]) const {
    const long long nb = nb0 + (long long)b * hop;
#pragma unroll
    for (int c = 0; c < R; ++c) {
      const int i = ql + c * qs;
      const long long n = nb + i;
      if (i >= t1 && i < t1 + hop && n < n0) {
        if (epi == EPI_STORE) st_stream(&row[n], x[c]);
        else row[n] = cmul(row[n], cconj(x[c]));
      }
    }
  }
};

// Transforms: the register-resident core (fft_tile.cuh: x32_first / x32_last), one warp per block,
// with an exchange buffer of its own next to the half spectrum.
template <int G> struct OsBody {
  static constexpr int L = X32::K;
  static constexpr int NTB = TileCfg<double>::NT;
  static constexpr int NT = NTB;
  using Args = OsArgs;
  static constexpr int P = X32::P;
  static constexpr int NPHASE = 2 + 2 * G;
  static constexpr size_t SMEM = X32Ex::BYTES + (size_t)P * (L / 2 + 1) * sizeof(double2);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    double2 *ex = (double2 *)smraw;
    double2 *xs = (double2 *)((char *)smraw + X32Ex::BYTES);
    const OsGroup g = a.groups[by];
    const long long n_first = (long long)bx * P * g.hop;
    if (n_first >= a.n0) return;   // whole CTA: no block of this tile holds outputs
    if constexpr (PH == 0) {
      OsSigLoader<L, X32::C> ld;
      ld.x = a.sig + (size_t)a.descs[g.first].chan * a.n0; ld.start = n_first - g.t1; ld.n0 = a.n0; ld.nmask = a.N - 1; ld.hop = g.hop;
      x32_first<-1, X32_WARP, X32Ex>(ex, a.tw, ld, tid);
    } else if constexpr (PH == 1) {
      OsHalfStorer<L> st{xs};
      x32_last<-1, X32_WARP, X32Ex>(ex, st, tid);
    } else {
      constexpr int r = (PH - 2) / 2;
      if (r >= g.count) return;
      if constexpr (PH % 2 == 0) inv_first(a, g, r, n_first, ex, xs, tid);
      else inv_last(a, g, r, n_first, ex, tid);
    }
  }
  // the inverse transform of row r of the group: one copy of the code for all G rows
  HD_NOINLINE static void inv_first(const Args &a, const OsGroup &g, int r, long long n_first, double2 *ex,
                                    const double2 *xs, int tid) {
    OsSpecLoader<L, X32::C> ld;
    ld.xs = xs; ld.H = a.H + g.hoff + (long long)r * L;
    x32_first<+1, X32_WARP, X32Ex>(ex, a.tw, ld, tid);
  }
  HD_NOINLINE static void inv_last(const Args &a, const OsGroup &g, int r, long long n_first, const double2 *ex,
                                   int tid) {
    OsStorer st;
    st.row = a.W + (size_t)a.descs[g.first + r].row * a.n0;
    st.nb0 = n_first - g.t1; st.n0 = a.n0; st.t1 = g.t1; st.hop = g.hop; st.epi = a.epi;
    x32_last<+1, X32_WARP, X32Ex>(ex, st, tid);
  }
};

// largest |h[t]| of rows of h over t in [lo, hi), one partial per CTA (out[by * gridDim.x + bx]):
// the planner's test that an impulse response has no taps above its rounding floor far from t = 0
struct AbsMaxArgs { const double2 *h; double *out; long long pitch, lo, hi; int nblk; };
struct AbsMaxBody {
  using Args = AbsMaxArgs;
  static constexpr int NPHASE = 2;
  static constexpr size_t SMEM = NT * sizeof(double);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    double *sm = (double *)smraw;
    if constexpr (PH == 0) {
      const long long chunk = (a.hi - a.lo + a.nblk - 1) / a.nblk;
      const long long s = a.lo + bx * chunk, e = s + chunk < a.hi ? s + chunk : a.hi;
      double m = 0;
      for (long long i = s + tid; i < e; i += NT) {
        const double2 v = a.h[(size_t)by * a.pitch + i];
        m = fmax(m, fmax(fabs(v.x), fabs(v.y)));
      }
      sm[tid] = m;
    } else if (tid == 0) {
      double m = 0;
      for (int i = 0; i < NT; ++i) m = fmax(m, sm[i]);
      a.out[(size_t)by * a.nblk + bx] = m;
    }
  }
};

// ---- Body: first kernel of the two-kernel path: K1-point transforms over r1 --------
// (Band scales read the band buffer rather than evaluate x^ * conj(psi^) * norm while the tile is filled:
// the evaluation slows the first kernel of Np/K' = 2 scales by more than the band-product launch it saves.)
// MODE_COARSE: coarse spectra of expansion rows (coarse_value), rows of N = Nc points
enum { MODE_DENSE = 0, MODE_BAND = 1, MODE_REAL = 2, MODE_CPLX = 3, MODE_COARSE = 4 };

// Coarse spectrum of expansion row d at coarse index r < Nc: the band product shifted to the centre
// bin and divided by the transform of the interpolation kernel (see "Band-limited expansion path"
// below); zero outside the band.  Nx: length of the signal's spectrum.
template <typename T> HD cx<T> coarse_value(const Fam &fam, const ScaleDesc &d, const cx<T> *spec, int r, unsigned Nx) {
  const int Nc = 1 << d.ip_log2Nc;
  const int kp = r < Nc / 2 ? r : r - Nc;       // signed offset from the centre bin
  const int k = d.ip_kc + kp;
  if (k < d.k_lo || k > d.k_hi) return mk<T>(0, 0);
  const cx<T> b = band_value<T>(fam, d, spec, (unsigned)k & (Nx - 1), k, Nx);
  // 1 / phi^(kp / Nc),  phi^(xi) = taps / I0(beta) * sinh(z) / z,  z = sqrt(beta^2 - (pi taps xi)^2)
  const double pw = 3.14159265358979323846 * (double)d.ip_w;
  const double x = pw * ((double)kp / (double)Nc);
  // > 0: |xi| <= 1/4 < 1 - xi_max.  The fused multiply-add is spelled out: left to the compiler, the
  // contraction differs between the kernels that inline this function, and so would the last bit
  const double bb = d.ip_beta * d.ip_beta;
  const double z = sqrt(fma(-x, x, bb));
  const double f = d.ip_dc * (z / sinh(z));
  return mk<T>((T)((double)b.x * f), (T)((double)b.y * f));
}

template <typename T> struct PassAArgs {
  const ScaleDesc *descs;
  const cx<T> *spec;   // x^ (MODE_DENSE, MODE_COARSE)
  const cx<T> *Bbuf;   // band products (MODE_BAND)
  const void *in;      // T* (MODE_REAL) or cx<T>* (MODE_CPLX), rows of `in_pitch`
  cx<T> *Z;            // [ny][U][K2]
  const cx<T> *tw;
  Fam fam;
  NTab nt;
  long long in_pitch, n_in;
  unsigned N;
  int first, row0;
  int pf_dist;         // L2 prefetch distance in tiles for the band-product rows (0 = off)
  unsigned K2;         // row length of Z: 1024 (second kernel = PassB) or 2^20 (pre-pass of the
                       // three-level path for Np > 2^20, where the rows are transformed again)
  unsigned Nx;         // MODE_COARSE: length of the signal's spectrum (N is the coarse length)
};

// REG: the fp64 dense rows of K1 = 1024 fill the register-resident core (fft_tile.cuh:
// x32_exchange_out / x32_last) straight from their spectrum loads: a thread's share of the tile is one
// column (b = tid % 4, positions tid / 4 + 32 i) of the three-pass core's fill as well, so phase 0
// loads, transforms and writes the exchange, and phase 1 finishes and stores.  No tile in shared memory.
template <typename T, int K1, int MODE, int SIGN> struct PassABody {
  static constexpr int NTB = TileCfg<T>::NT;   // threads per CTA of this kernel
  static constexpr int NT = NTB;
  using V = cx<T>;
  using Args = PassAArgs<T>;
  using LY = Lay<T, K1>;
  static constexpr int NP = Plan<K1>::NP;
  static constexpr int P = LY::P;
  static constexpr int T2 = P < K2C ? P : K2C;  // r2 values per tile (a.K2 is a multiple of it)
  static constexpr bool REG = sizeof(T) == 8 && K1 == X32::K && MODE == MODE_DENSE;
  static constexpr int NPHASE = REG ? 2 : (NP == 1 ? 1 : NP + 1);
  static constexpr size_t SMEM = REG ? X32Ex::BYTES : LY::BYTES;

  // Morlet, dense scale: a thread's bins are k0, k0 + D, k0 + 2D, ... (D = (NT/T2)*K2), so
  //   g(k + D) = g(k) * rho(k),  rho(k + D) = rho(k) * exp(-a^2),  a = s * w_D,
  // replaces the exp per bin by two multiplies.  Re-seeded with exact exp() when the
  // band is entered, at the signed-bin wrap and every 16 steps (error <= ~1e-14 relative).
  // Batches of UB bins: the spectrum loads of a batch are issued together (independent of the
  // recurrence), then the Gaussian values follow one another.  One load per iteration, as the
  // plain loop compiles, leaves every thread waiting a full L2 round trip 32 times per tile.
  static constexpr int DPOS = NT / T2 > 0 ? NT / T2 : 1;
  static constexpr int UB = CWTB_PASSA_BATCH;
  struct GaussWalk {
    const Args &a;
    const ScaleDesc &d;
    unsigned rb;   // r2 of the thread's bins: r20 + b
    const V *sp;   // the thread's bin of position 0
    long long D;
    double aa, q, g = 0, rho = 0;
    long long kprev = 0;
    int since = 1 << 30;
    HD GaussWalk(const Args &a_, const ScaleDesc &d_, int r20, int b) : a(a_), d(d_), rb((unsigned)(r20 + b)) {
      sp = a.spec + (size_t)d.chan * a.N + rb;
      D = (long long)DPOS * a.K2;
      const double wd = 6.283185307179586 * ((double)D * a.fam.dw);
      aa = d.s * wd;
      q = exp(-aa * aa);
    }
    // spectrum values of positions pos0 + u*DPOS (kk[u] = INT_MAX: outside the band or past K1)
    HD void load(int pos0, V (&raw)[UB], int (&kk)[UB]) const {
#pragma unroll
      for (int u = 0; u < UB; ++u) {
        const int pos = pos0 + u * DPOS;
        const unsigned r = (unsigned)pos * a.K2 + rb;
        const int k = (int)r - (r >= a.N / 2 ? (int)a.N : 0);
        const bool in = pos < K1 && k >= d.k_lo && k <= d.k_hi;
        kk[u] = in ? k : (int)0x7fffffff;
        raw[u] = in ? ldg(&sp[(size_t)pos * a.K2]) : mk<T>(0, 0);
      }
    }
    // exact g(k) and rho(k), out of line: the register-resident fill unrolls 32 steps of the walk
    HD_NOINLINE static double2 seed(double s, double dw, double f0, double aa, int k) {
      const double f = s * (6.283185307179586 * ((double)k * dw));
      const double dd = f - f0;
      return make_double2(exp(-0.5 * dd * dd), exp(-aa * dd - 0.5 * aa * aa));
    }
    // the next value of the walk: raw * Gaussian * amp, or zero outside the band
    HD V next(V raw, int kk) {
      if (kk == (int)0x7fffffff) { since = 1 << 30; return mk<T>(0, 0); }
      const int k = kk;
      // (a value in the subnormal range has lost its relative precision: with band_eps = 0 the
      // band reaches bins where exp() is below 1e-308, and the recurrence would carry that
      // error up to the peak -- re-seed until the value is a normal number again)
      if (since >= 16 || (long long)k != kprev + D || g < 1e-290) {
        const double2 gr = seed(d.s, a.fam.dw, a.fam.f0, aa, k);
        g = gr.x;
        rho = gr.y;
        since = 0;
      } else {
        g *= rho;
        rho *= q;
        ++since;
      }
      kprev = k;
      return cscale(raw, (T)(g * d.amp));
    }
  };

  struct Src {
    const Args &a;
    ScaleDesc d;
    int by, p;
    V twist0;
    HD Src(const Args &a_, int by_, int p_) : a(a_), by(by_), p(p_) {
      if (MODE == MODE_DENSE || MODE == MODE_BAND || MODE == MODE_COARSE) d = a.descs[a.first + by];
    }
    // element r = pos*K2 + r2 of the K'-point input
    HD V get(int pos, int r2) const {
      const unsigned r = (unsigned)pos * a.K2 + (unsigned)r2;
      if (MODE == MODE_DENSE) {
        const int k = (int)r - (r >= a.N / 2 ? (int)a.N : 0);
        // outside the scale's band the response is below the pruning threshold: same rule as
        // the pruned classes (their band product is exactly zero there); skips the exp
        if (a.fam.family != 3 && (k < d.k_lo || k > d.k_hi)) return mk<T>(0, 0);
        return band_value<T>(a.fam, d, a.spec, r, k, a.N);
      } else if (MODE == MODE_BAND) {
        V v = ldg(&a.Bbuf[d.boff + r]);
        if (p == 0 || NP > 1) return v;   // multi-pass plans apply the twist in pass 1
        const int k1 = pos - ((int)r >= d.rsplit ? K1 : 0);
        // e^{2 pi i k1 p / (K1 M)} = e^{2 pi i (k1 p K2) / N}
        V w = nroot_t<T>(a.nt, (unsigned)k1 * (unsigned)p * a.K2);
        return cmul(v, w);
      } else if (MODE == MODE_COARSE) {
        return coarse_value<T>(a.fam, d, a.spec, (int)r, a.Nx);
      } else if (MODE == MODE_REAL) {
        const T *row = (const T *)a.in + (size_t)(a.row0 + by) * a.in_pitch;
        return mk<T>((long long)r < a.n_in ? ldg(&row[r]) : (T)0, (T)0);
      } else {
        const V *row = (const V *)a.in + (size_t)(a.row0 + by) * a.in_pitch;
        return (long long)r < a.n_in ? ldg(&row[r]) : mk<T>(0, 0);
      }
    }
  };

  // the register-resident fill unrolls its 32 positions: one copy of the families' evaluation
  HD_NOINLINE static V get_out_of_line(const Args &a, int by, int p, int pos, int r2) { return Src(a, by, p).get(pos, r2); }

  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    V *sm = (V *)smraw;
    const int NTILE2 = (int)(a.K2 / T2);
    const int p = bx / NTILE2;
    const int r20 = (bx % NTILE2) * T2;
    const int M = (int)(a.N / ((unsigned)K1 * a.K2));
    ZStorer<T, SIGN> st;
    st.Z = a.Z + (size_t)by * a.N;
    st.nt = a.nt;
    st.p = p;
    st.M = M;
    st.r20 = r20;
    st.bmax = T2;
    st.K2 = a.K2;
    if constexpr (NP == 1) {
      Src src(a, by, p);
      for (int b = tid; b < T2; b += NT) {
        V x[K1];
#pragma unroll
        for (int i = 0; i < K1; ++i) x[i] = src.get(i, r20 + b);
        dftR<K1, SIGN, T>(x);
        st.store(b, 0, 1, x);
      }
    } else if constexpr (REG) {
      if constexpr (PH == 0) {
        static_assert(T2 == X32::P && DPOS == X32::C && X32::K % (DPOS * UB) == 0, "dense fill vs core columns");
        Src src(a, by, p);
        const int b = tid % T2, n1 = tid / T2;   // X32_BMAJOR
        V x[X32::C];
        if (a.fam.family == 0) {
          GaussWalk gw(a, src.d, r20, b);
#pragma unroll
          for (int it = 0; it < X32::C / UB; ++it) {
            V raw[UB];
            int kk[UB];
            gw.load(n1 + it * UB * DPOS, raw, kk);
#pragma unroll
            for (int u = 0; u < UB; ++u) x[it * UB + u] = gw.next(raw[u], kk[u]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < X32::C; ++i) x[i] = get_out_of_line(a, by, p, n1 + DPOS * i, r20 + b);
        }
        x32_exchange_out<SIGN, X32Ex>(sm, a.tw, b, n1, x);
      } else {
        x32_last<SIGN, X32_BMAJOR, X32Ex>(sm, st, tid);
      }
    } else if constexpr (PH == 0) {
      Src src(a, by, p);
      // warm L2 with the band-product rows of the tile `pf_dist` blocks ahead (same scale)
      if (MODE == MODE_BAND && a.pf_dist > 0 && T2 * sizeof(V) >= 256) {
        const int tiles = M * NTILE2;
        const int t = bx + a.pf_dist;
        if (t < tiles) {
          const int r20n = (t % NTILE2) * T2;
          const V *base = a.Bbuf + src.d.boff + r20n;
          for (int pos = tid; pos < K1; pos += NT)
            TileBarrier::prefetch_l2(base + (size_t)pos * a.K2, (unsigned)(T2 * sizeof(V)));
        }
      }
      // the same for the rows of a batched row transform (coherence smoothing): the
      // tile `pf_dist` blocks ahead of this one in the same row
      if (MODE == MODE_CPLX && a.pf_dist > 0 && T2 * sizeof(V) >= 256) {
        const int t = bx + a.pf_dist;
        if (t < M * NTILE2) {
          const V *row = (const V *)a.in + (size_t)(a.row0 + by) * a.in_pitch + (t % NTILE2) * T2;
          for (int pos = tid; pos < K1; pos += NT)
            if ((long long)pos * a.K2 + (t % NTILE2) * T2 + T2 <= a.n_in)
              TileBarrier::prefetch_l2(row + (size_t)pos * a.K2, (unsigned)(T2 * sizeof(V)));
        }
      }
      if (MODE == MODE_DENSE && a.fam.family == 0 && T2 <= NT) {
        const int b = tid % T2;
        GaussWalk gw(a, src.d, r20, b);
        for (int pos0 = tid / T2; pos0 < K1; pos0 += DPOS * UB) {
          V raw[UB];
          int kk[UB];
          gw.load(pos0, raw, kk);
#pragma unroll
          for (int u = 0; u < UB; ++u) {
            const int pos = pos0 + u * DPOS;
            if (pos >= K1) break;
            sm[LY::phys(b, pos)] = gw.next(raw[u], kk[u]);
          }
        }
      } else {
        // (the compiler batches four loads per round trip on its own; eight in flight measured ...)
        CWTB_PRAGMA_UNROLL_A
        for (int idx = tid; idx < K1 * T2; idx += NT) {
          const int b = idx % T2, pos = idx / T2;
          sm[LY::phys(b, pos)] = src.get(pos, r20 + b);
        }
      }
    } else if constexpr (PH == 1) {
      if (MODE == MODE_BAND && p != 0) {
        SmemTwistLoader<T, K1, Plan<K1>::R1> ld;
        ld.sm = sm;
        ld.nt = a.nt;
        ld.rsplit_row = a.descs[a.first + by].rsplit / (int)a.K2;
        ld.pk2 = (unsigned)p * a.K2;
        tile_first<T, K1, SIGN>(sm, a.tw, ld, tid);
      } else {
        SmemLoader<T, K1> ld;
        ld.sm = sm;
        tile_first<T, K1, SIGN>(sm, a.tw, ld, tid);
      }
    } else if constexpr (PH == 2 && NP == 3) {
      tile_second<T, K1, SIGN>(sm, a.tw, tid);
    } else {
      pass_last<T, K1, SIGN>(sm, st, tid);
    }
  }
};

// ==================================================================================================
// Band-limited expansion path.  A scale whose response is confined to the bins [k_lo, k_hi]
// (Kb of the Np bins) is a trigonometric polynomial of Kb terms: it is fully determined by
// Nc >= 2 Kb samples.  Instead of running Np/K' pruned transforms of K' points each, the engine
//   (1) forms the band product shifted to the centre bin kc and divided by the transform of the
//       interpolation kernel (coarse_value), while it fills the tiles of
//   (2) the inverse transform on the coarse grid of Nc points (CoarseRowsBody, CoarseABody +
//       CoarseBBody: the batched FFT's tiles, one launch each for all coarse lengths), and
//   (3) expands the Nc samples to the Np output points with a polyphase Kaiser-Bessel kernel of
//       `taps` real weights per output and re-modulates by e^{2 pi i kc n / Np} (ExpandBody):
//         W[R m + rho] = e^{2 pi i kc n/Np} * sum_t c[m + t - (taps/2 - 1)] * h[t][rho],  R = Np / Nc.
// With phi the kernel and phi^ its transform, sum_m e^{2 pi i k m/Nc} phi(x - m) =
// sum_l phi^(k/Nc + l) e^{2 pi i (k/Nc + l) x}: the l = 0 term is the exact value after the division
// by phi^(k/Nc), the others are the aliasing error, bounded on the host by
// max_{|xi| <= xi_max} sum_{l != 0} |phi^(xi + l)| / |phi^(xi)| (engine.cu: kb_alias_bound).  The host
// picks (Nc, taps) so that the bound stays below the context's expansion tolerance (default
// 5e-13: measured error 1e-13, three orders inside the 1e-10 parity gate; 0 = path off).
// Cost per output point: 2*taps + 8 fp64 FMAs, one 16-byte shared-memory read, one 16-byte store --
// a streaming kernel bounded by the W store, with no intermediate in global memory.
// ==================================================================================================
// ---- coarse transforms of the expansion rows: ragged launches over every coarse length ----------
// The expansion rows of one coarse length that are consecutive in the class-sorted descriptor array
// form a segment; their coarse rows are consecutive in C and Z (descs[].ip_coff).  A launch covers up
// to CSEG_MAX segments; CTA bx belongs to the last segment whose cta0 <= bx and runs the tile of that
// segment's length -- the same radix plan, twiddles and arithmetic as a per-length launch.
struct CoarseSeg { int first, count, log2Nc, cta0; };
constexpr int CSEG_MAX = 32;
HD constexpr size_t cmax(size_t a, size_t b) { return a > b ? a : b; }
template <typename T> struct CoarseArgs {
  const ScaleDesc *descs;
  const cx<T> *spec;   // x^ of the signal(s), Nx points per channel
  cx<T> *Z;            // CoarseABody -> CoarseBBody intermediate, rows at descs[].ip_coff
  cx<T> *C;            // coarse samples, rows at descs[].ip_coff
  const cx<T> *tw;
  Fam fam;
  NTab nt[11];         // CoarseABody: e^{2 pi i e / Nc} for Nc = 2^(10 + i)
  unsigned Nx;
  int nseg;
  int pf_dist;         // CoarseBBody: PassBArgs::pf_dist
  CoarseSeg seg[CSEG_MAX];
};
template <typename T> HD const CoarseSeg &coarse_seg(const CoarseArgs<T> &a, int bx) {
  int s = 0;
  while (s + 1 < a.nseg && bx >= a.seg[s + 1].cta0) ++s;
  return a.seg[s];
}

// Nc <= 1024: one tile of P rows per CTA.  Phase 0 fills the tile with coarse_value, then the
// passes of the batched row transform (RowsBody) run from shared memory.
template <typename T> struct CoarseRowsBody {
  static constexpr int NTB = TileCfg<T>::NT;
  static constexpr int NT = NTB;
  using V = cx<T>;
  using Args = CoarseArgs<T>;
  template <int K> static constexpr size_t bytes() { return Lay<T, K>::BYTES; }
  static constexpr size_t SMEM = cmax(cmax(cmax(bytes<64>(), bytes<128>()), cmax(bytes<256>(), bytes<512>())), bytes<1024>());
  static constexpr int NPHASE = 4;
  // CTAs of a segment of `rows` rows of 2^log2Nc points
  HD static int ctas(int log2Nc, int rows) {
    const int P = TileCfg<T>::TILE >> log2Nc;
    return (rows + P - 1) / P;
  }
  struct Storer {
    V *out;   // row 0 of the tile
    int nb;   // valid rows
    int K;
    template <int R> HD void store(int b, int ql, int qs, V (&x)[R]) const {
      if (b >= nb) return;
#pragma unroll
      for (int c = 0; c < R; ++c) out[(size_t)b * K + ql + c * qs] = x[c];
    }
  };
  template <int K, int PH> HD static void tile(const Args &a, const CoarseSeg &g, int bx, int tid, V *sm) {
    using LY = Lay<T, K>;
    constexpr int NP = Plan<K>::NP;
    static_assert(NP >= 2, "coarse rows: multi-pass tile plans only");
    const int row0 = (bx - g.cta0) * LY::P;
    const int nb = g.count - row0 < LY::P ? g.count - row0 : LY::P;
    if constexpr (PH == 0) {
      for (int idx = tid; idx < LY::P * K; idx += NT) {
        const int b = idx / K, pos = idx % K;
        V v = mk<T>(0, 0);
        if (b < nb) v = coarse_value<T>(a.fam, a.descs[g.first + row0 + b], a.spec, pos, a.Nx);
        sm[LY::phys(b, pos)] = v;
      }
    } else if constexpr (PH == 1) {
      SmemLoader<T, K> ld;
      ld.sm = sm;
      tile_first<T, K, +1>(sm, a.tw, ld, tid);
    } else if constexpr (PH == 2 && NP == 3) {
      tile_second<T, K, +1>(sm, a.tw, tid);
    } else if constexpr (PH == NP) {
      Storer st{a.C + a.descs[g.first].ip_coff + (size_t)row0 * K, nb, K};
      pass_last<T, K, +1>(sm, st, tid);
    }
  }
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *smraw) {
    const CoarseSeg &g = coarse_seg(a, bx);
    V *sm = (V *)smraw;
    switch (g.log2Nc) {
      case 6: tile<64, PH>(a, g, bx, tid, sm); break;
      case 7: tile<128, PH>(a, g, bx, tid, sm); break;
      case 8: tile<256, PH>(a, g, bx, tid, sm); break;
      case 9: tile<512, PH>(a, g, bx, tid, sm); break;
      case 10: tile<1024, PH>(a, g, bx, tid, sm); break;
    }
  }
};

// 1024 < Nc <= 2^20: the two-kernel row transform (K1 = Nc / 1024, K2 = 1024).  The first kernel is
// PassABody in MODE_COARSE, which forms the coarse spectrum while it fills its tile.
template <typename T> struct CoarseABody {
  static constexpr int NTB = TileCfg<T>::NT;
  static constexpr int NT = NTB;
  using V = cx<T>;
  using Args = CoarseArgs<T>;
  template <int K1> using A = PassABody<T, K1, MODE_COARSE, +1>;
  static constexpr size_t SMEM = cmax(cmax(cmax(cmax(A<2>::SMEM, A<4>::SMEM), cmax(A<8>::SMEM, A<16>::SMEM)),
                                           cmax(cmax(A<32>::SMEM, A<64>::SMEM), cmax(A<128>::SMEM, A<256>::SMEM))),
                                      cmax(A<512>::SMEM, A<1024>::SMEM));
  static constexpr int NPHASE = 4;
  template <int K1> HD static int per_row() { return K2C / A<K1>::T2; }
  HD static int ctas(int log2Nc, int rows) {
    switch (log2Nc - 10) {
      case 1: return rows * per_row<2>();
      case 2: return rows * per_row<4>();
      case 3: return rows * per_row<8>();
      case 4: return rows * per_row<16>();
      case 5: return rows * per_row<32>();
      case 6: return rows * per_row<64>();
      case 7: return rows * per_row<128>();
      case 8: return rows * per_row<256>();
      case 9: return rows * per_row<512>();
      case 10: return rows * per_row<1024>();
    }
    return 0;
  }
  template <int K1, int PH> HD static void tile(const Args &a, const CoarseSeg &g, int bx, int tid, void *sm) {
    if constexpr (PH < A<K1>::NPHASE) {
      const int local = bx - g.cta0, per = per_row<K1>();
      PassAArgs<T> pa{};
      pa.descs = a.descs; pa.spec = a.spec; pa.tw = a.tw; pa.fam = a.fam; pa.nt = a.nt[g.log2Nc - 10];
      pa.Z = a.Z + a.descs[g.first].ip_coff;
      pa.N = 1u << g.log2Nc; pa.Nx = a.Nx; pa.first = g.first; pa.K2 = K2C;
      A<K1>::template phase<PH>(pa, local % per, local / per, tid, sm);
    }
  }
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *sm) {
    const CoarseSeg &g = coarse_seg(a, bx);
    switch (g.log2Nc - 10) {
      case 1: tile<2, PH>(a, g, bx, tid, sm); break;
      case 2: tile<4, PH>(a, g, bx, tid, sm); break;
      case 3: tile<8, PH>(a, g, bx, tid, sm); break;
      case 4: tile<16, PH>(a, g, bx, tid, sm); break;
      case 5: tile<32, PH>(a, g, bx, tid, sm); break;
      case 6: tile<64, PH>(a, g, bx, tid, sm); break;
      case 7: tile<128, PH>(a, g, bx, tid, sm); break;
      case 8: tile<256, PH>(a, g, bx, tid, sm); break;
      case 9: tile<512, PH>(a, g, bx, tid, sm); break;
      case 10: tile<1024, PH>(a, g, bx, tid, sm); break;
    }
  }
};

// second kernel of the same rows: PassBBody from Z into C
template <typename T> struct CoarseBBody {
  using B = PassBBody<T, +1, K2C, false>;
  static constexpr int NTB = B::NTB;
  static constexpr int NT = NTB;
  using Args = CoarseArgs<T>;
  static constexpr size_t SMEM = B::SMEM;
  static constexpr int NPHASE = B::NPHASE;
  HD static int per_row(int log2Nc) {
    constexpr int P = B::LY::P;
    return ((1 << (log2Nc - 10)) + P - 1) / P;
  }
  HD static int ctas(int log2Nc, int rows) { return rows * per_row(log2Nc); }
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *sm) {
    const CoarseSeg &g = coarse_seg(a, bx);
    const int local = bx - g.cta0, per = per_row(g.log2Nc);
    const long long off = a.descs[g.first].ip_coff;
    const unsigned Nc = 1u << g.log2Nc;
    PassBArgs<T> pb{};
    pb.Z = a.Z + off; pb.out = a.C + off; pb.tw = a.tw;
    pb.pitch = Nc; pb.nout = Nc; pb.N = Nc; pb.post = 1.0;
    pb.epi = EPI_STORE; pb.pf_dist = a.pf_dist; pb.ny = g.count; pb.ileave = 1;
    B::template phase<PH>(pb, local % per, local / per, tid, sm);
  }
};

template <typename T> struct ExpandArgs {
  const ScaleDesc *descs;
  const cx<T> *C;      // coarse samples (inverse transforms of the coarse spectra)
  const double *wt;    // weight tables [taps][R] (fp64 for both engines)
  cx<T> *W;            // [rows][n0]
  NTab nt;
  long long n0;
  unsigned N;
  int first;
  int epi;             // EPI_STORE / EPI_MULCONJ
  int log2N;           // R = N / Nc = 1 << (log2N - ip_log2Nc) per row: one launch serves every
                       // coarse length (each row has N / (NT * 32) tiles whatever its R)
};

// CTA tile: RB = min(R, NT) consecutive phases rho  x  NRUN = NT / RB runs of L = 32 consecutive
// coarse positions m.  A thread keeps its `TAPS` weights (fixed rho) and a sliding window of TAPS
// coarse samples in registers and walks its run (fully unrolled: window slots are compile-time
// registers): one new sample (shared-memory read, the same address for the lanes of a run) and one
// 16-byte store per output; lanes run over rho, so a warp stores min(R, 32) consecutive points
// per run.  The kernel is bound by the fp64 pipe (2 taps + ~12 other fp64 instructions per point);
// 8 accumulator chains and 4 CTAs per SM give that pipe the parallelism it needs.
template <typename T, int TAPS, int EPI = EPI_STORE> struct ExpandBody {
  static constexpr int NTB = TileCfg<T>::NT;
  static constexpr int NT = NTB;
  static constexpr int MINB = sizeof(T) == 8 ? 4 : 2;   // CTAs per SM the register budget is capped for
  using V = cx<T>;
  using Args = ExpandArgs<T>;
  static constexpr int L = 32;                       // coarse positions per run
  static constexpr int MINR = 4;                     // smallest expansion factor R = Np / Nc
  static constexpr int MAXRUN = NT / MINR;
  static constexpr int STAGE = MAXRUN * L + TAPS;    // staged coarse samples (incl. halo)
  HD static int skew(int i) { return i + (i >> 5); } // runs start 33 elements apart: no bank conflict
  static constexpr int NPHASE = 2;
  static constexpr size_t SMEM = (size_t)(STAGE + STAGE / 32 + 2) * sizeof(V);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    V *sm = (V *)smraw;
    const ScaleDesc &d = a.descs[a.first + by];
    const int log2R = a.log2N - d.ip_log2Nc;
    const int R = 1 << log2R;
    const int Nc = 1 << d.ip_log2Nc;
    const int RB = R < NT ? R : NT;
    const int NRUN = NT / RB;
    const int MT = NRUN * L;                         // coarse positions per CTA
    const int mtiles = (Nc + MT - 1) / MT;
    const int mt = bx % mtiles, rb = bx / mtiles;
    if (rb * RB >= R) return;                        // short coarse grid: fewer tiles than the launch has
    const int m0 = mt * MT;
    if constexpr (PH == 0) {
      const V *c = a.C + d.ip_coff;
      for (int i = tid; i < MT + TAPS; i += NT) {
        const int m = (m0 - (TAPS / 2 - 1) + i) & (Nc - 1);     // periodic on the coarse grid
        sm[skew(i)] = ldg(&c[m]);
      }
    } else {
      const int rl = tid & (RB - 1), j = tid / RB;
      const int rho = rb * RB + rl;
      const int ms = m0 + j * L;                     // first coarse position of this thread's run
      // outputs n = R m + rho for m = ms .. ms + L - 1; kept while m < Nc and n < n0
      const long long nfirst = ((long long)ms << log2R) + rho;
      long long keep = (a.n0 - nfirst + R - 1) >> log2R;      // steps with n < n0
      if (keep > Nc - ms) keep = Nc - ms;
      const int smax = keep < 0 ? 0 : (keep > L ? L : (int)keep);
      if (smax == 0) return;
      T hw[TAPS];
      const double *wt = a.wt + d.ip_woff + rho;
#pragma unroll
      for (int t = 0; t < TAPS; ++t) hw[t] = (T)ldg(&wt[(size_t)t * R]);
      const V *run = sm + 33 * j;                    // skew(j*L + i) = 33 j + i + (i >> 5), i < L + TAPS
      V win[TAPS];
#pragma unroll
      for (int t = 0; t < TAPS - 1; ++t) win[t] = run[t + (t >> 5)];
      // re-modulation e^{2 pi i kc n / Np}: table value (fp64 roots) every RESEED steps, recurrence
      // (step e^{2 pi i kc R / Np}) in between, in the engine's arithmetic: fp64 drifts 1e-16 per
      // step (16 steps), fp32 6e-8 per step (8 steps: 5e-7 of the 1e-5 budget)
      constexpr int RESEED = sizeof(T) == 8 ? 16 : 8;
      const unsigned kc = (unsigned)d.ip_kc;
      const unsigned nlo = (unsigned)nfirst;
      const V stepw = nroot_t<T>(a.nt, kc << log2R);
      V tw = mk<T>(1, 0);
      V *p = a.W + (size_t)d.row * a.n0 + nfirst;
#pragma unroll
      for (int s = 0; s < L; ++s) {
        win[(s + TAPS - 1) % TAPS] = run[(s + TAPS - 1) + ((s + TAPS - 1) >> 5)];
        if (s % RESEED == 0) tw = nroot_t<T>(a.nt, kc * (nlo + ((unsigned)s << log2R)));
        // 8 independent chains (4 per component): the fp64 pipe needs that much parallelism per warp;
        // the fp32 kernel is bound by instruction issue (ncu: 70 % issue slots busy, 49 instructions per
        // point for 24 useful ones) and runs two chains per component
        constexpr int NCH = sizeof(T) == 8 ? 4 : 2;
        T ar[4] = {0, 0, 0, 0}, ai[4] = {0, 0, 0, 0};
#pragma unroll
        for (int t = 0; t < TAPS; ++t) {
          const V cv = win[(s + t) % TAPS];
          ar[t & (NCH - 1)] += cv.x * hw[t];
          ai[t & (NCH - 1)] += cv.y * hw[t];
        }
        const V acc = NCH == 4 ? mk<T>((ar[0] + ar[1]) + (ar[2] + ar[3]), (ai[0] + ai[1]) + (ai[2] + ai[3]))
                               : mk<T>(ar[0] + ar[1], ai[0] + ai[1]);
        const V x = cmul(acc, tw);
        tw = cmul(tw, stepw);
        if (s < smax) {
          if (EPI == EPI_MULCONJ) *p = cmul(*p, cconj(x));
          else st_stream(p, x);
        }
        p += R;
      }
    }
  }
};

#ifndef CWTB_HOST_EMU
// ---- the fp64 expansion with the tap sums on the tensor cores ---------------------------------------
// The tap sum  acc[m][rho] = sum_t c[m + t - (taps/2 - 1)] * h[t][rho]  is a Toeplitz product: for 8
// consecutive coarse positions m and 8 consecutive phases rho it is an (8 x taps) x (taps x 8) real
// matrix product per component, i.e. taps/4 `mma.sync.m8n8k4.f64` (SASS DMMA.8x8x4) for the real and
// as many for the imaginary part.  On H100 the fp64 tensor-core rate is twice the DFMA rate, and the
// accumulation happens inside the instruction: the scalar kernel's 2 x taps DFMA + 6 DADD per point
// (of ~38 fp64 instructions, the pipe that bounds it) become taps/2 DMMA per 64 points.
//   A fragment (8 x 4, row m, column t):  lane holds c[m0 + lane/4 + 4 ks + lane%4]   (shared memory)
//   B fragment (4 x 8, row t, column rho): lane holds h[4 ks + lane%4][rho0 + lane/4] (registers)
//   C fragment (8 x 8): lane holds acc[m0 + lane/4][rho0 + 2 (lane%4) + {0, 1}]: two adjacent outputs,
//                       stored as two 16-byte streaming stores (sm_90 has no 32-byte store) after an
//                       exchange with the neighbour lane, so that each store instruction fills whole sectors.
// A warp owns 8 phases and a run of L coarse positions; a CTA (4 warps) covers min(R, 32) phases
// x 4 L / (min(R, 32) / 8) coarse positions = 32 L outputs.  Tap counts 10 and 14 are padded to 12 / 16
// with zero weights.  Not part of the host-emulation build (warp-collective instruction): the
// emulated tests run the scalar ExpandBody, which stays the fp32 engine's kernel and the fallback.
// (An fp32 counterpart on 3xTF32 -- x = x_hi + x_lo, three mma.sync.m16n8k8.tf32 per component and eight
// taps -- gives the same 5e-7 parity but needs three MMAs and the hi/lo splits per tap pair; the fp32
// engine keeps the scalar kernel.)
__device__ __forceinline__ void dmma884(double &c0, double &c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
template <int TAPS, int EPI = EPI_STORE> struct ExpandMmaBody {
  static constexpr int NTB = 128;
  static constexpr int NT = NTB;
  static constexpr int MINB = 4;
  using V = double2;
  using Args = ExpandArgs<double>;
#ifndef CWTB_MMA_L
#define CWTB_MMA_L 128
#endif
  static constexpr int L = CWTB_MMA_L;              // coarse positions per warp run (8 L outputs per warp)
  static constexpr int KS = (TAPS + 3) / 4;         // k-steps of four taps
  static constexpr int KS4 = (TAPS + 4) / 4;        // R = 4: one more tap column (see compute<true>)
  static constexpr int OUT_PER_CTA = 32 * L;
  static constexpr int STAGE = 8 * L + 4 * KS4;     // staged coarse samples incl. halo (R = 4: 4 runs of 2 L)
  // two stages: the next tile's coarse samples arrive while this one computes and stores
  static constexpr size_t SMEM = 2 * (size_t)STAGE * sizeof(V);
  // work item w of a launch over `gm` tiles per row: row w / gm, tile w % gm
  struct Tile {
    const ScaleDesc *d;
    int log2R, Nc, wpb, MT, m0, rb;
    bool r4, live;
  };
  __device__ static Tile tile(const Args &a, unsigned w, unsigned gm) {
    Tile t;
    const int bx = (int)(w % gm);
    t.d = &a.descs[a.first + (int)(w / gm)];
    t.log2R = a.log2N - t.d->ip_log2Nc;
    t.r4 = t.log2R == 2;
    const int R = 1 << t.log2R;
    t.Nc = 1 << t.d->ip_log2Nc;
    t.wpb = t.r4 ? 1 : ((R < 32 ? R : 32) >> 3);   // warps side by side in rho: 1, 2 or 4
    t.MT = (4 / t.wpb) * (t.r4 ? 2 * L : L);        // coarse positions per tile: 4 / wpb warp runs
    const int mtiles = (t.Nc + t.MT - 1) / t.MT;
    t.rb = bx / mtiles;
    t.m0 = (bx % mtiles) * t.MT;
    t.live = !(t.rb * 32 >= R && t.rb > 0);         // short rows use the first tiles of a row only
    return t;
  }
  // the tile's coarse samples incl. halo, periodic on the coarse grid: one 16-byte cp.async each
  __device__ static void load(const Args &a, const Tile &t, V *sm) {
    if (!t.live) return;
    const V *c = a.C + t.d->ip_coff;
    const int n = t.MT + 4 * (t.r4 ? KS4 : KS);
    for (int i = (int)threadIdx.x; i < n; i += NT) cp_async(&sm[i], &c[(t.m0 - (TAPS / 2 - 1) + i) & (t.Nc - 1)]);
  }
  // Persistent: CTA b works on items b, b + gridDim.x, ... of the launch's rows x gm tiles.  Each tile
  // reads ~1 K coarse samples and writes 4096 outputs; prefetching the next tile's samples keeps the
  // store stream going where a fresh CTA would first wait for its loads.
  __device__ static void run_tiles(const Args &a, unsigned gm, unsigned total, V *sm) {
    unsigned w = blockIdx.x;
    Tile cur = tile(a, w, gm);
    load(a, cur, sm);
    for (int st = 0; w < total; w += gridDim.x, st ^= 1) {
      cp_async_wait();
      __syncthreads();   // this tile's samples are in, and every warp is done with the other stage
      const unsigned wn = w + gridDim.x;
      Tile nxt = cur;
      if (wn < total) {
        nxt = tile(a, wn, gm);
        load(a, nxt, sm + (st ^ 1) * STAGE);
      }
      if (cur.live) {
        if (cur.r4) compute<true>(a, cur, sm + st * STAGE);
        else compute<false>(a, cur, sm + st * STAGE);
      }
      cur = nxt;
    }
  }
  // R4 = false (R >= 8): MMA rows = 8 consecutive coarse positions, columns = 8 consecutive phases.
  // R4 = true  (R == 4): the 8 columns are 2 coarse positions x 4 phases, the rows step by two coarse
  //   positions: acc[m0 + 2 i + dm][rho] = sum_t' c[m0 + 2 i + t' - (taps/2 - 1)] * h[t' - dm][rho],
  //   t' < taps + 1 (B holds the weights shifted by dm, zero outside).  A warp then covers 16 coarse
  //   positions per MMA block and runs over 2 L of them: the same 8 L outputs per warp.
  template <bool R4>
  __device__ static void compute(const Args &a, const Tile &tl, const V *sm) {
    constexpr int KSr = R4 ? KS4 : KS;
    constexpr int Lr = R4 ? 2 * L : L;              // coarse positions per warp run
    constexpr int MB = R4 ? 16 : 8;                 // coarse positions per MMA block
    const ScaleDesc &d = *tl.d;
    const int log2R = tl.log2R;
    const int R = 1 << log2R;
    const int Nc = tl.Nc;
    const int wpb = tl.wpb, rb = tl.rb, m0 = tl.m0;
    {
      const int tid = (int)threadIdx.x;
      const int wid = tid >> 5, lane = tid & 31;
      const int g = lane >> 2, q = lane & 3;
      const int pb = wid % wpb, j = wid / wpb;
      const int rho0 = R4 ? 0 : rb * 32 + pb * 8;
      const int ms = m0 + j * Lr;
      double bf[KSr];
#pragma unroll
      for (int ks = 0; ks < KSr; ++ks) {
        const int t = 4 * ks + q - (R4 ? (g >> 2) : 0);
        const int rho = R4 ? (g & 3) : rho0 + g;
        bf[ks] = (t >= 0 && t < TAPS) ? ldg(&a.wt[d.ip_woff + (size_t)t * R + rho]) : 0.0;
      }
      // re-modulation e^{2 pi i kc n / Np} of this lane's two outputs: table values for the first
      // block, then steps of e^{2 pi i kc 64 / Np ... } = one MMA block of coarse positions further
      const unsigned kc = (unsigned)d.ip_kc;
      const int mlane = R4 ? 2 * g + (q >> 1) : g;              // coarse position of this lane inside a block
      const int rlane = R4 ? 2 * (q & 1) : rho0 + 2 * q;        // first of its two adjacent phases
      const unsigned n00 = ((unsigned)(ms + mlane) << log2R) + (unsigned)rlane;
      V tw0 = nroot(a.nt, kc * n00);
      V tw1 = cmul(tw0, nroot(a.nt, kc));
      const V stepb = nroot(a.nt, (kc * (unsigned)MB) << log2R);
      const V *run = sm + j * Lr + (R4 ? 2 * g : g) + q;
      V *rowp = a.W + (size_t)d.row * a.n0;
#pragma unroll 4
      for (int mb = 0; mb < Lr / MB; ++mb) {
        if (ms + MB * mb >= Nc) break;                // warp-uniform: short coarse grids end inside the run
        double cr0 = 0, cr1 = 0, ci0 = 0, ci1 = 0;
#pragma unroll
        for (int ks = 0; ks < KSr; ++ks) {
          const V s = run[MB * mb + 4 * ks];
          dmma884(cr0, cr1, s.x, bf[ks]);
          dmma884(ci0, ci1, s.y, bf[ks]);
        }
        const int m = ms + MB * mb + mlane;
        const long long n = ((long long)m << log2R) + rlane;
        const V x0 = cmul(make_double2(cr0, ci0), tw0);
        const V x1 = cmul(make_double2(cr1, ci1), tw1);
        tw0 = cmul(tw0, stepb);
        tw1 = cmul(tw1, stepb);
        // Lanes q and q^1 hold outputs n .. n+3 (same m).  Stored as they sit, each 16-byte store
        // instruction fills every 32-byte sector half (measured: half the write rate).  The pair swaps
        // one value so that each instruction writes whole sectors: the even lane stores n, n+2, the odd
        // lane n+1, n+3.
        const bool odd = q & 1;
        const V snd = odd ? x0 : x1;
        const V rcv = make_double2(__shfl_xor_sync(0xffffffffu, snd.x, 1), __shfl_xor_sync(0xffffffffu, snd.y, 1));
        const long long na = odd ? n - 1 : n;
        V ya = odd ? rcv : x0;                      // output na
        V yb = odd ? x1 : rcv;                      // output na + 2
        if (m < Nc) {
          V *p = rowp + na;
          const bool sa = na < a.n0, sb = na + 2 < a.n0;
          if (EPI == EPI_MULCONJ) {
            if (sa) p[0] = cmul(p[0], cconj(ya));
            if (sb) p[2] = cmul(p[2], cconj(yb));
          } else {
            if (sa) st_stream(p, ya);
            if (sb) st_stream(p + 2, yb);
          }
        }
      }
    }
  }
};
#endif

// ---- Body: band product B[r] = x^[k] * conj(psi_ft) * norm / Np for pruned scales ------
template <typename T> struct BandArgs {
  const ScaleDesc *descs;
  const cx<T> *spec;
  cx<T> *Bbuf;
  Fam fam;
  unsigned N;
  int first;
};
template <typename T> struct BandBody {
  using V = cx<T>;
  using Args = BandArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  static constexpr int PER = 4;
  template <bool MORSE> HD static void fill(const Args &a, int bx, int by, int tid) {
    const ScaleDesc d = a.descs[a.first + by];
    const int K = 1 << d.log2K;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int r = (bx * PER + i) * NT + tid;
      if (r >= K) return;
      const int k = r - (r >= d.rsplit ? K : 0);
      V v = mk<T>(0, 0);
      if (k >= d.k_lo && k <= d.k_hi) v = band_value<T, MORSE>(a.fam, d, a.spec, (unsigned)k & (a.N - 1), k, a.N);
      a.Bbuf[d.boff + r] = v;
    }
  }
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) { fill<false>(a, bx, by, tid); }
};
// the band products of Morse rows: BandBody with the Morse response compiled in (inlined into BandBody
// itself, its log and expm1 take the kernel from 32 to 36 registers in fp32 and from 34 to 38 in fp64)
template <typename T> struct BandBodyMorse : BandBody<T> {
  using Args = typename BandBody<T>::Args;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    BandBody<T>::template fill<true>(a, bx, by, tid);
  }
};

// ---- Body: batched K-point FFT over matrix rows (N <= 1024): forward FFT of short
// signals, the c2c test hook, the Gaussian smoothing transforms ----------------------
template <typename T> struct RowsArgs {
  const void *in;      // T* if real_in else cx<T>*
  cx<T> *out;
  const cx<T> *tw;
  const double *grow;  // EPI_GAUSS: per-row coefficient (null: plain store)
  long long in_pitch, out_pitch, n_in, nout;
  double post;
  int nrows, real_in, n;
};

template <typename T, int K> struct RowsLoader {
  using V = cx<T>;
  const RowsArgs<T> *a;
  int row0;
  int base, stride;
  HD void begin(int base_, int stride_, int, int) { base = base_; stride = stride_; }
  HD V get(int b, int pos) const {
    const int row = row0 + b;
    if (row >= a->nrows || pos >= a->n_in) return mk<T>(0, 0);
    if (a->real_in) return mk<T>(ldg((const T *)a->in + (size_t)row * a->in_pitch + pos), (T)0);
    return ldg((const V *)a->in + (size_t)row * a->in_pitch + pos);
  }
  template <int R> HD void load(int b, V (&x)[R]) const {
#pragma unroll
    for (int i = 0; i < R; ++i) x[i] = get(b, base + i * stride);
  }
};
template <typename T> struct RowsStorer {
  using V = cx<T>;
  const RowsArgs<T> *a;
  int row0;
  template <int R> HD void store(int b, int ql, int qs, V (&x)[R]) const {
    const int row = row0 + b;
    if (row >= a->nrows) return;
#pragma unroll
    for (int c = 0; c < R; ++c) {
      const int q = ql + c * qs;
      if (q >= a->nout) continue;
      V v = x[c];
      if (a->grow) {
        Epilogue<T> e;
        e.mode = EPI_GAUSS; e.g = a->grow[row]; e.invn = 1.0 / (double)a->n; e.post = a->post; e.nfreq = a->n;
        v = e.apply(v, v, q);
      }
      a->out[(size_t)row * a->out_pitch + q] = v;
    }
  }
};
template <typename T, int K, int SIGN> struct RowsBody {
  static constexpr int NTB = TileCfg<T>::NT;   // threads per CTA of this kernel
  static constexpr int NT = NTB;
  using V = cx<T>;
  using Args = RowsArgs<T>;
  using LY = Lay<T, K>;
  static constexpr int NP = Plan<K>::NP;
  static constexpr int NPHASE = NP;
  static constexpr size_t SMEM = LY::BYTES;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *smraw) {
    V *sm = (V *)smraw;
    const int row0 = bx * LY::P;
    RowsStorer<T> st;
    st.a = &a;
    st.row0 = row0;
    RowsLoader<T, K> ld;
    ld.a = &a;
    ld.row0 = row0;
    if constexpr (NP == 1) {
      for (int b = tid; b < LY::P; b += NT) {
        V x[K];
#pragma unroll
        for (int i = 0; i < K; ++i) x[i] = ld.get(b, i);
        dftR<K, SIGN, T>(x);
        st.store(b, 0, 1, x);
      }
    } else if constexpr (PH == 0) {
      tile_first<T, K, SIGN>(sm, a.tw, ld, tid);
    } else if constexpr (PH == 1 && NP == 3) {
      tile_second<T, K, SIGN>(sm, a.tw, tid);
    } else {
      pass_last<T, K, SIGN>(sm, st, tid);
    }
  }
};

// ---- Body: direct O(N^2) transform for tiny padded lengths (Np < 32) ---------------
template <typename T> struct TinyArgs {
  const ScaleDesc *descs;
  const cx<T> *spec;
  cx<T> *W;
  Fam fam;
  long long n0;
  unsigned N;
  int first;
  int epi;
};
template <typename T> struct TinyBody {
  using V = cx<T>;
  using Args = TinyArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const ScaleDesc d = a.descs[a.first + by];
    const int n = bx * NT + tid;
    if (n >= a.n0) return;
    double sr = 0, si = 0;
    for (unsigned r = 0; r < a.N; ++r) {
      const int k = (int)r - (r >= a.N / 2 && a.N > 1 ? (int)a.N : 0);
      V v = band_value<T>(a.fam, d, a.spec, r, k, a.N);
      double sn, cs;
      sincospi_hd(2.0 * (double)((r * (unsigned)n) % a.N) / (double)a.N, &sn, &cs);
      sr += (double)v.x * cs - (double)v.y * sn;
      si += (double)v.x * sn + (double)v.y * cs;
    }
    V *dst = &a.W[(size_t)d.row * a.n0 + n];
    V val = mk<T>((T)sr, (T)si);
    *dst = a.epi == EPI_MULCONJ ? cmul(*dst, cconj(val)) : val;
  }
};
// forward DFT of a tiny real signal
template <typename T> struct TinyFwdArgs {
  const T *sig;
  cx<T> *spec;
  long long n0;
  unsigned N;
};
template <typename T> struct TinyFwdBody {
  using Args = TinyFwdArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int, int, int tid, void *) {
    if ((unsigned)tid >= a.N) return;
    double sr = 0, si = 0;
    for (unsigned n = 0; n < a.N && (long long)n < a.n0; ++n) {
      double sn, cs;
      sincospi_hd(2.0 * (double)(((unsigned)tid * n) % a.N) / (double)a.N, &sn, &cs);
      sr += (double)a.sig[n] * cs;
      si -= (double)a.sig[n] * sn;
    }
    a.spec[tid] = mk<T>((T)sr, (T)si);
  }
};


// ---- Body: icwt reduction  out[n] (+)= sum_j Re(W[j,n]) / sqrt(s_j)   (wavelet.py:169-170) ----
template <typename T> struct IcwtArgs {
  const cx<T> *W;
  const double *inv_sqrt_s;   // per row: 1 / sqrt(s_j)
  double *out;
  long long n, pitch;
  int rows, accumulate;
  int rows_per_block;         // gridDim.y blocks of rows; > 1 block: partial sums meet in `out` by atomics
};
// One column per thread, rows in blocks of `rows_per_block` (blockIdx.y), 8 independent loads in
// flight per thread: a streaming read of W at HBM rate (4.29 GB at config 2).
template <typename T> struct IcwtBody {
  using Args = IcwtArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long n = (long long)bx * NT + tid;
    if (n >= a.n) return;
    const int j0 = by * a.rows_per_block;
    const int j1 = j0 + a.rows_per_block < a.rows ? j0 + a.rows_per_block : a.rows;
    const cx<T> *p = a.W + (size_t)j0 * a.pitch + n;
    double acc0 = 0, acc1 = 0;
    int j = j0;
    for (; j + 8 <= j1; j += 8) {
      double v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = (double)ldg(&p[(size_t)u * a.pitch]).x;
#pragma unroll
      for (int u = 0; u < 8; u += 2) {
        acc0 += v[u] * a.inv_sqrt_s[j + u];
        acc1 += v[u + 1] * a.inv_sqrt_s[j + u + 1];
      }
      p += (size_t)8 * a.pitch;
    }
    for (; j < j1; ++j, p += a.pitch) acc0 += (double)ldg(p).x * a.inv_sqrt_s[j];
    const double acc = acc0 + acc1;
    if (a.rows_per_block >= a.rows) {
      a.out[n] = a.accumulate ? a.out[n] + acc : acc;
    } else {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
      atomicAdd(&a.out[n], acc);
#else
      a.out[n] += acc;
#endif
    }
  }
};

// ---- Body: coherence inputs (wavelet.py:506-514) ---------------------------------------
//   C   = (|W1|^2 + i |W2|^2) / s   (two real fields packed into one complex field: the
//         smoothing filter is real, so one complex transform smooths both)
//   A12 = W1 conj(W2) / s,   aWCT = angle(W1 conj(W2))
// in the engine type T; the angle is written as double whatever T is
template <typename T> struct WctPrepArgs {
  const cx<T> *W1, *W2;
  const double *scale;   // per row
  cx<T> *C, *A12;
  double *aWCT;          // may be null
  long long n;
};
template <typename T> struct WctPrepBody {
  using Args = WctPrepArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long n = (long long)bx * NT + tid;
    if (n >= a.n) return;
    const size_t i = (size_t)by * a.n + n;
    const cx<T> w1 = a.W1[i], w2 = a.W2[i];
    const T s = (T)a.scale[by];
    const cx<T> w12 = cmul(w1, cconj(w2));
    a.C[i] = mk<T>((w1.x * w1.x + w1.y * w1.y) / s, (w2.x * w2.x + w2.y * w2.y) / s);
    a.A12[i] = mk<T>(w12.x / s, w12.y / s);
    if (a.aWCT) {
      if constexpr (sizeof(T) == 8) a.aWCT[i] = atan2(w12.y, w12.x);
      else a.aWCT[i] = (double)atan2f(w12.y, w12.x);
    }
  }
};

// ---- Body: white-noise surrogates on the device (seeded mode of the Monte-Carlo significance) ----
// Counter-based Philox4x32-10 (Salmon et al. 2011): sample pair (2j, 2j+1) of series `ser` of
// surrogate unit `unit` (a pair of the coherence test, a triple of the partial / multiple
// coherence test) is a pure function of (seed, unit, ser, j) -- independent of the launch
// geometry, of the rank that draws it and of how the units are batched.  Two 53-bit uniforms ->
// two standard normals (Box-Muller).  The reference's surrogates are white noise as well
// (helpers.py:146-173 filters a length-1 axis, SURVEY 8a row 10); this mode reproduces their
// distribution, not numpy's bit stream (the host-RNG mode does that).  The draw is in double for
// every T: the fp32 surrogates are the fp64 ones rounded.
// Counter words: (j lo, j hi, unit lo, c3).  Pairs: c3 = (unit hi << 1) | ser.  Triples:
// c3 = 2^31 | (unit hi << 2) | ser, a tag bit that pairs below 2^62 never set, so triple t and pair
// t of one seed share no series.
template <typename T> struct NoiseArgs {
  T *out;                   // [n_units][nser][n]
  unsigned long long seed;
  long long unit0;          // global index of the first unit
  long long n;
  int n_units;
  int nser;                 // 2 (pairs) or 3 (triples)
};
HD void philox4x32_10(unsigned c0, unsigned c1, unsigned c2, unsigned c3, unsigned k0, unsigned k1, unsigned (&o)[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned long long p0 = (unsigned long long)0xD2511F53u * c0;
    const unsigned long long p1 = (unsigned long long)0xCD9E8D57u * c2;
    const unsigned n0 = (unsigned)(p1 >> 32) ^ c1 ^ k0, n1 = (unsigned)p1;
    const unsigned n2 = (unsigned)(p0 >> 32) ^ c3 ^ k1, n3 = (unsigned)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  o[0] = c0; o[1] = c1; o[2] = c2; o[3] = c3;
}
// Two standard normals (Box-Muller) from one Philox4x32-10 block: two 53-bit uniforms in (0, 1),
// offset by half an ulp so that log() is finite
HD void philox_normals(const unsigned (&o)[4], double &e0, double &e1) {
  const double u1 = ((double)(o[0] >> 5) * 67108864.0 + (double)(o[1] >> 6) + 0.5) * (1.0 / 9007199254740992.0);
  const double u2 = ((double)(o[2] >> 5) * 67108864.0 + (double)(o[3] >> 6) + 0.5) * (1.0 / 9007199254740992.0);
  const double r = sqrt(-2.0 * log(u1));
  double sn, cs;
  sincospi_hd(2.0 * u2, &sn, &cs);
  e0 = r * cs;
  e1 = r * sn;
}
template <typename T> struct NoiseBody {
  using Args = NoiseArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long j = (long long)bx * NT + tid;        // sample pair index
    if (2 * j >= a.n) return;
    const long long unit = a.unit0 + by / a.nser;
    const int ser = by % a.nser;
    const unsigned hi = (unsigned)((unsigned long long)unit >> 32);
    const unsigned c3 = a.nser == 2 ? (hi << 1) | (unsigned)ser : 0x80000000u | (hi << 2) | (unsigned)ser;
    unsigned o[4];
    philox4x32_10((unsigned)j, (unsigned)((unsigned long long)j >> 32), (unsigned)unit, c3,
                  (unsigned)a.seed, (unsigned)(a.seed >> 32), o);
    double e0, e1;
    philox_normals(o, e0, e1);
    T *dst = a.out + (size_t)by * a.n + 2 * j;
    dst[0] = (T)e0;
    if (2 * j + 1 < a.n) dst[1] = (T)e1;
  }
};

// ---- Body: phase-randomised surrogates of the data (Theiler et al. 1992; Prichard & Theiler 1994) --
// For a real series x of length n with X = FFT_n(x) (the series' own length, not padded), surrogate
// unit u of a series in phase group g is x' = Re IFFT_n(X') with
//   X'_k = X_k e^{i phi(u,g,k)} for 1 <= k < n/2,   X'_{n-k} = conj(X'_k),   X'_0 = X_0,
//   X'_{n/2} = X_{n/2} for even n.
// |X'| = |X| bin by bin: the power spectrum, the mean and the variance of the series are kept.
// Series of one group share phi, so their cross spectrum X_a conj(X_b), hence their coherence, is
// kept too; series of different groups get independent phases.  phi = 2 pi U, U uniform in (0, 1)
// (53 bits of one Philox4x32-10 block, NoiseBody's conversion), a pure function of (seed, u, g, k):
// independent of the launch geometry, of the batching, of the rank and of which series uses it.
// Counter words: (k, g, u lo, 2^31 | (u hi << 2) | 3).  The white-noise pairs never set bit 31 of the
// last word (units below 2^62) and the triples never set both of its low bits (ser <= 2), so for
// 0 <= u < 2^61 no counter coincides with one of NoiseBody's.  k < 2^32 and 0 <= g < 2^31.
// One thread per bin pair (k, n - k) of one series of one unit: the Hermitian half is written, not
// recomputed.  fp64 whatever the coherence precision.
struct PhaseRotArgs {
  const double2 *spec;      // [nser][n] spectra of the data
  double2 *out;             // [n_units][nser][n] rotated spectra
  unsigned long long seed;
  long long unit0;          // global index of the first unit
  long long n;
  int nser;
  int group[3];             // phase group of each series
};
struct PhaseRotBody {
  using Args = PhaseRotArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long k = (long long)bx * NT + tid;
    if (2 * k > a.n) return;
    const int ser = by % a.nser;
    const double2 *src = a.spec + (size_t)ser * a.n;
    double2 *dst = a.out + (size_t)by * a.n;
    if (k == 0 || 2 * k == a.n) {   // mean and Nyquist bin stay
      dst[k] = src[k];
      return;
    }
    const unsigned long long unit = (unsigned long long)(a.unit0 + by / a.nser);
    unsigned o[4];
    philox4x32_10((unsigned)k, (unsigned)a.group[ser], (unsigned)unit, 0x80000000u | ((unsigned)(unit >> 32) << 2) | 3u,
                  (unsigned)a.seed, (unsigned)(a.seed >> 32), o);
    const double u = ((double)(o[0] >> 5) * 67108864.0 + (double)(o[1] >> 6) + 0.5) * (1.0 / 9007199254740992.0);
    double sn, cs;
    sincospi_hd(2.0 * u, &sn, &cs);
    const double2 x = src[k];
    const double2 r = make_double2(x.x * cs - x.y * sn, x.x * sn + x.y * cs);
    dst[k] = r;
    dst[a.n - k] = make_double2(r.x, -r.y);
  }
};

// ---- Bodies: AR(1) red-noise surrogates on the device (the power test's red-noise null) ----------
// Unit u of length n is x = m + sigma z with z[0] = e[0], z[i] = g z[i-1] + sqrt(1 - g^2) e[i] (the
// background of Torrence & Compo 1998, section 4), |g| < 1.  e[2j], e[2j+1] are the two normals of
// one Philox4x32-10 block (philox_normals, NoiseBody's conversion), a pure function of (seed, s, u,
// j): counter words (j, 2^31 | s, u lo, 2^31 | (u hi << 2) | 3), s the series tag (0, 1 or 2).  Tag 0
// is the power test's stream; the cross-wavelet and coherence tests draw their second series under
// tag 1 and the third series of the partial and multiple coherence under tag 2, so the series of one
// unit are independent even with equal parameters, and the first series is the power test's unit.
// PhaseRotBody's second word is a phase group below 2^31 and NoiseBody's a sample index below 2^26,
// so bit 31 of the second word keeps every tag apart from both for 0 <= u < 2^61 (j < 2^31), and the
// tag's two low bits keep the tags apart from each other.
// The recurrence is a linear scan over the whole series: z_end = g^L z_start + b over a stretch of L
// samples, b its end state from a zero start.  A thread owns AR1_CH consecutive samples (whole
// normal pairs), a CTA NT of those stretches.  Ar1BlockBody forms every CTA's (g^L, b), Ar1CarryBody
// chains them per unit into each CTA's carry-in, Ar1WriteBody redraws the normals from the thread's
// carry-in and writes x once.  The carries are in double and |g| < 1, so a rounding error decays
// along the series instead of growing.  The draw is in double for every T (fp32: the fp64 surrogate
// rounded).  The stretches depend on NT, the draws (seed, u, j) do not.
constexpr int AR1_CH = 32;   // samples per thread (even)
template <typename T> struct Ar1Args {
  T *out;                   // [n_units][nser][n]: unit by's series at out + by nser n
  double *blk;              // [n_units][nblk][2]: (g^L, b) of each CTA, then (., carry-in)
  unsigned long long seed;
  long long unit0;          // global index of the first unit
  long long n;
  double g, s, m, sigma;    // s = sqrt(1 - g^2)
  int nblk, n_units;
  int nser;                 // series per unit in out (the pairs of the cross test: 2)
  unsigned tag;             // series tag s of the counter
};
// Samples [i0, i1) of unit `unit` from the state z before i0: the state after i1 - 1, and x into dst
// (null: nothing written)
template <typename T>
HD double ar1_run(const Ar1Args<T> &a, unsigned long long unit, long long i0, long long i1, double z, T *dst) {
  for (long long i = i0; i < i1; i += 2) {
    unsigned o[4];
    philox4x32_10((unsigned)(i >> 1), 0x80000000u | a.tag, (unsigned)unit, 0x80000000u | ((unsigned)(unit >> 32) << 2) | 3u,
                  (unsigned)a.seed, (unsigned)(a.seed >> 32), o);
    double e0, e1;
    philox_normals(o, e0, e1);
    z = i == 0 ? e0 : fma(a.g, z, a.s * e0);
    if (dst) dst[i] = (T)(a.m + a.sigma * z);
    if (i + 1 < i1) {
      z = fma(a.g, z, a.s * e1);
      if (dst) dst[i + 1] = (T)(a.m + a.sigma * z);
    }
  }
  return z;
}
// the samples [i0, i1) of thread tid of CTA bx, and g^(i1 - i0)
template <typename T> HD double ar1_span(const Ar1Args<T> &a, int bx, int tid, long long &i0, long long &i1) {
  i0 = ((long long)bx * NT + tid) * AR1_CH;
  i1 = i0 + AR1_CH < a.n ? i0 + AR1_CH : a.n;
  double p = 1.0;
  for (long long i = i0; i < i1; ++i) p *= a.g;
  return p;
}
// (g^L, b) of the thread's stretch into sm [2][NT]
template <typename T> HD void ar1_local(const Ar1Args<T> &a, int bx, int by, int tid, double *sm) {
  long long i0, i1;
  sm[tid] = ar1_span(a, bx, tid, i0, i1);
  sm[NT + tid] = ar1_run<T>(a, (unsigned long long)(a.unit0 + by), i0, i1, 0.0, nullptr);
}
template <typename T> struct Ar1BlockBody {   // grid (nblk, n_units)
  using Args = Ar1Args<T>;
  static constexpr int NPHASE = 2;
  static constexpr size_t SMEM = 2 * NT * sizeof(double);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    double *sm = (double *)smraw;
    if constexpr (PH == 0) {
      ar1_local(a, bx, by, tid, sm);
    } else if (tid == 0) {
      double A = 1.0, B = 0.0;
      for (int t = 0; t < NT; ++t) {
        B = fma(sm[t], B, sm[NT + t]);
        A *= sm[t];
      }
      double *d = a.blk + 2 * ((size_t)by * a.nblk + bx);
      d[0] = A;
      d[1] = B;
    }
  }
};
struct Ar1CarryArgs { double *blk; int nblk, n_units; };
struct Ar1CarryBody {   // one thread per unit
  using Args = Ar1CarryArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const int u = bx * NT + tid;
    if (u >= a.n_units) return;
    double *d = a.blk + 2 * (size_t)u * a.nblk;
    double z = 0.0;
    for (int b = 0; b < a.nblk; ++b) {
      const double A = d[2 * b], B = d[2 * b + 1];
      d[2 * b + 1] = z;
      z = fma(A, z, B);
    }
  }
};
template <typename T> struct Ar1WriteBody {   // grid (nblk, n_units)
  using Args = Ar1Args<T>;
  static constexpr int NPHASE = 3;
  static constexpr size_t SMEM = 2 * NT * sizeof(double);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    double *sm = (double *)smraw;
    if constexpr (PH == 0) {
      ar1_local(a, bx, by, tid, sm);
    } else if constexpr (PH == 1) {
      if (tid == 0) {   // each thread's carry-in into sm[NT + t]
        double z = a.blk[2 * ((size_t)by * a.nblk + bx) + 1];
        for (int t = 0; t < NT; ++t) {
          const double A = sm[t], B = sm[NT + t];
          sm[NT + t] = z;
          z = fma(A, z, B);
        }
      }
    } else {
      long long i0, i1;
      ar1_span(a, bx, tid, i0, i1);
      ar1_run<T>(a, (unsigned long long)(a.unit0 + by), i0, i1, sm[NT + tid], a.out + (size_t)by * a.n * a.nser);
    }
  }
};

// ---- Body: out[i] = (T)(Re in[i] * f): the surrogates of the inverse transform, in the engine type --
template <typename T> struct RealPartArgs { const double2 *in; T *out; long long count; double f; };
template <typename T> struct RealPartBody {
  using Args = RealPartArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const long long i = (long long)bx * NT + tid;
    if (i < a.count) a.out[i] = (T)(a.in[i].x * a.f);
  }
};

// ---- Body: scale-axis boxcar (mothers.py:100-102; scipy convolve2d 'same', zero fill) ------
//   out[i] = sum_t win[t] * in[i - (t - off)],  off = (K-1)//2, rows outside [0, m) are zero
// Sums in the engine type T, like WctFinalBody; any K (no shared memory).
template <typename T> struct BoxcarArgs {
  const cx<T> *in;
  cx<T> *out;
  const double *win;
  long long n;
  int rows, K;
};
template <typename T> struct BoxcarBody {
  using Args = BoxcarArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long n = (long long)bx * NT + tid;
    if (n >= a.n) return;
    const int off = (a.K - 1) / 2;
    T re = 0, im = 0;
    for (int t = 0; t < a.K; ++t) {
      const int q = by - (t - off);
      if (q < 0 || q >= a.rows) continue;
      const cx<T> v = a.in[(size_t)q * a.n + n];
      const T w = (T)a.win[t];
      re += w * v.x;
      im += w * v.y;
    }
    a.out[(size_t)by * a.n + n] = mk<T>(re, im);
  }
};

// ---- selection bits of the cluster test (cwtb_coherence*_cluster_test) -------------------------
// Point (j, n) of a map R is selected where R[j, n] is finite, R[j, n] > thr[j] (a NaN thr selects
// nothing) and lo[j] <= n < hi[j].  The selection of a map is a bitmask [rows][words] of uint32,
// words = ceil(n / 32): column n is bit n % 32 of word n / 32, the bits past the last column are 0.
struct SelArgs {
  unsigned *bits;           // [rows][words], or null: no selection wanted
  const double *thr;        // [rows]
  const long long *lo, *hi; // [rows]
  long long words;
  int measure;              // Wct3FinalBody: the measure selected (0 partial, 1 multiple)
};
HD bool cluster_sel(const SelArgs &s, int row, long long n, double r) {
  return isfinite(r) && r > s.thr[row] && n >= s.lo[row] && n < s.hi[row];
}
// The lanes of a warp whose column lies below n_valid, for warps whose lanes hold chunks of cw
// consecutive columns (lane l: column c0 + l % cw, c0 a multiple of cw), cw in {8, 16, 32}
HD unsigned sel_lanes(int cw, long long n_valid) {
  const unsigned c = n_valid >= cw ? (cw == 32 ? ~0u : (1u << cw) - 1u) : (1u << n_valid) - 1u;
  unsigned m = 0;
  for (int h = 0; h < 32; h += cw) m |= c << h;
  return m;
}
// Selection bit p of (row, n) into s.bits.  On the device the lanes `lanes` (sel_lanes) vote and
// the first lane of each chunk stores its cw bits as one 8-, 16- or 32-bit word at byte n / 8: one
// writer per chunk, no atomics.  The emulation build sets or clears the bit itself.  A lane of a
// row < 0 votes and stores nothing.
HD void sel_store(const SelArgs &s, int row, long long n, int cw, bool p, unsigned lanes) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  const unsigned b = __ballot_sync(lanes, p);
  if (row >= 0 && (n & (cw - 1)) == 0) {
    const unsigned v = b >> ((threadIdx.x & 31) & ~(unsigned)(cw - 1));
    unsigned char *dst = (unsigned char *)(s.bits + (size_t)row * s.words) + (n >> 3);
    if (cw == 32) *(unsigned *)dst = v;
    else if (cw == 16) *(unsigned short *)dst = (unsigned short)v;
    else *dst = (unsigned char)v;
  }
#else
  (void)cw;
  (void)lanes;
  if (row < 0) return;
  unsigned &w = s.bits[(size_t)row * s.words + (n >> 5)];
  const unsigned bit = 1u << (n & 31);
  w = p ? (w | bit) : (w & ~bit);
#endif
}

// ---- Body: selection bits of a resident double field (the observed map of a cluster test) -------
// One thread per column of row by; a warp's lanes are 32 aligned columns.
struct ThreshBitsArgs { const double *R; SelArgs sel; long long n; };
struct ThreshBitsBody {
  using Args = ThreshBitsArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long n0 = (long long)bx * NT + (tid & ~31), n = n0 + (tid & 31);
    if (n0 >= a.n) return;   // the whole warp
    const bool p = n < a.n && cluster_sel(a.sel, by, n, ld_stream(&a.R[(size_t)by * a.n + n]));
    sel_store(a.sel, by, n, 32, p, ~0u);
  }
};

// ---- the wavelet power |W|^2 of a coefficient, as the power test compares and selects it ---------
// Every read of the resident power's tests forms P through this one function, the observed and the
// surrogate power alike, so their comparison is bit-consistent: double products rounded on their own
// (no contraction), exact for the widened parts of an fp32 W.  The same arithmetic as CxView's |F|^2.
template <typename T> HD double power_of(const cx<T> &v) { return norm2_rn((double)v.x, (double)v.y); }

// ---- Body: a surrogate unit's power against the resident power (cwtb_power_surrogate_counts /
// _cluster_test) ---------------------------------------------------------------------------------
// One thread per column of row by, a warp's lanes 32 aligned columns.  With cnt: k += 1 where the
// unit's P_i >= P_obs or P_i is not finite (count_exceed's rule; no atomics: the count launches of
// successive units run in order on one stream).  SEL: the selection bits of P (cluster_sel).  The
// observed map's bits are this kernel on the resident W without counters.
template <typename T> struct PowerCountArgs {
  const cx<T> *W;           // [rows][n] the unit's transform
  const cx<T> *obs;         // [rows][n] the resident W (with cnt)
  unsigned *cnt;            // [rows][n] exceedance counters, or null
  SelArgs sel;
  long long n;
};
template <typename T, bool SEL> struct PowerCountBody {
  using Args = PowerCountArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long n0 = (long long)bx * NT + (tid & ~31), n = n0 + (tid & 31);
    if (n0 >= a.n) return;   // the whole warp
    bool p = false;
    if (n < a.n) {
      const size_t o = (size_t)by * a.n + n;
      const double P = power_of<T>(ld_stream(&a.W[o]));
      if (a.cnt && (!isfinite(P) || P >= power_of<T>(ld_stream(&a.obs[o])))) a.cnt[o] += 1u;
      p = SEL && cluster_sel(a.sel, by, n, P);
    }
    if constexpr (SEL) sel_store(a.sel, by, n, 32, p, ~0u);
  }
};

// ---- Body: coherence  WCT = |S12|^2 / (S1 S2)  after the scale boxcar; optional histogram
// of floor(WCT * nbins) over masked points (wavelet.py:513, 624-630) ---------------------
// Fields, staging and sums in the engine type T; WCT is written (and binned) as double.
// Counting (cnt given, Monte-Carlo mode): every row is finished, not only those below maxscale,
// and each point's counter goes up by one where the surrogate's value reaches the observed one
// (count_exceed).  The histogram is binned as without counting.
template <typename T> struct WctFinalArgs {
  const cx<T> *C, *A12;     // time-smoothed fields
  const double *win;
  double *WCT;              // may be null (Monte-Carlo mode)
  const unsigned char *mask;   // [rows][n], may be null
  unsigned long long *hist;    // [rows][nbins], may be null
  long long n;
  int rows, K, maxscale, nbins;
  const double *obs;        // observed WCT [rows][n] (the resident coherence), with cnt
  unsigned *cnt;            // exceedance counters [rows][n], or null
  SelArgs sel;              // selection bits of every row (the SEL instantiation)
};
// One surrogate value r2 against the observed value at point o: an exceedance where r2 >= obs or
// r2 is not finite (the conservative choice).  No atomics: within a launch every point belongs to
// one thread, and the final launches of successive surrogate units run in order on one stream.
HD void count_exceed(unsigned *cnt, const double *obs, size_t o, double r2) {
  if (!isfinite(r2) || r2 >= obs[o]) cnt[o] += 1u;
}
// Tile: RS = 32 output rows x CW = 32 columns.  Phase 0 stages the RS + K - 1 input rows of both
// time-smoothed fields for these columns in shared memory (each input element is read from global
// memory (RS + K - 1) / RS times instead of K times); in phase 1 a thread produces 4 consecutive
// rows of one column, so every staged value feeds up to four accumulators.
// SEL: the instantiation that writes selection bits (a.sel); the others ignore a.sel, so their code
// is that of a kernel without them.
template <typename T, int KMAX_, bool SEL = false> struct WctFinalBody {
  using Args = WctFinalArgs<T>;
  using V = cx<T>;
  static constexpr int NPHASE = 2;
  static constexpr int RS = 32, CW = 32, KMAX = KMAX_, RG = 4;   // KMAX sizes the shared memory
  static constexpr size_t SMEM = (size_t)2 * (RS + KMAX - 1) * CW * sizeof(V) + KMAX * sizeof(T);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    const int K = a.K, off = (K - 1) / 2;
    const int nrow = RS + K - 1;
    V *sc = (V *)smraw;                               // [nrow][CW] of C
    V *sx = sc + (size_t)(RS + KMAX - 1) * CW;        // [nrow][CW] of A12
    T *sw = (T *)(sx + (size_t)(RS + KMAX - 1) * CW);
    const int i0 = by * RS;
    const long long n0 = (long long)bx * CW;
    // Monte-Carlo mode without counting or selection bits: rows below maxscale only
    const int rows_out = SEL || a.WCT || a.cnt ? a.rows : a.maxscale;
    if (i0 >= rows_out) return;
    const int qlo = i0 + off - K + 1;
    if constexpr (PH == 0) {
      for (int idx = tid; idx < nrow * CW; idx += NT) {
        const int r = idx / CW, col = idx % CW;
        const int q = qlo + r;
        const long long n = n0 + col;
        V c = mk<T>(0, 0), x = c;
        if (q >= 0 && q < a.rows && n < a.n) {
          c = a.C[(size_t)q * a.n + n];
          x = a.A12[(size_t)q * a.n + n];
        }
        sc[idx] = c;
        sx[idx] = x;
      }
      for (int t = tid; t < K; t += NT) sw[t] = (T)a.win[t];
    } else {
      for (int task = tid; task < (RS / RG) * CW; task += NT) {
        const int col = task % CW, g = task / CW;
        const long long n = n0 + col;
        if (n >= a.n) continue;
        T cr[RG] = {0, 0, 0, 0}, ci[RG] = {0, 0, 0, 0}, xr[RG] = {0, 0, 0, 0}, xi[RG] = {0, 0, 0, 0};
        // staged row u feeds output row i0 + RG g + e with tap t = e + K - 1 - (u - RG g)
        for (int du = 0; du < K + RG - 1; ++du) {
          const int u = RG * g + du;
          const V c = sc[u * CW + col], x = sx[u * CW + col];
#pragma unroll
          for (int e = 0; e < RG; ++e) {
            const int t = e + K - 1 - du;
            if (t >= 0 && t < K) {
              const T w = sw[t];
              cr[e] += w * c.x; ci[e] += w * c.y;
              xr[e] += w * x.x; xi[e] += w * x.y;
            }
          }
        }
#pragma unroll
        for (int e = 0; e < RG; ++e) {
          const int i = i0 + RG * g + e;
          if (i >= rows_out) break;
          // the ratio in double: numerator and denominator go as amplitude^4 and would leave
          // float's range near 2^+-31 times a unit series, the fields (amplitude^2) do not
          const double r2 = ((double)xr[e] * xr[e] + (double)xi[e] * xi[e]) / ((double)cr[e] * ci[e]);
          const size_t o = (size_t)i * a.n + n;
          if (a.WCT) a.WCT[o] = r2;
          if (a.cnt) count_exceed(a.cnt, a.obs, o, r2);
          // a warp's lanes are the CW = 32 columns of one row here (rows_out = rows: no lane breaks)
          if constexpr (SEL) sel_store(a.sel, i, n, CW, cluster_sel(a.sel, i, n, r2), sel_lanes(CW, a.n - n0));
          if (a.hist && i < a.maxscale && a.mask[o] && r2 == r2) {
            int bin = (int)floor(r2 * a.nbins);
            bin = bin < 0 ? 0 : (bin >= a.nbins ? a.nbins - 1 : bin);
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
            atomicAdd(&a.hist[(size_t)i * a.nbins + bin], 1ull);
#else
            a.hist[(size_t)i * a.nbins + bin] += 1ull;
#endif
          }
        }
      }
    }
  }
};

// ---- Body: partial / multiple coherence inputs of three series y, x1, x2 -------------------
//   A  = (|Wy|^2 + i |W1|^2) / s,   B = |W2|^2 / s   (real autos packed as in WctPrepBody)
//   Xy1 = Wy conj(W1) / s,   Xy2 = Wy conj(W2) / s,   X12 = W1 conj(W2) / s
// Each point's three coefficients are read once; the crosses may be written over the transforms
// (Xy1 over Wy, Xy2 over W1, X12 over W2): every thread reads its point before it writes it.
template <typename T> struct Wct3PrepArgs {
  const cx<T> *Wy, *W1, *W2;
  const double *scale;   // per row
  cx<T> *A, *B, *Xy1, *Xy2, *X12;
  long long n;
};
template <typename T> struct Wct3PrepBody {
  using Args = Wct3PrepArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long n = (long long)bx * NT + tid;
    if (n >= a.n) return;
    const size_t i = (size_t)by * a.n + n;
    const cx<T> wy = a.Wy[i], w1 = a.W1[i], w2 = a.W2[i];
    const T s = (T)a.scale[by];
    const cx<T> y1 = cmul(wy, cconj(w1)), y2 = cmul(wy, cconj(w2)), x12 = cmul(w1, cconj(w2));
    a.A[i] = mk<T>((wy.x * wy.x + wy.y * wy.y) / s, (w1.x * w1.x + w1.y * w1.y) / s);
    a.B[i] = mk<T>((w2.x * w2.x + w2.y * w2.y) / s, (T)0);
    a.Xy1[i] = mk<T>(y1.x / s, y1.y / s);
    a.Xy2[i] = mk<T>(y2.x / s, y2.y / s);
    a.X12[i] = mk<T>(x12.x / s, x12.y / s);
  }
};

// ---- Body: scale boxcar of the five time-smoothed fields of Wct3PrepBody, then
//   RP2 = |Sy1 S2 - Sy2 conj(S12)|^2 / ((Sy S2 - |Sy2|^2) (S1 S2 - |S12|^2))       (partial)
//   RM2 = (S2 |Sy1|^2 + S1 |Sy2|^2 - 2 Re(Sy1 S12 conj(Sy2))) / (Sy (S1 S2 - |S12|^2))  (multiple)
// The second is 1 - det G3 / (Sy (S1 S2 - |S12|^2)) with the 1 - x cancelled exactly.  No clamping:
// a zero or negative denominator gives inf / NaN.  The fields are widened to double when they are
// staged, and the boxcar sums and the combination run in double for every T: in fp32 the
// differences above cancel badly, and the kernel is bound by its global reads, not by arithmetic.
// Tile: RS output rows x CW columns; phase 0 stages the RS + K - 1 input rows of the five fields
// for these columns, phase 1 gives each of the NT = (RS / RG) CW threads RG consecutive rows of
// one column.
// PP, if given, receives the partial phase atan2(u.y, u.x): the angle of the smoothed partial cross
// spectrum of y and x1 with x2 removed, in the sign convention of aWCT (angle of W_y conj(W_x1)).
// A zero u gives 0 (np.angle(0)), a NaN gives NaN.
// Monte-Carlo mode (RP2, RM2 and PP all null): only the rows below maxscale and only the measures
// whose histogram is given; a measure's histogram counts floor(R2 nbins), clamped to
// [0, nbins - 1], over the points with mask != 0.  A non-finite R2 (a zero denominator) is not
// counted.  Counting (cntP or cntM given, Monte-Carlo mode): every row is finished, and each
// measure with counters counts its exceedances of the observed field (count_exceed).
template <typename T> struct Wct3FinalArgs {
  const cx<T> *A, *B, *Xy1, *Xy2, *X12;   // time-smoothed fields
  const double *win;
  double *RP2, *RM2, *PP;                // [rows][n], any may be null
  const unsigned char *mask;             // [rows][n], Monte-Carlo mode
  unsigned long long *histP, *histM;     // [rows][nbins], either may be null
  long long n;
  int rows, K, maxscale, nbins;
  const double *obsP, *obsM;             // observed RP2 / RM2 [rows][n], with the counters
  unsigned *cntP, *cntM;                 // exceedance counters [rows][n], either may be null
  SelArgs sel;                           // selection bits of sel.measure, every row (SEL)
};
// one count for R2 in its row's histogram; non-finite R2 is skipped before any conversion to int
HD void hist_count(unsigned long long *hist, int row, int nbins, double r2) {
  if (!isfinite(r2)) return;
  const double x = floor(r2 * nbins);
  const int bin = x < 0.0 ? 0 : (x >= (double)nbins ? nbins - 1 : (int)x);
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  atomicAdd(&hist[(size_t)row * nbins + bin], 1ull);
#else
  hist[(size_t)row * nbins + bin] += 1ull;
#endif
}
// SEL: as WctFinalBody's, for the measure a.sel.measure
template <typename T, int KMAX_, int RS_, int CW_, bool SEL = false> struct Wct3FinalBody {
  using Args = Wct3FinalArgs<T>;
  using V = cx<T>;
  static constexpr int NPHASE = 2;
  static constexpr int NF = 5, RS = RS_, CW = CW_, KMAX = KMAX_, RG = 4;
  static_assert((RS / RG) * CW == NT, "one task per thread");
  static constexpr size_t PLANE = (size_t)(RS + KMAX - 1) * CW;   // double2 per staged field
  static constexpr size_t SMEM = NF * PLANE * sizeof(double2) + KMAX * sizeof(double);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    const int K = a.K, off = (K - 1) / 2;
    const int nrow = RS + K - 1;
    double2 *st = (double2 *)smraw;                   // NF planes [nrow][CW]
    double *sw = (double *)(st + NF * PLANE);
    const int i0 = by * RS;
    const long long n0 = (long long)bx * CW;
    const int rows_out = SEL || a.RP2 || a.RM2 || a.PP || a.cntP || a.cntM ? a.rows : a.maxscale;
    if (i0 >= rows_out) return;
    const int qlo = i0 + off - K + 1;
    if constexpr (PH == 0) {
      const V *src[NF] = {a.A, a.B, a.Xy1, a.Xy2, a.X12};
      for (int idx = tid; idx < nrow * CW; idx += NT) {
        const int r = idx / CW, col = idx % CW;
        const int q = qlo + r;
        const long long n = n0 + col;
        const bool in = q >= 0 && q < a.rows && n < a.n;
        const size_t g = in ? (size_t)q * a.n + n : 0;
#pragma unroll
        for (int f = 0; f < NF; ++f) {
          double2 v = mk<double>(0.0, 0.0);
          if (in) {
            const V x = src[f][g];
            v = mk<double>((double)x.x, (double)x.y);
          }
          st[f * PLANE + idx] = v;
        }
      }
      for (int t = tid; t < K; t += NT) sw[t] = a.win[t];
    } else {
      const int task = tid, col = task % CW, grp = task / CW;
      const long long n = n0 + col;
      if (n >= a.n) return;
      double acc[NF][2][RG];
#pragma unroll
      for (int f = 0; f < NF; ++f)
#pragma unroll
        for (int e = 0; e < RG; ++e) acc[f][0][e] = acc[f][1][e] = 0.0;
      // staged row u feeds output row i0 + RG grp + e with tap t = e + K - 1 - (u - RG grp)
      for (int du = 0; du < K + RG - 1; ++du) {
        const int u = RG * grp + du;
        double2 v[NF];
#pragma unroll
        for (int f = 0; f < NF; ++f) v[f] = st[f * PLANE + u * CW + col];
#pragma unroll
        for (int e = 0; e < RG; ++e) {
          const int t = e + K - 1 - du;
          if (t >= 0 && t < K) {
            const double w = sw[t];
#pragma unroll
            for (int f = 0; f < NF; ++f) {
              acc[f][0][e] += w * v[f].x;
              acc[f][1][e] += w * v[f].y;
            }
          }
        }
      }
      unsigned selp = 0;   // bit e: row i0 + RG grp + e selected
#pragma unroll
      for (int e = 0; e < RG; ++e) {
        const int i = i0 + RG * grp + e;
        if (i >= rows_out) break;
        const double Sy = acc[0][0][e], S1 = acc[0][1][e], S2 = acc[1][0][e];
        const double2 Sy1 = mk<double>(acc[2][0][e], acc[2][1][e]);
        const double2 Sy2 = mk<double>(acc[3][0][e], acc[3][1][e]);
        const double2 S12 = mk<double>(acc[4][0][e], acc[4][1][e]);
        const double ny1 = Sy1.x * Sy1.x + Sy1.y * Sy1.y, ny2 = Sy2.x * Sy2.x + Sy2.y * Sy2.y;
        const double d12 = S1 * S2 - (S12.x * S12.x + S12.y * S12.y);
        const size_t o = (size_t)i * a.n + n;
        const bool binned = (a.histP || a.histM) && i < a.maxscale && a.mask[o];
        const bool selP = SEL && a.sel.measure == 0, selM = SEL && a.sel.measure != 0;
        if (a.RP2 || a.PP || (a.histP && binned) || a.cntP || selP) {
          const double2 u = csub(cscale(Sy1, S2), cmul(Sy2, cconj(S12)));
          if (a.RP2 || (a.histP && binned) || a.cntP || selP) {
            const double rp = (u.x * u.x + u.y * u.y) / ((Sy * S2 - ny2) * d12);
            if (a.RP2) a.RP2[o] = rp;
            if (a.histP && binned) hist_count(a.histP, i, a.nbins, rp);
            if (a.cntP) count_exceed(a.cntP, a.obsP, o, rp);
            if (selP && cluster_sel(a.sel, i, n, rp)) selp |= 1u << e;
          }
          if (a.PP) a.PP[o] = u.x == 0.0 && u.y == 0.0 ? 0.0 : atan2(u.y, u.x);
        }
        if (a.RM2 || (a.histM && binned) || a.cntM || selM) {
          const double2 z = cmul(cmul(Sy1, S12), cconj(Sy2));
          const double rm = (S2 * ny1 + S1 * ny2 - 2.0 * z.x) / (Sy * d12);
          if (a.RM2) a.RM2[o] = rm;
          if (a.histM && binned) hist_count(a.histM, i, a.nbins, rm);
          if (a.cntM) count_exceed(a.cntM, a.obsM, o, rm);
          if (selM && cluster_sel(a.sel, i, n, rm)) selp |= 1u << e;
        }
      }
      // The selection bits after the row loop: a warp holds 32 / CW groups, and a group past the
      // last row has left that loop early.  Every lane with a column votes for every e.
      if constexpr (SEL) {
        const unsigned lanes = sel_lanes(CW, a.n - n0);
#pragma unroll
        for (int e = 0; e < RG; ++e) {
          const int i = i0 + RG * grp + e;
          sel_store(a.sel, i < a.rows ? i : -1, n, CW, (selp >> e) & 1u, lanes);
        }
      }
    }
  }
};

// ---- Body: |W|^2 and its row means (SURVEY 8f: device-side derived products) ---------------
template <typename T> struct PowerArgs {
  const cx<T> *W;
  double *power;     // [rows][n] or null
  double *rowsum;    // [rows] accumulated with atomics, or null
  long long n;
  const double *rowmul;        // per-row factor of the stored power (rectification 1/s_j), or null
  const long long *lo, *hi;    // per-row column range [lo, hi) of the row sum, or null (all)
};
template <typename T> struct PowerBody {
  using Args = PowerArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  static constexpr int PER = 64;   // columns per thread, in four rounds of 16 independent 16-byte loads
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    // one atomic per warp for the row sum; four rounds per CTA: the atomics of a row all hit one
    // address and serialise in L2 (2048 of them per 2^20-point row with one round per CTA cost as
    // much as the 4.29 GB read)
    double acc = 0;
    const double mul = a.rowmul ? a.rowmul[by] : 1.0;
    const long long lo = a.lo ? a.lo[by] : 0, hi = a.hi ? a.hi[by] : a.n;
    const cx<T> *row = a.W + (size_t)by * a.n;
    for (int rd = 0; rd < 4; ++rd) {
      const long long n0 = ((long long)bx * 4 + rd) * 16 * NT + tid;
      if (n0 - tid >= a.n) break;
      cx<T> w[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const long long n = n0 + (long long)i * NT;
        w[i] = n < a.n ? ldg(&row[n]) : mk<T>(0, 0);
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const long long n = n0 + (long long)i * NT;
        const double p = ((double)w[i].x * w[i].x + (double)w[i].y * w[i].y) * mul;
        if (a.power && n < a.n) st_stream(&a.power[(size_t)by * a.n + n], p);
        if (n >= lo && n < hi) acc += p;
      }
    }
    if (a.rowsum) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
      // one atomic per warp (every lane reaches this point: no early return above)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
      if ((tid & 31) == 0) atomicAdd(&a.rowsum[by], acc);
#else
      a.rowsum[by] += acc;
#endif
    }
  }
};

// ---- Body: scale-averaged power  out[n] = sum_j w_j |W[j,n]|^2  (TC98 eq. 24; the sample
// scripts' `scale_avg`, simple_sample.py:88-91).  Rows with w_j = 0 are not read. ------------
template <typename T> struct ScaleAvgArgs {
  const cx<T> *W;
  const double *w;   // per row
  double *out;
  long long n;
  int rows;
  const int *sel;    // rows with a non-zero weight, ascending (device)
  int nsel;
  int sel_per_block; // gridDim.y blocks of selected rows; > 1 block: atomics into `out`
};
template <typename T> struct ScaleAvgBody {
  using Args = ScaleAvgArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long n = (long long)bx * NT + tid;
    if (n >= a.n) return;
    const int i0 = by * a.sel_per_block;
    const int i1 = i0 + a.sel_per_block < a.nsel ? i0 + a.sel_per_block : a.nsel;
    double acc0 = 0, acc1 = 0;
    int i = i0;
    for (; i + 4 <= i1; i += 4) {
      cx<T> v[4];
      double wj[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = a.sel[i + u];
        wj[u] = a.w[j];
        v[u] = ldg(&a.W[(size_t)j * a.n + n]);
      }
      acc0 += wj[0] * ((double)v[0].x * v[0].x + (double)v[0].y * v[0].y);
      acc1 += wj[1] * ((double)v[1].x * v[1].x + (double)v[1].y * v[1].y);
      acc0 += wj[2] * ((double)v[2].x * v[2].x + (double)v[2].y * v[2].y);
      acc1 += wj[3] * ((double)v[3].x * v[3].x + (double)v[3].y * v[3].y);
    }
    for (; i < i1; ++i) {
      const int j = a.sel[i];
      const cx<T> v = ldg(&a.W[(size_t)j * a.n + n]);
      acc0 += a.w[j] * ((double)v.x * v.x + (double)v.y * v.y);
    }
    const double acc = acc0 + acc1;
    if (a.sel_per_block >= a.nsel) {
      a.out[n] = acc;
    } else {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
      atomicAdd(&a.out[n], acc);
#else
      a.out[n] += acc;
#endif
    }
  }
};

// ---- Bodies: reductions of a resident field (cwtb_coherence_*, cwtb_field_*) ---------------
// One template per operation, over a view that says how the field is read and what a point adds:
//   CohView     the resident coherence (cwtb_wct_resident): WCT and aWCT, two [rows][n] double
//               fields whose flat indices have the same alignment
//   CxView<T>   a [rows][n] complex field of cx<T> (W or the cross spectrum); every sum is formed
//               in double, after widening
// A view supplies, for RowStatsBody: K sums per row, E elements per 16-byte vector, VPT 16-byte
// vectors per thread per chunk, load (vector q), add (element e of a vector) and add_at (element
// p, at a chunk's odd edge); for SelScaleAvgBody: NA sums per column, SEL, Pt, point, acc and put
// (and keep with SEL); for
// WindowBody: copy.

// Row stats [count, sum WCT, sum cos aWCT, sum sin aWCT] of the points with WCT > thr_j; aWCT is
// not read when want_phase == 0.  Scale average [sum w_j WCT, sum w_j cos aWCT, sum w_j sin aWCT]
// as three planes of n.  Window: WCT to o0, aWCT to o1, either may be null.
// The same reads serve the resident partial coherence (RP2 and its phase, cwtb_wct3_resident).
// CohMagView: a double field without a phase (the multiple coherence RM2): no phase field is read
// whatever want_phase, the phase sums and planes stay 0 and o1 is not written.
template <bool PHASE> struct CohViewT {
  const double *WCT, *aWCT;   // aWCT: unused (may be null) without PHASE
  int want_phase;
  static constexpr int K = 4, E = 2, VPT = 16, NA = 3;   // VPT: two loads each, one per field
  static constexpr bool SEL = false;                     // SelScaleAvgBody: every column of a row
  struct Vec { double2 w, g; };
  HD Vec load(size_t q) const {
    Vec v{ld_stream((const double2 *)WCT + q), make_double2(0, 0)};
    if constexpr (PHASE) {
      if (want_phase) v.g = ld_stream((const double2 *)aWCT + q);
    }
    return v;
  }
  HD void add1(double (&s)[K], double w, double ang, bool has_thr, double t) const {
    if (has_thr && !(w > t)) return;
    s[0] += 1.0;
    s[1] += w;
    if (PHASE && want_phase) {
      double sn, cs;
      sincos_hd(ang, &sn, &cs);
      s[2] += cs;
      s[3] += sn;
    }
  }
  HD void add(double (&s)[K], const Vec &v, int e, bool has_thr, double t) const {
    add1(s, e ? v.w.y : v.w.x, e ? v.g.y : v.g.x, has_thr, t);
  }
  HD void add_at(double (&s)[K], size_t p, bool has_thr, double t) const {
    add1(s, WCT[p], PHASE && want_phase ? aWCT[p] : 0.0, has_thr, t);
  }
  struct Pt { double w, a; };
  HD Pt point(size_t p) const {
    if constexpr (PHASE) return Pt{ld_stream(&WCT[p]), ld_stream(&aWCT[p])};
    else return Pt{ld_stream(&WCT[p]), 0.0};
  }
  HD static void acc(double (&s)[NA], double wj, const Pt &v) {
    if constexpr (PHASE) {
      double sn, cs;
      sincos_hd(v.a, &sn, &cs);
      s[0] += wj * v.w;
      s[1] += wj * cs;
      s[2] += wj * sn;
    } else {
      s[0] += wj * v.w;
    }
  }
  HD static void put(double *out, long long n, long long N, const double (&s)[NA]) {
    st_stream(&out[n], s[0]);
    st_stream(&out[N + n], s[1]);
    st_stream(&out[2 * N + n], s[2]);
  }
  HD void copy(size_t src, double *o0, double *o1, size_t dst) const {
    if (o0) o0[dst] = WCT[src];
    if constexpr (PHASE) {
      if (o1) o1[dst] = aWCT[src];
    }
  }
};
using CohView = CohViewT<true>;
using CohMagView = CohViewT<false>;

// The same double fields with their surrogate exceedance counts k (uint32 [rows][n], the same flat
// index; cwtb_coherence*_surrogate_counts) from M units.  Row stats: CohViewT's four sums over the
// points whose value is finite, whose k <= kmax and, with a threshold, whose value > thr_j.
// Window: the p-value (1 + k) / (1 + M) to o0, NaN where the value is not finite.
template <bool PHASE> struct CohCountViewT {
  const double *WCT, *aWCT;   // aWCT: unused (may be null) without PHASE
  const unsigned *cnt;
  long long kmax, m;          // m: the units M the counts hold
  int want_phase;
  static constexpr int K = 4, E = 2, VPT = 16;
  struct Vec { double2 w, g; uint2 k; };
  HD Vec load(size_t q) const {
    Vec v{ld_stream((const double2 *)WCT + q), make_double2(0, 0), ld_stream((const uint2 *)cnt + q)};
    if constexpr (PHASE) {
      if (want_phase) v.g = ld_stream((const double2 *)aWCT + q);
    }
    return v;
  }
  HD void add1(double (&s)[K], double w, double ang, unsigned k, bool has_thr, double t) const {
    if (!isfinite(w) || (long long)k > kmax) return;
    if (has_thr && !(w > t)) return;
    s[0] += 1.0;
    s[1] += w;
    if (PHASE && want_phase) {
      double sn, cs;
      sincos_hd(ang, &sn, &cs);
      s[2] += cs;
      s[3] += sn;
    }
  }
  HD void add(double (&s)[K], const Vec &v, int e, bool has_thr, double t) const {
    add1(s, e ? v.w.y : v.w.x, e ? v.g.y : v.g.x, e ? v.k.y : v.k.x, has_thr, t);
  }
  HD void add_at(double (&s)[K], size_t p, bool has_thr, double t) const {
    add1(s, WCT[p], PHASE && want_phase ? aWCT[p] : 0.0, cnt[p], has_thr, t);
  }
  HD void copy(size_t src, double *o0, double *, size_t dst) const {
    const double w = WCT[src];
    o0[dst] = isfinite(w) ? (double)(1 + (long long)cnt[src]) / (double)(1 + m) : w - w;   // inf - inf: NaN
  }
  HD bool finite(size_t o) const { return isfinite(ld_stream(&WCT[o])); }   // CountHistBody
};

// 16 bytes of a complex field: one double2, or two float2
template <typename T> struct CxVec16;
template <> struct CxVec16<double> {
  using V = double2;
  static constexpr int E = 1;
  HD static double re(const V &v, int) { return v.x; }
  HD static double im(const V &v, int) { return v.y; }
};
template <> struct CxVec16<float> {
  using V = float4;
  static constexpr int E = 2;
  HD static double re(const V &v, int e) { return (double)(e ? v.z : v.x); }
  HD static double im(const V &v, int e) { return (double)(e ? v.w : v.y); }
};

// Row stats [count, sum |F|^2, sum |F|, sum cos arg F, sum sin arg F] of the points with
// re^2 + im^2 > thr_j, with cos = re / |F|, sin = im / |F| and a zero coefficient counted as phase
// 0 (np.angle(0) == 0).  Scale average sum_j w_j F[j,n] as complex128.  Window: complex128 to o0.
template <typename T> struct CxView {
  const cx<T> *F;
  using V16 = CxVec16<T>;
  using Vec = typename V16::V;
  static constexpr int K = 5, E = V16::E, VPT = 32, NA = 2;
  static constexpr bool SEL = false;
  HD Vec load(size_t q) const { return ld_stream((const Vec *)F + q); }
  HD static void add1(double (&s)[K], double re, double im, bool has_thr, double t) {
    const double p = norm2_rn(re, im);
    if (has_thr && !(p > t)) return;
    const double m = sqrt(p);
    s[0] += 1.0;
    s[1] += p;
    s[2] += m;
    if (m > 0) {
      s[3] += re / m;
      s[4] += im / m;
    } else {
      s[3] += 1.0;
    }
  }
  HD void add(double (&s)[K], const Vec &v, int e, bool has_thr, double t) const {
    add1(s, V16::re(v, e), V16::im(v, e), has_thr, t);
  }
  HD void add_at(double (&s)[K], size_t p, bool has_thr, double t) const {
    add1(s, F[p].x, F[p].y, has_thr, t);
  }
  using Pt = cx<T>;
  HD Pt point(size_t p) const { return ld_stream(&F[p]); }
  HD static void acc(double (&s)[NA], double wj, const Pt &v) {
    s[0] += wj * (double)v.x;
    s[1] += wj * (double)v.y;
  }
  HD static void put(double *out, long long n, long long, const double (&s)[NA]) {
    st_stream((double2 *)out + n, make_double2(s[0], s[1]));
  }
  HD void copy(size_t src, double *o0, double *, size_t dst) const {
    const cx<T> v = F[src];
    ((double2 *)o0)[dst] = make_double2((double)v.x, (double)v.y);
  }
};

// The power P = power_of(F) of a complex field, as the power tests form it.  Window: P to o0.
template <typename T> struct CxPowerView {
  const cx<T> *F;
  HD void copy(size_t src, double *o0, double *, size_t dst) const { o0[dst] = power_of<T>(F[src]); }
};

// A complex field with the surrogate exceedance counts of its power P = power_of(F) (the resident
// power, cwtb_power_surrogate_counts), CohCountViewT's counterpart.  Row stats: CxView's five sums
// over the points whose P is finite, whose k <= kmax and, with a threshold, whose P > thr_j.  Window:
// the p-value (1 + k) / (1 + M) to o0, NaN where P is not finite.
template <typename T> struct CxCountView {
  const cx<T> *F;
  const unsigned *cnt;
  long long kmax, m;
  using V16 = CxVec16<T>;
  static constexpr int K = CxView<T>::K, E = V16::E, VPT = 32;
  struct Vec { typename V16::V w; unsigned k[E]; };
  HD Vec load(size_t q) const {
    Vec v;
    v.w = ld_stream((const typename V16::V *)F + q);
#pragma unroll
    for (int e = 0; e < E; ++e) v.k[e] = ld_stream(&cnt[q * E + e]);
    return v;
  }
  HD void add1(double (&s)[K], double re, double im, unsigned k, bool has_thr, double t) const {
    if (!isfinite(norm2_rn(re, im)) || (long long)k > kmax) return;
    CxView<T>::add1(s, re, im, has_thr, t);
  }
  HD void add(double (&s)[K], const Vec &v, int e, bool has_thr, double t) const {
    add1(s, V16::re(v.w, e), V16::im(v.w, e), v.k[e], has_thr, t);
  }
  HD void add_at(double (&s)[K], size_t p, bool has_thr, double t) const {
    add1(s, F[p].x, F[p].y, cnt[p], has_thr, t);
  }
  HD void copy(size_t src, double *o0, double *, size_t dst) const {
    const double P = power_of<T>(F[src]);
    o0[dst] = isfinite(P) ? (double)(1 + (long long)cnt[src]) / (double)(1 + m) : P - P;   // inf - inf: NaN
  }
  HD bool finite(size_t o) const { return isfinite(power_of<T>(ld_stream(&F[o]))); }   // CountHistBody
};

// A complex field over one cluster of its last cluster test (cwtb_cross_cluster_row_stats): CxView's
// five sums over the points whose label (int32 [rows][n], the field's flat index; 0 off the
// clusters, c + 1 on cluster c) is `want`.  Row stats only.
template <typename T> struct CxLabelView {
  const cx<T> *F;
  const int *lab;
  int want;
  using V16 = CxVec16<T>;
  static constexpr int K = CxView<T>::K, E = V16::E, VPT = 32;
  struct Vec { typename V16::V w; int l[E]; };
  HD Vec load(size_t q) const {
    Vec v;
    v.w = ld_stream((const typename V16::V *)F + q);
#pragma unroll
    for (int e = 0; e < E; ++e) v.l[e] = ld_stream(&lab[q * E + e]);
    return v;
  }
  HD void add(double (&s)[K], const Vec &v, int e, bool has_thr, double t) const {
    if (v.l[e] == want) CxView<T>::add1(s, V16::re(v.w, e), V16::im(v.w, e), has_thr, t);
  }
  HD void add_at(double (&s)[K], size_t p, bool has_thr, double t) const {
    if (lab[p] == want) CxView<T>::add1(s, F[p].x, F[p].y, has_thr, t);
  }
};

// Per-row sums of a view over the columns [lo_j, hi_j) where thr is null or the view's point
// passes thr_j (false for a NaN threshold).  CTA (bx, j) covers the fixed chunk
// [lo_j + bx CHUNK, lo_j + (bx + 1) CHUNK) of row j's range with 16-byte streaming loads, reduces
// its threads' sums in a fixed order and writes its partial; RowSumBody<K> adds the partials of a
// row in chunk order.  No atomics: repeated calls are bit-identical.
template <typename View> struct RowStatsArgs {
  View f;
  const long long *lo, *hi;   // per row
  const double *thr;          // per row, or null
  double *part;               // [rows][nchunk][K]
  long long n;
  int nchunk;
};
template <typename View> struct RowStatsBody {
  using Args = RowStatsArgs<View>;
  static constexpr int NTB = 256, NPHASE = 3, K = View::K;
  static constexpr int U = 4;                                              // 16-byte loads in flight
  static constexpr long long CHUNK = (long long)View::E * View::VPT * NTB;
  static constexpr size_t SMEM = (size_t)K * (NTB + 32) * sizeof(double);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    double *sm = (double *)smraw;          // [K][NTB] thread sums, then [K][32] lane sums
    if constexpr (PH == 0) {
      double s[K] = {};
      const long long lo = a.lo[by], hi = a.hi[by];
      const long long c0 = lo + (long long)bx * CHUNK;
      if (c0 < hi) {
        const long long c1 = c0 + CHUNK < hi ? c0 + CHUNK : hi;
        const bool has_thr = a.thr != nullptr;
        const double t = has_thr ? a.thr[by] : 0.0;
        constexpr size_t E = View::E;
        const size_t p0 = (size_t)by * a.n + c0, p1 = (size_t)by * a.n + c1;
        const size_t v0 = (p0 + E - 1) / E, v1 = p1 / E;   // [v0, v1): whole 16-byte vectors
        if constexpr (E == 2) {                             // an odd element at either end
          if (tid == 0 && (p0 & 1)) a.f.add_at(s, p0, has_thr, t);
          if (tid == 1 && (p1 & 1) && p1 - 1 >= E * v0) a.f.add_at(s, p1 - 1, has_thr, t);
        }
        for (size_t q0 = v0 + (size_t)tid; q0 < v1; q0 += (size_t)NTB * U) {
          typename View::Vec w[U] = {};
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const size_t q = q0 + (size_t)NTB * u;
            if (q < v1) w[u] = a.f.load(q);
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            if (q0 + (size_t)NTB * u < v1) {
#pragma unroll
              for (int e = 0; e < (int)E; ++e) a.f.add(s, w[u], e, has_thr, t);
            }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < K; ++k) sm[k * NTB + tid] = s[k];
    } else if constexpr (PH == 1) {
      if (tid < K * 32) {
        const int k = tid >> 5, l = tid & 31;
        double v = 0;
        for (int i = l; i < NTB; i += 32) v += sm[k * NTB + i];
        sm[K * NTB + tid] = v;
      }
    } else {
      if (tid < K) {
        double v = 0;
        for (int l = 0; l < 32; ++l) v += sm[K * NTB + tid * 32 + l];
        a.part[((size_t)by * a.nchunk + bx) * K + tid] = v;
      }
    }
  }
};

// out[j][k] = sum over chunks b (in order) of part[j][b][k], k < K (the K sums per row of
// RowStatsBody)
struct RowSumArgs { const double *part; double *out; int rows, nchunk; };
template <int K> struct RowSumBody {
  using Args = RowSumArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const int i = bx * NT + tid;
    if (i >= K * a.rows) return;
    const double *p = a.part + (size_t)(i / K) * a.nchunk * K + (i % K);
    double v = 0;
    for (int b = 0; b < a.nchunk; ++b) v += p[(size_t)b * K];
    a.out[i] = v;
  }
};

// The real part of a complex field for the reconstruction (cwtb_*_reconstruct): NA = 1 sum
// w_j Re F[j, n], each step rounded on its own (add_mul_rn), over the points that SelScaleAvgBody's
// column range and threshold on P = power_of(F) pass and that the form's predicate keeps:
//   RE_ALL    every point
//   RE_COUNT  P finite and k <= kmax (CxCountView's cut; cnt: the power's counts)
//   RE_LABEL  mark[label] != 0 (lab: the label image of the last cluster test, mark: a byte table
//             over the labels [0, n_clusters])
enum ReForm { RE_ALL, RE_COUNT, RE_LABEL };
template <typename T, int FORM> struct CxReView {
  const cx<T> *F;
  const unsigned *cnt = nullptr;
  long long kmax = 0;
  const int *lab = nullptr;
  const unsigned char *mark = nullptr;
  static constexpr int NA = 1;
  static constexpr bool SEL = true;
  struct Pt { cx<T> v; unsigned k; };   // k: the count (RE_COUNT) or the label (RE_LABEL)
  HD Pt point(size_t p) const {
    Pt r{ld_stream(&F[p]), 0u};
    if constexpr (FORM == RE_COUNT) r.k = ld_stream(&cnt[p]);
    if constexpr (FORM == RE_LABEL) r.k = (unsigned)ld_stream(&lab[p]);
    return r;
  }
  HD bool keep(const Pt &v, bool has_thr, double t) const {
    if constexpr (FORM == RE_LABEL) {
      if (!mark[v.k]) return false;
    }
    if (FORM == RE_COUNT || has_thr) {
      const double P = power_of<T>(v.v);
      if (has_thr && !(P > t)) return false;
      if constexpr (FORM == RE_COUNT) return isfinite(P) && (long long)v.k <= kmax;
    }
    return true;
  }
  HD static void acc(double (&s)[NA], double wj, const Pt &v) { s[0] = add_mul_rn(s[0], wj, (double)v.v.x); }
  HD static void put(double *out, long long n, long long, const double (&s)[NA]) { st_stream(&out[n], s[0]); }
};

// The view's NA weighted sums over the selected rows (the selected-rows pattern of ScaleAvgBody),
// four rows at a time: one thread per column adds the rows in order, no atomics.  A view with SEL
// (CxReView) also takes a per-row column range [lo_j, hi_j), an optional per-row threshold and its
// own predicate (keep): a point outside them adds nothing.  Views without SEL read none of them.
template <typename View> struct SelScaleAvgArgs {
  View f;
  const double *w;     // per row
  const int *sel;      // rows with a non-zero weight, ascending (device)
  int nsel;
  double *out;         // NA doubles per column, laid out by View::put
  long long n;
  const long long *lo = nullptr, *hi = nullptr;   // per row (SEL)
  const double *thr = nullptr;                    // per row, or null (SEL)
};
template <typename View> struct SelScaleAvgBody {
  using Args = SelScaleAvgArgs<View>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const long long n = (long long)bx * NT + tid;
    if (n >= a.n) return;
    double s[View::NA] = {};
    if constexpr (View::SEL) {
      const bool has_thr = a.thr != nullptr;
      auto in = [&](int j) { return n >= a.lo[j] && n < a.hi[j]; };
      auto add = [&](int j, const typename View::Pt &v) {
        if (a.f.keep(v, has_thr, has_thr ? a.thr[j] : 0.0)) View::acc(s, a.w[j], v);
      };
      int i = 0;
      for (; i + 4 <= a.nsel; i += 4) {
        typename View::Pt v[4] = {};
        bool on[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = a.sel[i + u];
          on[u] = in(j);
          if (on[u]) v[u] = a.f.point((size_t)j * a.n + n);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (on[u]) add(a.sel[i + u], v[u]);
      }
      for (; i < a.nsel; ++i) {
        const int j = a.sel[i];
        if (in(j)) add(j, a.f.point((size_t)j * a.n + n));
      }
      View::put(a.out, n, a.n, s);
      return;
    }
    int i = 0;
    for (; i + 4 <= a.nsel; i += 4) {
      typename View::Pt v[4];
      double wj[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = a.sel[i + u];
        wj[u] = a.w[j];
        v[u] = a.f.point((size_t)j * a.n + n);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) View::acc(s, wj[u], v[u]);
    }
    for (; i < a.nsel; ++i) {
      const int j = a.sel[i];
      View::acc(s, a.w[j], a.f.point((size_t)j * a.n + n));
    }
    View::put(a.out, n, a.n, s);
  }
};

// Strided sub-grid: out[r][c] = field[row0 + r row_step][col0 + c col_step], written by the
// view's copy.  Grid: (ceil(ncols / NT), nrows).
template <typename View> struct WindowArgs {
  View f;
  double *o0, *o1;     // [nrows][ncols] outputs (see the view)
  long long n;
  int row0, row_step;
  long long col0, col_step, ncols;
};
template <typename View> struct WindowBody {
  using Args = WindowArgs<View>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long c = (long long)bx * NT + tid;
    if (c >= a.ncols) return;
    const size_t src = (size_t)(a.row0 + (long long)by * a.row_step) * a.n + a.col0 + c * a.col_step;
    a.f.copy(src, a.o0, a.o1, (size_t)by * a.ncols + c);
  }
};

// ---- Body: histogram of the exceedance counts k in [0, nb) over the columns [lo_j, hi_j) of every
// row, of the points whose observed value is finite (cwtb_coherence*_count_hist, cwtb_power_count_hist)
// CTA (bx, j) covers the chunk [lo_j + bx CHUNK, lo_j + (bx + 1) CHUNK) of row j.  SHARED: the CTA
// counts into a uint32 histogram in shared memory (nb <= SMEM_BINS) and adds its non-zero bins to
// the 64-bit global histogram at the end; otherwise every point is one 64-bit atomic in global
// memory.  Integer sums: the result does not depend on the order, repeated calls are bit-identical.
// View: a counting view (CohCountViewT, CxCountView): its counts and finite().
template <typename View> struct CountHistArgs {
  View f;
  const long long *lo, *hi;   // per row
  unsigned long long *hist;   // [nb], zeroed by the caller
  long long n, nb;
};
template <typename View, bool SHARED> struct CountHistBody {
  using Args = CountHistArgs<View>;
  static constexpr int NPHASE = SHARED ? 3 : 1;
  static constexpr int SMEM_BINS = 12288;                  // 48 KiB: four CTAs per SM
  static constexpr long long CHUNK = 32LL * NT;
  static constexpr size_t SMEM = SHARED ? SMEM_BINS * sizeof(unsigned) : 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    unsigned *sh = (unsigned *)smraw;
    if constexpr (SHARED && PH == 0) {
      for (long long b = tid; b < a.nb; b += NT) sh[b] = 0u;
    } else if constexpr (PH == (SHARED ? 1 : 0)) {
      const long long c0 = a.lo[by] + (long long)bx * CHUNK;
      const long long c1 = c0 + CHUNK < a.hi[by] ? c0 + CHUNK : a.hi[by];
      for (long long n = c0 + tid; n < c1; n += NT) {
        const size_t o = (size_t)by * a.n + n;
        if (!a.f.finite(o)) continue;
        const unsigned k = ld_stream(&a.f.cnt[o]);
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
        if constexpr (SHARED) atomicAdd(&sh[k], 1u);
        else atomicAdd(&a.hist[k], 1ull);
#else
        if constexpr (SHARED) sh[k] += 1u;
        else a.hist[k] += 1ull;
#endif
      }
    } else {
      for (long long b = tid; b < a.nb; b += NT)
        if (sh[b]) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
          atomicAdd(&a.hist[b], (unsigned long long)sh[b]);
#else
          a.hist[b] += sh[b];
#endif
        }
    }
  }
};

// ---- cluster labelling of a selection bitmask (cwtb_coherence*_cluster_test) --------------------
// Clusters are the 8-connected components of the set bits of a bitmask [rows][words] (SelArgs'
// layout, n columns, rows * n < 2^32 so that a point's flat index j n + col fits 32 bits).  The
// labelling works on runs, the maximal horizontal stretches of set bits of a row:
//   ClusterCountBody    CTA (chunk, j): the runs that start and end in a chunk of CHW words of row j
//   ClusterScanBody     one CTA: exclusive offsets of the chunks, the runs of every row, the total
//   (the host reads the total and sizes the run tables from it)
//   ClusterExtractBody  CTA (chunk, j): run k's first point start[k] and end[k] (one past its last),
//                       flat indices in row-major order, its parent k and its sums zeroed
//   ClusterUnionBody    thread per run: unions with every run of the row above whose columns reach
//                       [start - 1, end] (8-connectivity; time is not circular)
//   ClusterSumBody      thread per run: q_j * length (and, for a table, the point count and the box)
//                       into its root's sums
//   ClusterMaxBody      the largest root sum into qmax[unit]
// Union-find: a union links the larger of two roots to the smaller with a compare-and-swap, so the
// root of a cluster is its smallest run, the run of its first point in row-major order, whatever
// order the unions run in.  find() halves paths with plain stores: a non-root is never the target
// of a link, and every value stored is an ancestor of the node.
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
HD unsigned uf_find(unsigned *parent, unsigned x) {
  volatile unsigned *p = parent;
  unsigned y = p[x];
  while (y != x) {
    const unsigned z = p[y];
    if (z != y) p[x] = z;
    x = y;
    y = z;
  }
  return x;
}
#else
HD unsigned uf_find(unsigned *p, unsigned x) {
  while (p[x] != x) {
    if (p[p[x]] != p[x]) p[x] = p[p[x]];
    x = p[x];
  }
  return x;
}
#endif
HD void uf_union(unsigned *parent, unsigned a, unsigned b) {
  for (;;) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) { const unsigned t = a; a = b; b = t; }
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
    if (atomicCAS(&parent[a], a, b) == a) return;
#else
    parent[a] = b;
    return;
#endif
  }
}
HD void atomic_add_u64(unsigned long long *p, unsigned long long v) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  atomicAdd(p, v);
#else
  *p += v;
#endif
}
HD void atomic_max_u64(unsigned long long *p, unsigned long long v) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  atomicMax(p, v);
#else
  if (v > *p) *p = v;
#endif
}
HD void atomic_max_u32(unsigned *p, unsigned v) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  atomicMax(p, v);
#else
  if (v > *p) *p = v;
#endif
}
HD void atomic_min_u32(unsigned *p, unsigned v) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  atomicMin(p, v);
#else
  if (v < *p) *p = v;
#endif
}
HD int popc32(unsigned x) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  return __popc(x);
#else
  return __builtin_popcount(x);
#endif
}
HD int ffs32(unsigned x) {   // index of the lowest set bit, x != 0
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  return __ffs(x) - 1;
#else
  return __builtin_ctz(x);
#endif
}

// The per-cluster sums of a table (the observed map and the test hook): point count, last row,
// first column and one past the last column; the first row is the root's.
struct ClusterStats {
  unsigned long long *pts;
  unsigned *rmax, *cmin, *cmax;
};
struct ClusterArgs {
  const unsigned *bits;       // [rows][words]
  long long n, words;
  int rows, cpr;              // cpr: chunks per row
  unsigned *chunk;            // [rows cpr]: packed counts (starts << 16 | ends), then start offsets
  unsigned *chunk_end;        // [rows cpr]: end offsets
  unsigned *rowbeg;           // [rows + 1]: first run of each row; rowbeg[rows] = runs
  unsigned *total;            // [2]: runs counted by starts and by ends
  unsigned *start, *end, *parent;   // [runs]
  unsigned long long *qsum;         // [runs]: root sums of q_j * length
  const unsigned long long *q;      // [rows]: the weight of a point of each row
  ClusterStats st;                  // pts null: no table
  unsigned long long *qmax;         // the unit's maximum
  unsigned runs;
};
// The run starts and ends of word w of row j, as bit sets (bits past the row's end are 0)
HD void run_bits(const ClusterArgs &a, int j, long long w, unsigned &st, unsigned &en) {
  const unsigned *r = a.bits + (size_t)j * a.words;
  const unsigned m = r[w];
  const unsigned prev = w > 0 ? r[w - 1] >> 31 : 0u;
  const unsigned next = w + 1 < a.words ? r[w + 1] & 1u : 0u;
  st = m & ~((m << 1) | prev);
  en = m & ~((m >> 1) | (next << 31));
}
struct ClusterCountBody {
  using Args = ClusterArgs;
  static constexpr int NPHASE = 2, WPT = 8;
  static constexpr long long CHW = (long long)WPT * NT;   // words per chunk
  // a chunk holds at most 16 CHW run starts (an alternating mask) and as many ends: each count has 16 bits
  static_assert(16 * CHW < 65536, "ClusterCountBody: the packed run counts of a chunk need 16 * CHW < 2^16");
  static constexpr size_t SMEM = NT * sizeof(unsigned);
  // the packed start / end counts of this thread's words of chunk bx of row by
  HD static unsigned count(const Args &a, int bx, int by, int tid) {
    const long long w0 = (long long)bx * CHW + (long long)tid * WPT;
    unsigned c = 0;
    for (long long w = w0; w < w0 + WPT && w < a.words; ++w) {
      unsigned st, en;
      run_bits(a, by, w, st, en);
      c += ((unsigned)popc32(st) << 16) | (unsigned)popc32(en);
    }
    return c;
  }
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    unsigned *sh = (unsigned *)smraw;
    if constexpr (PH == 0) {
      sh[tid] = count(a, bx, by, tid);
    } else if (tid == 0) {
      unsigned c = 0;
      for (int t = 0; t < NT; ++t) c += sh[t];
      a.chunk[(size_t)by * a.cpr + bx] = c;
    }
  }
};
// One CTA.  Thread t scans the chunks [t G, (t + 1) G), G = ceil(chunks / NT).
struct ClusterScanBody {
  using Args = ClusterArgs;
  static constexpr int NPHASE = 3;
  static constexpr size_t SMEM = 2 * NT * sizeof(unsigned);
  template <int PH> HD static void phase(const Args &a, int, int, int tid, void *smraw) {
    unsigned *ss = (unsigned *)smraw, *se = ss + NT;
    const long long nch = (long long)a.rows * a.cpr, G = (nch + NT - 1) / NT;
    const long long c0 = tid * G, c1 = c0 + G < nch ? c0 + G : nch;
    if constexpr (PH == 0) {
      unsigned s = 0, e = 0;
      for (long long c = c0; c < c1; ++c) {
        s += a.chunk[c] >> 16;
        e += a.chunk[c] & 0xFFFFu;
      }
      ss[tid] = s;
      se[tid] = e;
    } else if constexpr (PH == 1) {
      if (tid == 0) {
        unsigned s = 0, e = 0;
        for (int t = 0; t < NT; ++t) {
          const unsigned ts = ss[t], te = se[t];
          ss[t] = s;
          se[t] = e;
          s += ts;
          e += te;
        }
        a.total[0] = s;
        a.total[1] = e;
        a.rowbeg[a.rows] = s;
      }
    } else {
      unsigned s = ss[tid], e = se[tid];
      for (long long c = c0; c < c1; ++c) {
        const unsigned v = a.chunk[c];
        if (c % a.cpr == 0) a.rowbeg[c / a.cpr] = s;
        a.chunk[c] = s;
        a.chunk_end[c] = e;
        s += v >> 16;
        e += v & 0xFFFFu;
      }
    }
  }
};
struct ClusterExtractBody {
  using Args = ClusterArgs;
  using CB = ClusterCountBody;
  static constexpr int NPHASE = 3;
  static constexpr size_t SMEM = NT * sizeof(unsigned);
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *smraw) {
    unsigned *sh = (unsigned *)smraw;
    if constexpr (PH == 0) {
      sh[tid] = CB::count(a, bx, by, tid);
    } else if constexpr (PH == 1) {
      if (tid == 0) {
        unsigned c = 0;
        for (int t = 0; t < NT; ++t) {
          const unsigned v = sh[t];
          sh[t] = c;
          c += v;
        }
      }
    } else {
      const size_t ci = (size_t)by * a.cpr + bx;
      unsigned ks = a.chunk[ci] + (sh[tid] >> 16), ke = a.chunk_end[ci] + (sh[tid] & 0xFFFFu);
      const long long w0 = (long long)bx * CB::CHW + (long long)tid * CB::WPT;
      const unsigned base = (unsigned)((unsigned long long)by * (unsigned long long)a.n);
      for (long long w = w0; w < w0 + CB::WPT && w < a.words; ++w) {
        unsigned st, en;
        run_bits(a, by, w, st, en);
        for (; st; st &= st - 1, ++ks) {
          a.start[ks] = base + (unsigned)(32 * w + ffs32(st));
          a.parent[ks] = ks;
          a.qsum[ks] = 0ull;
          if (a.st.pts) {
            a.st.pts[ks] = 0ull;
            a.st.rmax[ks] = 0u;
            a.st.cmin[ks] = 0xFFFFFFFFu;
            a.st.cmax[ks] = 0u;
          }
        }
        for (; en; en &= en - 1, ++ke) a.end[ke] = base + (unsigned)(32 * w + ffs32(en)) + 1u;
      }
    }
  }
};
// the row of run k (rowbeg is sorted: the last row whose first run is <= k)
HD int run_row(const ClusterArgs &a, unsigned k) {
  int lo = 0, hi = a.rows - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (a.rowbeg[mid] <= k) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}
struct ClusterUnionBody {
  using Args = ClusterArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const unsigned long long k = (unsigned long long)bx * NT + tid;
    if (k >= a.runs) return;
    const int j = run_row(a, (unsigned)k);
    if (j == 0) return;
    const unsigned n = (unsigned)a.n;
    // in row j - 1: the runs p with end[p] >= s and start[p] <= e, s = start - 1 col, e = end col
    const unsigned s = a.start[k] - n, e = a.end[k] - n;
    unsigned lo = a.rowbeg[j - 1], hi = a.rowbeg[j];
    while (lo < hi) {   // the first run of row j - 1 with end >= s
      const unsigned mid = lo + (hi - lo) / 2;
      if (a.end[mid] < s) lo = mid + 1;
      else hi = mid;
    }
    for (unsigned p = lo; p < a.rowbeg[j] && a.start[p] <= e; ++p) uf_union(a.parent, (unsigned)k, p);
  }
};
struct ClusterSumBody {
  using Args = ClusterArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const unsigned long long k = (unsigned long long)bx * NT + tid;
    if (k >= a.runs) return;
    const unsigned r = uf_find(a.parent, (unsigned)k);
    const int j = run_row(a, (unsigned)k);
    const unsigned len = a.end[k] - a.start[k];
    atomic_add_u64(&a.qsum[r], a.q[j] * len);
    if (a.st.pts) {
      const unsigned c0 = a.start[k] - (unsigned)j * (unsigned)a.n;
      atomic_add_u64(&a.st.pts[r], len);
      atomic_max_u32(&a.st.rmax[r], (unsigned)j);
      atomic_min_u32(&a.st.cmin[r], c0);
      atomic_max_u32(&a.st.cmax[r], c0 + len);
      a.parent[k] = r;   // a find of another thread may store an ancestor over r: not a flat forest
    }
  }
};
struct ClusterMaxBody {
  using Args = ClusterArgs;
  static constexpr int NPHASE = 2;
  static constexpr size_t SMEM = NT * sizeof(unsigned long long);
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *smraw) {
    unsigned long long *sh = (unsigned long long *)smraw;
    if constexpr (PH == 0) {
      const unsigned long long k = (unsigned long long)bx * NT + tid;
      sh[tid] = k < a.runs && a.parent[k] == (unsigned)k ? a.qsum[k] : 0ull;
    } else if (tid == 0) {
      unsigned long long m = 0;
      for (int t = 0; t < NT; ++t) m = sh[t] > m ? sh[t] : m;
      if (m) atomic_max_u64(a.qmax, m);
    }
  }
};
// ---- Body: the label image [rows][n] int32 of a labelled bitmask: 0 off the clusters, else
// cid[root of the point's run] (the table rank + 1) ----------------------------------------------
struct ClusterPaintArgs { ClusterArgs c; const int *cid; int *labels; };
struct ClusterPaintBody {
  using Args = ClusterPaintArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const ClusterArgs &c = a.c;
    const long long n = (long long)bx * NT + tid;
    if (n >= c.n) return;
    const size_t o = (size_t)by * c.n + n;
    int lab = 0;
    if ((c.bits[(size_t)by * c.words + (n >> 5)] >> (n & 31)) & 1u) {
      unsigned lo = c.rowbeg[by], hi = c.rowbeg[by + 1] - 1;   // the last run of the row starting <= o
      while (lo < hi) {
        const unsigned mid = lo + (hi - lo + 1) / 2;
        if (c.start[mid] <= (unsigned)o) lo = mid;
        else hi = mid - 1;
      }
      lab = a.cid[uf_find(c.parent, lo)];
    }
    a.labels[o] = lab;
  }
};

// ---- Body: strided window of an int32 image [rows][n] (the cluster labels) -------------------------
struct LabelWindowArgs {
  const int *in;
  int *out;            // [nrows][ncols]
  long long n;
  int row0, row_step;
  long long col0, col_step, ncols;
};
struct LabelWindowBody {
  using Args = LabelWindowArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long k = (long long)bx * NT + tid;
    if (k >= a.ncols) return;
    a.out[(size_t)by * a.ncols + k] = a.in[(size_t)(a.row0 + (long long)by * a.row_step) * a.n + a.col0 + k * a.col_step];
  }
};

// ---- Body: real -> complex widening / complex -> real part ---------------------------------
struct R2CArgs { const double *in; double2 *out; long long count; };
struct R2CBody {
  using Args = R2CArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const long long i = (long long)bx * NT + tid;
    if (i < a.count) a.out[i] = make_double2(a.in[i], 0.0);
  }
};

// ---- Body: out[i] = in[i] * f ------------------------------------------------------------
struct ScaleCopyArgs { const double *in; double *out; long long count; double f; };
struct ScaleCopyBody {
  using Args = ScaleCopyArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const long long i = (long long)bx * NT + tid;
    if (i < a.count) a.out[i] = a.in[i] * a.f;
  }
};

// ---- Body: complex64 -> complex128 (fp32 transforms returned through the reference API) ----
struct WidenArgs { const float2 *in; double2 *out; long long count; };
struct WidenBody {
  using Args = WidenArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long i = ((long long)bx * 4 + u) * NT + tid;
      if (i < a.count) {
        const float2 v = a.in[i];
        a.out[i] = make_double2((double)v.x, (double)v.y);
      }
    }
  }
};

// ---- Bluestein (chirp-z) pieces: DFT of ARBITRARY length n through power-of-two transforms ----
// (un-padded mode, pycwt/helpers.py:15-19: with pyfftw installed the reference transforms at the
// signal's own length).  With w_s[k] = e^{s i pi k^2 / n}  (s = -1 forward, +1 inverse):
//   X[k] = sum_j x[j] e^{s 2 pi i jk/n} = w_s[k] * sum_j (x[j] w_s[j]) conj(w_s[k-j]),
// a linear convolution of length 2n-1 evaluated with transforms of length L = 2^m >= 2n-1:
//   a = x * w_s (zero-padded to L),  b[m] = conj(w_s[|m|]) for |m| < n (wrapped mod L),
//   X[k] = w_s[k] / L * IFFT_L( FFT_L(a) * FFT_L(b) )[k].
// One table wm[k] = e^{-i pi k^2/n} serves both signs (w_+ = conj(wm)); k^2 is reduced mod 2n in
// integers so the phase is exact.
struct BlueChirpArgs { double2 *wm; unsigned n; };
struct BlueChirpBody {
  using Args = BlueChirpArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const unsigned long long k = (unsigned long long)bx * NT + tid;
    if (k >= a.n) return;
    const unsigned long long m = (k * k) % (2ull * a.n);
    double sn, cs;
    sincospi_hd((double)m / (double)a.n, &sn, &cs);
    a.wm[k] = make_double2(cs, -sn);
  }
};

HD double2 blue_w(const double2 *wm, unsigned k, int sign) {   // w_s[k]
  const double2 v = wm[k];
  return sign < 0 ? v : make_double2(v.x, -v.y);
}

struct BlueFilterArgs { const double2 *wm; double2 *b; unsigned n, L; int sign; };
struct BlueFilterBody {
  using Args = BlueFilterArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const unsigned m = (unsigned)bx * NT + tid;
    if (m >= a.L) return;
    double2 v = make_double2(0.0, 0.0);
    if (m < a.n) v = blue_w(a.wm, m, -a.sign);             // conj(w_s[m])
    else if (m > a.L - a.n) v = blue_w(a.wm, a.L - m, -a.sign);
    a.b[m] = v;
  }
};

// a[r][k] = in[r][k] * w_s[k]   (rows of a generic transform)
struct BluePreArgs {
  const void *in; double2 *out; const double2 *wm;
  long long in_pitch, out_pitch; unsigned n; int real_in, sign;
};
struct BluePreBody {
  using Args = BluePreArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const unsigned k = (unsigned)bx * NT + tid;
    if (k >= a.n) return;
    double2 x;
    if (a.real_in) x = make_double2(((const double *)a.in)[(size_t)by * a.in_pitch + k], 0.0);
    else x = ((const double2 *)a.in)[(size_t)by * a.in_pitch + k];
    a.out[(size_t)by * a.out_pitch + k] = cmul(x, blue_w(a.wm, k, a.sign));
  }
};

// a[r][k] = x^[k] * norm_j conj(psi^(s_j w_k)) / n * w_+[k]: product of wavelet.py:102-104 and the
// chirp pre-multiplication of the inverse transform in one pass
struct BlueProdArgs {
  const ScaleDesc *descs; const double2 *spec; double2 *out; const double2 *wm;
  Fam fam; long long out_pitch; unsigned n; int first;
};
struct BlueProdBody {
  using Args = BlueProdArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const unsigned k = (unsigned)bx * NT + tid;
    if (k >= a.n) return;
    const ScaleDesc d = a.descs[a.first + by];
    // numpy fftfreq ordering for any n: bins 0 .. (n-1)/2 are non-negative
    const int ks = k < (a.n + 1) / 2 ? (int)k : (int)k - (int)a.n;
    double2 v = make_double2(0.0, 0.0);
    if (a.fam.family == 3 || (ks >= d.k_lo && ks <= d.k_hi)) v = band_value<double>(a.fam, d, a.spec, k, ks, a.n);
    a.out[(size_t)by * a.out_pitch + k] = cmul(v, blue_w(a.wm, k, +1));
  }
};

struct BlueMulArgs { double2 *x; const double2 *bf; unsigned L; };
struct BlueMulBody {
  using Args = BlueMulArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const unsigned m = (unsigned)bx * NT + tid;
    if (m >= a.L) return;
    double2 *p = a.x + (size_t)by * a.L + m;
    *p = cmul(*p, a.bf[m]);
  }
};

// F[r][k] *= filt[r][k] * post: a caller-supplied real frequency response per row (time smoothing
// with a filter other than Morlet's Gaussian: cwtb_set_smooth_filter); the table is double for
// every engine type T
template <typename T> struct FilterMulArgs { cx<T> *f; const double *filt; long long pitch; unsigned n; double post; };
template <typename T> struct FilterMulBody {
  using Args = FilterMulArgs<T>;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const unsigned k = (unsigned)bx * NT + tid;
    if (k >= a.n) return;
    const T m = (T)(a.filt[(size_t)by * a.n + k] * a.post);
    cx<T> *p = a.f + (size_t)by * a.pitch + k;
    p->x *= m; p->y *= m;
  }
};

// out[row][k] = epilogue(y[r][k] * w_s[k] * scale)
struct BluePostArgs {
  const double2 *y; double2 *out; const double2 *wm; const ScaleDesc *descs;   // descs may be null
  long long out_pitch, nout; double scale; unsigned L; int first, row0, sign, epi;
};
struct BluePostBody {
  using Args = BluePostArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const long long k = (long long)bx * NT + tid;
    if (k >= a.nout) return;
    const int row = a.descs ? a.descs[a.first + by].row : a.row0 + by;
    double2 v = cmul(a.y[(size_t)by * a.L + k], blue_w(a.wm, (unsigned)k, a.sign));
    v.x *= a.scale; v.y *= a.scale;
    double2 *o = a.out + (size_t)row * a.out_pitch + k;
    if (a.epi == EPI_MULCONJ) v = cmul(*o, cconj(v));
    *o = v;
  }
};

// F[r][k] *= exp(g_r * w_k^2) * post,  w_k = 2 pi fftfreq(n)[k]: the Gaussian time filter of
// Morlet.smooth (mothers.py:83-91) for a transform length that is not a power of two
struct BlueGaussArgs { double2 *f; const double *g; long long pitch; unsigned n; double post; };
struct BlueGaussBody {
  using Args = BlueGaussArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int by, int tid, void *) {
    const unsigned k = (unsigned)bx * NT + tid;
    if (k >= a.n) return;
    const long long ks = k < (a.n + 1) / 2 ? (long long)k : (long long)k - (long long)a.n;
    const double w = 6.283185307179586 * ((double)ks * (1.0 / (double)a.n));
    const double m = exp(a.g[by] * (w * w)) * a.post;
    double2 *p = a.f + (size_t)by * a.pitch + k;
    p->x *= m; p->y *= m;
  }
};

// ---- Body: pass twiddle tables in [c][j] layout (see fft_tile.cuh: tw_offset) -------------
struct PassTwArgs {
  double2 *out64;
  float2 *out32;
};
struct PassTwBody {
  using Args = PassTwArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const int idx = bx * NT + tid;
    if (idx >= TW_TOTAL) return;
    int L = 32;
    while (L < 1024 && idx >= tw_offset(2 * L)) L *= 2;
    const int R = tw_radix(L), Ln = L / R;
    const int rel = idx - tw_offset(L);
    const int c = rel / Ln + 1, j = rel % Ln;
    double sn, cs;
    sincospi_hd(2.0 * (double)(j * c) / (double)L, &sn, &cs);
    (void)R;
    a.out64[idx] = make_double2(cs, sn);
    a.out32[idx] = make_float2((float)cs, (float)sn);
  }
};

// ---- Body: twiddle tables ---------------------------------------------------------
struct TabArgs {
  double2 *out64;
  float2 *out32;
  unsigned count;
  double step;  // entry i = e^{2 pi i * i * step}
};
struct TabBody {
  using Args = TabArgs;
  static constexpr int NPHASE = 1;
  static constexpr size_t SMEM = 0;
  template <int PH> HD static void phase(const Args &a, int bx, int, int tid, void *) {
    const unsigned i = (unsigned)bx * NT + tid;
    if (i >= a.count) return;
    double sn, cs;
    sincospi_hd(2.0 * ((double)i * a.step), &sn, &cs);
    if (a.out64) a.out64[i] = make_double2(cs, sn);
    if (a.out32) a.out32[i] = make_float2((float)cs, (float)sn);
  }
};

}  // namespace cwtb
