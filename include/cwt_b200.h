/*
 * cwt_b200.h -- C ABI of the H100-native continuous-wavelet-transform engine.
 *
 * Drop-in boundary for the hot path of regeirk/pycwt.  The reference has no FFI
 * layer (it is pure Python); its "interface" for this path is the array math
 * inside pycwt/wavelet.py and pycwt/mothers.py.  Each entry point below names
 * the reference lines it replaces.  A host in any language binds these symbols
 * (ctypes / cffi / cgo / JNI); no torch or C++ types cross the boundary.
 *
 * Conventions
 *   - every function returns 0 on success, a negative cwtb_status otherwise,
 *     and never throws; cwtb_last_error(ctx) gives the message;
 *   - the caller owns every host buffer it passes; device buffers are owned by
 *     the context and addressed through opaque handles or raw device pointers
 *     obtained from cwtb_* accessors;
 *   - a context is bound to one device and one stream; calls on one context
 *     must be serialised by the caller (ctypes releases the GIL, so one context
 *     per host thread / per GPU);
 *   - complex numbers are interleaved (re, im) pairs of double (fp64 engine) or
 *     float (fp32 engine), C order, rows = scales.
 */
#ifndef CWT_B200_H
#define CWT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cwtb_ctx cwtb_ctx;

enum cwtb_status {
  CWTB_OK = 0,
  CWTB_ERR_ARG = -1,       /* bad argument (size, enum, NULL)            */
  CWTB_ERR_CUDA = -2,      /* CUDA runtime error (see cwtb_last_error)   */
  CWTB_ERR_NOMEM = -3,     /* device / pinned allocation failed          */
  CWTB_ERR_STATE = -4,     /* call sequence error (no transform resident) */
  CWTB_ERR_UNSUPPORTED = -5,
  CWTB_ERR_COMM = -6       /* NCCL error / libnccl not loadable           */
};

/* Mother-wavelet families, pycwt/mothers.py:13-233.  MexicanHat == DOG m=2.
 * CWTB_MORSE is the generalized Morse wavelet of Olhede & Walden (2002), unit energy:
 *   psi_ft(w) = A w^be exp(-w^ga) for w > 0, else 0,  A = sqrt(ga 2^((2be+1)/ga) / Gamma((2be+1)/ga)),
 * with 1 <= be <= 256 passed as `param` and 1 <= ga <= 12 taken from the context
 * (cwtb_set_morse_ga, default 3); ga = 1, be = m is Paul(m)'s response. */
enum cwtb_family {
  CWTB_MORLET = 0,  /* param = f0 (mothers.py:26-28)  */
  CWTB_PAUL = 1,    /* param = m  (mothers.py:118-122) */
  CWTB_DOG = 2,     /* param = m  (mothers.py:170-173) */
  CWTB_TABLE = 3,   /* caller supplies psi_ft on the [S, Np] grid (duck-typed wavelets) */
  CWTB_MORSE = 4    /* param = be; ga from cwtb_set_morse_ga */
};

enum cwtb_precision { CWTB_F64 = 0, CWTB_F32 = 1 };

/* ---- lifecycle ---------------------------------------------------------- */
int cwtb_device_count(void);
int cwtb_create(int device, cwtb_ctx **out);
void cwtb_destroy(cwtb_ctx *ctx);
const char *cwtb_last_error(cwtb_ctx *ctx);
const char *cwtb_version(void);

/* Relative cut-off below which the analytic frequency response is treated as
 * zero when the per-scale band is pruned (default 1e-16: at the level of the fp64
 * rounding of the transform itself -- parity against the reference fixtures is the
 * same 5e-16 as with 1e-20).  eps = 0 keeps every bin whose response
 * is representable (the reference's own underflow-to-zero set). */
int cwtb_set_band_eps(cwtb_ctx *ctx, double eps);
/* Tolerance of the band-limited expansion path (replaces the per-scale inverse FFT of
 * pycwt/wavelet.py:105-106 for scales whose band is at most 1/32 of the transform length): such a
 * scale is transformed on a coarse grid of Nc >= 2 * (band width) points and expanded to the
 * output points by a polyphase Kaiser-Bessel interpolation; (Nc, taps) are chosen so that the
 * relative aliasing error bound max sum_l |phi^(xi+l)|/|phi^(xi)| stays <= eps.  Defaults:
 * 5e-13 for the fp64 engine (measured error vs the reference ~1e-13), 2e-7 for the fp32 engine.
 * eps = 0 switches the path off: every scale runs the exact pruned transforms. */
int cwtb_set_expand_eps(cwtb_ctx *ctx, double eps_fp64, double eps_fp32);
/* Transform-length policy of pycwt/helpers.py:7-30.  pad_to_pow2 != 0 (default): the signal is
 * zero-padded to the next power of two (the reference's scipy branch, :27-30).  0: transforms
 * run at the signal's own length (what the reference does when pyfftw is installed, :15-19) --
 * Bluestein's algorithm on the power-of-two kernels, fp64 only, single-channel calls, n0 <= 2^24;
 * the smoothing filter of wct / smooth / wct_mc then is circular at the rows' own length, as in
 * the reference.  Power-of-two lengths are unaffected. */
int cwtb_set_padding(cwtb_ctx *ctx, int pad_to_pow2);
/* Arithmetic of cwtb_xwt, cwtb_wct, cwtb_wct_mc and cwtb_wct_mc_seeded: CWTB_F64 (what a new
 * context starts with) or CWTB_F32.  In fp32 the two transforms run in the fp32 engine (its band
 * and expansion tolerances, relative error <= 1e-5 each) and the coherence products, the time
 * smoothing and the scale boxcar are computed in float; the device holds half the bytes per
 * scale-point.  Host inputs stay double: the series and host surrogates are rounded to float on
 * the device, and device-drawn surrogates are drawn in double and rounded.  Outputs keep their
 * types: W12 complex128 (after an fp32 cwtb_xwt the resident job is an fp32 one; cwtb_get_w widens
 * it on the device), WCT and aWCT double, histogram counts int64, binned from the coherence as
 * double.  WCT differs from fp64 by at most 2.5e-4 (DESIGN.md section 6).  Un-padded transforms
 * (cwtb_set_padding(ctx, 0) with n0 not a power of two) have no fp32 path: the calls then return
 * CWTB_ERR_UNSUPPORTED.  cwtb_smooth always runs in fp64.  Returns CWTB_ERR_ARG for any other
 * value. */
int cwtb_set_coherence_precision(cwtb_ctx *ctx, int precision);
/* Time-smoothing filter of cwtb_smooth / cwtb_wct / cwtb_wct_mc.  Default (table == NULL): the
 * Gaussian exp(-0.5 (s/dt)^2 k^2) of Morlet.smooth (pycwt/mothers.py:83-91).  With a table
 * [n_rows][n] of real frequency responses (n = the transform length of the rows: next power of
 * two, or the rows' own length in un-padded mode) the following calls multiply the transforms of
 * their rows by it instead -- the smoothing operator of wavelets the reference has none for
 * (Paul, DOG: SURVEY 8f rank 4; pycwt_b200.mothers.enable_generic_smoothing).  The table stays in
 * force until replaced or cleared; calls whose rows / length differ fail with CWTB_ERR_STATE. */
int cwtb_set_smooth_filter(cwtb_ctx *ctx, const double *table, int n_rows, int64_t n);
/* Shape parameter ga of CWTB_MORSE (default 3) for the following calls with that family, the second
 * parameter of the family kept on the context like the smoothing filter above, so that every entry
 * point keeps its (family, param) pair.  A resident plan built for one ga is never reused for another.
 * Returns CWTB_ERR_ARG for ga outside [1, 12]. */
int cwtb_set_morse_ga(cwtb_ctx *ctx, double ga);

/* Pinned host memory (so D2H of multi-GiB results runs at PCIe speed and can
 * overlap with compute).  numpy wraps the returned pointer. */
int cwtb_host_alloc(cwtb_ctx *ctx, size_t bytes, void **out);
int cwtb_host_free(cwtb_ctx *ctx, void *p);

/* ---- cwt: pycwt/wavelet.py:91-106 (+ :123 trim to n0) -------------------- */
/*
 * Computes, for every scale s_j (j < n_scales),
 *   W[j, n] = ifft_k( fft(signal, Np)[k] * sqrt(s_j*w1*Np) * conj(psi_ft(s_j*w_k)) )[n],
 *   n < n0,  w_k = 2*pi*fftfreq(Np, dt)[k],
 * with Np = next power of two >= n0 (pycwt/helpers.py:27-30).
 *
 * signal      host pointer, n0 reals (double if signal_is_f32 == 0, else float)
 * scales      host pointer, n_scales doubles (resolved by the caller exactly as
 *             wavelet.py:75-88 does)
 * family/param  mother wavelet; for CWTB_TABLE `table` is a host [n_scales, Np]
 *             complex128 array holding sqrt(s*w1*Np)*conj(psi_ft) already
 * precision   arithmetic of the engine (fp64 or fp32)
 * The result stays resident on the device (see "what stays resident" below);
 * fetch it with cwtb_get_* or post-process it with cwtb_icwt...
 */
int cwtb_cwt(cwtb_ctx *ctx, const void *signal, int signal_is_f32, int64_t n0,
             double dt, const double *scales, int n_scales, int family,
             double param, int precision, const void *table);

/* Same, but the signal is already on the device (double or float, n0 reals);
 * used by benchmarks (`value` leg) and by the batched path. */
int cwtb_cwt_dev(cwtb_ctx *ctx, const void *d_signal, int signal_is_f32,
                 int64_t n0, double dt, const double *scales, int n_scales,
                 int family, double param, int precision);

/* Copy W (n_scales x n0, complex of the engine precision, or converted to
 * complex128 when out_f64 != 0) to host memory.  rows [row0, row0+nrows). */
int cwtb_get_w(cwtb_ctx *ctx, void *out, int out_f64, int row0, int nrows);
/* Forward spectrum of the zero-padded signal, bins [1, Np/2), divided by
 * sqrt(Np): the `fft` return value of wavelet.py:123.  Np/2-1 complex128. */
int cwtb_get_signal_fft(cwtb_ctx *ctx, void *out);
int64_t cwtb_padded_length(cwtb_ctx *ctx);
/* Number of transforms this context has started: a handle to a device-resident result stays
 * valid while this value is unchanged. */
int64_t cwtb_job_serial(cwtb_ctx *ctx);
/* Raw device pointer of the resident W (engine precision), for zero-copy
 * consumers (DLPack / __cuda_array_interface__ wrappers); NULL when none is resident. */
void *cwtb_w_device_ptr(cwtb_ctx *ctx);

/* ---- what stays resident --------------------------------------------------------------------
 * A context holds at most one resident transform W, besides the resident coherence, partial /
 * multiple coherence and cross spectrum of the calls below, which have lifetimes of their own.
 *   - These calls leave a transform resident: cwtb_cwt, cwtb_cwt_dev, cwtb_cwt_to_host, cwtb_xwt
 *     (W12), cwtb_cwt_batch and cwtb_cwt_batch_dev (the last chunk of channels: n_scales x its
 *     channels rows), cwtb_bench_last and cwtb_profile_last (the transform they re-run).
 *   - These leave none: cwtb_wct, cwtb_wct_resident, cwtb_wct3, cwtb_wct3_resident,
 *     cwtb_xwt_resident, every Monte-Carlo call (cwtb_*_mc*), and any call of the first list that
 *     fails once it has begun planning.
 *   - Every other call leaves the resident transform as it is: cwtb_smooth, cwtb_fft_c2c,
 *     cwtb_icwt_sum_host, the surrogate test hooks, the setters, every read and every release.
 * cwtb_job_serial changes when a call of the first two lists begins planning (not at the re-runs).
 * cwtb_get_w, cwtb_icwt_sum, the power calls, cwtb_field_* on CWTB_FIELD_W and cwtb_w_device_ptr
 * read the resident transform: CWTB_ERR_STATE (NULL) when there is none.  cwtb_get_signal_fft,
 * cwtb_padded_length and cwtb_last_plan describe the plan of the last call that planned, whether or
 * not its transform is resident.
 * cwtb_resident_shape reports what is resident, with the sizes every read of it copies: rows (0 when
 * nothing is), n0 and precision (the element type of a complex product; CWTB_F64 for the coherence
 * products, which are double).  Any output may be NULL.  CWTB_ERR_ARG for an unknown product. */
enum cwtb_product {
  CWTB_PRODUCT_W = 0,           /* the transform (CWTB_FIELD_W)                         */
  CWTB_PRODUCT_CROSS = 1,       /* the cross spectrum (CWTB_FIELD_CROSS)               */
  CWTB_PRODUCT_COHERENCE = 2,   /* WCT and aWCT of cwtb_wct_resident                   */
  CWTB_PRODUCT_COHERENCE3 = 3,  /* RP2, the partial phase and RM2 of cwtb_wct3_resident */
  CWTB_PRODUCT_POWER = 5        /* the kept W of cwtb_power_resident (CWTB_FIELD_POWER)     */
};
int cwtb_resident_shape(cwtb_ctx *ctx, int product, int *rows, int64_t *n0, int *precision);

/* Whole call for host callers: H2D signal, transform, one D2H of W into `out`
 * (page-locked memory from cwtb_host_alloc makes the copy run at PCIe speed; the
 * kernels take ~2 % of the copy time at the north-star size, so there is nothing
 * to overlap).  Equivalent to cwtb_cwt + cwtb_get_w. */
int cwtb_cwt_to_host(cwtb_ctx *ctx, const void *signal, int signal_is_f32,
                     int64_t n0, double dt, const double *scales, int n_scales,
                     int family, double param, int precision, void *out,
                     int out_f64);

/* ---- icwt: pycwt/wavelet.py:169-170 -------------------------------------- */
/* out[n] = sum_j Re(W[j,n]) / sqrt(s_j) for the resident W (the caller applies
 * dj*sqrt(dt)/(cdelta*psi(0))).  out: n0 doubles. */
int cwtb_icwt_sum(cwtb_ctx *ctx, double *out);
/* Same reduction for a caller-supplied host W (n_scales x n complex128). */
int cwtb_icwt_sum_host(cwtb_ctx *ctx, const void *W, const double *scales,
                       int n_scales, int64_t n, double *out);

/* ---- derived products of the resident W (SURVEY 8f rank 2) ---------------- */
/* power[j,n] = |W[j,n]|^2 (doubles, n_scales x n0). */
int cwtb_get_power(cwtb_ctx *ctx, double *out);
/* global wavelet spectrum: mean_n |W[j,n]|^2, n_scales doubles
 * (`power.mean(axis=1)`, pycwt/sample/simple_sample.py:79). */
int cwtb_global_power(cwtb_ctx *ctx, double *out);
/* power[j,n] = row_scale[j] * |W[j,n]|^2; row_scale (one factor per row, NULL = 1) carries the
 * rectification 1/s_j of Liu et al. 2007 (`power /= scales[:, None]`, docs/tutorial/cwt.md:49-53)
 * and/or a variance normalisation. */
int cwtb_get_power_scaled(cwtb_ctx *ctx, const double *row_scale, double *out);
/* mean of |W[j,n]|^2 over the columns lo[j] <= n < hi[j] of every row (NaN for an empty range):
 * the global spectrum restricted to the inside of the cone of influence, whose columns form one
 * centred range per scale. */
int cwtb_global_power_ranges(cwtb_ctx *ctx, const int64_t *lo, const int64_t *hi, double *out);
/* scale-averaged power out[n] = sum_j weights[j] * |W[j,n]|^2, n0 doubles (Torrence & Compo 1998
 * eq. 24; `scale_avg`, pycwt/sample/simple_sample.py:88-91: weights[j] = dj*dt/Cdelta/s_j inside
 * the period band, 0 outside).  Rows with weight 0 are not read. */
int cwtb_scale_avg_power(cwtb_ctx *ctx, const double *weights, double *out);

/* ---- xwt / wct: pycwt/wavelet.py:394-399, 498-514; mothers.py:61-104 ------ */
/* Two signals of equal length -> W12 = W1*conj(W2) (n_scales x n0 complex128). */
int cwtb_xwt(cwtb_ctx *ctx, const double *y1, const double *y2, int64_t n0,
             double dt, const double *scales, int n_scales, int family,
             double param, void *W12_out);
/* Wavelet coherence of two signals (Morlet smoothing operator):
 *   WCT = |S(W12/s)|^2 / (S(|W1|^2/s) * S(|W2|^2/s)),  aWCT = angle(W12),
 * S = Gaussian time filter exp(-0.5*(s/dt)^2*k^2) (FFT, zero-pad to Np) followed
 * by a boxcar of `boxcar_len` >= 1 taps with half-weight ends along the scale axis
 * (helpers.py:176-191, scipy convolve2d 'same' alignment).
 * WCT_out, aWCT_out: n_scales x n0 doubles (either may be NULL). */
int cwtb_wct(cwtb_ctx *ctx, const double *y1, const double *y2, int64_t n0,
             double dt, double dj, const double *scales, int n_scales, int family,
             double param, int boxcar_len, double *WCT_out, double *aWCT_out);
/* ---- resident coherence ---------------------------------------------------------------------
 * cwtb_wct_resident computes what cwtb_wct computes (same arguments, same precision:
 * cwtb_set_coherence_precision) but keeps WCT and aWCT (n_scales x n0 doubles each) in a device
 * buffer of their own.  Only cwtb_wct_resident writes that buffer: it stays valid across later
 * cwt / xwt / wct / Monte-Carlo calls, until the next cwtb_wct_resident or cwtb_coherence_release
 * (which frees it; so does cwtb_destroy).  cwtb_coherence_serial changes at both, and is bumped
 * before the buffer is written, so a cwtb_wct_resident that fails part-way changes it too.  The
 * reading calls return CWTB_ERR_STATE when nothing is resident and CWTB_ERR_ARG for bad ranges. */
int cwtb_wct_resident(cwtb_ctx *ctx, const double *y1, const double *y2, int64_t n0,
                      double dt, double dj, const double *scales, int n_scales, int family,
                      double param, int boxcar_len);
int64_t cwtb_coherence_serial(cwtb_ctx *ctx);
int cwtb_coherence_release(cwtb_ctx *ctx);
/* Strided sub-grid of either field (outputs may be NULL), nrows x ncols doubles:
 * out[r][c] = field[row0 + r*row_step][col0 + c*col_step], steps >= 1, every index inside the
 * field.  Whole rows with unit steps are plain device-to-host copies. */
int cwtb_coherence_window(cwtb_ctx *ctx, int row0, int nrows, int row_step, int64_t col0,
                          int64_t ncols, int64_t col_step, double *WCT_out, double *aWCT_out);
/* Per row j, over the columns [lo[j], hi[j]) (lo / hi NULL: the whole row) where thr is NULL or
 * WCT > thr[j] (false for a NaN threshold): out[j] = [count, sum WCT, sum cos aWCT, sum sin aWCT]
 * (S x 4 doubles).  aWCT is not read when want_phase == 0 (its sums are 0).  Deterministic: fixed
 * partition and summation order, repeated calls are bit-identical. */
int cwtb_coherence_row_stats(cwtb_ctx *ctx, const int64_t *lo, const int64_t *hi, const double *thr,
                             int want_phase, double *out);
/* out[3][n0]: sum_j weights[j]*WCT[j,n], sum_j weights[j]*cos aWCT[j,n], sum_j weights[j]*sin
 * aWCT[j,n].  Rows with weight 0 are not read.  Deterministic. */
int cwtb_coherence_scale_avg(cwtb_ctx *ctx, const double *weights, double *out);

/* ---- resident cross spectrum ----------------------------------------------------------------
 * cwtb_xwt_resident runs what cwtb_xwt runs (same arguments without W12_out, same precision:
 * cwtb_set_coherence_precision; un-padded transforms only in fp64, CWTB_TABLE unsupported) and
 * keeps W12 = W1 conj(W2) (n_scales x n0, complex of the engine precision) in a device buffer of
 * its own, the transform's W buffer handed over without a copy.  Lifetime:
 *   - only cwtb_xwt_resident writes that buffer: it survives every other call (cwt*, xwt, wct,
 *     wct_resident, wct_mc*, smooth, cwt_batch*);
 *   - it dies at the next cwtb_xwt_resident or cwtb_cross_release (which frees it; so does
 *     cwtb_destroy).  cwtb_cross_serial changes at both, and is bumped before the buffer is
 *     written, so a cwtb_xwt_resident that fails part-way changes it too;
 *   - afterwards no transform is resident: cwtb_get_w, cwtb_icwt_sum and the power calls return
 *     CWTB_ERR_STATE until the next transform.
 * cwtb_xwt itself is unchanged: its W12 stays the resident transform. */
int cwtb_xwt_resident(cwtb_ctx *ctx, const double *y1, const double *y2, int64_t n0,
                      double dt, const double *scales, int n_scales, int family, double param);
int64_t cwtb_cross_serial(cwtb_ctx *ctx);
int cwtb_cross_release(cwtb_ctx *ctx);

/* ---- resident wavelet power and its tests against surrogates ----------------------------------
 * cwtb_power_resident runs what cwtb_cwt runs on one real series (same arguments, in the precision
 * of cwtb_set_coherence_precision; un-padded transforms only in fp64, CWTB_TABLE unsupported) and
 * keeps its W (n_scales x n0, complex of that precision) in a device buffer of its own, the
 * transform's W buffer handed over without a copy, as cwtb_xwt_resident does.  The power
 * P = re^2 + im^2 of a coefficient is formed in double (exact products for an fp32 W), by one
 * function for the kept W and for every surrogate.  Lifetime:
 *   - only cwtb_power_resident writes that buffer: it survives every other call (cwt*, xwt*, wct*,
 *     the Monte-Carlo calls, the power tests below) byte for byte;
 *   - it dies at the next cwtb_power_resident or cwtb_power_release (which frees it; so does
 *     cwtb_destroy).  cwtb_power_serial changes at both, and is bumped before the buffer is
 *     written, so a cwtb_power_resident that fails part-way changes it too;
 *   - afterwards no transform is resident, as after cwtb_xwt_resident.
 * The cwtb_field_* calls read it as CWTB_FIELD_POWER. */
int cwtb_power_resident(cwtb_ctx *ctx, const double *signal, int64_t n0, double dt, const double *scales,
                        int n_scales, int family, double param);
int64_t cwtb_power_serial(cwtb_ctx *ctx);
int cwtb_power_release(cwtb_ctx *ctx);
/* cwtb_scale_avg_power on the kept W */
int cwtb_power_scale_avg(cwtb_ctx *ctx, const double *weights, double *out);
/* The nulls of the tests against surrogates (power, cross spectrum, coherence).  CWTB_NULL_AR1: unit u is x = m + sigma z, z[0] = e[0],
 * z[i] = g z[i-1] + sqrt(1 - g^2) e[i], e standard normals that are a pure function of (seed, u, i)
 * (the Philox4x32-10 stream of cwtb_wct_mc_seeded under a counter tag of its own: no counter of
 * the white-noise pairs or triples or of the phase-randomised surrogates recurs for
 * 0 <= u < 2^61), drawn on the device by a parallel scan in double (fp32: rounded).
 * CWTB_NULL_PHASE: the phase-randomised surrogates of the series (cwtb_wct_mc_phase, one series in
 * phase group 0): the periodogram is kept exactly. */
enum cwtb_null { CWTB_NULL_AR1 = 0, CWTB_NULL_PHASE = 1 };
/* Test hook: the AR(1) units first_unit .. first_unit + n_units - 1, out[n_units][n0] doubles.
 * CWTB_ERR_ARG: |g| >= 1, a non-finite g, m or sigma, n0 < 1, a negative unit number. */
int cwtb_mc_ar1_surrogates(cwtb_ctx *ctx, double g, double m, double sigma, uint64_t seed,
                           int64_t first_unit, int n_units, int64_t n0, double *out);
/* Point-wise test: for each unit, draw it (`null`; `series` [n0] is the data of the phase null, g,
 * m, sigma the AR(1) null's parameters), transform it with the kept W's plan, exactly as one
 * cwtb_cwt of it in the kept W's precision would, and count on every point
 *   k[s, n] += 1  where  P_unit[s, n] >= P_obs[s, n]  or P_unit[s, n] is not finite
 * into uint32 counters [n_scales][n0] that live with the kept W (4 bytes per scale-point).  Reset,
 * accumulation, CWTB_ERR_STATE (serial, n_scales, n0) and the 2^32 - 1 limit as
 * cwtb_coherence_surrogate_counts; CWTB_ERR_ARG also for an unknown null and the errors of
 * cwtb_mc_ar1_surrogates / cwtb_mc_phase_surrogates.  The units are transformed one at a time. */
int cwtb_power_surrogate_counts(cwtb_ctx *ctx, const double *series, int null, double g, double m, double sigma,
                                uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double dt,
                                const double *scales, int n_scales, int family, double param, int64_t serial,
                                int reset);
/* Cluster test: the units of cwtb_power_surrogate_counts, and the selection, clusters, weights,
 * qmax_out, checks and lifetime of cwtb_coherence_cluster_test with P in place of the coherence
 * (finite P > thr[j] on [lo[j], hi[j])).  The counts are neither read nor changed. */
int cwtb_power_cluster_test(cwtb_ctx *ctx, const double *series, int null, double g, double m, double sigma,
                            uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double dt,
                            const double *scales, int n_scales, int family, double param, int64_t serial,
                            const double *thr, const int64_t *lo, const int64_t *hi, const uint64_t *q,
                            uint64_t *qmax_out);
/* Strided sub-grid of P = re^2 + im^2 of the kept W (the tests' P, in double), nrows x ncols doubles,
 * with the layout and checks of cwtb_field_window: 8 bytes per point cross the bus, not 16. */
int cwtb_power_window(cwtb_ctx *ctx, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                      int64_t col_step, double *out);
/* Reading the counts and clusters, as the cwtb_coherence_* calls of the same names read the
 * coherence's: the p-value window (NaN where P is not finite), the row stats of
 * cwtb_field_row_stats (S x 5) over the points with a finite P and k <= kmax, the histogram of k,
 * the cluster table and the label window. */
int cwtb_power_pvalue_window(cwtb_ctx *ctx, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                             int64_t col_step, double *p_out);
int cwtb_power_pvalue_row_stats(cwtb_ctx *ctx, const int64_t *lo, const int64_t *hi, const double *thr,
                                int64_t kmax, double *out);
int cwtb_power_count_hist(cwtb_ctx *ctx, const int64_t *lo, const int64_t *hi, int64_t nbins, int64_t *out);
int cwtb_power_cluster_table(cwtb_ctx *ctx, int64_t cap, int64_t *count, uint64_t *Q, int64_t *points,
                             int64_t *box);
int cwtb_power_cluster_labels(cwtb_ctx *ctx, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                              int64_t col_step, int32_t *out);
/* cwtb_field_reconstruct of the kept W over the points with a finite P and k <= kmax of the last
 * cwtb_power_surrogate_counts (and P > thr[j] where thr is not NULL).  CWTB_ERR_STATE without a
 * power or without counts. */
int cwtb_power_pvalue_reconstruct(cwtb_ctx *ctx, const double *weights, const int64_t *lo, const int64_t *hi,
                                  const double *thr, int64_t kmax, double *out);
/* cwtb_field_reconstruct of the kept W over the points that the last cwtb_power_cluster_test labelled
 * c + 1 for some c in clusters[0 .. n_clusters) (rows of its table; a repeated row counts once,
 * n_clusters == 0 gives zeros).  CWTB_ERR_STATE before a cluster test, CWTB_ERR_ARG for a row outside
 * the table, n_clusters < 0 or a NULL clusters with n_clusters > 0. */
int cwtb_power_cluster_reconstruct(cwtb_ctx *ctx, const double *weights, const int64_t *lo, const int64_t *hi,
                                   const int64_t *clusters, int64_t n_clusters, double *out);

/* ---- tests of the resident cross spectrum against surrogate pairs -------------------------------
 * The tests of the power above on W12 of cwtb_xwt_resident, with P = |W12|^2 formed by the same
 * function.  |W12|^2 is common power: a burst in one series alone can reach it, so these test common
 * power, not association (the coherence tests do).  The nulls draw two series per unit:
 *   CWTB_NULL_AR1: series s (0, 1) is the AR(1) unit of cwtb_mc_ar1_surrogates with its own g[s],
 *     m[s], sigma[s] under the series tag s of the counter (tag 0 is that call's stream, so series 0
 *     of unit u is its unit u; tag 1 is a stream of its own);
 *   CWTB_NULL_PHASE: the phase-randomised surrogates of `series` [2][n0] (the two transformed
 *     series) in phase groups 0 and 1 (cwtb_mc_phase_surrogates): each keeps its periodogram, with
 *     phases independent of the other's.
 * A unit [2][n0] is transformed exactly as one cwtb_xwt of its two series in the resident W12's
 * precision, one unit at a time.  The counts (uint32, 4 bytes per scale-point) and the clusters
 * live with W12: they die at the next cwtb_xwt_resident, cwtb_cross_release and cwtb_destroy. */
/* Test hook: the AR(1) pairs first_unit .. first_unit + n_units - 1, out[n_units][2][n0] doubles;
 * the errors of cwtb_mc_ar1_surrogates for either series. */
int cwtb_mc_ar1_pair_surrogates(cwtb_ctx *ctx, const double *g, const double *m, const double *sigma,
                                uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double *out);
/* Point-wise test: k[s, n] += 1 where |W12_unit|^2 >= |W12_obs|^2 or is not finite; reset,
 * accumulation, limits and errors as cwtb_power_surrogate_counts.  g, m, sigma [2] (read by the AR(1)
 * null only), series [2][n0] (read by the phase null only). */
int cwtb_cross_surrogate_counts(cwtb_ctx *ctx, const double *series, int null, const double *g, const double *m,
                                const double *sigma, uint64_t seed, int64_t first_unit, int n_units, int64_t n0,
                                double dt, const double *scales, int n_scales, int family, double param,
                                int64_t serial, int reset);
/* Cluster test of finite |W12|^2 > thr[j] on [lo[j], hi[j]), as cwtb_power_cluster_test. */
int cwtb_cross_cluster_test(cwtb_ctx *ctx, const double *series, int null, const double *g, const double *m,
                            const double *sigma, uint64_t seed, int64_t first_unit, int n_units, int64_t n0,
                            double dt, const double *scales, int n_scales, int family, double param, int64_t serial,
                            const double *thr, const int64_t *lo, const int64_t *hi, const uint64_t *q,
                            uint64_t *qmax_out);
/* Reading the counts and clusters, as the cwtb_power_* calls of the same names: the row stats are
 * the five sums of cwtb_field_row_stats, the phase sums included. */
int cwtb_cross_pvalue_window(cwtb_ctx *ctx, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                             int64_t col_step, double *p_out);
int cwtb_cross_pvalue_row_stats(cwtb_ctx *ctx, const int64_t *lo, const int64_t *hi, const double *thr,
                                int64_t kmax, double *out);
int cwtb_cross_count_hist(cwtb_ctx *ctx, const int64_t *lo, const int64_t *hi, int64_t nbins, int64_t *out);
int cwtb_cross_cluster_table(cwtb_ctx *ctx, int64_t cap, int64_t *count, uint64_t *Q, int64_t *points,
                             int64_t *box);
int cwtb_cross_cluster_labels(cwtb_ctx *ctx, int row0, int nrows, int row_step, int64_t col0, int64_t ncols,
                              int64_t col_step, int32_t *out);
/* out[n_scales][5]: the five sums of cwtb_field_row_stats over the points that the last
 * cwtb_cross_cluster_test labelled `cluster` + 1 (row `cluster` of its table), on the columns
 * [lo[j], hi[j]) of each row (pass the cluster's box: nothing outside it is read).  CWTB_ERR_STATE
 * before a cluster test, CWTB_ERR_ARG for a cluster outside the table.  Deterministic. */
int cwtb_cross_cluster_row_stats(cwtb_ctx *ctx, int64_t cluster, const int64_t *lo, const int64_t *hi,
                                 double *out);

/* ---- partial and multiple wavelet coherence of three series (Mihanovic et al. 2009; Ng & Chan
 * 2012) -------------------------------------------------------------------------------------------
 * y, x1, x2: three signals of n0 samples (standardised by the caller as for cwtb_wct).  With S the
 * smoothing operator of cwtb_wct (same boxcar_len, same time filter, cwtb_set_smooth_filter
 * included), S_a = S(|W_a|^2/s) and S_ab = S(W_a conj(W_b)/s):
 *   RP2 = |S_y1 S_2 - S_y2 S_21|^2 / ((S_y S_2 - |S_y2|^2) (S_1 S_2 - |S_12|^2))   (y with x1, x2 removed)
 *   RM2 = 1 - det G3 / (S_y (S_1 S_2 - |S_12|^2))                                  (y on x1 and x2)
 * G3 the 3 x 3 smoothed spectral matrix.  RP2_out, RM2_out: n_scales x n0 doubles, either may be
 * NULL.  No clamping: a denominator that is zero or rounds to <= 0 gives inf or NaN; both measures
 * are ill-conditioned where x1 and x2 are nearly coherent (|S_12|^2 -> S_1 S_2).  The smoothed fields
 * are combined in double in both precisions.  Precision: cwtb_set_coherence_precision; un-padded
 * transforms only in fp64, CWTB_TABLE unsupported.  Lifetime: the resident coherence, partial /
 * multiple coherence and cross spectrum are not written (their handles survive the call); afterwards
 * no transform is resident
 * (cwtb_get_w, cwtb_icwt_sum and the power calls return CWTB_ERR_STATE until the next transform). */
int cwtb_wct3(cwtb_ctx *ctx, const double *y, const double *x1, const double *x2, int64_t n0,
              double dt, double dj, const double *scales, int n_scales, int family, double param,
              int boxcar_len, double *RP2_out, double *RM2_out);

/* ---- resident partial and multiple coherence ---------------------------------------------------
 * cwtb_wct3_resident computes what cwtb_wct3 computes (same arguments without the outputs, same
 * precision switch and errors) and keeps three n_scales x n0 double fields in one device buffer of
 * their own: RP2 at offset 0, the partial phase at offset a and RM2 at offset 2a (in doubles),
 * a = (n_scales*n0 rounded up to a multiple of 32).  24 bytes per scale-point.  The partial phase is
 *   phi = atan2(Im u, Re u),  u = S_y1 S_2 - S_y2 conj(S_12),
 * the angle of the smoothed partial cross spectrum of y and x1 with x2 removed, in the sign convention
 * of cwtb_wct's aWCT (angle of W_y conj(W_x1)); a zero u gives 0, a NaN one NaN.  aWCT is the angle
 * of the unsmoothed cross spectrum, phi of a smoothed quantity, so the two differ even where x2
 * plays no role.  RP2 and RM2 are bit-identical to cwtb_wct3's.  Lifetime:
 *   - only cwtb_wct3_resident writes that buffer: it survives every other call (cwt*, xwt*, wct*,
 *     wct3, the Monte-Carlo calls), and the resident coherence and cross spectrum survive it;
 *   - it dies at the next cwtb_wct3_resident or cwtb_coherence3_release (which frees it; so does
 *     cwtb_destroy).  cwtb_coherence3_serial changes at both, and is bumped before anything else,
 *     so a cwtb_wct3_resident that fails part-way leaves nothing resident;
 *   - afterwards no transform is resident, as after cwtb_wct3.
 * The reading calls take a measure: CWTB_MEASURE_PARTIAL (RP2 with the partial phase) or
 * CWTB_MEASURE_MULTIPLE (RM2, which has no phase: asking for its phase is CWTB_ERR_ARG).  They
 * return CWTB_ERR_STATE when nothing is resident and CWTB_ERR_ARG for a bad measure or range; the
 * reductions are deterministic, as those of cwtb_coherence_*. */
enum cwtb_measure { CWTB_MEASURE_PARTIAL = 0, CWTB_MEASURE_MULTIPLE = 1 };
int cwtb_wct3_resident(cwtb_ctx *ctx, const double *y, const double *x1, const double *x2, int64_t n0,
                       double dt, double dj, const double *scales, int n_scales, int family, double param,
                       int boxcar_len);
int64_t cwtb_coherence3_serial(cwtb_ctx *ctx);
int cwtb_coherence3_release(cwtb_ctx *ctx);
/* Strided sub-grid of the measure (R_out) and of the partial phase (phase_out; PARTIAL only), either
 * may be NULL, nrows x ncols doubles: the layout and checks of cwtb_coherence_window. */
int cwtb_coherence3_window(cwtb_ctx *ctx, int measure, int row0, int nrows, int row_step, int64_t col0,
                           int64_t ncols, int64_t col_step, double *R_out, double *phase_out);
/* out[j] = [count, sum R, sum cos phi, sum sin phi] over the columns [lo[j], hi[j]) (NULL: the
 * whole row) where thr is NULL or R > thr[j] (false for a NaN threshold), S x 4 doubles;
 * want_phase != 0 (PARTIAL only) reads the phase, otherwise its sums are 0. */
int cwtb_coherence3_row_stats(cwtb_ctx *ctx, int measure, const int64_t *lo, const int64_t *hi,
                              const double *thr, int want_phase, double *out);
/* out[3][n0]: sum_j weights[j]*R[j,n], sum_j weights[j]*cos phi[j,n], sum_j weights[j]*sin phi[j,n];
 * for MULTIPLE the two phase planes are 0.  Rows with weight 0 are not read. */
int cwtb_coherence3_scale_avg(cwtb_ctx *ctx, int measure, const double *weights, double *out);

/* Reading calls on a resident complex field: CWTB_FIELD_W (the resident transform's W),
 * CWTB_FIELD_CROSS (the cross spectrum) or CWTB_FIELD_POWER (the kept W of cwtb_power_resident).
 * They return CWTB_ERR_STATE when the field is not resident, CWTB_ERR_UNSUPPORTED for the W of a batched transform and CWTB_ERR_ARG for bad
 * ranges.  Outputs are complex128 / double whatever the field's precision (fp32 fields are widened
 * on the device); the reductions are deterministic (fixed partition and summation order, no
 * atomics: repeated calls are bit-identical). */
/* A complex field has the id of its product (cwtb_resident_shape), so that one id sizes every read of
 * it.  Ids 2 and 3 are the double products, and 4 is no product: it was an unknown product before
 * the power came, and callers that probe for one keep getting CWTB_ERR_ARG from it. */
enum cwtb_field { CWTB_FIELD_W = 0, CWTB_FIELD_CROSS = 1, CWTB_FIELD_POWER = 5 };
/* rows [row0, row0 + nrows), nrows x n0 complex128 */
int cwtb_field_get(cwtb_ctx *ctx, int field, int row0, int nrows, void *out);
/* strided sub-grid, nrows x ncols complex128: out[r][c] = F[row0 + r*row_step][col0 + c*col_step],
 * steps >= 1, every index inside the field (the checks of cwtb_coherence_window) */
int cwtb_field_window(cwtb_ctx *ctx, int field, int row0, int nrows, int row_step, int64_t col0,
                      int64_t ncols, int64_t col_step, void *out);
/* Per row j, over the columns [lo[j], hi[j]) (lo / hi NULL: the whole row) where thr is NULL or
 * re^2 + im^2 > thr[j] (in double, false for a NaN threshold): out[j] = [count, sum |F|^2,
 * sum |F|, sum cos phi, sum sin phi] (S x 5 doubles), |F| = sqrt(re^2 + im^2), cos phi = re/|F|,
 * sin phi = im/|F|; a zero coefficient has phase 0 (adds (1, 0)). */
int cwtb_field_row_stats(cwtb_ctx *ctx, int field, const int64_t *lo, const int64_t *hi,
                         const double *thr, double *out);
/* Reconstruction over a selection (Torrence & Compo 1998, eq. 29 restricted to selected points), the
 * column-wise counterpart of cwtb_field_row_stats: out[n] = sum_j weights[j] * Re F[j,n] (n0 doubles)
 * over the points with lo[j] <= n < hi[j] and, where thr is not NULL, re^2 + im^2 > thr[j] (in double,
 * false for a NaN threshold).  The inverse transform's factor dj sqrt(dt) / (Cdelta psi(0)) is the
 * caller's; pass weights[j] = 1 / sqrt(s_j) on the rows to sum and 0 elsewhere: rows with weight 0
 * or an empty range are not read, and a column without a selected point is 0.  For CWTB_FIELD_W and
 * CWTB_FIELD_POWER only: CWTB_ERR_ARG for CWTB_FIELD_CROSS (no inverse is defined for it), an unknown
 * field, a NULL weights / lo / hi / out, lo[j] < 0, lo[j] > hi[j] or hi[j] > n0.  Each column adds
 * its rows in ascending order, each step weights[j] * Re F rounded and then added rounded (no fused
 * multiply-add, no atomics): repeated calls are bit-identical. */
int cwtb_field_reconstruct(cwtb_ctx *ctx, int field, const double *weights, const int64_t *lo,
                           const int64_t *hi, const double *thr, double *out);
/* out[n] = sum_j weights[j] * W12[j,n] (n0 complex128) over the cross spectrum.  Rows with weight
 * 0 are not read. */
int cwtb_cross_scale_avg(cwtb_ctx *ctx, const double *weights, void *out);

/* Morlet.smooth on a caller-supplied host array (mothers.py:61-104).
 * in: n_scales x n (complex128 if is_complex else float64); out same type.  At most 65535 scales
 * (one launch row each): more are refused with CWTB_ERR_ARG. */
int cwtb_smooth(cwtb_ctx *ctx, const void *in, int is_complex, int n_scales,
                int64_t n, double dt, const double *scales, int boxcar_len,
                void *out);

/* ---- Monte-Carlo coherence significance: pycwt/wavelet.py:609-630 --------- */
/* Accumulates, over `n_pairs` surrogate pairs of length n0, the histogram
 * hist[s, floor(R2*nbins)] += 1 for rows s < maxscale and points with
 * mask[s, n] != 0 (period <= coi).  `noise` is a host array
 * [n_pairs, 2, n0] of doubles drawn by the caller (exact-parity mode: the caller
 * uses numpy's RNG exactly as the reference does).  hist: n_scales x nbins int64,
 * accumulated into (not cleared). */
int cwtb_wct_mc(cwtb_ctx *ctx, const double *noise, int n_pairs, int64_t n0,
                double dt, double dj, const double *scales, int n_scales,
                int family, double param, int boxcar_len, const uint8_t *mask,
                int maxscale, int nbins, int64_t *hist);
/* The same accumulation with the surrogates drawn ON THE DEVICE (SURVEY 8b vi "seed"): pair number
 * first_pair + i is standard-normal white noise from the counter-based Philox4x32-10 stream keyed
 * by (seed, pair number), so a run does not depend on how the pairs are split over calls, ranks
 * or GPUs.  Statistically equivalent to the reference's surrogates (which are white noise too,
 * helpers.py:146-173), not bit-identical to numpy's stream; no host RNG and no H2D of noise. */
int cwtb_wct_mc_seeded(cwtb_ctx *ctx, uint64_t seed, int64_t first_pair, int n_pairs, int64_t n0,
                       double dt, const double *scales, int n_scales, int family, double param,
                       int boxcar_len, const uint8_t *mask, int maxscale, int nbins, int64_t *hist);
/* Test hook: the surrogates of the seeded mode, out[n_pairs][2][n0]. */
int cwtb_mc_surrogates(cwtb_ctx *ctx, uint64_t seed, int64_t first_pair, int n_pairs, int64_t n0,
                       double *out);

/* ---- Monte-Carlo significance of the partial and multiple coherence (cwtb_wct3) ------------- */
/* Null: three mutually independent white-noise series of n0 samples per triple, not standardised,
 * each triple through the whole cwtb_wct3 pipeline (same smoothing, boxcar, time filter table).
 * Accumulates, over `n_triples` triples, hist_partial[s, b] += 1 for RP2 and hist_multiple[s, b] += 1
 * for RM2 with b = clamp(floor(R2*nbins), 0, nbins-1), for rows s < maxscale and points with
 * mask[s, n] != 0; a non-finite R2 (a zero denominator) is not counted.  Either histogram may be
 * NULL (its measure is then not evaluated), not both; each is n_scales x nbins int64, accumulated
 * into (not cleared).  `noise`: host array [n_triples][3][n0] of doubles (y, x1, x2 of each triple).
 * Precision, errors and lifetime as cwtb_wct3: the resident coherence and cross spectrum survive
 * the call; afterwards no transform is resident. */
int cwtb_wct3_mc(cwtb_ctx *ctx, const double *noise, int n_triples, int64_t n0, double dt,
                 const double *scales, int n_scales, int family, double param, int boxcar_len,
                 const uint8_t *mask, int maxscale, int nbins, int64_t *hist_partial,
                 int64_t *hist_multiple);
/* The same with the triples drawn on the device: series r (0 = y, 1 = x1, 2 = x2) of triple
 * first_triple + i is a pure function of (seed, triple number, r), from the Philox4x32-10 stream of
 * cwtb_wct_mc_seeded with a tag bit of its own, so triple t and pair t of one seed share no series
 * and no split over calls, ranks or GPUs changes a triple. */
int cwtb_wct3_mc_seeded(cwtb_ctx *ctx, uint64_t seed, int64_t first_triple, int n_triples, int64_t n0,
                        double dt, const double *scales, int n_scales, int family, double param,
                        int boxcar_len, const uint8_t *mask, int maxscale, int nbins,
                        int64_t *hist_partial, int64_t *hist_multiple);
/* Test hook: the triples of the seeded mode, out[n_triples][3][n0]. */
int cwtb_mc_surrogates3(cwtb_ctx *ctx, uint64_t seed, int64_t first_triple, int n_triples, int64_t n0,
                        double *out);

/* ---- Monte-Carlo significance against phase-randomised surrogates of the data -------------- */
/* Null: the data themselves with their Fourier phases randomised (Theiler et al. 1992; multivariate
 * form Prichard & Theiler 1994).  With X = FFT_n0(x) at the series' own length, unit u of a series
 * in phase group g is x' = Re IFFT_n0(X'), X'_k = X_k e^{i phi(u,g,k)} for 1 <= k < n0/2,
 * X'_{n0-k} = conj(X'_k), X'_0 = X_0 and, for even n0, X'_{n0/2} = X_{n0/2}: every series keeps its
 * power spectrum, mean and variance; series of one group share phi and keep their cross spectrum and
 * coherence; series of different groups become independent.  phi = 2 pi U, U uniform in (0, 1) from
 * the Philox4x32-10 stream keyed by `seed`, a pure function of (seed, u, g, k) with a counter tag of
 * its own (no counter of cwtb_wct_mc_seeded / cwtb_wct3_mc_seeded recurs for 0 <= u < 2^61), so no
 * split over calls, ranks or GPUs changes a unit.  Transforms and rotation run in fp64; an fp32
 * coherence gets the fp64 surrogates rounded.
 * series: host [nser][n0] doubles, nser = 2 or 3; group[nser]: phase group (>= 0) of each series.
 * nser = 2: hist_a = coherence histogram, hist_b must be NULL.
 * nser = 3 (y, x1, x2): hist_a = partial, hist_b = multiple, either may be NULL, not both.
 * Everything else (mask, maxscale, nbins, accumulate-into, precision, smoothing filter, lifetime of
 * resident results) as cwtb_wct_mc_seeded / cwtb_wct3_mc_seeded.
 * CWTB_ERR_ARG: nser not 2 or 3, a negative group or unit number, n0 < 4, a null pointer;
 * CWTB_ERR_UNSUPPORTED: CWTB_TABLE wavelets, n0 > 2^26, or n0 > 2^24 that is not a power of two. */
int cwtb_wct_mc_phase(cwtb_ctx *ctx, const double *series, int nser, const int *group, uint64_t seed,
                      int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                      int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                      int maxscale, int nbins, int64_t *hist_a, int64_t *hist_b);
/* Test hook: the surrogates themselves, out[n_units][nser][n0]. */
int cwtb_mc_phase_surrogates(cwtb_ctx *ctx, const double *series, int nser, const int *group,
                             uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double *out);
/* cwtb_wct_mc_phase with the null of choice (cwtb_wct_mc_phase is this call with CWTB_NULL_PHASE):
 *   CWTB_NULL_PHASE: the phase-randomised surrogates of `series` in the phase groups `group`, as
 *     cwtb_wct_mc_phase (g, m, sigma and held are not read);
 *   CWTB_NULL_AR1: series s of unit u is the AR(1) series of cwtb_mc_ar1_surrogates with its own
 *     g[s], m[s], sigma[s] under the series tag s of the counter (tag 0 is that call's stream, tag 1
 *     the second series of cwtb_mc_ar1_pair_surrogates, tag 2 a stream of its own), at the data's
 *     length n0, in double (fp32: rounded).  held[s] = 1 (held may be NULL: none) keeps row s of
 *     `series` [nser][n0] in every unit instead, uploaded once per call in the coherence precision
 *     as cwtb_wct3 uploads its inputs; only x1 and x2 of three series can be held.  `group` is not
 *     read; `series` only for the held rows.
 * CWTB_ERR_ARG also for an unknown null, AR(1) parameters that cwtb_mc_ar1_surrogates refuses (of
 * the drawn series), a held flag other than 0 / 1, on y or on a series of a pair, and held rows
 * without `series`. */
int cwtb_wct_mc_null(cwtb_ctx *ctx, const double *series, int nser, int null, const int *group, const double *g,
                     const double *m, const double *sigma, const int *held, uint64_t seed, int64_t first_unit,
                     int n_units, int64_t n0, double dt, const double *scales, int n_scales, int family,
                     double param, int boxcar_len, const uint8_t *mask, int maxscale, int nbins, int64_t *hist_a,
                     int64_t *hist_b);
/* Test hook: the AR(1) units of nser = 1, 2 or 3 series (tags 0 .. nser - 1),
 * out[n_units][nser][n0]; nser = 2 is cwtb_mc_ar1_pair_surrogates, nser = 1 cwtb_mc_ar1_surrogates. */
int cwtb_mc_ar1_series_surrogates(cwtb_ctx *ctx, int nser, const double *g, const double *m, const double *sigma,
                                  uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double *out);

/* ---- point-wise tests of the resident coherence against phase-randomised surrogates ----------
 * cwtb_coherence_surrogate_counts (two series: the resident coherence of cwtb_wct_resident) and
 * cwtb_coherence3_surrogate_counts (three: the resident RP2 and RM2 of cwtb_wct3_resident) run the
 * units first_unit .. first_unit + n_units - 1 of cwtb_wct_mc_phase (same arguments, same surrogates,
 * same histograms accumulated into hist / hist_partial, hist_multiple) and also count, for every
 * point of every row (the cone of influence and the rows from maxscale on included),
 *   k[s, n] += 1  where  R2_unit[s, n] >= R2_obs[s, n]  or R2_unit[s, n] is not finite,
 * into uint32 counters [n_scales][n0] per measure that live with the resident product (4 bytes per
 * scale-point for the coherence, 8 for the partial and multiple coherence), allocated at the first
 * call.  reset != 0 zeroes them first; otherwise the units are added to the ones already counted, so
 * units [0, a) then [a, M) give the counts of [0, M).  CWTB_ERR_STATE: `serial` is not the product's
 * current serial (cwtb_coherence_serial / cwtb_coherence3_serial), or n_scales / n0 differ from the
 * resident product's.  CWTB_ERR_ARG: the arguments of cwtb_wct_mc_phase, or a total of units above
 * 2^32 - 1.  The counts compare like with like only when the call runs the plan the product was
 * computed with (the same scales, precision, padding mode and smoothing filter).  Lifetime: the
 * counts die with their product (a new cwtb_wct_resident / cwtb_wct3_resident, the release calls,
 * cwtb_destroy); a counting call that fails leaves none readable. */
int cwtb_coherence_surrogate_counts(cwtb_ctx *ctx, const double *series, const int *group, uint64_t seed,
                                    int64_t first_unit, int n_units, int64_t n0, double dt,
                                    const double *scales, int n_scales, int family, double param,
                                    int boxcar_len, const uint8_t *mask, int maxscale, int nbins,
                                    int64_t *hist, int64_t serial, int reset);
int cwtb_coherence3_surrogate_counts(cwtb_ctx *ctx, const double *series, const int *group, uint64_t seed,
                                     int64_t first_unit, int n_units, int64_t n0, double dt,
                                     const double *scales, int n_scales, int family, double param,
                                     int boxcar_len, const uint8_t *mask, int maxscale, int nbins,
                                     int64_t *hist_partial, int64_t *hist_multiple, int64_t serial,
                                     int reset);
/* The same with the null of choice, as cwtb_wct_mc_null (the calls above are these with
 * CWTB_NULL_PHASE).  The counts remember the null of their units: reset == 0 on counts of another
 * null is CWTB_ERR_STATE. */
int cwtb_coherence_surrogate_counts_null(cwtb_ctx *ctx, const double *series, int null, const int *group,
                                         const double *g, const double *m, const double *sigma, const int *held,
                                         uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double dt,
                                         const double *scales, int n_scales, int family, double param,
                                         int boxcar_len, const uint8_t *mask, int maxscale, int nbins, int64_t *hist,
                                         int64_t serial, int reset);
int cwtb_coherence3_surrogate_counts_null(cwtb_ctx *ctx, const double *series, int null, const int *group,
                                          const double *g, const double *m, const double *sigma, const int *held,
                                          uint64_t seed, int64_t first_unit, int n_units, int64_t n0, double dt,
                                          const double *scales, int n_scales, int family, double param,
                                          int boxcar_len, const uint8_t *mask, int maxscale, int nbins,
                                          int64_t *hist_partial, int64_t *hist_multiple, int64_t serial, int reset);
/* Reading the counts of M units.  They return CWTB_ERR_STATE when the product or its counts are not
 * resident, and the errors of the corresponding cwtb_coherence*_window / _row_stats calls.
 * p-value window: p = (1 + k) / (1 + M) in double, NaN where the observed value is not finite, with
 * the layout and checks of cwtb_coherence_window. */
int cwtb_coherence_pvalue_window(cwtb_ctx *ctx, int row0, int nrows, int row_step, int64_t col0,
                                 int64_t ncols, int64_t col_step, double *p_out);
int cwtb_coherence3_pvalue_window(cwtb_ctx *ctx, int measure, int row0, int nrows, int row_step,
                                  int64_t col0, int64_t ncols, int64_t col_step, double *p_out);
/* The row stats of cwtb_coherence_row_stats / cwtb_coherence3_row_stats over the points whose
 * observed value is finite and whose count k <= kmax (and R > thr[j] where thr is given).  A
 * selection p <= alpha is the cut kmax = the largest k with (1 + k) / (1 + M) <= alpha. */
int cwtb_coherence_pvalue_row_stats(cwtb_ctx *ctx, const int64_t *lo, const int64_t *hi, const double *thr,
                                    int64_t kmax, int want_phase, double *out);
int cwtb_coherence3_pvalue_row_stats(cwtb_ctx *ctx, int measure, const int64_t *lo, const int64_t *hi,
                                     const double *thr, int64_t kmax, int want_phase, double *out);
/* out[k] (nbins = M + 1 int64, else CWTB_ERR_ARG) = the number of points with count k over the
 * columns [lo[j], hi[j]) of every row j whose observed value is finite: the histogram that decides
 * a Benjamini-Hochberg / -Yekutieli step-up test on the host.  Integer sums: bit-identical. */
int cwtb_coherence_count_hist(cwtb_ctx *ctx, const int64_t *lo, const int64_t *hi, int64_t nbins,
                              int64_t *out);
int cwtb_coherence3_count_hist(cwtb_ctx *ctx, int measure, const int64_t *lo, const int64_t *hi,
                               int64_t nbins, int64_t *out);

/* ---- cluster tests of the resident coherence against phase-randomised surrogates -------------
 * cwtb_coherence_cluster_test (the resident coherence) and cwtb_coherence3_cluster_test (the
 * resident RP2 or RM2, by `measure`) take the arguments of cwtb_coherence*_surrogate_counts (same
 * units, surrogates and histograms) and, per row j of the map, a threshold thr[j], a column range
 * [lo[j], hi[j]) and a weight q[j] <= 2^32.  In the resident map and in the map of every unit, point
 * (j, n) is selected where the value is finite, > thr[j] (a NaN selects nothing) and
 * lo[j] <= n < hi[j].  Clusters are the 8-connected components of the selection in the
 * (row, column) grid; column 0 and column n0 - 1 are not neighbours.  A cluster's Q is the sum of
 * q[j] over its points, in uint64.  qmax_out[i] (n_units uint64) receives the largest Q of unit
 * first_unit + i, 0 without clusters; the clusters of the resident map are kept with the product
 * (the label image takes 4 bytes per scale-point).  The counts of an earlier surrogate-count call
 * are neither read nor changed.  CWTB_ERR_UNSUPPORTED: n_scales * n0 >= 2^32.  CWTB_ERR_ARG: a
 * weight above 2^32, a column range outside [0, n0) or lo > hi, an unknown measure, and the
 * errors of cwtb_coherence*_surrogate_counts, whose CWTB_ERR_STATE cases apply too.  Lifetime:
 * the clusters die with their product (a new cwtb_wct_resident / cwtb_wct3_resident, the release
 * calls, cwtb_destroy) and with the next cluster test of it; a call that fails leaves none
 * readable. */
int cwtb_coherence_cluster_test(cwtb_ctx *ctx, const double *series, const int *group, uint64_t seed,
                                int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                int maxscale, int nbins, int64_t *hist, int64_t serial, const double *thr,
                                const int64_t *lo, const int64_t *hi, const uint64_t *q, uint64_t *qmax_out);
int cwtb_coherence3_cluster_test(cwtb_ctx *ctx, const double *series, const int *group, uint64_t seed,
                                 int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                 int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                 int maxscale, int nbins, int64_t *hist_partial, int64_t *hist_multiple,
                                 int64_t serial, const double *thr, const int64_t *lo, const int64_t *hi,
                                 const uint64_t *q, int measure, uint64_t *qmax_out);
/* The same with the null of choice, as cwtb_wct_mc_null (the calls above are these with
 * CWTB_NULL_PHASE). */
int cwtb_coherence_cluster_test_null(cwtb_ctx *ctx, const double *series, int null, const int *group, const double *g,
                                     const double *m, const double *sigma, const int *held, uint64_t seed,
                                     int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                     int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                     int maxscale, int nbins, int64_t *hist, int64_t serial, const double *thr,
                                     const int64_t *lo, const int64_t *hi, const uint64_t *q, uint64_t *qmax_out);
int cwtb_coherence3_cluster_test_null(cwtb_ctx *ctx, const double *series, int null, const int *group, const double *g,
                                      const double *m, const double *sigma, const int *held, uint64_t seed,
                                      int64_t first_unit, int n_units, int64_t n0, double dt, const double *scales,
                                      int n_scales, int family, double param, int boxcar_len, const uint8_t *mask,
                                      int maxscale, int nbins, int64_t *hist_partial, int64_t *hist_multiple,
                                      int64_t serial, const double *thr, const int64_t *lo, const int64_t *hi,
                                      const uint64_t *q, int measure, uint64_t *qmax_out);
/* The clusters of the resident map of the last cluster test, ordered by Q descending, ties by the
 * row-major index of the cluster's first point: *count = their number, and the first
 * min(cap, count) rows into Q[cap], points[cap] (point count) and box[cap][4] = first row, last
 * row + 1, first column, last column + 1.  CWTB_ERR_STATE: no product resident, or no cluster test
 * has completed for it. */
int cwtb_coherence_cluster_table(cwtb_ctx *ctx, int64_t cap, int64_t *count, uint64_t *Q, int64_t *points,
                                 int64_t *box);
int cwtb_coherence3_cluster_table(cwtb_ctx *ctx, int64_t cap, int64_t *count, uint64_t *Q, int64_t *points,
                                  int64_t *box);
/* Window of the label image: 0 off the clusters, c + 1 on the cluster of table row c, int32, with
 * the layout and checks of cwtb_coherence_window and the errors of the table calls. */
int cwtb_coherence_cluster_labels(cwtb_ctx *ctx, int row0, int nrows, int row_step, int64_t col0,
                                  int64_t ncols, int64_t col_step, int32_t *out);
int cwtb_coherence3_cluster_labels(cwtb_ctx *ctx, int row0, int nrows, int row_step, int64_t col0,
                                   int64_t ncols, int64_t col_step, int32_t *out);
/* Test hook: labels a host bitmask bits [n_scales][ceil(n0 / 32)] (column n: bit n % 32 of word
 * n / 32; no bit set past column n0 - 1) with the weights q[n_scales] through the cluster tests'
 * labeller: the table as cwtb_coherence_cluster_table returns it, the label image labels
 * [n_scales][n0] (may be NULL) and the largest Q into *qmax.  The shape is checked before anything
 * is read or allocated: CWTB_ERR_UNSUPPORTED for n_scales * n0 >= 2^32, CWTB_ERR_ARG for more than
 * 65535 scales (one launch row each). */
int cwtb_cluster_label_bits(cwtb_ctx *ctx, const uint32_t *bits, int n_scales, int64_t n0, const uint64_t *q,
                            int64_t cap, int64_t *count, uint64_t *Q, int64_t *points, int64_t *box,
                            int32_t *labels, uint64_t *qmax);

/* ---- batched transform of independent channels (SURVEY 8d config 5) ------- */
/* X: host [n_chan, n0] (float or double).  The per-channel transforms stay on
 * the device; `power_out` (may be NULL) receives the per-channel global wavelet
 * spectra [n_chan, n_scales] (doubles); `W_out` (may be NULL) receives all
 * coefficients [n_chan, n_scales, n0] in the engine precision.  The channels are
 * processed in chunks (CWTB_BATCH_MB of coefficients each).  With `power_out` only,
 * the chunks are pipelined: the input copy of chunk k+1 (straight from the caller's
 * array, pageable memory is fine) overlaps the kernels of chunk k, the spectra are
 * accumulated on the device and copied back once; the call returns when
 * `power_out` is complete. */
int cwtb_cwt_batch(cwtb_ctx *ctx, const void *X, int x_is_f32, int n_chan,
                   int64_t n0, double dt, const double *scales, int n_scales,
                   int family, double param, int precision, double *power_out,
                   void *W_out);

/* Device-resident variant: d_X [n_chan][n0] already on the device in the engine's real type;
 * one chunk (n_chan * n_scales rows <= 60000); W [n_chan][n_scales][n0] stays resident
 * (cwtb_w_device_ptr); power_out (may be NULL): host [n_chan][n_scales] mean |W|^2. */
int cwtb_cwt_batch_dev(cwtb_ctx *ctx, const void *d_X, int n_chan, int64_t n0, double dt,
                       const double *scales, int n_scales, int family, double param,
                       int precision, double *power_out);

/* ---- timing / introspection (bench.py, tests) ----------------------------- */
/* Device time (ms, CUDA events on the context's stream) of the kernels of the
 * last cwtb_cwt* / cwtb_xwt / cwtb_wct / cwtb_wct_mc call, excluding H2D/D2H; and the number
 * of kernel launches. */
double cwtb_last_kernel_ms(cwtb_ctx *ctx);
int cwtb_last_launch_count(cwtb_ctx *ctx);
/* Fills `out` (capacity n) with one int per scale of the last call:
 * log2 of the pruned transform length K' (0 if the scale used the direct small-N
 * kernel), or -log2(Nc) if the scale ran on the expansion path with a coarse grid of Nc points,
 * -1 for every scale of an un-padded transform, or CWTB_PLAN_OS (-2) if it ran as an overlap-save
 * convolution with its truncated impulse response (coarse grids have at least 2^6 points, so the
 * codes do not overlap).
 * Returns the number written. */
#define CWTB_PLAN_OS (-2)
int cwtb_last_plan(cwtb_ctx *ctx, int *out, int n);
/* Re-run the kernels of the last cwtb_cwt_dev call `iters` times and return the
 * mean device time per iteration in ms (events on the launching stream). */
int cwtb_bench_last(cwtb_ctx *ctx, int iters, double *ms_out);
/* One pass of the last cwtb_cwt_dev transform with a CUDA event pair around every kernel
 * launch, on a single stream (the normal run overlaps independent kernel chains on three
 * streams); writes "name|launches|total_ms|rows" lines (rows = scale rows processed) to out. */
int cwtb_profile_last(cwtb_ctx *ctx, char *out, size_t cap);
/* The same table for ANY sequence of calls (xwt, wct, wct_mc, smooth, batches): every kernel
 * launched between begin and end is bracketed by an event pair, on one stream. */
int cwtb_profile_begin(cwtb_ctx *ctx);
int cwtb_profile_end(cwtb_ctx *ctx, char *out, size_t cap);
/* Device memory helpers for benchmarks (inputs resident in HBM). */
int cwtb_dev_alloc(cwtb_ctx *ctx, size_t bytes, void **out);
int cwtb_dev_free(cwtb_ctx *ctx, void *p);
int cwtb_memcpy_h2d(cwtb_ctx *ctx, void *dst, const void *src, size_t bytes);
int cwtb_memcpy_d2h(cwtb_ctx *ctx, void *dst, const void *src, size_t bytes);
int cwtb_sync(cwtb_ctx *ctx);

/* Test hook: plain batched complex DFT of `batch` rows of length n through the engine's own
 * kernels (any n >= 2; lengths other than 2^k go through Bluestein's algorithm, fp64 only; any
 * batch, run in chunks of at most 65535 rows);
 * sign = -1 forward, +1 inverse (unnormalised).
 * in/out: host complex128 (precision selects the arithmetic). */
int cwtb_fft_c2c(cwtb_ctx *ctx, const void *in, void *out, int64_t n, int batch,
                 int sign, int precision);

/* ---- multi-GPU (SURVEY.md 8b vii, 8e) ------------------------------------------------------
 * One context per GPU (one process per GPU, or one host thread per context).  The transform
 * itself needs no collective: channels (pycwt.cwt per channel, wavelet.py:13-124), scales and
 * Monte-Carlo surrogate pairs (wavelet.py:609-630) are independent units that the caller
 * block-partitions over the ranks.  These entry points move the REDUCED products over
 * NVLink / NVSwitch with NCCL (bound at run time from libnccl.so.2; CWTB_ERR_COMM if absent):
 * per-channel spectra (all-gather), surrogate histograms (all-reduce), timings (max).
 * Buffers are host arrays, staged through device memory owned by the context.
 *   rank 0:  cwtb_comm_unique_id(id);  the host program hands the 128 bytes to every rank
 *   all:     cwtb_comm_init(ctx, world, rank, id);  ...collectives...;  cwtb_comm_destroy(ctx)
 * world == 1 needs no NCCL: the collectives are copies / no-ops. */
int cwtb_comm_unique_id(void *id128);
int cwtb_comm_init(cwtb_ctx *ctx, int world, int rank, const void *id128);
int cwtb_comm_destroy(cwtb_ctx *ctx);
int cwtb_comm_world(cwtb_ctx *ctx);
int cwtb_comm_rank(cwtb_ctx *ctx);
/* recv[r*bytes .. (r+1)*bytes) = rank r's `send` (bytes per rank, equal on all ranks) */
int cwtb_comm_allgather(cwtb_ctx *ctx, const void *send, void *recv, size_t bytes);
/* in place, every rank gets the result */
int cwtb_comm_allreduce_sum_i64(cwtb_ctx *ctx, int64_t *buf, size_t count);
int cwtb_comm_allreduce_max_f64(cwtb_ctx *ctx, double *buf, size_t count);
int cwtb_comm_broadcast(cwtb_ctx *ctx, void *buf, size_t bytes, int root);

#ifdef __cplusplus
}
#endif
#endif /* CWT_B200_H */
