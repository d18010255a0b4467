"""Tests of the resident wavelet power against AR(1) and phase-randomised surrogates, on the GPU.

The checks of test_emu_power_test.py on the device: the AR(1) units against the host restatement,
the counts, p-values, FDR threshold and clusters against a recount of the hooks' surrogates through
engine-level `cwt`, nothing else moving, lifetime and errors.  Then config 4's first series
(n0 = 2^18, 145 scales), fp64 and fp32, and config 2's geometry (2^20 x 256), fp64: the counts and
unit maxima of a few units against the recount.  Last, that the tests do what they claim: the
family-wise error of the cluster test and the point-wise rate on AR(1) noise, and a burst found.
"""
import numpy as np
import pytest
from scipy.stats import binom

import test_emu_cluster_test as C
import test_emu_power_test as E
from test_emu_surrogate_significance import red
from test_gpu_surrogate_pvalues import eng, api  # noqa: F401  (fixtures)

F64, F32 = E.F64, E.F32


def _unpad_after(fn, *a):
    from pycwt_b200 import helpers
    try:
        fn(*a)
    finally:
        helpers.set_fft_padding(True)


@pytest.mark.gpu
@pytest.mark.parametrize("g", [-0.9, 0.0, 0.5, 0.95])
@pytest.mark.parametrize("n", [4, 1001, 65537, 2 ** 17])
def test_ar1_units_match_host(eng, g, n):
    E.test_ar1_units_match_host(eng, g, n)


@pytest.mark.gpu
def test_ar1_units_split_and_seed(eng):
    E.test_ar1_units_split_and_seed(eng)
    # many units in one call: more than one launch of MAX_ROWS units is not needed, many CTAs are
    whole = eng.mc_ar1_surrogates(0.3, 0.0, 1.0, 8, 0, 64, 2 ** 20)
    part = eng.mc_ar1_surrogates(0.3, 0.0, 1.0, 8, 63, 1, 2 ** 20)
    assert np.array_equal(whole[63], part[0])


@pytest.mark.gpu
@pytest.mark.parametrize("null,prec,wav,n0,padded", E.CASES + [('ar1', 'fp32', 'morlet', 4096, True),
                                                              ('phase', 'fp64', 'dog', 4097, False)])
def test_counts_are_the_definition(api, eng, null, prec, wav, n0, padded):
    _unpad_after(E.test_counts_are_the_definition, api, eng, None, null, prec, wav, n0, padded)


@pytest.mark.gpu
def test_readers(api, eng):
    E.test_readers(api, eng)


@pytest.mark.gpu
@pytest.mark.parametrize("null,prec", [('ar1', 'fp64'), ('phase', 'fp32'), ('ar1', 'fp32')])
def test_cluster_test_against_recount(api, eng, null, prec):
    E.test_cluster_test_against_recount(api, eng, null, prec)


@pytest.mark.gpu
def test_nothing_else_moves(api, eng):
    E.test_nothing_else_moves(api, eng)


@pytest.mark.gpu
def test_lifetime_and_errors(api, eng):
    _unpad_after(E.test_lifetime_and_errors, api, eng, None)


# ---- config sizes: the recount by row blocks ------------------------------------------------------
def _recount_blocks(h, null, seed, M, thr=None, rows=32):
    """(k [S, n0], unit maxima of the selection P > thr inside the cone) of units 0 .. M - 1, each
    through engine-level `cwt` with W left on the device and read back in blocks of rows."""
    from pycwt_b200._engine import FIELD_W
    eng = h.engine
    S, n0 = h.shape
    prec = F32 if h.precision == 'fp32' else F64
    k = np.zeros((S, n0), dtype=np.int64)
    q = C.weights(h.scales)
    lo, hi = h.coi_ranges()
    qmax = []
    for x in E.surrogates(h, null, seed, 0, M):
        eng.cwt(x, h.dt, h.scales, *h.wavelet._engine_spec(), precision=prec, fetch=False)
        sel = np.zeros((S, n0), dtype=bool) if thr is not None else None
        for r0 in range(0, S, rows):
            nr = min(rows, S - r0)
            W = eng.field_window(FIELD_W, r0, nr, 1, 0, n0, 1)
            Pi = W.real * W.real + W.imag * W.imag
            del W
            Wo = h.window(slice(r0, r0 + nr))
            Po = Wo.real * Wo.real + Wo.imag * Wo.imag
            del Wo
            k[r0:r0 + nr] += (Pi >= Po) | ~np.isfinite(Pi)
            if sel is not None:
                cols = np.arange(n0)[None]
                sel[r0:r0 + nr] = np.isfinite(Pi) & (Pi > thr[r0:r0 + nr, None]) & \
                    (cols >= lo[r0:r0 + nr, None]) & (cols < hi[r0:r0 + nr, None])
        if sel is not None:
            Q = C.reference(sel, q)[0]
            qmax.append(int(Q[0]) if Q.size else 0)
    return k, qmax


def _check_config(api, h, null, M, seed):
    from pycwt_b200.resident import _cluster_weights
    W0 = h.wave().tobytes()
    h.surrogate_test(mc_count=M, seed=seed, null=null)
    Pobs = h.power()
    thr = np.quantile(Pobs, 0.95, axis=1)
    del Pobs
    res = h.cluster_test(thr, mc_count=M, seed=seed, null=null)
    k, qmax = _recount_blocks(h, null, seed, M, thr)
    S, n0 = h.shape
    for r0 in range(0, S, 32):
        W = h.window(slice(r0, r0 + 32))
        Po = W.real * W.real + W.imag * W.imag
        assert np.array_equal(h.pvalues(slice(r0, r0 + 32)), E.p_of(k[r0:r0 + 32], M, Po), equal_nan=True)
    _, unit_area = _cluster_weights(h)
    assert np.array_equal(res.null_max, np.array(qmax, dtype=float) * unit_area)
    assert h.wave().tobytes() == W0
    print("  %s %s %s: %d clusters, unit maxima %s" % (h.shape, h.precision, null, res.area.size, qmax))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
def test_config4_units(api, prec):
    """Config 4's first series (n0 = 2^18, 145 scales): 8 units, counts and maxima against the
    recount, both nulls split over the two precisions."""
    import workloads as wl
    c = wl.C4
    y = wl.config4_signals()[0]
    h = api.power_resident(y, c["dt"], dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=api.Morlet(c["f0"]),
                           precision=prec)
    assert h.shape == (145, 2 ** 18)
    _check_config(api, h, 'ar1' if prec == 'fp64' else 'phase', 8, 31)


@pytest.mark.gpu
def test_config2_units(api):
    """Config 2's geometry (2^20 points, 256 scales), fp64: 2 AR(1) units against the recount."""
    import workloads as wl
    c = wl.C2
    h = api.power_resident(wl.config2_signal(), c["dt"], dj=c["dj"], s0=c["s0"], J=c["J"],
                           wavelet=api.Morlet(c["f0"]))
    assert h.shape == (256, 2 ** 20)
    _check_config(api, h, 'ar1', 2, 32)


# ---- it tests what it claims ---------------------------------------------------------------------
KW = dict(dj=1 / 4, s0=2.0, J=28)


def _chi2_level(api, h, x):
    """The 95 % chi-squared level of `significance()` for the standardised series, power units."""
    g = api.ar1(x)[0]
    return api.significance(1.0, h.dt, h.scales, 0, g)[0]


@pytest.mark.gpu
def test_red_noise_rates(api):
    """40 AR(1) datasets (g = 0.7, n0 = 2048, periods 2 .. 256 at dj = 1/4), M = 99 units of the
    AR(1) null.  Family-wise error: `cluster_test` at the 95 % chi-squared level of
    `significance()`; the number of datasets with a cluster at p <= 0.05 is Binomial(40, <= 0.05):
    more than 6 has probability below 0.002.  Point-wise rate: the mean share of the points inside
    the cone of influence with p <= 0.05 lies in [0.03, 0.07].  Observed with these seeds on an
    H100: 3 of 40 datasets, a mean point-wise share of 0.0513."""
    rs = np.random.RandomState(77)
    hits, shares = 0, []
    for d in range(40):
        x = red(rs, 2048, 0.7)[0]
        h = api.power_resident(x, 1.0, **KW)
        res = h.cluster_test(_chi2_level(api, h, x), mc_count=99, seed=4000 + d)
        hits += bool((res.pvalue <= 0.05).any())
        h.surrogate_test(mc_count=99, seed=5000 + d)
        lo, hi = h.coi_ranges()
        cols = np.arange(h.n0)[None]
        cone = (cols >= lo[:, None]) & (cols < hi[:, None])
        shares.append(float((h.pvalues()[cone] <= 0.05).mean()))
    rate = float(np.mean(shares))
    print("  datasets with a cluster at p <= 0.05: %d of 40; mean point-wise share at p <= 0.05: %.4f"
          % (hits, rate))
    assert hits <= 6 and binom.sf(hits - 1, 40, 0.05) > 0.002
    assert 0.03 <= rate <= 0.07


@pytest.mark.gpu
@pytest.mark.parametrize("null", ['ar1', 'phase'])
def test_burst_found(api, null):
    """A sinusoidal burst of period 32 over samples [4000, 4400) (Hann window, amplitude 2.5) in AR(1)
    noise (g = 0.5), n0 = 8192, M = 99: the largest cluster at the 95 % chi-squared level has
    p <= 0.05, most of its points lie within one octave of period 32 and inside the burst's time span
    widened by two periods.  Observed with these seeds on an H100, under both nulls: 387 clusters, the
    largest of area 7.6 at p = 0.020 over rows [13, 18) and columns [4037, 4350), all of its points
    within the octave and the span."""
    rs = np.random.RandomState(12)
    n = np.arange(8192)
    win = np.where((n >= 4000) & (n < 4400), np.sin(np.pi * (n - 4000) / 400.0) ** 2, 0.0)
    x = red(rs, 8192, 0.5)[0] + 2.5 * win * np.sin(2 * np.pi * n / 32.0)
    h = api.power_resident(x, 1.0, **KW)
    res = h.cluster_test(_chi2_level(api, h, x), mc_count=99, seed=9, null=null)
    lab = h.cluster_labels() == 1
    near = np.abs(np.log2(h.period / 32.0)) <= 1.0
    share_scale = lab[near].sum() / lab.sum()
    share_time = lab[:, 3936:4464].sum() / lab.sum()
    print("  burst, %s null: %d clusters, largest area %.1f at p = %.3f, rows %s cols %s, share near "
          "period 32 %.3f, inside the span %.3f" % (null, res.area.size, res.area[0], res.pvalue[0],
                                                    res.rows[0], res.cols[0], share_scale, share_time))
    assert res.pvalue[0] <= 0.05
    assert share_scale >= 0.75 and share_time >= 0.75
