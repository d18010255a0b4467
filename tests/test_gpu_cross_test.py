"""Tests of the resident cross spectrum against AR(1) and phase-randomised surrogate pairs, on the GPU.

The checks of test_emu_cross_test.py on the device: the AR(1) pairs against the power test's units
and the host restatement, the counts, p-values, reductions and clusters against a recount of the
hooks' pairs through engine-level `xwt`, scaling by powers of two, nothing else moving, lifetime and
errors.  Then config 4's pair (n0 = 2^18, 145 scales) in fp64 under the AR(1) null and in fp32 under
the phase null: the counts and unit maxima of 8 pairs against the recount.  Last, that the tests do
what they claim: the family-wise error of the cluster test and the point-wise rate on independent
AR(1) pairs, a common burst found with its lag, and a burst in one series alone found too (common
power is not association).
"""
import numpy as np
import pytest
from scipy.stats import binom

import test_emu_cluster_test as C
import test_emu_cross_test as X
from test_emu_surrogate_significance import red
from test_gpu_surrogate_pvalues import eng, api  # noqa: F401  (fixtures)

F64, F32 = X.F64, X.F32


def _unpad_after(fn, *a):
    from pycwt_b200 import helpers
    try:
        fn(*a)
    finally:
        helpers.set_fft_padding(True)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4, 1001, 65537])
def test_ar1_pairs(eng, n):
    X.check_ar1_pairs(eng, n)


@pytest.mark.gpu
def test_ar1_pair_errors(eng):
    X.test_ar1_pair_errors(eng)


@pytest.mark.gpu
@pytest.mark.parametrize("null,prec,wav,n0,padded", X.CASES + [('ar1', 'fp32', 'morlet', 4096, True),
                                                              ('phase', 'fp64', 'dog', 4097, False)])
def test_counts_are_the_definition(api, null, prec, wav, n0, padded):
    _unpad_after(X.check_counts_are_the_definition, api, null, prec, wav, n0, padded)


@pytest.mark.gpu
@pytest.mark.parametrize("null,prec", [('phase', 'fp64'), ('ar1', 'fp32')])
def test_readers(api, null, prec):
    X.check_readers(api, null, prec)


@pytest.mark.gpu
@pytest.mark.parametrize("null,prec", [('ar1', 'fp64'), ('phase', 'fp32'), ('ar1', 'fp32')])
def test_cluster_test_against_recount(api, null, prec):
    X.check_cluster_test(api, null, prec)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,exps", [('fp64', [(200, -190), (-200, 180)]), ('fp32', [(24, 20), (-40, 30)])])
@pytest.mark.parametrize("null", ['ar1', 'phase'])
def test_scaling(api, prec, exps, null):
    X.check_scaling(api, prec, exps, null)


@pytest.mark.gpu
def test_nothing_else_moves(api):
    X.check_nothing_else_moves(api)


@pytest.mark.gpu
def test_lifetime_and_errors(api):
    _unpad_after(X.check_lifetime_and_errors, api)


# ---- config 4: the recount by row blocks -----------------------------------------------------------
def _recount_blocks(h, null, seed, M, thr, rows=32):
    """(k [S, n0], unit maxima of the selection |W12|^2 > thr inside the cone) of pairs 0 .. M - 1,
    each through engine-level `xwt`, compared in blocks of rows."""
    eng = h.engine
    S, n0 = h.shape
    k = np.zeros((S, n0), dtype=np.int64)
    q = C.weights(h.scales)
    lo, hi = h.coi_ranges()
    cols = np.arange(n0)[None]
    qmax = []
    for x in X.surrogates(h, null, seed, 0, M):
        W12 = eng.xwt(x[0], x[1], h.dt, h.scales, *h.wavelet._engine_spec(), precision=X.engine_prec(h))
        sel = np.zeros((S, n0), dtype=bool)
        for r0 in range(0, S, rows):
            nr = min(rows, S - r0)
            W = W12[r0:r0 + nr]
            Pi = W.real * W.real + W.imag * W.imag
            Wo = h.window(slice(r0, r0 + nr))
            Po = Wo.real * Wo.real + Wo.imag * Wo.imag
            k[r0:r0 + nr] += (Pi >= Po) | ~np.isfinite(Pi)
            sel[r0:r0 + nr] = np.isfinite(Pi) & (Pi > thr[r0:r0 + nr, None]) & \
                (cols >= lo[r0:r0 + nr, None]) & (cols < hi[r0:r0 + nr, None])
        del W12
        Q = C.reference(sel, q)[0]
        qmax.append(int(Q[0]) if Q.size else 0)
    return k, qmax


@pytest.mark.gpu
@pytest.mark.parametrize("prec,null", [('fp64', 'ar1'), ('fp32', 'phase')])
def test_config4_units(api, prec, null):
    """Config 4's pair (n0 = 2^18, 145 scales): 8 pairs, counts and maxima against the recount,
    read in blocks of rows.  Observed on an H100: 289 clusters at `h.signif` in both precisions."""
    from pycwt_b200.resident import _cluster_weights
    import workloads as wl
    c = wl.C4
    y = wl.config4_signals()
    h = api.xwt_resident(y[0], y[1], c["dt"], dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=api.Morlet(c["f0"]),
                         precision=prec)
    assert h.shape == (145, 2 ** 18)
    M, seed = 8, 31
    W0 = h.cross_spectrum().tobytes()
    h.surrogate_test(mc_count=M, seed=seed, null=null)
    sig = h.signif
    res = h.cluster_test(sig, mc_count=M, seed=seed, null=null)
    k, qmax = _recount_blocks(h, null, seed, M, sig ** 2)
    S, n0 = h.shape
    for r0 in range(0, S, 32):
        W = h.window(slice(r0, r0 + 32))
        Po = W.real * W.real + W.imag * W.imag
        assert np.array_equal(h.pvalues(slice(r0, r0 + 32)), X.p_of(k[r0:r0 + 32], M, Po), equal_nan=True)
    _, unit_area = _cluster_weights(h)
    assert np.array_equal(res.null_max, np.array(qmax, dtype=float) * unit_area)
    assert h.cross_spectrum().tobytes() == W0
    print("  %s %s %s: %d clusters, unit maxima %s" % (h.shape, prec, null, res.area.size, qmax))


# ---- it tests what it claims ---------------------------------------------------------------------
KW = dict(dj=1 / 4, s0=2.0, J=28)


def check_red_noise_rates(api, datasets=40, M=99):
    rs = np.random.RandomState(78)
    hits, shares = 0, []
    for d in range(datasets):
        y1 = red(rs, 2048, 0.7)[0]
        y2 = red(rs, 2048, 0.3)[0]
        h = api.xwt_resident(y1, y2, 1.0, **KW)
        res = h.cluster_test(h.signif, mc_count=M, seed=4000 + d)
        hits += bool((res.pvalue <= 0.05).any())
        h.surrogate_test(mc_count=M, seed=5000 + d)
        lo, hi = h.coi_ranges()
        cols = np.arange(h.n0)[None]
        cone = (cols >= lo[:, None]) & (cols < hi[:, None])
        shares.append(float((h.pvalues()[cone] <= 0.05).mean()))
    return hits, float(np.mean(shares))


@pytest.mark.gpu
def test_red_noise_rates(api):
    """40 pairs of independent AR(1) series (g = 0.7 and 0.3, n0 = 2048, periods 2 .. 256 at
    dj = 1/4), M = 99 pairs of the AR(1) null.  Family-wise error: `cluster_test` at `h.signif`; the
    number of datasets with a cluster at p <= 0.05 is Binomial(40, <= 0.05): more than 6 has
    probability below 0.002.  Point-wise rate: the mean share of the points inside the cone of
    influence with p <= 0.05 lies in [0.03, 0.07].  Observed with these seeds on an H100: 2 of 40
    datasets, a mean point-wise share of 0.0512."""
    hits, rate = check_red_noise_rates(api)
    print("  datasets with a cluster at p <= 0.05: %d of 40; mean point-wise share at p <= 0.05: %.4f"
          % (hits, rate))
    assert hits <= 6 and binom.sf(hits - 1, 40, 0.05) > 0.002
    assert 0.03 <= rate <= 0.07


def burst_pair(common, amp=2.5, seed=12):
    """Two AR(1) series (g = 0.5, n0 = 8192) with a Hann-windowed period-32 burst over [4000, 4400):
    in both, y2 a quarter period behind y1 (`common`), or in y1 alone; and the noise-free bursts."""
    rs = np.random.RandomState(seed)
    n = np.arange(8192)
    win = np.where((n >= 4000) & (n < 4400), np.sin(np.pi * (n - 4000) / 400.0) ** 2, 0.0)
    b1 = amp * win * np.sin(2 * np.pi * n / 32.0)
    b2 = amp * win * np.sin(2 * np.pi * (n - 8) / 32.0) if common else 0.0 * n
    return red(rs, 8192, 0.5)[0] + b1, red(rs, 8192, 0.5)[0] + b2, b1, b2


def check_burst(api, null, common, amp=2.5):
    """(result, shares near period 32 and inside the span, mean phase of cluster 0, its reference)."""
    y1, y2, b1, b2 = burst_pair(common, amp)
    h = api.xwt_resident(y1, y2, 1.0, **KW)
    res = h.cluster_test(h.signif, mc_count=99, seed=9, null=null)
    lab = h.cluster_labels() == 1
    near = np.abs(np.log2(h.period / 32.0)) <= 1.0
    share_scale = lab[near].sum() / lab.sum()
    share_time = lab[:, 3936:4464].sum() / lab.sum()
    mp = h.mean_phase(cluster=0)
    ref = None
    if common:
        # the lag's angle with the sign of angle(W1 conj W2), from the noise-free pair
        W12 = api.xwt(b1, b2, 1.0, normalize=False, **KW)[0]
        j = int(np.argmin(np.abs(np.log2(h.period / 32.0))))
        ref = float(np.angle(W12[j, 4100:4300].sum()))
    return res, share_scale, share_time, mp, ref


@pytest.mark.gpu
@pytest.mark.parametrize("null", ['ar1', 'phase'])
def test_common_burst_found(api, null):
    """A Hann-windowed burst of period 32 over samples [4000, 4400) (amplitude 2.5) in both of two
    independent AR(1) series (g = 0.5, n0 = 8192), y2 a quarter period behind, M = 99: the largest
    cluster at `h.signif` has p <= 0.05, at least 75 % of its points lie within one octave of period
    32 and inside the burst's span widened by two periods, and `mean_phase(cluster=0)` is the lag's
    angle within 0.3 rad.  Observed with these seeds on an H100, under both nulls: 118 clusters, the
    largest of area 6.4 at p = 0.010 over rows [14, 18) and columns [4066, 4341), all of its points
    within the octave and the span, mean phase 1.668 rad against 1.571 for the noise-free pair."""
    res, ss, st, mp, ref = check_burst(api, null, True)
    print("  common burst, %s null: %d clusters, largest area %.1f at p = %.3f, rows %s cols %s, share "
          "near period 32 %.3f, inside the span %.3f, phase %.3f (noise-free %.3f)"
          % (null, res.area.size, res.area[0], res.pvalue[0], res.rows[0], res.cols[0], ss, st, mp.angle, ref))
    assert res.pvalue[0] <= 0.05
    assert ss >= 0.75 and st >= 0.75
    assert abs(np.angle(np.exp(1j * (mp.angle - ref)))) <= 0.3


@pytest.mark.gpu
def test_burst_in_one_series(api):
    """The burst in y1 alone, at amplitude 6: |W12|^2 is common power, and the AR(1) test finds the
    burst as a significant patch although y2 has nothing there (Maraun & Kurths 2004; the coherence
    tests are the tests of association).  At amplitude 2.5 a burst in one series is not the largest
    patch.  The phase null's result is printed, not asserted.  Observed with these seeds on an H100:
    114 clusters, the largest of area 3.7 over rows [14, 18) and columns [4126, 4316), all of its
    points within the octave and the span, at p = 0.010 (AR(1)) and p = 0.030 (phase)."""
    for null in ('ar1', 'phase'):
        res, ss, st, mp, _ = check_burst(api, null, False, amp=6.0)
        print("  burst in y1 only, %s null: %d clusters, largest area %.1f at p = %.3f, rows %s cols %s, "
              "share near period 32 %.3f, inside the span %.3f"
              % (null, res.area.size, res.area[0], res.pvalue[0], res.rows[0], res.cols[0], ss, st))
        if null == 'ar1':
            assert res.pvalue[0] <= 0.05
            assert ss >= 0.75 and st >= 0.75
