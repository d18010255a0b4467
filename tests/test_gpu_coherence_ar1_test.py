"""Tests of the resident coherence and the partial and multiple coherence against AR(1) red-noise
surrogates (`null='ar1'`), on the GPU.

The checks of test_emu_coherence_ar1_test.py on the device, then config 4's geometry (n0 = 2^18, 145
scales): the counts and unit maxima of a few units against a recount through engine-level `wct` /
`wct3`, read in blocks of rows, for the pair and the conditional triple in fp64 and fp32.  Last,
that the tests do what they claim: the family-wise error of the cluster test and the point-wise rate
on independent AR(1) pairs, the cluster error of the conditional partial test when x1 and x2 share a
driver, and bursts found by the pair test and by the conditional partial test.
"""
import numpy as np
import pytest
from scipy.stats import binom

import test_emu_cluster_test as C
import test_emu_coherence_ar1_test as A
import test_emu_surrogate_pvalues as P
from test_emu_surrogate_significance import red
from test_gpu_surrogate_pvalues import eng, api  # noqa: F401  (fixtures)

F64, F32 = A.F64, A.F32


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4, 1001, 65537])
def test_units(eng, n):
    A.test_units(eng, n)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser,conditional", A.NULLS)
@pytest.mark.parametrize("n0,K", [(4096, 6), (600, 36)])
def test_counts_are_the_definition(eng, nser, conditional, n0, K, prec):
    A.check_counts(eng, nser, conditional, n0, K, prec)


@pytest.mark.gpu
@pytest.mark.parametrize("nser,conditional,prec,wav,n0,padded", A.CASES)
def test_public(api, eng, nser, conditional, prec, wav, n0, padded):
    from pycwt_b200 import helpers, mothers
    old = mothers.enable_generic_smoothing(True)
    try:
        A.test_public(api, eng, None, nser, conditional, prec, wav, n0, padded)
    finally:
        mothers.enable_generic_smoothing(old)
        helpers.set_fft_padding(True)
        eng.set_padding(True)


@pytest.mark.gpu
def test_no_units_of_another_null(eng):
    A.test_no_units_of_another_null(eng)


# ---- config 4: the recount by row blocks -----------------------------------------------------------
def _recount_blocks(h, U, M, measure, thr, rows=32):
    """(k [S, n0] of `measure`, unit maxima of the selection R > thr inside the cone) of the units U,
    each through engine-level `wct` / `wct3`, compared in blocks of rows."""
    S, n0 = h.shape
    k = np.zeros((S, n0), dtype=np.int64)
    q = C.weights(h.scales)
    lo, hi = h.coi_ranges()
    qmax = []
    for u in U:
        R = A.handle_fields(h, u[None])[measure][0]
        sel = np.zeros((S, n0), dtype=bool)
        for r0 in range(0, S, rows):
            sl = slice(r0, min(S, r0 + rows))
            w = h.window(sl)
            o = w[0] if measure == 0 else w[2]
            k[sl] += (R[sl] >= o) | ~np.isfinite(R[sl])
            sel[sl] = C.select(R[sl], thr[sl], lo[sl], hi[sl])
        del R
        Q = C.reference(sel, q)[0]
        qmax.append(int(Q[0]) if Q.size else 0)
    return k, qmax


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
@pytest.mark.parametrize("nser", [2, 3])
def test_config4_units(api, prec, nser):
    """Config 4's geometry (n0 = 2^18, 145 scales): 3 units of the AR(1) null (the conditional one for
    three series), counts and maxima against the recount, read in blocks of rows."""
    from pycwt_b200.resident import _cluster_weights
    import workloads as wl
    c = wl.C4
    y = list(wl.config4_signals())
    if nser == 3:
        y.append(red(np.random.RandomState(4), y[0].size, 0.6)[0] + 0.3 * y[1])
    fn = api.wct_resident if nser == 2 else api.wct3_resident
    h = fn(*y, c["dt"], dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=api.Morlet(c["f0"]), precision=prec)
    assert h.shape == (145, 2 ** 18)
    M, seed = 3, 31
    h.surrogate_test(mc_count=M, seed=seed, null='ar1')
    S, n0 = h.shape
    thr = np.full(S, 0.8)
    res = h.cluster_test(thr, mc_count=M, seed=seed, null='ar1')
    k, qmax = _recount_blocks(h, A.handle_units(h, seed, M), M, 0, thr)
    for r0 in range(0, S, 32):
        sl = slice(r0, r0 + 32)
        o = h.window(sl)[0]
        p = h.pvalues(sl) if nser == 2 else h.pvalues(sl, measure='partial')
        assert np.array_equal(p, P.p_of(k[sl], M, o), equal_nan=True)
    _, unit_area = _cluster_weights(h)
    assert np.array_equal(res.null_max, np.array(qmax, dtype=float) * unit_area)
    print("  %s %s nser %d: %d clusters, unit maxima %s" % (h.shape, prec, nser, res.area.size, qmax))


# ---- it tests what it claims ---------------------------------------------------------------------
KW = dict(dj=1 / 4, s0=2.0, J=28)


def _cone(h):
    lo, hi = h.coi_ranges()
    cols = np.arange(h.n0)[None]
    return (cols >= lo[:, None]) & (cols < hi[:, None])


@pytest.mark.gpu
def test_red_noise_rates_pair(api):
    """40 pairs of independent AR(1) series (g = 0.8 and 0.5, n0 = 2048, dj = 1/4), M = 99 pairs of
    the AR(1) null, `sig` from `surrogate_significance(null='ar1')` of another seed.  Family-wise
    error: the number of datasets with a cluster at p <= 0.05 is Binomial(40, <= 0.05), more than 6
    has probability 0.0034.  Point-wise rate: the mean share of the points inside the cone with
    p <= 0.05 lies in [0.03, 0.07]."""
    rs = np.random.RandomState(91)
    hits, shares = 0, []
    for d in range(40):
        y1, y2 = red(rs, 2048, 0.8)[0], red(rs, 2048, 0.5)[0]
        h = api.wct_resident(y1, y2, 1.0, **KW)
        sig = h.surrogate_significance(mc_count=99, seed=3000 + d, null='ar1')
        res = h.cluster_test(sig, mc_count=99, seed=4000 + d, null='ar1')
        hits += bool((res.pvalue <= 0.05).any())
        h.surrogate_test(mc_count=99, seed=5000 + d, null='ar1')
        shares.append(float((h.pvalues()[_cone(h)] <= 0.05).mean()))
    rate = float(np.mean(shares))
    print("  pair: datasets with a cluster at p <= 0.05: %d of 40; mean point-wise share: %.4f" % (hits, rate))
    assert hits <= 6 and binom.sf(hits - 1, 40, 0.05) > 0.002
    assert 0.03 <= rate <= 0.07


def _triple(rs, n=2048):
    """y independent AR(1) noise; x1 and x2 share a strong AR(1) driver."""
    drv = red(rs, n, 0.8)[0]
    return red(rs, n, 0.6)[0], drv + 0.4 * red(rs, n, 0.5)[0], drv + 0.4 * red(rs, n, 0.5)[0]


@pytest.mark.gpu
def test_red_noise_rates_triple(api):
    """40 triples with y independent of x1 and x2, which share a strong AR(1) driver: the conditional
    AR(1) test's RP2 clusters at p <= 0.05 appear in at most 6 of 40 datasets.  The rate of
    `conditional=False` is printed, not asserted."""
    rs = np.random.RandomState(92)
    hits = {True: 0, False: 0}
    for d in range(40):
        h = api.wct3_resident(*_triple(rs), 1.0, **KW)
        for cond in (True, False):
            sig = h.surrogate_significance(mc_count=99, seed=3000 + d, null='ar1', conditional=cond)[0]
            res = h.cluster_test(sig, mc_count=99, seed=4000 + d, null='ar1', conditional=cond)
            hits[cond] += bool((res.pvalue <= 0.05).any())
    print("  triple: datasets with an RP2 cluster at p <= 0.05: conditional %d of 40, unconditional %d of 40"
          % (hits[True], hits[False]))
    assert hits[True] <= 6


def _burst(n=8192, amp=2.5):
    t = np.arange(n)
    win = np.where((t >= 4000) & (t < 4400), np.sin(np.pi * (t - 4000) / 400.0) ** 2, 0.0)
    return amp * win * np.sin(2 * np.pi * t / 32.0)


def _found(h, res):
    """p of the first cluster, and whether it lies near period 32 and inside the burst's span."""
    lab = h.cluster_labels() == 1
    near = np.abs(np.log2(h.period / 32.0)) <= 1.0
    return float(res.pvalue[0]), lab[near][:, 3936:4464].sum() / max(lab.sum(), 1)


@pytest.mark.gpu
def test_burst_pair(api):
    rs = np.random.RandomState(12)
    b = _burst()
    h = api.wct_resident(red(rs, 8192, 0.5)[0] + b, red(rs, 8192, 0.5)[0] + b, 1.0, **KW)
    sig = h.surrogate_significance(mc_count=99, seed=1, null='ar1')
    res = h.cluster_test(sig, mc_count=99, seed=9, null='ar1')
    p, share = _found(h, res)
    print("  pair burst: cluster 0 at p = %.3f, %.2f of it near period 32 inside the burst" % (p, share))
    assert p <= 0.05 and share > 0.5


@pytest.mark.gpu
def test_burst_partial(api):
    rs = np.random.RandomState(13)
    b = _burst()
    y, x1, x2 = red(rs, 8192, 0.5)[0] + b, red(rs, 8192, 0.5)[0] + b, red(rs, 8192, 0.5)[0]
    h = api.wct3_resident(y, x1, x2, 1.0, **KW)
    sig = h.surrogate_significance(mc_count=99, seed=1, null='ar1')[0]
    res = h.cluster_test(sig, mc_count=99, seed=9, null='ar1')
    p, share = _found(h, res)
    print("  partial burst: cluster 0 at p = %.3f, %.2f of it near period 32 inside the burst" % (p, share))
    assert p <= 0.05 and share > 0.5
