"""Cluster tests of the resident coherence against phase-randomised surrogates, on the GPU.

The checks of test_emu_cluster_test.py on the device: the labeller against SciPy on the masks of
that file, every unit's largest cluster sum and the observed table and labels against a recount of
the hook's surrogates through engine-level `wct` / `wct3`, nothing else moving.  Then config 4's
data sizes (n0 = 2^18, 145 scales, K = 14), fp64 and fp32, pairs and triples: the maxima of 8 units
against the recount and a 50-unit `cluster_test`.  Last, that the test does what it claims: its
family-wise error on independent red noise, and a shared oscillation found.
"""
import numpy as np
import pytest
from scipy.stats import binom
from test_emu_surrogate_significance import red

import test_emu_cluster_test as C
import test_emu_surrogate_pvalues as P
import test_gpu_surrogate_significance as G
from test_gpu_surrogate_pvalues import eng, api  # noqa: F401  (fixtures)

F64, F32 = P.F64, P.F32
NBINS = P.NBINS


@pytest.mark.gpu
@pytest.mark.parametrize("name,sel", C.masks(), ids=[m[0] for m in C.masks()])
def test_labeller_matches_scipy(eng, name, sel):
    C.check_hook(eng, sel)


@pytest.mark.gpu
def test_labeller_large(eng):
    """Many CTAs per row and many rows: random masks around the percolation density, a full map."""
    rs = np.random.RandomState(5)
    for S, n0, d in ((64, 70001, 0.41), (300, 4096, 0.6), (3, 2 ** 17, 0.95)):
        C.check_hook(eng, rs.rand(S, n0) < d)
    C.check_hook(eng, np.ones((40, 40000), dtype=bool))
    alt = np.zeros((33, 65537), dtype=bool)
    alt[:, 1::2] = True
    C.check_hook(eng, alt)


@pytest.mark.gpu
def test_labeller_rejects(eng):
    C.test_labeller_rejects(eng)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser,measure", [(2, None), (3, 0), (3, 1)])
@pytest.mark.parametrize("n0,K", [(512, 6), (600, 36), (4096, 80)])
def test_units_are_the_definition(eng, nser, measure, n0, K, prec):
    C.check_units(eng, nser, n0, K, prec, measure=measure)


@pytest.mark.gpu
@pytest.mark.parametrize("nser,measure", [(2, None), (3, 1)])
def test_units_unpadded(eng, nser, measure):
    eng.set_padding(False)
    try:
        C.check_units(eng, nser, 4099, 6, F64, M=3, measure=measure)
    finally:
        eng.set_padding(True)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
def test_public_pair(api, eng, prec):
    C.test_public_pair(api, eng, prec)


@pytest.mark.gpu
@pytest.mark.parametrize("measure,conditional", [('partial', True), ('multiple', False)])
def test_public_triple(api, eng, measure, conditional):
    C.test_public_triple(api, eng, measure, conditional)


@pytest.mark.gpu
def test_lifetime_and_errors(api, eng):
    C.test_lifetime_and_errors(api, eng)


@pytest.mark.gpu
def test_engine_errors(eng):
    C.test_engine_errors(eng)


# ---- config 4 --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser", [2, 3])
def test_config4_units(eng, nser, prec):
    """Config 4's data sizes: the maxima of 8 units and the observed table against the recount."""
    c, prob, data = G._config4()
    x = data[:nser]
    sj = prob["sj"]
    S, n0 = sj.size, x.shape[1]
    groups = (0, 1) if nser == 2 else (0, 1, 1)
    measure = None if nser == 2 else 0
    if nser == 2:
        serial = eng.wct_resident(x[0], x[1], c["dt"], c["dj"], sj, P.MORLET, c["f0"], 14, precision=prec)
    else:
        serial = eng.wct3_resident(*x, c["dt"], c["dj"], sj, P.MORLET, c["f0"], 14, precision=prec)
    before = P.observed(eng, nser)
    obs = before[0]
    thr = np.nanquantile(np.where(np.isfinite(obs), obs, np.nan), 0.9, axis=1)
    lo, hi = np.zeros(S, dtype=np.int64), np.full(S, n0, dtype=np.int64)
    q = C.weights(sj)
    hs = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    qmax = eng.cluster_test(x, groups, 17, 0, 8, c["dt"], sj, P.MORLET, c["f0"], 14, prob["mask"],
                            prob["maxscale"], NBINS, *hs, serial=serial, thr=thr, lo=lo, hi=hi, q=q,
                            measure=measure, precision=prec)
    after = P.observed(eng, nser)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before, after))
    assert all(np.array_equal(a, b) for a, b in zip(hs, G._run(eng, c, prob, x, groups, 17, 0, 8, prec)))
    surr = eng.mc_phase_surrogates(x, groups, 17, 0, 8)
    ref = []
    for u in range(8):
        if nser == 2:
            R = eng.wct(surr[u, 0], surr[u, 1], c["dt"], c["dj"], sj, P.MORLET, c["f0"], 14, want_angle=False,
                        precision=prec)[0]
        else:
            R = eng.wct3(*surr[u], c["dt"], c["dj"], sj, P.MORLET, c["f0"], 14, precision=prec)[0]
        Q = C.reference(C.select(R, thr, lo, hi), q)[0]
        ref.append(int(Q[0]) if Q.size else 0)
    assert np.array_equal(qmax, np.array(ref, dtype=np.uint64))
    Q, pts, box = eng.cluster_table(nser == 3)
    rQ, rpts, rbox, rlab = C.reference(C.select(obs, thr, lo, hi), q)
    assert np.array_equal(Q, rQ) and np.array_equal(pts, rpts) and np.array_equal(box, rbox)
    assert np.array_equal(eng.cluster_labels(nser == 3, 0, S, 1, 0, n0, 1), rlab)
    print("  config 4, %d series, prec %d: %d clusters, unit maxima %s" % (nser, prec, Q.size, list(qmax)))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
@pytest.mark.parametrize("nser", [2, 3])
def test_config4_public(api, nser, prec):
    """A 50-unit cluster_test at config 4's sizes, with the levels of 50 other units as threshold."""
    import workloads as wl
    c = wl.C4
    y, x1 = wl.config4_signals()
    x2 = 0.6 * x1 + wl.chirp(c["n"], phase=2.1) + 0.5 * np.random.RandomState(2).randn(c["n"])
    kw = dict(dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=api.Morlet(c["f0"]), precision=prec)
    if nser == 2:
        h = api.wct_resident(y, x1, c["dt"], **kw)
        sig = h.surrogate_significance(mc_count=50, seed=23)
        res = h.cluster_test(sig, mc_count=50, seed=24)
    else:
        h = api.wct3_resident(y, x1, x2, c["dt"], **kw)
        sig = h.surrogate_significance(mc_count=50, seed=23)[1]
        res = h.cluster_test(sig, mc_count=50, seed=24, measure='multiple')
    assert h.shape == (145, 2 ** 18)
    assert res.null_max.shape == (50,) and res.area.size > 0
    assert set(np.unique(res.pvalue)) <= {(1 + k) / 51 for k in range(51)}
    lab = h.cluster_labels(slice(None, None, 4), slice(None, None, 64))
    assert lab.max() <= res.area.size
    print("  config 4 public, %d series, %s: %d clusters, largest area %.1f (p = %.3f), null max median %.1f"
          % (nser, prec, res.area.size, res.area[0], res.pvalue[0], np.median(res.null_max)))


# ---- it tests what it claims ---------------------------------------------------------------------
@pytest.mark.gpu
def test_red_noise_familywise_rate(api):
    """40 datasets of two independent AR(1) series (a = 0.7), n0 = 2048, periods 2 .. 256 (dj = 1/4),
    M = 99: the cluster-forming threshold is `surrogate_significance` at 95 % from units of one seed,
    the null from another.  Under the null, the number of datasets with a cluster at p <= 0.05 is
    Binomial(40, <= 0.05): more than 6 has probability below 0.002.  Observed with these seeds on an
    H100: 2 of 40.  The point-wise test of the first dataset paints points with p <= 0.05."""
    rs = np.random.RandomState(2024)
    hits = 0
    for d in range(40):
        x = red(rs, 2048, 0.7, 2)
        h = api.wct_resident(x[0], x[1], 1.0, dj=1 / 4, s0=2.0, J=28)
        sig = h.surrogate_significance(mc_count=99, seed=1000 + d)
        res = h.cluster_test(sig, mc_count=99, seed=2000 + d)
        hits += bool((res.pvalue <= 0.05).any())
        if d == 0:
            h.surrogate_test(mc_count=99, seed=3000)
            assert (h.pvalues()[P.coi_mask(h)] <= 0.05).sum() > 0
    print("  datasets with a cluster at p <= 0.05: %d of 40" % hits)
    assert hits <= 6 and binom.sf(hits - 1, 40, 0.05) > 0.002


@pytest.mark.gpu
def test_shared_sinusoid_found(api):
    """The wandering shared sinusoid of test_emu_surrogate_pvalues.test_shared_sinusoid_found
    (period 32, n0 = 2048, periods 8 .. 128, M = 99): its largest cluster has p <= 0.05, and most of
    its points lie within one octave of period 32.  Observed with these seeds on an H100: 7 clusters,
    the largest of area 139.1 at p = 0.010 over rows [0, 16), 81 % of its points within the octave."""
    rs = np.random.RandomState(11)
    n = np.arange(2048)
    s = 2.5 * np.sin(2 * np.pi * n / 32.0 + np.cumsum(0.2 * rs.randn(2048)))
    x = red(rs, 2048, 0.5, 2) + s
    h = api.wct_resident(x[0], x[1], 1.0, dj=1 / 4, s0=8 / 1.033, J=16)
    sig = h.surrogate_significance(mc_count=99, seed=7)
    res = h.cluster_test(sig, mc_count=99, seed=8)
    assert res.pvalue[0] <= 0.05
    lab = h.cluster_labels()
    rows = (lab == 1).sum(axis=1)
    near = np.abs(np.log2(h.period / 32.0)) <= 1.0
    share = rows[near].sum() / rows.sum()
    print("  sinusoid: %d clusters, largest area %.1f at p = %.3f, rows %s, share near period 32 %.3f"
          % (res.area.size, res.area[0], res.pvalue[0], res.rows[0], share))
    assert share >= 0.75
    assert abs(np.log2(h.period[rows.argmax()] / 32.0)) <= 1.0

