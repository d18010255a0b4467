"""Point-wise tests of the resident coherence against phase-randomised surrogates, on the GPU.

The checks of test_emu_surrogate_pvalues.py on the device: the counts against the recount of the
hook's surrogates through engine-level `wct` / `wct3`, bit for bit, on every row; the histograms,
levels and resident fields unchanged; accumulation, reset and the reductions.  Then config 4's data
sizes (n0 = 2^18, 145 scales, K = 14), fp64 and fp32, pairs and triples: the counts of 8 units
against the recount, the levels of a 50-unit `surrogate_test` against `surrogate_significance`, and
`fdr_threshold` against SciPy over all 38 M p-values.
"""
import numpy as np
import pytest

import test_emu_overlap_save as osv
import test_emu_surrogate_pvalues as P
import test_gpu_surrogate_significance as G

F64, F32 = P.F64, P.F32
NBINS = P.NBINS


@pytest.fixture(scope="module")
def eng():
    e = osv.make_engine()
    yield e
    e.set_padding(True)
    e.close()


@pytest.fixture
def api(eng, monkeypatch):
    import pycwt_b200
    from pycwt_b200 import _engine
    monkeypatch.setattr(_engine, "default_engine", lambda *a, **k: eng)
    return pycwt_b200


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser", [2, 3])
@pytest.mark.parametrize("n0,K", [(512, 6), (600, 36), (4096, 80)])
def test_counts_are_the_definition(eng, nser, n0, K, prec):
    P.check_counts_are_the_definition(eng, nser, n0, K, prec)


@pytest.mark.gpu
@pytest.mark.parametrize("nser", [2, 3])
def test_counts_unpadded(eng, nser):
    eng.set_padding(False)
    try:
        P.check_counts_are_the_definition(eng, nser, 4099, 6, F64, M=3)
    finally:
        eng.set_padding(True)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
def test_public_pair(api, eng, prec):
    P.test_public_pair(api, eng, prec)


@pytest.mark.gpu
@pytest.mark.parametrize("conditional", [True, False])
def test_public_triple(api, eng, conditional):
    P.test_public_triple(api, eng, conditional)


@pytest.mark.gpu
def test_red_noise_rate_and_sinusoid(api):
    P.test_red_noise_rate(api)
    P.test_shared_sinusoid_found(api)


def _stats(p):
    return "min p %.4f, %d NaN" % (np.nanmin(p), np.isnan(p).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser", [2, 3])
def test_config4_counts(eng, nser, prec):
    """Config 4's data sizes: the counts of 8 units against the recount, bit for bit, every row."""
    c, prob, data = G._config4()
    x = data[:nser]
    sj = prob["sj"]
    groups = (0, 1) if nser == 2 else (0, 1, 1)
    if nser == 2:
        serial = eng.wct_resident(x[0], x[1], c["dt"], c["dj"], sj, P.MORLET, c["f0"], 14, precision=prec)
    else:
        serial = eng.wct3_resident(*x, c["dt"], c["dj"], sj, P.MORLET, c["f0"], 14, precision=prec)
    before = P.observed(eng, nser)
    hs = [np.zeros((sj.size, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    eng.surrogate_counts(x, groups, 17, 0, 8, c["dt"], sj, P.MORLET, c["f0"], 14, prob["mask"], prob["maxscale"],
                         NBINS, *hs, serial=serial, precision=prec)
    after = P.observed(eng, nser)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before, after))
    assert all(np.array_equal(a, b) for a, b in zip(hs, G._run(eng, c, prob, x, groups, 17, 0, 8, prec)))
    obs = before[:nser - 1]
    k = P.recount(eng, x, groups, 17, 0, 8, sj, 14, prec, obs, dt=c["dt"], f0=c["f0"])
    for p, kk, o in zip(P.counted_p(eng, nser), k, obs):
        assert np.array_equal(p, P.p_of(kk, 8, o), equal_nan=True)
        print("  config 4, %d series, prec %d: %s" % (nser, prec, _stats(p)))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
@pytest.mark.parametrize("nser", [2, 3])
def test_config4_public(api, nser, prec):
    """A 50-unit surrogate_test: levels bit-identical to surrogate_significance, fields unchanged,
    fdr_threshold against SciPy over all 38 M p-values, pvalue_fraction against NumPy."""
    from scipy.stats import false_discovery_control
    import workloads as wl
    c = wl.C4
    y, x1 = wl.config4_signals()
    x2 = 0.6 * x1 + wl.chirp(c["n"], phase=2.1) + 0.5 * np.random.RandomState(2).randn(c["n"])
    kw = dict(dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=api.Morlet(c["f0"]), precision=prec)
    if nser == 2:
        h = api.wct_resident(y, x1, c["dt"], **kw)
        before = h.coherence().tobytes()
        lev = [h.surrogate_test(mc_count=50, seed=23)]
        ref = [h.surrogate_significance(mc_count=50, seed=23)]
        assert h.coherence().tobytes() == before
        measures = [{}]
    else:
        h = api.wct3_resident(y, x1, x2, c["dt"], **kw)
        before = h.partial().tobytes() + h.multiple().tobytes()
        lev = h.surrogate_test(mc_count=50, seed=23)
        ref = h.surrogate_significance(mc_count=50, seed=23)
        assert h.partial().tobytes() + h.multiple().tobytes() == before
        measures = [{'measure': 'partial'}, {'measure': 'multiple'}]
    assert h.shape == (145, 2 ** 18)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(lev, ref))
    cone = P.coi_mask(h)
    for kwm in measures:
        p = h.pvalues(**kwm)
        fin = np.isfinite(p)
        assert set(np.unique(p[fin])) <= {(1 + k) / 51 for k in range(51)}
        for method in ('bh', 'by'):
            for inside in (True, False):
                P.check_fdr(h.fdr_threshold(0.05, method, inside, **kwm), p[fin & (cone if inside else True)],
                            0.05, method)
        num, den = ((p <= 0.05) & fin & cone).sum(axis=1), (fin & cone).sum(axis=1)
        ref = np.where(den > 0, num / np.maximum(den, 1), np.nan)
        assert np.array_equal(h.pvalue_fraction(0.05, **kwm), ref, equal_nan=True)
        res = h.fdr_threshold(0.05, **kwm)
        print("  config 4 %s %s %s: BH %s, %s" % (nser, prec, kwm, res, _stats(p)))
    h.release()
