"""Monte-Carlo significance against phase-randomised surrogates of the data, on the GPU.

The checks of test_emu_surrogate_significance.py on the device: the surrogates against the NumPy
restatement of their definition (also at 2^18 samples and at lengths near it that run through
Bluestein's algorithm), the coupling of phase groups, the uniformity and purity of the phase stream,
and the histograms of `wct_mc_phase` against `wct_mc` / `wct3_mc` fed the hook's surrogates, bit
for bit.  At config 4's data sizes (n0 = 2^18, 145 scales, K = 14) the histograms of the partial and
multiple coherence are compared with the oracle composition of test_emu_partial_significance.py fed
the hook's surrogates: flips only at points within nbins 1e-10 / D of a bin edge.  Then the public
seeded calls.
"""
import numpy as np
import pytest

from oracle import cwt_oracle as orc
import test_emu_overlap_save as osv
import test_emu_surrogate_significance as T
from test_emu_partial_significance import oracle_hists

F64, F32 = T.F64, T.F32
NBINS = T.NBINS


@pytest.fixture(scope="module")
def eng():
    e = osv.make_engine()
    yield e
    e.set_padding(True)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("nser", [2, 3])
@pytest.mark.parametrize("n0", T.LENGTHS + [2 ** 18, 250000, 250001, 2 ** 21])
def test_surrogates_keep_the_spectrum(eng, n0, nser):
    T.check_surrogates_keep_the_spectrum(eng, n0, nser)


@pytest.mark.gpu
@pytest.mark.parametrize("n0", [2048, 3000, 4097, 2 ** 18, 250001])
def test_coupling(eng, n0):
    T.check_coupling(eng, n0)


@pytest.mark.gpu
def test_phases_uniform_and_pure(eng):
    T.check_phases_uniform_and_pure(eng)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser", [2, 3])
@pytest.mark.parametrize("n0,K,S", [(512, 6, 20), (600, 36, 20), (20000, 14, 40), (65536, 77, 45)])
def test_histogram_is_pipeline_of_surrogates(eng, nser, n0, K, S, prec):
    T.check_histogram_is_pipeline_of_surrogates(eng, nser, n0, K, prec, S=S)


@pytest.mark.gpu
@pytest.mark.parametrize("nser", [2, 3])
def test_histogram_unpadded(eng, nser):
    eng.set_padding(False)
    try:
        T.check_histogram_is_pipeline_of_surrogates(eng, nser, 6000, 14, F64, units=2, S=40)
    finally:
        eng.set_padding(True)


def _config4():
    import pycwt_b200 as pycwt
    import workloads as wl
    from pycwt_b200 import wavelet as wv
    c = wl.C4
    m = pycwt.Morlet(c["f0"])
    prob = wv._mc_problem(c["dt"], c["dj"], c["s0"], c["J"], m, N=c["n"])
    assert prob["N"] == 2 ** 18 and prob["sj"].size == 145 and wv._boxcar_len(m, c["dj"]) == 14
    y, x1 = wl.config4_signals()
    x2 = 0.6 * x1 + wl.chirp(c["n"], phase=2.1) + 0.5 * np.random.RandomState(2).randn(c["n"])
    data = np.stack([(v - v.mean()) / v.std() for v in (y, x1, x2)])
    return c, prob, data


def _run(eng, c, prob, data, groups, seed, first, units, prec):
    hs = [np.zeros((prob["sj"].size, NBINS), dtype=np.int64) for _ in range(data.shape[0] - 1)]
    eng.wct_mc_phase(data, groups, seed, first, units, c["dt"], prob["sj"], T.MORLET, c["f0"], 14, prob["mask"],
                     prob["maxscale"], NBINS, *hs, precision=prec)
    return hs


@pytest.mark.gpu
def test_config4_sizes_against_oracle(eng):
    """Config 4's data sizes.  Three series, fp64: one unit of the conditional null against the
    oracle composition of the hook's surrogates.  Both precisions and both numbers of series: equal
    to the host-fed Monte-Carlo calls bit for bit (5 units); fp32 levels within 1e-2 of fp64."""
    from pycwt_b200 import wavelet as wv
    c, prob, data = _config4()
    pts = int(prob["mask"][:prob["maxscale"]].sum())
    levels = {}
    for nser, groups in ((2, (0, 1)), (3, (0, 1, 1))):
        x = data[:nser]
        noise = eng.mc_phase_surrogates(x, groups, 4321, 10, 5)
        for prec in (F64, F32):
            hs = _run(eng, c, prob, x, groups, 4321, 10, 5, prec)
            hh = [np.zeros_like(h) for h in hs]
            if nser == 2:
                eng.wct_mc(noise, c["dt"], c["dj"], prob["sj"], T.MORLET, c["f0"], 14, prob["mask"], prob["maxscale"],
                           NBINS, hh[0], precision=prec)
                assert hs[0].sum() == 5 * pts
            else:
                eng.wct3_mc(noise, c["dt"], prob["sj"], T.MORLET, c["f0"], 14, prob["mask"], prob["maxscale"], NBINS,
                            *hh, precision=prec)
            for a, b in zip(hs, hh):
                assert a.sum() > 0 and np.array_equal(a, b)
            levels[nser, prec] = [wv._mc_levels(prob, h, 0.95) for h in hs]
        for a, b in zip(levels[nser, F64], levels[nser, F32]):
            ok = np.isfinite(a)
            assert (np.isfinite(b) == ok).all()
            print("  config 4 sizes, %d series: fp32 levels differ from fp64 by %.1e" % (nser, np.abs(a - b)[ok].max()))
            assert np.abs(a - b)[ok].max() < 1e-2
    # the oracle composition of one unit's surrogates (y, x1, x2), fp64
    noise = eng.mc_phase_surrogates(data, (0, 1, 1), 4321, 10, 1)
    hs = _run(eng, c, prob, data, (0, 1, 1), 4321, 10, 1, F64)
    hP, hM, nP, nM = oracle_hists(noise, prob, c["dt"], c["dj"], c["s0"], c["J"], orc.Morlet(c["f0"]))
    for h, href, near, label in ((hs[0], hP, nP, "RP2"), (hs[1], hM, nM, "RM2")):
        assert h.sum() == href.sum() and href.sum() > 5e6
        diff = np.abs(h - href).sum(axis=1)
        print("  config 4 sizes %s: %d samples, %d bin flips, %d near an edge"
              % (label, int(href.sum()), int(diff.sum()) // 2, int(near.sum())))
        assert (diff <= 2 * near).all()


@pytest.mark.gpu
def test_public_seeded_calls():
    import pycwt_b200 as pycwt
    rs = np.random.RandomState(4)
    y = T.red(rs, 5000, 0.6, 3)
    y[2] += y[1]
    kw = dict(dj=1 / 12, mc_count=20)
    a = pycwt.wct3_surrogate_significance(*y, 1.0, seed=9, **kw)
    b = pycwt.wct3_surrogate_significance(*y, 1.0, seed=9, **kw)
    c = pycwt.wct3_surrogate_significance(*y, 1.0, seed=10, **kw)
    d = pycwt.wct3_surrogate_significance(*y, 1.0, seed=9, precision="fp32", **kw)
    u = pycwt.wct3_surrogate_significance(*y, 1.0, seed=9, conditional=False, **kw)
    RP2 = pycwt.partial_wct(*y, 1.0, dj=1 / 12)[0]
    for k in (0, 1):
        ok = np.isfinite(a[k]) & (a[k] > 0)
        assert a[k].shape == (RP2.shape[0],) and ok.any() and (a[k][ok] < 1).all()
        assert np.array_equal(a[k], b[k], equal_nan=True)
        assert not np.array_equal(a[k], c[k], equal_nan=True)
        assert np.abs(a[k] - d[k])[ok].max() < 1e-2
    s2 = pycwt.wct_surrogate_significance(y[0], y[1], 1.0, seed=9, **kw)
    assert np.array_equal(s2, pycwt.wct_surrogate_significance(y[0], y[1], 1.0, seed=9, **kw), equal_nan=True)
    ok = np.isfinite(a[0]) & (a[0] > 0)
    print("  levels (median over rows): coherence %.3f, RP2 conditional %.3f / unconditional %.3f, "
          "RM2 conditional %.3f / unconditional %.3f"
          % (np.median(s2[ok]), np.median(a[0][ok]), np.median(u[0][ok]), np.median(a[1][ok]), np.median(u[1][ok])))
