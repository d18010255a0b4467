"""Monte-Carlo significance of the partial and multiple wavelet coherence on the GPU.

  * Histograms explained point by point (the pattern of test_gpu_coherence_parity.py::
    test_mc_histogram_explained): the histograms of `wct3_mc_seeded` and of `wct3_mc` fed the same
    triples are equal bit for bit, and equal the binned extended-precision RP2 / RM2 of the engine's
    own transforms of those triples (`ref_wct3`), except at points within nbins EPS kappa of a bin
    edge, kappa_P / kappa_M and EPS as in test_gpu_partial_coherence.py.
  * Config 4's Monte-Carlo geometry (N = 49152, padded to 65536, 145 scales, K = 14): a few
    triples in host-RNG mode against the oracle composition of test_emu_partial_significance.py.
  * The public seeded call: repeatable for one seed, different for another.
"""
import numpy as np
import pytest

from oracle import cwt_oracle as orc
import test_emu_overlap_save as osv
from test_gpu_partial_coherence import EPS, ref_wct3
from test_emu_partial_significance import oracle_hists

MORLET = 0
F64, F32 = 0, 1
NBINS = 1000


@pytest.fixture(scope="module")
def eng():
    e = osv.make_engine()
    yield e
    e.set_padding(True)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("K", [14, 36, 77])
def test_mc3_histogram_explained(eng, K, prec):
    """Per row and measure, sum |h - h_ref| <= 2 x (points within nbins EPS kappa of an edge)."""
    n0, S, maxscale, seed, triples = 600, 45, 37, 77, 2      # maxscale not a multiple of 32 or 64
    sj = 2.0 * 2 ** (np.arange(S) / 8.0)
    mask = ((np.arange(n0)[None, :] + 3 * np.arange(S)[:, None]) % 7 != 0).astype(np.uint8)
    hs = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(2)]
    eng.wct3_mc_seeded(seed, 0, triples, n0, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hs, precision=prec)
    noise = eng.mc_surrogates3(seed, 0, triples, n0)
    hh = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(2)]
    eng.wct3_mc(noise, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hh, precision=prec)
    assert np.array_equal(hs[0], hh[0]) and np.array_equal(hs[1], hh[1])
    href = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(2)]
    near = [np.zeros(S, dtype=np.int64) for _ in range(2)]
    npad = orc.next_pow2(n0)
    for t in range(triples):
        Ws = [eng.cwt(noise[t, r], 1.0, sj, MORLET, 6.0, precision=prec) for r in range(3)]
        rp, rm, kP, kM = ref_wct3(Ws, 1.0, sj, K, npad)
        for k, (R, kap) in enumerate(((rp, kP), (rm, kM))):
            R = np.asarray(R, dtype=np.float64)
            x = R * NBINS
            edge = np.abs(x - np.round(x)) <= NBINS * EPS[prec] * np.asarray(kap, dtype=np.float64)
            for i in range(maxscale):
                m = mask[i].astype(bool)
                b = np.clip(np.floor(x[i, m]), 0, NBINS - 1).astype(np.int64)
                href[k][i] += np.bincount(b, minlength=NBINS)
                near[k][i] += int(edge[i, m].sum())
    for k, label in ((0, "RP2"), (1, "RM2")):
        assert href[k][maxscale:].sum() == 0 and hs[k][maxscale:].sum() == 0
        diff = np.abs(hs[k] - href[k]).sum(axis=1)
        print("  MC3 K = %d %s %s: %d points binned, %d within EPS kappa of an edge, %d bin counts differ"
              % (K, "fp64" if prec == F64 else "fp32", label, href[k].sum(), near[k].sum(), diff.sum()))
        assert (diff <= 2 * near[k]).all(), {i: (diff[i], near[k][i]) for i in range(S) if diff[i] > 2 * near[k][i]}


@pytest.mark.gpu
def test_config4_monte_carlo_triples():
    """Config 4's Monte-Carlo geometry, 2 triples in host-RNG mode against the oracle composition:
    flips only at points within nbins 1e-10 / D of an edge; the levels of both measures."""
    import pycwt_b200 as pycwt
    import workloads as wl
    from pycwt_b200 import wavelet as wv
    c = wl.C4
    m = pycwt.Morlet(c["f0"])
    prob = wv._mc_problem(c["dt"], c["dj"], c["s0"], c["J"], m)
    assert prob["N"] == 49152 and prob["sj"].size == 145
    np.random.seed(4321)
    wv.rednoise(prob["N"], 0.3, 1)
    noise = [tuple(wv.rednoise(prob["N"], a, 1) for a in (0.3, 0.5, 0.2)) for _ in range(2)]
    h = wv._mc_histogram(prob, c["dt"], c["dj"], m, lambda i: noise[i], range(2), nser=3)
    hP, hM, nP, nM = oracle_hists(noise, prob, c["dt"], c["dj"], c["s0"], c["J"], orc.Morlet(c["f0"]))
    for k, (href, near, label) in enumerate(((hP, nP, "RP2"), (hM, nM, "RM2"))):
        assert h[k].sum() == href.sum() and href.sum() > 5e6
        diff = np.abs(h[k] - href).sum(axis=1)
        s, sr = wv._mc_levels(prob, h[k], 0.95), wv._mc_levels(prob, href, 0.95)
        ok = np.isfinite(sr)
        assert (np.isfinite(s) == ok).all()
        dl = float(np.abs(s[ok] - sr[ok]).max())
        print("  config 4 MC %s: %d samples, %d bin flips, %d near an edge, levels differ by %.1e"
              % (label, int(href.sum()), int(diff.sum()) // 2, int(near.sum()), dl))
        assert (diff <= 2 * near).all()
        assert dl < 1e-6


@pytest.mark.gpu
def test_public_seeded_call():
    import pycwt_b200 as pycwt
    args = (0.2, 0.4, 0.1, 1.0, 1 / 12, 2.0, 60)
    a = pycwt.wct3_significance(*args, mc_count=20, progress=False, seed=9)
    b = pycwt.wct3_significance(*args, mc_count=20, progress=False, seed=9)
    c = pycwt.wct3_significance(*args, mc_count=20, progress=False, seed=10)
    for k in (0, 1):
        ok = np.isfinite(a[k])
        assert ok.any() and ((a[k][ok] > 0) & (a[k][ok] < 1)).all()
        assert np.array_equal(a[k], b[k], equal_nan=True)
        assert not np.array_equal(a[k], c[k], equal_nan=True)
    ok = np.isfinite(a[0])
    print("  seeded levels: RP2 median %.3f, RM2 median %.3f" % (np.median(a[0][ok]), np.median(a[1][ok])))
