"""Full-size parity of every BASELINE.json configuration on the GPU box: the engine's result on the
bench's own inputs (workloads.py) against the CPU oracle, EVERY row, at the tolerances of the
north star (fp64: 1e-10 of max|W_ref|; fp32 engine: 1e-5).  The oracle runs in chunks of scales so
that its multi-GiB temporaries stay bounded; each test takes tens of seconds of host time."""
import numpy as np
import pytest

import workloads as wl
from conftest import relerr
from oracle import cwt_oracle as orc

pytestmark = pytest.mark.gpu

TOL64 = 1e-10
TOL32 = 1e-5


@pytest.fixture(scope="module")
def pycwt():
    import pycwt_b200
    return pycwt_b200


def _oracle_rows(x, dt, mother, sj, rows):
    fr = 1.0 / (mother.flambda() * sj[rows])
    return orc.cwt(x, dt, wavelet=mother, freqs=fr, workers=-1)[0]


# Per-row bounds of config 2, by the row's class in last_plan (error / max|W_ref[j]|): expansion rows at
# the expansion tolerance, exact and overlap-save rows at 1e-14 (DESIGN 6).  Measured on H100 against the
# fp64 oracle: 5.2e-14, 6.4e-15 and 2.7e-15.  The exact rows 0..19 (s = 2 .. 4.8) lie above the chirp's
# band, where the oracle's own rounding is of the order of the bound; they are also checked against the
# longdouble reference of test_gpu_row_parity.py (measured: 6.0e-15).
C2_OUT_OF_BAND = 20
C2_BOUND = {"expansion": 5e-13, "exact": 1e-14, "overlap-save": 1e-14}


def _row_class(p):
    return "expansion" if p < -2 else ("overlap-save" if p == -2 else "exact")


def _check_config2_rows(x, c, sj, plan, err, W):
    from test_gpu_row_parity import ref_rows, row_err
    worst = {}
    for j, p in enumerate(plan):
        k = _row_class(p)
        worst[k] = max(worst.get(k, 0.0), float(err[j]))
    print("config 2 per-row error by class: %s" % ", ".join("%s %.2e" % kv for kv in sorted(worst.items())))
    bad = [(j, _row_class(plan[j]), float(err[j])) for j in range(len(plan))
           if err[j] > C2_BOUND[_row_class(plan[j])]]
    assert not bad, bad
    rows = np.arange(C2_OUT_OF_BAND)
    e = row_err(W[rows], ref_rows(x, c["dt"], sj[rows], 0, c["f0"]))
    print("config 2 rows 0..%d (above the chirp's band): against the longdouble reference %.2e, against "
          "the fp64 oracle %.2e" % (C2_OUT_OF_BAND - 1, e.max(), err[rows].max()))
    assert all(_row_class(plan[j]) == "exact" for j in rows), plan[:C2_OUT_OF_BAND]
    assert (e < C2_BOUND["exact"]).all(), e


def test_config2_every_row(pycwt):
    """Config 2 (the bench's input: chirp N = 2^20, s0 = 2, dj = 1/16, 256 scales, Morlet(6), fp64):
    all 256 rows of W and of |W|^2 against the oracle."""
    c = wl.C2
    x = wl.config2_signal()
    W, sj, freqs, coi, fft, fftfreqs = pycwt.cwt(x, c["dt"], c["dj"], c["s0"], c["J"], pycwt.Morlet(c["f0"]))
    assert W.shape == (c["J"] + 1, c["n"]) and W.dtype == np.complex128
    np.testing.assert_array_equal(sj, wl.config2_scales())
    plan = pycwt.default_engine().last_plan(len(sj))
    assert min(plan) < 0 < max(plan)        # both the exact and the expansion path are in play
    m = orc.Morlet(c["f0"])
    # pass 1: the global normalisation max|W_ref|, from the oracle itself
    wmax, pmax, worst, worst_p = 0.0, 0.0, 0.0, 0.0
    chunks = [np.arange(r0, min(r0 + 32, len(sj))) for r0 in range(0, len(sj), 32)]
    diffs = []
    for rows in chunks:
        Wr = _oracle_rows(x, c["dt"], m, sj, rows)
        wmax = max(wmax, float(np.abs(Wr).max()))
        pr = np.abs(Wr) ** 2
        pmax = max(pmax, float(pr.max()))
        d = np.abs(W[rows] - Wr).max(axis=1)
        dp = np.abs(np.abs(W[rows]) ** 2 - pr).max(axis=1)
        diffs.append((rows, d, dp, np.abs(Wr).max(axis=1)))
    for rows, d, dp, _ in diffs:
        worst = max(worst, float(d.max()) / wmax)
        worst_p = max(worst_p, float(dp.max()) / pmax)
    print("config 2: max|dW|/max|W| = %.2e, power %.2e" % (worst, worst_p))
    assert worst < TOL64 and worst_p < TOL64
    # per row, against the row's own maximum, with the bound of the row's class
    err = np.concatenate([d / rmax for rows, d, dp, rmax in diffs])
    _check_config2_rows(x, c, sj, plan, err, W)
    ref_fft = np.fft.fft(x)[1:c["n"] // 2] / np.sqrt(c["n"])
    assert relerr(fft, ref_fft) < 1e-12


def test_config2_widest_band_mode(pycwt):
    """band_eps = 0 (every representable bin kept) with the expansion off at N = 2^20: the dense
    kernel's Gaussian recurrence must not start from subnormal values (rows 41, 54, 57 were off by
    2e-10 of max|W| before the re-seeding rule of kernels.cuh: PassABody, dense Morlet)."""
    from pycwt_b200 import _engine
    c = wl.C2
    x = wl.config2_signal()
    sj = wl.config2_scales()
    rows = np.array([0, 23, 39, 41, 51, 54, 57, 71, 100])
    eng = pycwt.default_engine()
    eng.set_band_eps(0.0)
    eng.set_expand_eps(0.0, 0.0)
    try:
        W = eng.cwt(x, c["dt"], sj[rows], _engine.MORLET, c["f0"])
    finally:
        eng.set_band_eps(1e-16)
        eng.set_expand_eps()
    Wr = _oracle_rows(x, c["dt"], orc.Morlet(c["f0"]), sj, rows)
    err = np.abs(W - Wr).max(axis=1) / np.abs(Wr).max()
    print("config 2, band_eps = 0: worst row error %.2e" % err.max())
    assert (err < 1e-12).all(), err


@pytest.mark.parametrize("family", ["paul", "dog"])
def test_config3_every_row_fp32(pycwt, monkeypatch, family):
    """Config 3: Paul(4) / DOG(2), N = 2^18, 128 scales, float32 chirp, fp32 engine; every row against
    the oracle at the contract's 1e-5 of max|W|, and every row against its own scale sigma_j (the row's
    maximum, or its rms response to white noise of the signal's energy where that is larger: rows
    outside the chirp's band) with the per-row bounds of test_gpu_fp32_row_parity.py."""
    from test_gpu_fp32_row_parity import EXACT32, EXPAND32, ref32, sigma_err
    monkeypatch.setenv("CWTB_PRECISION", "fp32")
    c = wl.C3
    p = c[family]
    x = wl.config3_signal()
    mother = pycwt.Paul(p["m"]) if family == "paul" else pycwt.DOG(p["m"])
    ref = orc.Paul(p["m"]) if family == "paul" else orc.DOG(p["m"])
    W, sj, *_ = pycwt.cwt(x, c["dt"], p["dj"], p["s0"], p["J"], mother)
    assert W.shape == (p["J"] + 1, c["n"])      # no NaN rows at these scales
    Wr = orc.cwt(x.astype(np.float64), c["dt"], p["dj"], p["s0"], p["J"], ref, workers=-1)[0]
    err = relerr(W, Wr)
    rows = np.abs(W - Wr).max(axis=1) / np.abs(Wr).max()
    print("config 3 %s: max|dW|/max|W| = %.2e (worst row %d)" % (family, err, int(rows.argmax())))
    assert err < TOL32 and (rows < TOL32).all()
    assert relerr(np.abs(W) ** 2, np.abs(Wr) ** 2) < TOL32
    plan = np.array(pycwt.default_engine().last_plan(len(sj)))
    fam = 1 if family == "paul" else 2
    e = sigma_err(W, *ref32(x, c["dt"], sj, fam, float(p["m"])))
    bound = np.where(plan < 0, EXPAND32, EXACT32)
    print("config 3 %s per row / sigma_j: expansion rows %.2e, exact rows %.2e"
          % (family, e[plan < 0].max(initial=0), e[plan >= 0].max(initial=0)))
    assert (e <= bound).all(), [(j, int(plan[j]), float(e[j])) for j in np.flatnonzero(e > bound)]


def test_config4_xwt_wct_every_row(pycwt):
    """Config 4 deterministic part: xwt and wct(sig=False) of the two N = 2^18 series, all 145 scales."""
    c = wl.C4
    y1, y2 = wl.config4_signals()
    m, mo = pycwt.Morlet(c["f0"]), orc.Morlet(c["f0"])
    W12, coi, freq, signif = pycwt.xwt(y1, y2, c["dt"], c["dj"], c["s0"], c["J"], wavelet=m)
    o = orc.xwt(y1, y2, c["dt"], c["dj"], c["s0"], c["J"], wavelet=mo)
    assert W12.shape == (c["J"] + 1, c["n"])
    e_x = relerr(W12, o[0])
    assert e_x < TOL64
    np.testing.assert_allclose(signif, o[3], rtol=1e-12)
    WCT, aWCT, coi, freq, sig = pycwt.wct(y1, y2, c["dt"], c["dj"], c["s0"], c["J"], sig=False, wavelet=m)
    ow = orc.wct(y1, y2, c["dt"], c["dj"], c["s0"], c["J"], sig=False, wavelet=mo)
    e_w = relerr(WCT, ow[0])
    # the phase angle of the unsmoothed cross spectrum: compare on the circle, where |W12| is not tiny
    big = np.abs(o[0]) > 1e-6 * np.abs(o[0]).max()
    dphi = np.angle(np.exp(1j * (aWCT - ow[1])))
    e_a = float(np.abs(dphi[big]).max())
    print("config 4: xwt %.2e, wct %.2e, angle %.2e" % (e_x, e_w, e_a))
    assert e_w < TOL64 and e_a < 1e-8


def test_config4_monte_carlo_real_geometry(pycwt):
    """Config 4 Monte-Carlo part at the real geometry (s0 = 2, dj = 1/12, J = 144: surrogates of
    49152 samples, 145 scales), 8 surrogate pairs, seeded: the GPU histograms equal the oracle's
    (a coherence value within 1e-13 of a bin edge may flip: at most a handful of 5e7 samples)."""
    c = wl.C4
    from pycwt_b200 import wavelet as wv
    m = pycwt.Morlet(c["f0"])
    prob = wv._mc_problem(c["dt"], c["dj"], c["s0"], c["J"], m)
    assert prob["N"] == 49152 and prob["sj"].size == 145
    np.random.seed(1234)
    sig_o, hist_o = orc.wct_significance(0.3, 0.5, c["dt"], c["dj"], c["s0"], c["J"], wavelet=orc.Morlet(c["f0"]),
                                         mc_count=8, rng=np.random, return_hist=True)
    np.random.seed(1234)
    wv.rednoise(prob["N"], 0.3, 1)                  # the reference's set-up draw
    hist = wv._mc_histogram(prob, c["dt"], c["dj"], m,
                            lambda i: (wv.rednoise(prob["N"], 0.3, 1), wv.rednoise(prob["N"], 0.5, 1)), range(8))
    flips = int(np.abs(hist - hist_o).sum())
    assert hist.sum() == hist_o.sum() and hist.sum() > 1e7
    assert flips <= 8, flips
    sig = wv._mc_levels(prob, hist, 0.95)
    ok = ~np.isnan(sig_o)
    assert (np.isnan(sig) == np.isnan(sig_o)).all()
    assert np.abs(sig[ok] - sig_o[ok]).max() < 1e-6
    print("config 4 MC: %d samples, %d bin flips" % (int(hist.sum()), flips))


def test_config5_batch_channels(pycwt):
    """Config 5 (per-GPU share: 1024 channels of N = 2^16, 128 scales, fp32): the global spectra
    of 32 random channels of the 1024-channel batch, and every coefficient of 8 channels of a
    64-channel batch, against per-channel oracle calls."""
    c = wl.C5
    eng = pycwt.default_engine()
    sj = wl.geometric_scales(c["s0"], c["dj"], c["J"])
    mo = orc.Morlet(c["f0"])
    fr = 1.0 / (mo.flambda() * sj)
    X = wl.config5_channels(0, c["per_gpu"])
    from pycwt_b200 import _engine
    power, _ = eng.cwt_batch(X, c["dt"], sj, _engine.MORLET, c["f0"], _engine.F32, want_power=True)
    assert power.shape == (c["per_gpu"], sj.size)
    pick = np.random.RandomState(7).choice(c["per_gpu"], 32, replace=False)
    worst = 0.0
    for ch in pick:
        Wr = orc.cwt(X[ch].astype(np.float64), c["dt"], wavelet=mo, freqs=fr, workers=-1)[0]
        pr = (np.abs(Wr) ** 2).mean(axis=1)
        worst = max(worst, float(np.abs(power[ch] - pr).max() / pr.max()))
    print("config 5: spectra of 32 of 1024 channels, worst %.2e" % worst)
    assert worst < TOL32
    _, W = eng.cwt_batch(X[:64], c["dt"], sj, _engine.MORLET, c["f0"], _engine.F32, want_power=False, want_w=True)
    assert W.shape == (64, sj.size, c["n"]) and W.dtype == np.complex64
    for ch in np.random.RandomState(8).choice(64, 8, replace=False):
        Wr = orc.cwt(X[ch].astype(np.float64), c["dt"], wavelet=mo, freqs=fr, workers=-1)[0]
        assert relerr(W[ch], Wr) < TOL32
