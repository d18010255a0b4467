"""Monte-Carlo significance against phase-randomised surrogates of the data
(`wct_surrogate_significance`, `wct3_surrogate_significance`, `Engine.wct_mc_phase`,
`Engine.mc_phase_surrogates`), checked on the host-emulation build of the kernels (tests/_emu).

  * the surrogates are what the definition says: spectrum moduli, mean, Nyquist bin, mean and
    variance of the data kept; series of one phase group keep their cross spectrum, others do not;
  * the phases are uniform, a pure function of (seed, unit, group, bin) restated in NumPy here
    (`philox4x32_10`, `phases`, `surrogate`), independent of how the units are split over calls;
  * the histograms are those of `wct_mc` / `wct3_mc` fed the hook's surrogates, bit for bit;
  * the public calls: repeatability, seeding, the rows and NaN pattern of the data's geometry,
    errors, no cache;
  * the levels against the white-noise null for white data, and the calibration of the
    conditional null where x1 and x2 share a driver;
  * world sizes 2 and 3 over gloo.
"""
import os
import socket
import sys

import numpy as np
import pytest

from conftest import ROOT

NBINS = 1000
F64, F32 = 0, 1
MORLET = 0


@pytest.fixture(scope="module")
def emu():
    from pycwt_b200 import build as _build, _engine
    lib = _build.build_emulation(os.path.join(ROOT, "tests", "_emu"))
    eng = _engine.Engine(0, lib_path=lib)
    assert "emulation" in eng.version()
    yield eng
    eng.set_padding(True)
    eng.close()


@pytest.fixture
def api(emu, monkeypatch):
    """The public API on the emulation build."""
    import pycwt_b200
    from pycwt_b200 import _engine
    monkeypatch.setattr(_engine, "default_engine", lambda *a, **k: emu)
    return pycwt_b200


# ---- NumPy restatement of the surrogate definition ---------------------------------------------
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, seed):
    """Philox4x32-10 (Salmon et al. 2011) of the counters (c0, c1, c2, c3), key = the two words of
    `seed`; arrays of uint64 holding 32-bit words."""
    c = [np.asarray(v, dtype=np.uint64) & _M32 for v in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return c


def phases(seed, unit, group, n):
    """U(seed, unit, group, k) for k = 0 .. n // 2: phi = 2 pi U.  Counter words
    (k, group, unit lo, 2^31 | (unit hi << 2) | 3); 53 bits of the first two output words."""
    k = np.arange(n // 2 + 1, dtype=np.uint64)
    o = philox4x32_10(k, group, unit & 0xFFFFFFFF, 0x80000000 | ((unit >> 32) << 2) | 3, seed)
    return ((o[0] >> np.uint64(5)).astype(float) * 67108864.0 + (o[1] >> np.uint64(6)).astype(float) + 0.5) \
        / 9007199254740992.0


def surrogate(x, seed, unit, group):
    n = x.size
    X = np.fft.fft(x)
    k = np.arange(1, (n + 1) // 2)                    # 1 <= k < n / 2
    Y = X.copy()
    Y[k] = X[k] * np.exp(2j * np.pi * phases(seed, unit, group, n)[k])
    Y[n - k] = np.conj(Y[k])
    return np.fft.ifft(Y).real


def red(rs, n, a, nser=1):
    """AR(1) series [nser, n] with coefficient a."""
    from scipy.signal import lfilter
    return lfilter([1.0], [1.0, -a], rs.randn(nser, n + 200), axis=1)[:, 200:]


LENGTHS = [256, 2048, 300, 3000, 301, 4097]      # 2^k (one- and two-kernel rows), even, odd


# ---- 1-3: the surrogates -------------------------------------------------------------------------
def check_surrogates_keep_the_spectrum(eng, n0, nser):
    rs = np.random.RandomState(n0 + nser)
    x = red(rs, n0, 0.7, nser) + 0.3
    groups = (0, 1, 1)[:nser]
    out = eng.mc_phase_surrogates(x, groups, 77, 5, 3)
    assert out.shape == (3, nser, n0) and out.dtype == np.float64 and np.isfinite(out).all()
    X = np.fft.fft(x, axis=1)
    top = np.abs(X).max()
    for u in range(3):
        Y = np.fft.fft(out[u], axis=1)
        assert np.abs(np.abs(Y) - np.abs(X)).max() <= 1e-12 * top
        assert np.abs(Y[:, 0] - X[:, 0]).max() <= 1e-12 * top
        if n0 % 2 == 0:
            assert np.abs(Y[:, n0 // 2] - X[:, n0 // 2]).max() <= 1e-12 * top
        assert np.abs(out[u].mean(axis=1) - x.mean(axis=1)).max() <= 1e-12
        assert np.abs(out[u].var(axis=1) / x.var(axis=1) - 1).max() <= 1e-12
        for r in range(nser):
            assert np.abs(out[u, r] - x[r]).max() > 0.1 * x[r].std()
            if u:
                assert np.abs(out[u, r] - out[u - 1, r]).max() > 0.1 * x[r].std()
            # the NumPy restatement of the keying and of the rotation
            ref = surrogate(x[r], 77, 5 + u, groups[r])
            assert np.abs(out[u, r] - ref).max() <= 1e-12 * np.abs(x).max()
    return x, out


@pytest.mark.parametrize("nser", [2, 3])
@pytest.mark.parametrize("n0", LENGTHS)
def test_surrogates_keep_the_spectrum(emu, n0, nser):
    check_surrogates_keep_the_spectrum(emu, n0, nser)


def circ_corr(a, b):
    """|mean e^{i (a - b)}| of two sets of angles."""
    return np.abs(np.exp(1j * (a - b)).mean())


def check_coupling(eng, n0):
    rs = np.random.RandomState(3)
    x = red(rs, n0, 0.5, 3)
    x[2] += 0.8 * x[1]
    X = np.fft.fft(x, axis=1)
    cross = X[1] * X[2].conj()
    k = np.arange(1, (n0 + 1) // 2)
    a = eng.mc_phase_surrogates(x, (0, 1, 1), 9, 0, 2)
    b = eng.mc_phase_surrogates(x, (0, 1, 2), 9, 0, 2)
    for u in range(2):
        A, B = np.fft.fft(a[u], axis=1), np.fft.fft(b[u], axis=1)
        assert np.abs(A[1] * A[2].conj() - cross).max() <= 1e-12 * np.abs(cross).max()
        assert np.abs(B[1] * B[2].conj() - cross)[k].max() > 0.1 * np.abs(cross).max()
        # series 0 and 1 are the same in both (phases belong to the group, not to the series' slot)
        assert np.array_equal(a[u, :2], b[u, :2])
        rot = np.angle(A[:, k] / X[:, k])              # the applied phases
        assert circ_corr(rot[1], rot[2]) > 1 - 1e-9
        assert circ_corr(rot[0], rot[1]) < 4 / np.sqrt(k.size)
        rotb = np.angle(B[:, k] / X[:, k])
        assert circ_corr(rotb[1], rotb[2]) < 4 / np.sqrt(k.size)
        assert circ_corr(rotb[0], rotb[2]) < 4 / np.sqrt(k.size)


@pytest.mark.parametrize("n0", [2048, 3000, 4097])
def test_coupling(emu, n0):
    check_coupling(emu, n0)


def check_phases_uniform_and_pure(eng, n0=32768, units=8):
    from scipy import stats
    rs = np.random.RandomState(5)
    x = rs.randn(2, n0)
    X = np.fft.fft(x, axis=1)
    k = np.arange(1, n0 // 2)
    out = eng.mc_phase_surrogates(x, (0, 1), 1234567890123, 0, units)
    U = []
    for u in range(units):
        Y = np.fft.fft(out[u], axis=1)
        got = np.mod(np.angle(Y[:, k] / X[:, k]) / (2 * np.pi), 1.0)
        for r in range(2):
            ref = phases(1234567890123, u, r, n0)[k]
            d = np.abs(got[r] - ref)
            assert np.minimum(d, 1 - d).max() < 1e-6      # angles recovered through two transforms
            U.append(ref)
    U = np.concatenate(U)
    assert U.size >= 1e5 and U.min() > 0 and U.max() < 1
    p = stats.kstest(U, "uniform").pvalue
    print("  KS test of %d phases against the uniform law: p = %.3f" % (U.size, p))
    assert p > 1e-3
    # the stream is keyed by the unit number, not by the call
    small = x[:, :3000]
    whole = eng.mc_phase_surrogates(small, (0, 1), 42, 0, 6)
    parts = np.concatenate([eng.mc_phase_surrogates(small, (0, 1), 42, 0, 2),
                            eng.mc_phase_surrogates(small, (0, 1), 42, 2, 4)])
    assert np.array_equal(whole, parts)
    assert not np.array_equal(eng.mc_phase_surrogates(small, (0, 1), 43, 0, 1)[0], whole[0])
    # units beyond 2^32 use the high counter word
    big = (1 << 40) + 3
    assert np.abs(eng.mc_phase_surrogates(small, (0, 1), 42, big, 1)[0, 1] - surrogate(small[1], 42, big, 1)).max() < 1e-11


def test_phases_uniform_and_pure(emu):
    check_phases_uniform_and_pure(emu)


# ---- 4: histograms ---------------------------------------------------------------------------------
def check_histogram_is_pipeline_of_surrogates(eng, nser, n0, K, prec, units=3, S=20, seed=31):
    rs = np.random.RandomState(n0 + K)
    x = red(rs, n0, 0.6, nser)
    x[-1] += 0.7 * x[-2]
    groups = (0, 1) if nser == 2 else (0, 1, 1)
    sj = 2.0 * 2 ** (np.arange(S) / 4.0)
    maxscale = S - 3
    mask = ((np.arange(n0)[None, :] + 3 * np.arange(S)[:, None]) % 7 != 0).astype(np.uint8)
    hs = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    eng.wct_mc_phase(x, groups, seed, 2, units, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hs, precision=prec)
    noise = eng.mc_phase_surrogates(x, groups, seed, 2, units)
    hh = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    if nser == 2:
        eng.wct_mc(noise, 1.0, 0.25, sj, MORLET, 6.0, K, mask, maxscale, NBINS, hh[0], precision=prec)
    else:
        eng.wct3_mc(noise, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hh, precision=prec)
    for a, b in zip(hs, hh):
        assert a[:maxscale].sum() == units * int(mask[:maxscale].sum()) or nser == 3
        assert a.sum() > 0 and a[maxscale:].sum() == 0
        assert np.array_equal(a, b)
    # accumulate-into, and a split over two calls
    eng.wct_mc_phase(x, groups, seed, 2, 1, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hh, precision=prec)
    eng.wct_mc_phase(x, groups, seed, 3, units - 1, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hh, precision=prec)
    for a, b in zip(hs, hh):
        assert np.array_equal(2 * a, b)
    return hs


@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser", [2, 3])
@pytest.mark.parametrize("n0,K", [(512, 6), (600, 36)])
def test_histogram_is_pipeline_of_surrogates(emu, nser, n0, K, prec):
    """Padded lengths (600 runs at 1024), 2^k, and a boxcar longer than 32."""
    check_histogram_is_pipeline_of_surrogates(emu, nser, n0, K, prec)


@pytest.mark.parametrize("nser", [2, 3])
def test_histogram_unpadded(emu, nser):
    """The un-padded transforms (fp64) of a length that is not 2^k."""
    emu.set_padding(False)
    try:
        check_histogram_is_pipeline_of_surrogates(emu, nser, 600, 6, F64, units=2)
    finally:
        emu.set_padding(True)


def test_one_histogram_of_three_series(emu):
    rs = np.random.RandomState(2)
    x = rs.randn(3, 256)
    sj = 2.0 * 2 ** (np.arange(8) / 2.0)
    mask = np.ones((8, 256), dtype=np.uint8)
    both = [np.zeros((8, NBINS), dtype=np.int64) for _ in range(2)]
    emu.wct_mc_phase(x, (0, 1, 1), 1, 0, 2, 1.0, sj, MORLET, 6.0, 3, mask, 6, NBINS, *both)
    for k in (0, 1):
        one = [None, None]
        one[k] = np.zeros((8, NBINS), dtype=np.int64)
        emu.wct_mc_phase(x, (0, 1, 1), 1, 0, 2, 1.0, sj, MORLET, 6.0, 3, mask, 6, NBINS, *one)
        assert np.array_equal(one[k], both[k])


# ---- 5: public calls ---------------------------------------------------------------------------------
def test_public_calls(api, emu, tmp_path, monkeypatch):
    from pycwt_b200 import wavelet as wv
    monkeypatch.setenv("HOME", str(tmp_path))
    monkeypatch.setenv("XDG_CACHE_HOME", str(tmp_path / "cache"))
    rs = np.random.RandomState(8)
    y = red(rs, 400, 0.5, 3)
    kw = dict(dj=1 / 4, mc_count=4)
    a = api.wct_surrogate_significance(y[0], y[1], 1.0, seed=5, **kw)
    b = api.wct_surrogate_significance(y[0], y[1], 1.0, seed=5, **kw)
    c = api.wct_surrogate_significance(y[0], y[1], 1.0, seed=6, **kw)
    assert np.array_equal(a, b, equal_nan=True) and not np.array_equal(a, c, equal_nan=True)
    np.random.seed(11)
    d = api.wct_surrogate_significance(y[0], y[1], 1.0, **kw)
    np.random.seed(11)
    e = api.wct_surrogate_significance(y[0], y[1], 1.0, **kw)
    np.random.seed(12)
    f = api.wct_surrogate_significance(y[0], y[1], 1.0, **kw)
    assert np.array_equal(d, e, equal_nan=True) and not np.array_equal(d, f, equal_nan=True)
    # rows and NaN pattern: _mc_levels on the geometry of the data, row for row with wct
    WCT, _, coi, freq, _ = api.wct(y[0], y[1], 1.0, dj=1 / 4, sig=False)
    assert a.shape == (WCT.shape[0],)
    m = api.Morlet(6)
    p = wv._wct_problem((y[0], y[1]), 1.0, 1 / 4, -1, -1, m, True, 'fp64')
    prob = wv._mc_problem(1.0, 1 / 4, p.s0, p.J, m, N=400)
    inside = (1 / freq)[:, None] <= coi[None, :]
    assert np.array_equal(prob['mask'].astype(bool), inside)
    # the reference's convention: the last row with points inside the cone keeps the template's NaN
    assert np.array_equal(np.isnan(a), np.arange(a.size) == prob['maxscale']) and np.isnan(prob['sig95'][prob['maxscale']])
    rows = np.arange(a.size) < prob['maxscale']
    assert ((a[rows] > 0) & (a[rows] < 1)).all() and (a[~rows & ~np.isnan(a)] == 0).all()
    hist = wv._surrogate_histogram(p, prob, (0, 1), 5, 0, 4, engine=emu)
    assert np.array_equal(wv._mc_levels(prob, hist[0], 0.95), a, equal_nan=True)
    assert hist[0][:prob['maxscale']].sum() == 4 * int(prob['mask'][:prob['maxscale']].sum())
    # three series, both nulls, fp32
    sp, sm = api.wct3_surrogate_significance(*y, 1.0, seed=5, **kw)
    sp2, sm2 = api.wct3_surrogate_significance(*y, 1.0, seed=5, conditional=False, **kw)
    sp3, sm3 = api.wct3_surrogate_significance(*y, 1.0, seed=5, precision='fp32', **kw)
    for s in (sp, sm, sp2, sm2, sp3, sm3):
        assert s.shape == a.shape and np.array_equal(np.isnan(s), np.isnan(a))
    assert not np.array_equal(sp, sp2, equal_nan=True)
    assert np.nanmax(np.abs(sp - sp3)) < 0.01 and np.nanmax(np.abs(sm - sm3)) < 0.01
    assert (sm[rows] >= sp[rows] - 0.05).all()
    # errors
    with pytest.raises(ValueError):
        api.wct_surrogate_significance(y[0], y[1][:-1], 1.0, **kw)
    bad = y[1].copy()
    bad[7] = np.nan
    with pytest.raises(ValueError):
        api.wct_surrogate_significance(y[0], bad, 1.0, **kw)
    with pytest.raises(ValueError):
        api.wct3_surrogate_significance(y[0], y[1], bad, 1.0, **kw)
    with pytest.raises(AttributeError):
        api.wct_surrogate_significance(y[0], y[1], 1.0, wavelet='paul', **kw)     # no generic smoothing
    with pytest.raises(ValueError):
        api.wct3_surrogate_significance(*y, 1.0, wavelet=api.Morlet(8), **kw)      # deltaj0 = -1
    with pytest.raises(ValueError):
        api.wct_surrogate_significance(y[0], y[1], 1.0, precision='fp16', **kw)
    assert not [f for _, _, fs in os.walk(str(tmp_path)) for f in fs]              # nothing cached


def test_engine_errors(emu):
    import ctypes
    P = ctypes.c_void_p
    x = np.random.RandomState(0).randn(3, 64)
    sj = np.array([2.0, 4.0, 8.0])
    mask = np.ones((3, 64), dtype=np.uint8)
    h = np.zeros((3, NBINS), dtype=np.int64)
    with pytest.raises(ValueError):
        emu.wct_mc_phase(x[:2], (0, 1), 1, 0, 1, 1.0, sj, MORLET, 6.0, 3, mask, 2, NBINS, h, h.copy())
    with pytest.raises(ValueError):
        emu.wct_mc_phase(x, (0, 1, 1), 1, 0, 1, 1.0, sj, MORLET, 6.0, 3, mask, 2, NBINS, None, None)
    with pytest.raises(ValueError):
        emu.mc_phase_surrogates(x, (0, 1), 1, 0, 1)
    with pytest.raises(ValueError):
        emu.mc_phase_surrogates(np.where(np.arange(64) == 3, np.inf, x), (0, 1, 1), 1, 0, 1)

    def hook(series, nser, groups, first=0, n0=64):
        g = np.asarray(groups, dtype=np.int32)
        out = np.empty((1, 3, 64))
        return emu.lib.cwtb_mc_phase_surrogates(emu.h, series.ctypes.data_as(P), nser, g.ctypes.data_as(P), 1, first,
                                                1, n0, out.ctypes.data_as(P))
    assert hook(x, 3, (0, 1, 1)) == 0
    assert hook(x, 4, (0, 1, 1, 1)) == -1 and hook(x, 1, (0,)) == -1
    assert hook(x, 3, (0, -1, 1)) == -1
    assert hook(x, 3, (0, 1, 1), n0=3) == -1
    assert hook(x, 3, (0, 1, 1), first=-1) == -1
    from pycwt_b200 import _engine
    g = np.array([0, 1, 1], dtype=np.int32)
    args = (sj.ctypes.data_as(P), 3, _engine.TABLE, 6.0, 3, mask.ctypes.data_as(P), 2, NBINS, h.ctypes.data_as(P), None)
    unsupported = emu.lib.cwtb_wct_mc_phase(emu.h, x.ctypes.data_as(P), 3, g.ctypes.data_as(P), 1, 0, 1, 64, 1.0, *args)
    assert unsupported not in (0, -1)
    assert hook(x, 3, (0, 1, 1), n0=(1 << 24) + 2) == unsupported      # beyond the Bluestein limit
    assert emu.lib.cwtb_wct_mc_phase(emu.h, None, 3, g.ctypes.data_as(P), 1, 0, 1, 64, 1.0, sj.ctypes.data_as(P), 3,
                                     MORLET, 6.0, 3, mask.ctypes.data_as(P), 2, NBINS, h.ctypes.data_as(P), None) == -1


# ---- 6: against the white null -------------------------------------------------------------------------
def test_white_data_agree_with_white_null(api):
    """Two independent white series: the surrogate null is white noise of the data's length, so on
    rows with many points inside the cone of influence the levels are those of
    `wct_significance(seed=)`, up to the Monte-Carlo scatter and to the one realisation's spectrum
    not being exactly flat.  Tolerance: the standard deviation of either level over 5 seeds with 40
    surrogates, measured here (printed; 0.02 on the emulation build, where the largest difference
    of the seed-averaged levels is 0.036), times 5, at least 0.03."""
    rs = np.random.RandomState(21)
    n0, dj = 512, 1 / 4
    y = rs.randn(2, n0)
    m = api.Morlet(6)
    s0 = 2 / m.flambda()
    J = int(np.round(np.log2(n0 / s0) / dj))
    sur = np.array([api.wct_surrogate_significance(y[0], y[1], 1.0, dj=dj, mc_count=40, seed=s) for s in range(5)])
    wht = np.array([api.wct_significance(0.0, 0.0, 1.0, dj, s0, J, mc_count=40, progress=False, cache=False, seed=s)
                    for s in range(5)])
    # the white null's surrogates have their own length and cone: compare rows well inside both
    rows = np.arange(2, 14)
    assert np.isfinite(sur[:, rows]).all() and np.isfinite(wht[:, rows]).all()
    spread = max(sur[:, rows].std(axis=0).max(), wht[:, rows].std(axis=0).max())
    d = np.abs(sur[:, rows].mean(axis=0) - wht[:, rows].mean(axis=0))
    tol = max(0.03, 5 * spread)
    print("  surrogate null:", np.round(sur[:, rows].mean(axis=0), 3))
    print("  white null    :", np.round(wht[:, rows].mean(axis=0), 3))
    print("  spread over seeds %.4f, largest difference %.4f, tolerance %.4f" % (spread, d.max(), tol))
    assert d.max() < tol


# ---- 7: calibration of the conditional null ----------------------------------------------------------------
def test_conditional_null_is_calibrated(api):
    """x1 and x2 share a strong band-limited driver, y is independent red noise: under this null
    hypothesis the fraction of in-cone points of the data's RP2 above the 95 % level is 0.05 on
    average.  Over 24 realisations (n0 = 512, 60 surrogates each) the fraction of one realisation has
    a standard deviation of 0.019 (the points of one RP2 field are strongly correlated), so the
    mean of 24 has a standard error of 0.004; observed on the emulation build: 0.0455.  The band
    asserted for the conditional null, [0.03, 0.07], is 0.05 +- 5 standard errors.  The fraction
    for the white-noise level of `wct3_significance` is printed beside it (0.036 here); no
    direction is asserted for it."""
    n0, dj, level, reals = 512, 1 / 4, 0.95, 24
    m = api.Morlet(6)
    s0 = 2 / m.flambda()
    J = int(np.round(np.log2(n0 / s0) / dj))
    t = np.arange(n0)
    white = api.wct3_significance(0.0, 0.0, 0.0, 1.0, dj, s0, J, significance_level=level, mc_count=60,
                                  progress=False, seed=1)[0]
    frac_c, frac_w = [], []
    for r in range(reals):
        rs = np.random.RandomState(100 + r)
        drv = red(rs, n0, 0.9)[0] * np.sin(2 * np.pi * t / 24.0 + rs.uniform(0, 6.28))   # band around period 24
        drv *= 3.0 / drv.std()
        x1 = drv + rs.randn(n0)
        x2 = np.roll(drv, 3) + rs.randn(n0)
        y = red(rs, n0, 0.7)[0]
        RP2, coi, freq = api.partial_wct(y, x1, x2, 1.0, dj=dj)
        sig = api.wct3_surrogate_significance(y, x1, x2, 1.0, dj=dj, significance_level=level, mc_count=60,
                                              seed=r)[0]
        inside = ((1 / freq)[:, None] <= coi[None, :]) & np.isfinite(sig)[:, None] & (sig > 0)[:, None]
        frac_c.append((RP2 > sig[:, None])[inside].mean())
        ok = inside & np.isfinite(white)[:, None] & (white > 0)[:, None]
        frac_w.append((RP2 > white[:, None])[ok].mean())
    fc, fw = float(np.mean(frac_c)), float(np.mean(frac_w))
    print("  fraction of in-cone RP2 above the 95 %% level over %d realisations: conditional null %.4f "
          "(std of one %.4f), white-noise null %.4f (std of one %.4f); nominal %.2f"
          % (reals, fc, np.std(frac_c), fw, np.std(frac_w), 1 - level))
    assert 0.03 <= fc <= 0.07


# ---- 8: multi-rank ---------------------------------------------------------------------------------------------
def _shard_data():
    rs = np.random.RandomState(17)
    y = red(rs, 300, 0.6, 3)
    y[2] += y[1]
    return y


SHARD_KW = dict(dj=0.5, mc_count=5, seed=42)


def _shard_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    from pycwt_b200 import distributed as D, _engine
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        eng = _engine.Engine(0, lib_path=os.path.join(ROOT, "tests", "_emu", "libcwtb200_emu.so"))
        y = _shard_data()
        comm = D.TorchComm(dist)
        s2 = D.wct_surrogate_significance_sharded(y[0], y[1], 1.0, engine=eng, comm=comm, **SHARD_KW)
        s3 = D.wct3_surrogate_significance_sharded(*y, 1.0, engine=eng, comm=comm, **SHARD_KW)
        q.put((rank, [s2.tolist()] + [s.tolist() for s in s3]))
        eng.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_gloo(world):
    """Every rank of a world of 2 or 3 gets the levels of one process running every unit."""
    pytest.importorskip("torch")
    import torch.multiprocessing as mp
    from pycwt_b200 import build as _build, _engine, distributed as D
    eng = _engine.Engine(0, lib_path=_build.build_emulation(os.path.join(ROOT, "tests", "_emu")))
    y = _shard_data()
    single = [D.wct_surrogate_significance_sharded(y[0], y[1], 1.0, engine=eng, **SHARD_KW)]
    single += list(D.wct3_surrogate_significance_sharded(*y, 1.0, engine=eng, **SHARD_KW))
    eng.close()
    for s in single:
        assert np.isnan(s).any() and np.isfinite(s).any()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r in range(world):
        for a, b in zip(got[r], single):
            assert np.array_equal(np.asarray(a), b, equal_nan=True)
