"""Resident cross-wavelet transform (`xwt_resident`) and the complex-field additions of
`ResidentTransform` (`window`, `global_power(signif=)`, `significant_fraction`), checked on the
host-emulation build of the kernels (tests/_emu, the fixture pattern of test_emu_kernels.py).

  * the fetch is bit-identical to `xwt(...)[0]` in both precisions, `signif`, `coi` and `freq`
    equal `xwt`'s;
  * `window` equals numpy slicing of the fetch;
  * every reduction agrees with numpy on the fetch, with the points selected as
    re^2 + im^2 > signif^2: counts exact, means within 1e-12 relative, circular sums within
    1e-12 of the count, `scale_avg` within 1e-12 of the numpy sum;
  * the handle survives cwt / xwt / wct / wct_resident / significance / cwt_resident and dies with
    the next xwt_resident or release().
"""
import os

import numpy as np
import pytest

from conftest import ROOT, golden_cwt_kwargs, load_golden
from test_emu_coherence_fp32 import chirp_pair
from test_emu_coherence_resident import WINDOWS, check_mean_phase

TOL = 1e-12

EXTRA_WINDOWS = [
    (slice(0, 0), slice(None)),
    (slice(None), slice(7, 7)),
    (slice(4, 5), slice(None)),
    (slice(None), slice(9, 10)),
    (slice(-1, None), slice(-1, None)),
    (slice(None, None, 3), slice(None, None, 3)),
]


@pytest.fixture(scope="module")
def emu():
    from pycwt_b200 import build as _build, _engine
    lib = _build.build_emulation(os.path.join(ROOT, "tests", "_emu"))
    eng = _engine.Engine(0, lib_path=lib)
    assert "emulation" in eng.version()
    yield eng
    eng.close()


@pytest.fixture
def api(emu, monkeypatch):
    """The public API on the emulation build."""
    import pycwt_b200
    from pycwt_b200 import _engine
    monkeypatch.setattr(_engine, "default_engine", lambda *a, **k: emu)
    return pycwt_b200


def ao_baltic():
    g = load_golden("ao_baltic_xwt_wct")
    return g["y1"], g["y2"], float(g["dt"]), dict(dj=1 / 12)


def chirp():
    a, b = chirp_pair(2 ** 13)
    return a, b, 1.0, dict(dj=1 / 4, s0=2.0, J=44)


CASES = {"ao_baltic": ao_baltic, "chirp8k": chirp}


# ---- numpy on the fetched field ---------------------------------------------------------------
def _close(a, b, tol=TOL):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    assert a.shape == b.shape
    assert (np.isnan(a) == np.isnan(b)).all(), (a, b)
    ok = ~np.isnan(b)
    assert (np.abs(a[ok] - b[ok]) <= tol * np.maximum(np.abs(b[ok]), 1e-300)).all(), \
        np.abs(a[ok] - b[ok]).max()


def _norm2(F):
    """re^2 + im^2, each operation rounded (what the engine compares against a threshold)."""
    return F.real * F.real + F.imag * F.imag


def _points(h, F, inside_coi, thr2):
    """[S, n0] mask of the points a reduction uses; thr2: threshold on re^2 + im^2."""
    S, n0 = F.shape
    m = np.ones((S, n0), dtype=bool)
    if inside_coi:
        m &= h.period[:, None] <= h.coi[None, :]
    if thr2 is not None:
        with np.errstate(invalid="ignore"):
            m &= _norm2(F) > np.asarray(thr2)[:, None]
    return m


def _row_sum(m, X):
    return np.einsum('ij,ij->i', m.astype(float), X)


def _mean(m, X):
    cnt = m.sum(axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(cnt > 0, _row_sum(m, X) / cnt, np.nan)


def _unit(F):
    """cos and sin of the phase as re / |F|, im / |F|; phase 0 for a zero coefficient."""
    m = np.sqrt(_norm2(F))
    safe = np.where(m > 0, m, 1.0)
    return np.where(m > 0, F.real / safe, 1.0), np.where(m > 0, F.imag / safe, 0.0)


def signif_with_gaps(F):
    """A |F| threshold per scale with NaN entries and rows that no point passes."""
    S = F.shape[0]
    thr = np.quantile(np.abs(F), 0.6, axis=1)
    thr[::5] = np.nan
    thr[1] = 2 * np.abs(F).max()
    thr[S - 2] = np.inf
    thr[3] = 0.0
    return thr


def check_cross_reductions(h, W12, signif):
    """Every reduction of a ResidentCrossWavelet against numpy on the fetched W12."""
    S, n0 = W12.shape
    per = h.period
    absF = np.sqrt(_norm2(W12))
    thr2 = np.asarray(signif) ** 2
    lo, hi = h.coi_ranges()
    cols = np.arange(n0)
    assert np.array_equal((cols[None, :] >= lo[:, None]) & (cols[None, :] < hi[:, None]),
                          _points(h, W12, True, None))
    for inside in (False, True):
        for sg, t2 in ((None, None), (signif, thr2)):
            _close(h.global_power(inside_coi=inside, signif=sg), _mean(_points(h, W12, inside, t2), absF))
    m = _points(h, W12, True, thr2)
    inside = _points(h, W12, True, None).sum(axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        _close(h.significant_fraction(signif), np.where(inside > 0, m.sum(axis=1) / inside, np.nan))

    cos, sin = _unit(W12)
    bands = [(-np.inf, np.inf), (per[2], per[S // 2]), (per[S // 3], per[-1] * 2)]
    for pmin, pmax in bands:
        rows = (per >= pmin) & (per < pmax)
        for inside in (True, False):
            for sg, t2 in ((None, None), (signif, thr2)):
                m = _points(h, W12, inside, t2) & rows[:, None]
                z = _row_sum(m, cos) + 1j * _row_sum(m, sin)
                cnt = m.sum(axis=1)
                ps = h.mean_phase(pmin, pmax, inside_coi=inside, signif=sg, per_scale=True)
                assert np.array_equal(ps.count, cnt)
                check_mean_phase(ps, z, cnt)
                band = h.mean_phase(pmin, pmax, inside_coi=inside, signif=sg)
                assert band.count == cnt.sum()
                check_mean_phase(band, z.sum(), cnt.sum())
        if rows.any() and h.wavelet.cdelta != -1:
            w = np.where(rows, h.dj * h.dt / h.wavelet.cdelta / np.asarray(h.scales), 0.0)
            ref = (w[:, None] * W12).sum(axis=0)
            got = h.scale_avg(pmin, pmax)
            assert got.dtype == np.complex128 and got.shape == (n0,)
            bound = (np.abs(w)[:, None] * np.abs(W12)).sum(axis=0)
            assert (np.abs(got - ref) <= TOL * bound).all()


# ---- tests ------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp64", "fp32"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_fetch_window_and_reductions(api, case, precision):
    y1, y2, dt, kw = CASES[case]()
    W12, coi, freq, signif = api.xwt(y1, y2, dt, precision=precision, **kw)
    W12 = np.array(W12)
    h = api.xwt_resident(y1, y2, dt, precision=precision, **kw)
    assert isinstance(h, api.ResidentCrossWavelet)
    assert h.shape == W12.shape and h.precision == precision
    assert np.array_equal(h.coi, coi) and np.array_equal(h.freq, freq)
    assert np.array_equal(h.signif, signif)
    assert np.array_equal(h.period, 1 / freq)
    got = h.cross_spectrum()
    assert got.dtype == np.complex128 and np.array_equal(got, W12)
    for rows, cols in WINDOWS + EXTRA_WINDOWS:
        w = h.window(rows, cols)
        assert w.dtype == np.complex128
        assert np.array_equal(w, W12[rows, cols]), (rows, cols)
    assert np.array_equal(h.window(), W12)
    check_cross_reductions(h, W12, signif_with_gaps(W12))
    # xwt's own significance level, in the sample script's |W12|^2 / signif > 1 convention
    check_cross_reductions(h, W12, np.sqrt(h.signif))


def test_reductions_are_deterministic(api):
    y1, y2, dt, kw = chirp()
    for precision in ("fp64", "fp32"):
        h = api.xwt_resident(y1, y2, dt, precision=precision, **kw)
        thr = signif_with_gaps(h.cross_spectrum())
        calls = [lambda: h.global_power(inside_coi=True, signif=thr),
                 lambda: h.significant_fraction(thr),
                 lambda: h.mean_phase(signif=thr, per_scale=True),
                 lambda: h.mean_phase(),
                 lambda: h.scale_avg(4.0, 40.0),
                 lambda: h.window(slice(None, None, 3), slice(1, None, 3))]
        for f in calls:
            a, b = f(), f()
            for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
                assert np.array_equal(x, y, equal_nan=True)


def test_paul_dog(api):
    a, b = chirp_pair(700, seed=3)
    for mo in (api.Paul(4), api.DOG(2)):
        for p in ("fp64", "fp32"):
            kw = dict(dj=0.25, s0=1.0, J=20, wavelet=mo, precision=p)
            W12, _, _, signif = api.xwt(a, b, 0.5, **kw)
            W12 = np.array(W12)
            h = api.xwt_resident(a, b, 0.5, **kw)
            assert np.array_equal(h.cross_spectrum(), W12)
            assert np.array_equal(h.signif, signif)
            check_cross_reductions(h, W12, signif_with_gaps(W12))


def test_unpadded_mode_runs_fp64(api, emu):
    from pycwt_b200 import helpers
    y1, y2, dt, kw = ao_baltic()
    helpers.set_fft_padding(False)
    try:
        W12 = np.array(api.xwt(y1, y2, dt, **kw)[0])
        for p in ("fp64", "fp32"):      # no fp32 Bluestein transforms: both run in fp64
            h = api.xwt_resident(y1, y2, dt, precision=p, **kw)
            assert np.array_equal(h.cross_spectrum(), W12)
            check_cross_reductions(h, W12, signif_with_gaps(W12))
    finally:
        helpers.set_fft_padding(True)
        emu.set_padding(True)


def _all_methods(h, signif):
    return [lambda: h.cross_spectrum(), lambda: h.window(), lambda: h.global_power(),
            lambda: h.significant_fraction(signif), lambda: h.mean_phase(),
            lambda: h.scale_avg(0, np.inf)]


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_lifetime(api, emu, precision):
    from pycwt_b200 import _engine
    y1, y2, dt, kw = ao_baltic()
    h = api.xwt_resident(y1, y2, dt, precision=precision, **kw)
    W12 = h.cross_spectrum().copy()
    thr = signif_with_gaps(W12)
    first = [h.global_power(inside_coi=True, signif=thr), h.mean_phase(signif=thr, per_scale=True),
             h.scale_avg(0, np.inf)]
    # a live coherence handle survives xwt_resident
    hc = api.wct_resident(y1, y2, dt, precision=precision, **kw)
    WCT = hc.coherence().copy()
    h2 = api.xwt_resident(y1, y2, dt, precision=precision, **kw)
    assert np.array_equal(hc.coherence(), WCT)
    assert not np.array_equal(h2._serial, h._serial)
    for f in _all_methods(h, thr):
        with pytest.raises(_engine.EngineError):
            f()
    h.release()                               # a stale handle does not free its successor
    h = h2

    # other work on the same engine leaves the cross spectrum alone
    api.cwt(y1, dt, **kw)
    api.xwt(y2, y1, dt, precision=precision, **kw)
    api.wct(y2, y1, dt, sig=False, **kw)
    hc2 = api.wct_resident(y2, y1, dt, precision=precision, **kw)
    api.wct_significance(0.5, 0.4, dt, 1 / 4, 2 * dt, 8, mc_count=1, cache=False, progress=False)
    api.wct_significance(0.5, 0.4, dt, 1 / 4, 2 * dt, 8, mc_count=2, cache=False, progress=False,
                         seed=3)
    r = api.cwt_resident(y1, dt, **kw)
    assert np.array_equal(h.cross_spectrum(), W12)
    again = [h.global_power(inside_coi=True, signif=thr), h.mean_phase(signif=thr, per_scale=True),
             h.scale_avg(0, np.inf)]
    for a, b in zip(first, again):
        for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            assert np.array_equal(x, y, equal_nan=True)
    assert r.power().shape == r.shape         # cwt_resident after it is a normal transform
    hc2.release()

    # after xwt_resident no transform is resident
    api.xwt_resident(y2, y1, dt, precision=precision, **kw).release()
    with pytest.raises(_engine.EngineError):
        r.wave()
    assert emu.lib.cwtb_get_w(emu.h, W12.ctypes.data, 1, 0, 1) == -4
    assert emu.lib.cwtb_global_power(emu.h, np.empty(64).ctypes.data) == -4
    assert emu.lib.cwtb_field_get(emu.h, 0, 0, 1, W12.ctypes.data) == -4
    assert not emu.lib.cwtb_w_device_ptr(emu.h)

    h.release()                               # stale: a no-op
    h = api.xwt_resident(y1, y2, dt, precision=precision, **kw)
    h.release()
    for f in _all_methods(h, thr):
        with pytest.raises(_engine.EngineError):
            f()
    h.release()                               # idempotent
    assert emu.lib.cwtb_field_get(emu.h, 1, 0, 1, W12.ctypes.data) == -4


def test_failed_call_invalidates_the_old_handle(api, emu):
    from pycwt_b200 import _engine
    y1, y2, dt, kw = ao_baltic()
    h = api.xwt_resident(y1, y2, dt, **kw)
    before = emu.cross_serial()
    with pytest.raises(_engine.EngineError):
        # more rows than one launch takes: refused after the serial bump
        emu.xwt_resident(y1, y2, dt, np.full(60001, 2.0), 0, 6.0)
    assert emu.cross_serial() != before
    with pytest.raises(_engine.EngineError):
        h.global_power()


def test_c_status_codes(api, emu):
    """CWTB_ERR_STATE with nothing resident, CWTB_ERR_ARG for bad ranges and steps,
    CWTB_ERR_UNSUPPORTED for CWTB_TABLE and a batched W."""
    import ctypes
    lib, hdl = emu.lib, emu.h
    out = np.empty(64, dtype=np.complex128)
    p = out.ctypes.data_as(ctypes.c_void_p)
    emu.cross_release()
    assert lib.cwtb_field_row_stats(hdl, 1, None, None, None, p) == -4
    assert lib.cwtb_cross_scale_avg(hdl, p, p) == -4
    assert lib.cwtb_field_window(hdl, 1, 0, 1, 1, 0, 1, 1, p) == -4
    y1, y2, dt, kw = ao_baltic()
    S, n0 = api.xwt_resident(y1, y2, dt, **kw).shape
    assert lib.cwtb_field_get(hdl, 2, 0, 1, p) == -1                      # unknown field
    assert lib.cwtb_field_get(hdl, 1, S - 1, 2, p) == -1
    assert lib.cwtb_field_window(hdl, 1, 0, 1, 0, 0, 1, 1, p) == -1       # row step 0
    assert lib.cwtb_field_window(hdl, 1, 0, 1, 1, 0, 1, -2, p) == -1      # column step < 1
    assert lib.cwtb_field_window(hdl, 1, S - 1, 2, 1, 0, 1, 1, p) == -1   # past the last row
    assert lib.cwtb_field_window(hdl, 1, 0, 1, 1, n0 - 3, 2, 2, p) == 0   # ends on the last column
    assert lib.cwtb_field_window(hdl, 1, 0, 1, 1, n0 - 3, 3, 2, p) == -1  # past the last column
    assert lib.cwtb_field_window(hdl, 1, 0, 1, 1, -1, 1, 1, p) == -1
    lo = np.zeros(S, dtype=np.int64)
    hi = np.full(S, n0 + 1, dtype=np.int64)
    res = np.empty((S, 5))
    rp = res.ctypes.data_as(ctypes.c_void_p)
    assert lib.cwtb_field_row_stats(hdl, 1, lo.ctypes.data_as(ctypes.c_void_p),
                                    hi.ctypes.data_as(ctypes.c_void_p), None, rp) == -1
    hi[:] = 0
    lo[3] = 1
    assert lib.cwtb_field_row_stats(hdl, 1, lo.ctypes.data_as(ctypes.c_void_p),
                                    hi.ctypes.data_as(ctypes.c_void_p), None, rp) == -1
    assert lib.cwtb_field_row_stats(hdl, 1, None, None, None, rp) == 0     # NULL ranges: whole rows
    assert np.array_equal(res[:, 0], np.full(S, n0))
    sj = np.ascontiguousarray(api.xwt_resident(y1, y2, dt, **kw).scales)
    y1c, y2c = np.ascontiguousarray(y1, dtype=float), np.ascontiguousarray(y2, dtype=float)
    assert lib.cwtb_xwt_resident(hdl, y1c.ctypes.data, y2c.ctypes.data, n0, dt, sj.ctypes.data,
                                 sj.size, 3, 0.0) == -5                    # CWTB_TABLE
    # the W of a batched transform
    X = np.stack([y1, y2]).astype(np.float64)
    emu.cwt_batch(X, dt, sj, 0, 6.0, want_power=True)
    assert lib.cwtb_field_get(hdl, 0, 0, 1, p) == -5
    assert lib.cwtb_field_row_stats(hdl, 0, None, None, None, rp) == -5


def test_bad_arguments(api):
    y1, y2, dt, kw = ao_baltic()
    h = api.xwt_resident(y1, y2, dt, **kw)
    S = h.shape[0]
    for bad in (dict(rows=slice(None, None, -1)), dict(cols=slice(None, None, 0)),
                dict(cols=slice(None, None, 1.5)), dict(rows=3), dict(cols=[1, 2]),
                dict(rows=slice(0.5, 4)), dict(cols=None), dict(rows=slice(None, None, True))):
        with pytest.raises(ValueError):
            h.window(**bad)
    neg = np.ones(S)
    neg[4] = -1.0
    for f in (h.global_power, h.significant_fraction, h.mean_phase):
        with pytest.raises(ValueError):
            f(signif=neg)
        with pytest.raises(ValueError):
            f(signif=np.ones(S - 1))
    with pytest.raises(ValueError):
        h.scale_avg(1e9, 2e9)
    # Morlet(f0=8) has no Cdelta
    h8 = api.xwt_resident(y1, y2, dt, wavelet=api.Morlet(8), **kw)
    with pytest.raises(ValueError):
        h8.scale_avg(0, np.inf)
    h8.global_power()

    class Duck(object):
        """A duck-typed mother wavelet: xwt has no device path for it."""

        def __init__(self):
            self._m = api.Morlet(6)

        def __getattr__(self, name):
            if name == '_engine_spec':      # not one of the engine's analytic families
                raise AttributeError(name)
            return getattr(self._m, name)
    for call in (api.xwt, api.xwt_resident):
        with pytest.raises(NotImplementedError):
            call(y1, y2, dt, wavelet=Duck(), **kw)


# ---- ResidentTransform additions ----------------------------------------------------------------
def check_transform_additions(r, W):
    """window, global_power(signif=) and significant_fraction of a ResidentTransform against numpy
    on its fetched W; signif is in power units (|W|^2 > signif)."""
    S, n0 = W.shape
    P = _norm2(W)
    for rows, cols in WINDOWS + EXTRA_WINDOWS:
        w = r.window(rows, cols)
        assert w.dtype == np.complex128 and np.array_equal(w, W[rows, cols]), (rows, cols)
    thr = np.quantile(P, 0.55, axis=1)
    thr[::4] = np.nan
    thr[2] = np.inf
    for inside in (False, True):
        _close(r.global_power(inside_coi=inside, signif=thr), _mean(_points(r, W, inside, thr), P))
    # without signif the existing kernel path runs
    _close(r.global_power(signif=None), P.mean(axis=1))
    m = _points(r, W, True, thr)
    inside = _points(r, W, True, None).sum(axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        _close(r.significant_fraction(thr), np.where(inside > 0, m.sum(axis=1) / inside, np.nan))
    a, b = r.significant_fraction(thr), r.significant_fraction(thr)
    assert np.array_equal(a, b, equal_nan=True)
    bad = np.ones(S)
    bad[1] = -2.0
    with pytest.raises(ValueError):
        r.global_power(signif=bad)
    with pytest.raises(ValueError):
        r.significant_fraction(np.ones(S + 1))


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_resident_transform_additions_nino3(api, monkeypatch, precision):
    monkeypatch.setenv("CWTB_PRECISION", precision)
    g = load_golden("nino3_morlet_default")
    r = api.cwt_resident(g["x"], float(g["dt"]), **golden_cwt_kwargs(g))
    W = np.array(r.wave())
    check_transform_additions(r, W)
