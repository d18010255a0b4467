"""Resident wavelet coherence (`wct_resident`), checked on the host-emulation build of the kernels
(tests/_emu, the fixture pattern of test_emu_kernels.py).

  * the full fetches are bit-identical to `wct(sig=False)` in both precisions;
  * `window` equals numpy slicing of the fetched fields;
  * every reduction agrees with numpy on the fetched fields: means within 1e-12 relative, the
    circular sums (bounded by the point count) within 1e-12 of the count;
  * the handle survives cwt / xwt / wct / significance and dies with the next wct_resident or
    release().
"""
import os

import numpy as np
import pytest

from conftest import ROOT, load_golden
from test_emu_coherence_fp32 import chirp_pair

TOL = 1e-12


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

WINDOWS = [
    (slice(None), slice(None)),
    (slice(3, 40, 5), slice(-100, None, 7)),
    (slice(-5, None), slice(1, -1, 3)),
    (slice(None, None, 4), slice(2, 147, 13)),
    (slice(0, 1), slice(None, None, 64)),
    (slice(10, 1000, 7), slice(-3, None)),
    (slice(2, 3), slice(5, 5)),
    (slice(None, None, 2), slice(None)),
]


# ---- numpy on the fetched fields --------------------------------------------------------------
def _points(h, WCT, inside_coi, sig95):
    """[S, n0] mask of the points a reduction uses."""
    S, n0 = WCT.shape
    m = np.ones((S, n0), dtype=bool)
    if inside_coi:
        m &= h.period[:, None] <= h.coi[None, :]
    if sig95 is not None:
        with np.errstate(invalid="ignore"):
            m &= WCT > np.asarray(sig95)[:, None]
    return m


def _close(a, b, tol=TOL):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    assert a.shape == b.shape
    assert (np.isnan(a) == np.isnan(b)).all(), (a, b)
    ok = ~np.isnan(b)
    assert (np.abs(a[ok] - b[ok]) <= tol * np.maximum(np.abs(b[ok]), 1e-300)).all(), \
        np.abs(a[ok] - b[ok]).max()


def check_reductions(h, WCT, aWCT, sig95):
    """Every reduction of the handle against numpy on the fetched fields."""
    S, n0 = WCT.shape
    per = h.period
    # the in-COI column ranges of the shared helper are the reference's `period <= coi` mask
    lo, hi = h.coi_ranges()
    cols = np.arange(n0)
    assert np.array_equal((cols[None, :] >= lo[:, None]) & (cols[None, :] < hi[:, None]),
                          _points(h, WCT, True, None))
    def masked_row_sum(m, X):
        return np.einsum('ij,ij->i', m.astype(float), X)

    for inside in (False, True):
        for thr in (None, sig95):
            m = _points(h, WCT, inside, thr)
            cnt = m.sum(axis=1)
            with np.errstate(invalid="ignore", divide="ignore"):
                ref = np.where(cnt > 0, masked_row_sum(m, WCT) / cnt, np.nan)
            _close(h.global_coherence(inside_coi=inside, sig95=thr), ref)
    m = _points(h, WCT, True, sig95)
    inside = _points(h, WCT, True, None).sum(axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        _close(h.significant_fraction(sig95), np.where(inside > 0, m.sum(axis=1) / inside, np.nan))

    cos, sin = np.cos(aWCT), np.sin(aWCT)
    bands = [(-np.inf, np.inf), (per[2], per[S // 2]), (per[S // 3], per[-1] * 2)]
    for pmin, pmax in bands:
        rows = (per >= pmin) & (per < pmax)
        for inside in (True, False):
            for thr in (None, sig95):
                m = _points(h, WCT, inside, thr) & rows[:, None]
                z = masked_row_sum(m, cos) + 1j * masked_row_sum(m, sin)
                cnt = m.sum(axis=1)
                ps = h.mean_phase(pmin, pmax, inside_coi=inside, sig95=thr, per_scale=True)
                assert np.array_equal(ps.count, cnt)
                check_mean_phase(ps, z, cnt)
                band = h.mean_phase(pmin, pmax, inside_coi=inside, sig95=thr)
                assert band.count == cnt.sum()
                check_mean_phase(band, z.sum(), cnt.sum())
        mean, phase = h.scale_avg(pmin, pmax)
        ref = WCT[rows].mean(axis=0)
        assert np.abs(mean - ref).max() <= TOL * np.abs(ref).max()
        z = cos[rows].sum(axis=0) + 1j * sin[rows].sum(axis=0)
        # the angle is as well defined as |sum e^{i aWCT}| is large against the rounding of the sum
        assert (np.abs(z) * np.abs(np.exp(1j * phase) - z / np.abs(z)) <= TOL * rows.sum()).all()


def check_mean_phase(mp, z, cnt):
    """angle = arg z, strength = |z| / count, NaN for an empty set; z is a sum of `cnt` unit
    vectors, so its rounding is bounded by the count."""
    angle, strength = np.asarray(mp.angle, dtype=float), np.asarray(mp.strength, dtype=float)
    z, cnt = np.asarray(z), np.asarray(cnt)
    empty = cnt == 0
    assert np.isnan(angle[empty]).all() and np.isnan(strength[empty]).all()
    assert not np.isnan(angle[~empty]).any()
    zk = np.where(empty, 0, z)
    got = np.where(empty, 0, strength * cnt * np.exp(1j * np.where(empty, 0, angle)))
    assert (np.abs(got - zk) <= TOL * np.maximum(cnt, 1)).all(), np.abs(got - zk).max()


def sig95_with_gaps(h, WCT):
    """A threshold per scale with NaN entries and rows that no point passes."""
    S = WCT.shape[0]
    thr = np.quantile(WCT, 0.6, axis=1)
    thr[::5] = np.nan
    thr[1] = 2.0
    thr[S - 2] = np.inf
    return thr


# ---- tests ------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp64", "fp32"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_fetch_window_and_reductions(api, case, precision):
    y1, y2, dt, kw = CASES[case]()
    WCT, aWCT, coi, freq, _ = api.wct(y1, y2, dt, sig=False, precision=precision, **kw)
    h = api.wct_resident(y1, y2, dt, precision=precision, **kw)
    assert h.shape == WCT.shape
    assert np.array_equal(h.coi, coi) and np.array_equal(h.freq, freq)
    assert np.array_equal(h.period, 1 / freq)
    assert np.array_equal(h.coherence(), WCT)
    assert np.array_equal(h.phase(), aWCT)
    for rows, cols in WINDOWS:
        w, a = h.window(rows, cols)
        assert np.array_equal(w, WCT[rows, cols]) and np.array_equal(a, aWCT[rows, cols]), (rows, cols)
    assert np.array_equal(h.window()[0], WCT)
    check_reductions(h, WCT, aWCT, sig95_with_gaps(h, WCT))


def test_reductions_are_deterministic(api):
    y1, y2, dt, kw = chirp()
    h = api.wct_resident(y1, y2, dt, **kw)
    thr = sig95_with_gaps(h, h.coherence())
    calls = [lambda: h.global_coherence(inside_coi=True, sig95=thr),
             lambda: h.significant_fraction(thr),
             lambda: h.mean_phase(sig95=thr, per_scale=True),
             lambda: h.mean_phase(),
             lambda: h.scale_avg(4.0, 40.0)]
    for f in calls:
        a, b = f(), f()
        for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            assert np.array_equal(x, y, equal_nan=True)


def test_paul_dog_generic_smoothing(api):
    from pycwt_b200 import mothers
    a, b = chirp_pair(700, seed=3)
    old = mothers.enable_generic_smoothing(True)
    try:
        for mo in (api.Paul(4), api.DOG(2), api.DOG(6)):
            for p in ("fp64", "fp32"):
                kw = dict(dj=0.25, s0=1.0, J=20, wavelet=mo, precision=p)
                WCT, aWCT = api.wct(a, b, 0.5, sig=False, **kw)[:2]
                h = api.wct_resident(a, b, 0.5, **kw)
                assert np.array_equal(h.coherence(), WCT) and np.array_equal(h.phase(), aWCT)
                _close(h.global_coherence(), WCT.mean(axis=1))
    finally:
        mothers.enable_generic_smoothing(old)


def test_unpadded_mode_runs_fp64(api, emu):
    from pycwt_b200 import helpers
    y1, y2, dt, kw = ao_baltic()
    helpers.set_fft_padding(False)
    try:
        WCT, aWCT = api.wct(y1, y2, dt, sig=False, **kw)[:2]
        for p in ("fp64", "fp32"):      # no fp32 Bluestein transforms: both run in fp64
            h = api.wct_resident(y1, y2, dt, precision=p, **kw)
            assert np.array_equal(h.coherence(), WCT) and np.array_equal(h.phase(), aWCT)
            check_reductions(h, WCT, aWCT, sig95_with_gaps(h, WCT))
    finally:
        helpers.set_fft_padding(True)
        emu.set_padding(True)


def _all_methods(h, sig95):
    return [lambda: h.coherence(), lambda: h.phase(), lambda: h.window(),
            lambda: h.global_coherence(), lambda: h.significant_fraction(sig95),
            lambda: h.mean_phase(), lambda: h.scale_avg(0, np.inf),
            lambda: h.significance(mc_count=1, cache=False, seed=1, progress=False)]


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_lifetime(api, emu, precision):
    from pycwt_b200 import _engine
    y1, y2, dt, kw = ao_baltic()
    h = api.wct_resident(y1, y2, dt, precision=precision, **kw)
    WCT, aWCT = h.coherence(), h.phase()
    g0 = h.global_coherence(inside_coi=True)
    # other work on the same engine leaves the coherence alone
    api.cwt(y1, dt, **kw)
    api.xwt(y1, y2, dt, precision=precision, **kw)
    api.wct(y2, y1, dt, sig=False, **kw)
    sig = h.significance(mc_count=4, cache=False, seed=11, progress=False)
    ref = api.wct(y1, y2, dt, sig=True, mc_count=4, cache=False, seed=11, progress=False,
                  precision=precision, **kw)[4]
    assert np.array_equal(sig, ref, equal_nan=True)
    assert np.array_equal(h.coherence(), WCT) and np.array_equal(h.phase(), aWCT)
    assert np.array_equal(h.global_coherence(inside_coi=True), g0, equal_nan=True)
    m = _points(h, WCT, False, sig)
    with np.errstate(invalid="ignore", divide="ignore"):
        _close(h.global_coherence(sig95=sig), np.where(m, WCT, 0).sum(axis=1) / m.sum(axis=1))

    # a second wct_resident replaces it
    h2 = api.wct_resident(y2, y1, dt, precision=precision, **kw)
    for f in _all_methods(h, sig):
        with pytest.raises(_engine.EngineError):
            f()
    h.release()                               # a stale handle does not free its successor
    assert np.array_equal(h2.coherence(), api.wct(y2, y1, dt, sig=False, precision=precision, **kw)[0])
    assert h2.shape == h.shape and np.array_equal(h2.coi, h.coi)     # host data stay readable
    h2.release()
    for f in _all_methods(h2, sig):
        with pytest.raises(_engine.EngineError):
            f()
    h2.release()                              # idempotent


def test_refused_boxcar_invalidates_the_old_handle(api, emu):
    from pycwt_b200 import _engine
    y1, y2, dt, kw = ao_baltic()
    h = api.wct_resident(y1, y2, dt, **kw)
    before = emu.coherence_serial()
    with pytest.raises(_engine.EngineError):
        # a boxcar of no taps, refused when the window is uploaded: fails after the serial bump
        emu.wct_resident(y1, y2, dt, 1 / 12, h.scales, 0, 6.0, 0)
    assert emu.coherence_serial() != before
    with pytest.raises(_engine.EngineError):
        h.global_coherence()


def test_c_status_codes(api, emu):
    """CWTB_ERR_STATE with nothing resident, CWTB_ERR_ARG for bad ranges and steps."""
    import ctypes
    lib, hdl = emu.lib, emu.h
    out = np.empty(64)
    p = out.ctypes.data_as(ctypes.c_void_p)
    emu.coherence_release()
    assert lib.cwtb_coherence_row_stats(hdl, None, None, None, 0, p) == -4
    assert lib.cwtb_coherence_scale_avg(hdl, p, p) == -4
    assert lib.cwtb_coherence_window(hdl, 0, 1, 1, 0, 1, 1, p, None) == -4
    y1, y2, dt, kw = ao_baltic()
    h = api.wct_resident(y1, y2, dt, **kw)
    S, n0 = h.shape
    assert lib.cwtb_coherence_window(hdl, 0, 1, 0, 0, 1, 1, p, None) == -1          # row step 0
    assert lib.cwtb_coherence_window(hdl, 0, 1, 1, 0, 1, -2, p, None) == -1         # column step < 1
    assert lib.cwtb_coherence_window(hdl, S - 1, 2, 1, 0, 1, 1, p, None) == -1      # past the last row
    assert lib.cwtb_coherence_window(hdl, 0, 1, 1, n0 - 3, 2, 2, p, None) == 0      # ends on the last column
    assert lib.cwtb_coherence_window(hdl, 0, 1, 1, n0 - 3, 3, 2, p, None) == -1     # past the last column
    assert lib.cwtb_coherence_window(hdl, 0, 1, 1, -1, 1, 1, p, None) == -1
    lo = np.zeros(S, dtype=np.int64)
    hi = np.full(S, n0 + 1, dtype=np.int64)
    res = np.empty((S, 4))
    assert lib.cwtb_coherence_row_stats(hdl, lo.ctypes.data_as(ctypes.c_void_p),
                                        hi.ctypes.data_as(ctypes.c_void_p), None, 0,
                                        res.ctypes.data_as(ctypes.c_void_p)) == -1
    hi[:] = 0
    lo[3] = 1
    assert lib.cwtb_coherence_row_stats(hdl, lo.ctypes.data_as(ctypes.c_void_p),
                                        hi.ctypes.data_as(ctypes.c_void_p), None, 0,
                                        res.ctypes.data_as(ctypes.c_void_p)) == -1
    # lo = hi = NULL: whole rows
    assert lib.cwtb_coherence_row_stats(hdl, None, None, None, 0, res.ctypes.data_as(ctypes.c_void_p)) == 0
    assert np.array_equal(res[:, 0], np.full(S, n0))
    _close(res[:, 1] / n0, h.coherence().mean(axis=1))


def test_bad_slices(api):
    y1, y2, dt, kw = ao_baltic()
    h = api.wct_resident(y1, y2, dt, **kw)
    for bad in (dict(rows=slice(None, None, -1)), dict(cols=slice(None, None, 0)),
                dict(cols=slice(None, None, 1.5)), dict(rows=3), dict(cols=[1, 2]),
                dict(rows=slice(0.5, 4)), dict(cols=None), dict(rows=slice(None, None, True))):
        with pytest.raises(ValueError):
            h.window(**bad)
    with pytest.raises(ValueError):
        h.global_coherence(sig95=np.zeros(3))
    with pytest.raises(ValueError):
        h.scale_avg(1e9, 2e9)
