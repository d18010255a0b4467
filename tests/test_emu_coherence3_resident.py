"""Resident partial and multiple coherence (`wct3_resident`), checked on the host-emulation build of
the kernels (tests/_emu, the fixture pattern of test_emu_partial_coherence.py).

  * `partial()` / `multiple()` are bit-identical to `partial_wct` / `multiple_wct` in both
    precisions, for Morlet K = 5, 14, 77, Paul(4) and DOG(2) with generic smoothing, and at an odd
    un-padded length (fp64 fallback);
  * the partial phase against the angle of u = S_y1 S_2 - S_y2 conj(S_12) composed from the oracle's
    `cwt` and `smooth`: |gamma_ref| |e^{i phi} - e^{i phi_ref}| D <= 1e-10 with gamma_ref = sqrt(RP2_ref)
    and D = (1 - R2_y2)(1 - R2_12), the scaling of `scaled_err`; fp32 against fp64 within 1e-3;
  * `window` equals numpy slicing of the full fetches;
  * every reduction of both measures agrees with numpy on the fetched fields (means within 1e-12
    relative, circular sums within 1e-12 of the point count), with hand-made thresholds and with
    those of `wct3_significance`;
  * argument errors, lifetime against every other call, and the significance methods against
    the public calls with the same arguments.
"""
import ctypes
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import cwt_oracle as orc
from test_emu_partial_coherence import CASES, MOTHERS, chirp_triple, generic, oracle_wct3
from test_emu_coherence_resident import (WINDOWS, _close, _points, check_mean_phase, check_reductions,
                                         sig95_with_gaps)

TOL = 1e-10
TOL32 = 1e-3
TOLR = 1e-12
ERR_ARG, ERR_STATE = -1, -4


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


def _vp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ---- oracle composition of the partial phase ----------------------------------------------------
def oracle_u(y, x1, x2, dt, dj, s0, J, mother):
    """u = S_y1 S_2 - S_y2 conj(S_12) from the oracle's transforms and smoothing operator (the
    composition of `oracle_wct3`)."""
    Ws = []
    for v in (y, x1, x2):
        v = np.asarray(v, dtype=float)
        W, sj = orc.cwt((v - v.mean()) / v.std(), dt, dj, s0, J, mother)[:2]
        Ws.append(W)
    if isinstance(mother, orc.Morlet):
        def sm(F):
            return orc.smooth(F, dt, dj, sj, mother.deltaj0)
    else:
        def sm(F):
            return orc.smooth_generic(F, dt, dj, sj, mother)
    inv = 1.0 / sj[:, None]
    Wy, W1, W2 = Ws
    S2 = sm(np.abs(W2) ** 2 * inv)
    Sy1, Sy2, S12 = (sm(a * b.conj() * inv) for a, b in ((Wy, W1), (Wy, W2), (W1, W2)))
    return Sy1 * S2 - Sy2 * S12.conj()


def phase_err(phi, phi_ref, rp_ref, D):
    """max |gamma_ref| |e^{i phi} - e^{i phi_ref}| D over every point (all finite)."""
    assert phi.shape == phi_ref.shape
    assert np.isfinite(phi).all() and np.isfinite(phi_ref).all()
    return float((np.sqrt(rp_ref) * np.abs(np.exp(1j * phi) - np.exp(1j * phi_ref)) * D).max())


def case_args(api, name, precision):
    n, dt, dj, s0, J, wav = CASES[name]
    y, x1, x2 = chirp_triple(n, seed=len(name))
    return (y, x1, x2, dt), dict(dj=dj, s0=s0, J=J, wavelet=MOTHERS[wav][0](api), precision=precision)


# ---- numpy on the fetched fields ----------------------------------------------------------------
class _PartialView(object):
    """The handle's partial measure under the method names of `ResidentCoherence`, so that
    `check_reductions` of test_emu_coherence_resident.py applies unchanged."""

    def __init__(self, h):
        self._h = h

    def __getattr__(self, name):
        return getattr(self._h, name)

    def global_coherence(self, inside_coi=False, sig95=None):
        return self._h.global_coherence('partial', inside_coi=inside_coi, sig=sig95)

    def significant_fraction(self, sig95):
        return self._h.significant_fraction(sig95, measure='partial')

    def mean_phase(self, period_min=-np.inf, period_max=np.inf, inside_coi=True, sig95=None,
                   per_scale=False):
        return self._h.mean_phase(period_min, period_max, inside_coi=inside_coi, sig=sig95,
                                  per_scale=per_scale)

    def scale_avg(self, period_min, period_max):
        return self._h.scale_avg(period_min, period_max)[:2]


def check_multiple(h, RM2, sig):
    """The reductions of RM2 against numpy on the fetched field."""
    for inside in (False, True):
        for thr in (None, sig):
            m = _points(h, RM2, inside, thr)
            cnt = m.sum(axis=1)
            with np.errstate(invalid="ignore", divide="ignore"):
                ref = np.where(cnt > 0, np.einsum('ij,ij->i', m.astype(float), RM2) / cnt, np.nan)
            _close(h.global_coherence('multiple', inside_coi=inside, sig=thr), ref, TOLR)
    m = _points(h, RM2, True, sig)
    inside = _points(h, RM2, True, None).sum(axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        _close(h.significant_fraction(sig, measure='multiple'),
               np.where(inside > 0, m.sum(axis=1) / inside, np.nan), TOLR)
    per = h.period
    S = len(per)
    for pmin, pmax in [(-np.inf, np.inf), (per[2], per[S // 2])]:
        rows = (per >= pmin) & (per < pmax)
        ref = RM2[rows].mean(axis=0)
        rm = h.scale_avg(pmin, pmax)[2]
        assert np.abs(rm - ref).max() <= TOLR * np.abs(ref).max()


def check_all(h, RP2, phase, RM2, sig_p, sig_m):
    check_reductions(_PartialView(h), RP2, phase, sig_p)
    check_multiple(h, RM2, sig_m)


# ---- tests --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_fetch_equals_public_calls_and_phase_against_oracle(api, name):
    def body():
        phases, fields = {}, {}
        for p in ("fp64", "fp32"):
            args, kw = case_args(api, name, p)
            RP2, coi, freq = api.partial_wct(*args, **kw)
            RM2 = api.multiple_wct(*args, **kw)[0]
            h = api.wct3_resident(*args, **kw)
            assert h.shape == RP2.shape
            assert np.array_equal(h.partial(), RP2) and np.array_equal(h.multiple(), RM2)
            assert np.array_equal(h.coi, coi) and np.array_equal(h.freq, freq)
            phases[p], fields[p] = h.phase(), (RP2, RM2)
            assert (np.abs(phases[p]) <= np.pi).all()
            h.release()
        n, dt, dj, s0, J, wav = CASES[name]
        y, x1, x2 = chirp_triple(n, seed=len(name))
        rp, _, Dp, _, _ = oracle_wct3(y, x1, x2, dt, dj, s0, J, MOTHERS[wav][1])
        phi_ref = np.angle(oracle_u(y, x1, x2, dt, dj, s0, J, MOTHERS[wav][1]))
        e64 = phase_err(phases["fp64"], phi_ref, rp, Dp)
        e32 = phase_err(phases["fp32"], phases["fp64"], fields["fp64"][0], Dp)
        print("  %s: partial phase |g| |de^{i phi}| D: fp64 vs oracle %.2e, fp32 vs fp64 %.2e"
              % (name, e64, e32))
        assert e64 <= TOL and e32 <= TOL32
    generic(body)


def test_unpadded_odd_length(api, emu):
    """At an odd un-padded length the pipeline runs in fp64 whatever precision is asked for."""
    from pycwt_b200 import helpers
    y, x1, x2 = chirp_triple(1001, seed=5)
    helpers.set_fft_padding(False)
    orc.PAD_NEXT_POW2 = False
    try:
        rp, _, Dp, _, _ = oracle_wct3(y, x1, x2, 1.0, 1 / 4, 2.0, 30, orc.Morlet(6))
        phi_ref = np.angle(oracle_u(y, x1, x2, 1.0, 1 / 4, 2.0, 30, orc.Morlet(6)))
        got = {}
        for p in ("fp64", "fp32"):
            kw = dict(dj=1 / 4, s0=2.0, J=30, precision=p)
            h = api.wct3_resident(y, x1, x2, 1.0, **kw)
            assert np.array_equal(h.partial(), api.partial_wct(y, x1, x2, 1.0, **kw)[0])
            assert np.array_equal(h.multiple(), api.multiple_wct(y, x1, x2, 1.0, **kw)[0])
            got[p] = (h.partial(), h.phase(), h.multiple())
            sig = sig95_with_gaps(h, got[p][0])
            check_all(h, *got[p], sig, sig95_with_gaps(h, got[p][2]))
    finally:
        helpers.set_fft_padding(True)
        orc.PAD_NEXT_POW2 = True
        emu.set_padding(True)
    for a, b in zip(got["fp64"], got["fp32"]):
        assert np.array_equal(a, b)
    assert phase_err(got["fp64"][1], phi_ref, rp, Dp) <= TOL


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_window_and_reductions(api, precision):
    args, kw = case_args(api, "morlet K=14", precision)
    h = api.wct3_resident(*args, **kw)
    RP2, phase, RM2 = h.partial(), h.phase(), h.multiple()
    for rows, cols in WINDOWS + [(slice(None, None, 3), slice(None, None, 3)), (slice(84, 85), slice(None))]:
        a, b, c = h.window(rows, cols)
        assert np.array_equal(a, RP2[rows, cols]), (rows, cols)
        assert np.array_equal(b, phase[rows, cols]), (rows, cols)
        assert np.array_equal(c, RM2[rows, cols]), (rows, cols)
    full = h.window()
    assert all(np.array_equal(x, y) for x, y in zip(full, (RP2, phase, RM2)))
    # hand-made thresholds: NaN rows, rows no point passes, quantiles
    check_all(h, RP2, phase, RM2, sig95_with_gaps(h, RP2), sig95_with_gaps(h, RM2))
    # the levels of wct3_significance (NaN from its last row with points outside the cone on)
    n, dt, dj, s0, J, _ = CASES["morlet K=14"]
    sp, sm = h.significance(mc_count=2, seed=3, progress=False)
    assert np.isnan(sp).any() and np.isnan(sm).any()
    check_all(h, RP2, phase, RM2, sp, sm)
    # the multiple measure's phase planes are zero
    from pycwt_b200 import _engine
    out = h.engine.coherence3_scale_avg(_engine.MEASURE_MULTIPLE, np.ones(len(h.scales)))
    assert not out[1:].any()
    # repeated reductions are bit-identical
    calls = [lambda: h.global_coherence('multiple', inside_coi=True, sig=sm),
             lambda: h.significant_fraction(sp),
             lambda: h.mean_phase(sig=sp, per_scale=True),
             lambda: h.scale_avg(4.0, 40.0)]
    for f in calls:
        a, b = f(), f()
        for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            assert np.array_equal(x, y, equal_nan=True)
    h.release()


def test_argument_errors(api, emu):
    from pycwt_b200 import _engine
    args, kw = case_args(api, "morlet K=5", "fp64")
    h = api.wct3_resident(*args, **kw)
    S, n0 = h.shape
    for bad in ("coherence", 0, None, "Partial"):
        with pytest.raises(ValueError):
            h.global_coherence(bad)
        with pytest.raises(ValueError):
            h.significant_fraction(np.zeros(S), measure=bad)
    for f in (lambda s: h.global_coherence(sig=s), lambda s: h.significant_fraction(s),
              lambda s: h.mean_phase(sig=s), lambda s: h.global_coherence('multiple', sig=s)):
        for s in (np.zeros(S - 1), np.zeros((S, 1)), 0.5):
            with pytest.raises(ValueError):
                f(s)
    for bad in (dict(rows=slice(None, None, -1)), dict(cols=slice(None, None, 0)),
                dict(cols=slice(None, None, 1.5)), dict(rows=3), dict(cols=[1, 2]),
                dict(rows=slice(None, None, True))):
        with pytest.raises(ValueError):
            h.window(**bad)
    with pytest.raises(ValueError):
        h.scale_avg(1e9, 2e9)
    # a phase asked of the multiple coherence, an unknown measure: CWTB_ERR_ARG
    with pytest.raises(_engine.EngineError):
        emu.coherence3_window(_engine.MEASURE_MULTIPLE, 0, 1, 1, 0, 4, 1, want_phase=True)
    with pytest.raises(_engine.EngineError):
        emu.coherence3_row_stats(_engine.MEASURE_MULTIPLE, np.zeros(S), np.full(S, n0), want_phase=True)
    lib, hdl = emu.lib, emu.h
    out = np.empty(4 * S)
    lo, hi = np.zeros(S, dtype=np.int64), np.full(S, n0, dtype=np.int64)
    assert lib.cwtb_coherence3_window(hdl, 1, 0, 1, 1, 0, 2, 1, _vp(out), _vp(out)) == ERR_ARG
    assert lib.cwtb_coherence3_window(hdl, 1, 0, 1, 1, 0, 2, 1, _vp(out), None) == 0
    assert lib.cwtb_coherence3_window(hdl, 0, 0, 1, 1, 0, 2, 1, _vp(out), _vp(out)) == 0
    assert lib.cwtb_coherence3_row_stats(hdl, 1, _vp(lo), _vp(hi), None, 1, _vp(out)) == ERR_ARG
    for m in (2, -1):
        assert lib.cwtb_coherence3_window(hdl, m, 0, 1, 1, 0, 2, 1, _vp(out), None) == ERR_ARG
        assert lib.cwtb_coherence3_row_stats(hdl, m, _vp(lo), _vp(hi), None, 0, _vp(out)) == ERR_ARG
        assert lib.cwtb_coherence3_scale_avg(hdl, m, _vp(out), _vp(out)) == ERR_ARG
    assert lib.cwtb_coherence3_window(hdl, 0, 0, 1, 0, 0, 1, 1, _vp(out), None) == ERR_ARG   # row step 0
    assert lib.cwtb_coherence3_window(hdl, 0, S - 1, 2, 1, 0, 1, 1, _vp(out), None) == ERR_ARG
    assert lib.cwtb_coherence3_window(hdl, 0, 0, 1, 1, n0 - 3, 3, 2, _vp(out), None) == ERR_ARG
    h.release()


def _all_methods(h):
    S = len(h.scales)
    return [h.partial, h.multiple, h.phase, h.window, h.global_coherence,
            lambda: h.significant_fraction(np.zeros(S)), h.mean_phase,
            lambda: h.scale_avg(0, np.inf),
            lambda: h.significance(mc_count=1, seed=1, progress=False),
            lambda: h.surrogate_significance(mc_count=1, seed=1)]


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_lifetime(api, emu, precision):
    from pycwt_b200 import _engine
    y, x1, x2 = chirp_triple(1024, seed=9)
    kw = dict(dj=1 / 4, s0=2.0, J=30, precision=precision)
    h = api.wct3_resident(y, x1, x2, 1.0, **kw)
    fields = (h.partial(), h.phase(), h.multiple())
    g0 = h.global_coherence(inside_coi=True)
    serial = emu.coherence3_serial()
    # other work on the same engine leaves it alone
    api.cwt(y, 1.0, dj=1 / 4, s0=2.0, J=30)
    api.xwt(y, x1, 1.0, **kw)
    api.wct(y, x2, 1.0, sig=False, **kw)
    hc = api.wct_resident(y, x1, 1.0, **kw)
    hx = api.xwt_resident(y, x2, 1.0, **kw)
    api.partial_wct(x2, y, x1, 1.0, **kw)
    api.multiple_wct(y, x1, x2, 1.0, dj=1 / 64, s0=2.0, J=100, precision=precision)   # K = 77
    api.wct3_significance(0.1, 0.2, 0.3, 1.0, 1 / 4, 2.0, 30, mc_count=2, seed=4, progress=False,
                          precision=precision)
    api.wct3_surrogate_significance(y, x1, x2, 1.0, mc_count=2, seed=4, **kw)
    assert emu.coherence3_serial() == serial
    assert all(np.array_equal(a, b) for a, b in zip((h.partial(), h.phase(), h.multiple()), fields))
    assert np.array_equal(h.global_coherence(inside_coi=True), g0, equal_nan=True)

    # wct_resident / xwt_resident handles survive a wct3_resident
    WCT, aWCT, W12 = hc.coherence(), hc.phase(), hx.cross_spectrum()
    h2 = api.wct3_resident(x1, y, x2, 1.0, **kw)
    assert np.array_equal(hc.coherence(), WCT) and np.array_equal(hc.phase(), aWCT)
    assert np.array_equal(hx.cross_spectrum(), W12)
    # ... and the old handle dies
    for f in _all_methods(h):
        with pytest.raises(_engine.EngineError, match="no longer resident"):
            f()
    h.release()                               # a stale handle does not free its successor
    assert np.array_equal(h2.partial(), api.partial_wct(x1, y, x2, 1.0, **kw)[0])
    assert h2.shape == h.shape and np.array_equal(h2.coi, h.coi)
    # no transform is resident afterwards: the C side refuses to read W
    out = np.empty(2 * 1024, dtype=np.complex128)
    assert emu.lib.cwtb_field_get(emu.h, _engine.FIELD_W, 0, 1, _vp(out)) == ERR_STATE
    h2.release()
    for f in _all_methods(h2):
        with pytest.raises(_engine.EngineError):
            f()
    h2.release()                              # idempotent
    assert np.array_equal(hc.coherence(), WCT)
    hc.release()
    hx.release()


def test_c_status_without_slot(api, emu):
    """CWTB_ERR_STATE from every reading call with nothing resident; a refused call leaves nothing."""
    from pycwt_b200 import _engine
    lib, hdl = emu.lib, emu.h
    y, x1, x2 = chirp_triple(256, seed=1)
    h = api.wct3_resident(y, x1, x2, 1.0, dj=1 / 4, s0=2.0, J=20)
    before = emu.coherence3_serial()
    sj = np.asarray(h.scales)
    with pytest.raises(_engine.EngineError):
        # a boxcar of no taps, refused when the window is uploaded: after the serial bump
        emu.wct3_resident(y, x1, x2, 1.0, 0.25, sj, 0, 6.0, 0)
    assert emu.coherence3_serial() != before
    with pytest.raises(_engine.EngineError):
        h.partial()
    out = np.empty(64)
    for m in (0, 1):
        assert lib.cwtb_coherence3_window(hdl, m, 0, 1, 1, 0, 1, 1, _vp(out), None) == ERR_STATE
        assert lib.cwtb_coherence3_row_stats(hdl, m, None, None, None, 0, _vp(out)) == ERR_STATE
        assert lib.cwtb_coherence3_scale_avg(hdl, m, _vp(out), _vp(out)) == ERR_STATE
    h = api.wct3_resident(y, x1, x2, 1.0, dj=1 / 4, s0=2.0, J=20)
    emu.coherence3_release()
    assert lib.cwtb_coherence3_row_stats(hdl, 0, None, None, None, 1, _vp(out)) == ERR_STATE
    with pytest.raises(_engine.EngineError):
        h.multiple()


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_significance_methods(api, precision):
    args, kw = case_args(api, "morlet K=5", precision)
    kw.pop("wavelet")
    y, x1, x2, dt = args
    h = api.wct3_resident(*args, **kw)
    from pycwt_b200.helpers import ar1
    al = [ar1(v)[0] for v in (y, x1, x2)]
    mc = dict(dt=dt, dj=kw["dj"], s0=kw["s0"], J=kw["J"], significance_level=0.9, precision=precision)
    got = h.significance(0.9, mc_count=3, seed=21, progress=False)
    ref = api.wct3_significance(*al, mc_count=3, seed=21, progress=False, **mc)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(got, ref))
    np.random.seed(5)
    got = h.significance(0.9, mc_count=2, progress=False)
    np.random.seed(5)
    ref = api.wct3_significance(*al, mc_count=2, progress=False, **mc)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(got, ref))
    for cond in (True, False):
        got = h.surrogate_significance(0.9, mc_count=3, seed=8, conditional=cond)
        ref = api.wct3_surrogate_significance(y, x1, x2, dt, dj=kw["dj"], s0=kw["s0"], J=kw["J"],
                                              significance_level=0.9, mc_count=3, seed=8,
                                              precision=precision, conditional=cond)
        assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(got, ref))
    np.random.seed(6)
    got = h.surrogate_significance(mc_count=2)
    np.random.seed(6)
    ref = api.wct3_surrogate_significance(y, x1, x2, dt, dj=kw["dj"], s0=kw["s0"], J=kw["J"],
                                          mc_count=2, precision=precision)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(got, ref))
    assert np.array_equal(h.partial(), api.partial_wct(*args, **kw)[0])
    h.release()


def test_zero_partial_spectrum(emu):
    """y = 0: u = 0 at every point, so the partial phase is 0 (np.angle(0)); RP2 and RM2 have a zero
    numerator (their denominators hold S_y, which rounding of the smoothing may leave at 0 or not)."""
    _, x1, x2 = chirp_triple(512, seed=4)
    sj = 2.0 * 2 ** (np.arange(21) / 4)
    emu.wct3_resident(np.zeros(512), x1, x2, 1.0, 0.25, sj, 0, 6.0, 5)
    from pycwt_b200 import _engine
    rp, ph = emu.coherence3_window(_engine.MEASURE_PARTIAL, 0, 21, 1, 0, 512, 1, want_phase=True)
    rm = emu.coherence3_window(_engine.MEASURE_MULTIPLE, 0, 21, 1, 0, 512, 1)[0]
    assert np.array_equal(ph, np.zeros((21, 512)))
    assert ((rp == 0) | np.isnan(rp)).all() and ((rm == 0) | np.isnan(rm)).all()
    emu.coherence3_release()
