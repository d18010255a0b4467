"""Partial and multiple wavelet coherence (`partial_wct`, `multiple_wct`), checked on the
host-emulation build of the kernels (tests/_emu, the fixture pattern of test_emu_kernels.py).

  * fp64 against a composition of the oracle's `cwt` and `smooth` (or `smooth_generic` for Paul /
    DOG), on every point: |RP2 - ref| * D <= 1e-10 with D = (1 - R2_y2)(1 - R2_12) the oracle's
    denominator, and |RM2 - ref| * D <= 1e-10 with D = 1 - R2_12.  Both measures are ill-conditioned
    as D -> 0, so the bound is on the error times D;
  * fp32 against fp64 under the same scaling, 1e-3;
  * identities that tie the new outputs to the already-tested `wct`: 1 - RM2 = (1 - R2_y2)(1 - RP2),
    y = x1 gives RP2 = RM2 = 1, RM2 is symmetric in x1 and x2, 0 <= RP2, RM2 <= 1 and
    RM2 >= max(R2_y1, R2_y2);
  * the errors of `wct`, and the resident coherence and cross spectrum survive the calls.
"""
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import cwt_oracle as orc

TOL = 1e-10
TOL32 = 1e-3


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


def chirp_triple(n, seed=0):
    """y, x1, x2 sharing a chirp driver with different phases and independent noise: every row
    has points of low and of high coherence, and x1, x2 are far from coherent with each other."""
    rs = np.random.RandomState(seed)
    t = np.arange(n) / n
    ph = 2 * np.pi * (20 * t + (n / 16) * t ** 2)
    return (np.sin(ph) + 0.5 * rs.randn(n), np.sin(ph + 0.7) + 0.5 * rs.randn(n),
            np.sin(ph + 2.1) + 0.5 * rs.randn(n))


# ---- oracle composition ----------------------------------------------------------------------
def oracle_wct3(y, x1, x2, dt, dj, s0, J, mother):
    """RP2, RM2 and their denominators D from the oracle's transforms and smoothing operator, in
    the det G3 form of the definition (the engine evaluates the cancelled form)."""
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
    Sy, S1, S2 = (sm(np.abs(W) ** 2 * inv) for W in Ws)
    Wy, W1, W2 = Ws
    Sy1, Sy2, S12 = (sm(a * b.conj() * inv) for a, b in ((Wy, W1), (Wy, W2), (W1, W2)))
    R2 = {"y1": np.abs(Sy1) ** 2 / (Sy * S1), "y2": np.abs(Sy2) ** 2 / (Sy * S2),
          "12": np.abs(S12) ** 2 / (S1 * S2)}
    d12 = S1 * S2 - np.abs(S12) ** 2
    RP2 = np.abs(Sy1 * S2 - Sy2 * S12.conj()) ** 2 / ((Sy * S2 - np.abs(Sy2) ** 2) * d12)
    det = (Sy * S1 * S2 + 2 * (Sy1 * S12 * Sy2.conj()).real
           - Sy * np.abs(S12) ** 2 - S1 * np.abs(Sy2) ** 2 - S2 * np.abs(Sy1) ** 2)
    RM2 = 1 - det / (Sy * d12)
    return RP2, RM2, (1 - R2["y2"]) * (1 - R2["12"]), 1 - R2["12"], R2


def scaled_err(got, ref, D):
    """max |got - ref| * D over every point (all finite)."""
    assert got.shape == ref.shape
    assert np.isfinite(got).all() and np.isfinite(ref).all()
    return float((np.abs(got - ref) * D).max())


# (name, n, dt, dj, s0, J, wavelet): K = round(2 deltaj0 / dj)
CASES = {
    "morlet K=5": (1024, 1.0, 1 / 4, 2.0, 30, "morlet"),
    "morlet K=14": (1024, 1.0, 1 / 12, 2.0, 84, "morlet"),
    "morlet K=77": (512, 1.0, 1 / 64, 2.0, 320, "morlet"),
    "paul4 K=36": (700, 0.5, 1 / 12, 1.0, 70, "paul"),
    "dog2 K=11": (700, 0.5, 1 / 4, 1.0, 24, "dog"),
}
MOTHERS = {"morlet": (lambda a: a.Morlet(6), orc.Morlet(6)), "paul": (lambda a: a.Paul(4), orc.Paul(4)),
           "dog": (lambda a: a.DOG(2), orc.DOG(2))}


def run_case(api, name, precision="fp64", pad=True):
    n, dt, dj, s0, J, wav = CASES[name]
    y, x1, x2 = chirp_triple(n, seed=len(name))
    kw = dict(dj=dj, s0=s0, J=J, wavelet=MOTHERS[wav][0](api), precision=precision)
    RP2, coi, freq = api.partial_wct(y, x1, x2, dt, **kw)
    RM2, coi2, freq2 = api.multiple_wct(y, x1, x2, dt, **kw)
    assert RP2.dtype == np.float64 and RP2.shape == (J + 1, n) and RM2.shape == RP2.shape
    WCT, _, coi_w, freq_w, _ = api.wct(y, x1, dt, sig=False, **kw)
    assert np.array_equal(coi, coi_w) and np.array_equal(freq, freq_w)
    assert np.array_equal(coi2, coi_w) and np.array_equal(freq2, freq_w)
    return (y, x1, x2, dt, kw), RP2, RM2


def generic(fn):
    """Run fn with the generic smoothing of Paul / DOG enabled."""
    from pycwt_b200 import mothers
    old = mothers.enable_generic_smoothing(True)
    try:
        return fn()
    finally:
        mothers.enable_generic_smoothing(old)


# ---- tests -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_fp64_against_oracle(api, name):
    def body():
        (y, x1, x2, dt, kw), RP2, RM2 = run_case(api, name)
        n, dt, dj, s0, J, wav = CASES[name]
        rp, rm, Dp, Dm, _ = oracle_wct3(y, x1, x2, dt, dj, s0, J, MOTHERS[wav][1])
        ep, em = scaled_err(RP2, rp, Dp), scaled_err(RM2, rm, Dm)
        print("  %s: max |dRP2| D %.2e, max |dRM2| D %.2e" % (name, ep, em))
        assert ep <= TOL and em <= TOL
    generic(body)


def test_unpadded_odd_length(api, emu):
    """set_fft_padding(False) at an odd length: the transforms and the smoothing run un-padded,
    in fp64 whatever precision is asked for."""
    from pycwt_b200 import helpers
    y, x1, x2 = chirp_triple(1001, seed=5)
    helpers.set_fft_padding(False)
    orc.PAD_NEXT_POW2 = False
    try:
        rp, rm, Dp, Dm, _ = oracle_wct3(y, x1, x2, 1.0, 1 / 4, 2.0, 30, orc.Morlet(6))
        out = {}
        for p in ("fp64", "fp32"):
            kw = dict(dj=1 / 4, s0=2.0, J=30, precision=p)
            out[p] = (api.partial_wct(y, x1, x2, 1.0, **kw)[0], api.multiple_wct(y, x1, x2, 1.0, **kw)[0])
    finally:
        helpers.set_fft_padding(True)
        orc.PAD_NEXT_POW2 = True
        emu.set_padding(True)
    assert np.array_equal(out["fp64"][0], out["fp32"][0]) and np.array_equal(out["fp64"][1], out["fp32"][1])
    assert scaled_err(out["fp64"][0], rp, Dp) <= TOL and scaled_err(out["fp64"][1], rm, Dm) <= TOL


@pytest.mark.parametrize("name", ["morlet K=14", "morlet K=77", "paul4 K=36"])
def test_fp32_against_fp64(api, name):
    def body():
        (y, x1, x2, dt, kw), RP2, RM2 = run_case(api, name, "fp64")
        _, RP32, RM32 = run_case(api, name, "fp32")
        R2y2 = api.wct(y, x2, dt, sig=False, **kw)[0]
        R212 = api.wct(x1, x2, dt, sig=False, **kw)[0]
        ep = scaled_err(RP32, RP2, (1 - R2y2) * (1 - R212))
        em = scaled_err(RM32, RM2, 1 - R212)
        print("  %s fp32 vs fp64: max |dRP2| D %.2e, max |dRM2| D %.2e" % (name, ep, em))
        assert ep <= TOL32 and em <= TOL32
    generic(body)


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
@pytest.mark.parametrize("name", ["morlet K=5", "morlet K=77", "dog2 K=11"])
def test_identities(api, name, precision):
    tol = TOL if precision == "fp64" else TOL32

    def body():
        (y, x1, x2, dt, kw), RP2, RM2 = run_case(api, name, precision)
        R2y1, R2y2, R212 = (api.wct(a, b, dt, sig=False, **kw)[0] for a, b in ((y, x1), (y, x2), (x1, x2)))
        D12 = 1 - R212
        # 1 - RM2 = (1 - R2_y2)(1 - RP2)
        assert (np.abs((1 - RM2) - (1 - R2y2) * (1 - RP2)) * D12).max() <= tol
        # symmetric in x1, x2
        assert (np.abs(api.multiple_wct(y, x2, x1, dt, **kw)[0] - RM2) * D12).max() <= tol
        # bounds
        slack = tol / (D12 * (1 - R2y2))
        assert (RP2 >= -slack).all() and (RP2 <= 1 + slack).all()
        assert (RM2 >= -tol / D12).all() and (RM2 <= 1 + tol / D12).all()
        assert (RM2 >= np.maximum(R2y1, R2y2) - tol / D12).all()
        # y = x1: x1 explains y completely, with or without x2
        RP2s = api.partial_wct(x1, x1, x2, dt, **kw)[0]
        RM2s = api.multiple_wct(x1, x1, x2, dt, **kw)[0]
        assert (np.abs(RP2s - 1) * D12 ** 2).max() <= tol
        assert (np.abs(RM2s - 1) * D12).max() <= tol
    generic(body)


def test_errors(api):
    from pycwt_b200 import mothers
    y, x1, x2 = chirp_triple(256)
    for f in (api.partial_wct, api.multiple_wct):
        with pytest.raises(ValueError):
            f(y, x1, x2[:-1], 1.0)
        with pytest.raises(ValueError):
            f(y, x1[:-1], x2, 1.0)
        with pytest.raises(ValueError):
            f(np.stack([y, y]), np.stack([x1, x1]), np.stack([x2, x2]), 1.0, J=10)
        old = mothers.enable_generic_smoothing(False)
        try:
            for mo in (api.Paul(4), api.DOG(2)):
                with pytest.raises(AttributeError):
                    f(y, x1, x2, 1.0, wavelet=mo)
        finally:
            mothers.enable_generic_smoothing(old)
        with pytest.raises(ValueError):
            f(y, x1, x2, 1.0, wavelet=api.Morlet(8))          # deltaj0 = -1
        with pytest.raises(ValueError):
            f(y, x1, x2, 1.0, precision="fp16")

        class Duck(object):
            def __init__(self):
                self._m = api.Morlet(6)

            def __getattr__(self, name):
                if name == '_engine_spec':      # not one of the engine's analytic families
                    raise AttributeError(name)
                return getattr(self._m, name)
        with pytest.raises(NotImplementedError):
            f(y, x1, x2, 1.0, wavelet=Duck())


def test_resident_handles_survive(api, emu):
    from pycwt_b200 import _engine
    y, x1, x2 = chirp_triple(1024, seed=9)
    kw = dict(dj=1 / 4, s0=2.0, J=30)
    hc = api.wct_resident(y, x1, 1.0, **kw)
    hx = api.xwt_resident(y, x2, 1.0, **kw)
    WCT, aWCT, W12 = hc.coherence(), hc.phase(), hx.cross_spectrum()
    cs, xs = emu.coherence_serial(), emu.cross_serial()
    for p in ("fp64", "fp32"):
        api.partial_wct(y, x1, x2, 1.0, precision=p, **kw)
        api.multiple_wct(x2, y, x1, 1.0, precision=p, dj=1 / 64, s0=2.0, J=100)   # K = 77
    assert emu.coherence_serial() == cs and emu.cross_serial() == xs
    assert np.array_equal(hc.coherence(), WCT) and np.array_equal(hc.phase(), aWCT)
    assert np.array_equal(hx.cross_spectrum(), W12)
    # no transform is resident afterwards: the C side refuses to read W (CWTB_ERR_STATE)
    import ctypes
    out = np.empty(2 * 1024, dtype=np.complex128)
    assert emu.lib.cwtb_field_get(emu.h, _engine.FIELD_W, 0, 1, out.ctypes.data_as(ctypes.c_void_p)) == -4
    hc.release()
    hx.release()


def test_engine_outputs(api, emu):
    """Engine.wct3: either measure may be skipped, and both equal what the public calls return."""
    y, x1, x2 = chirp_triple(512, seed=2)
    sj = 2.0 * 2 ** (np.arange(25) / 4)
    yn = [(v - v.mean()) / v.std() for v in (y, x1, x2)]
    RP2, RM2 = emu.wct3(*yn, 1.0, 0.25, sj, 0, 6.0, 5)
    assert np.array_equal(emu.wct3(*yn, 1.0, 0.25, sj, 0, 6.0, 5, want_multiple=False)[0], RP2)
    only = emu.wct3(*yn, 1.0, 0.25, sj, 0, 6.0, 5, want_partial=False)
    assert only[0] is None and np.array_equal(only[1], RM2)
    assert np.array_equal(api.partial_wct(y, x1, x2, 1.0, dj=0.25, s0=2.0, J=24)[0], RP2)
    assert np.array_equal(api.multiple_wct(y, x1, x2, 1.0, dj=0.25, s0=2.0, J=24)[0], RM2)
