"""The generalized Morse family on the device.

  * config 2's geometry at full size (Np = 2^20, 256 scales, fp64) and config 3's (2^18, 128 scales) in
    the fp32 engine, Morse(3, 20), row by row against the extended-precision reference of
    test_emu_morse.py at the bounds the fp64 / fp32 row-parity files hold the other analytic families
    to (every fourth row of config 2: the longdouble reference of 256 rows of 2^20 points is minutes
    of host time);
  * xwt and wct (generic smoothing, deltaj0 = 0.6) against a host numpy oracle in fp64: the reference
    rows, their product, and oracle/cwt_oracle.smooth_generic;
  * the resident handles: power_resident / xwt_resident / wct_resident equal the non-resident calls,
    their surrogate and cluster tests repeat for a seed, and `reconstruct` of a band-limited signal
    gives it back.
"""
import numpy as np
import pytest

import pycwt_b200 as pycwt
import test_emu_morse as M
import test_gpu_fp32_row_parity as p32
import test_gpu_row_parity as rp
import workloads
from oracle import cwt_oracle as orc
from pycwt_b200 import _engine
from pycwt_b200.mothers import Morse, enable_generic_smoothing

MORSE, F32 = _engine.MORSE, _engine.F32
BE, GA = 20.0, 3.0


@pytest.fixture(scope="module")
def eng():
    e = _engine.Engine(0)
    yield e
    e.close()


def _bounds(plan, log2N, exact, expand):
    return np.array([expand if (p < 0 and p != M.OS) else exact for p in plan])


@pytest.mark.gpu
def test_config2_rows_fp64(eng):
    x = workloads.config2_signal()
    sj = workloads.config2_scales()
    W = eng.cwt(x, 1.0, sj, MORSE, (BE, GA))
    plan = eng.last_plan(len(sj))
    rows = np.arange(0, len(sj), 4)
    err = rp.row_err(W[rows], M.morse_rows(x, 1.0, sj[rows], BE, GA))
    bound = _bounds(np.array(plan)[rows], 20, rp.EXACT, rp.EPS64)
    for j, e, b in zip(rows, err, bound):
        print("  config 2 Morse(3, 20) s = %-9.4g %-22s row_err %.2e (bound %.0e)"
              % (sj[j], M.kind(plan[j], 20), e, b))
    print("  classes:", sorted({M.kind(p, 20) for p in plan}))
    assert (err <= bound).all()


@pytest.mark.gpu
def test_config3_rows_fp32(eng):
    x = workloads.config3_signal()
    c = workloads.C3["paul"]
    sj = workloads.geometric_scales(c["s0"], c["dj"], c["J"])
    W = eng.cwt(x, 1.0, sj, MORSE, (BE, GA), precision=F32)
    plan = eng.last_plan(len(sj))
    R, sig = M.morse_ref32(x, 1.0, sj, BE, GA)
    err = p32.sigma_err(W, R, sig)
    bound = _bounds(plan, 18, p32.EXACT32, p32.EXPAND32)
    print("  config 3 fp32 Morse(3, 20): worst err/sigma %.2e, classes %s"
          % (err.max(), sorted({M.kind(p, 18) for p in plan})))
    assert (err <= bound).all(), dict(zip(sj[err > bound], err[err > bound]))


def _series(n=2 ** 14):
    rs = np.random.RandomState(3)
    t = np.arange(n)
    y1 = np.sin(2 * np.pi * t / 40) + 0.7 * rs.randn(n)
    y2 = np.sin(2 * np.pi * t / 40 + 0.9) + 0.7 * rs.randn(n)
    return y1, y2


def _geometry(n, mother, dj=1 / 12):
    s0 = 2 / mother.flambda()
    J = int(np.round(np.log2(n / s0) / dj))
    return dj, s0, J, s0 * 2 ** (np.arange(J + 1) * dj)


@pytest.mark.gpu
def test_xwt_wct_against_host_oracle():
    mother = Morse(GA, BE, deltaj0=0.6)
    y1, y2 = _series()
    dj, s0, J, sj = _geometry(len(y1), mother)
    y1n, y2n = [(y - y.mean()) / y.std() for y in (y1, y2)]
    W1 = M.morse_rows(y1n, 1.0, sj, BE, GA, dtype=np.float64)
    W2 = M.morse_rows(y2n, 1.0, sj, BE, GA, dtype=np.float64)
    W12 = pycwt.xwt(y1, y2, 1.0, dj, s0, J, wavelet=mother)[0]
    e = rp.row_err(W12, W1 * W2.conj())
    print("  xwt Morse(3, 20): worst row %.2e" % e.max())
    assert (e <= 2 * rp.EPS64).all()       # a product of two rows, expansion rows among them
    old = enable_generic_smoothing(True)
    try:
        WCT, aWCT = pycwt.wct(y1, y2, 1.0, dj, s0, J, sig=False, wavelet=mother)[:2]
    finally:
        enable_generic_smoothing(old)
    inv_s = 1.0 / sj[:, None]
    S1 = orc.smooth_generic(np.abs(W1) ** 2 * inv_s, 1.0, dj, sj, mother)
    S2 = orc.smooth_generic(np.abs(W2) ** 2 * inv_s, 1.0, dj, sj, mother)
    S12 = orc.smooth_generic(W1 * W2.conj() * inv_s, 1.0, dj, sj, mother)
    ref = np.abs(S12) ** 2 / (S1 * S2)
    d = np.abs(WCT - ref).max()
    print("  wct Morse(3, 20), deltaj0 = 0.6: max |WCT - oracle| %.2e" % d)
    assert d <= 1e-10
    assert np.abs(np.angle(np.exp(1j * (aWCT - np.angle(W1 * W2.conj()))))).max() <= 1e-9
    # without a smoothing window: the existing error
    with pytest.raises((ValueError, AttributeError)):
        pycwt.wct(y1, y2, 1.0, dj, s0, J, sig=False, wavelet=Morse())


@pytest.mark.gpu
def test_resident_products_and_tests():
    mother = Morse(GA, BE, deltaj0=0.6)
    y1, y2 = _series()
    dj, s0, J, sj = _geometry(len(y1), mother)
    y1n = (y1 - y1.mean()) / y1.std()
    # power
    h = pycwt.power_resident(y1, 1.0, dj, s0, J, wavelet=mother)
    W = pycwt.cwt(y1n, 1.0, dj, s0, J, wavelet=mother)[0]
    assert np.abs(h.window() - W).max() <= 1e-12 * np.abs(W).max()
    h.surrogate_test(mc_count=20, seed=11)
    p1 = h.pvalues()
    h.surrogate_test(mc_count=20, seed=11)
    assert np.array_equal(p1, h.pvalues())
    thr = np.full(len(h.scales), 4.0)
    r1, r2 = h.cluster_test(thr, mc_count=20, seed=12), h.cluster_test(thr, mc_count=20, seed=12)
    assert np.array_equal(r1.pvalue, r2.pvalue) and np.array_equal(r1.area, r2.area)
    # cross spectrum
    hx = pycwt.xwt_resident(y1, y2, 1.0, dj, s0, J, wavelet=mother)
    W12 = pycwt.xwt(y1, y2, 1.0, dj, s0, J, wavelet=mother)[0]
    assert np.abs(hx.window() - W12).max() <= 1e-12 * np.abs(W12).max()
    hx.surrogate_test(mc_count=20, seed=13)
    q1 = hx.pvalues()
    hx.surrogate_test(mc_count=20, seed=13)
    assert np.array_equal(q1, hx.pvalues())
    # coherence
    old = enable_generic_smoothing(True)
    try:
        hc = pycwt.wct_resident(y1, y2, 1.0, dj, s0, J, wavelet=mother)
        WCT = pycwt.wct(y1, y2, 1.0, dj, s0, J, sig=False, wavelet=mother)[0]
        assert np.abs(hc.window()[0] - WCT).max() <= 1e-12
        hc.surrogate_test(mc_count=10, seed=14)
        c1 = hc.pvalues()
        hc.surrogate_test(mc_count=10, seed=14)
        assert np.array_equal(c1, hc.pvalues())
        sig = np.full(len(hc.scales), 0.8)
        k1, k2 = hc.cluster_test(sig, mc_count=10, seed=15), hc.cluster_test(sig, mc_count=10, seed=15)
        assert np.array_equal(k1.pvalue, k2.pvalue)
    finally:
        enable_generic_smoothing(old)


@pytest.mark.gpu
def test_reconstruct_band_limited_signal():
    """Two tones, periods 32 and 100, well inside the scales: the full reconstruction gives them back
    away from the ends.  Bound 1e-3 of the signal's amplitude: the reconstruction's only approximation
    is the sum over scales at dj = 1/12 in place of the integral over ln s, which the extended-precision
    rows put at 8e-5 here; the device rows add rounding only."""
    mother = Morse(GA, BE)
    n = 4096
    t = np.arange(n)
    x = np.sin(2 * np.pi * t / 32) + 0.5 * np.sin(2 * np.pi * t / 100 + 0.3)
    dj, s0, J, sj = _geometry(n, mother)
    h = pycwt.power_resident(x, 1.0, dj, s0, J, wavelet=mother, normalize=False)
    rec = h.reconstruct()
    W = M.morse_rows(x, 1.0, sj, BE, GA, dtype=np.float64)
    host = dj / (mother.cdelta * mother.psi(0.0).real) * (W.real / np.sqrt(sj)[:, None]).sum(axis=0)
    mid = slice(600, n - 600)
    print("  reconstruct: |rec - x| %.2e, |rec - host restatement| %.2e"
          % (np.abs(rec - x)[mid].max(), np.abs(rec - host).max()))
    assert np.abs(rec - host).max() <= 1e-10
    assert np.abs(rec - x)[mid].max() <= 1e-3 * 1.5
