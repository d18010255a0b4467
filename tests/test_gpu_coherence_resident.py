"""Resident wavelet coherence (`wct_resident`) at config 4 on the GPU (two 2^18-point series,
s0 = 2, dj = 1/12, J = 144), in fp64 and fp32: fetches bit-identical to `wct(sig=False)`, every
reduction against numpy on the fetched fields, repeated reductions bit-identical, and the handle
alive after a seeded Monte-Carlo run of 8 surrogate pairs."""
import numpy as np
import pytest

from test_emu_coherence_resident import WINDOWS, check_reductions, sig95_with_gaps

pytestmark = pytest.mark.gpu

DT, DJ, S0, J = 1.0, 1 / 12, 2.0, 144


@pytest.fixture(scope="module")
def pycwt(has_cuda):
    if not has_cuda:
        pytest.skip("no CUDA device")
    import pycwt_b200
    return pycwt_b200


@pytest.fixture(scope="module")
def signals():
    import workloads
    return workloads.config4_signals()


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_config4_resident_coherence(pycwt, signals, precision):
    y1, y2 = signals
    kw = dict(dj=DJ, s0=S0, J=J, precision=precision)
    WCT, aWCT, coi, freq, _ = pycwt.wct(y1, y2, DT, sig=False, **kw)
    WCT, aWCT = np.array(WCT), np.array(aWCT)          # own copies: the pinned buffers are pooled
    h = pycwt.wct_resident(y1, y2, DT, **kw)
    assert h.shape == (J + 1, y1.size)
    assert np.array_equal(h.coi, coi) and np.array_equal(h.freq, freq)
    assert np.array_equal(h.coherence(), WCT)
    assert np.array_equal(h.phase(), aWCT)
    for rows, cols in WINDOWS + [(slice(None, None, 3), slice(None, None, 3)),
                                 (slice(None), slice(None, None, 64)),
                                 (slice(7, 100, 9), slice(-70001, -3, 1001))]:
        w, a = h.window(rows, cols)
        assert np.array_equal(w, WCT[rows, cols]) and np.array_equal(a, aWCT[rows, cols]), (rows, cols)

    sig95 = sig95_with_gaps(h, WCT)
    check_reductions(h, WCT, aWCT, sig95)

    per = h.period
    calls = [lambda: h.global_coherence(),
             lambda: h.global_coherence(inside_coi=True, sig95=sig95),
             lambda: h.significant_fraction(sig95),
             lambda: h.mean_phase(sig95=sig95),
             lambda: h.mean_phase(per[10], per[100], inside_coi=False, per_scale=True),
             lambda: h.scale_avg(per[20], per[60])]
    first = [f() for f in calls]
    for f, a in zip(calls, first):
        b = f()
        for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            assert np.array_equal(x, y, equal_nan=True)

    # 8 seeded surrogate pairs at the real geometry run on the same engine; the handle survives
    sig = h.significance(mc_count=8, cache=False, seed=5, progress=False)
    assert sig.shape == (J + 1,)
    for f, a in zip(calls, first):
        b = f()
        for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            assert np.array_equal(x, y, equal_nan=True)
    assert np.array_equal(h.coherence(), WCT)
    h.release()
