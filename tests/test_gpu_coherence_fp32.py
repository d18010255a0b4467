"""fp32 coherence on the GPU at config 4 size against the fp64 engine (which the other GPU tests
hold to the reference at 1e-10): the cross-wavelet transform, its angle and the coherence on
every row, and the Monte-Carlo histograms and levels at the real geometry in both RNG modes."""
import numpy as np
import pytest

from test_emu_coherence_fp32 import WCT_BOUND, check_fp32_coherence, check_fp32_histograms

pytestmark = pytest.mark.gpu

DT, DJ, S0, J = 1.0, 1 / 12, 2.0, 144


@pytest.fixture(scope="module")
def pycwt():
    import pycwt_b200
    return pycwt_b200


def test_config4_fp32_every_row(pycwt):
    import workloads
    y1, y2 = workloads.config4_signals()
    W64 = pycwt.xwt(y1, y2, DT, dj=DJ, s0=S0, J=J)[0]
    W32 = pycwt.xwt(y1, y2, DT, dj=DJ, s0=S0, J=J, precision='fp32')[0]
    assert W32.shape == (145, 2 ** 18) and W32.dtype == np.complex128
    WCT64, aWCT64 = pycwt.wct(y1, y2, DT, dj=DJ, s0=S0, J=J, sig=False)[:2]
    WCT32, aWCT32 = pycwt.wct(y1, y2, DT, dj=DJ, s0=S0, J=J, sig=False, precision='fp32')[:2]
    assert WCT32.dtype == np.float64 and aWCT32.dtype == np.float64
    for i in range(W64.shape[0]):
        check_fp32_coherence(W32[i], aWCT32[i], WCT32[i], W64[i], aWCT64[i], WCT64[i])
    assert WCT_BOUND <= 1e-3


@pytest.mark.parametrize("seeded", [False, True])
def test_config4_monte_carlo_fp32(pycwt, seeded):
    from pycwt_b200 import _engine, wavelet as wv
    m = pycwt.Morlet(6)
    prob = wv._mc_problem(DT, DJ, S0, J, m)
    assert prob["N"] == 49152 and prob["sj"].size == 145
    h = {}
    for p in (_engine.F64, _engine.F32):
        if seeded:
            h[p] = wv._mc_histogram_seeded(prob, DT, DJ, m, 17, 0, 8, precision=p)
        else:
            noise = np.random.RandomState(17).randn(8, 2, prob["N"])
            h[p] = wv._mc_histogram(prob, DT, DJ, m, lambda i: (noise[i, 0], noise[i, 1]), range(8),
                                    precision=p)
    check_fp32_histograms(h[_engine.F32], h[_engine.F64], prob)
