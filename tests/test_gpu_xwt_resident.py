"""Resident cross-wavelet transform (`xwt_resident`) at config 4 on the GPU (two 2^18-point
series, s0 = 2, dj = 1/12, J = 144), in fp64 and fp32: the fetch bit-identical to `xwt`, every
reduction against numpy on the fetch, repeated reductions bit-identical, also after a seeded
Monte-Carlo run of 8 surrogate pairs on the same engine.  And the complex-field additions of
`ResidentTransform` on config 2's 2^20-point fp64 transform and config 3's Paul(4) in fp32."""
import numpy as np
import pytest

from test_emu_coherence_resident import WINDOWS
from test_emu_xwt_resident import (EXTRA_WINDOWS, check_cross_reductions, check_transform_additions,
                                   signif_with_gaps)

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


def _same(a, b):
    for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
        assert np.array_equal(x, y, equal_nan=True)


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_config4_resident_cross_spectrum(pycwt, signals, precision):
    y1, y2 = signals
    kw = dict(dj=DJ, s0=S0, J=J, precision=precision)
    W12, coi, freq, signif = pycwt.xwt(y1, y2, DT, **kw)
    W12 = np.array(W12)                                # own copy: the pinned buffers are pooled
    h = pycwt.xwt_resident(y1, y2, DT, **kw)
    assert h.shape == (J + 1, y1.size)
    assert np.array_equal(h.coi, coi) and np.array_equal(h.freq, freq)
    assert np.array_equal(h.signif, signif)
    assert np.array_equal(h.cross_spectrum(), W12)
    for rows, cols in WINDOWS + EXTRA_WINDOWS + [(slice(None), slice(None, None, 64)),
                                                 (slice(7, 100, 9), slice(-70001, -3, 1001))]:
        assert np.array_equal(h.window(rows, cols), W12[rows, cols]), (rows, cols)

    check_cross_reductions(h, W12, signif_with_gaps(W12))
    check_cross_reductions(h, W12, np.sqrt(h.signif))

    per = h.period
    thr = signif_with_gaps(W12)
    calls = [lambda: h.global_power(),
             lambda: h.global_power(inside_coi=True, signif=thr),
             lambda: h.significant_fraction(thr),
             lambda: h.mean_phase(signif=np.sqrt(h.signif)),
             lambda: h.mean_phase(per[10], per[100], inside_coi=False, per_scale=True),
             lambda: h.scale_avg(per[48], per[60]),
             lambda: h.window(slice(None, None, 3), slice(None, None, 3))]
    first = [f() for f in calls]
    for f, a in zip(calls, first):
        _same(a, f())

    # 8 seeded surrogate pairs at the real geometry run on the same engine; the handle survives
    sig = pycwt.wct(y1, y2, DT, sig=True, mc_count=8, cache=False, seed=5, progress=False, **kw)[4]
    assert sig.shape == (J + 1,)
    for f, a in zip(calls, first):
        _same(a, f())
    assert np.array_equal(h.cross_spectrum(), W12)
    h.release()


def test_config2_resident_transform_additions(pycwt):
    import workloads as wl
    x, sj = wl.config2_signal(), wl.config2_scales()
    r = pycwt.cwt_resident(x, wl.C2["dt"], dj=wl.C2["dj"], s0=wl.C2["s0"], J=wl.C2["J"])
    assert r.shape == (sj.size, x.size)
    rows = slice(0, sj.size, 8)                        # a row subset of W for the numpy side
    Wsub = r.window(rows)
    assert np.array_equal(Wsub[5], r.window(slice(40, 41))[0])      # gather == whole-row copy
    check_transform_additions(_RowSubset(r, rows), Wsub)


def test_config3_paul_fp32_resident_transform_additions(pycwt, monkeypatch):
    import workloads as wl
    monkeypatch.setenv("CWTB_PRECISION", "fp32")
    p = wl.C3["paul"]
    r = pycwt.cwt_resident(wl.config3_signal(), wl.C3["dt"], dj=p["dj"], s0=p["s0"], J=p["J"],
                           wavelet=pycwt.Paul(p["m"]))
    W = np.array(r.wave())
    check_transform_additions(r, W)


class _RowSubset(object):
    """A ResidentTransform seen through every `step`-th row: the numpy side of the checks holds
    only those rows of a 2^20-point transform (host memory); thresholds are spread over all rows
    with +inf on the others, so the per-row results of the subset are the handle's."""

    def __init__(self, r, rows):
        self.r = r
        self.rows = rows
        self.idx = np.arange(*rows.indices(r.shape[0]))
        self.scales = np.asarray(r.scales)[self.idx]
        self.period = r.period[self.idx]
        self.coi = r.coi
        self.n0 = r.n0
        self.shape = (self.idx.size, r.n0)

    def coi_ranges(self):
        lo, hi = self.r.coi_ranges()
        return lo[self.idx], hi[self.idx]

    def _full(self, signif):
        t = np.full(self.r.shape[0], np.inf)
        signif = np.asarray(signif, dtype=float)
        if signif.shape != self.idx.shape:
            t = np.full(self.r.shape[0] + 1, np.nan)       # wrong length on the handle too
        else:
            t[self.idx] = signif
        return t

    def window(self, rows=slice(None), cols=slice(None)):
        return self.r.window(self.rows, cols)[rows]

    def global_power(self, inside_coi=False, signif=None):
        if signif is None:
            return self.r.global_power(inside_coi=inside_coi)[self.idx]
        return self.r.global_power(inside_coi=inside_coi, signif=self._full(signif))[self.idx]

    def significant_fraction(self, signif):
        return self.r.significant_fraction(self._full(signif))[self.idx]
