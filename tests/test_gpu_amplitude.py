"""Amplitude invariance on the device at the configs' geometries: the checks of
tests/test_emu_amplitude.py (its module notes give the exponent ranges), one exponent pair per
product near each end of its range.  Only array equality and host arithmetic: no reference
transform.

  * config 2 (Morlet, 2^20 points, fp64): 50 of its 256 scales, which run the dense, overlap-save
    and expansion classes with both coarse launches; the plan and the kernels launched must not
    move;
  * config 3 (Paul(4) and DOG(2), 2^18 points, fp32);
  * config 4 (two and three series of 2^18 points): xwt, wct, partial_wct, multiple_wct, and the
    resident pair and triple in fp64 and fp32 with 8 surrogate units of counts and clusters;
  * a slice of config 5's batch (16 channels of 2^16 points, fp32).
"""
import numpy as np
import pytest

import test_emu_amplitude as A
import test_gpu_fp64_row_parity as rp64
import workloads as wl

pytestmark = pytest.mark.gpu
F64, F32 = A.F64, A.F32


@pytest.fixture(scope="module")
def eng():
    from pycwt_b200 import _engine
    e = _engine.default_engine()
    yield e


@pytest.fixture(scope="module")
def api():
    import pycwt_b200
    return pycwt_b200


def kernel_names(prof):
    """Names (without spaces) of the kernels of a profile, the forward transform's excluded."""
    return {p["name"].replace(" ", "") for p in prof if not p["name"].startswith("fwd:")}


def expected_kernels(plan):
    """The kernels a config 2 plan launches: the exact classes (test_gpu_fp64_row_parity), the
    overlap-save rows, and the expansion rows with their coarse launches."""
    want = set(rp64.expected_kernels([c for c in plan if c >= 0], 20))
    if A.overlap_save(plan):
        want.add("OsBody<4>")
    if A.coarse_pair(plan):
        want |= {"coarse:CoarseABody<double>", "coarse:CoarseBBody<double>"}
    if A.coarse_ragged(plan):
        want.add("coarse:CoarseRowsBody<double>")
    return want


def test_config2_rows(eng):
    """Every second of config 2's first 48 scales (its dense and overlap-save rows) and every eighth
    beyond (the expansion rows): the plan pinned by class, and the same kernels launched at 2^900,
    2^-900 and 2^0, each expansion kernel among them."""
    sj = wl.config2_scales()
    sj = np.concatenate([sj[:48:2], sj[48::8]])
    cell = A.cwt_cell("config 2", wl.C2["n"], sj, A.MORLET, 6.0, (F64,),
                      [A.dense(20), A.overlap_save, A.expansion, A.coarse_ragged, A.coarse_pair])
    x = wl.config2_signal()
    plan = A.check_cwt_cell(eng, cell, F64, x=x)
    names = []
    for k in (0,) + A.ends(1, F64):
        eng.profile_begin()
        try:
            eng.cwt(np.ldexp(x, k), 1.0, sj, A.MORLET, 6.0, F64)
        finally:
            prof = eng.profile_end()
        assert eng.last_plan(len(sj)) == plan, k
        names.append(kernel_names(prof))
    print("  config 2 plan:", plan)
    print("  kernels:", sorted(names[0]))
    assert names[1] == names[0] and names[2] == names[0], names
    got = names[0]
    want = expected_kernels(plan)
    assert want <= got, sorted(want - got)
    assert any(n.startswith("ExpandMmaBody<") for n in got), sorted(got)
    exact = rp64.launched(prof)
    assert exact == rp64.expected_kernels([c for c in plan if c >= 0], 20), (sorted(exact), plan)


@pytest.mark.parametrize("fam,par,key", [(A.PAUL, 4.0, "paul"), (A.DOG, 2.0, "dog")])
def test_config3(eng, fam, par, key):
    c = wl.C3[key]
    sj = wl.geometric_scales(c["s0"], c["dj"], c["J"])
    cell = A.cwt_cell("config 3 " + key, wl.C3["n"], sj, fam, par, (F32,), [])
    A.check_cwt_cell(eng, cell, F32, x=wl.config3_signal().astype(np.float64))


KW4 = dict(dj=wl.C4["dj"], s0=wl.C4["s0"], J=wl.C4["J"])


def _series(count):
    y1, y2 = wl.config4_signals()
    if count == 2:
        return [y1, y2]
    return [y1, y2, wl.chirp(wl.C4["n"], 1.9) + 0.5 * np.random.RandomState(3).randn(wl.C4["n"])]


@pytest.mark.parametrize("prec", [F64, F32])
def test_config4_xwt_wct(api, prec):
    y = _series(2)
    A.check_xwt(api, y, KW4, prec, A.pair_exps(A.XWT, prec))
    A.check_wct(api, y, KW4, prec, A.coh_exps(2))


@pytest.mark.parametrize("prec", [F64, F32])
def test_config4_partial_multiple(api, prec):
    A.check_wct3(api, _series(3), KW4, prec, A.coh_exps(3))


@pytest.mark.parametrize("prec", [F64, F32])
def test_config4_resident_pair(api, eng, prec):
    A.check_resident_coherence(api, eng, _series(2), KW4, prec, A.coh_exps(2)[2:], M=8)


@pytest.mark.parametrize("prec", [F64, F32])
def test_config4_resident_triple(api, eng, prec):
    A.check_resident_coherence(api, eng, _series(3), KW4, prec, A.coh_exps(3)[2:], M=8)


@pytest.mark.parametrize("prec", [F64, F32])
def test_config4_resident_cross(api, eng, prec):
    A.check_resident_cross(api, eng, _series(2), KW4, prec, A.pair_exps(A.XWT, prec))


def test_config5_batch_slice(eng):
    X = wl.config5_channels(0, 16)
    sj = wl.geometric_scales(wl.C5["s0"], wl.C5["dj"], wl.C5["J"])
    k = A.RANGE[(2, F32)]
    A.check_cwt_batch(eng, X, sj, A.MORLET, 6.0, F32, [tuple(k if c % 2 else 1 - k for c in range(16))])
