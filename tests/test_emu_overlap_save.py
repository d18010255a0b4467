"""Overlap-save rows (kernels.cuh: OsBody) on the host-emulation build of the kernels.  The checks are
`check_*` functions of an engine: tests/test_gpu_row_parity.py runs them on the GPU.

Rows whose band stays clear of Nyquist have a short impulse response; the planner truncates it and
convolves block by block instead of running the two-kernel exact path (last_plan code -2).  Checked:
  * Morlet and DOG rows that take the class match the oracle within 1e-14 of max|W|, with an odd n0
    (blocks that reach past the signal read the zero padding) and with n0 = Np (the first and last
    blocks wrap around to real samples at the other end);
  * rows whose band reaches Nyquist, and Paul rows, keep their path;
  * the class equals the path it replaces (CWTB_OS=0) row by row;
  * re-planning: a context with the switch off, a change of geometry and back, and a plan whose
    expansion weight tables are new while every overlap-save candidate is rejected;
  * the cross-wavelet epilogue and the resident products on a plan that uses the class.
"""
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import cwt_oracle as orc

OS = -2
N0 = 50001                                    # Np = 2^16
SJ = 2.0 * 2 ** (np.arange(0, 28) / 4.0)      # s = 2 .. 25: Nyquist-cut, overlap-save, expansion rows


def make_engine(lib_path=None, **env):
    """An engine whose context reads `env` (CWTB_* switches) at creation; lib_path None: the
    library the package loads."""
    from pycwt_b200 import _engine
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return _engine.Engine(0, lib_path=lib_path)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def emu_lib():
    from pycwt_b200 import build as _build
    return _build.build_emulation(os.path.join(ROOT, "tests", "_emu"))


def _engine(os_on):
    eng = make_engine(emu_lib(), CWTB_OS="1" if os_on else "0")
    assert "emulation" in eng.version()
    return eng


@pytest.fixture(scope="module")
def emu():
    eng = _engine(True)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def emu_off():
    eng = _engine(False)
    yield eng
    eng.close()


def _signal(n0):
    rs = np.random.RandomState(7)
    t = np.arange(n0) / n0
    return np.sin(2 * np.pi * (40 * t + 3000 * t ** 2)) + 0.3 * rs.randn(n0)


@pytest.fixture(scope="module")
def signal():
    return _signal(N0)


def check_rows_match_oracle(eng, n0, fam, ref, par):
    signal = _signal(n0)
    W = eng.cwt(signal, 1.0, SJ, fam, par)
    plan = eng.last_plan(len(SJ))
    rows = [j for j, p in enumerate(plan) if p == OS]
    assert len(rows) >= 6, plan
    assert plan[0] != OS            # s = 2: the band reaches Nyquist
    Wr = orc.cwt(signal, 1.0, wavelet=ref, freqs=1 / (ref.flambda() * SJ))[0]
    wmax = np.abs(Wr).max()
    for j in rows:
        assert np.abs(W[j] - Wr[j]).max() < 1e-14 * wmax, (j, np.abs(W[j] - Wr[j]).max() / wmax)
    assert np.abs(W - Wr).max() < 2e-13 * wmax
    return W, plan


def check_nyquist_and_paul_rows_rejected(eng, signal):
    eng.cwt(signal, 1.0, np.array([2.0, 2.5, 3.0]), 0, 6.0)
    assert OS not in eng.last_plan(3)
    eng.cwt(signal, 1.0, SJ, 1, 4.0)
    assert OS not in eng.last_plan(len(SJ))


def check_equals_replaced_path_per_row(eng, eng_off, signal, fam, par, sj=SJ):
    W = eng.cwt(signal, 1.0, sj, fam, par)
    plan = eng.last_plan(len(sj))
    W0 = eng_off.cwt(signal, 1.0, sj, fam, par)
    assert OS in plan and OS not in eng_off.last_plan(len(sj))
    for j, p in enumerate(plan):
        d = np.abs(W[j] - W0[j]).max() / np.abs(W0[j]).max()
        if p == OS:
            assert d < 1e-14, (j, d)
        else:
            assert d == 0, (j, p, d)
    return W, plan


def check_replanning(eng, eng_off, signal):
    W1 = eng.cwt(signal, 1.0, SJ, 0, 6.0)
    p1 = eng.last_plan(len(SJ))
    # another geometry on the same context: shorter odd signal, Np = 2^14
    y = signal[:9001]
    W2 = eng.cwt(y, 1.0, SJ[:20], 0, 6.0)
    p2 = eng.last_plan(20)
    assert OS in p2
    m = orc.Morlet(6)
    Wr2 = orc.cwt(y, 1.0, wavelet=m, freqs=1 / (m.flambda() * SJ[:20]))[0]
    assert np.abs(W2 - Wr2).max() < 1e-14 * np.abs(Wr2).max()
    # back to the first geometry: the same plan and the same numbers
    assert np.array_equal(eng.cwt(signal, 1.0, SJ, 0, 6.0), W1)
    assert eng.last_plan(len(SJ)) == p1
    # the switch off: the plan of the parent paths
    eng_off.cwt(signal, 1.0, SJ, 0, 6.0)
    assert OS not in eng_off.last_plan(len(SJ))


def check_batched_channels_equal_single_channel(eng, signal):
    rs = np.random.RandomState(12)
    X = np.stack([signal, rs.randn(signal.size)])
    _, W = eng.cwt_batch(X, 1.0, SJ, 0, 6.0, precision=0, want_w=True)
    for ch in range(2):
        assert np.array_equal(W[ch], eng.cwt(X[ch], 1.0, SJ, 0, 6.0))
        assert OS in eng.last_plan(len(SJ))


def check_new_weight_tables_survive_rejected_candidates(eng_off, signal, lib_path=None, **env):
    """CWTB_WTAB_MB=0 starts the expansion weight cache over on every plan.  The Paul plan has new
    tables and overlap-save candidates (bands clear of Nyquist) that are all rejected: the tables must
    still reach the device, whatever the planning of the candidates' impulse responses does."""
    eng = make_engine(lib_path, CWTB_WTAB_MB="0", **env)
    try:
        eng.cwt(signal, 1.0, SJ, 0, 6.0)
        W = eng.cwt(signal, 1.0, SJ, 1, 4.0)
        plan = eng.last_plan(len(SJ))
        assert OS not in plan and min(plan) < -2, plan
        assert np.array_equal(W, eng_off.cwt(signal, 1.0, SJ, 1, 4.0))
    finally:
        eng.close()


def check_cross_product_epilogue(eng, eng_off, signal):
    rs = np.random.RandomState(11)
    y2 = signal + 0.5 * rs.randn(signal.size)
    X = eng.xwt(signal, y2, 1.0, SJ, 0, 6.0)
    assert OS in eng.last_plan(len(SJ))
    X0 = eng_off.xwt(signal, y2, 1.0, SJ, 0, 6.0)
    for j in range(len(SJ)):
        assert np.abs(X[j] - X0[j]).max() < 2e-14 * np.abs(X0[j]).max(), j
    return X, y2


def check_resident_products(eng, eng_off, signal):
    from pycwt_b200 import cwt_resident
    kw = dict(dj=0.25, s0=2.0, J=27, wavelet="morlet")
    r = cwt_resident(signal, 1.0, engine=eng, **kw)
    assert OS in eng.last_plan(28)
    W = r.wave()
    gp, sap, ic = r.global_power(), r.scale_avg_power(4.0, 16.0), r.icwt()
    r0 = cwt_resident(signal, 1.0, engine=eng_off, **kw)
    W0 = r0.wave()
    assert np.abs(W - W0).max() < 1e-14 * np.abs(W0).max()
    np.testing.assert_allclose(gp, r0.global_power(), rtol=1e-12)
    np.testing.assert_allclose(sap, r0.scale_avg_power(4.0, 16.0), rtol=1e-12, atol=1e-12 * np.abs(sap).max())
    np.testing.assert_allclose(ic, r0.icwt(), rtol=0, atol=1e-12 * np.abs(ic).max())


@pytest.mark.parametrize("n0", [N0, 2 ** 16])
@pytest.mark.parametrize("fam,ref,par", [(0, orc.Morlet(6), 6.0), (2, orc.DOG(2), 2.0), (2, orc.DOG(6), 6.0)])
def test_rows_match_oracle(emu, n0, fam, ref, par):
    check_rows_match_oracle(emu, n0, fam, ref, par)


def test_nyquist_and_paul_rows_rejected(emu, signal):
    check_nyquist_and_paul_rows_rejected(emu, signal)


@pytest.mark.parametrize("fam,par", [(0, 6.0), (2, 2.0)])
def test_equals_replaced_path_per_row(emu, emu_off, signal, fam, par):
    check_equals_replaced_path_per_row(emu, emu_off, signal, fam, par)


def test_replanning(emu, emu_off, signal):
    check_replanning(emu, emu_off, signal)


def test_batched_channels_equal_single_channel(emu, signal):
    check_batched_channels_equal_single_channel(emu, signal)


def test_new_weight_tables_survive_rejected_candidates(emu_off, signal):
    check_new_weight_tables_survive_rejected_candidates(emu_off, signal, emu_lib())


def test_cross_product_epilogue(emu, emu_off, signal):
    check_cross_product_epilogue(emu, emu_off, signal)


def test_resident_products(emu, emu_off, signal):
    check_resident_products(emu, emu_off, signal)
