"""Coarse transforms of the expansion rows (kernels.cuh: CoarseRowsBody, CoarseABody, CoarseBBody)
on the host-emulation build of the kernels.

The coarse spectra are formed while the transforms fill their tiles, and every coarse length runs
in one ragged launch (lengths up to 1024) or one launch pair (longer ones).  Checked:
  * expansion rows (plan code -log2(Nc)) of Morlet and DOG match the oracle within the expansion
    tolerance, at an odd n0 and at n0 = Np, in fp64 and fp32, and each such row of Morlet, DOG and
    Paul matches the exact path (expand_eps = 0) row by row;
  * the coarse transforms take three launches whatever the number of coarse lengths;
  * batched channels give each channel's single-channel rows bit for bit;
  * the cross-wavelet epilogue on a plan with expansion rows.
"""
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import cwt_oracle as orc

N0 = 50001                                    # Np = 2^16
SJ = 2.0 * 2 ** (np.arange(0, 60) / 6.0)      # s = 2 .. 2^10.8: coarse lengths 2^7 .. 2^13
TOL = {0: 2e-13, 1: 2e-6}                     # F64, F32: expansion tolerance over max|W|


@pytest.fixture(scope="module")
def emu():
    from pycwt_b200 import build as _build, _engine
    lib = _build.build_emulation(os.path.join(ROOT, "tests", "_emu"))
    eng = _engine.Engine(0, lib_path=lib)
    assert "emulation" in eng.version()
    yield eng
    eng.close()


def _signal(n0, seed=7):
    rs = np.random.RandomState(seed)
    t = np.arange(n0) / n0
    return np.sin(2 * np.pi * (40 * t + 3000 * t ** 2)) + 0.3 * rs.randn(n0)


def _expansion_rows(plan):
    return [j for j, p in enumerate(plan) if p < -2]


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("n0", [N0, 2 ** 16])
@pytest.mark.parametrize("fam,ref,par", [(0, orc.Morlet(6), 6.0), (2, orc.DOG(2), 2.0), (1, orc.Paul(4), 4.0)])
def test_rows_match_oracle_and_exact_path(emu, n0, fam, ref, par, prec):
    x = _signal(n0)
    W = emu.cwt(x, 1.0, SJ, fam, par, prec)
    plan = emu.last_plan(len(SJ))
    rows = _expansion_rows(plan)
    assert len(rows) >= 20, plan
    wmax = np.abs(W).max()
    if fam != 1:   # (the oracle's Paul overflows at the largest of these scales)
        Wr = orc.cwt(x, 1.0, wavelet=ref, freqs=1 / (ref.flambda() * SJ))[0]
        assert max(np.abs(W[j] - Wr[j]).max() for j in rows) < TOL[prec] * np.abs(Wr).max()
    emu.set_expand_eps(0, 0)
    try:
        We = emu.cwt(x, 1.0, SJ, fam, par, prec)
        assert not _expansion_rows(emu.last_plan(len(SJ)))
    finally:
        emu.set_expand_eps()
    for j in rows:
        rmax = np.abs(We[j]).max()
        assert np.abs(W[j] - We[j]).max() <= TOL[prec] * max(rmax, 1e-3 * wmax), j


def test_coarse_launch_count(emu):
    # the launches of a transform with expansion rows, less those of the same transform without them:
    # the coarse transforms (three launches) plus one expansion launch per tap count
    x = _signal(N0)
    for fam, par in ((0, 6.0), (2, 2.0)):
        emu.cwt(x, 1.0, SJ, fam, par)
        plan = emu.last_plan(len(SJ))
        rows = _expansion_rows(plan)
        with_exp = emu.last_launch_count()
        taps_launches = with_exp - _launches_without(emu, x, fam, par, rows) - 3
        assert 1 <= taps_launches <= 5, (with_exp, taps_launches)
        lengths = {-plan[j] for j in rows}
        assert min(lengths) <= 10 < max(lengths) and len(lengths) > 3, plan   # both kinds, several lengths


def _launches_without(emu, x, fam, par, rows):
    keep = [j for j in range(len(SJ)) if j not in rows]
    emu.cwt(x, 1.0, SJ[keep], fam, par)
    assert not _expansion_rows(emu.last_plan(len(keep)))
    return emu.last_launch_count()


@pytest.mark.parametrize("prec", [0, 1])
def test_batched_channels(emu, prec):
    n0 = 20001
    X = np.stack([_signal(n0, seed) for seed in (1, 2, 3)])
    _, W = emu.cwt_batch(X, 1.0, SJ, 0, 6.0, precision=prec, want_w=True)
    for ch in range(len(X)):
        assert np.array_equal(W[ch], emu.cwt(X[ch], 1.0, SJ, 0, 6.0, prec))
        assert _expansion_rows(emu.last_plan(len(SJ)))


def test_cross_product_epilogue(emu):
    from pycwt_b200 import _engine
    y1, y2 = _signal(N0, 1), _signal(N0, 2)
    for prec in (_engine.F64, _engine.F32):
        W12 = emu.xwt(y1, y2, 1.0, SJ, _engine.MORLET, 6.0, prec)
        W1 = emu.cwt(y1, 1.0, SJ, _engine.MORLET, 6.0, prec)
        assert _expansion_rows(emu.last_plan(len(SJ)))
        W2 = emu.cwt(y2, 1.0, SJ, _engine.MORLET, 6.0, prec)
        ref = W1 * np.conj(W2)
        tol = 1e-12 if prec == _engine.F64 else 1e-5
        assert np.abs(W12 - ref).max() <= tol * np.abs(ref).max()
