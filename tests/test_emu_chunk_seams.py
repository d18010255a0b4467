"""The engine's chunk seams that are cheap on the host emulation (tests/_emu), so that the CPU suite
holds them:

  * the Bluestein rows past the launch row limit: fft_c2c of 65535, 65536 and 70000 rows of 3 points
    (L = 8), whose chunks blue_chunk_rows caps at 65535 rows, against numpy (test_gpu_chunk_seams.py);
  * the seeded-draw hooks (mc_surrogates, mc_surrogates3, mc_phase_surrogates,
    mc_ar1_series_surrogates) across their launches of MAX_ROWS / nser units (MAX_ROWS for the AR(1)
    hook, one launch per series): the launch record shows the seam, one call equals two calls split
    there, and the units on both sides of it equal Philox restatements (the normal noise here, the
    phase and AR(1) units those of test_emu_surrogate_significance.py and test_emu_cross_test.py);
  * launch groups of the two-kernel classes (CWTB_GROUP = 3 with one and two chains) on an Np = 2^16
    cell: seam rows against the longdouble reference and every row bit for bit against one group;
  * the calls whose launches take one row per scale refuse more scales than a launch has rows, at
    the call, with the limit in the message.
"""
import numpy as np
import pytest

import test_emu_cross_test as X
import test_emu_surrogate_significance as T
import test_gpu_chunk_seams as G
from test_emu_overlap_save import emu_lib, make_engine

MAX_ROWS = G.MAX_ROWS
N0 = 6


@pytest.fixture(scope="module")
def emu():
    eng = make_engine(emu_lib())
    assert "emulation" in eng.version()
    yield eng
    eng.close()


@pytest.mark.parametrize("rows", [65535, 65536, 70000])
def test_bluestein_row_cap(emu, rows):
    """More rows of a length that is not 2^k than one launch takes: chunks of at most 65535 rows."""
    G.check_bluestein_rows(emu, 3, rows)


def _drawn(eng, draw, first, count):
    return G.profiled(eng, lambda: draw(first, count))


def normals_host(seed, unit, ser, nser, n):
    """Series `ser` of unit `unit` of the seeded normal noise (kernels.cuh: NoiseBody): pair j of
    samples from Philox4x32-10 of the counter words (j lo, j hi, unit lo, c3) with
    c3 = (unit hi << 1) | ser for pairs, 2^31 | (unit hi << 2) | ser for triples, through Box-Muller."""
    j = np.arange((n + 1) // 2, dtype=np.uint64)
    hi = unit >> 32
    c3 = (hi << 1) | ser if nser == 2 else 0x80000000 | (hi << 2) | ser
    o = T.philox4x32_10(j, j >> np.uint64(32), unit & 0xFFFFFFFF, c3, seed)
    u1 = ((o[0] >> np.uint64(5)).astype(float) * 67108864.0 + (o[1] >> np.uint64(6)).astype(float) + 0.5) \
        / 9007199254740992.0
    u2 = ((o[2] >> np.uint64(5)).astype(float) * 67108864.0 + (o[3] >> np.uint64(6)).astype(float) + 0.5) \
        / 9007199254740992.0
    r = np.sqrt(-2.0 * np.log(u1))
    e = np.empty(2 * j.size)
    e[0::2] = r * np.cos(2 * np.pi * u2)
    e[1::2] = r * np.sin(2 * np.pi * u2)
    return e[:n]


# The split of 40000 units into two calls away from the seams is test_emu_host_paths.py's
# test_surrogates_of_more_units_than_one_launch_has_rows; here the split falls on the seam, the
# launch record shows it, and the units on both sides of it are checked against a restatement.
@pytest.mark.parametrize("nser", [2, 3])
def test_normal_noise_hook_seam(emu, nser):
    draw = (lambda u0, n: emu.mc_surrogates(11, u0, n, N0)) if nser == 2 else \
        (lambda u0, n: emu.mc_surrogates3(11, u0, n, N0))
    batch = MAX_ROWS // nser
    whole, prof = _drawn(emu, draw, 0, batch + 2)
    assert G.launches(prof, "NoiseBody") == (2, nser * (batch + 2)), prof
    assert np.array_equal(whole, np.concatenate([draw(0, batch), draw(batch, 2)]))
    for u in (batch - 1, batch, batch + 1):
        ref = np.array([normals_host(11, u, r, nser, N0) for r in range(nser)])
        # sincospi on the device, cos / sin of 2 pi u2 here: a few ulp of r <= 8.6
        assert np.abs(whole[u] - ref).max() <= 1e-14, u


@pytest.mark.parametrize("groups", [(0, 0), (0, 0, 1)], ids=["pair", "triple"])
def test_phase_hook_seam(emu, groups):
    nser = len(groups)
    x = np.random.RandomState(6).randn(nser, N0)
    draw = lambda u0, n: emu.mc_phase_surrogates(x, groups, 11, u0, n)   # noqa: E731
    batch = MAX_ROWS // nser
    whole, prof = _drawn(emu, draw, 0, batch + 2)
    assert G.launches(prof, "PhaseRotBody", tagged=True) == (2, nser * (batch + 2)), prof
    assert np.array_equal(whole, np.concatenate([draw(0, batch), draw(batch, 2)]))
    for u in (batch - 1, batch, batch + 1):
        ref = np.array([T.surrogate(x[r], 11, u, groups[r]) for r in range(nser)])
        assert np.abs(whole[u] - ref).max() <= 1e-13 * np.abs(x).max(), u


@pytest.mark.parametrize("nser", [1, 3])
def test_ar1_hook_seam(emu, nser):
    g, m, sigma = (0.7, -0.4, 0.55)[:nser], (0.0, 3.0, -1.0)[:nser], (1.0, 2.5, 0.75)[:nser]
    draw = lambda u0, n: emu.mc_ar1_series_surrogates(g, m, sigma, 5, u0, n, N0)   # noqa: E731
    batch = MAX_ROWS
    whole, prof = _drawn(emu, draw, 0, batch + 2)
    assert G.launches(prof, "Ar1BlockBody", tagged=True) == (2 * nser, nser * (batch + 2)), prof
    assert np.array_equal(whole, np.concatenate([draw(0, batch), draw(batch, 2)]))
    for u in (batch - 1, batch, batch + 1):
        for r in range(nser):
            ref = X.ar1_host(g[r], m[r], sigma[r], 5, u, N0, r)
            tol = 16 * np.finfo(float).eps * sigma[r] / (1 - abs(g[r])) * \
                max(1.0, float(np.abs(ref - m[r]).max()) / sigma[r])
            assert float(np.abs(whole[u, r].astype(np.longdouble) - ref).max()) <= tol, (u, r)


@pytest.mark.parametrize("chains", [1, 2])
def test_two_kernel_launch_groups(chains):
    G.check_groups(3, chains, G.F64, emu_lib())


def test_refusals_name_the_limit(emu):
    """One row per scale in a launch: more scales than 65535 (60000 rows of a transform) are refused
    at the call, with the limit in the message."""
    from pycwt_b200._engine import EngineError
    x = np.random.RandomState(1).randn(40)
    with pytest.raises(EngineError, match="at most 60000"):
        emu.cwt(x, 1.0, np.full(60001, 2.0), 0, 6.0)
    with pytest.raises(EngineError, match="65535 scales"):
        emu.smooth(np.zeros((MAX_ROWS + 1, 4)), 1.0, np.full(MAX_ROWS + 1, 2.0), 3)
    with pytest.raises(EngineError, match="65535 scales"):
        emu.cluster_label_bits(np.zeros((MAX_ROWS + 1, 1), dtype=np.uint32), 4,
                               np.ones(MAX_ROWS + 1, dtype=np.uint64))
