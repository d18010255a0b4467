"""Row-by-row parity of the fp32 engine (precision F32) against a high-precision reference.

The reference is `ref_rows` of test_gpu_row_parity.py in fp64 (its own error, ~1e-15, is far below
the fp32 engine's), fed with the input the engine transforms: x.astype(float32).  Each row j is
measured against
    sigma_j = max(max_n |R_j|, nu_j),   nu_j = ||x||_2 ||F_j||_2 / Np,
F_j = sqrt(s_j w1 Np) conj(psi_ft(s_j omega)) the row's response: nu_j is the row's rms response to a
white input of the signal's energy, the level at which the rounding of the input's transform spreads
into every row.  A row far outside the band of a chirp stays checkable without an exception; for white
noise sigma_j = max_n |R_j| and the metric is row_err's.

Covered, each cell pinned to its plan (last_plan) and, on the device, to its launches:
  * the scalar expansion kernel ExpandBody<float, 6 | 8 | 10> (and its cross-product epilogue) for
    R = Np / Nc = 8 .. 2^14, both below and above the 256-thread CTA, n0 = Np, Np - 1, Np - 2, Np - 3,
    Np / 2 + 1;
  * its coarse transforms: CoarseRowsBody<float> (Nc = 2^6 .. 2^10), CoarseABody / CoarseBBody<float>
    (the register-resident K1 = 2 .. 16 tiles of Nc = 2^11 .. 2^14, longer grids, and Nc = 2^20 at
    Np = 2^23, the largest coarse length the planner gives);
  * the exact classes with the expansion off: SingleBody<float, 32 .. 1024>, DirectBody<float, 2 | 4 | 8>,
    two-kernel and dense rows, the three-level dense path (Np = 2^21), TinyBody and small transforms;
  * Morlet(6), DOG(2), DOG(3), Paul(4), the orders whose amplitude is evaluated in double (DOG(10),
    Paul(12), Paul(60)) and a caller-supplied response table;
  * xwt in fp32 against R1 conj(R2);
  * the concurrent stream graph against its serialised run, bit for bit, for every CWTB_PRIO x
    CWTB_CHAINS (check_graph of test_gpu_row_parity.py);
  * cwt_batch (bench config 5): chunked, pipelined and device-resident input, each channel bit-identical
    to its single-channel transform, every row and every power entry against the reference;
  * config 5's real geometry: the power of all 1024 channels, every coefficient of 8 channels.

Bounds, per row class (error / sigma_j), from the worst values measured on an H100 80GB HBM3 at a
700 W power limit (the cells here, the channel batch, config 5 and config 3 of test_gpu_fullsize.py):
  exact rows (TinyBody .. three-level dense)   9.7e-7 (config 3 Paul(4), two-kernel)   bound 3e-6
  expansion rows, eps32 = 2e-7 (8 / 10 taps)   6.8e-7 (config 5)                       bound 1.2e-6
  expansion rows, 6 taps (eps32 = 5e-6)        7.3e-7                                  bound: its eps
  xwt (a product of two rows)                  6.8e-7                                  twice the rows'
  mean power per (channel, scale), relative    7.1e-6 (config 5)                       bound 2e-5
A row's power error is up to 2 (max|R_j| / rms R_j) times its error over sigma_j when the error is a
gain error (the fp32 amplitude), and max / rms is about 5 for the white-noise rows of config 5.
The fp64 engine's Paul rows past xi_b = 1/4 (band half-width over 1/4 of the coarse grid), whose coarse
rounding noise comes back amplified by up to phi^(0) / phi^(xi) <= 64 (engine.cu: expand_gain), have
no fp32 counterpart: with 6 / 8 / 10 taps the planner's cost model always takes the next coarse length
instead (no such row for Paul(2, 4, 12, 60) over s = 16 .. 2^14 at Np = 2^16 and 2^18, nor for Paul(4)
with eps32 up to 1e-5).

Single-edit fp32 mutants on the emulation: the largest change of a row over sigma_j, then the tests
that fail, here and among the existing fp32 tests (test_emu_*, test_gpu_cwt, test_gpu_xwt_wct,
test_gpu_coherence_fp32 and config 3 of test_gpu_fullsize under --emu):
  ExpandBody fp32 RESEED 8 -> 32                  1.4e-6  the 2^20 and Paul(4) cells, the stream graph;
                                                          no existing test
  K1 <= 16 coarse first pass skips a tile column  O(1)    every cell with Nc = 2^11 .. 2^14; 17 existing
  DirectBody step e^{2 pi i NT / N} -> NT + 1     O(1)    every cell with DirectBody rows; 12 existing
  Morlet (float)(f - f0) -> (float)f - (float)f0  5.0e-7  none, here or existing: within the bound
  Paul / DOG amplitude in double from m > 16      3.7e-7  none, here or existing: within the bound

`pytest --emu` runs every cell on the host emulation except the kernel-name assertions and these
GPU-only tests: test_config5_real_geometry (1024 channels x 128 scales of 2^16 points).
"""
import re

import numpy as np
import pytest

import test_emu_overlap_save as osv
import test_gpu_row_parity as rp
from oracle import cwt_oracle as orc

MORLET, PAUL, DOG, TABLE = 0, 1, 2, 3
F32 = 1
EPS32 = 2e-7            # default fp32 expansion tolerance (engine set_expand_eps)
# per-row bounds (error / sigma_j)
EXACT32 = 3e-6
EXPAND32 = 1.2e-6      # tight enough to see ExpandBody's fp32 re-seeding interval go from 8 to 32 steps
POWER32 = 2e-5          # relative error of a row's mean power


# ------------------------------------------------------------------------------------------------
# reference and error model
# ------------------------------------------------------------------------------------------------
def ref32(x, dt, sj, fam, par, n0=None):
    """Reference rows of the fp32 input x (already rounded) and their sigma_j."""
    x = np.asarray(x, dtype=np.float64)
    Np = orc.next_pow2(x.size)
    R = rp.ref_rows(x, dt, sj, fam, par, n0=n0, dtype=np.float64)
    nx = np.linalg.norm(x)
    nu = np.array([nx * np.linalg.norm(rp.response(Np, dt, s, fam, par, np.float64)) / Np for s in sj])
    return R, np.maximum(np.abs(R).max(axis=1), nu)


def sigma_err(W, R, sig):
    """max_n |W[j] - R[j]| / sigma_j for each row j."""
    W, R = np.asarray(W), np.asarray(R)
    assert W.shape == R.shape, (W.shape, R.shape)
    assert np.isfinite(W).all(), "non-finite coefficients"
    return np.abs(W - R).max(axis=1) / sig


def test_nu_is_white_noise_rms():
    """CPU: nu_j is the rms of the rows of a white input, within a few percent."""
    n = 2 ** 16
    x = np.random.RandomState(3).randn(n)
    sj = 2.0 * 2 ** (np.arange(0, 17) / 4.0)         # s = 2 .. 32: wide bands, many bins per row
    for fam, par in ((MORLET, 6.0), (DOG, 2.0), (PAUL, 4.0)):
        R, sig = ref32(x, 1.0, sj, fam, par)
        nu = np.array([np.linalg.norm(x) * np.linalg.norm(rp.response(n, 1.0, s, fam, par, np.float64)) / n
                       for s in sj])
        rms = np.sqrt((np.abs(R) ** 2).mean(axis=1))
        assert np.abs(rms / nu - 1).max() < 0.03, (fam, rms / nu)
        assert np.array_equal(sig, np.abs(R).max(axis=1))    # white noise: sigma_j = max_n |R_j|


def test_fp64_reference_matches_longdouble():
    """CPU: the fp64 reference agrees with the longdouble one to 1e-13 per row."""
    x = rp.chirp_noise(5000).astype(np.float32)
    sj = 0.7 * 2 ** (np.arange(0, 44) / 4.0)
    for fam, par in ((MORLET, 6.0), (PAUL, 4.0), (DOG, 2.0), (DOG, 3.0), (DOG, 10.0), (PAUL, 12.0)):
        e = rp.row_err(rp.ref_rows(x, 1.0, sj, fam, par, dtype=np.float64), rp.ref_rows(x, 1.0, sj, fam, par))
        assert (e <= 1e-13).all(), (fam, par, e.max())


# ------------------------------------------------------------------------------------------------
# engine and launches
# ------------------------------------------------------------------------------------------------
def _emulated(eng):
    return "emulation" in eng.version()


@pytest.fixture(scope="module")
def eng():
    e = osv.make_engine()
    yield e
    e.close()


def launches(prof):
    """{(taps, epilogue): rows} of the fp32 expansion launches, and the set of the other kernel names."""
    expand, names = {}, set()
    for p in prof:
        m = re.search(r"ExpandBody<float,\s*(\d+)(?:,\s*(\d+))?>", p["name"])
        if m:
            key = (int(m.group(1)), int(m.group(2) or 0))
            expand[key] = expand.get(key, 0) + p["rows"]
        else:
            names.add(re.sub(r"^\w+:", "", p["name"]).replace(" ", ""))
    return expand, names


def expected_kernels(plan, log2N):
    """Names of the fp32 kernels a plan must launch (other than the expansion kernel)."""
    want = set()
    for p in plan:
        if p < -2:
            want.add("CoarseRowsBody<float>" if -p <= 10 else "CoarseABody<float>")
            if -p > 10:
                want.add("CoarseBBody<float>")
        elif p == 0:
            want.add("TinyBody<float>")
        elif p <= 10:
            want.add("SingleBody<float,%d>" % 2 ** p)
        elif p <= 13 and p < log2N:
            want.add("DirectBody<float,%d>" % 2 ** (p - 10))
    return want


# ------------------------------------------------------------------------------------------------
# plan-pinned cells
# ------------------------------------------------------------------------------------------------
# A cell: wavelet, Np, n0 values, scales and the plan of each: (log2 R, taps) for an expansion row,
# log2 K' (0: TinyBody) for an exact row.  `eps`: set_expand_eps(eps32=...) of the cell (0: the
# expansion off) -- a cell with a looser tolerance than the default is bounded by it as well.
def _cell(name, fam, par, log2N, n0s, rows, eps=EPS32, xwt=False, signal=rp.white, table=False):
    return dict(name=name, fam=fam, par=par, log2N=log2N, n0s=n0s, sj=np.array([r[0] for r in rows]),
                plan=[r[1] for r in rows], eps=eps, xwt=xwt, signal=signal, table=table)


NP16 = 2 ** 16
N0_EDGES = [NP16, NP16 - 1, NP16 - 2, NP16 - 3, NP16 // 2 + 1]
CELLS = [
    # R = 8 .. 1024 (Nc = 2^13 .. 2^6: K1 = 8, 4, 2 tiles and every CoarseRowsBody length), 8 and 10 taps
    _cell("morlet R 8..1024, n0 edges", MORLET, 6.0, 16, N0_EDGES,
          [(40.0, (3, 10)), (50.0, (3, 8)), (80.0, (4, 10)), (100.0, (4, 8)), (160.0, (5, 10)), (200.0, (5, 8)),
           (400.0, (6, 8)), (800.0, (7, 8)), (1500.0, (8, 8)), (3000.0, (9, 8)), (6000.0, (10, 8)),
           (8.0, 15), (20.0, 13)]),
    # 6 taps exist only for a looser tolerance
    _cell("6 taps, eps32 = 5e-6", MORLET, 6.0, 16, [NP16, NP16 - 3],
          [(40.0, (3, 8)), (400.0, (5, 6)), (800.0, (6, 6)), (1500.0, (7, 6)), (3000.0, (8, 6)), (6000.0, (9, 6))],
          eps=5e-6),
    # K1 = 16 (Nc = 2^14), longer coarse grids, R = 2^13 and 2^14 (Nc = 128, 64: 32 / 64 rb tiles per row)
    _cell("Np = 2^20, Nc = 2^14 .. 2^17, R = 2^14", MORLET, 6.0, 20, [2 ** 20 - 1],
          [(40.0, (3, 10)), (44.0, (3, 8)), (88.0, (4, 8)), (175.0, (5, 8)), (350.0, (6, 8)), (7e4, (13, 8)),
           (1e5, (14, 8)), (8.0, 20)]),
    # the largest coarse length the planner gives: Nc = 2^20 (coarse grids stop there), R = 8
    _cell("Np = 2^23, Nc = 2^20", MORLET, 6.0, 23, [2 ** 23 - 5], [(40.0, (3, 10)), (45.0, (3, 8))]),
    _cell("DOG(2)", DOG, 2.0, 16, [NP16, NP16 - 1],
          [(40.0, (3, 10)), (80.0, (4, 10)), (160.0, (5, 10)), (320.0, (5, 8)), (640.0, (6, 8)), (2560.0, (8, 8)),
           (5.0, 15), (20.0, 13)], signal=rp.chirp_noise),
    _cell("DOG(3)", DOG, 3.0, 16, [NP16, NP16 - 2],
          [(40.0, (3, 10)), (80.0, (4, 10)), (160.0, (5, 10)), (320.0, (5, 8)), (640.0, (6, 8)), (2560.0, (8, 8)),
           (5.0, 15), (20.0, 13)], signal=rp.chirp_noise),
    _cell("Paul(4)", PAUL, 4.0, 16, [NP16, NP16 - 3],
          [(160.0, (3, 8)), (320.0, (4, 8)), (640.0, (5, 8)), (1280.0, (6, 8)), (5000.0, (8, 8)), (40.0, 14),
           (80.0, 13)], signal=rp.chirp_noise),
    # orders above 8: the amplitude in double
    _cell("DOG(10)", DOG, 10.0, 16, [NP16, NP16 - 1],
          [(80.0, (3, 8)), (320.0, (5, 8)), (2560.0, (8, 8)), (10.0, 15), (40.0, 13)], signal=rp.chirp_noise),
    _cell("Paul(12)", PAUL, 12.0, 16, [NP16, NP16 - 1],
          [(160.0, (3, 10)), (640.0, (5, 10)), (1280.0, (5, 8)), (5000.0, (7, 8)), (20.0, 15), (80.0, 13)],
          signal=rp.chirp_noise),
    _cell("Paul(60)", PAUL, 60.0, 16, [NP16, NP16 - 2],
          [(320.0, (3, 10)), (1280.0, (5, 10)), (2560.0, (5, 8)), (10000.0, (7, 8)), (40.0, 15), (160.0, 13)],
          signal=rp.chirp_noise),
    # a response table (family 3): dense rows
    _cell("table", MORLET, 6.0, 12, [4096, 4001], [(3.0, 12), (30.0, 12), (300.0, 12)], table=True),
    # the cross-product epilogue (EPI_MULCONJ) on expansion and exact rows
    _cell("xwt", MORLET, 6.0, 16, [NP16, NP16 - 3],
          [(50.0, (3, 8)), (80.0, (4, 10)), (400.0, (6, 8)), (6000.0, (10, 8)), (8.0, 15), (20.0, 13)], xwt=True),
    # exact classes, expansion off: dense, two-kernel, DirectBody<8, 4, 2>, SingleBody<1024 .. 32>
    _cell("exact classes", MORLET, 6.0, 16, [NP16, NP16 - 1],
          [(4.0, 16), (8.0, 15), (16.0, 14), (30.0, 13), (60.0, 12), (120.0, 11), (240.0, 10), (480.0, 9),
           (960.0, 8), (1900.0, 7), (3800.0, 6), (7600.0, 5)], eps=0.0),
    _cell("exact classes, xwt", MORLET, 6.0, 16, [NP16 - 3],
          [(4.0, 16), (16.0, 14), (30.0, 13), (120.0, 11), (240.0, 10), (7600.0, 5)], eps=0.0, xwt=True),
    # Np = 2^21: the three-level dense path and pruned two-kernel rows
    _cell("three-level dense, Np = 2^21", MORLET, 6.0, 21, [2 ** 21 - 3],
          [(2.0, 21), (3.0, 21), (5.0, 20), (12.0, 19)], eps=0.0),
]
# small transforms: TinyBody (Np < 32) and the single-kernel classes of Np = 32 .. 1024
SMALL_N0 = [1, 3, 31, 33, 511, 513]


def _cell_ids():
    return [(c, n0) for c in CELLS for n0 in c["n0s"]]


def run_cell(eng, cell, n0):
    """The cell's transform, plan and profile."""
    fam, par, sj = cell["fam"], cell["par"], cell["sj"]
    x = cell["signal"](n0)
    y2 = rp.white(n0, 9) if cell["xwt"] else None
    table = None
    if cell["table"]:
        Np = orc.next_pow2(n0)
        table = np.array([rp.response(Np, 1.0, s, fam, par, np.float64) for s in sj])
    eng.set_expand_eps(eps32=cell["eps"])
    try:
        eng.profile_begin()
        try:
            if cell["xwt"]:
                # the series are rounded to fp32 on the device
                W = eng.xwt(x, y2, 1.0, sj, fam, par, F32)
            elif table is not None:
                W = eng.cwt(x.astype(np.float32), 1.0, sj, TABLE, 0.0, F32, table=table)
            else:
                W = eng.cwt(x.astype(np.float32), 1.0, sj, fam, par, F32)
        finally:
            prof = eng.profile_end()
        plan = eng.last_plan(len(sj))
    finally:
        eng.set_expand_eps()
    return x, y2, W, plan, prof


def row_classes(cell, plan):
    """(class, bound) of each row; a cell with a looser expansion tolerance is bounded by it."""
    xbound = max(EXPAND32, cell["eps"])
    return [("exact", EXACT32) if p >= 0 else ("expansion", xbound) for p in plan]


def check_cell(eng, cell, n0):
    fam, par, sj, log2N = cell["fam"], cell["par"], cell["sj"], cell["log2N"]
    Np = orc.next_pow2(n0)
    assert Np == 2 ** log2N
    x, y2, W, plan, prof = run_cell(eng, cell, n0)
    # it ran as intended: the plan of every row, and on the device the launches
    want = [-(log2N - p[0]) if isinstance(p, tuple) else p for p in cell["plan"]]
    assert plan == want, (cell["name"], n0, list(zip(sj, plan, want)))
    if not _emulated(eng):
        expand, names = launches(prof)
        rows_by_taps = {}
        for p in cell["plan"]:
            if isinstance(p, tuple):
                rows_by_taps[p[1]] = rows_by_taps.get(p[1], 0) + 1
        epis = (0, 1) if cell["xwt"] else (0,)
        assert expand == {(t, e): r for t, r in rows_by_taps.items() for e in epis}, (cell["name"], prof)
        missing = expected_kernels(plan, log2N) - names
        assert not missing, (cell["name"], missing, sorted(names))
    # it is accurate
    R, sig = ref32(x.astype(np.float32), 1.0, sj, fam, par)
    if cell["xwt"]:
        R2, sig2 = ref32(y2.astype(np.float32), 1.0, sj, fam, par)
        R, sig = R * np.conj(R2), sig * sig2
    err = sigma_err(W, R, sig)
    classes = row_classes(cell, plan)
    factor = 2 if cell["xwt"] else 1          # a product of two rows: twice the rows' bound
    for j, (p, (cls, bound)) in enumerate(zip(cell["plan"], classes)):
        kern = ("ExpandBody<float, %d%s> R = %d" % (p[1], ", 1" if cell["xwt"] else "", 2 ** p[0])
                if isinstance(p, tuple) else "exact log2K' = %d" % p)
        print("  %-36s n0 = %-8d s = %-8g %-34s %-14s err %.2e" % (cell["name"], n0, sj[j], kern, cls, err[j]))
    bad = [(sj[j], cls, float(err[j])) for j, (cls, bound) in enumerate(classes) if err[j] > factor * bound]
    assert not bad, (cell["name"], n0, bad)
    return err


@pytest.mark.gpu
@pytest.mark.parametrize("cell,n0", _cell_ids(), ids=["%s|n0=%d" % (c["name"], n0) for c, n0 in _cell_ids()])
def test_fp32_cell(eng, cell, n0):
    check_cell(eng, cell, n0)


@pytest.mark.gpu
@pytest.mark.parametrize("n0", SMALL_N0)
def test_fp32_small_transforms(eng, n0):
    """Np = 1 .. 1024: TinyBody below 32 points, single-kernel rows above, expansion off and on.  (No
    scale below f0 / pi: such a Morlet row lies past Nyquist in the tail of the response, and the fp32
    band threshold, 1e-9 of the wavelet's peak, is up to 1e-5 of that row's own maximum; s = 0.5
    measures 1.2e-5 on the emulation.)"""
    sj = np.array([1.0, 2.0, 4.0, 8.0, 16.0, 64.0])
    sj = sj[sj <= max(n0, 2)]
    x = rp.white(n0, 11).astype(np.float32)
    R, sig = ref32(x, 1.0, sj, MORLET, 6.0)
    for eps in (0.0, EPS32):
        eng.set_expand_eps(eps32=eps)
        try:
            W = eng.cwt(x, 1.0, sj, MORLET, 6.0, F32)
            plan = eng.last_plan(len(sj))
        finally:
            eng.set_expand_eps()
        Np = orc.next_pow2(n0)
        exact = [(p == 0) if Np < 32 else (5 <= p <= Np.bit_length() - 1) for p in plan]
        assert all(x or (eps and p < -2) for x, p in zip(exact, plan)), (n0, plan)
        err = sigma_err(W, R, sig)
        print("  n0 = %-4d expansion eps32 %g: plan %s, worst %.2e" % (n0, eps, plan, err.max()))
        assert (err <= np.where(exact, EXACT32, EXPAND32)).all(), (n0, err)


# ------------------------------------------------------------------------------------------------
# concurrent stream graph against its serialised run (fp32)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def graph_ref32():
    x = rp.white(rp.GRAPH_N0, 8).astype(np.float32)
    return x, rp.ref_rows(x, 1.0, rp.GRAPH_SJ, MORLET, 6.0, dtype=np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("chains", [1, 2])
@pytest.mark.parametrize("prio", [0, 1, 2])
def test_stream_graph_equals_serial_fp32(graph_ref32, prio, chains):
    x, ref = graph_ref32
    e = osv.make_engine(CWTB_PRIO=str(prio), CWTB_CHAINS=str(chains))
    try:
        for expand in (True, False):
            plan, err = rp.check_graph(e, x, ref, expand, 0, F32, (EXPAND32, EXACT32))
            print("  fp32 CWTB_PRIO=%d CWTB_CHAINS=%d expansion %-3s: bit-identical, classes %s, worst %.2e"
                  % (prio, chains, "on" if expand else "off", sorted(set(plan)), err.max()))
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------
# channel batch (bench config 5's path)
# ------------------------------------------------------------------------------------------------
BATCH_N0 = 20001                                               # Np = 2^15
BATCH_SJ = 2.0 * 2 ** (np.arange(0, 20) / 2.0)                 # s = 2 .. 1450: exact and expansion rows
BATCH_MB = 7          # 7 MiB of fp32 coefficients per chunk: 2 channels of 20 x 20001 (3.2 MB each)
BATCH_CH = 7          # chunks of 2, 2, 2 and 1 channels


def power_ref(X, sj, fam, par):
    """mean_n |R_j|^2 of each channel (rows [nch, S]) and the rows themselves."""
    R = [ref32(x, 1.0, sj, fam, par) for x in X]
    return np.array([(np.abs(r) ** 2).mean(axis=1) for r, _ in R]), R


@pytest.fixture(scope="module")
def batch_input():
    X = np.stack([rp.chirp_noise(BATCH_N0, seed) for seed in range(BATCH_CH)]).astype(np.float32)
    P, R = power_ref(X, BATCH_SJ, MORLET, 6.0)
    return X, P, R


@pytest.mark.gpu
@pytest.mark.parametrize("pipeline", [0, 1])
def test_cwt_batch_fp32(batch_input, pipeline):
    X, P, R = batch_input
    e = osv.make_engine(CWTB_BATCH_MB=str(BATCH_MB), CWTB_BATCH_PIPELINE=str(pipeline))
    try:
        single = [e.cwt(x, 1.0, BATCH_SJ, MORLET, 6.0, F32, out_f64=False) for x in X]
        plan = e.last_plan(len(BATCH_SJ))
        assert min(plan) < -2 < 0 < max(plan), plan            # expansion and exact rows
        # chunks of 2, 2, 2, 1 channels (W requested: the synchronous chunk loop)
        power, W = e.cwt_batch(X, 1.0, BATCH_SJ, MORLET, 6.0, F32, want_power=True, want_w=True)
        for ch in range(BATCH_CH):
            assert np.array_equal(W[ch], single[ch]), ch
            err = sigma_err(W[ch], *R[ch])
            assert (err <= np.where(np.array(plan) < 0, EXPAND32, EXACT32)).all(), (ch, err)
        perr = np.abs(power - P) / P
        print("  CWTB_BATCH_PIPELINE=%d: worst row %.2e, worst power %.2e"
              % (pipeline, max(sigma_err(W[ch], *R[ch]).max() for ch in range(BATCH_CH)), perr.max()))
        assert (perr <= POWER32).all(), perr.max()
        # power only: on the device with CWTB_BATCH_PIPELINE=1 the pipelined input copies
        p2, _ = e.cwt_batch(X, 1.0, BATCH_SJ, MORLET, 6.0, F32, want_power=True)
        assert (np.abs(p2 - P) / P <= POWER32).all()
        # device-resident input, every channel in one launch
        d = e.dev_alloc(X.nbytes)
        try:
            e.h2d(d, X)
            p3 = e.cwt_batch_dev(d, BATCH_CH, BATCH_N0, 1.0, BATCH_SJ, MORLET, 6.0, F32, want_power=True)
            Wd = e.get_w(BATCH_CH * len(BATCH_SJ), BATCH_N0, F32, out_f64=False)
        finally:
            e.dev_free(d)
        assert np.array_equal(Wd.reshape(W.shape), W)
        assert (np.abs(p3 - P) / P <= POWER32).all()
    finally:
        e.close()


@pytest.mark.gpu
def test_config5_real_geometry():
    """Config 5 (1024 channels of 2^16 points, 128 scales, Morlet, fp32): the power of every channel
    against the reference, per entry; every coefficient of 8 channels per row.  n0 = Np, so the mean
    power of a reference row is sum_k |X_k F_jk|^2 / Np^2 (Parseval): one matrix product for all
    channels, no inverse transforms."""
    import workloads as wl
    from pycwt_b200 import _engine
    c = wl.C5
    sj = wl.geometric_scales(c["s0"], c["dj"], c["J"])
    X = wl.config5_channels(0, c["per_gpu"])
    n = c["n"]
    e = _engine.Engine(0)
    try:
        if _emulated(e):
            pytest.skip("GPU-only: 1024 channels x 128 scales of 2^16 points")
        power, _ = e.cwt_batch(X, c["dt"], sj, MORLET, c["f0"], F32, want_power=True)
        F2 = np.array([np.abs(rp.response(n, c["dt"], s, MORLET, c["f0"], np.float64)) ** 2 for s in sj])
        P = np.empty_like(power)
        for c0 in range(0, len(X), 128):
            A = np.abs(np.fft.fft(X[c0:c0 + 128].astype(np.float64), axis=1)) ** 2
            P[c0:c0 + 128] = A @ F2.T / float(n) ** 2
        perr = np.abs(power - P) / P
        ch, j = np.unravel_index(perr.argmax(), perr.shape)
        print("  config 5: power of %d channels x %d scales, worst %.2e (channel %d, s = %g)"
              % (len(X), sj.size, perr.max(), ch, sj[j]))
        assert (perr <= POWER32).all(), (perr.max(), np.unravel_index(perr.argmax(), perr.shape))
        pick = np.random.RandomState(8).choice(len(X), 8, replace=False)
        _, W = e.cwt_batch(X[pick], c["dt"], sj, MORLET, c["f0"], F32, want_power=False, want_w=True)
        plan = e.last_plan(len(sj))
        worst = 0.0
        for i, ch in enumerate(pick):
            err = sigma_err(W[i], *ref32(X[ch], c["dt"], sj, MORLET, c["f0"]))
            worst = max(worst, err.max())
            assert (err <= np.where(np.array(plan) < 0, EXPAND32, EXACT32)).all(), (ch, err)
        print("  config 5: every coefficient of 8 channels, worst row %.2e" % worst)
    finally:
        e.close()
