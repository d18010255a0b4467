"""Row-by-row parity of the GPU-only kernel paths against an extended-precision reference.

`ref_rows` computes rows of the transform independently of every engine path: the full-length band
product (no pruning, no expansion, no overlap-save), in np.longdouble (80-bit on x86-64) from the
forward FFT to the trim to n0.  `row_err` measures each row against its own maximum, so a defect
confined to one phase, one tile or the end of one row cannot hide behind the largest row of the
transform.  The main input is white noise: with the sqrt(s) normalisation every row of its transform
has the same expected power.

Covered on the device:
  * the tensor-core expansion kernel (kernels.cuh: ExpandMmaBody) over a table of cells, each pinned
    to its plan (-log2 Nc from last_plan, taps and rows from the launch names): R = Np / Nc from 4 to
    2^14, 12 / 16 / 20 taps, Nc = 64 alone and in one launch with longer grids, every residue of n0
    mod 4, more tiles than the persistent grid and fewer, the cross-product epilogue, and the
    Morlet / DOG(2) / DOG(3) / Paul(4) responses;
  * the overlap-save rows (kernels.cuh: OsBody) through the checks of test_emu_overlap_save.py, plus
    per-row bounds against the reference;
  * the concurrent stream graph against its serialised run, bit for bit, for every CWTB_PRIO x
    CWTB_CHAINS, with two-kernel chains running beside the coarse / expansion streams.
`pytest --emu` runs the same checks on the host emulation (whose planner has no tensor-core kernel:
the cells set CWTB_EXPAND_MIN_R=2, the tensor-core kernel's own default, so that both plan the same
coarse grids); only the kernel-name assertions are skipped there.
"""
import math
import re

import numpy as np
import pytest

from conftest import load_golden
from oracle import cwt_oracle as orc
import test_emu_overlap_save as osv

MORLET, PAUL, DOG = 0, 1, 2
OS = osv.OS
LD = np.longdouble
PI_L = 4 * np.arctan(LD(1))
EPS64 = 5e-13          # default expansion tolerance (engine set_expand_eps)
EXACT = 1e-14          # exact rows (DESIGN 6)


# ------------------------------------------------------------------------------------------------
# reference
# ------------------------------------------------------------------------------------------------
def _conj_psi_ld(family, param, f):
    """conj(psi_ft(f)) of the reference's mothers (oracle/cwt_oracle.py) in the precision of f
    (longdouble or fp64); the Paul and DOG normalisation constants are fp64 (each within an ulp of
    their exact value)."""
    T = f.dtype.type
    if family == MORLET:
        return (4 * np.arctan(T(1))) ** T(-0.25) * np.exp(-(f - T(param)) ** 2 / 2)
    m = int(param)
    if family == PAUL:
        # (2m - 1)! as the engine forms it (in double); the reference's int64 np.prod(range(2, 2m))
        # is the same number up to m = 10 and wraps around from m = 11
        c = T(2.0 ** m / np.sqrt(m * float(math.factorial(2 * m - 1))))
        with np.errstate(over="ignore"):
            return np.where(f > 0, c * f ** m * np.exp(-np.maximum(f, 0)), T(0))
    c = T(1.0 / np.sqrt(orc._gamma(m + 0.5)))
    mag = c * f ** m * np.exp(-f ** 2 / 2)
    # conj(-(1j ** m)) exactly: m % 4 = 0 -> -1, 1 -> +i, 2 -> +1, 3 -> -i
    return mag * {0: -1, 1: 1j, 2: 1, 3: -1j}[m % 4]


def response(Np, dt, s, family, param, dtype=LD):
    """F[k] = sqrt(s w1 Np) conj(psi_ft(s omega_k)) on the Np signed bins, in `dtype`."""
    T = np.dtype(dtype).type
    pi = 4 * np.arctan(T(1))
    k = (np.fft.fftfreq(Np) * Np).astype(T)                    # signed bins, exact
    omega = 2 * pi * k / (T(Np) * T(dt))
    norm = np.sqrt(T(s) * (2 * pi / (T(Np) * T(dt))) * T(Np))   # sqrt(s w1 Np)
    return norm * _conj_psi_ld(family, param, T(s) * omega)


def ref_rows(x, dt, scales, family, param, n0=None, npad=None, dtype=LD):
    """Rows W[j, :n0] of the transform of x (zero-padded to the next power of two, or to `npad`) at the
    fp64 scales, as full-length band products computed in `dtype` (longdouble by default; fp64 is
    enough against the fp32 engine); complex128 result.  Paul's response is finite everywhere here,
    as in the engine (the reference's inf * 0 = NaN rows, s pi / dt > 709.78, are dropped by the
    Python layer, pycwt_b200/wavelet.py: _nan_rows)."""
    x = np.asarray(x, dtype=np.float64)
    n0 = x.size if n0 is None else n0
    Np = npad or orc.next_pow2(x.size)
    X = np.fft.fft(x.astype(dtype), Np)
    out = np.empty((len(scales), n0), dtype=np.complex128)
    for j, s in enumerate(np.asarray(scales, dtype=np.float64)):
        row = np.fft.ifft(X * response(Np, dt, s, family, param, dtype))
        out[j] = row[:n0]
    return out


def row_err(W, ref):
    """max_n |W[j] - ref[j]| / max_n |ref[j]| for each row j; the NaN pattern must match."""
    W, ref = np.asarray(W), np.asarray(ref)
    assert W.shape == ref.shape, (W.shape, ref.shape)
    assert (np.isnan(W) == np.isnan(ref)).all(), "NaN pattern differs"
    out = np.zeros(W.shape[0])
    for j in range(W.shape[0]):
        if np.isnan(ref[j]).all():
            continue
        m = np.abs(ref[j]).max()
        d = np.abs(W[j] - ref[j]).max()
        out[j] = d / m if m > 0 else d
    return out


def white(n0, seed=0):
    return np.random.RandomState(seed).randn(n0)


def chirp_noise(n0, seed=1):
    t = np.arange(n0) / n0
    return np.sin(2 * np.pi * (40 * t + (n0 / 16) * t ** 2)) + 0.5 * np.random.RandomState(seed).randn(n0)


def test_reference_self_check():
    """CPU: the reference agrees with the fp64 oracle row by row and with fixtures of the reference
    package, on every family (on Paul's rows that the oracle does not turn into NaN)."""
    x = white(3000, 5)
    sj = 0.7 * 2 ** (np.arange(0, 44) / 4.0)
    for fam, mother, par in ((MORLET, orc.Morlet(6), 6.0), (PAUL, orc.Paul(4), 4.0),
                             (DOG, orc.DOG(2), 2.0), (DOG, orc.DOG(3), 3.0)):
        with np.errstate(all="ignore"):
            Wo, so = orc.cwt(x, 1.0, wavelet=mother, freqs=1 / (mother.flambda() * sj))[:2]
        # the oracle drops its all-NaN rows; the reference runs at the scales the oracle kept
        assert len(so) >= 30 and np.isfinite(Wo).all()
        R = ref_rows(x, 1.0, so, fam, par)
        e = row_err(R, Wo)
        assert (e <= 2e-15).all(), (fam, par, e.max(), int(e.argmax()))
    assert np.isfinite(ref_rows(x, 1.0, sj[-4:], PAUL, 4.0)).all()
    for name in ("chirp4000_morlet", "nino3_dog3_odd"):
        g = load_golden(name)
        fam = {"morlet": MORLET, "paul": PAUL, "dog": DOG}[str(g["wavelet"])]
        R = ref_rows(g["x"], float(g["dt"]), g["sj"], fam, float(g["param"]))
        e = row_err(R[:, ::int(g["stride"])], g["W"])
        assert (e <= 1e-13).all(), (name, e.max())


# ------------------------------------------------------------------------------------------------
# engines
# ------------------------------------------------------------------------------------------------
def _emulated(eng):
    return "emulation" in eng.version()


@pytest.fixture(scope="module")
def eng():
    e = osv.make_engine(CWTB_EXPAND_MIN_R="2")
    yield e
    e.close()


def expand_launches(prof):
    """{(taps, epilogue): rows} of the tensor-core expansion launches of a profile."""
    out = {}
    for p in prof:
        m = re.search(r"ExpandMmaBody<(\d+)(?:,\s*(\d+))?>", p["name"])
        if m:
            key = (int(m.group(1)), int(m.group(2) or 0))
            out[key] = out.get(key, 0) + p["rows"]
    return out


# ------------------------------------------------------------------------------------------------
# B. tensor-core expansion cells
# ------------------------------------------------------------------------------------------------
# A cell: wavelet, Np, n0 values, scales and the plan the planner must give each of them:
# (log2 R, taps) for an expansion row (R = Np / Nc), None for an exact row.  The scales come from the
# band half-width (R grows with s at any Np); `eps`: set_expand_eps for the cell and its bound.
def _cell(name, fam, par, log2N, n0s, rows, eps=EPS64, xwt=False, signal=white):
    return dict(name=name, fam=fam, par=par, log2N=log2N, n0s=n0s, sj=np.array([r[0] for r in rows]),
                plan=[r[1] for r in rows], eps=eps, xwt=xwt, signal=signal)


NP16 = 2 ** 16
N0_EDGES = [NP16, NP16 - 1, NP16 - 2, NP16 - 3, NP16 // 2 + 1]   # every residue mod 4 ends a store pair
MORLET_MIX = [(3.0, None), (8.0, None), (13.0, None),
              (17.0, (2, 20)), (25.0, (2, 16)), (34.0, (3, 20)), (50.0, (3, 16)), (70.0, (4, 20)),
              (120.0, (4, 16)), (165.0, (5, 16)), (185.0, (4, 12)), (500.0, (5, 12)), (1000.0, (6, 12)),
              (2000.0, (7, 12))]
CELLS = [
    _cell("morlet R 4..128, n0 edges", MORLET, 6.0, 16, N0_EDGES, MORLET_MIX),
    # R = 4 with 12 taps exists only for a looser tolerance
    _cell("R = 4, 12 / 16 / 20 taps", MORLET, 6.0, 16, [NP16, NP16 - 3],
          [(17.0, (2, 20)), (22.0, (2, 16)), (30.0, (2, 12)), (60.0, (3, 12)), (8.0, None)], eps=1e-11),
    # Nc = 64 (R = 1024) in the 12-tap launch with Nc = 128 / 256 / 4096 rows: the launch's tile count
    # follows Nc = 64, the longer rows' extra tiles are dead
    _cell("Nc = 64 with longer grids", MORLET, 6.0, 16, [NP16, NP16 - 2],
          [(3000.0, (8, 12)), (8000.0, (9, 12)), (20000.0, (10, 12)), (185.0, (4, 12))]),
    # one row, Np = 2^12: Nc = 64 alone, 2 tiles for the whole grid
    _cell("Nc = 64 alone, Np = 2^12", MORLET, 6.0, 12, [4096, 4093], [(1000.0, (6, 12))]),
    # Np = 2^20: 4 rows x 256 tiles + the 2^14-phase weight table (Nc = 64: 512 tiles) in one 12-tap
    # launch, far more tiles than occupancy x SMs: the persistent loop wraps
    _cell("Np = 2^20, R = 16 and 2^14", MORLET, 6.0, 20, [2 ** 20 - 1],
          [(182.0, (4, 12)), (186.0, (4, 12)), (190.0, (4, 12)), (195.0, (4, 12)), (4e5, (14, 12)),
           (8.0, None)]),
    _cell("DOG(2)", DOG, 2.0, 16, [NP16, NP16 - 1],
          [(18.0, (2, 20)), (25.0, (2, 16)), (36.0, (3, 20)), (100.0, (4, 16)), (195.0, (4, 12)),
           (1000.0, (6, 12)), (5.0, None)], signal=chirp_noise),
    _cell("DOG(3)", DOG, 3.0, 16, [NP16, NP16 - 2],
          [(18.0, (2, 20)), (25.0, (2, 16)), (36.0, (3, 20)), (100.0, (4, 16)), (205.0, (4, 12)),
           (1000.0, (6, 12)), (5.0, None)], signal=chirp_noise),
    _cell("Paul(4)", PAUL, 4.0, 16, [NP16, NP16 - 3],
          [(52.0, (2, 20)), (70.0, (2, 16)), (105.0, (3, 20)), (300.0, (4, 16)), (550.0, (4, 12)),
           (3000.0, (6, 12)), (20.0, None)], signal=chirp_noise),
    # the cross-product epilogue (EPI_MULCONJ) on R = 4 / 8 / 64
    _cell("xwt R = 4, 8, 64", MORLET, 6.0, 16, [NP16, NP16 - 3],
          [(17.0, (2, 20)), (34.0, (3, 20)), (1000.0, (6, 12)), (8.0, None)], xwt=True),
]


def check_expansion_cell(eng, cell, n0):
    fam, par, sj, log2N = cell["fam"], cell["par"], cell["sj"], cell["log2N"]
    assert orc.next_pow2(n0) == 2 ** log2N
    x = cell["signal"](n0)
    eng.set_expand_eps(cell["eps"])
    try:
        eng.profile_begin()
        try:
            if cell["xwt"]:
                y2 = white(n0, 9)
                W = eng.xwt(x, y2, 1.0, sj, fam, par)
            else:
                W = eng.cwt(x, 1.0, sj, fam, par)
        finally:
            prof = eng.profile_end()
        plan = eng.last_plan(len(sj))
    finally:
        eng.set_expand_eps()
    # it ran as intended: the coarse grid of every row, and on the device the launches by tap count
    want = [-(log2N - p[0]) if p else None for p in cell["plan"]]
    for j, (w, p) in enumerate(zip(want, plan)):
        assert (p == w) if w is not None else (p > 0 or p == OS), (cell["name"], j, sj[j], plan)
    rows_by_taps = {}
    for p in cell["plan"]:
        if p:
            rows_by_taps[p[1]] = rows_by_taps.get(p[1], 0) + 1
    launches = expand_launches(prof)
    if not _emulated(eng):
        epis = (0, 1) if cell["xwt"] else (0,)
        assert launches == {(t, e): r for t, r in rows_by_taps.items() for e in epis}, (cell["name"], prof)
    # it is accurate
    ref = ref_rows(x, 1.0, sj, fam, par)
    if cell["xwt"]:
        ref = ref * np.conj(ref_rows(y2, 1.0, sj, fam, par))
    err = row_err(W, ref)
    xr = [j for j, p in enumerate(cell["plan"]) if p]
    er = [j for j, p in enumerate(cell["plan"]) if not p]
    for j in xr:
        print("  %-28s ExpandMmaBody<%d%s>  R = %-5d taps %d  n0 = %d  row_err %.2e"
              % (cell["name"], cell["plan"][j][1], ", 1" if cell["xwt"] else "", 2 ** cell["plan"][j][0],
                 cell["plan"][j][1], n0, err[j]))
    assert (err[xr] <= cell["eps"]).all(), (cell["name"], n0, dict(zip(sj[xr], err[xr])))
    assert (err[er] <= EXACT).all(), (cell["name"], n0, dict(zip(sj[er], err[er])))
    return err


def _cell_ids():
    return [(c, n0) for c in CELLS for n0 in c["n0s"]]


@pytest.mark.gpu
@pytest.mark.parametrize("cell,n0", _cell_ids(), ids=["%s|n0=%d" % (c["name"], n0) for c, n0 in _cell_ids()])
def test_expansion_cell(eng, cell, n0):
    check_expansion_cell(eng, cell, n0)


# ------------------------------------------------------------------------------------------------
# C. overlap-save rows
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def os_engines():
    # (CWTB_EXPAND_MIN_R=2 is the device's default; the emulation then plans the same rows)
    on = osv.make_engine(CWTB_OS="1", CWTB_EXPAND_MIN_R="2")
    off = osv.make_engine(CWTB_OS="0", CWTB_EXPAND_MIN_R="2")
    yield on, off
    on.close()
    off.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n0", [osv.N0, 2 ** 16])
@pytest.mark.parametrize("fam,mother,par", [(MORLET, orc.Morlet(6), 6.0), (DOG, orc.DOG(2), 2.0),
                                            (DOG, orc.DOG(6), 6.0)])
def test_overlap_save_rows(os_engines, n0, fam, mother, par):
    on, off = os_engines
    W, plan = osv.check_rows_match_oracle(on, n0, fam, mother, par)
    err = row_err(W, ref_rows(osv._signal(n0), 1.0, osv.SJ, fam, par))
    rows = [j for j, p in enumerate(plan) if p == OS]
    print("  overlap-save %s n0 = %d: rows %s, worst row_err %.2e" % (type(mother).__name__, n0, rows, err[rows].max()))
    assert (err[rows] <= EXACT).all(), dict(zip(rows, err[rows]))
    # white noise: the same rows against the parent paths, every other row bit-identical
    osv.check_equals_replaced_path_per_row(on, off, white(n0, 3), fam, par)


@pytest.mark.gpu
def test_overlap_save_partial_group(os_engines):
    """A row count whose last overlap-save group of four is partial."""
    on, off = os_engines
    x = white(osv.N0, 4)
    for k in range(len(osv.SJ), 0, -1):
        sj = osv.SJ[:k]
        on.cwt(x, 1.0, sj, MORLET, 6.0, fetch=False)
        if on.last_plan(k).count(OS) % 4:
            break
    W, plan = osv.check_equals_replaced_path_per_row(on, off, x, MORLET, 6.0, sj)
    rows = [j for j, p in enumerate(plan) if p == OS]
    assert len(rows) % 4 and len(rows) > 4, plan
    err = row_err(W, ref_rows(x, 1.0, sj, MORLET, 6.0))
    assert (err[rows] <= EXACT).all(), dict(zip(rows, err[rows]))


@pytest.mark.gpu
def test_overlap_save_config2_geometry(os_engines):
    """Config 2's geometry (Np = 2^20, s0 = 2, dj = 1/16, 256 scales, Morlet): its overlap-save rows
    against the reference and against the paths they replace; every other row bit-identical."""
    import workloads as wl
    on, off = os_engines
    sj = wl.config2_scales()
    x = white(wl.C2["n"], 6)
    W, plan = osv.check_equals_replaced_path_per_row(on, off, x, MORLET, wl.C2["f0"], sj)
    rows = [j for j, p in enumerate(plan) if p == OS]
    assert rows == list(range(20, 48)), rows
    err = row_err(W[rows], ref_rows(x, wl.C2["dt"], sj[rows], MORLET, wl.C2["f0"]))
    print("  config 2 overlap-save rows 20..47: worst row_err %.2e" % err.max())
    assert (err <= EXACT).all(), err


@pytest.mark.gpu
def test_overlap_save_engine_checks(os_engines):
    """The checks of test_emu_overlap_save.py on the device: Nyquist / Paul rows keep their path,
    re-planning, batched channels bit-identical to single-channel calls, weight tables of rejected
    candidates, the cross-product epilogue and the resident products."""
    on, off = os_engines
    signal = osv._signal(osv.N0)
    osv.check_nyquist_and_paul_rows_rejected(on, signal)
    osv.check_replanning(on, off, signal)
    osv.check_batched_channels_equal_single_channel(on, signal)
    osv.check_new_weight_tables_survive_rejected_candidates(off, signal, CWTB_OS="0", CWTB_EXPAND_MIN_R="2")
    X, y2 = osv.check_cross_product_epilogue(on, off, signal)
    plan = on.last_plan(len(osv.SJ))
    rows = [j for j, p in enumerate(plan) if p == OS]
    ref = ref_rows(signal, 1.0, osv.SJ[rows], MORLET, 6.0) * np.conj(ref_rows(y2, 1.0, osv.SJ[rows], MORLET, 6.0))
    err = row_err(X[rows], ref)
    assert (err <= 2 * EXACT).all(), err      # a product of two rows: twice the rows' bound
    osv.check_resident_products(on, off, signal)


# ------------------------------------------------------------------------------------------------
# D. concurrent stream graph against its serialised run
# ------------------------------------------------------------------------------------------------
# One Morlet geometry at Np = 2^17, run three ways on each configuration:
#   * overlap-save on: dense and overlap-save rows, expansion rows of 16 / 20 taps on coarse grids of
#     2^13 .. 2^15 points (the second pass, behind the long coarse transforms) and a 12-tap launch on
#     grids of 64 .. 1024 points (the first pass);
#   * overlap-save off (CWTB_OS=0): the same expansion launches next to dense and two-kernel rows of
#     three classes, which rotate over the chain streams while the coarse priority chain runs;
#   * expansion off: single-kernel, direct, two-kernel and dense rows.
# Single-kernel and direct rows never share a transform with expansion rows: every band narrow enough
# for them is planned for the expansion.
GRAPH_N0 = 2 ** 17 - 7
GRAPH_LOG2N = 17
GRAPH_SJ = np.concatenate([2.0 * 2 ** (np.arange(0, 50) / 8.0), 1500.0 * 2 ** (np.arange(0, 17) / 4.0)])


@pytest.fixture(scope="module")
def graph_ref():
    x = white(GRAPH_N0, 8)
    return x, ref_rows(x, 1.0, GRAPH_SJ, MORLET, 6.0)


def check_graph(eng, x, ref, expand, os_on, precision=0, bounds=(EPS64, EXACT)):
    """W three ways -- overlapped copy, transform then fetch, serialised (profiling) then fetch --
    bit-identical, and per row within the bounds of the reference: `bounds` (expansion rows, exact
    rows) of row_err.  The fp32 engine (precision 1) has no overlap-save rows."""
    sj = GRAPH_SJ
    if not expand:
        eng.set_expand_eps(0.0, 0.0)
    try:
        W1 = eng.cwt(x, 1.0, sj, MORLET, 6.0, precision)
        plan = eng.last_plan(len(sj))
        eng.cwt(x, 1.0, sj, MORLET, 6.0, precision, fetch=False)
        W2 = eng.get_w(len(sj), x.size, precision)
        eng.profile_begin()
        try:
            eng.cwt(x, 1.0, sj, MORLET, 6.0, precision, fetch=False)
        finally:
            prof = eng.profile_end()
        W3 = eng.get_w(len(sj), x.size, precision)
    finally:
        eng.set_expand_eps()
    log2N = GRAPH_LOG2N
    chain_classes = {p for p in plan if 13 < p <= log2N}     # two-kernel and dense classes
    if expand:
        # expansion launches in both passes
        assert any(-10 <= p < -2 for p in plan) and any(p < -10 for p in plan), plan
        if os_on and precision == 0:
            assert OS in plan and log2N in plan, plan
        else:
            # two-kernel rows, and more chain classes than one stream
            assert OS not in plan and any(13 < p < log2N for p in plan) and len(chain_classes) >= 3, plan
    else:
        # single-kernel (K' <= 2^10), direct (2^11 .. 2^13), two-kernel and dense rows
        assert set(plan) >= {5, 8, 12, 13, 14, 15, 16, log2N}, plan
    if not _emulated(eng):
        kernel = "ExpandMmaBody<" if precision == 0 else "ExpandBody<float"
        assert prof and (not expand or any(kernel in p["name"] for p in prof)), prof
    assert np.array_equal(W1, W2), "overlapped copy differs from transform-then-fetch"
    assert np.array_equal(W1, W3), "concurrent run differs from the serialised one"
    err = row_err(W1, ref)
    xr = [j for j, p in enumerate(plan) if p < -2]
    er = [j for j, p in enumerate(plan) if p > 0 or p == OS]
    assert (err[xr] <= bounds[0]).all(), dict(zip(xr, err[xr]))
    assert (err[er] <= bounds[1]).all(), dict(zip(er, err[er]))
    return plan, err


@pytest.mark.gpu
@pytest.mark.parametrize("chains", [1, 2])
@pytest.mark.parametrize("prio", [0, 1, 2])
def test_stream_graph_equals_serial(graph_ref, prio, chains):
    x, ref = graph_ref
    env = dict(CWTB_PRIO=str(prio), CWTB_CHAINS=str(chains), CWTB_EXPAND_MIN_R="2")
    engines = {os_on: osv.make_engine(CWTB_OS=str(os_on), **env) for os_on in (1, 0)}
    try:
        for os_on, expand in ((1, True), (0, True), (1, False)):
            plan, err = check_graph(engines[os_on], x, ref, expand, os_on)
            print("  CWTB_PRIO=%d CWTB_CHAINS=%d overlap-save %-3s expansion %-3s: bit-identical, classes %s, "
                  "worst row_err %.2e" % (prio, chains, "on" if os_on else "off", "on" if expand else "off",
                                          sorted(set(plan)), err.max()))
    finally:
        for e in engines.values():
            e.close()
