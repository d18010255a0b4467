"""Row-by-row parity of the fp64 engine's exact rows against an extended-precision reference.

The reference is `ref_rows` of test_gpu_row_parity.py (np.longdouble from the forward FFT to the trim),
each row measured against its own maximum (`row_err`), so a defect confined to one class, one tile or
the end of one row cannot hide behind the largest row of the transform.  The expansion is off
(set_expand_eps(0, 0)) in every cell: each row runs one of the exact classes, and each cell pins the
class of every row (last_plan) and, on the device, the exact-class kernels it launches.

Covered:
  * Np = 2^20, the register-resident dense first kernel PassABody<double, 1024, MODE_DENSE> with
    PassBBody<double, 1, 1024, true>: Morlet(6) (its Gaussian walk, a row whose band crosses the signed-bin
    wrap), DOG(2, 3, 6, 10), Paul(4, 12, 60) (the out-of-line family evaluation) and a response table;
    rows pruned to 2^18 / 2^19 that go dense through the planner's dense margin, K' = 2^17 two-kernel rows
    (band-mode first kernel, 1024-point second kernel), DirectBody and SingleBody rows;
    n0 = 2^20, 2^20 - 3, 2^19 + 1;
  * band_eps = 0 at Np = 2^20 (the Gaussian walk re-seeds on subnormal values), Morlet and DOG(2);
  * Np = 2^16: SingleBody<double, 32 .. 1024>, DirectBody<double, 2 | 4 | 8>, two-kernel rows with the
    512-point second kernel and the three-pass dense rows, for DOG(2), DOG(3), Paul(4) and a table;
  * the three-level path: Np = 2^21 (and 2^22 on the device only), the dense pre-pass with K1 = 2 / 4
    followed by the interleaved 2^20-point transforms (PassABody MODE_CPLX, then the register-resident
    PassBBody), and pruned two-kernel rows;
  * xwt (EPI_MULCONJ) on the exact classes against R1 conj(R2), DOG(2) and Paul(4);
  * TinyBody and the single-kernel classes of Np = 1 .. 1024, DOG(2) and Paul(4);
  * the transform hook fft_c2c at n = 2^20 and 2^21, both signs, against a longdouble np.fft.
Morlet at the Np = 2^16 classes is covered by check_graph of test_gpu_row_parity.py.  A Paul band has
positive frequencies only (at most Np / 2 bins), so up to Np = 2^21 a Paul row is never dense by its
band: its dense rows at Np = 2^20 come through the dense margin, at Np = 2^16 and 2^21 it has none, and
at Np = 2^22 the pruned length 2^21 is not built and the row runs dense.  A table row has no band and is
always dense.

Bounds: EXACT = 1e-14 of row_err per row (DESIGN 6), twice that for xwt (a product of two rows); fft_c2c
1e-14 of each output row's maximum.  Worst row_err per class on an H100 80GB HBM3 at a 700 W power
limit (host emulation in brackets):
  dense, Np = 2^20 (register-resident core)    5.1e-15 (5.1e-15)  Morlet(6), s = 1
  dense, Np = 2^20, band_eps = 0               4.3e-15 (4.6e-15)  Morlet(6), s = 2
  two-kernel, K' = 2^17                        2.1e-15 (2.1e-15)  Paul(60)
  DirectBody / SingleBody                      1.6e-15 / 2.2e-15 (1.7e-15 / 2.1e-15)  Paul(60)
  Np = 2^16 classes (512-point second kernel)  9.3e-16 (1.4e-15)
  three-level (Np = 2^21, 2^22)                1.3e-15 (1.5e-15)
  xwt                                          2.2e-15 (2.8e-15)  Paul(4), DirectBody
  small transforms / fft_c2c                   5.6e-16 / 8.5e-16 (6.2e-16 / 1.2e-15)

Single-edit fp64 mutants on the emulation: the largest row_err of a row of this file's cells, then the
tests that fail, here and in the existing suite:
  GaussWalk re-seed interval 16 -> 256          5.1e-15  none here: within the bound, equal to the unmutated
                                                         rows (a thread's column walks 32 bins and re-seeds
                                                         at the band's edge and the wrap); existing suite
                                                         not run
  subnormal guard `g < 1e-290` removed           3.4e-13  the band_eps = 0 Morlet cell (s = 16); existing suite
                                                         not run (its band_eps = 0 checks hold 1e-12)
  x32_exchange_out: cmul(wc, wa[a]) -> wc, a = 3  O(1)     every cell whose rows or forward transform run
                                                         the 1024-point core (Np >= 2^16), fft_c2c; dozens
                                                         of existing tests
  x32_last: second half stored at k1 + 256       O(1)     the same cells and tests (half of every output
                                                         tile is never written)
  Paul (2m - 1)! formed in int64                 NaN      the Paul(12) (x 2.4e2) and Paul(60) (non-finite)
                                                         cells; in the existing suite the fp32 file's Paul(12)
                                                         and Paul(60) cells, no fp64 test (none uses m > 10)

`pytest --emu` runs every cell on the host emulation except the kernel-name assertions and the
Np = 2^22 cell.
"""
import numpy as np
import pytest

import test_emu_overlap_save as osv
import test_gpu_row_parity as rp
from oracle import cwt_oracle as orc

MORLET, PAUL, DOG, TABLE = 0, 1, 2, 3
EXACT = rp.EXACT            # 1e-14: exact rows (DESIGN 6)
FFT_BOUND = 1e-14           # fft_c2c, relative to each output row's maximum
BAND_EPS = 1e-16            # the engine's default band threshold (cwtb_set_band_eps)
FAM_NAME = {MORLET: "Morlet", PAUL: "Paul", DOG: "DOG"}


# ------------------------------------------------------------------------------------------------
# CPU: the reference
# ------------------------------------------------------------------------------------------------
def test_fp64_reference_matches_longdouble_high_orders():
    """CPU: for the orders whose normalisation constant is a double (the engine forms it the same way),
    the fp64 reference agrees with the longdouble one within a fifth of EXACT (measured at most 1.1e-15,
    Paul(60) at s = 10), at the scales of the cells."""
    x = rp.white(5000, 2)
    for fam, par, sj in ((DOG, 10.0, [2.0, 8.0, 32.0, 512.0, 4096.0]),
                         (PAUL, 12.0, [4.0, 60.0, 120.0, 1900.0, 15000.0]),
                         (PAUL, 60.0, [10.0, 150.0, 280.0, 4500.0, 35000.0])):
        e = rp.row_err(rp.ref_rows(x, 1.0, sj, fam, par, npad=2 ** 20, dtype=np.float64)[:, :5000],
                       rp.ref_rows(x, 1.0, sj, fam, par, npad=2 ** 20)[:, :5000])
        print("  %s(%d): fp64 against longdouble reference, worst row %.2e" % (FAM_NAME[fam], par, e.max()))
        assert (e <= EXACT / 5).all(), (fam, par, e)


def test_table_reproduces_family_rows_on_emulation():
    """CPU (host emulation): a response table built from `response` gives the analytic family's rows,
    and both give the reference's."""
    n0 = 4001
    x = rp.white(n0, 4)
    Np = orc.next_pow2(n0)
    e = osv.make_engine(osv.emu_lib())
    try:
        assert "emulation" in e.version()
        e.set_expand_eps(0.0, 0.0)
        for fam, par, sj in ((MORLET, 6.0, [1.0, 2.0, 30.0, 300.0]), (DOG, 3.0, [2.0, 30.0, 300.0]),
                             (PAUL, 4.0, [2.0, 60.0, 600.0])):
            table = np.array([rp.response(Np, 1.0, s, fam, par, np.float64) for s in sj])
            Wt = e.cwt(x, 1.0, sj, TABLE, 0.0, table=table)
            assert e.last_plan(len(sj)) == [12] * len(sj)            # a table row is dense
            Wf = e.cwt(x, 1.0, sj, fam, par)
            ref = rp.ref_rows(x, 1.0, sj, fam, par)
            et, ef, d = rp.row_err(Wt, ref), rp.row_err(Wf, ref), rp.row_err(Wt, Wf)
            print("  table %s(%g): table %.2e, family %.2e, table against family %.2e"
                  % (FAM_NAME[fam], par, et.max(), ef.max(), d.max()))
            assert (et <= EXACT).all() and (ef <= EXACT).all() and (d <= EXACT).all(), (fam, et, ef, d)
    finally:
        e.close()


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


EXACT_KERNELS = ("TinyBody", "SingleBody", "DirectBody", "BandBody", "PassABody", "PassBBody")


def launched(prof):
    """Names (without spaces) of the exact-class kernels of a profile, the forward transform's excluded."""
    out = set()
    for p in prof:
        name = p["name"].replace(" ", "")
        if ":" not in name and name.startswith(EXACT_KERNELS):
            out.add(name)
    return out


def expected_kernels(plan, log2N):
    """The exact-class kernels a plan launches (engine.cu: run_classes)."""
    want = set()
    for p in set(plan):
        if p == 0:
            want.add("TinyBody<double>")
        elif p <= 10:
            # (single-kernel and direct classes read the band products, dense ones included)
            want |= {"BandBody<double>", "SingleBody<double,%d>" % 2 ** p}
        elif p <= 13 and p < log2N:
            want |= {"BandBody<double>", "DirectBody<double,%d>" % 2 ** (p - 10)}
        elif p == log2N and p > 20:
            # dense pre-pass of K0 = Np / 2^20 points, then the K0 interleaved 2^20-point transforms
            want |= {"PassABody<double,%d,0,1>" % 2 ** (p - 20), "PassABody<double,1024,3,1>",
                     "PassBBody<double,1,1024,true>"}
        elif p == log2N:
            # dense: 1024-point second kernel, K1 = Np / 1024 (the register-resident core at K1 = 1024)
            want |= {"PassABody<double,%d,0,1>" % 2 ** (p - 10), "PassBBody<double,1,1024,true>"}
        else:
            # band products, then first kernels of K' / K2 points: K2 = 512 up to K' = 2^16, 1024 above
            l2k = 10 if p > 16 else 9
            want |= {"BandBody<double>", "PassABody<double,%d,1,1>" % 2 ** (p - l2k),
                     "PassBBody<double,1,%d,%s>" % (2 ** l2k, "true" if l2k == 10 else "false")}
    return want


# ------------------------------------------------------------------------------------------------
# plan-pinned cells
# ------------------------------------------------------------------------------------------------
# A cell: wavelet, Np, n0 values, and (scale, log2 K') of every row; K' = Np for a dense row.
# `table`: the rows run as a response table (family 3) built from (family, param) per row.
# `band_eps`: set_band_eps of the cell (restored to the default after it).  `gpu_only`: skipped on the
# emulation (Np = 2^22).
def _cell(name, fam, par, log2N, n0s, rows, xwt=False, table=None, band_eps=BAND_EPS, gpu_only=False):
    return dict(name=name, fam=fam, par=par, log2N=log2N, n0s=n0s, sj=np.array([r[0] for r in rows], float),
                plan=[r[1] for r in rows], xwt=xwt, table=table, band_eps=band_eps, gpu_only=gpu_only)


N20 = [2 ** 20, 2 ** 20 - 3, 2 ** 19 + 1]
N16 = [2 ** 16, 2 ** 16 - 1]
# Np = 2^20, per family: a dense row by its band, rows of K' = 2^19 and 2^18 made dense by the dense
# margin, a K' = 2^17 two-kernel row, a DirectBody<8> row (K' = 2^13) and a SingleBody<1024> row.
DOG20 = [(2.0, 20), (8.0, 20), (16.0, 20), (32.0, 17), (512.0, 13), (4096.0, 10)]
CELLS = [
    # s = 1, 2: bands from negative frequencies past Nyquist, across the signed-bin wrap
    _cell("Np = 2^20 Morlet(6)", MORLET, 6.0, 20, N20,
          [(1.0, 20), (2.0, 20), (8.0, 20), (16.0, 20), (32.0, 17), (512.0, 13), (4096.0, 10)]),
    _cell("Np = 2^20 DOG(2)", DOG, 2.0, 20, N20, DOG20),
    _cell("Np = 2^20 DOG(3)", DOG, 3.0, 20, N20, DOG20),
    _cell("Np = 2^20 DOG(6)", DOG, 6.0, 20, N20, DOG20),
    _cell("Np = 2^20 DOG(10)", DOG, 10.0, 20, N20, DOG20),
    _cell("Np = 2^20 Paul(4)", PAUL, 4.0, 20, N20,
          [(2.0, 20), (50.0, 20), (100.0, 17), (1600.0, 13), (12000.0, 10)]),
    _cell("Np = 2^20 Paul(12)", PAUL, 12.0, 20, N20,
          [(4.0, 20), (60.0, 20), (120.0, 17), (1900.0, 13), (15000.0, 10)]),
    _cell("Np = 2^20 Paul(60)", PAUL, 60.0, 20, N20,
          [(10.0, 20), (150.0, 20), (280.0, 17), (4500.0, 13), (35000.0, 10)]),
    # a table row has no band: every row dense, whatever its width
    _cell("Np = 2^20 table", None, None, 20, N20, [(2.0, 20), (8.0, 20), (50.0, 20), (512.0, 20)],
          table=[(MORLET, 6.0), (DOG, 3.0), (PAUL, 4.0), (DOG, 2.0)]),
    # band_eps = 0: the bands reach bins whose response is subnormal.  From s = 16 a Morlet walk climbs
    # from the band's edge to its peak within one re-seeding interval of 16 steps (s w_D = pi per step)
    _cell("Np = 2^20 band_eps = 0, Morlet(6)", MORLET, 6.0, 20, [2 ** 20 - 3],
          [(1.0, 20), (2.0, 20), (4.0, 20), (8.0, 20), (12.0, 20), (16.0, 20)], band_eps=0.0),
    _cell("Np = 2^20 band_eps = 0, DOG(2)", DOG, 2.0, 20, [2 ** 20 - 3], [(2.0, 20), (4.0, 20), (8.0, 20)],
          band_eps=0.0),
    # Np = 2^16: three-pass dense (K1 = 64), two-kernel rows with the 512-point second kernel (K' = 2^14,
    # 2^15), DirectBody<8, 4, 2>, SingleBody<1024 .. 32>
    _cell("Np = 2^16 DOG(2)", DOG, 2.0, 16, N16,
          [(2.0, 16), (8.0, 15), (16.0, 14), (32.0, 13), (64.0, 12), (128.0, 11), (256.0, 10), (512.0, 9),
           (1024.0, 8), (2048.0, 7), (4096.0, 6), (8192.0, 5)]),
    _cell("Np = 2^16 DOG(3)", DOG, 3.0, 16, N16,
          [(2.0, 16), (8.0, 15), (16.0, 14), (32.0, 13), (64.0, 12), (128.0, 11), (256.0, 10), (512.0, 9),
           (1024.0, 8), (2048.0, 7), (4096.0, 6), (8192.0, 5)]),
    _cell("Np = 2^16 Paul(4)", PAUL, 4.0, 16, N16,
          [(2.0, 15), (16.0, 15), (50.0, 14), (100.0, 13), (200.0, 12), (400.0, 11), (800.0, 10), (1600.0, 9),
           (3200.0, 8), (6400.0, 7), (11000.0, 6)]),
    _cell("Np = 2^16 table", None, None, 16, N16, [(2.0, 16), (30.0, 16), (300.0, 16)],
          table=[(DOG, 2.0), (DOG, 3.0), (PAUL, 4.0)]),
    # three levels: dense pre-pass (K1 = 2, 4) and interleaved 2^20-point transforms; pruned two-kernel
    # rows of K' = 2^19 and 2^20 (at Np = 2^21 a Paul band has at most 2^20 bins: no dense Paul row)
    _cell("Np = 2^21 Morlet(6)", MORLET, 6.0, 21, [2 ** 21 - 3], [(2.0, 21), (4.0, 21), (16.0, 19)]),
    _cell("Np = 2^21 DOG(2)", DOG, 2.0, 21, [2 ** 21 - 3], [(2.0, 21), (4.0, 21), (16.0, 19)]),
    _cell("Np = 2^21 Paul(4)", PAUL, 4.0, 21, [2 ** 21 - 3], [(2.0, 20), (16.0, 20), (50.0, 19)]),
    _cell("Np = 2^22 Morlet(6)", MORLET, 6.0, 22, [2 ** 22 - 5], [(2.0, 22), (16.0, 20)], gpu_only=True),
    _cell("Np = 2^22 DOG(2)", DOG, 2.0, 22, [2 ** 22 - 5], [(2.0, 22), (16.0, 20)], gpu_only=True),
    _cell("Np = 2^22 Paul(4)", PAUL, 4.0, 22, [2 ** 22 - 5], [(2.0, 22), (50.0, 20)], gpu_only=True),
    # the cross-product epilogue (EPI_MULCONJ) on every exact class
    _cell("xwt Np = 2^20 DOG(2)", DOG, 2.0, 20, [2 ** 20 - 3], DOG20, xwt=True),
    _cell("xwt Np = 2^20 Paul(4)", PAUL, 4.0, 20, [2 ** 20 - 3],
          [(2.0, 20), (50.0, 20), (100.0, 17), (1600.0, 13), (12000.0, 10)], xwt=True),
    _cell("xwt Np = 2^16 DOG(2)", DOG, 2.0, 16, [2 ** 16 - 1],
          [(2.0, 16), (8.0, 15), (64.0, 12), (128.0, 11), (256.0, 10), (8192.0, 5)], xwt=True),
    _cell("xwt Np = 2^16 Paul(4)", PAUL, 4.0, 16, [2 ** 16 - 1],
          [(16.0, 15), (50.0, 14), (100.0, 13), (800.0, 10), (11000.0, 6)], xwt=True),
]


def _cell_ids():
    return [(c, n0) for c in CELLS for n0 in c["n0s"]]


def reference(cell, x, sj):
    """Reference rows of x: per row's family for a table cell."""
    if cell["table"] is None:
        return rp.ref_rows(x, 1.0, sj, cell["fam"], cell["par"])
    return np.concatenate([rp.ref_rows(x, 1.0, [s], fam, par) for s, (fam, par) in zip(sj, cell["table"])])


def run_cell(eng, cell, n0):
    """The cell's transform, plan and profile."""
    sj = cell["sj"]
    x = rp.white(n0)
    y2 = rp.white(n0, 9) if cell["xwt"] else None
    eng.set_expand_eps(0.0, 0.0)
    eng.set_band_eps(cell["band_eps"])
    try:
        eng.profile_begin()
        try:
            if cell["xwt"]:
                W = eng.xwt(x, y2, 1.0, sj, cell["fam"], cell["par"])
            elif cell["table"] is not None:
                Np = orc.next_pow2(n0)
                table = np.array([rp.response(Np, 1.0, s, fam, par, np.float64)
                                  for s, (fam, par) in zip(sj, cell["table"])])
                W = eng.cwt(x, 1.0, sj, TABLE, 0.0, table=table)
            else:
                W = eng.cwt(x, 1.0, sj, cell["fam"], cell["par"])
        finally:
            prof = eng.profile_end()
        plan = eng.last_plan(len(sj))
    finally:
        eng.set_expand_eps()
        eng.set_band_eps(BAND_EPS)
    return x, y2, W, plan, prof


def check_cell(eng, cell, n0):
    sj, log2N = cell["sj"], cell["log2N"]
    assert orc.next_pow2(n0) == 2 ** log2N
    if cell["gpu_only"] and _emulated(eng):
        pytest.skip("GPU-only: Np = %d on the host emulation" % 2 ** log2N)
    x, y2, W, plan, prof = run_cell(eng, cell, n0)
    # it ran as intended: the class of every row
    assert plan == cell["plan"], (cell["name"], n0, list(zip(sj, plan, cell["plan"])))
    # it is accurate
    ref = reference(cell, x, sj)
    if cell["xwt"]:
        ref = ref * np.conj(reference(cell, y2, sj))
    err = rp.row_err(W, ref)
    for j, p in enumerate(plan):
        print("  %-36s n0 = %-8d s = %-8g log2K' = %-3d row_err %.2e" % (cell["name"], n0, sj[j], p, err[j]))
    bound = 2 * EXACT if cell["xwt"] else EXACT         # a product of two rows: twice the rows' bound
    bad = {float(sj[j]): float(err[j]) for j in range(len(sj)) if not err[j] <= bound}
    assert not bad, (cell["name"], n0, bad)
    # and on the device through the kernels of its classes
    if not _emulated(eng):
        got, want = launched(prof), expected_kernels(plan, log2N)
        assert got == want, (cell["name"], sorted(got), sorted(want), prof)
    return err


@pytest.mark.gpu
@pytest.mark.parametrize("cell,n0", _cell_ids(), ids=["%s|n0=%d" % (c["name"], n0) for c, n0 in _cell_ids()])
def test_fp64_cell(eng, cell, n0):
    check_cell(eng, cell, n0)


SMALL_N0 = [1, 3, 31, 33, 511, 513]


@pytest.mark.gpu
@pytest.mark.parametrize("fam,par", [(DOG, 2.0), (PAUL, 4.0)], ids=["DOG(2)", "Paul(4)"])
@pytest.mark.parametrize("n0", SMALL_N0)
def test_fp64_small_transforms(eng, n0, fam, par):
    """Np = 1 .. 1024: TinyBody below 32 points, the single-kernel classes above."""
    sj = np.array([0.5, 1.0, 2.0, 4.0, 8.0, 16.0, 64.0])
    sj = sj[sj <= max(n0, 2)]
    x = rp.white(n0, 11)
    Np = orc.next_pow2(n0)
    eng.set_expand_eps(0.0, 0.0)
    try:
        eng.profile_begin()
        try:
            W = eng.cwt(x, 1.0, sj, fam, par)
        finally:
            prof = eng.profile_end()
        plan = eng.last_plan(len(sj))
    finally:
        eng.set_expand_eps()
    log2N = Np.bit_length() - 1
    assert all((p == 0) if Np < 32 else (5 <= p <= log2N) for p in plan), (n0, plan)
    err = rp.row_err(W, rp.ref_rows(x, 1.0, sj, fam, par))
    print("  %s(%d) n0 = %-4d plan %s, worst row_err %.2e" % (FAM_NAME[fam], par, n0, plan, err.max()))
    assert (err <= EXACT).all(), (n0, dict(zip(sj, err)))
    if not _emulated(eng):
        got, want = launched(prof), expected_kernels(plan, log2N)
        assert got == want, (n0, sorted(got), sorted(want), prof)


# ------------------------------------------------------------------------------------------------
# the transform hook
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("sign", [-1, 1])
@pytest.mark.parametrize("log2n", [20, 21])
def test_fft_c2c_rows(eng, log2n, sign):
    """Plain complex DFTs of 3 rows (engine.cu: fft_rows): PassABody MODE_CPLX then the register-resident
    PassBBody<double, sign, 1024>, behind a K0 = 2 pre-pass at n = 2^21.  Each row against a longdouble
    np.fft of the same input, relative to that row's maximum."""
    n, rows = 2 ** log2n, 3
    rs = np.random.RandomState(20 + log2n)
    x = rs.randn(rows, n) + 1j * rs.randn(rows, n)
    x[1] *= np.exp(-0.5 * ((np.arange(n) - n / 3) / (n / 50)) ** 2)      # a localised row: a smooth spectrum
    x[2] = np.exp(2j * np.pi * 12345.25 * np.arange(n) / n) + 1e-3 * x[2]  # one off-bin tone over noise
    eng.profile_begin()
    try:
        Y = eng.fft_c2c(x, sign)
    finally:
        prof = eng.profile_end()
    xl = x.astype(np.clongdouble)
    ref = np.fft.fft(xl, axis=1) if sign < 0 else np.fft.ifft(xl, axis=1) * n
    err = np.abs(Y - ref).max(axis=1) / np.abs(ref).max(axis=1)
    print("  fft_c2c n = 2^%d sign %+d: row errors %s" % (log2n, sign, " ".join("%.2e" % v for v in err)))
    assert np.isfinite(Y).all() and (err <= FFT_BOUND).all(), err
    if not _emulated(eng):
        want = {"PassABody<double,1024,3,%d>" % sign, "PassBBody<double,%d,1024,true>" % sign}
        if log2n > 20:
            want.add("PassABody<double,%d,3,%d>" % (2 ** (log2n - 20), sign))
        assert launched(prof) == want, prof
