"""Row-by-row parity of the generalized Morse family (CWTB_MORSE) against an extended-precision
reference, on the host emulation of the kernels.

The reference is the shape of `ref_rows` (test_gpu_row_parity.py): full-length band products in
np.longdouble from the forward FFT to the trim, with its own Morse response evaluated in log form
relative to the peak (`morse_response`).  Each row is measured against its own maximum (`row_err`,
fp64) or against sigma_j (`sigma_err`, fp32), at the bounds the fp64 and fp32 row-parity files hold
the other analytic families to: 1e-14 for an exact fp64 row, the expansion tolerance 5e-13 for an fp64
expansion row, 3e-6 / 1.2e-6 of sigma_j for an exact / expansion fp32 row.

Covered: every row class last_plan reports (expansion at several R, one- and two-kernel pruned rows,
dense rows, overlap-save rows, rows cut at Nyquist, un-padded Bluestein rows), in fp64 and fp32 where
the class exists there; the response table path against the native family; Morse(1, m) against Paul(m);
the resident plan not reused across a change of ga.
"""
import numpy as np
import pytest

import test_emu_overlap_save as osv
import test_gpu_fp32_row_parity as p32
import test_gpu_row_parity as rp
from oracle import cwt_oracle as orc

PAUL, TABLE, MORSE = 1, 3, 4
F64, F32 = 0, 1
LD = np.longdouble
EXACT, EPS64 = rp.EXACT, rp.EPS64
EXACT32, EXPAND32 = p32.EXACT32, p32.EXPAND32
OS = osv.OS


# ------------------------------------------------------------------------------------------------
# reference
# ------------------------------------------------------------------------------------------------
def morse_response(Np, dt, s, be, ga, dtype=LD):
    """F[k] = sqrt(s w1 Np) psi_ft(s omega_k) of Morse(ga, be) on the Np signed bins, in `dtype`:
    psi_ft(f) = psi_ft(f_p) exp(be u - (be/ga) expm1(ga u)), u = ln(f / f_p), f_p = (be/ga)^(1/ga)."""
    from scipy.special import gammaln
    T = np.dtype(dtype).type
    pi = 4 * np.arctan(T(1))
    ga_, be_ = T(ga), T(be)
    k = (np.fft.fftfreq(Np) * Np).astype(T)
    f = T(s) * (2 * pi * k / (T(Np) * T(dt)))
    bg = be_ / ga_
    lnfp = np.log(bg) / ga_
    r = (2 * be + 1) / ga
    lnA = T(0.5) * (np.log(ga_) + T(r) * np.log(T(2)) - T(gammaln(r)))    # lgamma in double: within an ulp
    lnpk = lnA + be_ * lnfp - bg
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        u = np.log(np.where(f > 0, f, T(1))) - lnfp
        v = np.exp(lnpk + be_ * u - bg * np.expm1(ga_ * u))
    norm = np.sqrt(T(s) * (2 * pi / (T(Np) * T(dt))) * T(Np))
    return norm * np.where(f > 0, v, T(0))


def morse_rows(x, dt, scales, be, ga, n0=None, npad=None, dtype=LD):
    """ref_rows for Morse(ga, be), complex128 [S, n0]."""
    x = np.asarray(x, dtype=np.float64)
    n0 = x.size if n0 is None else n0
    Np = npad or orc.next_pow2(x.size)
    X = np.fft.fft(x.astype(dtype), Np)
    out = np.empty((len(scales), n0), dtype=np.complex128)
    for j, s in enumerate(np.asarray(scales, dtype=np.float64)):
        out[j] = np.fft.ifft(X * morse_response(Np, dt, s, be, ga, dtype))[:n0]
    return out


def lift(Np, dt, s, be, ga):
    """psi_ft's peak over its largest value on the row's grid: 1 when the peak lies below Nyquist.  The
    band is pruned at band_eps of the peak, so a row whose peak lies past Nyquist carries that error
    times this factor relative to its own maximum."""
    k = np.arange(1, Np // 2 + 1)
    u = np.log(s * 2 * np.pi * k / (Np * dt)) - np.log(be / ga) / ga
    return float(np.exp(-(be * u - (be / ga) * np.expm1(ga * u)).max()))


def morse_ref32(x, dt, sj, be, ga, n0=None):
    """fp32 reference rows and sigma_j (p32.ref32 for Morse)."""
    x = np.asarray(x, dtype=np.float64)
    Np = orc.next_pow2(x.size)
    R = morse_rows(x, dt, sj, be, ga, n0=n0, dtype=np.float64)
    nx = np.linalg.norm(x)
    nu = np.array([nx * np.linalg.norm(morse_response(Np, dt, s, be, ga, np.float64)) / Np for s in sj])
    return R, np.maximum(np.abs(R).max(axis=1), nu)


def test_reference_matches_paul():
    """CPU: Morse(1, m)'s reference response is Paul(m)'s (the engine's Paul constant) to 1e-15."""
    for m in (1, 4, 12):
        for s in (0.5, 3.0, 40.0):
            a = morse_response(2 ** 12, 1.0, s, float(m), 1.0)
            b = rp.response(2 ** 12, 1.0, s, PAUL, float(m))
            assert np.abs(a - b).max() <= 1e-15 * np.abs(b).max(), (m, s)


# ------------------------------------------------------------------------------------------------
# engine
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    e = osv.make_engine(osv.emu_lib(), CWTB_EXPAND_MIN_R="2")
    assert "emulation" in e.version()
    yield e
    e.close()


def kind(p, log2N):
    """The class of a last_plan entry."""
    if p == OS:
        return "overlap-save"
    if p == -1:
        return "unpadded"
    if p < 0:
        return "expansion R=%d" % 2 ** (log2N + p)
    if p == log2N:
        return "dense"
    if p <= 10:
        return "pruned one-kernel"
    return "pruned two-kernel"


N0 = 50001                                       # Np = 2^16
SJ = 0.5 * 2 ** (np.arange(0, 40) / 3.0)      # s = 0.5 .. 4e3 (below 1, the rows are cut at Nyquist)
GA_BE = [(3.0, 20.0), (2.0, 4.5), (1.0, 3.0)]


def _classes(plan, sj, Np, be, ga, log2N):
    """Per-row class names, with rows whose band reaches Nyquist named apart."""
    out = []
    for p, s in zip(plan, sj):
        name = kind(p, log2N)
        resp = morse_response(Np, 1.0, s, be, ga, np.float64)
        if abs(resp[Np // 2 - 1]) > 1e-16 * np.abs(resp).max():     # the last positive bin
            name += " (cut at Nyquist)"
        out.append(name)
    return out


def run_fp64(emu, ga, be):
    """The fp64 rows of SJ checked row by row; the set of their class names."""
    x = rp.white(N0, 3)
    Np, log2N = 2 ** 16, 16
    W = emu.cwt(x, 1.0, SJ, MORSE, (be, ga))
    plan = emu.last_plan(len(SJ))
    err = rp.row_err(W, morse_rows(x, 1.0, SJ, be, ga))
    names = _classes(plan, SJ, Np, be, ga, log2N)
    for s, n, e in zip(SJ, names, err):
        print("  Morse(%g, %g) fp64 s = %-9.4g %-36s row_err %.2e" % (ga, be, s, n, e))
    for j, p in enumerate(plan):
        bound = (EPS64 if (p < 0 and p != OS) else EXACT) * max(1.0, lift(Np, 1.0, SJ[j], be, ga))
        assert err[j] <= bound, (SJ[j], names[j], err[j])
    return set(names)


@pytest.mark.parametrize("ga,be", GA_BE)
def test_rows_fp64(emu, ga, be):
    run_fp64(emu, ga, be)


SJ_EXACT = np.array([0.5, 1.0, 2.0, 64.0, 4096.0])


def run_fp64_exact(emu, ga, be):
    """Np = 2^20 with the expansion off: dense rows (through the dense margin: a band of positive
    frequencies never spans Np bins), two-kernel and one-kernel pruned rows."""
    n0, Np, log2N = 2 ** 20 - 3, 2 ** 20, 20
    x = rp.white(n0, 6)
    emu.set_expand_eps(0.0, 0.0)
    try:
        W = emu.cwt(x, 1.0, SJ_EXACT, MORSE, (be, ga))
        plan = emu.last_plan(len(SJ_EXACT))
    finally:
        emu.set_expand_eps()
    err = rp.row_err(W, morse_rows(x, 1.0, SJ_EXACT, be, ga))
    names = _classes(plan, SJ_EXACT, Np, be, ga, log2N)
    for s, n, e in zip(SJ_EXACT, names, err):
        print("  Morse(%g, %g) fp64 Np = 2^20 s = %-7g %-36s row_err %.2e" % (ga, be, s, n, e))
    for j in range(len(plan)):
        assert err[j] <= EXACT * max(1.0, lift(Np, 1.0, SJ_EXACT[j], be, ga)), (SJ_EXACT[j], names[j], err[j])
    return set(names)


def test_rows_fp64_exact_classes(emu):
    run_fp64_exact(emu, 3.0, 20.0)


@pytest.mark.parametrize("ga,be", GA_BE)
def test_rows_fp32(emu, ga, be):
    x = rp.white(N0, 5).astype(np.float32)
    log2N = 16
    W = emu.cwt(x, 1.0, SJ, MORSE, (be, ga), precision=F32)
    plan = emu.last_plan(len(SJ))
    R, sig = morse_ref32(x, 1.0, SJ, be, ga)
    err = p32.sigma_err(W, R, sig)
    for s, p, e in zip(SJ, plan, err):
        print("  Morse(%g, %g) fp32 s = %-9.4g %-22s err/sigma %.2e" % (ga, be, s, kind(p, log2N), e))
    for j, p in enumerate(plan):
        assert err[j] <= (EXPAND32 if p < 0 else EXACT32), (SJ[j], kind(p, log2N), err[j])


def test_every_class_is_hit(emu):
    """fp64 at Np = 2^16 (padded) and un-padded: every class of last_plan has at least one Morse row."""
    seen = set()
    for ga, be in GA_BE:
        seen |= run_fp64(emu, ga, be)
    seen |= run_fp64_exact(emu, 3.0, 20.0)
    # un-padded (Bluestein) rows
    x = rp.white(3001, 7)
    sj = np.array([0.5, 2.0, 9.0, 60.0])
    emu.set_padding(False)
    try:
        W = emu.cwt(x, 1.0, sj, MORSE, (20.0, 3.0))
        plan = emu.last_plan(len(sj))
    finally:
        emu.set_padding(True)
    err = rp.row_err(W, morse_rows(x, 1.0, sj, 20.0, 3.0, npad=3001))
    assert plan == [-1] * len(sj) and (err <= EXACT).all(), (plan, err)
    seen.add("unpadded")
    kinds = {n.split(" (")[0].split(" R=")[0] for n in seen}
    rs = {n for n in seen if n.startswith("expansion R=")}
    print("  classes:", sorted(seen), kinds)
    assert {"dense", "pruned one-kernel", "pruned two-kernel", "overlap-save", "expansion", "unpadded"} <= kinds
    assert len(rs) >= 3, rs
    assert any("cut at Nyquist" in n for n in seen)


def test_table_equals_family(emu):
    """A duck-typed object with Morse's psi_ft runs through CWTB_TABLE and agrees with the family."""
    import pycwt_b200 as pycwt
    from pycwt_b200.mothers import Morse

    class Duck(object):
        def __init__(self):
            self._m = Morse(3, 20)

        def psi_ft(self, f):
            return self._m.psi_ft(f)

        def flambda(self):
            return self._m.flambda()

        def coi(self):
            return self._m.coi()

    n0 = 4001
    x = rp.white(n0, 4)
    sj = np.array([1.0, 4.0, 30.0, 300.0])
    Np = orc.next_pow2(n0)
    emu.set_expand_eps(0.0, 0.0)
    try:
        table = pycwt.wavelet._response_table(Duck(), sj, Np, 1.0)
        Wt = emu.cwt(x, 1.0, sj, TABLE, 0.0, table=table)
        Wf = emu.cwt(x, 1.0, sj, MORSE, (20.0, 3.0))
    finally:
        emu.set_expand_eps()
    ref = morse_rows(x, 1.0, sj, 20.0, 3.0)
    for W in (Wt, Wf):
        assert (rp.row_err(W, ref) <= EXACT).all()
    assert (rp.row_err(Wt, Wf) <= EXACT).all()


@pytest.mark.parametrize("m", [1, 4, 12])
def test_morse_ga1_equals_paul(emu, m):
    """Morse(1, m) rows equal Paul(m) rows within 1e-13 of each row's maximum (not bit for bit: the
    response is evaluated differently), beyond the rows' pruning error when Paul's peak lies past
    Nyquist (`lift`)."""
    x = rp.white(N0, 8)
    Wm = emu.cwt(x, 1.0, SJ, MORSE, (float(m), 1.0))
    pm = emu.last_plan(len(SJ))
    Wp = emu.cwt(x, 1.0, SJ, PAUL, float(m))
    assert pm == emu.last_plan(len(SJ))
    d = rp.row_err(Wm, Wp) / np.maximum(1.0, [lift(2 ** 16, 1.0, s, float(m), 1.0) for s in SJ])
    print("  Morse(1, %d) against Paul(%d): worst row %.2e" % (m, m, d.max()))
    assert (d <= 1e-13).all(), d


def test_plan_not_reused_across_ga(emu):
    """The same (family, be, geometry) with another ga plans again: the rows follow ga."""
    x = rp.white(N0, 9)
    sj = SJ[::4]
    W3 = emu.cwt(x, 1.0, sj, MORSE, (20.0, 3.0))
    W2 = emu.cwt(x, 1.0, sj, MORSE, (20.0, 2.0))
    W3b = emu.cwt(x, 1.0, sj, MORSE, 20.0)          # be alone: ga = 3
    for W, ga in ((W3, 3.0), (W2, 2.0), (W3b, 3.0)):
        err = rp.row_err(W, morse_rows(x, 1.0, sj, 20.0, ga))
        assert (err <= EPS64).all(), (ga, err)
    assert np.array_equal(W3, W3b)


def test_argument_errors(emu):
    from pycwt_b200._engine import EngineError
    x = rp.white(1024)
    for be, ga in ((0.5, 3.0), (257.0, 3.0), (20.0, 0.5), (20.0, 13.0)):
        with pytest.raises(EngineError):
            emu.cwt(x, 1.0, [2.0], MORSE, (be, ga))
    assert emu.lib.cwtb_set_morse_ga(emu.h, 12.5) == -1
