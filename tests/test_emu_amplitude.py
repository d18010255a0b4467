"""Amplitude invariance of every product, checked on the host-emulation build of the kernels.

The engine has no data-dependent threshold: band pruning, the overlap-save truncation and the
expansion planner depend on the wavelet and the geometry only.  So scaling the input by a power of
two scales every intermediate by a power of two, which is exact while every intermediate stays in
the normal range.  Data in physical units (strain near 1e-21, counts near 1e9) with
`normalize=False` rely on that, and a data-derived threshold, a magnitude-keyed pruning rule or a
flush-to-zero flag would break it.  Asserted, for inputs scaled by 2^k (a pair by 2^a and 2^b with
a != b so that swapped series cannot pass):

  * W(2^k x) = 2^k W(x) and icwt, bit for bit, with the same plan (`last_plan`);
  * W12 -> 2^(a+b) W12 bit for bit (`xwt`, `xwt_resident`);
  * WCT, aWCT, RP2, RM2 and the partial phase unchanged bit for bit, a pair scaled by 2^a and 2^b
    and a triple by three different exponents (as far apart as 2^COH and 2^-COH: series in
    different units), and with a fixed seed the surrogate levels, the exceedance counts, the
    p-values, the FDR threshold and the clusters.  With `normalize=False` the coherence paths bring
    each series into [1/2, 1) by an exact power of two first (wavelet.py: `_unit_binade`): the
    pipeline smooths the two auto-spectra as the real and imaginary parts of one complex field, and
    without it the rounding of the larger would leak into the smaller by about 2^(2 |a - b|) ulp;
  * `normalize=True`: every product unchanged (the standardisation is exact under 2^k);
  * reductions the device forms with floating-point atomics (PowerBody's row sums, the multi-block
    ScaleAvgBody and IcwtBody), whose order of additions is not fixed on the device: within
    ATOMIC_TOL of 2^(degree k) times the unscaled result.

Largest |k| tested, per product (degree in the input) and precision; beyond it an intermediate
leaves the normal range (DESIGN.md section 6):

  product                                        degree   fp64   fp32
  cwt W, icwt, resident wave / window            1        900     64
  |W|^2 sums                                     2        450     48
  xwt / xwt_resident W12 (their red-noise level  4        200     48
    fits ar1 to the raw series: quartic sums)
  wct, partial / multiple coherence, resident    -        450    450
    coherence, surrogates and clusters (host: the
    std of the raw series, computed on every call)
  normalize=True (xwt's ar1 of the raw series)   4        200    200

The fp64 limits come from the squares and fourth powers of |W| s^-1/2: W of a unit series is O(1)
to O(sqrt(s)), so the degree-d intermediate reaches 2^(d k) and leaves fp64's exponent range
(2^-1022 .. 2^1024) near d |k| = 1000 with the response and the scale factors.  fp32 W is linear
but its forward spectrum grows by up to Np.  The coherence products see series in [1/2, 1)
whatever k, so no device intermediate bounds them.  On the engine's own `wct` (no host scaling,
`test_fp32_wct_against_longdouble_reference`) the fp32 coherence forms its smoothed fields
(degree 2) in float and their ratio in double: it holds while the fields do, to 2^+-32 at 2^18
points (DESIGN.md section 6).

One cell checks fp32 WCT at k = +-40 against the extended-precision reference of
test_gpu_coherence_parity.py (np.longdouble has a 15-bit exponent), under that file's error model.
tests/test_gpu_amplitude.py runs the same checks on the device at the configs' geometries.
"""
import os

import numpy as np
import pytest

from conftest import ROOT

F64, F32 = 0, 1
MORLET, PAUL, DOG, TABLE = 0, 1, 2, 3
PREC = {F64: 'fp64', F32: 'fp32'}
# largest |k| per degree in the input and engine precision (the module table)
# fp32 linear: 2^100 overflows nothing below Np = 2^28, but from 2^-80 down products
# inside the fp32 row transforms (a response or twiddle value times a spectral value) leave float's
# normal range (2^-126): TinyBody at 2^-90, a 2^16-point row at 2^-100, a 2^18-point Paul row at 2^-80
RANGE = {(1, F64): 900, (1, F32): 64,
         (2, F64): 450, (2, F32): 48,
         (4, F64): 200, (4, F32): 48}
# xwt, xwt_resident: degree 4, since their red-noise level fits ar1 to the raw series (quartic sums)
XWT = 4
# the coherence products: the series reach the device in [1/2, 1); the host's std of the raw series
# (computed on every call, used by xwt only) is quadratic
COH_RANGE = 450
NORM_RANGE = 200      # xwt fits ar1 to the raw series whatever `normalize`: quartic sums
ATOMIC_TOL = 1e-13


def ends(deg, prec):
    """Exponents near both ends of the range of a product of degree `deg`."""
    k = RANGE[(deg, prec)]
    return (k, -k)


def pair_exps(deg, prec):
    """(a, b), a != b, near each end of the range of a product of degree `deg`."""
    k = RANGE[(deg, prec)]
    return [(k, k - 3), (-k + 5, -k)]


def coh_exps(nser):
    """Exponents of the series of a coherence product: different for every series, near each end of
    the range, and the two ends at once."""
    k = COH_RANGE
    if nser == 2:
        return [(k, k - 3), (-k + 5, -k), (k, -k)]
    return [(k, k - 2, k - 5), (-k + 3, -k, -k + 7), (k, -k, 1)]


def assert_scaled(got, ref, e, name):
    """got == 2^e ref bit for bit (ldexp is exact in the normal range)."""
    want = np.ldexp(ref.real, e) + 1j * np.ldexp(ref.imag, e) if np.iscomplexobj(ref) else np.ldexp(ref, e)
    want = np.asarray(want, dtype=np.asarray(ref).dtype)
    assert np.isfinite(ref).all() or np.array_equal(np.isnan(got), np.isnan(ref)), name
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    assert not bad.any(), (name, e, int(bad.sum()), np.argwhere(bad)[:3].tolist())


def assert_close_scaled(got, ref, e, name, tol=ATOMIC_TOL):
    """A sum formed with atomics: within tol of 2^e ref, relative to the largest |2^e ref|."""
    ref, got = np.asarray(ref), np.asarray(got)
    want = np.ldexp(ref.real, e) + 1j * np.ldexp(ref.imag, e) if np.iscomplexobj(ref) else np.ldexp(ref, e)
    assert got.shape == want.shape and np.array_equal(np.isnan(got), np.isnan(want)), name
    ok = ~np.isnan(want)
    m = np.abs(want[ok]).max() if ok.any() else 0.0
    assert m > 0 and np.isfinite(m), (name, e, m)
    assert (np.abs(got[ok] - want[ok]) <= tol * m).all(), (name, e, np.abs(got[ok] - want[ok]).max() / m)


def assert_same(got, ref, name):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape and got.dtype == ref.dtype, (name, got.shape, ref.shape)
    bad = ~((got == ref) | (np.isnan(got) & np.isnan(ref)))
    assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:3].tolist(),
                           got[bad][:3].tolist(), ref[bad][:3].tolist())


def signal(n0, seed=0):
    """A chirp plus noise: every scale carries signal."""
    rs = np.random.RandomState(seed)
    t = np.arange(n0) / n0
    return np.sin(2 * np.pi * (40 * t + (n0 / 10) * t ** 2)) + 0.3 * rs.randn(n0)


def series(n0, count, seed=0):
    """`count` partly coherent series: a shared sinusoid under independent noise."""
    rs = np.random.RandomState(seed)
    t = np.arange(n0)
    base = np.sin(2 * np.pi * t / 37.0) + 0.5 * np.sin(2 * np.pi * t / 150.0)
    return [base + (0.4 + 0.2 * i) * rs.randn(n0) + 0.3 * np.roll(base, 5 * i) for i in range(count)]


# ------------------------------------------------------------------------------------------------
# transforms: Engine.cwt over the exact classes, overlap-save, both expansion kernels, the coarse
# launches, a response table and Bluestein
# ------------------------------------------------------------------------------------------------
def response_table(Np, dt, sj):
    """Rows of a response table (the duck-typed wavelet path): Morlet(6), DOG(2) and Paul(4) rows."""
    import test_gpu_row_parity as rp
    fams = [(MORLET, 6.0), (DOG, 2.0), (PAUL, 4.0)]
    return np.array([rp.response(Np, dt, s, *fams[j % 3], np.float64) for j, s in enumerate(sj)])


def cwt_cell(name, n0, sj, fam, par, precs, classes, pad=True, table=False):
    """`classes`: predicates on the plan that the cell must meet, one for every class it names; a
    dict {precision: predicates} where the precisions plan differently."""
    return dict(name=name, n0=n0, sj=np.asarray(sj, float), fam=fam, par=par, precs=precs,
                classes=classes, pad=pad, table=table)


def dense(log2N):
    return lambda p: log2N in p


def has(*codes):
    return lambda p: all(c in p for c in codes)


def expansion(p):
    return any(c < -2 for c in p)


def single(p):
    return any(5 <= c <= 10 for c in p)


def overlap_save(p):
    return -2 in p


def direct(log2N):
    return lambda p: any(11 <= c <= 13 and c < log2N for c in p)


def two_kernel(log2N):
    return lambda p: any(13 < c < log2N for c in p)


def coarse_ragged(p):
    """Expansion rows of coarse length <= 1024: the ragged coarse launch."""
    return any(-10 <= c < -2 for c in p)


def coarse_pair(p):
    """Expansion rows of coarse length > 1024: the coarse launch pair."""
    return any(c < -10 for c in p)


def bluestein(p):
    return len(p) > 0 and set(p) == {-1}


def check_cwt_cell(eng, cell, prec, x=None, exps=None):
    """W of the scaled signal equals the scaled W bit for bit, with the same plan; then the plan
    covers the cell's classes."""
    from oracle import cwt_oracle as orc
    x = signal(cell["n0"]) if x is None else x
    sj = cell["sj"]
    table = response_table(orc.next_pow2(cell["n0"]) if cell["pad"] else cell["n0"], 1.0, sj) \
        if cell["table"] else None
    fam = TABLE if cell["table"] else cell["fam"]
    eng.set_padding(cell["pad"])
    try:
        W0 = eng.cwt(x, 1.0, sj, fam, cell["par"] or 0.0, prec, table=table)
        plan = eng.last_plan(len(sj))
        for k in exps or ends(1, prec):
            W = eng.cwt(np.ldexp(x, k), 1.0, sj, fam, cell["par"] or 0.0, prec, table=table)
            assert eng.last_plan(len(sj)) == plan, (cell["name"], k)
            assert_scaled(W, W0, k, "%s W %s" % (cell["name"], PREC[prec]))
    finally:
        eng.set_padding(True)
    assert np.isfinite(W0).all(), cell["name"]
    classes = cell["classes"]
    for c in classes[prec] if isinstance(classes, dict) else classes:
        assert c(plan), (cell["name"], PREC[prec], plan)
    return plan


SJ16 = 2.0 * 2 ** (np.arange(0, 60) / 6.0)     # Np = 2^16: coarse lengths 2^7 .. 2^13
CWT_CELLS = [
    cwt_cell("Np = 2^16 Morlet: dense, overlap-save (fp64), two-kernel (fp32), direct, expansion with "
             "both coarse launches", 50001, SJ16, MORLET, 6.0, (F64, F32),
             {F64: [dense(16), overlap_save, direct(16), expansion, coarse_ragged, coarse_pair],
              F32: [dense(16), two_kernel(16), direct(16), expansion, coarse_ragged, coarse_pair]}),
    cwt_cell("Np = 2^16 Paul(4): two-kernel and expansion rows", 50001,
             [2.0, 16.0, 50.0, 100.0, 200.0, 800.0, 3200.0], PAUL, 4.0, (F64, F32),
             [two_kernel(16), expansion]),
    cwt_cell("Np = 2^13 Morlet: dense pair, direct, single, expansion, overlap-save (fp64)", 8192,
             2.0 * 2 ** (np.arange(45) / 4.0), MORLET, 6.0, (F64, F32),
             {F64: [dense(13), has(12, 11), has(10), expansion, overlap_save],
              F32: [dense(13), has(12, 11), has(10), expansion]}),
    cwt_cell("Np = 2^13 DOG(2): overlap-save", 8192, 2.0 * 2 ** (np.arange(30) / 4.0), DOG, 2.0,
             (F64,), [overlap_save]),
    cwt_cell("Np = 16 DOG(2): TinyBody", 13, [0.5, 1.0, 2.0, 4.0], DOG, 2.0, (F64, F32), [has(0)]),
    cwt_cell("Np = 1024 Paul(4): single-kernel classes", 1000, 2.0 * 2 ** (np.arange(24) / 4.0), PAUL,
             4.0, (F64, F32), [single]),
    cwt_cell("Np = 2^12 response table", 4001, [1.0, 2.0, 30.0, 300.0], None, None, (F64, F32),
             [has(12)], table=True),
    cwt_cell("n0 = 1001 un-padded (Bluestein)", 1001, 2.0 * 2 ** (np.arange(20) / 4.0), MORLET, 6.0,
             (F64,), [bluestein], pad=False),
]


@pytest.fixture(scope="module")
def emu():
    from pycwt_b200 import build as _build, _engine
    lib = _build.build_emulation(os.path.join(ROOT, "tests", "_emu"))
    eng = _engine.Engine(0, lib_path=lib)
    assert "emulation" in eng.version()
    yield eng
    eng.close()


@pytest.fixture
def api(emu, monkeypatch):
    """The public API on the emulation build."""
    import pycwt_b200
    from pycwt_b200 import _engine
    monkeypatch.setattr(_engine, "default_engine", lambda *a, **k: emu)
    return pycwt_b200


def _cwt_ids():
    return [(c, p) for c in CWT_CELLS for p in c["precs"]]


@pytest.mark.parametrize("cell,prec", _cwt_ids(), ids=["%s|%s" % (c["name"], PREC[p]) for c, p in _cwt_ids()])
def test_engine_cwt(emu, cell, prec):
    check_cwt_cell(emu, cell, prec)


def test_cells_cover_both_expansion_kernels(emu):
    """The DMMA fp64 and the scalar fp32 expansion kernels both run in the cells above."""
    cell = CWT_CELLS[0]
    for prec in (F64, F32):
        assert expansion(check_cwt_cell(emu, cell, prec, exps=(1,)))


def check_cwt_batch(eng, X, sj, fam, par, prec, exps):
    """cwt_batch: per channel c scaled by 2^e_c, W exactly scaled and the row sums of |W|^2 within
    ATOMIC_TOL of 2^(2 e_c) times the unscaled ones."""
    P0, W0 = eng.cwt_batch(X, 1.0, sj, fam, par, prec, want_power=True, want_w=True)
    plan = eng.last_plan(len(sj))
    for e in exps:
        Xs = np.stack([np.ldexp(x, int(k)) for x, k in zip(X, e)]).astype(X.dtype)
        P, W = eng.cwt_batch(Xs, 1.0, sj, fam, par, prec, want_power=True, want_w=True)
        assert eng.last_plan(len(sj)) == plan
        for c, k in enumerate(e):
            assert_scaled(W[c], W0[c], int(k), "cwt_batch W channel %d" % c)
            assert_close_scaled(P[c], P0[c], 2 * int(k), "cwt_batch power channel %d" % c)


@pytest.mark.parametrize("prec", [F64, F32])
def test_cwt_batch(emu, prec):
    X = np.stack([signal(4096, seed) for seed in range(3)])
    k = RANGE[(2, prec)]
    check_cwt_batch(emu, X, 2.0 * 2 ** (np.arange(36) / 4.0), MORLET, 6.0, prec,
                    [(k, -k, 1), (-k + 1, 3, k - 1)])
    if prec == F32:   # float32 input, the fp32 engine's own element type
        check_cwt_batch(emu, X.astype(np.float32), 2.0 * 2 ** (np.arange(36) / 4.0), DOG, 2.0, prec,
                        [(k, 2 - k, 0)])


def check_public_cwt(api, x, kw, ks):
    """`cwt`: W and the signal's spectrum scale by 2^k, sj / freqs / coi do not move; `icwt` of the
    result (IcwtBody: an atomic sum over scales) within ATOMIC_TOL of 2^k times the unscaled one."""
    W0, sj0, f0, coi0, fft0, _ = api.cwt(x, 1.0, **kw)
    r0 = api.icwt(W0, sj0, 1.0, kw.get("dj", 1 / 12), kw.get("wavelet", "morlet"))
    for k in ks:
        W, sj, f, coi, fft, _ = api.cwt(np.ldexp(x, k), 1.0, **kw)
        assert_scaled(W, W0, k, "cwt W")
        assert_scaled(fft, fft0, k, "cwt fft")
        assert_same(sj, sj0, "sj")
        assert_same(coi, coi0, "coi")
        assert_close_scaled(api.icwt(W, sj, 1.0, kw.get("dj", 1 / 12), kw.get("wavelet", "morlet")), r0, k,
                            "icwt")


def test_public_cwt_and_icwt(api):
    x = signal(3000, 2)
    check_public_cwt(api, x, dict(dj=1 / 8, s0=2.0, J=60), ends(1, F64))
    check_public_cwt(api, x, dict(dj=1 / 4, s0=1.0, J=30, wavelet=api.DOG(2)), ends(1, F64))


def check_resident_transform(api, eng, x, kw, ks):
    """cwt_resident: wave / window / power exact; the row sums and scale averages within ATOMIC_TOL."""
    def products(h):
        return dict(wave=h.wave(), window=h.window(slice(1, None, 3), slice(5, None, 7)),
                    power=h.power(), gp=h.global_power(), gpc=h.global_power(inside_coi=True),
                    sa=h.scale_avg_power(8.0, 64.0), icwt=h.icwt())
    ref = products(api.cwt_resident(x, 1.0, engine=eng, **kw))
    deg = dict(wave=1, window=1, power=2, gp=2, gpc=2, sa=2, icwt=1)
    for k in ks:
        got = products(api.cwt_resident(np.ldexp(x, k), 1.0, engine=eng, **kw))
        for name in ("wave", "power"):
            assert_scaled(got[name], ref[name], deg[name] * k, "resident " + name)
        for name in ("gp", "gpc", "sa", "icwt"):
            assert_close_scaled(got[name], ref[name], deg[name] * k, "resident " + name)
        for part in (0, 1) if isinstance(got["window"], tuple) else (None,):
            g = got["window"] if part is None else got["window"][part]
            r = ref["window"] if part is None else ref["window"][part]
            assert_scaled(g, r, k, "resident window")


def test_resident_transform(api, emu):
    check_resident_transform(api, emu, signal(5000, 4), dict(dj=1 / 8, s0=2.0, J=80), ends(2, F64))


# ------------------------------------------------------------------------------------------------
# cross spectrum, coherence, partial and multiple coherence
# ------------------------------------------------------------------------------------------------
KW = dict(dj=1 / 4, s0=2.0, J=20)


def check_xwt(api, y, kw, prec, exps):
    W0 = api.xwt(y[0], y[1], 1.0, normalize=False, precision=PREC[prec], **kw)[0]
    assert np.isfinite(W0).all()
    for a, b in exps:
        W = api.xwt(np.ldexp(y[0], a), np.ldexp(y[1], b), 1.0, normalize=False, precision=PREC[prec], **kw)[0]
        assert_scaled(W, W0, a + b, "xwt W12 %s (%d, %d)" % (PREC[prec], a, b))


def check_wct(api, y, kw, prec, exps):
    WCT0, aWCT0 = api.wct(y[0], y[1], 1.0, sig=False, normalize=False, precision=PREC[prec], **kw)[:2]
    assert np.isfinite(WCT0).all()
    for a, b in exps:
        WCT, aWCT = api.wct(np.ldexp(y[0], a), np.ldexp(y[1], b), 1.0, sig=False, normalize=False,
                            precision=PREC[prec], **kw)[:2]
        tag = "wct %s (%d, %d)" % (PREC[prec], a, b)
        assert_same(WCT, WCT0, "WCT " + tag)
        assert_same(aWCT, aWCT0, "aWCT " + tag)


def check_wct3(api, y, kw, prec, exps):
    RP0 = api.partial_wct(*y, 1.0, normalize=False, precision=PREC[prec], **kw)[0]
    RM0 = api.multiple_wct(*y, 1.0, normalize=False, precision=PREC[prec], **kw)[0]
    assert np.isfinite(RP0).all() and np.isfinite(RM0).all()
    for e in exps:
        ys = [np.ldexp(v, k) for v, k in zip(y, e)]
        assert_same(api.partial_wct(*ys, 1.0, normalize=False, precision=PREC[prec], **kw)[0], RP0,
                    "partial_wct %s %s" % (PREC[prec], e))
        assert_same(api.multiple_wct(*ys, 1.0, normalize=False, precision=PREC[prec], **kw)[0], RM0,
                    "multiple_wct %s %s" % (PREC[prec], e))


@pytest.mark.parametrize("prec", [F64, F32])
def test_xwt(api, prec):
    check_xwt(api, series(1000, 2), KW, prec, pair_exps(XWT, prec))


@pytest.mark.parametrize("prec", [F64, F32])
def test_wct(api, prec):
    check_wct(api, series(1000, 2), KW, prec, coh_exps(2))


@pytest.mark.parametrize("prec", [F64, F32])
def test_partial_multiple_wct(api, prec):
    check_wct3(api, series(1000, 3), KW, prec, coh_exps(3))


@pytest.mark.parametrize("prec", [F64, F32])
def test_normalize_true(api, prec):
    """With normalize=True the standardised series are the same bits: every product is unchanged."""
    y = series(1000, 3, seed=1)
    p = PREC[prec]
    ref = (api.xwt(y[0], y[1], 1.0, precision=p, **KW)[0],
           *api.wct(y[0], y[1], 1.0, sig=False, precision=p, **KW)[:2],
           api.partial_wct(*y, 1.0, precision=p, **KW)[0], api.multiple_wct(*y, 1.0, precision=p, **KW)[0])
    for e in ((NORM_RANGE, -NORM_RANGE, 17), (-NORM_RANGE + 1, NORM_RANGE - 2, -40)):
        ys = [np.ldexp(v, k) for v, k in zip(y, e)]
        got = (api.xwt(ys[0], ys[1], 1.0, precision=p, **KW)[0],
               *api.wct(ys[0], ys[1], 1.0, sig=False, precision=p, **KW)[:2],
               api.partial_wct(*ys, 1.0, precision=p, **KW)[0], api.multiple_wct(*ys, 1.0, precision=p, **KW)[0])
        for name, g, r in zip(("xwt", "WCT", "aWCT", "RP2", "RM2"), got, ref):
            assert_same(g, r, "normalize=True %s %s %s" % (name, p, e))


def test_fp32_wct_against_longdouble_reference(emu):
    """fp32 WCT of series scaled by 2^40 and 2^-40 against the longdouble
    reference fed the engine's own fp32 transforms, within test_gpu_coherence_parity's EPS kappa."""
    import test_gpu_coherence_parity as cp
    from oracle import cwt_oracle as orc
    y1, y2 = cp.white_pair(1000, 3)
    sj = 2.0 * 2 ** (np.arange(21) / 4.0)
    K = 3
    for a, b in ((40, 40), (-40, -40)):
        u1, u2 = np.ldexp(y1, a), np.ldexp(y2, b)
        WCT = emu.wct(u1, u2, 1.0, 0.25, sj, MORLET, 6.0, K, precision=F32)[0]
        W1 = emu.cwt(u1, 1.0, sj, MORLET, 6.0, precision=F32)
        W2 = emu.cwt(u2, 1.0, sj, MORLET, 6.0, precision=F32)
        R, _, kappa = cp.ref_coherence(W1, W2, 1.0, sj, K, orc.next_pow2(1000))
        assert np.isfinite(WCT).all(), (a, b)
        q = np.abs(WCT - R) / kappa
        print("  fp32 WCT (2^%d, 2^%d): worst |WCT - R| / kappa %.2e" % (a, b, q.max()))
        assert q.max() <= cp.EPS[F32], (a, b, float(q.max()))


# ------------------------------------------------------------------------------------------------
# resident handles and the surrogate tests
# ------------------------------------------------------------------------------------------------
def check_resident_cross(api, eng, y, kw, prec, exps):
    def products(h):
        return dict(W12=h.cross_spectrum(), win=h.window(slice(0, None, 2), slice(3, None, 5)),
                    gp=h.global_power(), gpc=h.global_power(inside_coi=True), sa=h.scale_avg(4.0, 40.0))
    ref = products(api.xwt_resident(y[0], y[1], 1.0, normalize=False, precision=PREC[prec], engine=eng, **kw))
    for a, b in exps:
        got = products(api.xwt_resident(np.ldexp(y[0], a), np.ldexp(y[1], b), 1.0, normalize=False,
                                        precision=PREC[prec], engine=eng, **kw))
        assert_scaled(got["W12"], ref["W12"], a + b, "xwt_resident W12")
        wg, wr = (got["win"], ref["win"]) if not isinstance(got["win"], tuple) else (got["win"][0], ref["win"][0])
        assert_scaled(wg, wr, a + b, "xwt_resident window")
        for name in ("gp", "gpc"):
            assert_close_scaled(got[name], ref[name], a + b, "xwt_resident " + name)
        sg, sr = got["sa"], ref["sa"]
        if isinstance(sg, tuple):
            assert_close_scaled(sg[0], sr[0], a + b, "xwt_resident scale_avg")
            assert_close_scaled(sg[1], sr[1], 0, "xwt_resident scale_avg phase")
        else:
            assert_close_scaled(sg, sr, a + b, "xwt_resident scale_avg")


@pytest.mark.parametrize("prec", [F64, F32])
def test_resident_cross(api, emu, prec):
    check_resident_cross(api, emu, series(1000, 2, 5), KW, prec, pair_exps(XWT, prec))


def _stats_pair(h):
    sig = np.full(len(h.scales), 0.6)
    return dict(WCT=h.coherence(), aWCT=h.phase(), win=h.window(slice(1, None, 3), slice(2, None, 9)),
                gc=h.global_coherence(), gci=h.global_coherence(inside_coi=True, sig95=sig),
                frac=h.significant_fraction(sig), mp=tuple(h.mean_phase(4.0, 40.0, per_scale=True)),
                sa=h.scale_avg(4.0, 40.0))


def _stats_triple(h):
    sig = np.full(len(h.scales), 0.6)
    return dict(RP2=h.partial(), RM2=h.multiple(), PP=h.phase(), win=h.window(slice(1, None, 3), slice(2, None, 9)),
                gp=h.global_coherence(), gm=h.global_coherence('multiple', inside_coi=True, sig=sig),
                frac=h.significant_fraction(sig), mp=tuple(h.mean_phase(4.0, 40.0, per_scale=True)),
                sa=h.scale_avg(4.0, 40.0))


EXACT_FIELDS = ("WCT", "aWCT", "RP2", "RM2", "PP")


def _surrogate_products(h, triple, M, seed):
    """Levels, counts, p-values, FDR and clusters of a fixed seed."""
    out = {}
    out["levels"] = h.surrogate_significance(mc_count=M, seed=seed)
    out["test"] = h.surrogate_test(mc_count=M, seed=seed)
    if triple:
        out["pv"] = (h.pvalues(), h.pvalues(measure='multiple'))
        out["fdr"] = tuple(h.fdr_threshold(q=0.2)) + tuple(h.fdr_threshold(q=0.2, measure='multiple'))
        sig = out["levels"][0]
    else:
        out["pv"] = h.pvalues()
        out["fdr"] = tuple(h.fdr_threshold(q=0.2))
        sig = out["levels"]
    out["frac"] = h.pvalue_fraction(0.25)
    res = h.cluster_test(np.where(np.isfinite(sig), sig, 0.5), mc_count=M, seed=seed + 1)
    out["clusters"] = tuple(res)
    out["labels"] = h.cluster_labels()
    return out


def _flatten(v):
    if isinstance(v, (tuple, list)):
        return [x for e in v for x in _flatten(e)]
    return [np.asarray(v)]


def check_resident_coherence(api, eng, y, kw, prec, exps, M=4, seed=21):
    """wct_resident / wct3_resident with normalize=False: fields exact, reductions within ATOMIC_TOL
    of the unscaled ones, surrogate levels, counts, p-values, FDR and clusters identical."""
    triple = len(y) == 3
    make = (lambda v: api.wct3_resident(*v, 1.0, normalize=False, precision=PREC[prec], engine=eng, **kw)) \
        if triple else \
        (lambda v: api.wct_resident(*v, 1.0, normalize=False, precision=PREC[prec], engine=eng, **kw))
    stats = _stats_triple if triple else _stats_pair
    h = make(y)
    ref, sref = stats(h), _surrogate_products(h, triple, M, seed)
    assert sref["clusters"][0].size > 0 and sref["labels"].max() > 0
    for e in exps:
        h = make([np.ldexp(v, k) for v, k in zip(y, e)])
        got, sgot = stats(h), _surrogate_products(h, triple, M, seed)
        for name, r in ref.items():
            tag = "%s %s %s" % (name, PREC[prec], e)
            for g1, r1 in zip(_flatten(got[name]), _flatten(r)):
                if name in EXACT_FIELDS or name == "win":
                    assert_same(g1, r1, tag)
                elif r1.dtype.kind == 'f' and np.isfinite(r1).any():
                    assert_close_scaled(g1, r1, 0, tag)
                else:
                    assert_same(g1, r1, tag)
        for name, r in sref.items():
            for g1, r1 in zip(_flatten(sgot[name]), _flatten(r)):
                assert_same(g1, r1, "%s %s %s" % (name, PREC[prec], e))


@pytest.mark.parametrize("prec", [F64, F32])
def test_resident_pair(api, emu, prec):
    check_resident_coherence(api, emu, series(512, 2, 7), KW, prec, coh_exps(2))


@pytest.mark.parametrize("prec", [F64, F32])
def test_resident_triple(api, emu, prec):
    check_resident_coherence(api, emu, series(512, 3, 8), KW, prec, coh_exps(3))
