"""Tests of the resident coherence and the partial and multiple coherence against AR(1) red-noise
surrogates of the data's length (`null='ar1'` of `wct_resident` / `wct3_resident`, of
`wct_surrogate_significance` / `wct3_surrogate_significance`, and the engine calls
`mc_ar1_series_surrogates`, `wct_mc_phase`, `surrogate_counts` and `cluster_test` with a
`CoherenceNull`), checked on the host-emulation build of the kernels (tests/_emu):

  * the units: series 0 and 1 are the cross test's AR(1) pair bit for bit, series 2 a host
    restatement under the series tag 2, equal parameters give three different series, and splitting
    the units over calls changes nothing;
  * the counts are the definition k = #{i : R2_i >= R2_obs or R2_i not finite}, bit for bit, against
    a recount of the hook's units (x1 and x2 held at the data for the conditional triple) through
    engine-level `wct` / `wct3` one unit at a time, on every row, fp64 and fp32, Morlet, Paul and DOG,
    the K > 32 boxcar, padded, 2^k and un-padded lengths, with accumulation and reset;
  * the histograms, levels, readers and clusters of the same recount;
  * inputs scaled by powers of two leave the counts and the clusters bit-identical;
  * nothing else moves: the resident fields stay byte-identical, the phase calls give what they gave,
    and counts of one null take no units of another;
  * errors and lifetime.
"""
import copy

import numpy as np
import pytest

import test_emu_cluster_test as C
import test_emu_cross_test as X
import test_emu_surrogate_pvalues as P
import test_emu_surrogate_significance as T
from test_emu_surrogate_significance import emu, api, red  # noqa: F401  (fixtures)

F64, F32 = T.F64, T.F32
NBINS = T.NBINS
MORLET = T.MORLET
AR1, PHASE = 0, 1
ERR_ARG, ERR_STATE = -1, -4


def cnull(nser, conditional=True):
    """An AR(1) null of the engine with distinct parameters per series."""
    from pycwt_b200._engine import CoherenceNull
    held = (0, 1, 1) if nser == 3 and conditional else (0,) * nser
    return CoherenceNull(AR1, None, (0.6, -0.3, 0.45)[:nser], (0.0, 0.5, -1.0)[:nser], (1.0, 2.0, 0.5)[:nser], held)


def units(eng, x, null, seed, first, count):
    """The units [count, nser, n0] of `null` for the data x [nser, n0]: the drawn series from the hook
    (they are a prefix 0 .. d - 1, so the hook's tags are theirs), the held ones the data's rows."""
    nser, n0 = x.shape
    d = sum(1 for h in null.held if not h)
    U = np.repeat(x[None].astype(np.float64), count, axis=0)
    U[:, :d] = eng.mc_ar1_series_surrogates(null.g[:d], null.m[:d], null.sigma[:d], seed, first, count, n0)
    return U


# ---- the units -----------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4, 1001, 9000])
def test_units(emu, n):
    g, m, sigma = (0.7, -0.4, 0.55), (0.0, 3.0, -1.0), (1.0, 2.5, 0.75)
    U = emu.mc_ar1_series_surrogates(g, m, sigma, 1234, 0, 4, n)
    assert U.shape == (4, 3, n)
    assert np.array_equal(U[:, :2], emu.mc_ar1_pair_surrogates(g[:2], m[:2], sigma[:2], 1234, 0, 4, n))
    assert np.array_equal(emu.mc_ar1_series_surrogates(g[:1], m[:1], sigma[:1], 1234, 0, 4, n)[:, 0],
                          emu.mc_ar1_surrogates(g[0], m[0], sigma[0], 1234, 0, 4, n))
    for u in (0, 3):
        ref = X.ar1_host(g[2], m[2], sigma[2], 1234, u, n, 2)
        tol = 16 * np.finfo(float).eps * sigma[2] / (1 - abs(g[2])) * \
            max(1.0, float(np.abs(ref - m[2]).max()) / sigma[2])
        assert float(np.abs(U[u, 2].astype(np.longdouble) - ref).max()) <= tol
    same = emu.mc_ar1_series_surrogates((0.5,) * 3, (0.0,) * 3, (1.0,) * 3, 7, 0, 2, n)
    for a, b in ((0, 1), (0, 2), (1, 2)):
        assert not np.array_equal(same[:, a], same[:, b])
        if n >= 1000:
            assert abs(np.corrcoef(same[0, a], same[0, b])[0, 1]) < 0.2
    a = emu.mc_ar1_series_surrogates(g, m, sigma, 1234, 0, 1, n)
    b = emu.mc_ar1_series_surrogates(g, m, sigma, 1234, 1, 3, n)
    assert np.array_equal(U, np.concatenate([a, b]))


# ---- counts are the definition (engine level) ----------------------------------------------------
def recount(eng, U, sj, K, prec, obs, dt=1.0, f0=6.0):
    """k per measure of the units U [M, nser, n0] through engine-level wct / wct3, unit by unit."""
    k = [np.zeros(o.shape, dtype=np.int64) for o in obs]
    for u in U:
        if len(u) == 2:
            R = [eng.wct(u[0], u[1], dt, 0.25, sj, MORLET, f0, K, want_angle=False, precision=prec)[0]]
        else:
            R = list(eng.wct3(*u, dt, 0.25, sj, MORLET, f0, K, precision=prec))
        for kk, r, o in zip(k, R, obs):
            kk += (~np.isfinite(r)) | (r >= o)
    return k


def check_counts(eng, nser, conditional, n0, K, prec, M=4, seed=31):
    x, sj, mask, serial = P.setup(eng, nser, n0, K, prec)
    S = sj.size
    maxscale = S - 3
    null = cnull(nser, conditional)
    before = P.observed(eng, nser)
    obs = before[:nser - 1]
    hs = P.count(eng, x, null, seed, 0, M, sj, mask, maxscale, K, prec, serial)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before, P.observed(eng, nser)))
    hh = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    eng.wct_mc_phase(x, null, seed, 0, M, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hh, precision=prec)
    assert all(np.array_equal(a, b) for a, b in zip(hs, hh))
    U = units(eng, x, null, seed, 0, M)
    if nser == 3 and conditional:
        assert all(np.array_equal(u[1:], x[1:]) for u in U)
    k = recount(eng, U, sj, K, prec, obs)
    ps = P.counted_p(eng, nser)
    for p, kk, o in zip(ps, k, obs):
        assert np.array_equal(p, P.p_of(kk, M, o), equal_nan=True)
        assert 0 < kk.sum() < M * kk.size
    # accumulation: [0, 2) then [2, M) is [0, M); reset starts over
    P.count(eng, x, null, seed, 0, 2, sj, mask, maxscale, K, prec, serial)
    P.count(eng, x, null, seed, 2, M - 2, sj, mask, maxscale, K, prec, serial, reset=False)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(P.counted_p(eng, nser), ps))
    P.count(eng, x, null, seed, 3, 1, sj, mask, maxscale, K, prec, serial)
    k1 = recount(eng, units(eng, x, null, seed, 3, 1), sj, K, prec, obs)
    assert all(np.array_equal(p, P.p_of(kk, 1, o), equal_nan=True) for p, kk, o in zip(P.counted_p(eng, nser), k1, obs))


NULLS = [(2, True), (3, True), (3, False)]


@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser,conditional", NULLS)
@pytest.mark.parametrize("n0,K", [(512, 6), (600, 36)])
def test_counts_are_the_definition(emu, nser, conditional, n0, K, prec):
    """2^k, and a padded length (600 runs at 1024) with a boxcar longer than 32."""
    check_counts(emu, nser, conditional, n0, K, prec)


@pytest.mark.parametrize("nser,conditional", NULLS)
def test_counts_unpadded(emu, nser, conditional):
    emu.set_padding(False)
    try:
        check_counts(emu, nser, conditional, 600, 6, F64, M=3)
    finally:
        emu.set_padding(True)


# ---- the public calls: levels, readers, clusters ---------------------------------------------------
@pytest.fixture
def generic(emu):
    """The generic smoothing of Paul / DOG on; the padding back on afterwards, in the package and in
    the engine the handles synchronise."""
    from pycwt_b200 import helpers, mothers
    old = mothers.enable_generic_smoothing(True)
    yield
    mothers.enable_generic_smoothing(old)
    helpers.set_fft_padding(True)
    emu.set_padding(True)


WAVELETS = {'morlet': lambda api: api.Morlet(6), 'paul': lambda api: api.Paul(4), 'dog': lambda api: api.DOG(2)}
KW = dict(dj=1 / 2, s0=2.0)


def handle(api, nser, wav, prec, n0, padded=True, normalize=True, scale=None):
    from pycwt_b200 import helpers
    helpers.set_fft_padding(padded)
    x = (P.pair if nser == 2 else P.triple)(n0, 5 + nser)
    if scale is not None:
        x = np.ldexp(x, np.array(scale)[:, None])
    fn = api.wct_resident if nser == 2 else api.wct3_resident
    return fn(*x, 1.0, wavelet=WAVELETS[wav](api), precision=prec, normalize=normalize, **KW)


def obs_fields(h):
    f = P.fields(h)
    return f[:1] if len(f) == 2 else [f[0], f[2]]


def handle_fields(h, U):
    """The measures of each unit through engine-level wct / wct3 under the handle's plan (smoothing
    filter, length policy and precision of `_wct_on_device`), [measure][unit]."""
    from pycwt_b200.wavelet import _wct_on_device, _wct_problem
    eng = h.engine
    p = _wct_problem(h._y, h.dt, h.dj, h.s0, h.J, h.wavelet, h.normalize, h.precision)
    out = []
    for u in U:
        q = copy.copy(p)
        q.yns = tuple(u)
        if len(u) == 2:
            out.append([_wct_on_device(eng, q, lambda *a, boxcar_len, precision: eng.wct(
                *a[:7], boxcar_len, want_angle=False, precision=precision)[0])])
        else:
            out.append(list(_wct_on_device(eng, q, lambda *a, boxcar_len, precision: eng.wct3(
                *a[:8], boxcar_len, precision=precision))))
    return [np.array(r) for r in zip(*out)]


def handle_units(h, seed, M, conditional=True):
    from pycwt_b200.wavelet import _coherence_null, _surrogate_problem
    p, _ = _surrogate_problem(h._y, h.dt, h.dj, h.s0, h.J, h.wavelet, h.normalize, h.precision)
    null = _coherence_null('ar1', p, h.normalize, conditional)
    return units(h.engine, np.stack(p.yns), null, seed, 0, M)


def kcount(R, o):
    return ((R >= o[None]) | ~np.isfinite(R)).sum(axis=0)


CASES = [   # (nser, conditional, precision, wavelet, n0, padded)
    (2, True, 'fp64', 'morlet', 256, True),
    (2, True, 'fp32', 'paul', 300, True),
    (2, True, 'fp64', 'dog', 301, False),
    (3, True, 'fp64', 'paul', 256, True),
    (3, True, 'fp32', 'morlet', 300, True),
    (3, False, 'fp64', 'dog', 300, True),
    (3, True, 'fp64', 'morlet', 301, False),
]


@pytest.mark.parametrize("nser,conditional,prec,wav,n0,padded", CASES)
def test_public(api, emu, generic, nser, conditional, prec, wav, n0, padded):
    h = handle(api, nser, wav, prec, n0, padded, normalize=(wav != 'dog'))
    before = [f.tobytes() for f in P.fields(h)]
    M, seed = 5, 17
    kw = {} if nser == 2 else dict(conditional=conditional)
    levels = h.surrogate_test(mc_count=M, seed=seed, null='ar1', **kw)
    assert h.surrogate_null == 'ar1' and h.surrogate_units == M and h.surrogate_seed == seed
    ref = h.surrogate_significance(mc_count=M, seed=seed, null='ar1', **kw)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(np.atleast_2d(levels), np.atleast_2d(ref)))
    assert [f.tobytes() for f in P.fields(h)] == before
    obs = obs_fields(h)
    R = handle_fields(h, handle_units(h, seed, M, conditional))
    ps = [P.p_of(kcount(r, o), M, o) for r, o in zip(R, obs)]
    measures = [{}] if nser == 2 else [dict(measure='partial'), dict(measure='multiple')]
    lo, hi = h.coi_ranges()
    cols = np.arange(h.n0)[None]
    cone = (cols >= lo[:, None]) & (cols < hi[:, None])
    for p, o, mk in zip(ps, obs, measures):
        assert np.array_equal(h.pvalues(**mk), p, equal_nan=True)
        fin = np.isfinite(p)
        for alpha in (0.35, 0.7):
            sel = cone & fin & (p <= alpha)
            tested = (cone & fin).sum(axis=1)
            frac = h.pvalue_fraction(alpha, **mk)
            assert np.array_equal(frac[tested > 0], sel.sum(axis=1)[tested > 0] / tested[tested > 0])
            gc = h.global_coherence(inside_coi=True, alpha=alpha, **mk)
            n = sel.sum(axis=1)
            ok = n > 0
            assert np.allclose(gc[ok], np.where(sel, o, 0).sum(axis=1)[ok] / n[ok], rtol=1e-13, atol=0)
            assert np.isnan(gc[~ok]).all()
        for method in ('bh', 'by'):
            for q in (0.05, 0.5):
                P.check_fdr(h.fdr_threshold(q, method, True, **mk), p[fin & cone], q, method)
    # the cluster test: null_max, table and labels of the recount, thresholded on the host and
    # labelled by scipy.ndimage.label
    m = 0 if nser == 2 else 1
    sig = np.nanquantile(obs[m], 0.6, axis=1)
    res = h.cluster_test(sig, mc_count=M, seed=seed, null='ar1', **kw, **measures[m])
    q = C.weights(h.scales)
    unit = h.dj * h.dt / np.min(h.scales) / 2.0 ** 32
    ref = np.array([C.reference(C.select(r, sig, lo, hi), q)[0][:1].sum() for r in R[m]], dtype=np.uint64)
    assert np.array_equal(res.null_max, ref.astype(float) * unit)
    rQ, rpts, rbox, rlab = C.reference(C.select(obs[m], sig, lo, hi), q)
    assert np.array_equal(res.area, rQ.astype(float) * unit) and np.array_equal(res.points, rpts)
    assert np.array_equal(res.rows, rbox[:, :2]) and np.array_equal(res.cols, rbox[:, 2:])
    assert np.array_equal(res.pvalue, np.array([(1 + np.sum(ref >= Qc)) / (1 + M) for Qc in rQ]))
    assert np.array_equal(h.cluster_labels(), rlab)
    assert [f.tobytes() for f in P.fields(h)] == before


# ---- engine-level clusters, K > 32 -----------------------------------------------------------------
@pytest.mark.parametrize("nser,conditional,measure", [(2, True, None), (3, True, 0), (3, False, 1)])
@pytest.mark.parametrize("prec", [F64, F32])
def test_cluster_units(emu, nser, conditional, measure, prec, n0=600, K=36, M=4, seed=23):
    x, sj, mask, serial = P.setup(emu, nser, n0, K, prec)
    S = sj.size
    null = cnull(nser, conditional)
    before = P.observed(emu, nser)
    obs = before[0] if nser == 2 else before[measure]
    thr, lo, hi = C.row_args(S, n0, obs)
    q = C.weights(sj)
    hs = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    qmax = emu.cluster_test(x, null, seed, 0, M, 1.0, sj, MORLET, 6.0, K, mask, S - 3, NBINS, *hs,
                            serial=serial, thr=thr, lo=lo, hi=hi, q=q, measure=measure, precision=prec)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before, P.observed(emu, nser)))
    ref = []
    for u in units(emu, x, null, seed, 0, M):
        if nser == 2:
            r = emu.wct(u[0], u[1], 1.0, 0.25, sj, MORLET, 6.0, K, want_angle=False, precision=prec)[0]
        else:
            r = emu.wct3(*u, 1.0, 0.25, sj, MORLET, 6.0, K, precision=prec)[measure]
        ref.append(C.reference(C.select(r, thr, lo, hi), q)[0][:1].sum())
    assert np.array_equal(qmax, np.array(ref, dtype=np.uint64)) and (qmax > 0).any()
    rQ, rpts, rbox, rlab = C.reference(C.select(obs, thr, lo, hi), q)
    Q, pts, box = emu.cluster_table(measure is not None)
    assert np.array_equal(Q, rQ) and np.array_equal(pts, rpts) and np.array_equal(box, rbox)
    assert np.array_equal(emu.cluster_labels(measure is not None, 0, S, 1, 0, n0, 1), rlab)


# ---- powers of two ---------------------------------------------------------------------------------
@pytest.mark.parametrize("nser", [2, 3])
def test_powers_of_two(api, emu, generic, nser):
    """normalize=False: the units take the data's mean and scale; scaling the inputs by powers of two
    scales every unit by the same powers, and the counts and clusters stay bit-identical."""
    runs = []
    for scale in ([0, 0, 0], [7, -5, 3], [-60, 40, 20]):
        h = handle(api, nser, 'morlet', 'fp64', 256, normalize=False, scale=scale[:nser])
        lv = h.surrogate_test(mc_count=4, seed=3, null='ar1')
        sig = np.nanquantile(obs_fields(h)[0], 0.6, axis=1)
        res = h.cluster_test(sig, mc_count=4, seed=4, null='ar1')
        runs.append((h.pvalues(), np.atleast_2d(lv), res.null_max, res.area, h.cluster_labels()))
    for r in runs[1:]:
        assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(runs[0], r))


# ---- nothing else moves ----------------------------------------------------------------------------
def test_nothing_else_moves(api, emu):
    x3 = P.triple(256, 2)
    hp = api.power_resident(x3[0], 1.0, **KW)
    hx = api.xwt_resident(x3[0], x3[1], 1.0, **KW)
    h = api.wct_resident(x3[0], x3[1], 1.0, **KW)
    h3 = api.wct3_resident(*x3, 1.0, **KW)
    keep = [hp.wave().tobytes(), hx.cross_spectrum().tobytes()]
    h.surrogate_test(mc_count=3, seed=2)
    h3.surrogate_test(mc_count=3, seed=2)
    phase = [h.pvalues(), h3.pvalues(), h3.pvalues(measure='multiple')]
    h.surrogate_test(mc_count=3, seed=2, null='ar1')
    h3.surrogate_test(mc_count=3, seed=2, null='ar1')
    h3.cluster_test(np.full(len(h3.scales), 0.5), mc_count=2, seed=1, null='ar1')
    assert h.surrogate_null == 'ar1' and h3.surrogate_null == 'ar1'
    assert [hp.wave().tobytes(), hx.cross_spectrum().tobytes()] == keep
    h.surrogate_test(mc_count=3, seed=2)
    h3.surrogate_test(mc_count=3, seed=2)
    assert h.surrogate_null == 'phase'
    again = [h.pvalues(), h3.pvalues(), h3.pvalues(measure='multiple')]
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(phase, again))
    # the phase calls of the C ABI are the null calls with CWTB_NULL_PHASE
    eng = h.engine
    x, sj, mask, serial = P.setup(eng, 3, 256, 6, F64)
    a = P.count(eng, x, (0, 1, 1), 9, 0, 3, sj, mask, 17, 6, F64, serial)
    pa = P.counted_p(eng, 3)
    from pycwt_b200._engine import CoherenceNull
    b = P.count(eng, x, CoherenceNull(PHASE, (0, 1, 1)), 9, 0, 3, sj, mask, 17, 6, F64, serial)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
    assert all(np.array_equal(u, v, equal_nan=True) for u, v in zip(pa, P.counted_p(eng, 3)))


def test_no_units_of_another_null(emu):
    """Counts of one null take no units of another: ERR_STATE, and the counts stay readable."""
    from pycwt_b200._engine import EngineError
    for nser in (2, 3):
        x, sj, mask, serial = P.setup(emu, nser, 256, 6, F64)
        groups = (0, 1) if nser == 2 else (0, 1, 1)
        P.count(emu, x, groups, 1, 0, 2, sj, mask, 17, 6, F64, serial)
        p0 = P.counted_p(emu, nser)
        with pytest.raises(EngineError, match="another null"):
            P.count(emu, x, cnull(nser), 1, 2, 1, sj, mask, 17, 6, F64, serial, reset=False)
        assert all(np.array_equal(u, v, equal_nan=True) for u, v in zip(p0, P.counted_p(emu, nser)))
        P.count(emu, x, cnull(nser), 1, 0, 2, sj, mask, 17, 6, F64, serial)
        with pytest.raises(EngineError, match="another null"):
            P.count(emu, x, groups, 1, 2, 1, sj, mask, 17, 6, F64, serial, reset=False)
        P.count(emu, x, cnull(nser), 1, 2, 1, sj, mask, 17, 6, F64, serial, reset=False)


# ---- errors and lifetime ---------------------------------------------------------------------------
def test_errors(api, emu):
    from pycwt_b200._engine import CoherenceNull, EngineError
    x, sj, mask, serial = P.setup(emu, 3, 256, 6, F64)
    good = cnull(3)
    cases = [
        (good._replace(g=(0.5, 1.0, 0.3), held=(0, 0, 0)), "AR\\(1\\)"),
        (good._replace(g=(np.nan, 0.0, 0.0)), "AR\\(1\\)"),
        (good._replace(sigma=(np.inf, 1.0, 1.0)), "AR\\(1\\)"),
        (good._replace(held=(1, 0, 0)), "held"),
        (good._replace(held=(0, 2, 1)), "held"),
        (CoherenceNull(7, (0, 1, 1)), "unknown null"),
    ]
    for null, msg in cases:
        with pytest.raises(EngineError, match=msg):
            P.count(emu, x, null, 1, 0, 1, sj, mask, 17, 6, F64, serial)
    # a held g is not read: |g| >= 1 on a held driver is fine
    P.count(emu, x, good._replace(g=(0.5, 2.0, np.nan)), 1, 0, 1, sj, mask, 17, 6, F64, serial)
    with pytest.raises(EngineError, match="serial"):
        P.count(emu, x, good, 1, 0, 1, sj, mask, 17, 6, F64, serial + 1)
    x2, sj2, mask2, serial2 = P.setup(emu, 2, 256, 6, F64)
    with pytest.raises(EngineError, match="held"):
        P.count(emu, x2, cnull(2)._replace(held=(0, 1)), 1, 0, 1, sj2, mask2, 17, 6, F64, serial2)
    with pytest.raises(ValueError, match="one entry per series"):
        P.count(emu, x2, cnull(3), 1, 0, 1, sj2, mask2, 17, 6, F64, serial2)
    with pytest.raises(EngineError, match="nser"):
        emu.mc_ar1_series_surrogates((0.1,) * 4, (0,) * 4, (1,) * 4, 1, 0, 1, 8)
    # C level: the table wavelets are unsupported
    hs = np.zeros((sj.size, NBINS), dtype=np.int64)
    with pytest.raises(EngineError, match="analytic"):
        emu.wct_mc_phase(x2, cnull(2), 1, 0, 1, 1.0, sj2, 3, 6.0, 6, mask2, 17, NBINS, hs)
    # Python level
    h = api.wct_resident(*P.pair(256), 1.0, **KW)
    with pytest.raises(ValueError, match="null"):
        h.surrogate_test(mc_count=2, null='white')
    with pytest.raises(ValueError, match="null"):
        h.cluster_test(np.ones(len(h.scales)), mc_count=2, null=None)
    with pytest.raises(ValueError, match="null"):
        api.wct_surrogate_significance(*P.pair(256), 1.0, mc_count=2, null='red', **KW)
    trend = np.arange(256.0) ** 3
    with pytest.raises((ValueError, Warning)):
        api.wct3_surrogate_significance(trend, *P.pair(256), 1.0, mc_count=2, null='ar1', **KW)
    # lifetime: the counts die with the product, a new product counts afresh
    h.surrogate_test(mc_count=2, seed=1, null='ar1')
    h.release()
    with pytest.raises(EngineError, match="no longer resident"):
        h.pvalues()
    h2 = api.wct_resident(*P.pair(256), 1.0, **KW)
    with pytest.raises(EngineError, match="surrogate test"):
        h2.pvalues()
    h2.surrogate_test(mc_count=2, seed=1, null='ar1')
    assert np.isfinite(h2.pvalues()).any()
