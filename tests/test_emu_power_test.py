"""Tests of the resident wavelet power against AR(1) and phase-randomised surrogates
(`power_resident`, `ResidentPower` and the engine calls `power_resident`, `mc_ar1_surrogates`,
`power_surrogate_counts`, `power_cluster_test`), checked on the host-emulation build of the kernels
(tests/_emu):

  * the AR(1) units equal a host restatement (Philox4x32-10 in NumPy, the recursion in longdouble)
    to a few ulp of sigma / (1 - |g|), and do not depend on how the units are split over calls;
  * the counts are the definition k = #{i : P_i >= P_obs or P_i not finite}, bit for bit, against a
    recount of the hooks' surrogates through engine-level `cwt` one unit at a time, for both nulls,
    fp64 and fp32, Morlet, Paul and DOG, padded, 2^k and un-padded lengths, with accumulation and
    reset;
  * the p-values, the FDR threshold (scipy.stats.false_discovery_control) and the clusters (the
    scipy.ndimage reference of test_emu_cluster_test) of the same recount;
  * nothing else moves: the power's W and the coherence, cross and triple slots stay byte-identical,
    and the other calls leave the power valid;
  * lifetime and errors.
"""
import numpy as np
import pytest

import test_emu_cluster_test as C
import test_emu_surrogate_pvalues as P
import test_emu_surrogate_significance as T
from test_emu_surrogate_significance import emu, api, red  # noqa: F401  (fixtures)

F64, F32 = T.F64, T.F32
POWER = 'power'   # pycwt_b200._engine.POWER
KW = dict(dj=0.5, s0=2.0)


# ---- host restatement of the AR(1) units -----------------------------------------------------------
def ar1_host(g, m, sigma, seed, unit, n):
    """Unit `unit` of the AR(1) null in longdouble: the normals of the Philox4x32-10 blocks with
    counter words (j, 2^31, unit lo, 2^31 | (unit hi << 2) | 3), Box-Muller as NoiseBody converts."""
    j = np.arange((n + 1) // 2, dtype=np.uint64)
    o = T.philox4x32_10(j, 0x80000000, unit & 0xFFFFFFFF, 0x80000000 | ((unit >> 32) << 2) | 3, seed)
    u1 = ((o[0] >> np.uint64(5)).astype(float) * 67108864.0 + (o[1] >> np.uint64(6)).astype(float) + 0.5) \
        / 9007199254740992.0
    u2 = ((o[2] >> np.uint64(5)).astype(float) * 67108864.0 + (o[3] >> np.uint64(6)).astype(float) + 0.5) \
        / 9007199254740992.0
    r = np.sqrt(-2.0 * np.log(u1))
    e = np.empty(2 * j.size)
    e[0::2] = r * np.cos(2 * np.pi * u2)
    e[1::2] = r * np.sin(2 * np.pi * u2)
    e = e[:n].astype(np.longdouble)
    gl = np.longdouble(g)
    s = np.sqrt(1 - gl * gl)
    z = np.empty(n, dtype=np.longdouble)
    z[0] = e[0]
    acc = z[0]
    for i in range(1, n):
        acc = gl * acc + s * e[i]
        z[i] = acc
    return np.longdouble(m) + np.longdouble(sigma) * z


@pytest.mark.parametrize("g", [-0.9, 0.0, 0.5, 0.95])
@pytest.mark.parametrize("n", [4, 1001, 65537, 2 ** 17])
def test_ar1_units_match_host(emu, g, n):
    units = (0, 5) if n <= 65537 else (3,)
    m, sigma = (0.0, 1.0) if g != 0.5 else (3.0, 2.5)
    for u in units:
        x = emu.mc_ar1_surrogates(g, m, sigma, 1234, u, 1, n)[0]
        ref = ar1_host(g, m, sigma, 1234, u, n)
        tol = 16 * np.finfo(float).eps * sigma / (1 - abs(g)) * max(1.0, float(np.abs(ref - m).max()) / sigma)
        err = float(np.abs(x.astype(np.longdouble) - ref).max())
        assert err <= tol, (g, n, u, err, tol)


def test_ar1_units_split_and_seed(emu):
    whole = emu.mc_ar1_surrogates(0.7, 0.0, 1.0, 99, 0, 7, 9000)
    a = emu.mc_ar1_surrogates(0.7, 0.0, 1.0, 99, 0, 3, 9000)
    b = emu.mc_ar1_surrogates(0.7, 0.0, 1.0, 99, 3, 4, 9000)
    assert np.array_equal(whole, np.concatenate([a, b]))
    assert not np.array_equal(whole, emu.mc_ar1_surrogates(0.7, 0.0, 1.0, 100, 0, 7, 9000))
    # units far apart in the unit number (the high word of the counter)
    far = emu.mc_ar1_surrogates(0.7, 0.0, 1.0, 99, 2 ** 40, 1, 64)
    assert np.abs(far[0] - ar1_host(0.7, 0.0, 1.0, 99, 2 ** 40, 64).astype(float)).max() < 1e-13


@pytest.mark.parametrize("g", [1.0, -1.0, 1.5, np.nan, np.inf])
def test_ar1_bad_coefficient(emu, g):
    from pycwt_b200._engine import EngineError
    with pytest.raises(EngineError, match="AR\\(1\\)"):
        emu.mc_ar1_surrogates(g, 0.0, 1.0, 1, 0, 1, 16)


def test_ar1_bad_mean_and_sigma(emu):
    from pycwt_b200._engine import EngineError
    for m, s in ((np.nan, 1.0), (0.0, np.inf)):
        with pytest.raises(EngineError, match="AR\\(1\\)"):
            emu.mc_ar1_surrogates(0.5, m, s, 1, 0, 1, 16)


# ---- the recount -------------------------------------------------------------------------------
def series(n, seed=3):
    return red(np.random.RandomState(seed), n, 0.6)[0] * 3.0 + 1.5


def surrogates(h, null, seed, first, count):
    """The units the handle's tests draw, from the hooks.  A phase-randomised unit is a pure function
    of (seed, unit, phase group, bin): the power's series in group 0 is the first of a pair."""
    eng = h.engine
    kind, g, m, sigma = h._null(null)
    if null == 'ar1':
        return eng.mc_ar1_surrogates(g, m, sigma, seed, first, count, h.n0)
    return eng.mc_phase_surrogates(np.stack([h._yn, h._yn]), (0, 1), seed, first, count)[:, 0]


def unit_powers(h, null, seed, first, count):
    """P_i [count, S, n0] of engine-level `cwt` of each unit, in the handle's precision."""
    eng = h.engine
    pow2 = h.n0 & (h.n0 - 1) == 0
    prec = F32 if h.precision == 'fp32' and (h._padding or pow2) else F64
    out = []
    for x in surrogates(h, null, seed, first, count):
        W = eng.cwt(x, h.dt, h.scales, *h.wavelet._engine_spec(), precision=prec)
        out.append(W.real * W.real + W.imag * W.imag)
    return np.array(out)


def recount(Pobs, Pi):
    return ((Pi >= Pobs[None]) | ~np.isfinite(Pi)).sum(axis=0)


def p_of(k, M, Pobs):
    return np.where(np.isfinite(Pobs), (1.0 + k) / (1.0 + M), np.nan)


CASES = [   # (null, precision, wavelet, n0, padded)
    ('ar1', 'fp64', 'morlet', 300, True),
    ('phase', 'fp64', 'morlet', 256, True),
    ('ar1', 'fp32', 'paul', 256, True),
    ('phase', 'fp32', 'dog', 300, True),
    ('ar1', 'fp64', 'dog', 301, False),
    ('phase', 'fp64', 'paul', 301, False),
    ('phase', 'fp32', 'morlet', 1000, True),
]
WAVELETS = {'morlet': lambda api: api.Morlet(6), 'paul': lambda api: api.Paul(4), 'dog': lambda api: api.DOG(2)}


def resident(api, null, prec, wav, n0, padded, normalize=True):
    from pycwt_b200 import helpers
    helpers.set_fft_padding(padded)
    return api.power_resident(series(n0), 1.0, wavelet=WAVELETS[wav](api), precision=prec,
                              normalize=normalize, **KW)


@pytest.fixture
def padding():
    from pycwt_b200 import helpers
    yield
    helpers.set_fft_padding(True)


@pytest.mark.parametrize("null,prec,wav,n0,padded", CASES)
def test_counts_are_the_definition(api, emu, padding, null, prec, wav, n0, padded):
    h = resident(api, null, prec, wav, n0, padded, normalize=(null == 'phase'))
    Pobs = h.power()
    W0 = h.wave().tobytes()
    M = 5
    h.surrogate_test(mc_count=M, seed=21, null=null)
    assert h.surrogate_units == M and h.surrogate_seed == 21
    Pi = unit_powers(h, null, 21, 0, M)
    assert np.array_equal(h.pvalues(), p_of(recount(Pobs, Pi), M, Pobs), equal_nan=True)
    assert h.wave().tobytes() == W0
    # accumulation over calls: [0, 2) then [2, M) equals [0, M); reset starts over
    eng = h.engine
    kind, g, m, sigma = h._null(null)
    args = (h._yn, kind, g, m, sigma, 21)
    geo = (h.dt, h.scales, *h.wavelet._engine_spec(), h._serial)
    S, n = h.shape
    eng.power_surrogate_counts(*args, 0, 2, *geo, reset=True)
    assert np.array_equal(eng.pvalue_window(POWER, 0, S, 1, 0, n, 1),
                          p_of(recount(Pobs, Pi[:2]), 2, Pobs), equal_nan=True)
    eng.power_surrogate_counts(*args, 2, M - 2, *geo, reset=False)
    assert np.array_equal(eng.pvalue_window(POWER, 0, S, 1, 0, n, 1),
                          p_of(recount(Pobs, Pi), M, Pobs), equal_nan=True)
    eng.power_surrogate_counts(*args, 2, M - 2, *geo, reset=True)
    assert np.array_equal(eng.pvalue_window(POWER, 0, S, 1, 0, n, 1),
                          p_of(recount(Pobs, Pi[2:]), M - 2, Pobs), equal_nan=True)


def test_readers(api, emu):
    h = api.power_resident(series(600), 1.0, **KW)
    Pobs = h.power()
    W = h.wave()
    # the device's |W|^2 is re^2 + im^2 in double, each product rounded on its own
    assert np.array_equal(Pobs, W.real * W.real + W.imag * W.imag)
    assert np.array_equal(h.power(slice(2, None, 5), slice(7, 590, 9)), Pobs[2::5, 7:590:9])
    assert h.power(slice(3, 3), slice(None)).shape == (0, 600)
    M = 7
    h.surrogate_test(mc_count=M, seed=5, null='phase')
    k = recount(Pobs, unit_powers(h, 'phase', 5, 0, M))
    p = p_of(k, M, Pobs)
    assert np.array_equal(h.pvalues(slice(1, None, 3), slice(5, 590, 7)), p[1::3, 5:590:7], equal_nan=True)
    assert np.array_equal(h.pvalues(), p, equal_nan=True)
    lo, hi = h.coi_ranges()
    cone = (np.arange(h.n0)[None] >= lo[:, None]) & (np.arange(h.n0)[None] < hi[:, None])
    fin = np.isfinite(p)
    for alpha in (0.25, 0.5):
        sel = cone & fin & (p <= alpha)
        tested = (cone & fin).sum(axis=1)
        frac = h.pvalue_fraction(alpha)
        assert np.array_equal(frac[tested > 0], sel.sum(axis=1)[tested > 0] / tested[tested > 0])
        assert np.isnan(frac[tested == 0]).all()
        num = np.where(sel, Pobs, 0).sum(axis=1)
        gp = h.global_power(inside_coi=True, alpha=alpha)
        cnt = sel.sum(axis=1)
        ok = cnt > 0
        assert np.allclose(gp[ok], num[ok] / cnt[ok], rtol=1e-12) and np.isnan(gp[~ok]).all()
    for method in ('bh', 'by'):
        for inside in (True, False):
            for q in (0.05, 0.3, 0.9):
                P.check_fdr(h.fdr_threshold(q, method, inside), p[fin & (cone if inside else True)], q, method)
    # the products of ResidentTransform
    signif = np.full(len(h.scales), np.median(Pobs))
    above = cone & (Pobs > signif[:, None])
    assert np.allclose(h.significant_fraction(signif), above.sum(axis=1) / (hi - lo), equal_nan=True)
    assert np.allclose(h.global_power(), Pobs.mean(axis=1), rtol=1e-12)
    sa = h.scale_avg_power(2.0, 40.0)
    sel_s, w = h._band_weights(2.0, 40.0)
    assert np.allclose(sa, (w[:, None] * Pobs).sum(axis=0), rtol=1e-12)
    W = h.wave()
    assert np.array_equal(h.window(slice(0, None, 2), slice(3, 50, 4)), W[0::2, 3:50:4])


@pytest.mark.parametrize("null,prec", [('ar1', 'fp64'), ('phase', 'fp32'), ('phase', 'fp64')])
def test_cluster_test_against_recount(api, emu, null, prec):
    h = api.power_resident(series(700, seed=8), 1.0, precision=prec, **KW)
    Pobs = h.power()
    W0 = h.wave().tobytes()
    M = 6
    h.surrogate_test(mc_count=3, seed=1, null=null)
    p0 = h.pvalues()
    sig = np.quantile(Pobs, 0.7, axis=1)
    res = h.cluster_test(sig, mc_count=M, seed=4, null=null)
    q = C.weights(h.scales)
    lo, hi = h.coi_ranges()
    cols = np.arange(h.n0)[None]
    cone = (cols >= lo[:, None]) & (cols < hi[:, None])

    def select(Pm):
        return np.isfinite(Pm) & (Pm > sig[:, None]) & cone

    rQ, rpts, rbox, rlab = C.reference(select(Pobs), q)
    from pycwt_b200.resident import _cluster_weights
    _, unit_area = _cluster_weights(h)
    assert np.array_equal(res.area, rQ.astype(float) * unit_area)
    assert np.array_equal(res.points, rpts)
    assert np.array_equal(np.column_stack([res.rows, res.cols]), rbox)
    assert np.array_equal(h.cluster_labels(), rlab)
    qmax = [C.reference(select(Pi), q)[0] for Pi in unit_powers(h, null, 4, 0, M)]
    qmax = np.array([int(x[0]) if x.size else 0 for x in qmax], dtype=float) * unit_area
    assert np.array_equal(res.null_max, qmax)
    reached = np.array([(qmax >= a).sum() for a in res.area])
    assert np.array_equal(res.pvalue, (1.0 + reached) / (1.0 + M))
    assert h.wave().tobytes() == W0
    assert np.array_equal(h.pvalues(), p0, equal_nan=True)   # the counts are kept


def test_nothing_else_moves(api, emu):
    x = series(512, seed=1)
    y = series(512, seed=2)
    z = series(512, seed=3)
    hc = api.wct_resident(x, y, 1.0, **KW)
    hx = api.xwt_resident(x, y, 1.0, **KW)
    h3 = api.wct3_resident(x, y, z, 1.0, **KW)
    h = api.power_resident(x, 1.0, **KW)
    before = [hc.coherence().tobytes(), hx.cross_spectrum().tobytes(), h3.partial().tobytes(), h.wave().tobytes()]
    h.surrogate_test(mc_count=3, seed=2)
    h.cluster_test(np.full(len(h.scales), 2.0), mc_count=3, seed=3, null='phase')
    after = [hc.coherence().tobytes(), hx.cross_spectrum().tobytes(), h3.partial().tobytes(), h.wave().tobytes()]
    assert before == after
    p = h.pvalues()
    # the other calls leave the power valid and byte-identical
    api.cwt(x, 1.0, **KW)
    api.xwt(x, y, 1.0, **KW)
    api.wct(x, y, 1.0, sig=False, **KW)
    hc.surrogate_test(mc_count=2, seed=1)
    hc.cluster_test(np.full(len(hc.scales), 0.5), mc_count=2, seed=1)
    api.cwt_resident(x, 1.0, **KW)
    assert h.wave().tobytes() == before[3]
    assert np.array_equal(h.pvalues(), p, equal_nan=True)
    assert hc.coherence().tobytes() == before[0]


def test_lifetime_and_errors(api, emu, padding):
    from pycwt_b200 import helpers
    from pycwt_b200._engine import EngineError
    x = series(256)
    h = api.power_resident(x, 1.0, **KW)
    with pytest.raises(EngineError, match="surrogate test"):
        h.pvalues()
    with pytest.raises(EngineError, match="cluster test"):
        h.cluster_labels()
    for bad in (0, -1, 2 ** 31, 1.5, True):
        with pytest.raises(ValueError, match="mc_count"):
            h.surrogate_test(mc_count=bad)
    with pytest.raises(ValueError, match="null"):
        h.surrogate_test(mc_count=2, null='white')
    with pytest.raises(ValueError, match="null"):
        h.cluster_test(np.ones(len(h.scales)), mc_count=2, null=None)
    with pytest.raises(ValueError, match="signif"):
        h.cluster_test(np.ones(3), mc_count=2)
    helpers.set_fft_padding(False)
    with pytest.raises(ValueError, match="padding"):
        h.surrogate_test(mc_count=2)
    helpers.set_fft_padding(True)
    h.surrogate_test(mc_count=2, seed=1)
    p_good = h.pvalues()
    # a stale serial at the engine level
    eng = h.engine
    kind, g, m, sigma = h._null('ar1')
    geo = (h.dt, h.scales, *h.wavelet._engine_spec())
    with pytest.raises(EngineError, match="serial"):
        eng.power_surrogate_counts(h._yn, kind, g, m, sigma, 1, 0, 1, *geo, h._serial + 1)
    with pytest.raises(EngineError, match="AR\\(1\\)"):
        eng.power_surrogate_counts(h._yn, kind, 1.0, m, sigma, 1, 0, 1, *geo, h._serial)
    with pytest.raises(EngineError, match="unknown null"):
        eng.power_surrogate_counts(h._yn, 7, g, m, sigma, 1, 0, 1, *geo, h._serial)
    with pytest.raises(EngineError, match="scales or length"):
        eng.power_surrogate_counts(h._yn, kind, g, m, sigma, 1, 0, 1, h.dt, h.scales[:-1],
                                   *h.wavelet._engine_spec(), h._serial)
    # each failing call returned before it began counting: the counts of the last good one stay
    assert np.array_equal(h.pvalues(), p_good, equal_nan=True)
    h2 = api.power_resident(x, 1.0, **KW)   # a new power_resident ends the old handle
    with pytest.raises(EngineError, match="no longer resident"):
        h.wave()
    with pytest.raises(EngineError, match="surrogate test"):
        h2.pvalues()
    h2.release()
    with pytest.raises(EngineError, match="no longer resident"):
        h2.wave()
    h2.release()   # releasing an invalid handle does nothing

    class Duck(object):
        def psi_ft(self, f):
            return np.exp(-f ** 2)

    with pytest.raises(TypeError, match="power_resident"):
        api.power_resident(x, 1.0, wavelet=Duck())
    with pytest.raises(ValueError, match="precision"):
        api.power_resident(x, 1.0, precision='fp16')
