"""Tests of the resident cross spectrum against AR(1) and phase-randomised surrogate pairs
(`xwt_resident`, `ResidentCrossWavelet` and the engine calls `mc_ar1_pair_surrogates`,
`cross_surrogate_counts`, `cross_cluster_test`, `cross_cluster_row_stats`), checked on the
host-emulation build of the kernels (tests/_emu):

  * the AR(1) pairs: series 0 is the power test's unit bit for bit, series 1 a host restatement
    under the series tag 1, the two differ with equal parameters, and splitting the units over calls
    changes nothing;
  * the counts are the definition k = #{i : P_i >= P_obs or P_i not finite}, P = |W12|^2, bit for
    bit, against a recount of the hooks' pairs through engine-level `xwt` one pair at a time, for
    both nulls, fp64 and fp32, Morlet, Paul and DOG, padded, 2^k and un-padded lengths, with
    accumulation and reset;
  * the p-values, fractions, FDR threshold, `global_power(alpha=)` and `mean_phase(alpha=)` of the
    same recount, and the clusters with `global_power(cluster=)` / `mean_phase(cluster=)`;
  * inputs scaled by powers of two leave the counts and the clusters bit-identical;
  * nothing else moves: W12 and the other resident slots stay byte-identical;
  * lifetime and errors.
"""
import numpy as np
import pytest

import test_emu_cluster_test as C
import test_emu_power_test as E
import test_emu_surrogate_pvalues as P
import test_emu_surrogate_significance as T
from test_emu_surrogate_significance import emu, api, red  # noqa: F401  (fixtures)

F64, F32 = T.F64, T.F32
CROSS = 'cross'   # pycwt_b200._engine.CROSS
KW = dict(dj=0.5, s0=2.0)


# ---- the AR(1) pairs -----------------------------------------------------------------------------
def ar1_host(g, m, sigma, seed, unit, n, tag):
    """Series `tag` of unit `unit` in longdouble: E.ar1_host with the counter's second word
    2^31 | tag."""
    j = np.arange((n + 1) // 2, dtype=np.uint64)
    o = T.philox4x32_10(j, 0x80000000 | tag, unit & 0xFFFFFFFF, 0x80000000 | ((unit >> 32) << 2) | 3, seed)
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
    z[0] = acc = e[0]
    for i in range(1, n):
        acc = gl * acc + s * e[i]
        z[i] = acc
    return np.longdouble(m) + np.longdouble(sigma) * z


def check_ar1_pairs(eng, n):
    g, m, sigma = (0.7, -0.4), (0.0, 3.0), (1.0, 2.5)
    pairs = eng.mc_ar1_pair_surrogates(g, m, sigma, 1234, 0, 4, n)
    assert pairs.shape == (4, 2, n)
    # series 0 is the power test's stream, bit for bit
    assert np.array_equal(pairs[:, 0], eng.mc_ar1_surrogates(g[0], m[0], sigma[0], 1234, 0, 4, n))
    # series 1: tag 1
    for u in (0, 3):
        ref = ar1_host(g[1], m[1], sigma[1], 1234, u, n, 1)
        tol = 16 * np.finfo(float).eps * sigma[1] / (1 - abs(g[1])) * \
            max(1.0, float(np.abs(ref - m[1]).max()) / sigma[1])
        assert float(np.abs(pairs[u, 1].astype(np.longdouble) - ref).max()) <= tol
    # equal parameters: two different series
    same = eng.mc_ar1_pair_surrogates((0.5, 0.5), (0.0, 0.0), (1.0, 1.0), 7, 0, 2, n)
    assert not np.array_equal(same[:, 0], same[:, 1])
    if n >= 1000:
        assert abs(np.corrcoef(same[0, 0], same[0, 1])[0, 1]) < 0.2
    # splitting the units over calls
    a = eng.mc_ar1_pair_surrogates(g, m, sigma, 1234, 0, 1, n)
    b = eng.mc_ar1_pair_surrogates(g, m, sigma, 1234, 1, 3, n)
    assert np.array_equal(pairs, np.concatenate([a, b]))
    far = eng.mc_ar1_pair_surrogates(g, m, sigma, 1234, 2 ** 40, 1, 64)
    assert np.abs(far[0, 1] - ar1_host(g[1], m[1], sigma[1], 1234, 2 ** 40, 64, 1).astype(float)).max() < 1e-12


@pytest.mark.parametrize("n", [4, 1001, 9000])
def test_ar1_pairs(emu, n):
    check_ar1_pairs(emu, n)


def test_ar1_pair_errors(emu):
    from pycwt_b200._engine import EngineError
    for g, m, s in (((0.5, 1.0), (0, 0), (1, 1)), ((0.5, 0.5), (0, np.nan), (1, 1)), ((0.5, 0.5), (0, 0), (1, np.inf))):
        with pytest.raises(EngineError, match="AR\\(1\\)"):
            emu.mc_ar1_pair_surrogates(g, m, s, 1, 0, 1, 16)
    with pytest.raises(ValueError, match="one entry per series"):
        emu.mc_ar1_pair_surrogates((0.5,), (0, 0), (1, 1), 1, 0, 1, 16)
    with pytest.raises(EngineError, match="bad argument"):
        emu.mc_ar1_pair_surrogates((0.5, 0.5), (0, 0), (1, 1), 1, -1, 1, 16)


# ---- the recount -------------------------------------------------------------------------------
def pair(n, seed=3):
    rs = np.random.RandomState(seed)
    return red(rs, n, 0.6)[0] * 3.0 + 1.5, red(rs, n, 0.3)[0] * 0.5 - 2.0


def surrogates(h, null, seed, first, count):
    """The pairs the handle's tests draw, from the hooks, [count, 2, n0]."""
    eng = h.engine
    kind, g, m, sigma = h._null(null)
    if null == 'ar1':
        return eng.mc_ar1_pair_surrogates(g, m, sigma, seed, first, count, h.n0)
    return eng.mc_phase_surrogates(h._yn, (0, 1), seed, first, count)


def engine_prec(h):
    pow2 = h.n0 & (h.n0 - 1) == 0
    return F32 if h.precision == 'fp32' and (h._padding or pow2) else F64


def unit_powers(h, null, seed, first, count):
    """|W12_i|^2 [count, S, n0] of engine-level `xwt` of each pair, in the handle's precision, formed
    as re*re + im*im in double (NumPy does not fuse)."""
    eng = h.engine
    out = []
    for x in surrogates(h, null, seed, first, count):
        W = eng.xwt(x[0], x[1], h.dt, h.scales, *h.wavelet._engine_spec(), precision=engine_prec(h))
        out.append(W.real * W.real + W.imag * W.imag)
    return np.array(out)


def obs_power(h):
    W = h.cross_spectrum()
    return W.real * W.real + W.imag * W.imag


recount, p_of = E.recount, E.p_of
CASES = E.CASES
WAVELETS = E.WAVELETS


def resident(api, prec, wav, n0, padded, normalize=True, seed=3):
    from pycwt_b200 import helpers
    helpers.set_fft_padding(padded)
    y1, y2 = pair(n0, seed)
    return api.xwt_resident(y1, y2, 1.0, wavelet=WAVELETS[wav](api), precision=prec, normalize=normalize, **KW)


padding = E.padding


def check_counts_are_the_definition(api, null, prec, wav, n0, padded):
    h = resident(api, prec, wav, n0, padded, normalize=(null == 'phase'))
    Pobs = obs_power(h)
    W0 = h.cross_spectrum().tobytes()
    M = 5
    h.surrogate_test(mc_count=M, seed=21, null=null)
    assert h.surrogate_units == M and h.surrogate_seed == 21
    Pi = unit_powers(h, null, 21, 0, M)
    assert np.array_equal(h.pvalues(), p_of(recount(Pobs, Pi), M, Pobs), equal_nan=True)
    assert h.cross_spectrum().tobytes() == W0
    # accumulation over calls: [0, 2) then [2, M) equals [0, M); reset starts over
    eng = h.engine
    kind, g, m, sigma = h._null(null)
    args = (h._yn, kind, g, m, sigma, 21)
    geo = (h.dt, h.scales, *h.wavelet._engine_spec(), h._serial)
    S, n = h.shape
    eng.cross_surrogate_counts(*args, 0, 2, *geo, reset=True)
    assert np.array_equal(eng.pvalue_window(CROSS, 0, S, 1, 0, n, 1),
                          p_of(recount(Pobs, Pi[:2]), 2, Pobs), equal_nan=True)
    eng.cross_surrogate_counts(*args, 2, M - 2, *geo, reset=False)
    assert np.array_equal(eng.pvalue_window(CROSS, 0, S, 1, 0, n, 1),
                          p_of(recount(Pobs, Pi), M, Pobs), equal_nan=True)
    eng.cross_surrogate_counts(*args, 2, M - 2, *geo, reset=True)
    assert np.array_equal(eng.pvalue_window(CROSS, 0, S, 1, 0, n, 1),
                          p_of(recount(Pobs, Pi[2:]), M - 2, Pobs), equal_nan=True)


@pytest.mark.parametrize("null,prec,wav,n0,padded", CASES)
def test_counts_are_the_definition(api, emu, padding, null, prec, wav, n0, padded):
    check_counts_are_the_definition(api, null, prec, wav, n0, padded)


def host_sums(W, sel):
    """Per row: count, sum |W|^2, sum |W|, sum cos arg W, sum sin arg W over sel (phase 0 at 0)."""
    Pw = W.real * W.real + W.imag * W.imag
    m = np.sqrt(Pw)
    safe = np.where(m > 0, m, 1.0)
    cs = np.where(m > 0, W.real / safe, 1.0)
    sn = np.where(m > 0, W.imag / safe, 0.0)
    return np.stack([sel.sum(axis=1), np.where(sel, Pw, 0).sum(axis=1), np.where(sel, m, 0).sum(axis=1),
                     np.where(sel, cs, 0).sum(axis=1), np.where(sel, sn, 0).sum(axis=1)], axis=1)


def check_mean_phase(mp, st):
    """MeanPhase of the whole band against host sums st [S, 5]."""
    cnt, c, s = st[:, 0].sum(), st[:, 3].sum(), st[:, 4].sum()
    assert mp.count == int(cnt)
    if cnt:
        assert abs(mp.angle - np.arctan2(s, c)) <= 1e-12
        assert abs(mp.strength - np.hypot(c, s) / cnt) <= 1e-13
    else:
        assert np.isnan(mp.angle)


def check_readers(api, null='phase', prec='fp64', n0=600):
    y1, y2 = pair(n0, 5)
    h = api.xwt_resident(y1, y2, 1.0, precision=prec, **KW)
    W = h.cross_spectrum()
    Pobs = W.real * W.real + W.imag * W.imag
    M = 7
    h.surrogate_test(mc_count=M, seed=5, null=null)
    p = p_of(recount(Pobs, unit_powers(h, null, 5, 0, M)), M, Pobs)
    assert np.array_equal(h.pvalues(slice(1, None, 3), slice(5, n0 - 10, 7)), p[1::3, 5:n0 - 10:7],
                          equal_nan=True)
    assert np.array_equal(h.pvalues(), p, equal_nan=True)
    lo, hi = h.coi_ranges()
    cols = np.arange(h.n0)[None]
    cone = (cols >= lo[:, None]) & (cols < hi[:, None])
    fin = np.isfinite(p)
    for alpha in (0.25, 0.5):
        sel = cone & fin & (p <= alpha)
        tested = (cone & fin).sum(axis=1)
        frac = h.pvalue_fraction(alpha)
        assert np.array_equal(frac[tested > 0], sel.sum(axis=1)[tested > 0] / tested[tested > 0])
        assert np.isnan(frac[tested == 0]).all()
        st = host_sums(W, sel)
        gp = h.global_power(inside_coi=True, alpha=alpha)
        ok = st[:, 0] > 0
        assert np.allclose(gp[ok], st[ok, 2] / st[ok, 0], rtol=1e-13, atol=0) and np.isnan(gp[~ok]).all()
        check_mean_phase(h.mean_phase(alpha=alpha), st)
        # with a threshold as well (|W12| units)
        sig = np.quantile(np.sqrt(Pobs), 0.5, axis=1)
        st2 = host_sums(W, sel & (Pobs > (sig ** 2)[:, None]))
        check_mean_phase(h.mean_phase(alpha=alpha, signif=sig), st2)
    for method in ('bh', 'by'):
        for inside in (True, False):
            for q in (0.05, 0.3, 0.9):
                P.check_fdr(h.fdr_threshold(q, method, inside), p[fin & (cone if inside else True)], q, method)
    # both None: today's results
    assert np.array_equal(h.global_power(), h.global_power(alpha=None, cluster=None), equal_nan=True)
    return h


def test_readers(api, emu):
    check_readers(api)


def check_cluster_test(api, null, prec, n0=700, M=6):
    y1, y2 = pair(n0, 8)
    h = api.xwt_resident(y1, y2, 1.0, precision=prec, **KW)
    W = h.cross_spectrum()
    Pobs = W.real * W.real + W.imag * W.imag
    h.surrogate_test(mc_count=3, seed=1, null=null)
    p0 = h.pvalues()
    sig = np.sqrt(np.quantile(Pobs, 0.7, axis=1))    # |W12| units
    res = h.cluster_test(sig, mc_count=M, seed=4, null=null)
    q = C.weights(h.scales)
    lo, hi = h.coi_ranges()
    cols = np.arange(h.n0)[None]
    cone = (cols >= lo[:, None]) & (cols < hi[:, None])
    thr = (sig ** 2)[:, None]     # squared on the host as the handle squares it

    def select(Pm):
        return np.isfinite(Pm) & (Pm > thr) & cone

    rQ, rpts, rbox, rlab = C.reference(select(Pobs), q)
    from pycwt_b200.resident import _cluster_weights
    _, unit_area = _cluster_weights(h)
    assert np.array_equal(res.area, rQ.astype(float) * unit_area)
    assert np.array_equal(res.points, rpts)
    assert np.array_equal(np.column_stack([res.rows, res.cols]), rbox)
    lab = h.cluster_labels()
    assert np.array_equal(lab, rlab)
    qmax = [C.reference(select(Pi), q)[0] for Pi in unit_powers(h, null, 4, 0, M)]
    qmax = np.array([int(x[0]) if x.size else 0 for x in qmax], dtype=float) * unit_area
    assert np.array_equal(res.null_max, qmax)
    reached = np.array([(qmax >= a).sum() for a in res.area])
    assert np.array_equal(res.pvalue, (1.0 + reached) / (1.0 + M))
    assert h.cross_spectrum().tobytes() == W.tobytes()
    assert np.array_equal(h.pvalues(), p0, equal_nan=True)   # the counts are kept
    # reductions over one cluster
    assert res.area.size >= 2
    for c in (0, 1, res.area.size - 1):
        st = host_sums(W, lab == c + 1)
        assert st[:, 0].sum() == res.points[c]
        gp = h.global_power(cluster=c)
        ok = st[:, 0] > 0
        assert np.allclose(gp[ok], st[ok, 2] / st[ok, 0], rtol=1e-13, atol=0) and np.isnan(gp[~ok]).all()
        check_mean_phase(h.mean_phase(cluster=c), st)
        mp = h.mean_phase(cluster=c, per_scale=True)
        assert np.array_equal(mp.count, st[:, 0].astype(np.int64))
        # the engine call reads the box only: the whole rows give the same sums
        S = len(h.scales)
        full = h.engine.cross_cluster_row_stats(c, np.zeros(S, np.int64), np.full(S, h.n0, np.int64))
        assert np.array_equal(full[:, 0], st[:, 0])
    return h, res


@pytest.mark.parametrize("null,prec", [('ar1', 'fp64'), ('phase', 'fp32'), ('phase', 'fp64')])
def test_cluster_test_against_recount(api, emu, null, prec):
    check_cluster_test(api, null, prec)


def check_scaling(api, prec, exps, null):
    """normalize=False: y1 2^a, y2 2^b leave the counts, p-values, cluster tables and labels
    bit-identical (the nulls' m and sigma, the units, W12 and signif all scale exactly)."""
    y1, y2 = pair(512, 11)
    out = []
    for a, b in [(0, 0)] + exps:
        h = api.xwt_resident(np.ldexp(y1, a), np.ldexp(y2, b), 1.0, normalize=False, precision=prec, **KW)
        h.surrogate_test(mc_count=4, seed=3, null=null)
        res = h.cluster_test(h.signif, mc_count=4, seed=6, null=null)
        out.append((h.pvalues(), res.area, res.points, res.rows, res.cols, res.pvalue, res.null_max,
                    h.cluster_labels(), h.fdr_threshold(0.3)))
    for (a, b), o in zip(exps, out[1:]):
        for x, y in zip(out[0], o):
            assert np.array_equal(np.asarray(x), np.asarray(y), equal_nan=True), (prec, null, a, b)


@pytest.mark.parametrize("prec,exps", [('fp64', [(200, -190), (-200, 180)]), ('fp32', [(24, 20), (-40, 30)])])
@pytest.mark.parametrize("null", ['ar1', 'phase'])
def test_scaling(api, emu, prec, exps, null):
    check_scaling(api, prec, exps, null)


def check_nothing_else_moves(api):
    x, y = pair(512, 1)
    z = pair(512, 2)[0]
    hc = api.wct_resident(x, y, 1.0, **KW)
    hp = api.power_resident(z, 1.0, **KW)
    h3 = api.wct3_resident(x, y, z, 1.0, **KW)
    h = api.xwt_resident(x, y, 1.0, **KW)
    hp.surrogate_test(mc_count=2, seed=1)
    hp.cluster_test(np.full(len(hp.scales), 2.0), mc_count=2, seed=2)
    pp, lp = hp.pvalues(), hp.cluster_labels()

    def state():
        return [hc.coherence().tobytes(), hp.wave().tobytes(), h3.partial().tobytes(),
                h.cross_spectrum().tobytes()]

    before = state()
    h.surrogate_test(mc_count=3, seed=2)
    h.cluster_test(h.signif, mc_count=3, seed=3, null='phase')
    assert state() == before
    assert np.array_equal(hp.pvalues(), pp, equal_nan=True) and np.array_equal(hp.cluster_labels(), lp)
    p, lab = h.pvalues(), h.cluster_labels()
    # the other calls leave the cross spectrum, its counts and clusters as they were
    api.cwt(x, 1.0, **KW)
    api.xwt(x, y, 1.0, **KW)
    api.wct(x, y, 1.0, sig=False, **KW)
    hp.surrogate_test(mc_count=2, seed=1, null='phase')
    hp.cluster_test(np.full(len(hp.scales), 2.0), mc_count=2, seed=2)
    hc.surrogate_test(mc_count=2, seed=1)
    api.cwt_resident(x, 1.0, **KW)
    assert h.cross_spectrum().tobytes() == before[3]
    assert np.array_equal(h.pvalues(), p, equal_nan=True)
    assert np.array_equal(h.cluster_labels(), lab)
    assert hc.coherence().tobytes() == before[0]


def test_nothing_else_moves(api, emu):
    check_nothing_else_moves(api)


def check_lifetime_and_errors(api):
    from pycwt_b200 import helpers
    from pycwt_b200._engine import EngineError
    x, y = pair(256)
    h = api.xwt_resident(x, y, 1.0, **KW)
    with pytest.raises(EngineError, match="surrogate test"):
        h.pvalues()
    with pytest.raises(EngineError, match="cluster test"):
        h.cluster_labels()
    with pytest.raises(EngineError, match="cluster test"):
        h.mean_phase(cluster=0)
    for bad in (0, -1, 2 ** 31, 1.5, True):
        with pytest.raises(ValueError, match="mc_count"):
            h.surrogate_test(mc_count=bad)
    with pytest.raises(ValueError, match="null"):
        h.surrogate_test(mc_count=2, null='white')
    with pytest.raises(ValueError, match="null"):
        h.cluster_test(h.signif, mc_count=2, null=None)
    with pytest.raises(ValueError, match="signif"):
        h.cluster_test(np.ones(3), mc_count=2)
    helpers.set_fft_padding(False)
    with pytest.raises(ValueError, match="padding"):
        h.surrogate_test(mc_count=2)
    with pytest.raises(ValueError, match="padding"):
        h.cluster_test(h.signif, mc_count=2)
    helpers.set_fft_padding(True)
    h.surrogate_test(mc_count=2, seed=1)
    p_good = h.pvalues()
    res = h.cluster_test(h.signif * 0.5, mc_count=2, seed=1)
    assert res.area.size > 0
    for bad in (-1, res.area.size, 1.0, True):
        with pytest.raises(ValueError, match="cluster"):
            h.global_power(cluster=bad)
    with pytest.raises(ValueError, match="signif or alpha"):
        h.mean_phase(cluster=0, alpha=0.5)
    with pytest.raises(ValueError, match="signif or alpha"):
        h.global_power(cluster=0, signif=h.signif)
    eng = h.engine
    S = len(h.scales)
    z, n = np.zeros(S, np.int64), np.full(S, h.n0, np.int64)
    with pytest.raises(EngineError, match="no such cluster"):
        eng.cross_cluster_row_stats(res.area.size, z, n)
    with pytest.raises(EngineError, match="no such cluster"):
        eng.cross_cluster_row_stats(-1, z, n)
    # a stale serial, bad parameters, an unknown null, another shape at the engine level
    kind, g, m, sigma = h._null('ar1')
    geo = (h.dt, h.scales, *h.wavelet._engine_spec())
    with pytest.raises(EngineError, match="serial"):
        eng.cross_surrogate_counts(h._yn, kind, g, m, sigma, 1, 0, 1, *geo, h._serial + 1)
    with pytest.raises(EngineError, match="AR\\(1\\)"):
        eng.cross_surrogate_counts(h._yn, kind, [g[0], 1.0], m, sigma, 1, 0, 1, *geo, h._serial)
    with pytest.raises(EngineError, match="unknown null"):
        eng.cross_surrogate_counts(h._yn, 7, g, m, sigma, 1, 0, 1, *geo, h._serial)
    with pytest.raises(EngineError, match="scales or length"):
        eng.cross_surrogate_counts(h._yn, kind, g, m, sigma, 1, 0, 1, h.dt, h.scales[:-1],
                                   *h.wavelet._engine_spec(), h._serial)
    with pytest.raises(EngineError, match="scales or length"):
        eng.cross_surrogate_counts(h._yn[:, :-1], kind, g, m, sigma, 1, 0, 1, *geo, h._serial)
    with pytest.raises(ValueError, match="\\[2, n0\\]"):
        eng.cross_surrogate_counts(h._yn[0], kind, g, m, sigma, 1, 0, 1, *geo, h._serial)
    # each failing counting call returned before it began counting: the counts of the last good one stay
    assert np.array_equal(h.pvalues(), p_good, equal_nan=True)
    # a failing cluster test leaves no clusters readable
    with pytest.raises(EngineError, match="unknown null"):
        eng.cross_cluster_test(h._yn, 7, g, m, sigma, 1, 0, 1, *geo, h._serial, (h.signif ** 2), *h.coi_ranges(),
                               C.weights(h.scales))
    with pytest.raises(EngineError, match="cluster test"):
        h.cluster_labels()
    with pytest.raises(EngineError, match="cluster test"):
        eng.cluster_table(CROSS)
    # the counts and clusters die with the product
    h.cluster_test(h.signif * 0.5, mc_count=2, seed=1)
    h2 = api.xwt_resident(x, y, 1.0, **KW)   # a new xwt_resident ends the old handle
    with pytest.raises(EngineError, match="no longer resident"):
        h.cross_spectrum()
    with pytest.raises(EngineError, match="surrogate test"):
        h2.pvalues()
    with pytest.raises(EngineError, match="surrogate counts"):
        eng.pvalue_window(CROSS, 0, 1, 1, 0, 1, 1)
    with pytest.raises(EngineError, match="cluster test"):
        h2.cluster_labels()
    h2.surrogate_test(mc_count=2, seed=1)
    h2.cluster_test(h2.signif * 0.5, mc_count=2, seed=1)
    h2.release()
    with pytest.raises(EngineError, match="no longer resident"):
        h2.pvalues()
    with pytest.raises(EngineError, match="no cross spectrum"):
        eng.pvalue_window(CROSS, 0, 1, 1, 0, 1, 1)
    with pytest.raises(EngineError, match="no cross spectrum"):
        eng.cluster_table(CROSS)
    h2.release()   # releasing an invalid handle does nothing


def test_lifetime_and_errors(api, emu, padding):
    check_lifetime_and_errors(api)
