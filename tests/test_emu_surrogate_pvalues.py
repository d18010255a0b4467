"""Point-wise tests of the resident coherence against phase-randomised surrogates (`surrogate_test`,
`pvalues`, `pvalue_fraction`, `fdr_threshold`, `global_coherence` / `mean_phase` with `alpha`, and
the engine calls `surrogate_counts`, `pvalue_window`, `pvalue_row_stats`, `count_hist`), checked on
the host-emulation build of the kernels (tests/_emu):

  * the counts are the definition k = #{i : R2_i >= R2_obs}, bit for bit, against a recount of the
    hook's surrogates through engine-level `wct` / `wct3` one unit at a time, on every row (also
    those from maxscale on), with the K > 32 boxcar, padded, 2^k and un-padded lengths;
  * nothing else moves: the histograms are those of `wct_mc_phase`, the levels those of
    `surrogate_significance`, the resident fields stay byte-identical;
  * accumulation over calls, reset, reading, FDR against SciPy, lifetime and errors;
  * the test does what it claims on red noise and on a shared sinusoid.
"""
import numpy as np
import pytest
from scipy.stats import false_discovery_control

import test_emu_surrogate_significance as T
from test_emu_surrogate_significance import emu, api, red  # noqa: F401  (fixtures)

F64, F32 = T.F64, T.F32
NBINS = T.NBINS
MORLET = T.MORLET
ERR_ARG, ERR_STATE = -1, -4


def setup(eng, nser, n0, K, prec, S=20, seed=5):
    """Data, scales, mask, and the resident product of the data (engine level)."""
    rs = np.random.RandomState(n0 + K + nser)
    x = red(rs, n0, 0.6, nser)
    x[-1] += 0.7 * x[-2]
    sj = 2.0 * 2 ** (np.arange(S) / 4.0)
    mask = ((np.arange(n0)[None, :] + 3 * np.arange(S)[:, None]) % 7 != 0).astype(np.uint8)
    if nser == 2:
        serial = eng.wct_resident(x[0], x[1], 1.0, 0.25, sj, MORLET, 6.0, K, precision=prec)
    else:
        serial = eng.wct3_resident(x[0], x[1], x[2], 1.0, 0.25, sj, MORLET, 6.0, K, precision=prec)
    return x, sj, mask, serial


def observed(eng, nser):
    """The resident fields, in the order the counts are kept (and the phases, to check they stay)."""
    S, n0, _ = eng._shape(2 if nser == 2 else 3)
    if nser == 2:
        return list(eng.coherence_window(0, S, 1, 0, n0, 1))
    return [eng.coherence3_window(0, 0, S, 1, 0, n0, 1, want_phase=True)[0],
            eng.coherence3_window(1, 0, S, 1, 0, n0, 1)[0],
            eng.coherence3_window(0, 0, S, 1, 0, n0, 1, want_value=False, want_phase=True)[1]]


def recount(eng, x, groups, seed, first, units, sj, K, prec, obs, dt=1.0, f0=6.0):
    """k per measure from the hook's surrogates through engine-level wct / wct3, unit by unit."""
    nser = x.shape[0]
    surr = eng.mc_phase_surrogates(x, groups, seed, first, units)
    k = [np.zeros(o.shape, dtype=np.int64) for o in obs]
    for u in range(units):
        if nser == 2:
            R = [eng.wct(surr[u, 0], surr[u, 1], dt, 0.25, sj, MORLET, f0, K, want_angle=False,
                         precision=prec)[0]]
        else:
            R = list(eng.wct3(*surr[u], dt, 0.25, sj, MORLET, f0, K, precision=prec))
        for kk, r, o in zip(k, R, obs):
            kk += (~np.isfinite(r)) | (r >= o)
    return k


def counted_p(eng, nser):
    """The p-value fields of the engine's counts, per measure."""
    S, n0, _ = eng._shape(2 if nser == 2 else 3)
    if nser == 2:
        return [eng.pvalue_window(None, 0, S, 1, 0, n0, 1)]
    return [eng.pvalue_window(m, 0, S, 1, 0, n0, 1) for m in (0, 1)]


def p_of(k, M, obs):
    return np.where(np.isfinite(obs), (1 + k) / (1 + M), np.nan)


def count(eng, x, groups, seed, first, units, sj, mask, maxscale, K, prec, serial, reset=True):
    nser = x.shape[0]
    hs = [np.zeros((sj.size, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    eng.surrogate_counts(x, groups, seed, first, units, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hs,
                         serial=serial, reset=reset, precision=prec)
    return hs


def check_counts_are_the_definition(eng, nser, n0, K, prec, M=5, seed=31):
    x, sj, mask, serial = setup(eng, nser, n0, K, prec)
    S = sj.size
    maxscale = S - 3
    groups = (0, 1) if nser == 2 else (0, 1, 1)
    before = observed(eng, nser)
    obs = before[:nser - 1]
    hs = count(eng, x, groups, seed, 0, M, sj, mask, maxscale, K, prec, serial)
    # nothing else moves: the resident fields, byte for byte, and the histograms of wct_mc_phase
    after = observed(eng, nser)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before, after))
    hh = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    eng.wct_mc_phase(x, groups, seed, 0, M, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hh, precision=prec)
    assert all(np.array_equal(a, b) for a, b in zip(hs, hh))
    # the counts are the definition, on every row
    k = recount(eng, x, groups, seed, 0, M, sj, K, prec, obs)
    ps = counted_p(eng, nser)
    for p, kk, o in zip(ps, k, obs):
        assert np.array_equal(p, p_of(kk, M, o), equal_nan=True)
        assert 0 < kk[maxscale:].sum() < M * kk[maxscale:].size      # rows from maxscale on are counted
        fin = np.isfinite(p)
        assert (p[fin] >= 1 / (M + 1)).all() and (p[fin] <= 1).all()
    # units [0, 2) plus [2, M) are one call over [0, M)
    count(eng, x, groups, seed, 0, 2, sj, mask, maxscale, K, prec, serial)
    count(eng, x, groups, seed, 2, M - 2, sj, mask, maxscale, K, prec, serial, reset=False)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(counted_p(eng, nser), ps))
    # reset zeroes them: two units on top of the five are the two units alone
    count(eng, x, groups, seed, 3, 2, sj, mask, maxscale, K, prec, serial)
    k2 = recount(eng, x, groups, seed, 3, 2, sj, K, prec, obs)
    assert all(np.array_equal(p, p_of(kk, 2, o), equal_nan=True) for p, kk, o in zip(counted_p(eng, nser), k2, obs))
    return k


@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser", [2, 3])
@pytest.mark.parametrize("n0,K", [(512, 6), (600, 36)])
def test_counts_are_the_definition(emu, nser, n0, K, prec):
    """2^k, and a padded length (600 runs at 1024) with a boxcar longer than 32."""
    check_counts_are_the_definition(emu, nser, n0, K, prec)


@pytest.mark.parametrize("nser", [2, 3])
def test_counts_unpadded(emu, nser):
    """The un-padded transforms (fp64) of a length that is not 2^k."""
    emu.set_padding(False)
    try:
        check_counts_are_the_definition(emu, nser, 600, 6, F64, M=3)
    finally:
        emu.set_padding(True)


def test_nan_observed_point(emu):
    """x1 == x2: the denominator of RP2 vanishes, and so does its p-value."""
    rs = np.random.RandomState(3)
    x = red(rs, 256, 0.5, 3)
    x[2] = x[1]
    sj = 2.0 * 2 ** (np.arange(8) / 2.0)
    serial = emu.wct3_resident(x[0], x[1], x[2], 1.0, 0.5, sj, MORLET, 6.0, 3)
    mask = np.ones((8, 256), dtype=np.uint8)
    count(emu, x, (0, 1, 1), 2, 0, 4, sj, mask, 6, 3, F64, serial)
    RP2 = emu.coherence3_window(0, 0, 8, 1, 0, 256, 1)[0]
    p = emu.pvalue_window(0, 0, 8, 1, 0, 256, 1)
    assert (~np.isfinite(RP2)).any()
    assert np.array_equal(np.isnan(p), ~np.isfinite(RP2))
    lo, hi = np.zeros(8, dtype=np.int64), np.full(8, 256, dtype=np.int64)
    assert emu.count_hist(0, lo, hi, 5).sum() == np.isfinite(RP2).sum()
    st = emu.pvalue_row_stats(0, lo, hi, 4)
    assert np.array_equal(st[:, 0], np.isfinite(RP2).sum(axis=1))


# ---- the public calls ----------------------------------------------------------------------------
def pair(n0=1024, seed=4):
    rs = np.random.RandomState(seed)
    x = red(rs, n0, 0.7, 2)
    x[1] += 0.6 * x[0]
    return x


def triple(n0=1024, seed=6):
    rs = np.random.RandomState(seed)
    x = red(rs, n0, 0.7, 3)
    x[0] += 0.5 * x[1]
    x[2] += 0.5 * x[1]
    return x


KW = dict(dj=1 / 4, s0=2.0, J=24)


def fields(h):
    if hasattr(h, 'coherence'):
        return [h.coherence(), h.phase()]
    return [h.partial(), h.phase(), h.multiple()]


def host_p(api, h, M, seed, conditional=True):
    """The handle's p-values per measure, recounted from the hook through engine-level wct / wct3."""
    from pycwt_b200.wavelet import _wct_problem
    eng = h.engine
    p = _wct_problem(h._y, h.dt, h.dj, h.s0, h.J, h.wavelet, h.normalize, h.precision)
    prec = F32 if h.precision == 'fp32' else F64
    nser = len(p.yns)
    groups = (0, 1) if nser == 2 else ((0, 1, 1) if conditional else (0, 1, 2))
    obs = fields(h)
    obs = obs[:1] if nser == 2 else [obs[0], obs[2]]
    k = recount(eng, np.stack(p.yns), groups, seed, 0, M, p.sj, p.klen, prec, obs)
    return [p_of(kk, M, o) for kk, o in zip(k, obs)], obs


@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
def test_public_pair(api, emu, prec):
    x = pair()
    h = api.wct_resident(x[0], x[1], 1.0, precision=prec, **KW)
    before = [f.tobytes() for f in fields(h)]
    g0 = h.global_coherence(inside_coi=True)
    m0 = h.mean_phase(per_scale=True)
    lev = h.surrogate_test(mc_count=6, seed=11)
    assert h.surrogate_units == 6 and h.surrogate_seed == 11
    assert np.array_equal(lev, h.surrogate_significance(mc_count=6, seed=11), equal_nan=True)
    assert np.array_equal(lev, api.wct_surrogate_significance(x[0], x[1], 1.0, mc_count=6, seed=11,
                                                              precision=prec, **KW), equal_nan=True)
    assert [f.tobytes() for f in fields(h)] == before
    # alpha=None: today's results, bit for bit
    assert np.array_equal(h.global_coherence(inside_coi=True), g0, equal_nan=True)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(h.mean_phase(per_scale=True), m0))
    (P,), (W,) = host_p(api, h, 6, 11)
    assert np.array_equal(h.pvalues(), P, equal_nan=True)
    assert np.array_equal(h.pvalues(slice(1, None, 3), slice(5, 900, 7)), P[1::3, 5:900:7], equal_nan=True)
    check_reductions(h, P, W, h.phase(), None)


@pytest.mark.parametrize("conditional", [True, False])
def test_public_triple(api, emu, conditional):
    x = triple()
    h = api.wct3_resident(*x, 1.0, **KW)
    before = [f.tobytes() for f in fields(h)]
    lev = h.surrogate_test(mc_count=5, seed=3, conditional=conditional)
    ref = h.surrogate_significance(mc_count=5, seed=3, conditional=conditional)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(lev, ref))
    ref = api.wct3_surrogate_significance(*x, 1.0, mc_count=5, seed=3, conditional=conditional, **KW)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(lev, ref))
    assert [f.tobytes() for f in fields(h)] == before
    Ps, Ws = host_p(api, h, 5, 3, conditional)
    for measure, P, W in zip(('partial', 'multiple'), Ps, Ws):
        assert np.array_equal(h.pvalues(measure=measure), P, equal_nan=True)
        check_reductions(h, P, W, h.phase(), measure)


def coi_mask(h):
    lo, hi = h.coi_ranges()
    n = np.arange(h.n0)
    return (n[None, :] >= lo[:, None]) & (n[None, :] < hi[:, None])


def check_reductions(h, P, W, phase, measure):
    """pvalue_fraction, global_coherence / mean_phase with alpha, fdr_threshold against NumPy / SciPy."""
    kw = {} if measure is None else dict(measure=measure)
    cone = coi_mask(h)
    fin = np.isfinite(P)
    M = h.surrogate_units
    sig = np.nanpercentile(W, 60, axis=1)
    for alpha in (1 / (M + 1), 0.5, 2.5 / (M + 1), 1.0):
        sel = fin & (P <= alpha)
        num, den = (sel & cone).sum(axis=1), (fin & cone).sum(axis=1)
        ref = np.where(den > 0, num / np.maximum(den, 1), np.nan)
        assert np.allclose(h.pvalue_fraction(alpha, **kw), ref, rtol=0, atol=0, equal_nan=True)
        for inside in (False, True):
            for s in (None, sig):
                pts = sel & (cone if inside else True) & (True if s is None else W > s[:, None])
                g = h.global_coherence(inside_coi=inside, alpha=alpha,
                                       **({} if s is None else {('sig95' if measure is None else 'sig'): s}), **kw)
                n = pts.sum(axis=1)
                ref = np.where(n > 0, np.where(pts, W, 0).sum(axis=1) / np.maximum(n, 1), np.nan)
                assert np.allclose(g, ref, rtol=1e-12, atol=0, equal_nan=True)
        if measure != 'multiple':
            pts = sel & cone & (W > sig[:, None])
            mp = h.mean_phase(alpha=alpha, per_scale=True, **({'sig95': sig} if measure is None else {'sig': sig}))
            c = np.where(pts, np.cos(phase), 0).sum(axis=1)
            sn = np.where(pts, np.sin(phase), 0).sum(axis=1)
            assert np.array_equal(mp.count, pts.sum(axis=1))
            ok = mp.count > 0
            assert np.allclose(mp.angle[ok], np.arctan2(sn, c)[ok], rtol=0, atol=1e-9)
    for method in ('bh', 'by'):
        for inside in (True, False):
            for q in (0.05, 0.3, 0.9, 1e-9):
                check_fdr(h.fdr_threshold(q, method, inside, **kw), P[fin & (cone if inside else True)], q, method)


def check_fdr(res, p, q, method):
    """FdrResult against scipy.stats.false_discovery_control on the same p-values."""
    assert res.tested == p.size
    if p.size == 0:
        assert res == (0.0, 0, 0)
        return
    rej = false_discovery_control(p, method=method) <= q
    assert res.rejected == int(rej.sum())
    assert res.alpha == (float(p[rej].max()) if rej.any() else 0.0)
    assert (p[rej] <= res.alpha).all() and not (p[~rej] <= res.alpha).any()


def test_fdr_ties_and_no_rejection(api, emu):
    """Small M: heavy ties.  q below the smallest reachable p: nothing rejected."""
    from pycwt_b200.resident import _fdr
    rs = np.random.RandomState(0)
    for M in (1, 2, 9, 99):
        for rej_rate in (0.0, 0.2, 0.9):
            k = rs.randint(0, M + 1, size=3000)
            k[: int(rej_rate * k.size)] = 0
            hist = np.bincount(k, minlength=M + 1)
            p = (1 + k) / (1 + M)
            for method in ('bh', 'by'):
                for q in (0.01, 0.05, 0.2, 0.6):
                    check_fdr(_fdr(hist, M, q, method), p, q, method)
    x = pair(512)
    h = api.wct_resident(x[0], x[1], 1.0, **KW)
    h.surrogate_test(mc_count=4, seed=1)
    res = h.fdr_threshold(0.1)
    assert res.rejected == 0 and res.alpha == 0.0 and res.tested > 0


def test_kmax():
    from pycwt_b200.resident import _kmax
    for M in (1, 5, 99, 999, 12345):
        for alpha in (1e-9, 1 / (M + 1), 0.01, 0.05, 0.1, 1 / 3, 0.5, 0.999, 1.0):
            k = _kmax(alpha, M)
            ok = [kk for kk in range(M + 1) if (1 + kk) / (1 + M) <= alpha]
            assert k == (max(ok) if ok else -1)


# ---- lifetime and errors -------------------------------------------------------------------------
def test_lifetime_and_errors(api, emu):
    from pycwt_b200 import _engine, helpers
    x = pair(512)
    y = triple(512)
    h = api.wct_resident(x[0], x[1], 1.0, **KW)
    h3 = api.wct3_resident(*y, 1.0, **KW)
    reads = lambda h, **kw: [lambda: h.pvalues(**kw), lambda: h.pvalue_fraction(0.05, **kw),  # noqa: E731
                             lambda: h.fdr_threshold(**kw), lambda: h.global_coherence(alpha=0.05, **kw)]
    for hh, kw in ((h, {}), (h3, {'measure': 'multiple'})):
        for f in reads(hh, **kw):
            with pytest.raises(_engine.EngineError, match="surrogate_test"):
                f()
    h.surrogate_test(mc_count=4, seed=2)
    h3.surrogate_test(mc_count=3, seed=2)
    p4 = h.pvalues()
    assert set(np.unique(p4[np.isfinite(p4)])) <= {(1 + k) / 5 for k in range(5)}
    # a second test with another M replaces the counts
    h.surrogate_test(mc_count=7, seed=2)
    p7 = h.pvalues()
    assert h.surrogate_units == 7 and np.nanmin(p7) >= 1 / 8
    assert set(np.unique(p7[np.isfinite(p7)])) <= {(1 + k) / 8 for k in range(8)}
    # argument errors
    for bad in (0, -1, 2 ** 31, 2.5, True):
        with pytest.raises(ValueError, match="mc_count"):
            h.surrogate_test(mc_count=bad)
    for bad in (0, -0.1, 1.5, np.nan):
        with pytest.raises(ValueError, match="alpha"):
            h.pvalue_fraction(bad)
        with pytest.raises(ValueError, match="alpha"):
            h.global_coherence(alpha=bad)
        with pytest.raises(ValueError, match="alpha"):
            h3.mean_phase(alpha=bad)
    for bad in (0, 1, -0.5, 2.0):
        with pytest.raises(ValueError, match="q must"):
            h.fdr_threshold(bad)
    with pytest.raises(ValueError, match="method"):
        h.fdr_threshold(0.05, method='holm')
    for f in (lambda: h3.pvalues(measure='x'), lambda: h3.pvalue_fraction(0.1, measure='both'),
              lambda: h3.fdr_threshold(measure=None), lambda: h3.global_coherence('rm', alpha=0.1)):
        with pytest.raises(ValueError, match="measure"):
            f()
    with pytest.raises(ValueError, match="rows"):
        h.pvalues(rows=slice(None, None, -1))
    # a changed padding mode
    helpers.set_fft_padding(False)
    try:
        with pytest.raises(ValueError, match="padding"):
            h.surrogate_test(mc_count=2, seed=1)
        with pytest.raises(ValueError, match="padding"):
            h3.surrogate_test(mc_count=2, seed=1)
    finally:
        helpers.set_fft_padding(True)
        emu.set_padding(True)
    # a failed test above left the counts of the last one readable: it never started
    assert np.array_equal(h.pvalues(), p7, equal_nan=True)
    # a newer wct_resident: the old handle is gone, the triple's counts stay
    h3p = h3.pvalues(measure='multiple')
    hn = api.wct_resident(x[1], x[0], 1.0, **KW)
    for f in reads(h):
        with pytest.raises(_engine.EngineError, match="no longer resident"):
            f()
    with pytest.raises(_engine.EngineError, match="surrogate_test"):
        hn.pvalues()
    assert np.array_equal(h3.pvalues(measure='multiple'), h3p, equal_nan=True)
    # the engine refuses to read counts of a product that has none
    assert emu.lib.cwtb_coherence_pvalue_window(emu.h, 0, 1, 1, 0, 1, 1, None) == ERR_STATE
    # release
    h3.release()
    for f in reads(h3, measure='partial'):
        with pytest.raises(_engine.EngineError, match="no longer resident"):
            f()
    hn.release()


def test_engine_errors(emu):
    x, sj, mask, serial = setup(emu, 2, 256, 3, F64, S=8)
    hs = [np.zeros((8, NBINS), dtype=np.int64)]
    args = (x, (0, 1), 1, 0, 2, 1.0, sj, MORLET, 6.0, 3, mask, 6, NBINS)
    from pycwt_b200._engine import EngineError
    with pytest.raises(EngineError, match="status -4"):            # not the product's serial
        emu.surrogate_counts(*args, *hs, serial=serial + 1)
    with pytest.raises(EngineError, match="status -4"):            # another scale vector
        emu.surrogate_counts(x, (0, 1), 1, 0, 2, 1.0, sj[:7], MORLET, 6.0, 3, mask[:7], 6, NBINS,
                             np.zeros((7, NBINS), dtype=np.int64), serial=serial)
    with pytest.raises(EngineError, match="status -4"):            # the triple has no product resident
        emu.coherence3_release()
        emu.surrogate_counts(np.vstack([x, x[:1]]), (0, 1, 1), 1, 0, 2, 1.0, sj, MORLET, 6.0, 3, mask, 6, NBINS,
                             *hs, None, serial=emu.coherence3_serial())
    emu.surrogate_counts(*args, *hs, serial=serial)
    lo, hi = np.zeros(8, dtype=np.int64), np.full(8, 256, dtype=np.int64)
    with pytest.raises(EngineError, match="M \\+ 1"):
        emu.count_hist(None, lo, hi, 4)
    assert emu.count_hist(None, lo, hi, 3).sum() == 8 * 256
    # the slot's release frees the counts with it
    emu.coherence_release()
    assert emu.lib.cwtb_coherence_count_hist(emu.h, None, None, 3, None) == ERR_STATE


# ---- it tests what it claims ---------------------------------------------------------------------
def test_red_noise_rate(api):
    """Two independent AR(1) series (a = 0.7), n0 = 2048, M = 99: the fraction of the 57080 in-cone
    points with p <= 0.05 is 0.0629 (observed with these seeds), inside [0.02, 0.08]; BH at
    q = 0.05 rejects none of them."""
    rs = np.random.RandomState(2024)
    x = red(rs, 2048, 0.7, 2)
    h = api.wct_resident(x[0], x[1], 1.0, dj=1 / 4, s0=2.0, J=30)
    h.surrogate_test(mc_count=99, seed=7)
    P = h.pvalues()
    cone = coi_mask(h)
    frac = (P[cone] <= 0.05).mean()
    assert 0.02 <= frac <= 0.08, frac
    assert h.fdr_threshold(0.05).rejected == 0


def test_shared_sinusoid_found(api):
    """Two series of independent red noise (a = 0.5) sharing a sinusoid of period 32 (amplitude 2.5)
    whose phase wanders (a random walk of 0.2 rad per sample), n0 = 2048, periods 8 .. 128, M = 99.
    A sinusoid of fixed phase would not do: it is one Fourier line, which phase randomisation keeps
    as a sinusoid in every surrogate, and two sinusoids of one period are coherent whatever their
    phases.  Observed with these seeds: BH at q = 0.05 rejects 9108 of the 32730 points in the cone
    (cut-off p = 0.01), 86 % of them within one octave of period 32, a band that holds 48 % of the
    cone; the row with the most rejections is period 32."""
    rs = np.random.RandomState(11)
    n = np.arange(2048)
    s = 2.5 * np.sin(2 * np.pi * n / 32.0 + np.cumsum(0.2 * rs.randn(2048)))
    x = red(rs, 2048, 0.5, 2) + s
    h = api.wct_resident(x[0], x[1], 1.0, dj=1 / 4, s0=8 / 1.033, J=16)
    h.surrogate_test(mc_count=99, seed=8)
    res = h.fdr_threshold(0.05)
    assert res.rejected > 0
    P = h.pvalues()
    cone = coi_mask(h)
    rej = cone & (P <= res.alpha)
    assert rej.sum() == res.rejected
    near = np.abs(np.log2(h.period / 32.0)) <= 1.0
    share = rej[near].sum() / rej.sum()
    assert share >= 0.75, share
    assert share > 1.5 * cone[near].sum() / cone.sum()
    assert abs(np.log2(h.period[rej.sum(axis=1).argmax()] / 32.0)) <= 0.5
