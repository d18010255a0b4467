"""Tests of the reconstruction over a selection (`ResidentPower.reconstruct`,
`ResidentTransform.reconstruct` and the engine calls `field_reconstruct`, `power_pvalue_reconstruct`,
`power_cluster_reconstruct`), checked on the host-emulation build of the kernels (tests/_emu):

  * every mode and combination of band, cone, signif, alpha and a set of clusters equals a longdouble
    restatement from the fetched W and the masks of `period`, `coi_ranges`, `power`, `pvalues` and
    `cluster_labels`, within a bound that covers the summation only;
  * bands that partition the scales, and single clusters, add up to the whole;
  * with everything selected it agrees with `icwt()`;
  * repeated calls are bit-identical and move nothing resident;
  * inputs scaled by 2^k give 2^k times the reconstruction, bit for bit;
  * lifetime and errors, at the Python and the C level;
  * two tones: the band around one gives it back.
"""
import ctypes

import numpy as np
import pytest

import test_emu_power_test as PT
from test_emu_power_test import padding  # noqa: F401  (fixture)
from test_emu_surrogate_significance import emu, api, red  # noqa: F401  (fixtures)

EPS = np.finfo(float).eps
ERR_ARG, ERR_STATE, ERR_UNSUPPORTED = -1, -4, -5
POWER_RANGE = {'fp64': 450, 'fp32': 48}    # |k| of a degree-2 product (test_emu_amplitude's table)


# ---- the restatement ------------------------------------------------------------------------------
def _selection(h, mode, r0, r1, W):
    """bool [r1 - r0, n0]: the points of rows r0 .. r1 - 1 that `mode` selects."""
    S, n0 = h.shape
    sel = np.repeat(h._band(mode.get('period_min', -np.inf), mode.get('period_max', np.inf))[r0:r1, None],
                    n0, axis=1)
    if mode.get('inside_coi'):
        lo, hi = h.coi_ranges()
        cols = np.arange(n0)[None]
        sel &= (cols >= lo[r0:r1, None]) & (cols < hi[r0:r1, None])
    P = W.real * W.real + W.imag * W.imag           # the device's P (test_emu_power_test.test_readers)
    if mode.get('signif') is not None:
        sel &= P > np.asarray(mode['signif'], dtype=float)[r0:r1, None]
    if mode.get('alpha') is not None:
        sel &= h.pvalues(slice(r0, r1)) <= mode['alpha']       # NaN where P is not finite: not selected
    if mode.get('cluster') is not None:
        rows = np.atleast_1d(np.asarray(mode['cluster'], dtype=np.int64))
        sel &= np.isin(h.cluster_labels(slice(r0, r1)), rows + 1)
    return sel


def restate(h, modes, block=None):
    """[(ref, bound)] per mode: fac * sum over the selected points of Re W / sqrt(s_j) in longdouble,
    and 2 (S_sel + 2) eps |fac| sum |Re W| / sqrt(s_j) per column.  W is read in row blocks."""
    S, n0 = h.shape
    block = block or S
    fac = h.dj * np.sqrt(h.dt) / (h.wavelet.cdelta * h.wavelet.psi(0))
    rs = 1.0 / np.sqrt(np.asarray(h.scales, dtype=float))
    acc = [[np.zeros(n0, dtype=np.longdouble), np.zeros(n0, dtype=np.longdouble), np.zeros(n0)] for _ in modes]
    for r0 in range(0, S, block):
        r1 = min(S, r0 + block)
        W = h.window(slice(r0, r1), slice(None))
        term = rs[r0:r1, None].astype(np.longdouble) * W.real.astype(np.longdouble)
        for a, mode in zip(acc, modes):
            sel = _selection(h, mode, r0, r1, W)
            a[0] += np.where(sel, term, 0).sum(axis=0)
            a[1] += np.where(sel, np.abs(term), 0).sum(axis=0)
            a[2] += sel.sum(axis=0)
    return [(fac * s, 2 * (cnt + 2) * EPS * abs(fac) * ab.astype(float)) for s, ab, cnt in acc]


def check(x, ref, bound, what):
    assert x.shape == ref.shape, what
    for part in ((np.real,) if not np.iscomplexobj(ref) else (np.real, np.imag)):
        err = np.abs(part(x).astype(np.longdouble) - part(ref)).astype(float)
        bad = err > bound
        assert not bad.any(), (what, int(bad.sum()), float(err.max()), np.argwhere(bad)[:3].tolist())


def modes_of(h, cluster_rows=None):
    """Every combination of band, cone, signif and alpha, and the cluster sets."""
    P = h.power()
    per = h.period
    band = (float(per[len(per) // 3]), float(per[2 * len(per) // 3]))
    sig = np.quantile(P, 0.6, axis=1)
    sig[1] = np.nan                                  # a NaN entry selects none of its scale
    out = []
    for b in ((-np.inf, np.inf), band):
        for inside in (False, True):
            for signif in (None, sig):
                for alpha in ((None, 0.5) if hasattr(h, 'pvalues') else (None,)):
                    m = dict(period_min=b[0], period_max=b[1], inside_coi=inside, signif=signif)
                    out.append(m if alpha is None else dict(m, alpha=alpha))
    for rows in cluster_rows or ():
        for inside in (False, True):
            out.append(dict(inside_coi=inside, cluster=rows))
    return out


def power_with_tests(api, null, prec, wav, n0, padded, normalize=True):
    """A resident power with counts and clusters, and the cluster sets of its table."""
    h = PT.resident(api, null, prec, wav, n0, padded, normalize=normalize)
    h.surrogate_test(mc_count=9, seed=11, null=null)
    res = h.cluster_test(np.quantile(h.power(), 0.7, axis=1), mc_count=4, seed=12, null=null)
    nc = len(res.area)
    sets = [[], 0] + ([[0, nc - 1, 0], list(range(nc))] if nc else [])
    return h, sets


# ---- 1. definition --------------------------------------------------------------------------------
@pytest.mark.parametrize("null,prec,wav,n0,padded", PT.CASES)
def test_definition(api, emu, padding, null, prec, wav, n0, padded):
    h, sets = power_with_tests(api, null, prec, wav, n0, padded)
    modes = modes_of(h, sets)
    for mode, (ref, bound) in zip(modes, restate(h, modes)):
        x = h.reconstruct(**mode)
        assert x.dtype == (np.float64 if wav == 'dog' else np.complex128)
        check(x, ref, bound, mode)
    # the transform's own W
    ht = api.cwt_resident(h._yn, 1.0, wavelet=PT.WAVELETS[wav](api), **PT.KW)
    modes = modes_of(ht)
    for mode, (ref, bound) in zip(modes, restate(ht, modes)):
        check(ht.reconstruct(**mode), ref, bound, ('transform', mode))


# ---- 2. additivity --------------------------------------------------------------------------------
@pytest.mark.parametrize("null,prec,wav,n0,padded", PT.CASES[:4])
def test_additivity(api, emu, padding, null, prec, wav, n0, padded):
    h, sets = power_with_tests(api, null, prec, wav, n0, padded)
    per = h.period
    edges = [-np.inf, float(per[len(per) // 4]), float(per[len(per) // 2]), np.inf]
    (ref, bound), = restate(h, [dict(inside_coi=True)])
    whole = h.reconstruct(inside_coi=True)
    parts = [h.reconstruct(a, b, inside_coi=True) for a, b in zip(edges[:-1], edges[1:])]
    check(sum(parts), ref, 2 * bound, 'bands')
    check(whole, ref, bound, 'whole')
    nc = len(h.engine.cluster_table(PT.POWER)[0])
    if nc:
        rows = list(range(nc))
        (ref, bound), = restate(h, [dict(cluster=rows)])
        check(sum(h.reconstruct(cluster=c) for c in rows), ref, 2 * bound, 'clusters')


# ---- 3. full selection against icwt() ---------------------------------------------------------------
@pytest.mark.parametrize("null,prec,wav,n0,padded", PT.CASES)
def test_full_selection_is_icwt(api, emu, padding, monkeypatch, null, prec, wav, n0, padded):
    h = PT.resident(api, null, prec, wav, n0, padded)
    x = h.reconstruct()
    (ref, bound), = restate(h, [{}])
    # the same series through cwt_resident in the power's precision
    monkeypatch.setenv('CWTB_PRECISION', prec)
    ht = api.cwt_resident(h._yn, 1.0, wavelet=PT.WAVELETS[wav](api), **PT.KW)
    assert ht.wave().tobytes() == h.wave().tobytes()
    check(ht.icwt(), ref, bound, 'icwt')
    check(x, ht.icwt(), 2 * bound, 'power against icwt')
    check(ht.reconstruct(), ht.icwt(), 2 * bound, 'transform against icwt')


# ---- 4. stability ---------------------------------------------------------------------------------
def test_repeated_calls_move_nothing(api, emu):
    x = PT.series(512, seed=4)
    y = PT.series(512, seed=5)
    hc = api.wct_resident(x, y, 1.0, **PT.KW)
    hx = api.xwt_resident(x, y, 1.0, **PT.KW)
    h, sets = power_with_tests(api, 'phase', 'fp64', 'morlet', 512, True)
    state = lambda: [hc.coherence().tobytes(), hx.cross_spectrum().tobytes(), h.wave().tobytes(),  # noqa: E731
                     h.pvalues().tobytes(), h.cluster_labels().tobytes()]
    before = state()
    modes = modes_of(h, sets)
    first = [h.reconstruct(**m).tobytes() for m in modes]
    assert [h.reconstruct(**m).tobytes() for m in modes] == first
    assert state() == before


# ---- 5. powers of two -----------------------------------------------------------------------------
@pytest.mark.parametrize("prec,wav", [('fp64', 'morlet'), ('fp32', 'paul'), ('fp64', 'dog')])
def test_powers_of_two(api, emu, prec, wav):
    y = PT.series(300, seed=6)
    sig = None

    def run(k):
        h = api.power_resident(np.ldexp(y, k), 1.0, wavelet=PT.WAVELETS[wav](api), precision=prec,
                               normalize=False, **PT.KW)
        s = np.ldexp(sig, 2 * k)
        h.surrogate_test(mc_count=5, seed=3, null='phase')
        res = h.cluster_test(s, mc_count=3, seed=4, null='phase')
        rows = list(range(len(res.area)))
        return [h.reconstruct(), h.reconstruct(2.0, 20.0, inside_coi=True), h.reconstruct(signif=s),
                h.reconstruct(alpha=0.5), h.reconstruct(signif=s, alpha=0.5, inside_coi=True),
                h.reconstruct(cluster=rows)], rows

    h0 = api.power_resident(y, 1.0, wavelet=PT.WAVELETS[wav](api), precision=prec, normalize=False, **PT.KW)
    sig = np.quantile(h0.power(), 0.7, axis=1)
    ref, rows = run(0)
    assert rows
    K = POWER_RANGE[prec]
    for k in (K, -K, 7):
        got, rows_k = run(k)
        assert rows_k == rows
        for i, (g, r) in enumerate(zip(got, ref)):
            want = np.ldexp(r.real, k) + 1j * np.ldexp(r.imag, k) if np.iscomplexobj(r) else np.ldexp(r, k)
            assert np.array_equal(g, want), (k, i)


# ---- 6. lifetime and errors -----------------------------------------------------------------------
def test_errors_python(api, emu, padding):
    from pycwt_b200._engine import EngineError
    x = PT.series(256)
    h = api.power_resident(x, 1.0, **PT.KW)
    with pytest.raises(EngineError, match="surrogate test"):
        h.reconstruct(alpha=0.5)
    with pytest.raises(EngineError, match="cluster test"):
        h.reconstruct(cluster=0)
    with pytest.raises(ValueError, match="no scale"):
        h.reconstruct(1e6, 2e6)
    with pytest.raises(ValueError, match="signif"):
        h.reconstruct(signif=np.ones(3))
    with pytest.raises(ValueError, match="negative"):
        h.reconstruct(signif=-np.ones(len(h.scales)))
    h.surrogate_test(mc_count=3, seed=1)
    with pytest.raises(ValueError, match="alpha"):
        h.reconstruct(alpha=0.0)
    res = h.cluster_test(np.quantile(h.power(), 0.7, axis=1), mc_count=2, seed=1)
    nc = len(res.area)
    for bad in (dict(cluster=0, signif=np.ones(len(h.scales))), dict(cluster=0, alpha=0.5)):
        with pytest.raises(ValueError, match="no signif or alpha"):
            h.reconstruct(**bad)
    for bad in (nc, -1, [0, nc], 1.5, True, [[0]]):
        with pytest.raises(ValueError, match="cluster"):
            h.reconstruct(cluster=bad)
    assert not h.reconstruct(cluster=[]).any()
    # a wavelet without Cdelta
    hp = api.cwt_resident(x, 1.0, wavelet=api.Paul(5), **PT.KW)
    assert hp.wavelet.cdelta == -1
    with pytest.raises(ValueError, match="Cdelta"):
        hp.reconstruct()
    # superseded and released handles
    ht = api.cwt_resident(x, 1.0, **PT.KW)
    api.cwt(x, 1.0, **PT.KW)
    with pytest.raises(EngineError, match="no longer resident"):
        ht.reconstruct()
    h2 = api.power_resident(x, 1.0, **PT.KW)
    with pytest.raises(EngineError, match="no longer resident"):
        h.reconstruct()
    h2.release()
    with pytest.raises(EngineError, match="no longer resident"):
        h2.reconstruct()


def test_errors_c(api, emu):
    from pycwt_b200 import _engine
    lib, c = emu.lib, emu.h
    x = PT.series(256)
    h = api.power_resident(x, 1.0, **PT.KW)
    S, n0 = h.shape
    w = np.ones(S)
    lo, hi = np.zeros(S, dtype=np.int64), np.full(S, n0, dtype=np.int64)
    out = np.empty(n0)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def field(fid, lo=lo, hi=hi, w=w, out=out, thr=None):
        return lib.cwtb_field_reconstruct(c, fid, None if w is None else P(w), None if lo is None else P(lo),
                                          None if hi is None else P(hi), thr, None if out is None else P(out))

    assert field(_engine.FIELD_POWER) == 0
    assert field(_engine.FIELD_W) == ERR_STATE             # no transform resident after power_resident
    assert field(_engine.FIELD_CROSS) == ERR_ARG
    assert field(4) == ERR_ARG
    for kw in (dict(w=None), dict(lo=None), dict(hi=None), dict(out=None)):
        assert field(_engine.FIELD_POWER, **kw) == ERR_ARG
    bad_lo = lo.copy()
    bad_lo[2] = 5
    bad_hi = hi.copy()
    bad_hi[2] = 4
    assert field(_engine.FIELD_POWER, lo=bad_lo, hi=bad_hi) == ERR_ARG      # lo > hi
    assert field(_engine.FIELD_POWER, hi=hi + 1) == ERR_ARG                 # hi > n0
    assert field(_engine.FIELD_POWER, lo=lo - 1) == ERR_ARG
    assert lib.cwtb_power_pvalue_reconstruct(c, P(w), P(lo), P(hi), None, 3, P(out)) == ERR_STATE
    cl = np.zeros(1, dtype=np.int64)
    assert lib.cwtb_power_cluster_reconstruct(c, P(w), P(lo), P(hi), P(cl), 1, P(out)) == ERR_STATE
    h.surrogate_test(mc_count=3, seed=1)
    assert lib.cwtb_power_pvalue_reconstruct(c, P(w), P(lo), P(hi), None, 3, P(out)) == 0
    assert lib.cwtb_power_pvalue_reconstruct(c, None, P(lo), P(hi), None, 3, P(out)) == ERR_ARG
    res = h.cluster_test(np.quantile(h.power(), 0.7, axis=1), mc_count=2, seed=1)
    nc = len(res.area)
    assert nc > 0
    assert lib.cwtb_power_cluster_reconstruct(c, P(w), P(lo), P(hi), P(cl), 1, P(out)) == 0
    for bad in (nc, -1):
        b = np.array([0, bad], dtype=np.int64)
        assert lib.cwtb_power_cluster_reconstruct(c, P(w), P(lo), P(hi), P(b), 2, P(out)) == ERR_ARG
    assert lib.cwtb_power_cluster_reconstruct(c, P(w), P(lo), P(hi), None, 1, P(out)) == ERR_ARG
    assert lib.cwtb_power_cluster_reconstruct(c, P(w), P(lo), P(hi), P(cl), -1, P(out)) == ERR_ARG
    assert lib.cwtb_power_cluster_reconstruct(c, P(w), P(lo), P(hi), None, 0, P(out)) == 0
    assert not out.any()
    # the W of a batched transform
    sj = np.asarray(h.scales, dtype=float)
    emu.cwt_batch(np.stack([x, x]), 1.0, sj, *h.wavelet._engine_spec())
    assert field(_engine.FIELD_W) == ERR_UNSUPPORTED
    h.release()
    assert field(_engine.FIELD_POWER) == ERR_STATE
    assert lib.cwtb_power_pvalue_reconstruct(c, P(w), P(lo), P(hi), None, 3, P(out)) == ERR_STATE


# ---- 7. filtering ---------------------------------------------------------------------------------
def test_band_gives_back_its_tone(api, emu):
    n0 = 2048
    t = np.arange(n0)
    fast, slow = np.sin(2 * np.pi * t / 8), 1.5 * np.sin(2 * np.pi * t / 64 + 0.3)
    ht = api.cwt_resident(fast + slow, 1.0, dj=1 / 12, s0=2.0)
    x = ht.reconstruct(5.0, 13.0)
    assert x.dtype == np.complex128
    lo, hi = ht.coi_ranges()
    sel = ht._band(5.0, 13.0)
    inside = slice(int(lo[sel].max()), int(hi[sel].min()))     # outside the cone of every row of the band
    err = x.real[inside] - fast[inside]
    rms = float(np.sqrt(np.mean(err ** 2)) / np.sqrt(np.mean(fast[inside] ** 2)))
    assert rms < 0.03, rms     # 0.0230 on this series: TC98 report a few per cent for eq. 29
    # the power's W of the same series, normalize=False, is the same W
    hp = api.power_resident(fast + slow, 1.0, dj=1 / 12, s0=2.0, normalize=False)
    assert np.array_equal(hp.reconstruct(5.0, 13.0), x)



# ---- a burst in red noise, found and given back ---------------------------------------------------
def burst_case(api):
    """An AR(1) series (g = 0.7, n0 = 4096) with a Hann-windowed period-32 burst of amplitude 4 over
    samples [2000, 2400): the clusters at p <= 0.05 of `cluster_test` at the 95 % chi-squared level of
    `significance()` with M = 199, reconstructed in data units.  Returns (rows, correlation with the
    burst over its span widened by two periods, rms outside that span over rms inside)."""
    rs = np.random.RandomState(12)
    n = np.arange(4096)
    win = np.where((n >= 2000) & (n < 2400), np.sin(np.pi * (n - 2000) / 400.0) ** 2, 0.0)
    burst = 4.0 * win * np.sin(2 * np.pi * n / 32.0)
    x = red(rs, 4096, 0.7)[0] + burst
    h = api.power_resident(x, 1.0, dj=1 / 4, s0=2.0, J=24)
    sig = api.significance(1.0, h.dt, h.scales, 0, api.ar1(x)[0])[0]
    res = h.cluster_test(sig, mc_count=199, seed=9)
    rows = np.flatnonzero(res.pvalue <= 0.05)
    rec = h.reconstruct(cluster=rows).real * x.std()
    span = (n >= 1936) & (n < 2464)
    corr = float(np.corrcoef(rec[span], burst[span])[0, 1])
    outside = float(np.sqrt(np.mean(rec[~span] ** 2)) / np.sqrt(np.mean(rec[span] ** 2)))
    return rows, corr, outside


def test_burst_given_back(api, emu):
    rows, corr, outside = burst_case(api)
    print("  burst: clusters %s at p <= 0.05, correlation %.4f, rms outside / inside %.4f"
          % (rows.tolist(), corr, outside))
    assert rows.size >= 1
    # this run: one cluster (rows [13, 18), columns [2069, 2337)) at p = 0.02, correlation 0.9649, nothing
    # outside the span (the device computes the same numbers)
    assert corr >= 0.95 and outside <= 0.01
