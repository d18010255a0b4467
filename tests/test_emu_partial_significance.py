"""Monte-Carlo significance of the partial and multiple wavelet coherence (`wct3_significance`,
`Engine.wct3_mc`, `Engine.wct3_mc_seeded`), checked on the host-emulation build of the kernels
(tests/_emu, the fixture pattern of test_emu_partial_coherence.py).

  * histograms of host surrogates against a composition in this file: the oracle's `cwt` of the
    unstandardised surrogates, `smooth` (or `smooth_generic` for Paul), the det G3 form of RP2 and
    RM2 and the binning rule clamp(floor(R2 nbins), 0, nbins - 1) over the points of the mask in
    rows below maxscale.  Per row sum |h - h_ref| <= 2 x (points within nbins 1e-10 / D of a bin
    edge), D the oracle's denominator of each measure (the bound of the partial-coherence tests);
  * the public call in host-RNG mode against that composition fed a replay of its draw order;
  * the seeded mode: the device triples, their independence from the pair streams, splits over
    calls, equality with the host-fed path, and agreement with the host-RNG mode within the
    Monte-Carlo scatter;
  * RM2 >= R2_y1 at every point, seen in the histograms of the same surrogates;
  * fp32 against fp64, errors, resident handles and a world size of 2 over gloo.
"""
import ctypes
import os
import socket
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import cwt_oracle as orc

TOL = 1e-10
NBINS = 1000


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


def generic(fn):
    """Run fn with the generic smoothing of Paul / DOG enabled."""
    from pycwt_b200 import mothers
    old = mothers.enable_generic_smoothing(True)
    try:
        return fn()
    finally:
        mothers.enable_generic_smoothing(old)


# ---- oracle composition ----------------------------------------------------------------------
def oracle_measures(triple, dt, dj, s0, J, mother):
    """RP2, RM2, their denominators D (as in test_emu_partial_coherence.oracle_wct3) and R2_y1 of
    one surrogate triple, NOT standardised (the Monte-Carlo null does not standardise)."""
    Ws = []
    for v in triple:
        W, sj = orc.cwt(np.asarray(v, dtype=float), dt, dj, s0, J, mother)[:2]
        Ws.append(W)
    if isinstance(mother, orc.Morlet):
        def sm(F):
            return orc.smooth(F, dt, dj, sj, mother.deltaj0)
    else:
        def sm(F):
            return orc.smooth_generic(F, dt, dj, sj, mother)
    inv = 1.0 / sj[:, None]
    Sy, S1, S2 = (sm(np.abs(W) ** 2 * inv) for W in Ws)
    Wy, W1, W2 = Ws
    Sy1, Sy2, S12 = (sm(a * b.conj() * inv) for a, b in ((Wy, W1), (Wy, W2), (W1, W2)))
    R2y1, R2y2, R212 = (np.abs(Sy1) ** 2 / (Sy * S1), np.abs(Sy2) ** 2 / (Sy * S2),
                        np.abs(S12) ** 2 / (S1 * S2))
    d12 = S1 * S2 - np.abs(S12) ** 2
    RP2 = np.abs(Sy1 * S2 - Sy2 * S12.conj()) ** 2 / ((Sy * S2 - np.abs(Sy2) ** 2) * d12)
    det = (Sy * S1 * S2 + 2 * (Sy1 * S12 * Sy2.conj()).real
           - Sy * np.abs(S12) ** 2 - S1 * np.abs(Sy2) ** 2 - S2 * np.abs(Sy1) ** 2)
    RM2 = 1 - det / (Sy * d12)
    return RP2, RM2, (1 - R2y2) * (1 - R212), 1 - R212, R2y1


def bin_rows(R, mask, maxscale, nbins=NBINS):
    """Histogram [S, nbins] of R under the binning rule; non-finite values are not counted."""
    h = np.zeros((R.shape[0], nbins), dtype=np.int64)
    for i in range(maxscale):
        v = R[i, mask[i].astype(bool)]
        v = v[np.isfinite(v)]
        h[i] = np.bincount(np.clip(np.floor(v * nbins), 0, nbins - 1).astype(np.int64), minlength=nbins)
    return h


def near_edge(R, D, mask, maxscale, nbins=NBINS):
    """Per row: masked points whose R lies within nbins TOL / D of a bin edge."""
    x = R * nbins
    edge = np.abs(x - np.round(x)) <= nbins * TOL / D
    out = np.zeros(R.shape[0], dtype=np.int64)
    for i in range(maxscale):
        out[i] = int(edge[i, mask[i].astype(bool)].sum())
    return out


def oracle_hists(noise, prob, dt, dj, s0, J, mother):
    """(hP, hM, nearP, nearM) of the triples noise[t] = (y, x1, x2)."""
    S = prob['sj'].size
    hP, hM = np.zeros((S, NBINS), np.int64), np.zeros((S, NBINS), np.int64)
    nP, nM = np.zeros(S, np.int64), np.zeros(S, np.int64)
    for tr in noise:
        rp, rm, Dp, Dm, _ = oracle_measures(tr, dt, dj, s0, J, mother)
        hP += bin_rows(rp, prob['mask'], prob['maxscale'])
        hM += bin_rows(rm, prob['mask'], prob['maxscale'])
        nP += near_edge(rp, Dp, prob['mask'], prob['maxscale'])
        nM += near_edge(rm, Dm, prob['mask'], prob['maxscale'])
    return hP, hM, nP, nM


def check_explained(h, h_ref, near, maxscale, label):
    assert h.shape == h_ref.shape
    assert h[maxscale:].sum() == 0 and h_ref[maxscale:].sum() == 0
    diff = np.abs(h - h_ref).sum(axis=1)
    print("  %s: %d points binned, %d near an edge, %d counts differ"
          % (label, h_ref.sum(), near.sum(), diff.sum()))
    assert h_ref.sum() > 0
    assert (diff <= 2 * near).all(), {i: (diff[i], near[i]) for i in range(diff.size) if diff[i] > 2 * near[i]}


# (n triples, dt, dj, s0, J, wavelet): K = round(2 deltaj0 / dj); N = ceil(6 s0 2^(J dj) / dt)
CASES = {
    "morlet K=5": (dict(dt=1.0, dj=1 / 4, s0=2.0, J=24), "morlet"),
    "morlet K=14": (dict(dt=1.0, dj=1 / 12, s0=2.0, J=60), "morlet"),
    "morlet K=77": (dict(dt=1.0, dj=1 / 64, s0=2.0, J=256), "morlet"),
    "paul4 K=12": (dict(dt=0.5, dj=1 / 4, s0=1.0, J=20), "paul"),
}
MOTHERS = {"morlet": (lambda a: a.Morlet(6), orc.Morlet(6)), "paul": (lambda a: a.Paul(4), orc.Paul(4))}


def host_triples(n, N, seed):
    rs = np.random.RandomState(seed)
    return rs.randn(n, 3, N)


def run_host(emu, prob, g, mother, noise, precision=0):
    from pycwt_b200 import wavelet as wv
    return wv._mc_histogram(prob, g["dt"], g["dj"], mother, lambda i: noise[i], range(len(noise)),
                            engine=emu, precision=precision, nser=3)


# ---- tests -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_histograms_against_oracle(api, emu, name):
    from pycwt_b200 import wavelet as wv
    g, wav = CASES[name]
    mother = MOTHERS[wav][0](api)

    def body():
        prob = wv._mc_problem(g["dt"], g["dj"], g["s0"], g["J"], mother)
        noise = host_triples(2, prob['N'], len(name))
        h = run_host(emu, prob, g, mother, noise)
        assert h.shape == (2, prob['sj'].size, NBINS) and h.dtype == np.int64
        hP, hM, nP, nM = oracle_hists(noise, prob, g["dt"], g["dj"], g["s0"], g["J"], MOTHERS[wav][1])
        check_explained(h[0], hP, nP, prob['maxscale'], name + " RP2")
        check_explained(h[1], hM, nM, prob['maxscale'], name + " RM2")
    generic(body)


def test_unpadded_odd_length(api, emu):
    """An odd surrogate length (N = 365) with the padding off: un-padded transforms and smoothing,
    in fp64 whatever precision is asked for."""
    from pycwt_b200 import helpers, wavelet as wv
    g = dict(dt=1.0, dj=1 / 4, s0=1.9, J=20)
    mother = api.Morlet(6)
    prob = wv._mc_problem(g["dt"], g["dj"], g["s0"], g["J"], mother)
    assert prob['N'] == 365
    noise = host_triples(2, prob['N'], 3)
    helpers.set_fft_padding(False)
    orc.PAD_NEXT_POW2 = False
    try:
        h64 = run_host(emu, prob, g, mother, noise, 0)
        h32 = run_host(emu, prob, g, mother, noise, 1)
        hP, hM, nP, nM = oracle_hists(noise, prob, g["dt"], g["dj"], g["s0"], g["J"], orc.Morlet(6))
    finally:
        helpers.set_fft_padding(True)
        orc.PAD_NEXT_POW2 = True
        emu.set_padding(True)
    assert np.array_equal(h64, h32)
    check_explained(h64[0], hP, nP, prob['maxscale'], "un-padded RP2")
    check_explained(h64[1], hM, nM, prob['maxscale'], "un-padded RM2")


def test_public_call_host_rng(api):
    """wct3_significance with np.random seeded equals the oracle composition fed a replay of the
    draw order: one set-up draw rednoise(N, al_y, 1), then y, x1, x2 of every triple."""
    from pycwt_b200 import wavelet as wv
    from pycwt_b200.helpers import rednoise
    al = (0.3, 0.5, 0.2)
    g = dict(dt=1.0, dj=1 / 4, s0=2.0, J=24)
    np.random.seed(2024)
    sp, sm = api.wct3_significance(*al, g["dt"], g["dj"], g["s0"], g["J"], mc_count=3, progress=False)
    prob = wv._mc_problem(g["dt"], g["dj"], g["s0"], g["J"], api.Morlet(6))
    np.random.seed(2024)
    rednoise(prob['N'], al[0], 1)
    noise = [tuple(rednoise(prob['N'], a, 1) for a in al) for _ in range(3)]
    hP, hM, nP, nM = oracle_hists(noise, prob, g["dt"], g["dj"], g["s0"], g["J"], orc.Morlet(6))
    assert nP.sum() == 0 and nM.sum() == 0          # nothing near an edge: the histograms must agree
    rp, rm = wv._mc_levels(prob, hP, 0.95), wv._mc_levels(prob, hM, 0.95)
    assert sp.shape == sm.shape == (g["J"] + 1,) and sp.dtype == sm.dtype == np.float64
    ok = np.isfinite(rp)
    assert (np.isfinite(sp) == ok).all() and (np.isfinite(sm) == ok).all() and ok.any()
    # rows without a level keep the template of wct_significance: NaN with valid points, 0 without
    assert np.array_equal(sp[~ok], prob['sig95'][~ok], equal_nan=True)
    assert np.array_equal(sm[~ok], prob['sig95'][~ok], equal_nan=True)
    assert np.abs(sp[ok] - rp[ok]).max() <= 1e-12 and np.abs(sm[ok] - rm[ok]).max() <= 1e-12
    assert ((sp[ok] > 0) & (sp[ok] < 1)).all() and ((sm[ok] > 0) & (sm[ok] < 1)).all()


def test_seeded_surrogates(emu):
    """The device triples: standard-normal white noise keyed by seed and triple number, three
    uncorrelated series, none of them a series of the pair with the same number."""
    z = emu.mc_surrogates3(7, 3, 2, 20001)                  # triples 3 and 4, odd length
    assert z.shape == (2, 3, 20001) and np.isfinite(z).all()
    flat = z.ravel()
    assert abs(flat.mean()) < 4 / np.sqrt(flat.size) and abs(flat.std() - 1) < 0.02
    assert abs(((flat[:-1] * flat[1:]).mean())) < 4 / np.sqrt(flat.size)
    assert abs((flat ** 4).mean() - 3) < 0.15 and np.abs(flat).max() < 7
    assert np.array_equal(emu.mc_surrogates3(7, 4, 1, 20001)[0], z[1])        # keyed by triple number
    assert not np.array_equal(emu.mc_surrogates3(8, 3, 1, 20001)[0], z[0])    # and by seed
    c = np.corrcoef(z[0])
    assert np.abs(c[np.triu_indices(3, 1)]).max() < 0.05
    pairs = emu.mc_surrogates(7, 3, 2, 20001)
    for t in range(2):
        for r in range(3):
            for p in range(2):
                for q in range(2):
                    assert np.abs(np.corrcoef(z[t, r], pairs[p, q])[0, 1]) < 0.05
    # the pair stream is unchanged by the triples: pairs 3 and 4 of seed 7, drawn alone
    assert np.array_equal(emu.mc_surrogates(7, 4, 1, 20001)[0], pairs[1])


def test_seeded_histograms(api, emu):
    """Splitting the triples over calls changes nothing; the seeded histograms equal those of
    wct3_mc fed the hook's surrogates; the levels agree with the host-RNG mode within the
    Monte-Carlo scatter (the bounds of test_emu_kernels.check_seeded_monte_carlo)."""
    from pycwt_b200 import wavelet as wv
    m = api.Morlet(6)
    dt, dj, s0, J = 1.0, 0.5, 2.0, 8
    prob = wv._mc_problem(dt, dj, s0, J, m)
    h_all = wv._mc_histogram_seeded(prob, dt, dj, m, 11, 0, 6, engine=emu, nser=3)
    h_split = (wv._mc_histogram_seeded(prob, dt, dj, m, 11, 0, 2, engine=emu, nser=3) +
               wv._mc_histogram_seeded(prob, dt, dj, m, 11, 2, 4, engine=emu, nser=3))
    assert h_all.shape == (2, J + 1, NBINS) and h_all[0].sum() > 0 and h_all[1].sum() > 0
    assert np.array_equal(h_all, h_split)
    noise = emu.mc_surrogates3(11, 0, 6, prob['N'])
    h_host = wv._mc_histogram(prob, dt, dj, m, lambda i: noise[i], range(6), engine=emu, nser=3)
    assert np.array_equal(h_all, h_host)
    # against the host-RNG mode (numpy stream): same distribution, different draws
    rs = np.random.RandomState(3)
    tau = int(np.ceil(-2 / np.log(0.3)))
    h_rng = wv._mc_histogram(prob, dt, dj, m, lambda i: tuple(rs.randn(prob['N'] + tau)[tau:] for _ in range(3)),
                             range(40), engine=emu, nser=3)
    h_dev = wv._mc_histogram_seeded(prob, dt, dj, m, 5, 0, 40, engine=emu, nser=3)
    for k in (0, 1):
        a, b = wv._mc_levels(prob, h_rng[k], 0.95), wv._mc_levels(prob, h_dev[k], 0.95)
        ok = np.isfinite(a)
        assert (np.isfinite(b) == ok).all()
        d = np.abs(a[ok] - b[ok])
        print("  %s: host-RNG vs seeded levels differ by %.3f (first 4 rows), %.3f (all)"
              % ("RP2" if k == 0 else "RM2", d[:4].max(), d.max()))
        assert d[:4].max() < 0.03 and d.max() < 0.15, d
    # the public seeded call: repeatable for one seed, different for another
    s1 = api.wct3_significance(0.1, 0.2, 0.3, dt, dj, s0, J, mc_count=4, progress=False, seed=5)
    s2 = api.wct3_significance(0.1, 0.2, 0.3, dt, dj, s0, J, mc_count=4, progress=False, seed=5)
    s3 = api.wct3_significance(0.1, 0.2, 0.3, dt, dj, s0, J, mc_count=4, progress=False, seed=6)
    for k in (0, 1):
        assert np.array_equal(s1[k], s2[k], equal_nan=True)
        assert not np.array_equal(s1[k], s3[k], equal_nan=True)


def test_multiple_dominates_pairwise(api, emu):
    """RM2 >= R2_y1 at every point, so over the same (y, x1) noise the cumulative counts of RM2
    are at most those of the two-series coherence at every bin, up to points where the two differ
    by less than their rounding; and the multiple level is not below the two-series level by more
    than one bin."""
    from pycwt_b200 import wavelet as wv
    g = dict(dt=1.0, dj=1 / 12, s0=2.0, J=60)
    m = api.Morlet(6)
    prob = wv._mc_problem(g["dt"], g["dj"], g["s0"], g["J"], m)
    noise = host_triples(3, prob['N'], 17)
    h3 = run_host(emu, prob, g, m, noise)
    h2 = wv._mc_histogram(prob, g["dt"], g["dj"], m, lambda i: noise[i, :2], range(3), engine=emu)
    close = np.zeros(prob['sj'].size, np.int64)
    for tr in noise:
        _, rm, _, Dm, r2y1 = oracle_measures(tr, g["dt"], g["dj"], g["s0"], g["J"], orc.Morlet(6))
        for i in range(prob['maxscale']):
            sel = prob['mask'][i].astype(bool)
            close[i] += int(((rm - r2y1)[i, sel] <= 2 * TOL / Dm[i, sel]).sum())
    ms = prob['maxscale']
    excess = (np.cumsum(h3[1], axis=1) - np.cumsum(h2, axis=1))[:ms].max(axis=1)
    assert (h3[1].sum(axis=1) == h2.sum(axis=1)).all()
    assert (excess <= close[:ms]).all(), (excess, close[:ms])
    s2, sm = wv._mc_levels(prob, h2, 0.95), wv._mc_levels(prob, h3[1], 0.95)
    ok = np.isfinite(s2)
    print("  multiple minus two-series level: min %.4f, median %.4f"
          % ((sm - s2)[ok].min(), np.median((sm - s2)[ok])))
    assert (sm[ok] >= s2[ok] - 1.0 / NBINS).all()


def test_fp32_against_fp64(api, emu):
    """Same surrogates in both precisions: equal counts per row; the levels within 2e-3, the bound
    of the two-series fp32 significance."""
    from pycwt_b200 import wavelet as wv

    def body():
        for name in ("morlet K=14", "paul4 K=12"):
            g, wav = CASES[name]
            mother = MOTHERS[wav][0](api)
            prob = wv._mc_problem(g["dt"], g["dj"], g["s0"], g["J"], mother)
            noise = host_triples(3, prob['N'], 23)
            h64 = run_host(emu, prob, g, mother, noise, 0)
            h32 = run_host(emu, prob, g, mother, noise, 1)
            for k, label in ((0, "RP2"), (1, "RM2")):
                assert h64[k].sum() > 0
                assert (h32[k].sum(axis=1) == h64[k].sum(axis=1)).all()
                s32, s64 = wv._mc_levels(prob, h32[k], 0.95), wv._mc_levels(prob, h64[k], 0.95)
                ok = np.isfinite(s64)
                assert (np.isfinite(s32) == ok).all() and ok.any()
                d = np.abs(s32[ok] - s64[ok]).max()
                moved = int(np.abs(h32[k] - h64[k]).sum()) // 2
                print("  %s %s fp32 vs fp64: %d of %d points change bin, levels within %.1e"
                      % (name, label, moved, int(h64[k].sum()), d))
                assert d <= 2e-3
    generic(body)


def test_errors(api, emu):
    from pycwt_b200 import mothers, _engine
    args = (0.1, 0.2, 0.3, 1.0, 0.5, 2.0, 8)
    old = mothers.enable_generic_smoothing(False)
    try:
        for mo in (api.Paul(4), api.DOG(2)):
            with pytest.raises(AttributeError):
                api.wct3_significance(*args, wavelet=mo, mc_count=1, progress=False)
    finally:
        mothers.enable_generic_smoothing(old)
    with pytest.raises(ValueError):
        api.wct3_significance(*args, wavelet=api.Morlet(8), mc_count=1, progress=False)   # deltaj0 = -1
    with pytest.raises(ValueError):
        api.wct3_significance(*args, precision="fp16", mc_count=1, progress=False)

    class Duck(object):
        def __init__(self):
            self._m = api.Morlet(6)

        def __getattr__(self, name):
            if name == '_engine_spec':
                raise AttributeError(name)
            return getattr(self._m, name)
    with pytest.raises(NotImplementedError):
        api.wct3_significance(*args, wavelet=Duck(), mc_count=1, progress=False)
    import inspect
    assert "cache" not in inspect.signature(api.wct3_significance).parameters
    # Engine argument checks
    S, n0 = 9, 64
    sj = 2.0 * 2 ** (np.arange(S) / 2)
    mask = np.ones((S, n0), np.uint8)
    h = np.zeros((S, NBINS), np.int64)
    noise = np.random.RandomState(0).randn(1, 3, n0)
    with pytest.raises(ValueError):
        emu.wct3_mc(noise, 1.0, sj, 0, 6.0, 3, mask, 4, NBINS, None, None)
    with pytest.raises(ValueError):
        emu.wct3_mc(noise[:, :2], 1.0, sj, 0, 6.0, 3, mask, 4, NBINS, h, None)
    with pytest.raises(ValueError):
        emu.wct3_mc(noise, 1.0, sj, 0, 6.0, 3, mask[:, 1:], 4, NBINS, h, None)
    with pytest.raises(ValueError):
        emu.wct3_mc(noise, 1.0, sj, 0, 6.0, 3, mask, 4, NBINS, h.astype(np.int32), None)
    with pytest.raises(ValueError):
        emu.wct3_mc_seeded(1, 0, 1, n0, 1.0, sj, 0, 6.0, 3, mask, 4, NBINS, None, None)
    for ms in (-1, S + 1):
        with pytest.raises(_engine.EngineError, match="bad argument"):
            emu.wct3_mc(noise, 1.0, sj, 0, 6.0, 3, mask, ms, NBINS, h, h.copy())
    with pytest.raises(_engine.EngineError, match="analytic"):
        emu.wct3_mc_seeded(1, 0, 1, n0, 1.0, sj, _engine.TABLE, 6.0, 3, mask, 4, NBINS, h, None)
    # the C ABI: CWTB_ERR_ARG (-1) for null surrogates, no histogram, or nbins < 1
    P = ctypes.c_void_p
    mk = mask.ctypes.data_as(P)
    hp = h.ctypes.data_as(P)
    assert emu.lib.cwtb_wct3_mc(emu.h, None, 1, n0, 1.0, sj.ctypes.data_as(P), S, 0, 6.0, 3, mk, 4, NBINS,
                                hp, None) == -1
    assert emu.lib.cwtb_wct3_mc(emu.h, noise.ctypes.data_as(P), 1, n0, 1.0, sj.ctypes.data_as(P), S, 0, 6.0, 3,
                                mk, 4, NBINS, None, None) == -1
    assert emu.lib.cwtb_wct3_mc_seeded(emu.h, 1, 0, 1, n0, 1.0, sj.ctypes.data_as(P), S, 0, 6.0, 3, mk, 4, 0,
                                       hp, None) == -1
    assert emu.lib.cwtb_mc_surrogates3(emu.h, 1, 0, 0, n0, noise.ctypes.data_as(P)) == -1
    assert h.sum() == 0
    # one histogram only: the other measure is neither needed nor touched
    hp1, hm1 = np.zeros_like(h), np.zeros_like(h)
    emu.wct3_mc(noise, 1.0, sj, 0, 6.0, 3, mask, 5, NBINS, hp1, hm1)
    only_p, only_m = np.zeros_like(h), np.zeros_like(h)
    emu.wct3_mc(noise, 1.0, sj, 0, 6.0, 3, mask, 5, NBINS, only_p, None)
    emu.wct3_mc(noise, 1.0, sj, 0, 6.0, 3, mask, 5, NBINS, None, only_m)
    assert np.array_equal(only_p, hp1) and np.array_equal(only_m, hm1) and hp1[:5].sum() == 5 * n0
    # accumulated into, not cleared
    emu.wct3_mc(noise, 1.0, sj, 0, 6.0, 3, mask, 5, NBINS, only_p, None)
    assert np.array_equal(only_p, 2 * hp1)


def test_resident_handles_survive(api, emu):
    from pycwt_b200 import _engine
    rs = np.random.RandomState(9)
    y, x1 = rs.randn(1024), rs.randn(1024)
    kw = dict(dj=1 / 4, s0=2.0, J=30)
    hc = api.wct_resident(y, x1, 1.0, **kw)
    hx = api.xwt_resident(y, x1, 1.0, **kw)
    WCT, aWCT, W12 = hc.coherence(), hc.phase(), hx.cross_spectrum()
    cs, xs = emu.coherence_serial(), emu.cross_serial()
    for p in ("fp64", "fp32"):
        api.wct3_significance(0.1, 0.2, 0.3, 1.0, 0.5, 2.0, 8, mc_count=2, progress=False, precision=p)
        api.wct3_significance(0.1, 0.2, 0.3, 1.0, 1 / 64, 2.0, 200, mc_count=1, progress=False, seed=3,
                              precision=p)                                          # K = 77
    assert emu.coherence_serial() == cs and emu.cross_serial() == xs
    assert np.array_equal(hc.coherence(), WCT) and np.array_equal(hc.phase(), aWCT)
    assert np.array_equal(hx.cross_spectrum(), W12)
    out = np.empty(2 * 1024, dtype=np.complex128)
    assert emu.lib.cwtb_field_get(emu.h, _engine.FIELD_W, 0, 1, out.ctypes.data_as(ctypes.c_void_p)) == -4
    hc.release()
    hx.release()


# ---- multi-rank ------------------------------------------------------------------------------
SHARD_ARGS = (0.2, 0.1, 0.4, 1.0, 0.5, 2.0, 8, 0.95, 'morlet')


def _mc3_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    from pycwt_b200 import distributed as D, _engine
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        eng = _engine.Engine(0, lib_path=os.path.join(ROOT, "tests", "_emu", "libcwtb200_emu.so"))
        sig = [D.wct3_significance_sharded(*SHARD_ARGS, mc_count=5, seed=42, engine=eng, comm=D.TorchComm(dist),
                                           device_rng=rng) for rng in (False, True)]
        q.put((rank, [[s.tolist() for s in pm] for pm in sig]))
        eng.close()
    finally:
        dist.destroy_process_group()


def test_sharded_significance_gloo():
    """World size 2 gives the levels of one process running every triple, in both RNG modes."""
    pytest.importorskip("torch")
    import torch.multiprocessing as mp
    from pycwt_b200 import build as _build, _engine, distributed as D
    eng = _engine.Engine(0, lib_path=_build.build_emulation(os.path.join(ROOT, "tests", "_emu")))
    single = [D.wct3_significance_sharded(*SHARD_ARGS, mc_count=5, seed=42, engine=eng, device_rng=rng)
              for rng in (False, True)]
    # the two-coefficient surrogate pair is what it was: the first two series of the triple stream
    p = D.surrogate_pair(42, 3, 100, 0.2, 0.1)
    t = D.surrogate_pair(42, 3, 100, 0.2, 0.1, 0.4)
    assert len(p) == 2 and len(t) == 3 and np.array_equal(p[0], t[0]) and np.array_equal(p[1], t[1])
    eng.close()
    for pm in single:
        for s in pm:
            assert np.isnan(s).any() and np.isfinite(s).any()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_mc3_worker, args=(r, 2, port, q)) for r in range(2)]
    for pr in procs:
        pr.start()
    got = [q.get(timeout=300) for _ in procs]
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    for _, sig in got:
        for k in (0, 1):
            for m in (0, 1):
                assert np.array_equal(np.array(sig[k][m]), single[k][m], equal_nan=True)
