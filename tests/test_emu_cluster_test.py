"""Cluster tests of the resident coherence against phase-randomised surrogates (`cluster_test`,
`cluster_labels`, and the engine calls `cluster_test`, `cluster_table`, `cluster_labels` and the
hook `cluster_label_bits`), checked on the host-emulation build of the kernels (tests/_emu):

  * the labeller equals scipy.ndimage.label with 8-connectivity up to renumbering, on masks no
    coherence map produces, with Q, point counts and boxes equal to integer sums on the host and
    the table in its contract order;
  * every unit's largest cluster sum equals a recount of the hook's surrogates through engine-level
    `wct` / `wct3`, thresholded on the host and labelled by SciPy, and the observed table and labels
    equal the same recount of the resident field, with the K > 32 boxcar, padded, 2^k and
    un-padded lengths;
  * nothing else moves: the fields, the counts of an earlier `surrogate_test`, the histograms;
  * lifetime and errors.
"""
import numpy as np
import pytest
from scipy import ndimage

import test_emu_surrogate_pvalues as P
import test_emu_surrogate_significance as T
from test_emu_surrogate_significance import emu, api, red  # noqa: F401  (fixtures)

F64, F32 = T.F64, T.F32
NBINS = T.NBINS
MORLET = T.MORLET
ERR_ARG, ERR_STATE, ERR_UNSUPPORTED = -1, -4, -5


# ---- host restatement of the contract ------------------------------------------------------------
def pack(sel):
    """bool [S, n0] -> uint32 [S, ceil(n0 / 32)], column n at bit n % 32 of word n / 32."""
    S, n0 = sel.shape
    words = (n0 + 31) // 32
    pad = np.zeros((S, words * 32), dtype=np.uint64)
    pad[:, :n0] = sel
    return (pad.reshape(S, words, 32) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)


def weights(sj):
    smin = np.min(sj)
    return np.floor(2.0 ** 32 * smin / np.asarray(sj, dtype=float) + 0.5).astype(np.uint64)


def reference(sel, q):
    """(Q, points, box [:, 4], labels) of the contract: SciPy's 8-connected labels renumbered in
    table order (Q descending, ties by the row-major index of the first point), integer sums."""
    lab, n = ndimage.label(sel, structure=np.ones((3, 3)))
    S, n0 = sel.shape
    Q = np.zeros(n + 1, dtype=np.uint64)
    for j in range(S):
        Q += np.bincount(lab[j], minlength=n + 1).astype(np.uint64) * np.uint64(q[j])
    pts = np.bincount(lab.ravel(), minlength=n + 1)[1:]
    box = np.array([[r.start, r.stop, c.start, c.stop] for r, c in ndimage.find_objects(lab)],
                   dtype=np.int64).reshape(n, 4)
    first = box[:, 0] * n0 + _first_cols(lab, box, n)     # the first point lies in the first row
    order = np.lexsort((first, ~Q[1:]))
    rank = np.zeros(n + 1, dtype=np.int32)
    rank[1 + order] = np.arange(1, n + 1)
    return Q[1:][order], pts[order], box[order], rank[lab]


def _first_cols(lab, box, n):
    """Per cluster, the first column of its points in its first row."""
    out = np.full(n, lab.shape[1], dtype=np.int64)
    for j in np.unique(box[:, 0]):
        row = lab[j]
        c = np.flatnonzero(row)
        cl = row[c] - 1
        starts = box[cl, 0] == j
        np.minimum.at(out, cl[starts], c[starts])
    return out


def check_hook(eng, sel, q=None):
    sel = np.asarray(sel, dtype=bool)
    S, n0 = sel.shape
    if q is None:
        q = weights(2.0 * 2 ** (np.arange(S) / 4.0))
    Q, pts, box, labels, qmax = eng.cluster_label_bits(pack(sel), n0, q)
    rQ, rpts, rbox, rlab = reference(sel, q)
    assert np.array_equal(labels, rlab)
    assert np.array_equal(Q, rQ) and np.array_equal(pts, rpts) and np.array_equal(box, rbox)
    assert qmax == (int(rQ[0]) if rQ.size else 0)
    return Q


def masks():
    rs = np.random.RandomState(17)
    out = []
    for d in (0.05, 0.3, 0.41, 0.7):
        out.append(('random%.2f' % d, rs.rand(37, 301) < d))
    out.append(('ones', np.ones((9, 100), dtype=bool)))
    alt = np.zeros((12, 256), dtype=bool)
    alt[:, ::2] = True
    out.append(('alternating', alt))
    alt2 = np.zeros((12, 257), dtype=bool)   # checkerboard: every run touches the next row's two
    alt2[::2, ::2] = True
    alt2[1::2, 1::2] = True
    out.append(('checkerboard', alt2))
    ser = np.zeros((15, 70), dtype=bool)     # a serpentine through every row
    ser[::2, 1:69] = True
    ser[1::4, 68] = True
    ser[3::4, 1] = True
    out.append(('serpentine', ser))
    cor = np.zeros((6, 45), dtype=bool)
    cor[0, 0] = cor[0, 44] = cor[5, 0] = cor[5, 44] = True
    out.append(('corners', cor))
    out.append(('n0<32', rs.rand(5, 13) < 0.5))
    out.append(('S=1', rs.rand(1, 200) < 0.5))
    out.append(('one point', np.ones((1, 1), dtype=bool)))
    out.append(('empty', np.zeros((4, 40), dtype=bool)))
    wrap = np.zeros((3, 64), dtype=bool)     # column 0 and column n0 - 1 are not neighbours
    wrap[1, 0] = wrap[0, 63] = wrap[2, 63] = True
    out.append(('no wrap', wrap))
    return out


@pytest.mark.parametrize("name,sel", masks(), ids=[m[0] for m in masks()])
def test_labeller_matches_scipy(emu, name, sel):
    check_hook(emu, sel)


def test_labeller_ties_and_weights(emu):
    """Equal Q: ordered by the first point; unequal weights per row decide the order."""
    sel = np.zeros((4, 40), dtype=bool)
    sel[0, 30:33] = sel[2, 1:4] = sel[3, 20] = sel[1, 10] = True
    Q = check_hook(emu, sel, np.array([1, 1, 1, 3], dtype=np.uint64))
    assert list(Q) == [3, 3, 3, 1]
    check_hook(emu, np.ones((3, 50), dtype=bool), np.full(3, 2 ** 32, dtype=np.uint64))


def test_labeller_rejects(emu):
    from pycwt_b200._engine import EngineError
    import ctypes
    # n_scales * n0 >= 2^32 is refused before anything is read or allocated
    c = ctypes.c_int64()
    for S, n0 in ((2, 2 ** 31), (65536, 65536), (1, 2 ** 32)):
        assert emu.lib.cwtb_cluster_label_bits(emu.h, None, S, n0, None, 0, ctypes.byref(c), None, None, None,
                                               None, None) == ERR_UNSUPPORTED
    bits = pack(np.ones((2, 40), dtype=bool))
    bits[1, 1] |= np.uint32(1 << 9)          # a bit past column 39
    with pytest.raises(EngineError, match="past the last column"):
        emu.cluster_label_bits(bits, 40, np.ones(2, dtype=np.uint64))
    for bad in (pack(np.ones((2, 40), dtype=bool))[:, :1], np.ones((2, 3), dtype=np.uint32), np.ones(4, np.uint32)):
        with pytest.raises(ValueError, match="ceil"):     # the hook reads exactly S x ceil(n0 / 32) words
            emu.cluster_label_bits(bad, 40, np.ones(2, dtype=np.uint64))
    with pytest.raises(ValueError, match="q must"):
        emu.cluster_label_bits(pack(np.ones((2, 40), dtype=bool)), 40, np.ones(3, dtype=np.uint64))
    with pytest.raises(EngineError, match="2\\^32"):
        emu.cluster_label_bits(pack(np.ones((2, 40), dtype=bool)), 40, np.full(2, 2 ** 32 + 1, dtype=np.uint64))


# ---- the units against a recount ----------------------------------------------------------------
def select(R, thr, lo, hi):
    n = np.arange(R.shape[1])
    with np.errstate(invalid='ignore'):
        return np.isfinite(R) & (R > thr[:, None]) & (n >= lo[:, None]) & (n < hi[:, None])


def row_args(S, n0, obs):
    """A threshold per row (one NaN row) and column ranges of several shapes."""
    thr = np.nanquantile(np.where(np.isfinite(obs), obs, np.nan), 0.2, axis=1)
    thr[3] = np.nan
    lo = np.zeros(S, dtype=np.int64)
    hi = np.full(S, n0, dtype=np.int64)
    lo[5:9] = n0 // 8
    hi[5:9] = n0 - n0 // 5
    lo[10] = hi[10] = n0 // 2
    return thr, lo, hi


def recount_qmax(eng, x, groups, seed, M, sj, K, prec, thr, lo, hi, q, measure):
    nser = x.shape[0]
    surr = eng.mc_phase_surrogates(x, groups, seed, 0, M)
    out = []
    for u in range(M):
        if nser == 2:
            R = eng.wct(surr[u, 0], surr[u, 1], 1.0, 0.25, sj, MORLET, 6.0, K, want_angle=False, precision=prec)[0]
        else:
            R = eng.wct3(*surr[u], 1.0, 0.25, sj, MORLET, 6.0, K, precision=prec)[measure]
        Q = reference(select(R, thr, lo, hi), q)[0]
        out.append(int(Q[0]) if Q.size else 0)
    return np.array(out, dtype=np.uint64)


def check_units(eng, nser, n0, K, prec, M=4, seed=23, measure=None):
    x, sj, mask, serial = P.setup(eng, nser, n0, K, prec)
    S = sj.size
    maxscale = S - 3
    groups = (0, 1) if nser == 2 else (0, 1, 1)
    before = P.observed(eng, nser)
    obs = before[0] if nser == 2 else before[measure]
    thr, lo, hi = row_args(S, n0, obs)
    q = weights(sj)
    # an earlier point-wise test keeps its counts
    P.count(eng, x, groups, 3, 0, 2, sj, mask, maxscale, K, prec, serial)
    p0 = P.counted_p(eng, nser)
    hs = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    qmax = eng.cluster_test(x, groups, seed, 0, M, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hs,
                            serial=serial, thr=thr, lo=lo, hi=hi, q=q,
                            measure=None if nser == 2 else measure, precision=prec)
    after = P.observed(eng, nser)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before, after))
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(P.counted_p(eng, nser), p0))
    hh = [np.zeros((S, NBINS), dtype=np.int64) for _ in range(nser - 1)]
    eng.wct_mc_phase(x, groups, seed, 0, M, 1.0, sj, MORLET, 6.0, K, mask, maxscale, NBINS, *hh, precision=prec)
    assert all(np.array_equal(a, b) for a, b in zip(hs, hh))
    ref = recount_qmax(eng, x, groups, seed, M, sj, K, prec, thr, lo, hi, q, measure)
    assert np.array_equal(qmax, ref)
    assert (ref > 0).any()
    m = None if nser == 2 else measure
    Q, pts, box = eng.cluster_table(m is not None)
    rQ, rpts, rbox, rlab = reference(select(obs, thr, lo, hi), q)
    assert rQ.size > 1
    assert np.array_equal(Q, rQ) and np.array_equal(pts, rpts) and np.array_equal(box, rbox)
    assert np.array_equal(eng.cluster_labels(m is not None, 0, S, 1, 0, n0, 1), rlab)
    assert np.array_equal(eng.cluster_labels(m is not None, 1, 5, 3, 7, 40, 9), rlab[1:16:3, 7:7 + 40 * 9:9])


@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("nser,measure", [(2, None), (3, 0), (3, 1)])
@pytest.mark.parametrize("n0,K", [(512, 6), (600, 36)])
def test_units_are_the_definition(emu, nser, measure, n0, K, prec):
    """2^k, and a padded length (600 runs at 1024) with a boxcar longer than 32."""
    check_units(emu, nser, n0, K, prec, measure=measure)


@pytest.mark.parametrize("nser,measure", [(2, None), (3, 1)])
def test_units_unpadded(emu, nser, measure):
    emu.set_padding(False)
    try:
        check_units(emu, nser, 600, 6, F64, M=3, measure=measure)
    finally:
        emu.set_padding(True)


# ---- the public calls ----------------------------------------------------------------------------
KW = P.KW


def check_public(h, res, sig, M, seed, groups, measure):
    """ClusterResult against the engine-level recount of the handle's surrogates."""
    from pycwt_b200.wavelet import _wct_problem
    eng = h.engine
    p = _wct_problem(h._y, h.dt, h.dj, h.s0, h.J, h.wavelet, h.normalize, h.precision)
    prec = F32 if h.precision == 'fp32' else F64
    lo, hi = h.coi_ranges()
    q = weights(h.scales)
    unit = h.dj * h.dt / np.min(h.scales) / 2.0 ** 32
    ref = recount_qmax(eng, np.stack(p.yns), groups, seed, M, p.sj, p.klen, prec, np.asarray(sig, dtype=float),
                       lo, hi, q, measure)
    assert np.array_equal(res.null_max, ref.astype(float) * unit)
    obs = h.coherence() if measure is None else (h.partial() if measure == 0 else h.multiple())
    rQ, rpts, rbox, rlab = reference(select(obs, np.asarray(sig, dtype=float), lo, hi), q)
    assert np.array_equal(res.area, rQ.astype(float) * unit)
    assert np.array_equal(res.points, rpts)
    assert np.array_equal(res.rows, rbox[:, :2]) and np.array_equal(res.cols, rbox[:, 2:])
    pv = np.array([(1 + np.sum(ref >= Qc)) / (1 + M) for Qc in rQ])
    assert np.array_equal(res.pvalue, pv)
    assert np.array_equal(h.cluster_labels(), rlab)
    assert np.array_equal(h.cluster_labels(slice(2, None, 4), slice(3, 800, 11)), rlab[2::4, 3:800:11])


@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
def test_public_pair(api, emu, prec):
    x = P.pair()
    h = api.wct_resident(x[0], x[1], 1.0, precision=prec, **KW)
    before = [f.tobytes() for f in P.fields(h)]
    sig = h.surrogate_significance(mc_count=6, seed=11)
    res = h.cluster_test(sig, mc_count=5, seed=12)
    assert isinstance(res, api.ClusterResult)
    assert [f.tobytes() for f in P.fields(h)] == before
    assert res.area.size > 0 and (np.diff(res.area) <= 0).all()
    check_public(h, res, sig, 5, 12, (0, 1), None)


@pytest.mark.parametrize("measure,conditional", [('partial', True), ('multiple', False)])
def test_public_triple(api, emu, measure, conditional):
    x = P.triple()
    h = api.wct3_resident(*x, 1.0, **KW)
    before = [f.tobytes() for f in P.fields(h)]
    sig = h.surrogate_significance(mc_count=5, seed=3, conditional=conditional)[0 if measure == 'partial' else 1]
    res = h.cluster_test(sig, mc_count=4, seed=4, measure=measure, conditional=conditional)
    assert [f.tobytes() for f in P.fields(h)] == before
    check_public(h, res, sig, 4, 4, (0, 1, 1) if conditional else (0, 1, 2), 0 if measure == 'partial' else 1)


def test_inside_coi_false(api, emu):
    x = P.pair(512)
    h = api.wct_resident(x[0], x[1], 1.0, **KW)
    sig = np.full(len(h.scales), 0.6)
    a = h.cluster_test(sig, mc_count=2, seed=1, inside_coi=False)
    b = h.cluster_test(sig, mc_count=2, seed=1)
    assert a.points.sum() > b.points.sum()
    sel = select(h.coherence(), sig, np.zeros(len(sig), dtype=np.int64), np.full(len(sig), 512))
    assert a.points.sum() == sel.sum()


# ---- lifetime and errors -------------------------------------------------------------------------
def test_lifetime_and_errors(api, emu):
    from pycwt_b200 import _engine, helpers
    x = P.pair(512)
    y = P.triple(512)
    h = api.wct_resident(x[0], x[1], 1.0, **KW)
    h3 = api.wct3_resident(*y, 1.0, **KW)
    S = len(h.scales)
    sig = np.full(S, 0.7)
    for hh in (h, h3):
        with pytest.raises(_engine.EngineError, match="cluster test"):
            hh.cluster_labels()
    for bad in (None, np.full(S - 1, 0.5), np.full((S, 1), 0.5), 0.5):
        with pytest.raises(ValueError, match="sig"):
            h.cluster_test(bad, mc_count=2)
    for bad in (0, -1, 2 ** 31, 2.5, True):
        with pytest.raises(ValueError, match="mc_count"):
            h.cluster_test(sig, mc_count=bad)
    with pytest.raises(ValueError, match="measure"):
        h3.cluster_test(sig, mc_count=2, measure='both')
    res = h.cluster_test(sig, mc_count=2, seed=5)
    lab = h.cluster_labels()
    assert lab.dtype == np.int32 and lab.max() == res.area.size
    assert h.cluster_labels(slice(0, 0)).shape == (0, 512)
    with pytest.raises(ValueError, match="rows"):
        h.cluster_labels(rows=slice(None, None, -1))
    # the point-wise counts are not touched: none were made
    with pytest.raises(_engine.EngineError, match="surrogate_test"):
        h.pvalues()
    # a changed padding mode
    helpers.set_fft_padding(False)
    try:
        with pytest.raises(ValueError, match="padding"):
            h.cluster_test(sig, mc_count=2, seed=1)
    finally:
        helpers.set_fft_padding(True)
        emu.set_padding(True)
    # a failed engine call leaves nothing readable
    assert np.array_equal(h.cluster_labels(), lab)
    with pytest.raises(_engine.EngineError):
        emu.cluster_test(np.stack([x[0], x[1]]), (0, 1), 1, 0, 1, 1.0, h.scales, MORLET, 6.0, 3,
                         np.ones((S, 512), dtype=np.uint8), S, NBINS, np.zeros((S, NBINS), dtype=np.int64),
                         serial=emu.coherence_serial() + 1, thr=sig, lo=np.zeros(S), hi=np.full(S, 512),
                         q=weights(h.scales))
    with pytest.raises(_engine.EngineError, match="cluster test"):
        h.cluster_labels()
    res = h.cluster_test(sig, mc_count=2, seed=5)
    # a newer wct_resident: the old handle is gone and the new product has no clusters
    hn = api.wct_resident(x[1], x[0], 1.0, **KW)
    with pytest.raises(_engine.EngineError, match="no longer resident"):
        h.cluster_labels()
    with pytest.raises(_engine.EngineError, match="cluster test"):
        hn.cluster_labels()
    # the triple's clusters survive the pair's product, and die with its release
    h3.cluster_test(np.full(S, 0.5), mc_count=2, seed=1, measure='multiple')
    l3 = h3.cluster_labels()
    emu.coherence_release()
    assert np.array_equal(h3.cluster_labels(), l3)
    h3.release()
    with pytest.raises(_engine.EngineError, match="no longer resident"):
        h3.cluster_labels()
    import ctypes
    c = ctypes.c_int64()
    assert emu.lib.cwtb_coherence3_cluster_table(emu.h, 0, ctypes.byref(c), None, None, None) == ERR_STATE
    assert emu.lib.cwtb_coherence_cluster_labels(emu.h, 0, 1, 1, 0, 1, 1, None) == ERR_STATE


def test_labels_of_the_other_product(api, emu):
    """The pair and the triple keep their clusters apart: a handle reads its own product's labels or
    gets an EngineError, whatever the other product holds."""
    from pycwt_b200 import _engine
    x = P.pair(512)
    y = P.triple(512)
    h = api.wct_resident(x[0], x[1], 1.0, **KW)
    h3 = api.wct3_resident(*y, 1.0, **KW)
    S = len(h.scales)
    h.cluster_test(np.full(S, 0.6), mc_count=2, seed=5)
    lab = h.cluster_labels()
    assert lab.max() > 0
    # before any triple test
    with pytest.raises(_engine.EngineError, match="cluster test"):
        h3.cluster_labels()
    # after a triple test that failed in the engine
    h3.cluster_test(np.full(S, 0.5), mc_count=2, seed=1)
    assert h3.cluster_labels().max() > 0
    with pytest.raises(_engine.EngineError):
        emu.cluster_test(np.stack(y), (0, 1, 1), 1, 0, 1, 1.0, h3.scales, MORLET, 6.0, 3,
                         np.ones((S, 512), dtype=np.uint8), S, NBINS, np.zeros((S, NBINS), dtype=np.int64), None,
                         serial=emu.coherence3_serial() + 1, thr=np.full(S, 0.5), lo=np.zeros(S),
                         hi=np.full(S, 512), q=weights(h3.scales), measure=0)
    with pytest.raises(_engine.EngineError, match="cluster test"):
        h3.cluster_labels()
    # a new triple product
    h3.cluster_test(np.full(S, 0.5), mc_count=2, seed=1)
    h3n = api.wct3_resident(*y[::-1], 1.0, **KW)
    with pytest.raises(_engine.EngineError, match="cluster test"):
        h3n.cluster_labels()
    # the pair's labels never moved; and the other way round
    assert np.array_equal(h.cluster_labels(), lab)
    h3n.cluster_test(np.full(S, 0.5), mc_count=2, seed=1, measure='multiple')
    hn = api.wct_resident(x[1], x[0], 1.0, **KW)
    with pytest.raises(_engine.EngineError, match="cluster test"):
        hn.cluster_labels()
    assert h3n.cluster_labels().max() > 0
    hn.release()
    h3n.release()


def test_engine_errors(emu):
    from pycwt_b200._engine import EngineError
    x, sj, mask, serial = P.setup(emu, 2, 256, 3, F64, S=8)
    hs = [np.zeros((8, NBINS), dtype=np.int64)]
    lo, hi = np.zeros(8, dtype=np.int64), np.full(8, 256, dtype=np.int64)
    kw = dict(serial=serial, thr=np.full(8, 0.5), lo=lo, hi=hi, q=weights(sj))
    args = (x, (0, 1), 1, 0, 2, 1.0, sj, MORLET, 6.0, 3, mask, 6, NBINS, *hs)
    emu.cluster_test(*args, **kw)
    with pytest.raises(EngineError, match="status -1"):
        emu.cluster_test(*args, **dict(kw, hi=np.full(8, 257)))
    with pytest.raises(EngineError, match="status -1"):
        emu.cluster_test(*args, **dict(kw, q=np.full(8, 2 ** 32 + 1, dtype=np.uint64)))
    with pytest.raises(EngineError, match="status -4"):
        emu.cluster_test(*args, **dict(kw, serial=serial + 1))
    x3, sj3, mask3, serial3 = P.setup(emu, 3, 256, 3, F64, S=8)
    with pytest.raises(EngineError, match="status -1"):
        emu.cluster_test(x3, (0, 1, 1), 1, 0, 2, 1.0, sj3, MORLET, 6.0, 3, mask3, 6, NBINS, *hs, None,
                         **dict(kw, serial=serial3, measure=2))
