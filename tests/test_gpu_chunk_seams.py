"""The engine's chunk loops across their seams, on the GPU.

Most host loops of engine.cu cut their work into chunks: rows of the two-kernel transforms, launch
groups of the two-kernel classes, rows of the Bluestein convolutions, uploads of the host icwt and
batches of Monte-Carlo units.  Every other test runs them at sizes where the loop runs once, so the
offsets of a second chunk and the short last chunk are checked here.  Each test:

  * picks a geometry with at least three chunks, the last one partial, through the size of the call or
    the existing switches (CWTB_GROUP, CWTB_CHAINS), never through a constant;
  * asserts from the launch record (profile_begin / profile_end: launches and rows per kernel) that the
    loop ran that many chunks, so a retuned chunk size fails the test instead of hiding the seam;
  * compares with a reference that does not run the loop: rows on both sides of every seam against an
    extended-precision transform and bit for bit against the same rows computed in one chunk, or the
    Monte-Carlo counts, histograms and every unit's largest cluster against a recount of the hooks'
    units, one unit at a time.

Worst errors measured on an H100 80GB HBM3 (700 W power limit) are in DESIGN 6.  `pytest --emu` runs the
geometries that the host emulation finishes in reasonable time; the others skip there.
"""
import numpy as np
import pytest

import test_emu_cluster_test as C
import test_emu_coherence_ar1_test as A
import test_emu_overlap_save as osv
import test_emu_power_test as E
import test_emu_surrogate_pvalues as P
import test_gpu_row_parity as rp

MORLET, DOG = 0, 2
F64, F32 = 0, 1
MAX_ROWS = 65535           # rows of one launch (gridDim.y)
BOUND = {F64: rp.EXACT, F32: 1e-5}


def emulated(eng):
    return "emulation" in eng.version()


@pytest.fixture(scope="module")
def eng():
    e = osv.make_engine()
    yield e
    e.set_padding(True)
    e.close()


def profiled(eng, fn):
    eng.profile_begin()
    try:
        out = fn()
    finally:
        prof = eng.profile_end()
    return out, prof


def launches(prof, name, tagged=False):
    """(launches, rows) of the kernels whose name starts with `name` (untagged ones only, unless
    `tagged`: the forward transform and the surrogate generators prefix theirs with 'tag:')."""
    nl = rows = 0
    for p in prof:
        nm = p["name"].replace(" ", "")
        if ":" in nm:
            if not tagged:
                continue
            nm = nm.split(":", 1)[1]
        if nm.startswith(name):
            nl += p["launches"]
            rows += p["rows"]
    return nl, rows


def seams(total, chunk):
    """First and last row, and the rows on both sides of every seam of chunks of `chunk` rows."""
    r = {0, total - 1}
    for s in range(chunk, total, chunk):
        r |= {s - 1, s}
    return sorted(r)


# ---- rows of the power-of-two transforms -----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("log2n", [20, 21])
def test_fft_rows_chunks(eng, log2n):
    """fft_rows: at n = 2^20 the two-kernel rows run in chunks of 256 MiB / (n 16 B) = 16 rows; at
    n = 2^21 the three-level rows in chunks of 512 MiB / (n 16 B) = 16 rows.  40 rows: 16, 16, 8."""
    if emulated(eng):
        pytest.skip("40 rows of 2^%d points: too long on the host emulation" % log2n)
    n, rows, chunk = 2 ** log2n, 40, 16
    rs = np.random.RandomState(log2n)
    x = rs.randn(rows, n) + 1j * rs.randn(rows, n)
    Y, prof = profiled(eng, lambda: eng.fft_c2c(x, -1))
    pa, pa_rows = launches(prof, "PassABody")
    pb, pb_rows = launches(prof, "PassBBody")
    if log2n == 20:
        assert (pa, pa_rows, pb, pb_rows) == (3, rows, 3, rows), prof
    else:
        # pre-pass per outer chunk (K0 = 2), then the 2 x nr interleaved 2^20-point rows in inner
        # chunks of 16: 32 + 32 + 16 rows
        k1 = launches(prof, "PassABody<double,2,")
        assert k1 == (3, rows), prof
        assert (pb, pb_rows) == (5, 2 * rows), prof
    R = seams(rows, chunk)
    ref = np.fft.fft(x[R].astype(np.clongdouble), axis=1)
    err = np.abs(Y[R] - ref).max(axis=1) / np.abs(ref).max(axis=1)
    one = eng.fft_c2c(x[R], -1)           # fewer rows than a chunk: one chunk
    print("  fft_c2c n = 2^%d, %d rows in chunks of %d: worst row error %.2e" % (log2n, rows, chunk, err.max()))
    assert (err <= BOUND[F64]).all(), dict(zip(R, err))
    assert np.array_equal(one, Y[R])


# ---- Bluestein rows and the launch row limit ---------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 1000])
@pytest.mark.parametrize("rows", [65535, 65536, 70000])
def test_bluestein_rows_past_the_launch_limit(eng, n, rows):
    """blue_rows: chunks of min(1 GiB / (L 16 B), 65535) rows.  n = 3 (L = 8): the row limit, one seam
    past 65535 rows; n = 1000 (L = 2048): 32768 rows, two seams at 70000."""
    if emulated(eng) and n > 3:
        pytest.skip("70000 rows of 1000 points: too long on the host emulation")
    check_bluestein_rows(eng, n, rows)


def check_bluestein_rows(eng, n, rows):
    L = 1 << (2 * n - 1).bit_length()
    chunk = min((1 << 30) // (L * 16), MAX_ROWS)
    rs = np.random.RandomState(n + rows)
    x = rs.randn(rows, n) + 1j * rs.randn(rows, n)
    Y, prof = profiled(eng, lambda: eng.fft_c2c(x, -1))
    nchunks = -(-rows // chunk)
    assert launches(prof, "BluePreBody") == (nchunks, rows), prof
    assert launches(prof, "BluePostBody") == (nchunks, rows), prof
    R = seams(rows, chunk)
    ref = np.fft.fft(x[R].astype(np.clongdouble), axis=1)
    err = np.abs(Y[R] - ref).max(axis=1) / np.abs(ref).max(axis=1)
    whole = np.abs(Y - np.fft.fft(x, axis=1)).max() / np.abs(Y).max()
    print("  Bluestein n = %d, %d rows in %d chunks: seam rows %.2e, all rows vs numpy %.2e"
          % (n, rows, nchunks, err.max(), whole))
    assert (err <= BOUND[F64]).all(), dict(zip(R, err))
    assert whole <= BOUND[F64]
    assert np.array_equal(eng.fft_c2c(x[R], -1), Y[R])


@pytest.mark.gpu
def test_unpadded_cwt_scale_chunks(eng):
    """run_job_exact: n0 = 100003 (L = 2^18) in chunks of 1 GiB / (L 16 B) = 256 scales; 600 scales
    give 256, 256, 88.  The seam rows against the longdouble un-padded transform, and bit for bit
    against the same scales in one chunk."""
    if emulated(eng):
        pytest.skip("600 rows of an L = 2^18 convolution: too long on the host emulation")
    n0, S, chunk = 100003, 600, 256
    x = rp.white(n0, 3)
    sj = 2.0 * 2 ** (np.arange(S) / 40.0)
    eng.set_padding(False)
    try:
        W, prof = profiled(eng, lambda: eng.cwt(x, 1.0, sj, MORLET, 6.0))
        R = seams(S, chunk)
        one = eng.cwt(x, 1.0, sj[R], MORLET, 6.0)
    finally:
        eng.set_padding(True)
    assert launches(prof, "BlueProdBody") == (3, S), prof
    ref = rp.ref_rows(x, 1.0, sj[R], MORLET, 6.0, npad=n0)
    err = rp.row_err(W[R], ref)
    print("  un-padded cwt n0 = %d, %d scales in chunks of %d: worst seam row_err %.2e" % (n0, S, chunk, err.max()))
    assert (err <= BOUND[F64]).all(), dict(zip(R, err))
    assert np.array_equal(one, W[R])


# ---- launch groups of the two-kernel classes ---------------------------------------------------------
# Np = 2^16 with the expansion and the overlap-save rows off: dense rows (K' = Np, three-pass first
# kernel) and band rows of K' = 2^14, 2^15 run as two-kernel classes in launch groups of CWTB_GROUP rows,
# the band products of a group in region (i % G) of the class's chain.
GROUP_N0 = 2 ** 16 - 1
GROUP_SJ = 2.0 * 2 ** (np.arange(0, 48) / 16.0)


def group_run(group, chains, prec, profile, lib=None):
    env = dict(CWTB_OS="0", CWTB_CHAINS=str(chains))
    if group:
        env["CWTB_GROUP"] = str(group)
    e = osv.make_engine(lib, **env)
    try:
        e.set_expand_eps(0.0, 0.0)
        x = rp.white(GROUP_N0, 4)
        run = lambda: e.cwt(x, 1.0, GROUP_SJ, DOG, 2.0, precision=prec)   # noqa: E731
        if profile:
            W, prof = profiled(e, run)
        else:
            W, prof = run(), None
        return W, e.last_plan(GROUP_SJ.size), prof, emulated(e)
    finally:
        e.close()


GROUP_REF = {}


def group_reference(prec, lib):
    if (prec, lib) not in GROUP_REF:
        W, plan, _, _ = group_run(0, 2, prec, False, lib)
        x = rp.white(GROUP_N0, 4)
        GROUP_REF[prec, lib] = W, plan, rp.ref_rows(x, 1.0, GROUP_SJ, DOG, 2.0, dtype=np.longdouble if prec == F64 else np.float64)
    return GROUP_REF[prec, lib]


def check_groups(group, chains, prec, lib=None):
    W0, plan, ref = group_reference(prec, lib)
    two = {}
    for j, p in enumerate(plan):
        if p >= 14:                      # two-kernel classes at Np = 2^16
            two.setdefault(p, []).append(j)
    assert max(len(v) for v in two.values()) > 2 * group, (plan, group)
    W, plan1, prof, _ = group_run(group, chains, prec, True, lib)
    W2, _, _, _ = group_run(group, chains, prec, False, lib)       # unprofiled: the chains on their streams
    assert plan1 == plan
    # one launch pair per group of every two-kernel class: >= 3 groups, the last partial
    want = sum(-(-len(v) // group) for v in two.values())
    assert launches(prof, "PassABody") == (want, sum(len(v) for v in two.values())), prof
    assert any(len(v) > 2 * group and (group == 1 or len(v) % group) for v in two.values()), two
    R = sorted(set(j for v in two.values() for i in seams(len(v), group) for j in [v[i]]))
    err = rp.row_err(W[R], ref[R])
    print("  CWTB_GROUP=%d CWTB_CHAINS=%d %s: two-kernel classes %s, worst seam row_err %.2e"
          % (group, chains, "fp64" if prec == F64 else "fp32", {k: len(v) for k, v in two.items()}, err.max()))
    assert (err <= BOUND[prec]).all(), dict(zip(R, err))
    # grouping changes no arithmetic: bit for bit the rows of one group of the default size
    assert np.array_equal(W, W0) and np.array_equal(W2, W0)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("chains", [1, 2])
@pytest.mark.parametrize("group", [1, 3, 5])
def test_two_kernel_launch_groups(group, chains, prec):
    check_groups(group, chains, prec)


# ---- host icwt uploads -------------------------------------------------------------------------------
@pytest.mark.gpu
def test_icwt_host_uploads(eng):
    """icwt_sum_host: uploads of 256 MiB / (n 16 B) rows; n = 2^20 gives 16, 40 rows give 16, 16, 8.
    Against a longdouble sum within the bound of 40 fp64 additions."""
    n, S, chunk = 2 ** 20, 40, 16
    rs = np.random.RandomState(12)
    W = rs.randn(S, n) + 1j * rs.randn(S, n)
    W[chunk] *= 1e3                       # the first row of the second upload dominates its columns
    sj = 2.0 * 2 ** (np.arange(S) / 4.0)
    out, prof = profiled(eng, lambda: eng.icwt_sum(W, sj))
    assert launches(prof, "IcwtBody") == (3, 3), prof
    terms = W.real.astype(np.longdouble) / np.sqrt(sj.astype(np.longdouble))[:, None]
    ref = terms.sum(axis=0)
    tol = 2 * S * np.finfo(float).eps * np.abs(terms).sum(axis=0)
    err = np.abs(out - ref)
    print("  icwt_sum_host %d rows of 2^20 in uploads of %d: worst |error| / bound %.2e"
          % (S, chunk, float((err / tol).max())))
    assert (err <= tol).all()


# ---- Monte-Carlo unit batches -------------------------------------------------------------------------
# mc_run / test_units draw units in batches of min(n_units, 256 MiB / (bytes per unit), MAX_ROWS / ndraw):
# bytes per unit = drawn rows x n0 x (16 for phase-randomised units, sizeof(T) for AR(1) units).  At
# n0 = 2^20 that is 8 .. 64 units; each test runs 2.5 batches and recounts every unit.
MC_N0 = 2 ** 20
MC_S, MC_K = 6, 6


def mc_batch(ndraw, resident):
    return min((256 << 20) // (ndraw * MC_N0 * resident), MAX_ROWS // ndraw)


def hook_units(eng, x, kind, null, seed, first, count):
    if kind == 'phase':
        return eng.mc_phase_surrogates(x, null, seed, first, count)
    return A.units(eng, x, null, seed, first, count)


MC_CASES = [   # (nser, null: 'phase' | 'ar1', conditional, measure of the cluster test)
    (2, 'phase', True, None), (2, 'ar1', True, None), (3, 'ar1', True, 0), (3, 'ar1', False, 1)]


def unit_fields(eng, u, sj, prec):
    """The measures of one unit through engine-level wct / wct3: [R2] or [RP2, RM2]."""
    if len(u) == 2:
        return [eng.wct(u[0], u[1], 1.0, 0.25, sj, MORLET, 6.0, MC_K, want_angle=False, precision=prec)[0]]
    return list(eng.wct3(*u, 1.0, 0.25, sj, MORLET, 6.0, MC_K, precision=prec))[:2]


def largest_cluster(sel, q):
    Q = C.reference(sel, q)[0]
    return int(Q[0]) if Q.size else 0


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("nser,kind,conditional,measure", MC_CASES,
                         ids=["pair-phase", "pair-ar1", "triple-ar1-conditional", "triple-ar1"])
def test_coherence_unit_batches(eng, nser, kind, conditional, measure, prec):
    """surrogate_counts and cluster_test over 2.5 batches: the counts, histograms and every unit's
    largest cluster bit for bit against the hook's units recounted through engine-level wct / wct3,
    the host-unit wct_mc / wct3_mc (one batch) and the labeller's restatement."""
    if emulated(eng):
        pytest.skip("units of 2^20 points: too long on the host emulation")
    n0 = MC_N0
    x, sj, mask, serial = P.setup(eng, nser, n0, MC_K, prec, S=MC_S)
    maxscale = MC_S - 2
    if kind == 'phase':
        null, ndraw, res = ((0, 1) if nser == 2 else (0, 1, 1)), nser, 16
    else:
        null = A.cnull(nser, conditional)
        ndraw, res = sum(1 for h in null.held if not h), 8 if prec == F64 else 4
    batch = mc_batch(ndraw, res)
    M, seed = 2 * batch + batch // 2, 41
    gen_kernel = "PhaseRotBody" if kind == 'phase' else "Ar1BlockBody"
    gen_want = (3, M * nser) if kind == 'phase' else (3 * ndraw, M * ndraw)
    obs = P.observed(eng, nser)[:nser - 1]
    hs, prof = profiled(eng, lambda: P.count(eng, x, null, seed, 0, M, sj, mask, maxscale, MC_K, prec, serial))
    assert launches(prof, gen_kernel, tagged=True) == gen_want, prof
    ps = P.counted_p(eng, nser)
    # the cluster test of the same units: a threshold per row, column ranges on two rows
    o = obs[0 if measure is None else measure]
    thr = np.nanquantile(np.where(np.isfinite(o), o, np.nan), 0.8, axis=1)
    lo = np.zeros(MC_S, dtype=np.int64)
    hi = np.full(MC_S, n0, dtype=np.int64)
    lo[1], hi[2] = n0 // 8, n0 - n0 // 5
    q = C.weights(sj)
    hc = [np.zeros_like(h) for h in hs]
    qmax, cprof = profiled(eng, lambda: eng.cluster_test(
        x, null, seed, 0, M, 1.0, sj, MORLET, 6.0, MC_K, mask, maxscale, P.NBINS, *hc, serial=serial,
        thr=thr, lo=lo, hi=hi, q=q, measure=measure, precision=prec))
    assert launches(cprof, gen_kernel, tagged=True) == gen_want, cprof
    k = [np.zeros(o.shape, dtype=np.int64) for o in obs]
    hh = [np.zeros_like(h) for h in hs]
    ref_qmax = []
    for u0 in range(0, M, 8):
        U = hook_units(eng, x, kind, null, seed, u0, min(8, M - u0))
        for u in U:
            R = unit_fields(eng, u, sj, prec)
            for kk, r, ob in zip(k, R, obs):
                kk += (~np.isfinite(r)) | (r >= ob)
            ref_qmax.append(largest_cluster(C.select(R[0 if measure is None else measure], thr, lo, hi), q))
        if nser == 2:
            eng.wct_mc(U, 1.0, 0.25, sj, MORLET, 6.0, MC_K, mask, maxscale, P.NBINS, hh[0], precision=prec)
        else:
            eng.wct3_mc(U, 1.0, sj, MORLET, 6.0, MC_K, mask, maxscale, P.NBINS, *hh, precision=prec)
    print("  %s nser %d %s: %d units in batches of %d, unit maxima %d .. %d"
          % (kind, nser, "fp64" if prec == F64 else "fp32", M, batch, min(ref_qmax), max(ref_qmax)))
    for p, kk, ob in zip(ps, k, obs):
        assert np.array_equal(p, P.p_of(kk, M, ob), equal_nan=True)
        assert 0 < kk.sum() < M * kk.size
    assert all(np.array_equal(a, b) for a, b in zip(hs, hh))
    assert all(np.array_equal(a, b) for a, b in zip(hc, hh))
    assert np.array_equal(qmax, np.array(ref_qmax, dtype=np.uint64))
    assert len(set(ref_qmax)) > 1


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
def test_power_unit_batches(eng, prec, monkeypatch):
    """The power test (test_units) over 2.5 batches of phase-randomised units: the p-values and every
    unit's largest cluster bit for bit against the hook's units recounted through engine-level cwt."""
    if emulated(eng):
        pytest.skip("units of 2^20 points: too long on the host emulation")
    import pycwt_b200
    from pycwt_b200 import _engine
    from pycwt_b200.resident import _cluster_weights
    monkeypatch.setattr(_engine, "default_engine", lambda *a, **k: eng)
    h = pycwt_b200.power_resident(E.series(MC_N0), 1.0, wavelet=pycwt_b200.Morlet(6), precision=prec,
                                  dj=0.5, s0=2.0, J=4)
    batch = mc_batch(1, 16)
    M, seed = 2 * batch + batch // 2, 17
    Pobs = h.power()
    _, prof = profiled(eng, lambda: h.surrogate_test(mc_count=M, seed=seed, null='phase'))
    assert launches(prof, "PhaseRotBody", tagged=True) == (3, M), prof
    thr = np.quantile(Pobs, 0.95, axis=1)
    res, cprof = profiled(eng, lambda: h.cluster_test(thr, mc_count=M, seed=seed, null='phase'))
    assert launches(cprof, "PhaseRotBody", tagged=True) == (3, M), cprof
    q = C.weights(h.scales)
    lo, hi = h.coi_ranges()
    k = np.zeros(Pobs.shape, dtype=np.int64)
    qmax = []
    for u0 in range(0, M, 8):
        Pi = E.unit_powers(h, 'phase', seed, u0, min(8, M - u0))
        k += E.recount(Pobs, Pi)
        qmax += [largest_cluster(C.select(p, thr, lo, hi), q) for p in Pi]
    print("  power test %s: %d units in batches of %d, unit maxima %d .. %d" % (prec, M, batch, min(qmax), max(qmax)))
    assert np.array_equal(h.pvalues(), E.p_of(k, M, Pobs), equal_nan=True)
    assert 0 < k.sum() < M * k.size
    _, unit_area = _cluster_weights(h)
    assert np.array_equal(res.null_max, np.array(qmax, dtype=float) * unit_area)
    assert len(set(qmax)) > 1
