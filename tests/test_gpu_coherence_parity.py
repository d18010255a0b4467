"""Point-by-point parity of the coherence kernels against an extended-precision reference.

`ref_smooth` / `ref_coherence` restate the coherence stage of the reference (wavelet.py:498-514,
mothers.py:83-102) in np.longdouble: the time smoothing by FFT (zero-padded to the transform length,
Gaussian exp(-0.5 (s/dt)^2 k^2) or a filter table), the trim to n0, the scale boxcar with half-weight
end taps in the alignment of convolve2d(..., 'same'), and R = |S12|^2 / (S1 S2).

They are fed the engine's own transforms (Engine.cwt of the same series at the same scales), so the
comparison isolates the kernels after the transform: WctPrepBody, the Gaussian folded into the
forward FFT (EPI_GAUSS, also on the three-level path of N = 2^21), BlueGaussBody and FilterMulBody,
the fused boxcar and ratio WctFinalBody<T, 16 | 64> with its histogram mode, and BoxcarBody (Morlet
smooth, and boxcars longer than 64 taps in wct).

Error model.  A smoothed field F is computed with an error of at most eps * M_F[i] in output row i,
where M_F[i] is the largest magnitude of the rows in the boxcar footprint of row i: the larger of
the time-smoothed row's maximum and the rms of the row before smoothing (an FFT filter spreads the
rounding of its input row's L2 norm over the row).  To first order that bounds
    |dR| <= eps * kappa,   kappa = 2 M12 / sqrt(S1 S2) + R (M1 / S1 + M2 / S2)
(|S12|^2 <= S1 S2 keeps the first term finite), and every coherence assertion is pointwise,
|WCT - R| <= EPS * kappa, on every row and column.  EPS per precision was measured on the H100
(see EPS below).

`pytest --emu` runs the same checks on the host emulation of the kernels.
"""
import numpy as np
import pytest

from oracle import cwt_oracle as orc
from conftest import load_golden, relerr
import test_emu_overlap_save as osv
from test_gpu_row_parity import LD, PI_L, ref_rows

MORLET, PAUL, DOG = 0, 1, 2
F64, F32 = 0, 1
CLD = np.clongdouble
# Largest |WCT - R| / kappa allowed, per engine precision.  Worst measured over the cells below on
# an H100 80GB HBM3 (700 W): fp64 1.7e-16 (config 4 and n0 = 2^20 + 3), fp32 8.4e-8 (config 4); the
# host emulation gives the same within 2x.  The bounds keep a margin of 12x (fp64) and 7x (fp32).
EPS = {F64: 2e-15, F32: 6e-7}
# the reference's own rounding, for its CPU self-check against the fp64 oracle
EPS_ORACLE = 1e-13


# ------------------------------------------------------------------------------------------------
# reference
# ------------------------------------------------------------------------------------------------
def boxcar_window(K):
    """helpers.py:176-191: K taps, half-weight ends, normalised (K = 1: one unit tap)."""
    w = np.ones(K, dtype=LD)
    w[0] = w[-1] = LD(0.5)
    return w / w.sum()


def ref_boxcar(T, K):
    """convolve2d(T, win[:, None], 'same') with zero fill: out[i] = sum_t w[t] T[i - (t - off)],
    off = (K - 1) // 2."""
    w = boxcar_window(K)
    m = T.shape[0]
    off = (K - 1) // 2
    out = np.zeros_like(T)
    for t in range(K):
        sh = t - off
        if 0 <= sh < m:
            out[sh:] += w[t] * T[:m - sh]
        elif sh < 0 and -sh < m:
            out[:m + sh] += w[t] * T[-sh:]
    return out


def footprint_max(a, K):
    """max over the rows q of the boxcar footprint of output row i, q = i - (t - off) for t < K."""
    m = a.size
    off = (K - 1) // 2
    return np.array([a[max(i + off - K + 1, 0):min(i + off, m - 1) + 1].max() for i in range(m)])


def ref_smooth(F, dt, scales, K, npad, table=None):
    """(smoothed field, time-smoothed field before the boxcar) of the rows F [S, n0], in longdouble.
    Real input gives real output (the smoothing filters are real and even)."""
    F = np.asarray(F)
    is_real = not np.iscomplexobj(F)
    S, n0 = F.shape
    X = np.fft.fft(F.astype(LD if is_real else CLD), npad, axis=1)
    if table is None:
        k = 2 * PI_L * (np.fft.fftfreq(npad) * npad).astype(LD) / LD(npad)
        sn = np.asarray(scales, dtype=np.float64).astype(LD) / LD(dt)
        filt = np.exp(LD(-0.5) * (sn[:, None] * k[None, :]) ** 2)
    else:
        filt = np.asarray(table, dtype=np.float64).astype(LD)
        assert filt.shape == (S, npad)
    T = np.fft.ifft(X * filt, axis=1)[:, :n0]
    if is_real:
        T = T.real
    return ref_boxcar(T, K), T


def row_mag(F, T):
    """Per row: the larger of max|T| and the rms of F (see the error model)."""
    F = np.asarray(F)
    rms = np.sqrt((np.abs(F.astype(CLD if np.iscomplexobj(F) else LD)) ** 2).mean(axis=1))
    return np.maximum(np.abs(T).max(axis=1), rms)


def ref_coherence(W1, W2, dt, scales, K, npad, table=None):
    """(R, angle of W1 W2*, kappa) in longdouble from the rows W1, W2 [S, n0]."""
    W1, W2 = np.asarray(W1).astype(CLD), np.asarray(W2).astype(CLD)
    s = np.asarray(scales, dtype=np.float64).astype(LD)[:, None]
    C1 = (W1.real ** 2 + W1.imag ** 2) / s
    C2 = (W2.real ** 2 + W2.imag ** 2) / s
    W12 = W1 * np.conj(W2)
    C12 = W12 / s
    S1, T1 = ref_smooth(C1, dt, scales, K, npad, table)
    S2, T2 = ref_smooth(C2, dt, scales, K, npad, table)
    S12, T12 = ref_smooth(C12, dt, scales, K, npad, table)
    R = (S12.real ** 2 + S12.imag ** 2) / (S1 * S2)
    M1 = footprint_max(row_mag(C1, T1), K)[:, None]
    M2 = footprint_max(row_mag(C2, T2), K)[:, None]
    M12 = footprint_max(row_mag(C12, T12), K)[:, None]
    kappa = 2 * M12 / np.sqrt(S1 * S2) + R * (M1 / S1 + M2 / S2)
    return R, np.angle(W12), kappa


def white_pair(n0, seed=0):
    """Two standardised series, partly coherent: R spans low and high values on every row."""
    rs = np.random.RandomState(seed)
    a = rs.randn(n0)
    b = 0.6 * a + rs.randn(n0)
    return (a - a.mean()) / a.std(), (b - b.mean()) / b.std()


def test_reference_self_check():
    """CPU: ref_smooth / ref_coherence against the fp64 oracle and the reference's fixtures."""
    rs = np.random.RandomState(3)
    for n0, S, K in ((300, 25, 1), (300, 25, 2), (257, 12, 7), (64, 9, 14), (301, 5, 19), (100, 6, 33)):
        sj = 0.7 * 2 ** (np.arange(S) / 3.0)
        Fr = rs.randn(S, n0)
        Fc = rs.randn(S, n0) + 1j * rs.randn(S, n0)
        dj = 2 * 0.6 / K                                  # oracle.smooth: K = round(2 deltaj0 / dj)
        for pad in (True, False):
            orc.PAD_NEXT_POW2 = pad
            try:
                npad = orc.transform_length(n0)
                for F in (Fr, Fc):
                    ref = ref_smooth(F, 1.0, sj, K, npad)[0]
                    assert relerr(ref, orc.smooth(F, 1.0, dj, sj)) <= EPS_ORACLE, (n0, S, K, pad)
                for mo in (orc.Paul(4), orc.DOG(2), orc.DOG(6)):
                    from pycwt_b200 import mothers
                    table = mothers.time_filter_table(mo, sj, 1.0, npad)
                    dj_g = 2 * mo.deltaj0 / K
                    ref = ref_smooth(Fc, 1.0, sj, K, npad, table)[0]
                    assert relerr(ref, orc.smooth_generic(Fc, 1.0, dj_g, sj, mo)) <= EPS_ORACLE, (mo.name, K, pad)
                # the coherence of the oracle's own transforms (scales spaced by the dj of K)
                y1, y2 = white_pair(n0, 4)
                m = orc.Morlet(6)
                W1, sw = orc.cwt(y1, 1.0, dj, 0.7, S - 1, m)[:2]
                W2 = orc.cwt(y2, 1.0, dj, 0.7, S - 1, m)[0]
                WCT, aWCT = orc.wct(y1, y2, 1.0, dj=dj, s0=0.7, J=S - 1, sig=False, normalize=False)[:2]
                R, ang, kappa = ref_coherence(W1, W2, 1.0, sw, K, npad)
                assert (np.abs(WCT - R) <= EPS_ORACLE * kappa).all(), (n0, S, K, pad)
                assert np.abs(aWCT - ang).max() <= 1e-15
            finally:
                orc.PAD_NEXT_POW2 = True
    # fixtures of the reference package
    g = load_golden("smooth_cases")
    for F, Sref in ((g["Wr"], g["Sr"]), (g["Wc"], g["Sc"])):
        ref = ref_smooth(F, float(g["dt"]), g["sj"], int(round(2 * 0.6 / float(g["dj"]))),
                         orc.next_pow2(F.shape[1]))[0]
        assert relerr(ref, Sref) <= 1e-15
    g = load_golden("nopad_wct_smooth")
    for F, Sref in ((g["Wr"], g["Sr"]), (g["Wc"], g["Sc"])):
        assert relerr(ref_smooth(F, 1.0, g["sj"], 5, F.shape[1])[0], Sref) <= 1e-15     # dj = 0.25
    for name, npad_of in (("ao_baltic_xwt_wct", orc.next_pow2), ("nopad_wct_smooth", int)):
        check_wct_fixture(load_golden(name), npad_of)


def check_wct_fixture(g, npad_of):
    """The fixture's WCT / aWCT against the reference computed from longdouble transforms at the
    fixture's transform length."""
    dt = float(g["dt"])
    y1, y2 = [(y - y.mean()) / y.std() for y in (g["y1"], g["y2"])]
    n0 = y1.size
    m = orc.Morlet(6)
    s0 = 2 * dt / m.flambda()
    J = int(np.round(np.log2(n0 * dt / s0) * 12))
    sj = s0 * 2 ** (np.arange(J + 1) / 12)
    npad = npad_of(n0)
    W1, W2 = (ref_rows(y, dt, sj, MORLET, 6.0, npad=npad) for y in (y1, y2))
    R, ang, kappa = ref_coherence(W1, W2, dt, sj, 14, npad)
    err_wct = (np.abs(g["WCT"] - R) / kappa).max()
    err_ang = np.abs(np.angle(np.exp(1j * (g["aWCT"] - ang)))).max()
    print("  fixture vs longdouble (npad %d): WCT max |dR| / kappa %.2e, aWCT %.2e" % (npad, err_wct, err_ang))
    assert err_wct <= EPS_ORACLE
    return err_wct, err_ang


# ------------------------------------------------------------------------------------------------
# engine cells: the coherence stage on the engine's own transforms
# ------------------------------------------------------------------------------------------------
def _emulated(eng):
    return "emulation" in eng.version()


@pytest.fixture(scope="module")
def eng():
    e = osv.make_engine()
    yield e
    e.set_padding(True)
    e.set_smooth_filter(None)
    e.close()


WAVELETS = {"morlet": (MORLET, 6.0, None), "paul4": (PAUL, 4.0, orc.Paul(4)),
            "dog2": (DOG, 2.0, orc.DOG(2)), "dog6": (DOG, 6.0, orc.DOG(6))}


def _cell(name, n0, S, K, prec=F64, pad=True, wav="morlet"):
    return dict(name=name, n0=n0, S=S, K=K, prec=prec, pad=pad, wav=wav)


# Scales run from a row whose Gaussian passes nearly every bin (s = 0.6 dt) to s = 1.5 n0 dt, where
# little more than DC survives (much larger scales underflow the fp32 rows to 0 / 0).
CELLS = [
    # (n0 = 2 has no coherence: the reference's normalisation sqrt(s omega[1] npad) is NaN for npad = 2;
    # the two-point rows are covered by test_smooth_rows)
    _cell("n0=3 S=5 K=3", 3, 5, 3),
    _cell("n0=31 S=33 K=2 fp32", 31, 33, 2, F32),
    _cell("n0=33 S=32 K=16", 33, 32, 16),
    _cell("n0=33 S=1 K=1 fp32", 33, 1, 1, F32),
    _cell("n0=1000 S=31 K=17 fp32", 1000, 31, 17, F32),
    _cell("n0=1000 S=33 K=64", 1000, 33, 64),
    _cell("n0=1000 S=5 K=77 (S < K) fp32", 1000, 5, 77, F32),
    _cell("n0=1000 S=1 K=14", 1000, 1, 14),
    _cell("n0=4097 S=145 K=150", 4097, 145, 150),
    _cell("n0=4097 S=145 K=63 fp32", 4097, 145, 63, F32),
    _cell("n0=4097 S=64 K=19", 4097, 64, 19),
    _cell("n0=4097 S=33 K=65 fp32", 4097, 33, 65, F32),
    _cell("Paul(4) n0=1000 S=60 K=36", 1000, 60, 36, wav="paul4"),
    _cell("DOG(2) n0=1000 S=60 K=34 fp32", 1000, 60, 34, F32, wav="dog2"),
    _cell("DOG(6) n0=4097 S=40 K=23", 4097, 40, 23, wav="dog6"),
    _cell("DOG(2) n0=1000 S=31 K=77 fp32", 1000, 31, 77, F32, wav="dog2"),
    _cell("un-padded n0=1000 S=40 K=14", 1000, 40, 14, pad=False),
    _cell("un-padded n0=1000 S=40 K=36 Paul(4)", 1000, 40, 36, pad=False, wav="paul4"),
    _cell("un-padded n0=4099 S=33 K=65", 4099, 33, 65, pad=False),
    # an odd length with a one-tap boxcar: the highest bins of row 0 (BlueGaussBody's frequency
    # split) are not averaged away by neighbouring rows
    _cell("un-padded n0=1001 S=20 K=1", 1001, 20, 1, pad=False),
    _cell("un-padded n0=100003 S=5 K=19", 100003, 5, 19, pad=False),
    _cell("n0=2^20+3 S=3 K=2", 2 ** 20 + 3, 3, 2),
    _cell("n0=2^20+3 S=4 K=77 fp32", 2 ** 20 + 3, 4, 77, F32),
]


def cell_scales(n0, S):
    if S == 1:
        return np.array([1.5 * n0 if n0 < 100 else 40.0])
    return 0.6 * (2.5 * n0) ** (np.arange(S) / (S - 1))


def run_coherence_cell(eng, cell, y1, y2, sj, dt=1.0):
    """Engine WCT / aWCT and the reference's R, kappa from the engine's own transforms; returns the
    worst |WCT - R| / kappa after the assertions of one cell."""
    fam, par, mother = WAVELETS[cell["wav"]]
    prec, K, n0 = cell["prec"], cell["K"], y1.size
    npad = orc.next_pow2(n0) if cell["pad"] else n0
    eng.set_padding(cell["pad"])
    table = None
    if mother is not None:
        from pycwt_b200 import mothers
        table = mothers.time_filter_table(mother, sj, dt, npad)
    eng.set_smooth_filter(table)
    try:
        WCT, aWCT = eng.wct(y1, y2, dt, 0.1, sj, fam, par, K, precision=prec)
        eng.wct_resident(y1, y2, dt, 0.1, sj, fam, par, K, precision=prec)
        Wr, Ar = eng.coherence_window(0, len(sj), 1, 0, n0, 1)
        # un-padded transforms run in fp64 whatever the precision asked for
        tprec = prec if cell["pad"] else F64
        W1 = eng.cwt(y1, dt, sj, fam, par, precision=tprec)
        W2 = eng.cwt(y2, dt, sj, fam, par, precision=tprec)
    finally:
        eng.set_smooth_filter(None)
        eng.set_padding(True)
    assert np.array_equal(Wr, WCT) and np.array_equal(Ar, aWCT), "wct_resident differs from wct"
    # the transforms are the ones wct used: its angle is the angle of their product to a few ulp
    ulp = np.finfo(np.float32 if tprec == F32 else np.float64).eps
    d = np.abs(aWCT - np.angle(W1 * np.conj(W2)))
    assert np.minimum(d, 2 * np.pi - d).max() <= 8 * ulp * np.pi, cell["name"]
    R, _, kappa = ref_coherence(W1, W2, dt, sj, K, npad, table)
    assert np.isfinite(WCT).all()
    q = np.abs(WCT - R) / kappa
    worst = float(q.max())
    i, n = np.unravel_index(int(q.argmax()), q.shape)
    print("  %-40s worst |WCT - R| / kappa %.2e (row %d, col %d; R %.3f)" % (cell["name"], worst, i, n, R[i, n]))
    assert worst <= EPS[tprec], (cell["name"], worst, i, n)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS, ids=[c["name"] for c in CELLS])
def test_coherence_cell(eng, cell):
    y1, y2 = white_pair(cell["n0"], 7)
    run_coherence_cell(eng, cell, y1, y2, cell_scales(cell["n0"], cell["S"]))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
def test_coherence_config4(eng, prec):
    """Config 4's transform (N = 2^18, s0 = 2, dj = 1/12, 145 rows, K = 14), every row."""
    import workloads as wl
    c4 = wl.C4
    y1, y2 = [(y - y.mean()) / y.std() for y in wl.config4_signals()]
    sj = c4["s0"] * 2 ** (np.arange(c4["J"] + 1) * c4["dj"])
    run_coherence_cell(eng, _cell("config 4 %s" % ("fp64" if prec == F64 else "fp32"), c4["n"], len(sj), 14, prec),
                       y1, y2, sj, c4["dt"])


# ---- Morlet.smooth / Engine.smooth (BoxcarBody) ------------------------------------------------
SMOOTH_CELLS = [(1, 3, 1), (1, 5, 2), (2, 5, 3), (2, 1, 14), (33, 5, 16), (1000, 31, 17), (1000, 5, 19),
                (1000, 40, 23), (300, 64, 34), (300, 60, 36), (4097, 33, 63), (4097, 33, 64), (300, 70, 65),
                (1000, 20, 77), (300, 145, 150), (2 ** 20 + 3, 3, 2), (2 ** 20 + 3, 4, 77)]


@pytest.mark.gpu
@pytest.mark.parametrize("n0,S,K", SMOOTH_CELLS, ids=["n0=%d S=%d K=%d" % c for c in SMOOTH_CELLS])
def test_smooth_rows(eng, n0, S, K):
    rs = np.random.RandomState(n0 + S + K)
    sj = cell_scales(max(n0, 2), S)
    npad = orc.next_pow2(n0)
    worst = 0.0
    for F in (rs.randn(S, n0), rs.randn(S, n0) + 1j * rs.randn(S, n0)):
        out = eng.smooth(F, 1.0, sj, K)
        assert out.dtype == F.dtype
        ref, T = ref_smooth(F, 1.0, sj, K, npad)
        M = footprint_max(row_mag(F, T), K)
        q = (np.abs(out - ref).max(axis=1) / M).max()
        worst = max(worst, float(q))
    print("  smooth n0 = %d S = %d K = %d: worst row error / footprint max %.2e" % (n0, S, K, worst))
    assert worst <= EPS[F64], worst


# ---- Monte-Carlo histograms (WctFinalBody's histogram mode, rows below maxscale) ----------------
@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("K", [14, 19, 36, 77])
def test_mc_histogram_explained(eng, K, prec):
    """Histograms of wct_mc_seeded and of wct_mc fed the same surrogates equal the binned reference
    R of the engine's own transforms of those surrogates, except at points whose R lies within
    EPS kappa of a bin edge: per row sum |h - h_ref| <= 2 x (near-edge points), zero without any."""
    n0, S, maxscale, nbins, seed, pairs = 600, 45, 37, 1000, 77, 2     # maxscale not a multiple of 32
    sj = 2.0 * 2 ** (np.arange(S) / 8.0)
    mask = ((np.arange(n0)[None, :] + 3 * np.arange(S)[:, None]) % 7 != 0).astype(np.uint8)
    h_seeded = np.zeros((S, nbins), dtype=np.int64)
    eng.wct_mc_seeded(seed, 0, pairs, n0, 1.0, sj, MORLET, 6.0, K, mask, maxscale, nbins, h_seeded, precision=prec)
    noise = eng.mc_surrogates(seed, 0, pairs, n0)
    h_host = np.zeros((S, nbins), dtype=np.int64)
    eng.wct_mc(noise, 1.0, 0.1, sj, MORLET, 6.0, K, mask, maxscale, nbins, h_host, precision=prec)
    assert np.array_equal(h_seeded, h_host)
    h_ref = np.zeros((S, nbins), dtype=np.int64)
    near = np.zeros(S, dtype=np.int64)
    npad = orc.next_pow2(n0)
    for p in range(pairs):
        W1 = eng.cwt(noise[p, 0], 1.0, sj, MORLET, 6.0, precision=prec)
        W2 = eng.cwt(noise[p, 1], 1.0, sj, MORLET, 6.0, precision=prec)
        R, _, kappa = ref_coherence(W1, W2, 1.0, sj, K, npad)
        x = R * nbins
        edge = np.abs(x - np.round(x)) <= nbins * EPS[prec] * kappa
        for i in range(maxscale):
            m = mask[i].astype(bool)
            b = np.clip(np.floor(x[i, m]).astype(np.int64), 0, nbins - 1)
            h_ref[i] += np.bincount(b, minlength=nbins)
            near[i] += int(edge[i, m].sum())
    assert h_ref[maxscale:].sum() == 0 and h_seeded[maxscale:].sum() == 0
    diff = np.abs(h_seeded - h_ref).sum(axis=1)
    print("  MC K = %d %s: %d points binned, %d within EPS kappa of an edge, %d bin counts differ"
          % (K, "fp64" if prec == F64 else "fp32", h_ref.sum(), near.sum(), diff.sum()))
    assert (diff <= 2 * near).all(), dict((i, (diff[i], near[i])) for i in range(S) if diff[i] > 2 * near[i])


# ------------------------------------------------------------------------------------------------
# public API at the boxcar widths of fine dj and of the generic smoothing (1e-10 against the oracle)
# ------------------------------------------------------------------------------------------------
TOL = 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize("dj", [1 / 16, 1 / 64])
def test_wct_fine_dj(dj):
    """Morlet K = round(1.2 / dj): 19 taps at dj = 1/16, 77 at dj = 1/64."""
    import pycwt_b200 as pycwt
    g = load_golden("ao_baltic_xwt_wct")
    y1, y2, dt = g["y1"], g["y2"], float(g["dt"])
    WCT, aWCT = pycwt.wct(y1, y2, dt, dj=dj, sig=False, wavelet=pycwt.Morlet(6))[:2]
    Wr, Ar = orc.wct(y1, y2, dt, dj=dj, sig=False, wavelet=orc.Morlet(6))[:2]
    assert relerr(WCT, Wr) < TOL and relerr(aWCT, Ar) < TOL
    h = pycwt.wct_resident(y1, y2, dt, dj=dj, wavelet=pycwt.Morlet(6))
    assert np.array_equal(h.coherence(), WCT) and np.array_equal(h.phase(), aWCT)


@pytest.mark.gpu
def test_generic_smoothing_default_dj():
    """Paul(4), DOG(2), DOG(6) with generic smoothing at dj = 1/12 (K = 36, 34, 23)."""
    import pycwt_b200 as pycwt
    from pycwt_b200 import mothers
    rs = np.random.RandomState(21)
    n = 700
    y1 = rs.randn(n).cumsum() * 0.1 + rs.randn(n)
    y2 = 0.5 * y1 + rs.randn(n)
    dt, dj, J = 0.5, 1 / 12, 60
    old = mothers.enable_generic_smoothing(True)
    try:
        for mo, mr in ((pycwt.Paul(4), orc.Paul(4)), (pycwt.DOG(2), orc.DOG(2)), (pycwt.DOG(6), orc.DOG(6))):
            WCT, aWCT = pycwt.wct(y1, y2, dt, dj, s0=2 * dt, J=J, sig=False, wavelet=mo)[:2]
            y1n, y2n = (y1 - y1.mean()) / y1.std(), (y2 - y2.mean()) / y2.std()
            W1, s = orc.cwt(y1n, dt, dj, 2 * dt, J, mr)[:2]
            W2 = orc.cwt(y2n, dt, dj, 2 * dt, J, mr)[0]
            inv = 1.0 / s[:, None]
            S1 = orc.smooth_generic(np.abs(W1) ** 2 * inv, dt, dj, s, mr)
            S2 = orc.smooth_generic(np.abs(W2) ** 2 * inv, dt, dj, s, mr)
            S12 = orc.smooth_generic(W1 * W2.conj() * inv, dt, dj, s, mr)
            assert relerr(WCT, np.abs(S12) ** 2 / (S1 * S2)) < TOL, mo.name
            # (DOG's real rows put many angles at +-pi: compared modulo 2 pi)
            assert np.abs(np.angle(np.exp(1j * (aWCT - np.angle(W1 * W2.conj()))))).max() < TOL * np.pi, mo.name
    finally:
        mothers.enable_generic_smoothing(old)


@pytest.mark.gpu
def test_wct_significance_fine_dj_seeded():
    """dj = 1/64 (K = 77 > the 65 rows): the seeded host RNG gives the oracle's surrogates."""
    import pycwt_b200 as pycwt
    dt, dj, s0, J = 1.0, 1 / 64, 2.0, 64
    rs = np.random.RandomState(5)
    sig_ref = orc.wct_significance(0.3, 0.2, dt, dj, s0, J, mc_count=4, rng=rs)
    np.random.set_state(np.random.RandomState(5).get_state())
    sig = pycwt.wct_significance(0.3, 0.2, dt, dj, s0, J, wavelet="morlet", mc_count=4,
                                 progress=False, cache=False)
    assert relerr(sig, sig_ref) < 1e-9
