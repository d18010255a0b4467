"""Partial and multiple wavelet coherence on the GPU.

Point by point against the extended-precision restatement of test_gpu_coherence_parity.py
(`ref_smooth`: time smoothing by FFT in np.longdouble, trim, scale boxcar), fed the engine's own
transforms of the three series, extended to the five smoothed fields S_y, S_1, S_2, S_y1, S_y2, S_12
(S_12 with the conjugate of x2's transform, as every cross here).

Error model.  As in test_gpu_coherence_parity.py, a smoothed field F carries an error of at most
eps * M_F at a point, M_F the footprint maximum of the row magnitudes (`footprint_max(row_mag)`).
To first order, with u = S_y1 S_2 - S_y2 conj(S_12), Dy = S_y S_2 - |S_y2|^2, D12 = S_1 S_2 - |S_12|^2
and N = S_2 |S_y1|^2 + S_1 |S_y2|^2 - 2 Re(S_y1 S_12 conj(S_y2)):
    |dRP2| <= eps * kappa_P,  kappa_P = 2 |u| u' / (Dy D12) + RP2 (Dy' / Dy + D12' / D12)
    |dRM2| <= eps * kappa_M,  kappa_M = N' / (S_y D12) + RM2 (M_y / S_y + D12' / D12)
where the primed quantities are the first-order bounds of the products with every field F replaced
by M_F in turn (u' = M_y1 S_2 + |S_y1| M_2 + M_y2 |S_12| + |S_y2| M_12, and so on).  The combination
itself runs in double, so its rounding is inside the same first-order terms.  EPS per precision was
measured on the H100 (see EPS below).

Also, at config 4's geometry, the public calls against the oracle composition under the bounds of
tests/test_emu_partial_coherence.py.
"""
import numpy as np
import pytest

from oracle import cwt_oracle as orc
import test_emu_overlap_save as osv
from test_gpu_coherence_parity import LD, CLD, ref_smooth, row_mag, footprint_max
from test_emu_partial_coherence import oracle_wct3, scaled_err, TOL, TOL32

MORLET = 0
F64, F32 = 0, 1
# Largest |R - R_ref| / kappa allowed, per engine precision: the bounds of test_gpu_coherence_parity.py.
# Worst measured over the cells below on an H100 80GB HBM3 (700 W): fp64 1.2e-16, fp32 3.3e-8, both at
# config 4; the host emulation gives the same or less.  Margins of 16x (fp64) and 18x (fp32).
EPS = {F64: 2e-15, F32: 6e-7}


@pytest.fixture(scope="module")
def eng():
    e = osv.make_engine()
    yield e
    e.set_padding(True)
    e.close()


def config4_triple(n=None):
    """config 4's two series and a third chirp with another phase and noise of its own."""
    import workloads as wl
    y, x1 = wl.config4_signals(n)
    n = y.size
    return y, x1, wl.chirp(n, phase=2.1) + 0.5 * np.random.RandomState(2).randn(n)


def ref_wct3(Ws, dt, scales, K, npad):
    """(RP2, RM2, kappa_P, kappa_M) in longdouble from the engine's transforms Wy, W1, W2."""
    s = np.asarray(scales, dtype=np.float64).astype(LD)[:, None]
    Wy, W1, W2 = (np.asarray(W).astype(CLD) for W in Ws)
    S, M = {}, {}
    for key, F in (("y", (Wy.real ** 2 + Wy.imag ** 2) / s), ("1", (W1.real ** 2 + W1.imag ** 2) / s),
                   ("2", (W2.real ** 2 + W2.imag ** 2) / s), ("y1", Wy * np.conj(W1) / s),
                   ("y2", Wy * np.conj(W2) / s), ("12", W1 * np.conj(W2) / s)):
        S[key], T = ref_smooth(F, dt, scales, K, npad)
        M[key] = footprint_max(row_mag(F, T), K)[:, None]
    Sy, S1, S2, Sy1, Sy2, S12 = S["y"], S["1"], S["2"], S["y1"], S["y2"], S["12"]
    ay1, ay2, a12 = np.abs(Sy1), np.abs(Sy2), np.abs(S12)
    u = Sy1 * S2 - Sy2 * np.conj(S12)
    Dy = Sy * S2 - ay2 ** 2
    D12 = S1 * S2 - a12 ** 2
    RP2 = np.abs(u) ** 2 / (Dy * D12)
    N = S2 * ay1 ** 2 + S1 * ay2 ** 2 - 2 * (Sy1 * S12 * np.conj(Sy2)).real
    RM2 = N / (Sy * D12)
    du = M["y1"] * S2 + ay1 * M["2"] + M["y2"] * a12 + ay2 * M["12"]
    dDy = M["y"] * S2 + Sy * M["2"] + 2 * ay2 * M["y2"]
    dD12 = M["1"] * S2 + S1 * M["2"] + 2 * a12 * M["12"]
    dN = (M["2"] * ay1 ** 2 + 2 * S2 * ay1 * M["y1"] + M["1"] * ay2 ** 2 + 2 * S1 * ay2 * M["y2"]
          + 2 * (M["y1"] * a12 * ay2 + ay1 * M["12"] * ay2 + ay1 * a12 * M["y2"]))
    kP = 2 * np.abs(u) * du / (Dy * D12) + RP2 * (dDy / Dy + dD12 / D12)
    kM = dN / (Sy * D12) + RM2 * (M["y"] / Sy + dD12 / D12)
    return RP2, RM2, kP, kM


def run_parity(eng, name, ys, sj, K, prec, pad=True, dt=1.0):
    n0 = ys[0].size
    npad = orc.next_pow2(n0) if pad else n0
    eng.set_padding(pad)
    try:
        RP2, RM2 = eng.wct3(*ys, dt, 0.1, sj, MORLET, 6.0, K, precision=prec)
        tprec = prec if pad else F64          # un-padded transforms run in fp64
        Ws = [eng.cwt(y, dt, sj, MORLET, 6.0, precision=tprec) for y in ys]
    finally:
        eng.set_padding(True)
    rp, rm, kP, kM = ref_wct3(Ws, dt, sj, K, npad)
    assert np.isfinite(RP2).all() and np.isfinite(RM2).all()
    qp = float((np.abs(RP2 - rp) / kP).max())
    qm = float((np.abs(RM2 - rm) / kM).max())
    print("  %-36s worst |dRP2| / kappa_P %.2e, |dRM2| / kappa_M %.2e" % (name, qp, qm))
    assert qp <= EPS[tprec] and qm <= EPS[tprec], (name, qp, qm)


def white_triple(n0, seed=0):
    rs = np.random.RandomState(seed)
    a = rs.randn(n0)
    b = 0.6 * a + rs.randn(n0)
    c = 0.4 * a + 0.3 * b + rs.randn(n0)
    return [(v - v.mean()) / v.std() for v in (a, b, c)]


CELLS = [  # name, n0, S, K, prec, pad
    ("n0=4097 S=145 K=150", 4097, 145, 150, F64, True),
    ("n0=4097 S=64 K=77 fp32", 4097, 64, 77, F32, True),
    ("n0=1000 S=60 K=36 fp32", 1000, 60, 36, F32, True),
    ("un-padded n0=4099 S=40 K=14", 4099, 40, 14, F64, False),
    ("un-padded n0=1001 S=33 K=65", 1001, 33, 65, F64, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS, ids=[c[0] for c in CELLS])
def test_parity_cell(eng, cell):
    name, n0, S, K, prec, pad = cell
    sj = 0.6 * (2.5 * n0) ** (np.arange(S) / (S - 1))
    run_parity(eng, name, white_triple(n0, 7), sj, K, prec, pad)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F64, F32])
def test_parity_config4(eng, prec):
    """Config 4's transform (N = 2^18, s0 = 2, dj = 1/12, 145 rows, K = 14), every row."""
    import workloads as wl
    c4 = wl.C4
    ys = [(y - y.mean()) / y.std() for y in config4_triple()]
    sj = c4["s0"] * 2 ** (np.arange(c4["J"] + 1) * c4["dj"])
    run_parity(eng, "config 4 %s" % ("fp64" if prec == F64 else "fp32"), ys, sj, 14, prec, dt=c4["dt"])


@pytest.mark.gpu
def test_config4_public_calls():
    """partial_wct / multiple_wct at config 4: fp64 against the oracle composition, fp32 against
    fp64, with the bounds of the CPU test."""
    import pycwt_b200 as pycwt
    import workloads as wl
    c4 = wl.C4
    y, x1, x2 = config4_triple()
    kw = dict(dj=c4["dj"], s0=c4["s0"], J=c4["J"])
    rp, rm, Dp, Dm, _ = oracle_wct3(y, x1, x2, c4["dt"], c4["dj"], c4["s0"], c4["J"], orc.Morlet(6))
    out = {}
    for p in ("fp64", "fp32"):
        out[p] = (pycwt.partial_wct(y, x1, x2, c4["dt"], precision=p, **kw)[0],
                  pycwt.multiple_wct(y, x1, x2, c4["dt"], precision=p, **kw)[0])
    e64 = (scaled_err(out["fp64"][0], rp, Dp), scaled_err(out["fp64"][1], rm, Dm))
    e32 = (scaled_err(out["fp32"][0], out["fp64"][0], Dp), scaled_err(out["fp32"][1], out["fp64"][1], Dm))
    print("  config 4: fp64 vs oracle |dRP2| D %.2e |dRM2| D %.2e; fp32 vs fp64 %.2e %.2e" % (e64 + e32))
    assert max(e64) <= TOL and max(e32) <= TOL32
