"""Resident partial and multiple coherence (`wct3_resident`) on the GPU.

  * At config 4's triple (three 2^18-point series, s0 = 2, dj = 1/12, J = 144, K = 14), fp64 and
    fp32: `partial()` / `multiple()` bit-identical to `partial_wct` / `multiple_wct`, windows equal
    to numpy slicing, every reduction of both measures against numpy on the fetched fields (the
    checks of test_emu_coherence3_resident.py), repeated reductions bit-identical, and the handle
    alive after seeded Monte-Carlo runs.
  * The partial phase point by point against the extended-precision restatement of
    test_gpu_partial_coherence.py (`ref_smooth` in np.longdouble of the engine's own transforms).
    With u = S_y1 S_2 - S_y2 conj(S_12) and u' its first-order bound given in that file's header
    (u' = M_y1 S_2 + |S_y1| M_2 + M_y2 |S_12| + |S_y2| M_12), an error of at most EPS u' in u moves
    e^{i phi} by at most 2 EPS u' / |u|, so the check is
        |u_ref| |e^{i phi} - e^{i phi_ref}| <= 2 EPS u'
    with that file's EPS (2e-15 fp64, 6e-7 fp32), at K = 14, 36 and 77 and at the un-padded lengths
    1001 and 4099.
"""
import numpy as np
import pytest

from oracle import cwt_oracle as orc
import test_emu_overlap_save as osv
from test_gpu_coherence_parity import LD, CLD, ref_smooth, row_mag, footprint_max
from test_gpu_partial_coherence import EPS, config4_triple, white_triple
from test_emu_coherence_resident import WINDOWS, sig95_with_gaps
from test_emu_coherence3_resident import check_all

pytestmark = pytest.mark.gpu

MORLET = 0
F64, F32 = 0, 1


@pytest.fixture(scope="module")
def eng():
    e = osv.make_engine()
    yield e
    e.set_padding(True)
    e.close()


# ---- the partial phase against the extended-precision restatement --------------------------------
def ref_u(Ws, dt, scales, K, npad):
    """(u, u') in longdouble from the engine's transforms Wy, W1, W2."""
    s = np.asarray(scales, dtype=np.float64).astype(LD)[:, None]
    Wy, W1, W2 = (np.asarray(W).astype(CLD) for W in Ws)
    S, M = {}, {}
    for key, F in (("2", (W2.real ** 2 + W2.imag ** 2) / s), ("y1", Wy * np.conj(W1) / s),
                   ("y2", Wy * np.conj(W2) / s), ("12", W1 * np.conj(W2) / s)):
        S[key], T = ref_smooth(F, dt, scales, K, npad)
        M[key] = footprint_max(row_mag(F, T), K)[:, None]
    u = S["y1"] * S["2"] - S["y2"] * np.conj(S["12"])
    du = M["y1"] * S["2"] + np.abs(S["y1"]) * M["2"] + M["y2"] * np.abs(S["12"]) + np.abs(S["y2"]) * M["12"]
    return u, du


CELLS = [  # name, n0, S, K, prec, pad
    ("n0=4097 S=64 K=14", 4097, 64, 14, F64, True),
    ("n0=4097 S=64 K=14 fp32", 4097, 64, 14, F32, True),
    ("n0=2048 S=60 K=36", 2048, 60, 36, F64, True),
    ("n0=1000 S=60 K=36 fp32", 1000, 60, 36, F32, True),
    ("n0=4097 S=64 K=77", 4097, 64, 77, F64, True),
    ("n0=4097 S=64 K=77 fp32", 4097, 64, 77, F32, True),
    ("un-padded n0=4099 S=40 K=14", 4099, 40, 14, F64, False),
    ("un-padded n0=1001 S=33 K=36", 1001, 33, 36, F64, False),
]


@pytest.mark.parametrize("cell", CELLS, ids=[c[0] for c in CELLS])
def test_partial_phase_parity(eng, cell):
    name, n0, S, K, prec, pad = cell
    sj = 0.6 * (2.5 * n0) ** (np.arange(S) / (S - 1))
    ys = white_triple(n0, 7)
    npad = orc.next_pow2(n0) if pad else n0
    eng.set_padding(pad)
    try:
        eng.wct3_resident(*ys, 1.0, 0.1, sj, MORLET, 6.0, K, precision=prec)
        phi = np.array(eng.coherence3_window(0, 0, S, 1, 0, n0, 1, want_value=False, want_phase=True)[1])
        eng.coherence3_release()
        tprec = prec if pad else F64          # un-padded transforms run in fp64
        Ws = [eng.cwt(y, 1.0, sj, MORLET, 6.0, precision=tprec) for y in ys]
    finally:
        eng.set_padding(True)
    u, du = ref_u(Ws, 1.0, sj, K, npad)
    phi_ref = np.angle(u.astype(np.complex128))
    assert np.isfinite(phi).all()
    err = np.abs(u).astype(np.float64) * np.abs(np.exp(1j * phi) - np.exp(1j * phi_ref))
    q = float((err / (2 * du.astype(np.float64))).max())
    print("  %-32s worst |u| |de^{i phi}| / (2 u') %.2e (EPS %.0e, margin %.0fx)"
          % (name, q, EPS[tprec], EPS[tprec] / max(q, 1e-300)))
    assert q <= EPS[tprec], (name, q)


# ---- config 4 ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pycwt(has_cuda):
    if not has_cuda:
        pytest.skip("no CUDA device")
    import pycwt_b200
    return pycwt_b200


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_config4_resident(pycwt, precision):
    import workloads as wl
    c4 = wl.C4
    y, x1, x2 = config4_triple()
    kw = dict(dj=c4["dj"], s0=c4["s0"], J=c4["J"], precision=precision)
    RP2, coi, freq = pycwt.partial_wct(y, x1, x2, c4["dt"], **kw)
    RP2 = np.array(RP2)                       # own copies: the pinned buffers are pooled
    RM2 = np.array(pycwt.multiple_wct(y, x1, x2, c4["dt"], **kw)[0])
    h = pycwt.wct3_resident(y, x1, x2, c4["dt"], **kw)
    assert h.shape == RP2.shape == (c4["J"] + 1, y.size)
    assert np.array_equal(h.coi, coi) and np.array_equal(h.freq, freq)
    assert np.array_equal(h.partial(), RP2) and np.array_equal(h.multiple(), RM2)
    phase = np.array(h.phase())
    assert np.isfinite(phase).all() and (np.abs(phase) <= np.pi).all()
    for rows, cols in WINDOWS + [(slice(None, None, 3), slice(None, None, 3)),
                                 (slice(7, 100, 9), slice(-70001, -3, 1001))]:
        a, b, c = h.window(rows, cols)
        assert np.array_equal(a, RP2[rows, cols]), (rows, cols)
        assert np.array_equal(b, phase[rows, cols]), (rows, cols)
        assert np.array_equal(c, RM2[rows, cols]), (rows, cols)

    check_all(h, RP2, phase, RM2, sig95_with_gaps(h, RP2), sig95_with_gaps(h, RM2))
    sp, sm = h.significance(mc_count=8, seed=5, progress=False)
    check_all(h, RP2, phase, RM2, sp, sm)

    per = h.period
    calls = [lambda: h.global_coherence(),
             lambda: h.global_coherence('multiple', inside_coi=True, sig=sm),
             lambda: h.significant_fraction(sp),
             lambda: h.mean_phase(sig=sp),
             lambda: h.mean_phase(per[10], per[100], inside_coi=False, per_scale=True),
             lambda: h.scale_avg(per[20], per[60])]
    first = [f() for f in calls]
    h.surrogate_significance(mc_count=4, seed=2)
    for f, a in zip(calls, first):
        b = f()
        for x, y_ in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            assert np.array_equal(x, y_, equal_nan=True)
    assert np.array_equal(h.partial(), RP2)
    h.release()
