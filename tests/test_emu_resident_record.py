"""The engine's record of what is resident (cwtb_resident_shape) on the host-emulation build of the
kernels (tests/_emu, the fixture pattern of test_emu_kernels.py).

  * the rule of include/cwt_b200.h ("what stays resident"): after every call, the four records,
    cwtb_w_device_ptr and cwtb_job_serial are what the rule says;
  * the binding sizes every read from the record: after a call that leaves no transform, the
    transform reads raise EngineError; after a batch or a transform of another length, reads
    whose sizes disagree with the record raise ValueError or EngineError instead of overrunning;
  * the Monte-Carlo calls check their histograms and masks with ValueError.
"""
import ctypes
import os

import numpy as np
import pytest

from conftest import ROOT

MORLET, F64, F32 = 0, 0, 1
W, CROSS, COH, COH3 = 0, 1, 2, 3
N0, SJ = 100, np.array([2.0, 4.0, 8.0, 16.0])            # the calls under test
N0_BASE, SJ_BASE = 160, np.array([2.0, 3.0, 5.0, 9.0, 14.0])   # what is resident before them


@pytest.fixture(scope="module")
def emu():
    from pycwt_b200 import build as _build, _engine
    lib = _build.build_emulation(os.path.join(ROOT, "tests", "_emu"))
    eng = _engine.Engine(0, lib_path=lib)
    assert "emulation" in eng.version()
    yield eng
    eng.close()


def series(n, k, seed=0):
    return np.random.RandomState(seed).randn(k, n)


def state(eng):
    """({product: (rows, n0, precision)}, cwtb_w_device_ptr set, cwtb_job_serial)."""
    rec = {}
    for p in (W, CROSS, COH, COH3):
        r, n, pr = ctypes.c_int(-1), ctypes.c_int64(-1), ctypes.c_int(-1)
        assert eng.lib.cwtb_resident_shape(eng.h, p, ctypes.byref(r), ctypes.byref(n), ctypes.byref(pr)) == 0
        rec[p] = (r.value, n.value, pr.value)
    return rec, bool(eng.lib.cwtb_w_device_ptr(eng.h)), eng.job_serial()


def make_all_resident(eng):
    """A transform, a cross spectrum, a coherence and a partial / multiple coherence, all
    N0_BASE x len(SJ_BASE), the cross spectrum in fp32."""
    a, b, c = series(N0_BASE, 3, seed=1)
    eng.set_padding(True)
    eng.set_smooth_filter(None)
    eng.xwt_resident(a, b, 1.0, SJ_BASE, MORLET, 6.0, precision=F32)
    eng.wct_resident(a, b, 1.0, 0.25, SJ_BASE, MORLET, 6.0, 3)
    eng.wct3_resident(a, b, c, 1.0, 0.25, SJ_BASE, MORLET, 6.0, 3)
    eng.cwt(a, 1.0, SJ_BASE, MORLET, 6.0, fetch=False)
    S = len(SJ_BASE)
    rec, wptr, _ = state(eng)
    assert rec == {W: (S, N0_BASE, F64), CROSS: (S, N0_BASE, F32), COH: (S, N0_BASE, F64),
                   COH3: (S, N0_BASE, F64)}, rec
    assert wptr


def mc_args(nser=2):
    mask = np.ones((len(SJ), N0), dtype=np.uint8)
    return mask, len(SJ), 10, [np.zeros((len(SJ), 10), dtype=np.int64) for _ in range(nser - 1)]


def run_cwt_dev(eng, precision, n_chan=None):
    x = series(N0, n_chan or 1, seed=2).astype(np.float32 if precision == F32 else np.float64)
    d = eng.dev_alloc(x.nbytes)
    try:
        eng.h2d(d, x)
        if n_chan is None:
            eng.cwt_dev(d, int(precision == F32), N0, 1.0, SJ, MORLET, 6.0, precision)
        else:
            eng.cwt_batch_dev(d, n_chan, N0, 1.0, SJ, MORLET, 6.0, precision, want_power=True)
    finally:
        eng.dev_free(d)


def mc(eng, name):
    a, b, c = series(N0, 3, seed=3)
    mask, maxscale, nbins, h = mc_args(3)
    args = (1.0, SJ, MORLET, 6.0, 3, mask, maxscale, nbins)
    if name == "wct_mc":
        eng.wct_mc(series(N0, 4, seed=4).reshape(2, 2, N0), 1.0, 0.25, SJ, MORLET, 6.0, 3, mask, maxscale,
                   nbins, h[0])
    elif name == "wct_mc_seeded":
        eng.wct_mc_seeded(5, 0, 2, N0, *args, h[0])
    elif name == "wct3_mc":
        eng.wct3_mc(series(N0, 6, seed=5).reshape(2, 3, N0), *args, h[0], h[1])
    elif name == "wct3_mc_seeded":
        eng.wct3_mc_seeded(5, 0, 2, N0, *args, h[0], h[1])
    elif name == "wct_mc_phase2":
        eng.wct_mc_phase(np.stack([a, b]), [0, 1], 5, 0, 2, *args, h[0])
    else:
        eng.wct_mc_phase(np.stack([a, b, c]), [0, 1, 1], 5, 0, 2, *args, h[0], h[1])


S = len(SJ)
a_, b_, c_ = series(N0, 3, seed=6)
KEEP = None
# name: (call, the transform afterwards (None: as before, 0: none), the slots the call writes)
RULE = {
    # a transform resident
    "cwt": (lambda e: e.cwt(a_, 1.0, SJ, MORLET, 6.0, fetch=False), (S, N0, F64), {}),
    "cwt_fp32": (lambda e: e.cwt(a_.astype(np.float32), 1.0, SJ, MORLET, 6.0, precision=F32, fetch=False),
                 (S, N0, F32), {}),
    "cwt_to_host": (lambda e: e.cwt(a_, 1.0, SJ, MORLET, 6.0), (S, N0, F64), {}),
    "cwt_to_host_fp32": (lambda e: e.cwt(a_, 1.0, SJ, MORLET, 6.0, precision=F32, out_f64=False),
                         (S, N0, F32), {}),
    "cwt_dev": (lambda e: run_cwt_dev(e, F64), (S, N0, F64), {}),
    "cwt_dev_fp32": (lambda e: run_cwt_dev(e, F32), (S, N0, F32), {}),
    "xwt": (lambda e: e.xwt(a_, b_, 1.0, SJ, MORLET, 6.0), (S, N0, F64), {}),
    "xwt_fp32": (lambda e: e.xwt(a_, b_, 1.0, SJ, MORLET, 6.0, precision=F32), (S, N0, F32), {}),
    "cwt_batch_power": (lambda e: e.cwt_batch(series(N0, 4), 1.0, SJ, MORLET, 6.0), (4 * S, N0, F64), {}),
    "cwt_batch_w": (lambda e: e.cwt_batch(series(N0, 4), 1.0, SJ, MORLET, 6.0, want_power=True, want_w=True),
                    (4 * S, N0, F64), {}),
    "cwt_batch_dev": (lambda e: run_cwt_dev(e, F64, n_chan=3), (3 * S, N0, F64), {}),
    "cwt_batch_dev_fp32": (lambda e: run_cwt_dev(e, F32, n_chan=3), (3 * S, N0, F32), {}),
    # none resident
    "wct_boxcar3": (lambda e: e.wct(a_, b_, 1.0, 0.25, SJ, MORLET, 6.0, 3), 0, {}),
    "wct_boxcar80": (lambda e: e.wct(a_, b_, 1.0, 0.25, SJ, MORLET, 6.0, 80), 0, {}),
    "wct3": (lambda e: e.wct3(a_, b_, c_, 1.0, 0.25, SJ, MORLET, 6.0, 3), 0, {}),
    "wct_resident": (lambda e: e.wct_resident(a_, b_, 1.0, 0.25, SJ, MORLET, 6.0, 3), 0, {COH: (S, N0, F64)}),
    "wct3_resident": (lambda e: e.wct3_resident(a_, b_, c_, 1.0, 0.25, SJ, MORLET, 6.0, 80), 0,
                      {COH3: (S, N0, F64)}),
    "xwt_resident": (lambda e: e.xwt_resident(a_, b_, 1.0, SJ, MORLET, 6.0), 0, {CROSS: (S, N0, F64)}),
    "wct_mc": (lambda e: mc(e, "wct_mc"), 0, {}),
    "wct_mc_seeded": (lambda e: mc(e, "wct_mc_seeded"), 0, {}),
    "wct3_mc": (lambda e: mc(e, "wct3_mc"), 0, {}),
    "wct3_mc_seeded": (lambda e: mc(e, "wct3_mc_seeded"), 0, {}),
    "wct_mc_phase2": (lambda e: mc(e, "wct_mc_phase2"), 0, {}),
    "wct_mc_phase3": (lambda e: mc(e, "wct_mc_phase3"), 0, {}),
    # left as it is
    "smooth": (lambda e: e.smooth(series(N0, S) + 0j, 1.0, SJ, 3), KEEP, {}),
    "fft_c2c": (lambda e: e.fft_c2c(series(64, 2) + 0j, -1), KEEP, {}),
    "icwt_sum_host": (lambda e: e.icwt_sum(series(N0, S) + 0j, SJ), KEEP, {}),
    "mc_surrogates": (lambda e: e.mc_surrogates(1, 0, 2, N0), KEEP, {}),
    "mc_surrogates3": (lambda e: e.mc_surrogates3(1, 0, 2, N0), KEEP, {}),
    "mc_phase_surrogates": (lambda e: e.mc_phase_surrogates(np.stack([a_, b_]), [0, 0], 1, 0, 2), KEEP, {}),
    "setters": (lambda e: (e.set_band_eps(1e-16), e.set_expand_eps(), e.set_padding(True),
                           e.set_smooth_filter(None),
                           e.lib.cwtb_set_coherence_precision(e.h, F64)), KEEP, {}),
    "reads": (lambda e: (e.get_w(len(SJ_BASE), N0_BASE), e.power(len(SJ_BASE), N0_BASE),
                         e.global_power(len(SJ_BASE)), e.icwt_sum(), e.signal_fft(),
                         e.field_get(CROSS), e.coherence_window(0, 2, 1, 0, 3, 1),
                         e.coherence3_scale_avg(0, np.ones(len(SJ_BASE)))), KEEP, {}),
    "cross_release": (lambda e: e.cross_release(), KEEP, {CROSS: (0, 0, F64)}),
    "coherence_release": (lambda e: e.coherence_release(), KEEP, {COH: (0, 0, F64)}),
    "coherence3_release": (lambda e: e.coherence3_release(), KEEP, {COH3: (0, 0, F64)}),
}


@pytest.mark.parametrize("name", list(RULE))
def test_rule(emu, name):
    call, w_after, writes = RULE[name]
    make_all_resident(emu)
    before, _, serial = state(emu)
    call(emu)
    rec, wptr, serial_after = state(emu)
    expect = dict(before)
    expect.update(writes)
    if w_after is not KEEP:
        expect[W] = w_after or (0, 0, F64)
    assert rec == expect, (rec, expect)
    assert wptr == (expect[W][0] > 0)
    # (a call may plan more than once: cwt_to_host's plain path, a batch's chunks)
    assert serial_after == serial if w_after is KEEP else serial_after > serial


def test_cwt_to_host_forked_copy(emu):
    """cwt_to_host's own path (the copy of the single-kernel rows overlaps the other chains): it
    plans once and leaves the transform it copied."""
    x = series(4096, 1, seed=10)[0]
    sj = 2.0 * 2 ** (np.arange(0, 24) / 2.0)
    make_all_resident(emu)
    serial = emu.job_serial()
    Wh = emu.cwt(x, 1.0, sj, MORLET, 6.0)
    rec, wptr, serial_after = state(emu)
    assert serial_after == serial + 1 and wptr and rec[W] == (len(sj), 4096, F64)
    assert np.array_equal(emu.get_w(len(sj), 4096), Wh)


def test_reruns_keep_the_transform(emu):
    run_cwt_dev(emu, F64, n_chan=None)
    before = state(emu)
    assert before[0][W] == (S, N0, F64) and before[1]
    emu.bench_last(2)
    assert state(emu) == before
    emu.profile_last()
    assert state(emu) == before


def test_unknown_product(emu):
    assert emu.lib.cwtb_resident_shape(emu.h, 4, None, None, None) == -1     # CWTB_ERR_ARG
    assert emu.lib.cwtb_resident_shape(emu.h, -1, None, None, None) == -1
    assert emu.lib.cwtb_resident_shape(emu.h, W, None, None, None) == 0     # every output may be NULL


@pytest.mark.parametrize("boxcar", [3, 80])
def test_no_transform_after_wct(emu, boxcar):
    from pycwt_b200._engine import EngineError
    emu.cwt(a_, 1.0, SJ, MORLET, 6.0, fetch=False)
    emu.wct(a_, b_, 1.0, 0.25, SJ, MORLET, 6.0, boxcar)
    assert not emu.lib.cwtb_w_device_ptr(emu.h)
    for read in (lambda: emu.get_w(S, N0), lambda: emu.power(S, N0), lambda: emu.global_power(S),
                 lambda: emu.icwt_sum(), lambda: emu.scale_avg_power(np.ones(S)), lambda: emu.field_get(W)):
        with pytest.raises(EngineError, match="no single transform resident"):
            read()
    out = np.empty((S, N0), dtype=np.complex128)
    assert emu.lib.cwtb_get_w(emu.h, out.ctypes.data, 1, 0, S) == -4      # CWTB_ERR_STATE


def test_batch_leaves_its_last_chunk(emu):
    X = series(N0, 4, seed=7)
    power, _ = emu.cwt_batch(X, 1.0, SJ, MORLET, 6.0)
    with pytest.raises(ValueError):
        emu.global_power(S)
    gp = emu.global_power(4 * S)
    assert gp.shape == (4 * S,)
    np.testing.assert_allclose(gp.reshape(4, S), power, rtol=1e-13)
    W = emu.get_w(4 * S, N0)
    np.testing.assert_allclose(W[S:2 * S], emu.cwt(X[1], 1.0, SJ, MORLET, 6.0), rtol=0, atol=1e-13 * abs(W).max())


def test_reads_follow_the_last_length(emu):
    from pycwt_b200._engine import EngineError
    emu.cwt(series(100, 1)[0], 1.0, SJ, MORLET, 6.0, fetch=False)
    a, b = series(5000, 2, seed=8)
    emu.wct(a, b, 1.0, 0.25, SJ, MORLET, 6.0, 3)
    with pytest.raises(EngineError):
        emu.icwt_sum()
    with pytest.raises(EngineError):
        emu.scale_avg_power(np.ones(S))
    emu.cwt(a, 1.0, SJ, MORLET, 6.0, fetch=False)
    assert emu.icwt_sum().shape == (5000,) and emu.scale_avg_power(np.ones(S)).shape == (5000,)


def test_get_w_element_type_is_the_transforms(emu):
    emu.cwt(a_, 1.0, SJ, MORLET, 6.0, fetch=False)
    assert emu.get_w(S, N0, precision=F32, out_f64=False).dtype == np.complex128
    emu.cwt(a_, 1.0, SJ, MORLET, 6.0, precision=F32, fetch=False)
    assert emu.get_w(S, N0, precision=F64, out_f64=False).dtype == np.complex64
    assert emu.get_w(S, N0, out_f64=True).dtype == np.complex128


@pytest.mark.parametrize("name", ["wct_mc", "wct_mc_seeded"])
def test_mc_histogram_and_mask_checks(emu, name):
    mask, maxscale, nbins, (h,) = mc_args(2)
    noise = series(N0, 4, seed=9).reshape(2, 2, N0)

    def call(hist, m=mask):
        if name == "wct_mc":
            return emu.wct_mc(noise, 1.0, 0.25, SJ, MORLET, 6.0, 3, m, maxscale, nbins, hist)
        return emu.wct_mc_seeded(5, 0, 2, N0, 1.0, SJ, MORLET, 6.0, 3, m, maxscale, nbins, hist)

    for bad in (np.zeros((S, nbins + 1), dtype=np.int64), np.zeros((S + 1, nbins), dtype=np.int64),
                np.zeros((S, nbins), dtype=np.int32), np.zeros((nbins, S), dtype=np.int64).T):
        with pytest.raises(ValueError):
            call(bad)
    with pytest.raises(ValueError):
        call(None)
    with pytest.raises(ValueError):
        call(h, mask[:, 1:])
    if name == "wct_mc":
        with pytest.raises(ValueError):
            emu.wct_mc(noise.reshape(1, 4, N0), 1.0, 0.25, SJ, MORLET, 6.0, 3, mask, maxscale, nbins, h)
    assert call(h) is h and h.sum() > 0
