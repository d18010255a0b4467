"""fp32 cross-wavelet transform, coherence and Monte-Carlo coherence significance, checked on the
host-emulation build of the kernels (tests/_emu, the fixture pattern of test_emu_kernels.py).

Contract of the fp32 coherence (DESIGN.md section 6):
  * W12 within 2e-5 of max|W12| (two transforms, each at the fp32 engine's 1e-5);
  * the angle within max|W12_ref| |e^{i aWCT32} - e^{i aWCT_ref}| <= 4e-5 max|W12_ref|, which
    follows from the W12 bound;
  * |WCT32 - WCT64| <= WCT_BOUND, about three times the largest error measured (config 4 on an
    H100); it must stay below the 1e-3 width of the significance histogram's bins;
  * Monte-Carlo histograms from the same surrogates: equal counts per row, every sample at most
    one bin away, 95 % levels within 2e-3.
"""
import os
import socket
import sys

import numpy as np
import pytest

from conftest import ROOT, load_golden, relerr
from oracle import cwt_oracle as orc

WCT_BOUND = 2.5e-4


def check_fp32_coherence(W12, aWCT, WCT, W12r, aWCTr, WCTr):
    assert W12.dtype == np.complex128 and WCT.dtype == np.float64 and aWCT.dtype == np.float64
    assert relerr(W12, W12r) <= 2e-5
    m = np.abs(W12r).max()
    assert (np.abs(W12r) * np.abs(np.exp(1j * aWCT) - np.exp(1j * aWCTr))).max() <= 4e-5 * m
    assert np.abs(WCT - WCTr).max() <= WCT_BOUND


def check_fp32_histograms(h32, h64, prob):
    from pycwt_b200 import wavelet as wv
    assert h64.sum() > 0
    assert (h32.sum(axis=1) == h64.sum(axis=1)).all()
    # a sample that moves by at most one bin changes the cumulative count at bin b by at most the
    # counts of bins b and b + 1
    nxt = np.concatenate([h64[:, 1:], np.zeros((h64.shape[0], 1), h64.dtype)], axis=1)
    assert (np.abs(np.cumsum(h32, axis=1) - np.cumsum(h64, axis=1)) <= h64 + nxt).all()
    s32, s64 = wv._mc_levels(prob, h32, 0.95), wv._mc_levels(prob, h64, 0.95)
    ok = np.isfinite(s64)
    assert (np.isfinite(s32) == ok).all() and ok.any()
    assert np.abs(s32[ok] - s64[ok]).max() <= 2e-3


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


def chirp_pair(n, seed=0):
    rs = np.random.RandomState(seed)
    t = np.arange(n) / n
    ph = 2 * np.pi * (50 * t + (n / 8) * t ** 2)
    return np.sin(ph) + 0.5 * rs.randn(n), np.sin(ph + 0.7) + 0.5 * rs.randn(n)


def test_ao_baltic_fixture_fp32(api):
    g = load_golden("ao_baltic_xwt_wct")
    W12 = api.xwt(g["y1"], g["y2"], float(g["dt"]), dj=1 / 12, wavelet=api.Morlet(6), precision='fp32')[0]
    WCT, aWCT = api.wct(g["y1"], g["y2"], float(g["dt"]), dj=1 / 12, sig=False, wavelet="morlet",
                        precision='fp32')[:2]
    assert W12.shape == (76, 147)
    check_fp32_coherence(W12, aWCT, WCT, g["W12"], g["aWCT"], g["WCT"])


def test_chirp_expansion_and_exact_rows_fp32(api, emu):
    """2^13 points, dj = 1/4: dense, several pruned classes and expansion rows in the fp32 plan."""
    a, b = chirp_pair(2 ** 13)
    kw = dict(dj=1 / 4, s0=2.0, J=44)
    W12 = api.xwt(a, b, 1.0, precision='fp32', **kw)[0]
    plan = emu.last_plan(45)
    assert min(plan) < 0 and len({p for p in plan if p > 0}) >= 2, plan
    WCT, aWCT = api.wct(a, b, 1.0, sig=False, precision='f32', **kw)[:2]
    W12r = orc.xwt(a, b, 1.0, **kw)[0]
    WCTr, aWCTr = orc.wct(a, b, 1.0, sig=False, **kw)[:2]
    check_fp32_coherence(W12, aWCT, WCT, W12r, aWCTr, WCTr)


def test_paul_dog_generic_smoothing_fp32(api):
    from pycwt_b200 import mothers
    a, b = chirp_pair(700, seed=3)
    old = mothers.enable_generic_smoothing(True)
    try:
        for mo in (api.Paul(4), api.DOG(2), api.DOG(6)):
            kw = dict(dj=0.25, s0=1.0, J=20, wavelet=mo)
            out = {}
            for p in ('fp64', 'fp32'):
                W12 = api.xwt(a, b, 0.5, precision=p, **kw)[0]
                WCT, aWCT = api.wct(a, b, 0.5, sig=False, precision=p, **kw)[:2]
                out[p] = (W12, aWCT, WCT)
            W12r, aWCTr, WCTr = out['fp64']
            check_fp32_coherence(*out['fp32'], W12r, aWCTr, WCTr)
    finally:
        mothers.enable_generic_smoothing(old)


def _morlet():
    import pycwt_b200
    return pycwt_b200.Morlet(6)


def _mc_geometry():
    """The geometry of test_gpu_xwt_wct.py::test_wct_mc_histogram_vs_oracle."""
    from pycwt_b200 import wavelet as wv
    return wv._mc_problem(1.0, 0.25, 2.0, 24, _morlet())


def test_monte_carlo_host_surrogates_fp32(emu):
    from pycwt_b200 import _engine, wavelet as wv
    prob = _mc_geometry()
    noise = np.random.RandomState(5).randn(3, 2, prob["N"])
    h = {p: wv._mc_histogram(prob, 1.0, 0.25, _morlet(), lambda i: (noise[i, 0], noise[i, 1]),
                             range(3), engine=emu, precision=p) for p in (_engine.F64, _engine.F32)}
    check_fp32_histograms(h[_engine.F32], h[_engine.F64], prob)


def test_monte_carlo_seeded_fp32(emu):
    from pycwt_b200 import _engine, wavelet as wv
    prob = _mc_geometry()
    h = {p: wv._mc_histogram_seeded(prob, 1.0, 0.25, _morlet(), 9, 0, 3, engine=emu, precision=p)
         for p in (_engine.F64, _engine.F32)}
    check_fp32_histograms(h[_engine.F32], h[_engine.F64], prob)


def test_unpadded_mode_runs_fp64(api, emu):
    """No fp32 transforms at a length that is not a power of two: the engine refuses, the public
    API computes in fp64."""
    from pycwt_b200 import _engine, helpers, wavelet as wv
    g = load_golden("ao_baltic_xwt_wct")
    y1, y2, dt = g["y1"], g["y2"], float(g["dt"])
    helpers.set_fft_padding(False)
    try:
        emu.set_padding(False)
        with pytest.raises(_engine.EngineError, match="fp64"):
            emu.xwt(y1, y2, dt, np.array([2.0, 4.0]), 0, 6.0, precision=_engine.F32)
        assert np.array_equal(api.xwt(y1, y2, dt, precision='fp32')[0], api.xwt(y1, y2, dt)[0])
        a = api.wct(y1, y2, dt, sig=False, precision='fp32')
        b = api.wct(y1, y2, dt, sig=False)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        sig = {}
        for p in ('fp32', 'fp64'):
            np.random.seed(4321)
            sig[p] = wv._wct_significance(0.2, 0.1, 1.0, 0.5, 2.0, 10, 0.95, 'morlet', mc_count=2,
                                          progress=False, cache=False, precision=p)
        assert np.array_equal(sig['fp32'], sig['fp64'], equal_nan=True)
    finally:
        helpers.set_fft_padding(True)
        emu.set_padding(True)


def test_explicit_fp64_is_the_default_and_nothing_leaks(api):
    a, b = chirp_pair(3000, seed=1)
    kw = dict(dj=1 / 4, s0=2.0, J=30)
    W0 = api.xwt(a, b, 1.0, **kw)[0]
    W32 = api.xwt(a, b, 1.0, precision='fp32', **kw)[0]
    assert not np.array_equal(W0, W32)
    assert np.array_equal(api.xwt(a, b, 1.0, precision='fp64', **kw)[0], W0)
    assert np.array_equal(api.xwt(a, b, 1.0, **kw)[0], W0)
    c0 = api.wct(a, b, 1.0, sig=False, **kw)
    api.wct(a, b, 1.0, sig=False, precision='float32', **kw)
    c1 = api.wct(a, b, 1.0, sig=False, precision='FP64', **kw)
    assert np.array_equal(c0[0], c1[0]) and np.array_equal(c0[1], c1[1])


def test_bad_precision_spelling(api):
    from pycwt_b200 import distributed as D
    a, b = chirp_pair(256)
    for bad in ('fp16', 'double', 64, None):
        with pytest.raises(ValueError):
            api.xwt(a, b, 1.0, precision=bad)
        with pytest.raises(ValueError):
            api.wct(a, b, 1.0, sig=False, precision=bad)
        with pytest.raises(ValueError):
            api.wct(a, b, 1.0, dj=0.5, s0=2.0, J=4, sig=True, precision=bad, mc_count=1, cache=False)
        with pytest.raises(ValueError):
            D.wct_significance_sharded(0.2, 0.1, 1.0, 0.5, 2.0, 8, mc_count=1, precision=bad)
        with pytest.raises(ValueError):
            D.wct_scale_sharded(a, b, 1.0, dj=0.5, s0=2.0, J=4, precision=bad)


def test_wct_hands_precision_to_significance(api, monkeypatch):
    from pycwt_b200 import wavelet as wv
    seen = {}

    def spy(*args, **kwargs):
        seen.update(kwargs)
        return np.zeros(3)
    monkeypatch.setattr(wv, "_wct_significance", spy)
    a, b = chirp_pair(256)
    api.wct(a, b, 1.0, dj=0.5, s0=2.0, J=4, sig=True, precision='fp32', mc_count=2)
    assert seen["precision"] == 'fp32' and seen["mc_count"] == 2


def _mc_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    from pycwt_b200 import distributed as D, _engine
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        eng = _engine.Engine(0, lib_path=os.path.join(ROOT, "tests", "_emu", "libcwtb200_emu.so"))
        sig = [D.wct_significance_sharded(0.2, 0.1, 1.0, 0.5, 2.0, 8, 0.95, 'morlet', mc_count=5, seed=42,
                                          engine=eng, comm=D.TorchComm(dist), device_rng=rng,
                                          precision='fp32') for rng in (False, True)]
        q.put((rank, [s.tolist() for s in sig]))
        eng.close()
    finally:
        dist.destroy_process_group()


def test_sharded_significance_fp32_gloo():
    """World size 2 gives the fp32 levels of one process running every pair."""
    pytest.importorskip("torch")
    import torch.multiprocessing as mp
    from pycwt_b200 import build as _build, _engine, distributed as D
    eng = _engine.Engine(0, lib_path=_build.build_emulation(os.path.join(ROOT, "tests", "_emu")))
    single = [D.wct_significance_sharded(0.2, 0.1, 1.0, 0.5, 2.0, 8, 0.95, 'morlet', mc_count=5, seed=42,
                                         engine=eng, device_rng=rng, precision='fp32') for rng in (False, True)]
    eng.close()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_mc_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for _, sig in got:
        for k in (0, 1):
            assert np.array_equal(np.array(sig[k]), single[k], equal_nan=True)
