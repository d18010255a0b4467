"""The engine's host control flow on the host-emulation build: the paths that decide what runs on
which stream, and when copies start, are the device's own.  Streams and events are inert there
(every launch runs in issue order), so each check shows through the profile or the launch count
that its path ran, and that the result is the one of the serial path.

  * the stream graph of one transform (CWTB_PRIO x CWTB_CHAINS): overlapped copy, transform then
    fetch and a profiled (serial) run are bit-identical in every configuration;
  * the pipelined channel batch (CWTB_BATCH_PIPELINE) equals the chunk-after-chunk path;
  * the phase angle of `wct`, copied while the smoothing runs, equals the resident one;
  * the profile lists every launch of a call;
  * device-drawn surrogates of more units than one launch has rows.
"""
import numpy as np
import pytest

from test_emu_overlap_save import emu_lib, make_engine
from pycwt_b200 import _engine

MORLET, F64, F32 = _engine.MORLET, _engine.F64, _engine.F32
OS = -2
GRAPH_N0 = 2 ** 16 - 5
# exact rows of K' = 2^14, 2^15 and dense ones (CWTB_DENSE_MARGIN=0), overlap-save rows, and expansion
# rows with coarse grids up to and above 1024 points
GRAPH_SJ = np.concatenate([2.0 * 2 ** (np.arange(0, 30) / 4.0), 400.0 * 2 ** np.arange(0, 8)])
GRAPH_ENV = dict(CWTB_EXPAND_MIN_R="2", CWTB_DENSE_MARGIN="0")


def _engine_with(**env):
    eng = make_engine(emu_lib(), **env)
    assert "emulation" in eng.version()
    return eng


def _total_launches(prof):
    return sum(p["launches"] for p in prof)


def _graph_run(eng, x, expand):
    if not expand:
        eng.set_expand_eps(0.0, 0.0)
    try:
        s0 = eng.job_serial()
        W1 = eng.cwt(x, 1.0, GRAPH_SJ, MORLET, 6.0)
        # one plan: cwtb_cwt_to_host took its early-copy path (the fall-back plans a second time)
        assert eng.job_serial() == s0 + 1
        plan = eng.last_plan(len(GRAPH_SJ))
        eng.cwt(x, 1.0, GRAPH_SJ, MORLET, 6.0, fetch=False)
        W2 = eng.get_w(len(GRAPH_SJ), x.size)
        launches = eng.last_launch_count()
        eng.profile_begin()
        try:
            eng.cwt(x, 1.0, GRAPH_SJ, MORLET, 6.0, fetch=False)
        finally:
            prof = eng.profile_end()
        W3 = eng.get_w(len(GRAPH_SJ), x.size)
    finally:
        eng.set_expand_eps()
    assert np.array_equal(W1, W2) and np.array_equal(W1, W3)
    assert _total_launches(prof) == launches, (launches, prof)
    return plan, prof, W1


@pytest.fixture(scope="module")
def graph_signal():
    return np.random.RandomState(8).randn(GRAPH_N0)


@pytest.fixture(scope="module")
def graph_serial(graph_signal):
    """W of the three plans with every launch on the engine's stream (CWTB_PRIO=0, CWTB_CHAINS=1)."""
    out = {}
    for os_on in (1, 0):
        eng = _engine_with(CWTB_OS=str(os_on), CWTB_PRIO="0", CWTB_CHAINS="1", **GRAPH_ENV)
        try:
            for expand in ((True, False) if os_on else (True,)):
                out[os_on, expand] = _graph_run(eng, graph_signal, expand)
        finally:
            eng.close()
    return out


def test_graph_plans(graph_serial):
    """The geometry has what the stream graph forks over."""
    log2N = 16
    plan, prof, _ = graph_serial[1, True]
    assert OS in plan and log2N in plan, plan
    assert any(-10 <= p < -2 for p in plan) and any(p < -10 for p in plan), plan
    names = " ".join(p["name"] for p in prof)
    for k in ("fwd:", "coarse:CoarseABody", "coarse:CoarseRowsBody", "ExpandBody<double", "OsBody"):
        assert k in names, (k, names)
    plan, _, _ = graph_serial[0, True]
    assert {14, 15, log2N} <= set(plan), plan      # three chain classes
    plan, _, _ = graph_serial[1, False]
    assert {14, 15, log2N} <= set(plan) and any(0 < p <= 10 for p in plan) and any(10 < p <= 13 for p in plan), plan


@pytest.mark.parametrize("chains", [1, 2, 3, 4])
@pytest.mark.parametrize("prio", [0, 1, 2])
def test_stream_graph(graph_signal, graph_serial, prio, chains):
    for os_on in (1, 0):
        eng = _engine_with(CWTB_OS=str(os_on), CWTB_PRIO=str(prio), CWTB_CHAINS=str(chains), **GRAPH_ENV)
        try:
            for expand in ((True, False) if os_on else (True,)):
                plan, prof, W = _graph_run(eng, graph_signal, expand)
                ref_plan, ref_prof, ref_W = graph_serial[os_on, expand]
                assert plan == ref_plan and prof == ref_prof
                assert np.array_equal(W, ref_W), (prio, chains, os_on, expand)
        finally:
            eng.close()


BATCH_N0 = 2001                                    # Np = 2048
BATCH_SJ = 2.0 * 2 ** (np.arange(0, 16) / 2.0)


@pytest.mark.parametrize("precision,in_dtype", [(F64, np.float64), (F64, np.float32), (F32, np.float32),
                                                (F32, np.float64)])
def test_batch_pipeline_equals_synchronous_chunks(precision, in_dtype):
    """7 channels in chunks of 1 MiB of coefficients (CWTB_BATCH_MB=1): 2 channels (fp64) or 4 (fp32),
    a short last chunk."""
    X = np.random.RandomState(3).randn(7, BATCH_N0).astype(in_dtype)
    per_chunk = (1 << 20) // ((16 if precision == F64 else 8) * BATCH_N0 * BATCH_SJ.size)
    chunks = -(-7 // per_chunk)
    assert per_chunk in (2, 4) and 7 % per_chunk
    out = {}
    for pipeline in (1, 0):
        eng = _engine_with(CWTB_BATCH_MB="1", CWTB_BATCH_PIPELINE=str(pipeline))
        try:
            eng.profile_begin()
            try:
                out[pipeline], _ = eng.cwt_batch(X, 1.0, BATCH_SJ, MORLET, 6.0, precision, want_power=True)
            finally:
                prof = eng.profile_end()
            power_launches = sum(p["launches"] for p in prof if p["name"].startswith("PowerBody"))
            assert power_launches == chunks, prof
            # the pipeline counts the launches of the whole batch, the chunk loop those of its last chunk
            if pipeline:
                assert eng.last_launch_count() == _total_launches(prof), prof
            else:
                assert eng.last_launch_count() < _total_launches(prof) / 2, prof
        finally:
            eng.close()
    assert out[1].shape == (7, BATCH_SJ.size) and np.isfinite(out[1]).all()
    assert np.array_equal(out[1], out[0])


@pytest.mark.parametrize("precision", [F64, F32])
def test_wct_angle_copied_early_equals_resident(precision):
    rs = np.random.RandomState(4)
    n0 = 3000
    t = np.arange(n0)
    y1 = np.sin(2 * np.pi * t / 50.0) + rs.randn(n0)
    y2 = np.sin(2 * np.pi * t / 50.0 + 1.0) + rs.randn(n0)
    sj = 2.0 * 2 ** (np.arange(0, 40) / 6.0)
    eng = _engine_with()
    try:
        WCT, A = eng.wct(y1, y2, 1.0, 1 / 6, sj, MORLET, 6.0, 3, precision=precision)
        eng.wct_resident(y1, y2, 1.0, 1 / 6, sj, MORLET, 6.0, 3, precision=precision)
        Wr, Ar = eng.coherence_window(0, sj.size, 1, 0, n0, 1)
    finally:
        eng.close()
    assert np.isfinite(A).all() and np.abs(A).max() > 0
    assert np.array_equal(A, Ar) and np.array_equal(WCT, Wr)


def test_profile_lists_every_launch():
    x = np.random.RandomState(5).randn(5000)
    sj = 2.0 * 2 ** (np.arange(0, 40) / 4.0)
    eng = _engine_with()
    try:
        eng.cwt(x, 1.0, sj, MORLET, 6.0, fetch=False)
        prof = eng.profile_last()
        assert prof and all(p["ms"] == 0.0 and p["rows"] >= p["launches"] > 0 for p in prof), prof
        assert _total_launches(prof) == eng.last_launch_count(), prof
        assert any(p["name"].startswith("fwd:") for p in prof), prof
        # any sequence of calls: an xwt's two transforms and their epilogues
        eng.profile_begin()
        try:
            eng.xwt(x, x[::-1].copy(), 1.0, sj, MORLET, 6.0)
        finally:
            prof2 = eng.profile_end()
        assert _total_launches(prof2) >= 2 * _total_launches(prof), (prof, prof2)
    finally:
        eng.close()


SHORT_N0 = 24


def test_surrogates_of_more_units_than_one_launch_has_rows():
    """40000 units of 2 or 3 series are more rows than one launch takes (65535): drawn in batches,
    they equal two calls of 20000 units each."""
    series = np.random.RandomState(6).randn(3, SHORT_N0)
    eng = _engine_with()
    try:
        for draw in (lambda u0, n: eng.mc_surrogates(11, u0, n, SHORT_N0),
                     lambda u0, n: eng.mc_surrogates3(11, u0, n, SHORT_N0),
                     lambda u0, n: eng.mc_phase_surrogates(series[:2], [0, 0], 11, u0, n),
                     lambda u0, n: eng.mc_phase_surrogates(series, [0, 0, 1], 11, u0, n)):
            whole = draw(0, 40000)
            assert np.array_equal(whole, np.concatenate([draw(0, 20000), draw(20000, 20000)]))
    finally:
        eng.close()
