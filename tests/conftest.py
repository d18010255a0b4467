"""pytest configuration: registers the `gpu` marker and shared helpers."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_addoption(parser):
    parser.addoption("--emu", action="store_true", default=False,
                     help="developer aid: run gpu-marked tests against the host-emulation "
                          "build of the kernels (tests/_emu), for debugging test logic "
                          "without a GPU.  Never used by the driver.")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    if config.getoption("--emu"):
        use_emulation_library()


def use_emulation_library():
    """Point the ctypes loader at tests/_emu/libcwtb200_emu.so (same kernel sources,
    compiled with -DCWTB_HOST_EMU so every CTA runs as a C++ loop on the CPU).  This is
    test-side patching: the package itself has no switch for it."""
    from pycwt_b200 import build as _build, _engine
    lib = _build.build_emulation(os.path.join(ROOT, "tests", "_emu"))
    _engine.LIB_PATH = lib
    _engine._default.clear()
    return lib


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)


def relerr(a, ref):
    """max|a - ref| / max|ref| (the parity metric of SURVEY 8d); NaN-pattern must match."""
    a = np.asarray(a)
    ref = np.asarray(ref)
    assert a.shape == ref.shape, (a.shape, ref.shape)
    nan_a, nan_r = np.isnan(a), np.isnan(ref)
    assert (nan_a == nan_r).all(), "NaN pattern differs"
    if nan_r.all():
        return 0.0
    d = np.abs(np.where(nan_r, 0, a - ref)).max()
    m = np.abs(np.where(nan_r, 0, ref)).max()
    return float(d / m) if m > 0 else float(d)


def golden_cwt_kwargs(g):
    kw = {str(k): float(v) for k, v in zip(g["kw_keys"], g["kw_vals"])}
    if "J" in kw:
        kw["J"] = int(kw["J"])
    return kw


@pytest.fixture(scope="session")
def has_cuda():
    try:
        import pycwt_b200._engine as eng
        return eng.device_count() > 0
    except Exception:
        return False
