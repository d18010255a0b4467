"""CPU-only tests: the C-ABI library loads and exports every symbol of include/cwt_b200.h
(no compute calls without a GPU), the product path fails loudly without a device, and the
host-side O(S) logic (scale resolution, NaN-row prediction, significance, helpers) matches
the reference fixtures."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_golden

import pycwt_b200 as pycwt
from pycwt_b200 import _engine, build as _build


def header_symbols():
    txt = open(os.path.join(ROOT, "include", "cwt_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(cwtb_[a-z0-9_]+)\s*\(", txt)))


@pytest.fixture(scope="module")
def lib():
    return _engine.load_library(_build.build())


def test_library_exports_every_declared_symbol(lib):
    syms = header_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(lib, s), "symbol %s declared in include/cwt_b200.h is not exported" % s
    # and the ctypes binding declares a prototype for each of them
    assert set(syms) == set(_engine._SIGNATURES), set(syms) ^ set(_engine._SIGNATURES)
    assert b"sm_90a" in lib.cwtb_version()


def test_no_cpu_fallback_without_device(lib):
    if lib.cwtb_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    with pytest.raises(_engine.EngineError):
        pycwt.cwt(np.random.randn(64), 1.0)
    with pytest.raises(_engine.EngineError):
        pycwt.Morlet().smooth(np.ones((3, 8)), 1.0, 0.25, np.ones(3))


def test_package_never_imports_the_oracle():
    import sys
    src = os.path.join(ROOT, "pycwt_b200")
    for fn in os.listdir(src):
        if fn.endswith(".py"):
            assert "oracle" not in open(os.path.join(src, fn)).read(), fn
    assert not any(m.startswith("oracle") for m in sys.modules
                   if getattr(sys.modules[m], "__file__", "") and "pycwt_b200" in (sys.modules[m].__file__ or ""))


def test_namespace_matches_reference_surface():
    for name in ["cwt", "icwt", "significance", "xwt", "wct", "wct_significance", "Morlet",
                 "Paul", "DOG", "MexicanHat", "ar1", "ar1_spectrum", "rednoise", "find", "fft",
                 "fft_kwargs", "get_cache_dir", "np", "chi2", "tqdm", "helpers", "mothers",
                 "wavelet"]:
        assert hasattr(pycwt, name), name
    assert pycwt.__version__.startswith("0.3.0a22")
    assert callable(pycwt.helpers.boxpdf)  # sample_xwt.py:52 uses pycwt.helpers.boxpdf
    import inspect
    assert str(inspect.signature(pycwt.cwt)) == \
        "(signal, dt, dj=0.08333333333333333, s0=-1, J=-1, wavelet='morlet', freqs=None)"
    assert list(inspect.signature(pycwt.wct).parameters)[:10] == \
        ["y1", "y2", "dt", "dj", "s0", "J", "sig", "significance_level", "wavelet", "normalize"]
    # the reference's parameters in the reference's order; `seed` (device-side surrogates) is an
    # optional trailing extension with a default that keeps the reference behaviour
    params = inspect.signature(pycwt.wct_significance).parameters
    assert list(params) == ["al1", "al2", "dt", "dj", "s0", "J", "significance_level", "wavelet", "mc_count",
                            "progress", "cache", "seed"] and params["seed"].default is None


@pytest.mark.parametrize("name", ["nino3_morlet_tutorial", "nino3_morlet_default",
                                  "nino3_paul_default", "nino3_dog_default", "chirp4000_paul",
                                  "chirp32k_morlet"])
def test_scale_resolution_and_nan_rows_bit_identical(name):
    from pycwt_b200.wavelet import _resolve_scales, _nan_rows
    g = load_golden(name)
    kw = {str(k): float(v) for k, v in zip(g["kw_keys"], g["kw_vals"])}
    mother = {"morlet": pycwt.Morlet, "paul": pycwt.Paul, "dog": pycwt.DOG}[str(g["wavelet"])](int(g["param"]))
    x = g["x"]
    sj, freqs = _resolve_scales(len(x), float(g["dt"]), kw.get("dj", 1 / 12), kw.get("s0", -1),
                                int(kw.get("J", -1)), mother, None)
    npad = pycwt.fft_kwargs(x)["n"]
    keep = ~_nan_rows(mother, sj, npad, float(g["dt"]))
    np.testing.assert_array_equal(sj[keep], g["sj"])
    np.testing.assert_array_equal(freqs[keep], g["freqs"])
    assert keep.sum() == int(g["shape"][0])


def test_mother_wavelet_constants():
    m = pycwt.Morlet(6)
    assert (m.dofmin, m.cdelta, m.gamma, m.deltaj0, m.name) == (2, 0.776, 2.32, 0.60, "Morlet")
    assert pycwt.Morlet(5).cdelta == -1
    p = pycwt.Paul(4)
    assert (p.dofmin, p.cdelta, p.gamma, p.deltaj0) == (2, 1.132, 1.17, 1.50)
    d = pycwt.DOG(2)
    assert (d.dofmin, d.cdelta, d.gamma, d.deltaj0) == (1, 3.541, 1.43, 1.40)
    assert pycwt.DOG(6).cdelta == 1.966 and pycwt.MexicanHat().name == "Mexican Hat"
    assert abs(m.flambda() - 4 * np.pi / (6 + np.sqrt(38))) < 1e-15
    assert abs(p.flambda() - 4 * np.pi / 9) < 1e-15 and abs(d.flambda() - 2 * np.pi / np.sqrt(2.5)) < 1e-15
    assert abs(m.psi_ft(0.0) - np.pi ** -0.25 * np.exp(-18)) < 1e-20
    assert p.psi(0) == pytest.approx(2 ** 4 * 2 / np.sqrt(np.pi * 40320.0))   # reference quirk kept
    assert abs(pycwt.DOG(2).psi(0.0) - 1 / np.sqrt(0.75 * np.sqrt(np.pi))) < 1e-12
    with pytest.raises(KeyError):
        pycwt.wavelet._check_parameter_wavelet("gabor")
    obj = object()
    assert pycwt.wavelet._check_parameter_wavelet(obj) is obj


def test_significance_and_helpers_match_reference():
    g = load_golden("significance_nino3")
    x, sj, alpha = g["x"], g["sj"], float(g["alpha"])
    m = pycwt.Morlet(6)
    np.testing.assert_allclose(np.array(pycwt.ar1(x)), g["ar1_full"], rtol=1e-14)
    s0, f0 = pycwt.significance(1.0, 0.25, sj, 0, alpha, significance_level=0.95, wavelet=m)
    np.testing.assert_allclose(s0, g["s0"], rtol=1e-13)
    np.testing.assert_allclose(f0, g["f0"], rtol=1e-13)
    std = x.std()
    s1, f1 = pycwt.significance(std ** 2, 0.25, sj, 1, alpha, significance_level=0.95,
                                dof=x.size - sj, wavelet=m)
    np.testing.assert_allclose(s1, g["s1"], rtol=1e-13)
    s2, f2 = pycwt.significance(std ** 2, 0.25, sj, 2, alpha, significance_level=0.95,
                                dof=[sj[3], sj[13]], wavelet=m)
    np.testing.assert_allclose(s2, g["s2"], rtol=1e-13)
    np.testing.assert_allclose(f2, g["f2"], rtol=1e-13)
    s3, f3 = pycwt.significance(x / std, 0.25, sj, 0, significance_level=0.9, wavelet="morlet")
    np.testing.assert_allclose(s3, g["s3"], rtol=1e-13)
    with pytest.raises(ValueError):
        pycwt.significance(1.0, 0.25, sj, 3, alpha)
    freqs = 1 / (m.flambda() * sj)
    np.testing.assert_allclose(pycwt.ar1_spectrum(freqs * 0.25, alpha), g["spec"], rtol=1e-14)
    np.testing.assert_array_equal(pycwt.helpers.rect(7, normalize=True), g["rect7"])
    np.testing.assert_array_equal(pycwt.helpers.rect(2), g["rect2"])
    with pytest.raises(Warning):
        pycwt.ar1(np.arange(10.0))      # pure trend: no AR(1) upper bound


def test_rednoise_consumes_rng_like_the_reference():
    np.random.seed(3)
    a = pycwt.rednoise(50, 0.8, 1)
    np.random.seed(3)
    tau = int(np.ceil(-2 / np.log(0.8)))
    b = np.random.randn(50 + tau, 1)[tau:].flatten()
    np.testing.assert_array_equal(a, b)


def test_cache_key_and_dir(tmp_path, monkeypatch):
    monkeypatch.setenv("HOME", str(tmp_path))
    d = pycwt.get_cache_dir()
    assert d == "%s/.cache/pycwt/" % tmp_path and os.path.isdir(d)
    # a cache hit short-circuits the Monte-Carlo loop (no GPU needed)
    aa = np.round(np.arctanh(np.array([0.1, 0.2]) * 4))
    aa = np.abs(aa) + 0.5 * (aa < 0)
    key = "wct_sig_{:0.5f}_{:0.5f}_{:0.5f}_{:0.5f}_{:d}_{}".format(aa[0], aa[1], 0.25, 2.0, 12, "Morlet")
    np.savetxt(os.path.join(d, key + ".gz"), np.arange(13.0))
    out = pycwt.wct_significance(0.1, 0.2, 1.0, 0.25, 2.0, 12, wavelet="morlet", progress=False)
    np.testing.assert_array_equal(out, np.arange(13.0))


def test_header_is_plain_c_and_c_example_links(tmp_path):
    """include/cwt_b200.h compiles as C99 and as C++; the C example links against the engine
    library and fails loudly where no device is present."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = os.path.join(ROOT, "include", "cwt_b200.h")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c", hdr],
                   check=True)
    subprocess.run([shutil.which("g++"), "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-x", "c++", hdr],
                   check=True)
    from pycwt_b200 import build
    lib = build.build()
    exe = str(tmp_path / "c_abi_example")
    subprocess.run([gcc, "-std=c99", "-Wall", "-I" + os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "c_abi_example.c"), "-L" + os.path.dirname(lib),
                    "-l:" + os.path.basename(lib), "-lm", "-Wl,-rpath," + os.path.dirname(lib), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    import pycwt_b200._engine as eng
    try:
        have = eng.device_count() > 0
    except Exception:
        have = False
    if have:
        assert r.returncode == 0 and "kernel launches" in r.stdout
    else:
        assert r.returncode != 0 and "cwtb_create failed" in r.stderr
