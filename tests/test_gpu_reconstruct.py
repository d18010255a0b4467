"""Tests of the reconstruction over a selection on the GPU.

The checks of test_emu_reconstruct.py on the device; then config 4's first series (n0 = 2^18,
145 scales), fp64 and fp32, and config 2's geometry (2^20 x 256), fp64, in every mode against the
longdouble restatement with W read back in row blocks; last, the burst in red noise given back.
"""
import numpy as np
import pytest

import test_emu_power_test as E
import test_emu_reconstruct as R
from test_gpu_surrogate_pvalues import eng, api  # noqa: F401  (fixtures)


def _unpad_after(fn, *a):
    from pycwt_b200 import helpers
    try:
        fn(*a)
    finally:
        helpers.set_fft_padding(True)


@pytest.mark.gpu
@pytest.mark.parametrize("null,prec,wav,n0,padded", E.CASES)
def test_definition(api, eng, null, prec, wav, n0, padded):
    _unpad_after(R.test_definition, api, eng, None, null, prec, wav, n0, padded)


@pytest.mark.gpu
@pytest.mark.parametrize("null,prec,wav,n0,padded", E.CASES[:4])
def test_additivity(api, eng, null, prec, wav, n0, padded):
    _unpad_after(R.test_additivity, api, eng, None, null, prec, wav, n0, padded)


@pytest.mark.gpu
@pytest.mark.parametrize("null,prec,wav,n0,padded", E.CASES)
def test_full_selection_is_icwt(api, eng, monkeypatch, null, prec, wav, n0, padded):
    _unpad_after(R.test_full_selection_is_icwt, api, eng, None, monkeypatch, null, prec, wav, n0, padded)


@pytest.mark.gpu
def test_repeated_calls_move_nothing(api, eng):
    R.test_repeated_calls_move_nothing(api, eng)


@pytest.mark.gpu
@pytest.mark.parametrize("prec,wav", [('fp64', 'morlet'), ('fp32', 'paul'), ('fp64', 'dog')])
def test_powers_of_two(api, eng, prec, wav):
    R.test_powers_of_two(api, eng, prec, wav)


@pytest.mark.gpu
def test_errors(api, eng):
    _unpad_after(R.test_errors_python, api, eng, None)
    R.test_errors_c(api, eng)


@pytest.mark.gpu
def test_band_gives_back_its_tone(api, eng):
    R.test_band_gives_back_its_tone(api, eng)


@pytest.mark.gpu
def test_burst_given_back(api, eng):
    R.test_burst_given_back(api, eng)


def _check_geometry(api, h, y, null):
    """Every mode against the restatement, W read back 16 rows at a time."""
    sig = api.significance(1.0, h.dt, h.scales, 0, api.ar1(y)[0])[0]
    h.surrogate_test(mc_count=3, seed=5, null=null)
    res = h.cluster_test(sig, mc_count=3, seed=6, null=null)
    per = h.period
    S = len(per)
    quarter = (float(per[3 * S // 8]), float(per[5 * S // 8]))
    modes = [{}, dict(period_min=quarter[0], period_max=quarter[1]), dict(inside_coi=True, signif=sig),
             dict(alpha=0.5), dict(inside_coi=True, signif=sig, alpha=0.5),
             dict(cluster=list(range(min(3, len(res.area)))))]
    for mode, (ref, bound) in zip(modes, R.restate(h, modes, block=16)):
        R.check(h.reconstruct(**mode), ref, bound, (h.shape, h.precision, mode))
    print("  %s %s: %d clusters" % (h.shape, h.precision, len(res.area)))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ['fp64', 'fp32'])
def test_config4(api, prec):
    import workloads as wl
    c = wl.C4
    y = wl.config4_signals()[0]
    h = api.power_resident(y, c["dt"], dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=api.Morlet(c["f0"]),
                           precision=prec)
    assert h.shape == (145, 2 ** 18)
    _check_geometry(api, h, y, 'ar1' if prec == 'fp64' else 'phase')


@pytest.mark.gpu
def test_config2(api):
    import workloads as wl
    c = wl.C2
    y = wl.config2_signal()
    h = api.power_resident(y, c["dt"], dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=api.Morlet(c["f0"]))
    assert h.shape == (256, 2 ** 20)
    _check_geometry(api, h, y, 'ar1')
