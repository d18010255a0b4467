"""CPU: the host formulas of the generalized Morse wavelets (pycwt_b200.mothers.Morse) against
extended-precision quadrature (mpmath), and the parameter handling of the Python surface.

Conventions (DESIGN.md section 1): psi_ft(w) = A w^be exp(-w^ga) for w > 0, unit energy, and
psi(t) = (2 pi)^-1/2 int psi_ft(w) e^(iwt) dw."""
import time

import mpmath
import numpy as np
import pytest

import pycwt_b200 as pycwt
from pycwt_b200 import _engine
from pycwt_b200.mothers import DOG, Morlet, Morse, Paul, time_filter_table
from pycwt_b200.wavelet import _check_parameter_wavelet, _nan_rows

PARAMS = [(3, 20), (1, 1), (1, 4), (2, 2.5), (12, 256), (1, 256), (12, 1), (6, 7.3)]
mpmath.mp.dps = 30


def _psi_ft_mp(mo, w):
    """psi_ft from its definition, A w^be exp(-w^ga), in mpmath."""
    ga, be = mpmath.mpf(mo.ga), mpmath.mpf(mo.be)
    r = (2 * be + 1) / ga
    A = mpmath.sqrt(ga * mpmath.mpf(2) ** r / mpmath.gamma(r))
    return A * w ** be * mpmath.exp(-w ** ga)


def _breaks(mo):
    lo, hi = mo._band(np.log(1e-40))
    return [0] + list(np.linspace(lo, hi, 48))


@pytest.mark.parametrize("ga,be", PARAMS)
def test_unit_energy_and_response(ga, be):
    mo = Morse(ga, be)
    energy = mpmath.quad(lambda w: _psi_ft_mp(mo, w) ** 2, _breaks(mo))
    assert abs(energy - 1) < 1e-12, energy
    lo, hi = mo._band(np.log(1e-12))
    w = np.linspace(lo, hi, 37)
    ref = np.array([float(_psi_ft_mp(mo, mpmath.mpf(v))) for v in w])
    assert np.abs(mo.psi_ft(w) - ref).max() <= 1e-12 * ref.max()
    assert (mo.psi_ft(np.array([-3.0, 0.0])) == 0).all()


@pytest.mark.parametrize("ga,be", PARAMS)
def test_psi_against_quadrature(ga, be):
    """psi(t) within 1e-10 |psi(0)| of the defining integral for |t| <= 10 t_e, psi(0) in closed form."""
    mo = Morse(ga, be)
    te = 1 / mo.coi()
    psi0 = float(mpmath.quad(lambda w: _psi_ft_mp(mo, w), _breaks(mo)) / mpmath.sqrt(2 * mpmath.pi))
    assert abs(mo.psi(0.0) - psi0) <= 1e-12 * psi0
    assert abs(mo._psi0 - psi0) <= 1e-12 * psi0
    ts = np.array([0.1, 0.37, 1.0, 2.2, 3.3, 5.1, 7.7, 9.99]) * te
    ts = np.concatenate([ts, -ts[::3]])
    got = mo.psi(ts)
    for t, g in zip(ts, got):
        ref = complex(mpmath.quad(lambda w: _psi_ft_mp(mo, w) * mpmath.expj(w * t), _breaks(mo))
                      / mpmath.sqrt(2 * mpmath.pi))
        assert abs(g - ref) <= 1e-10 * psi0, (ga, be, t / te, g, ref)
    # e-folding time: |psi(t_e)|^2 / |psi(0)|^2 = e^-2
    assert abs(abs(mo.psi(te)) ** 2 / psi0 ** 2 - np.exp(-2)) < 1e-9
    # beyond the table: finite and decaying
    far = mo.psi(np.array([25, 100, 1e4]) * te)
    assert np.isfinite(far).all() and (np.abs(far) < 0.05 * psi0).all()


@pytest.mark.parametrize("ga,be", PARAMS)
def test_flambda_coi_cdelta(ga, be):
    mo = Morse(ga, be)
    # flambda = 2 pi / x*, x* = s w at the scale s maximising s^(1/2) psi_ft(s w) for a fixed w
    x_star = mpmath.findroot(lambda x: mpmath.diff(lambda u: mpmath.log(mpmath.sqrt(u) * _psi_ft_mp(mo, u)), x),
                             mpmath.mpf(be / ga) ** (1 / mpmath.mpf(ga)))
    assert abs(2 * np.pi / float(x_star) - mo.flambda()) < 1e-10 * mo.flambda()
    # cdelta: sqrt(pi/2) / (ln 2 psi(0)) int_0^inf psi_ft(u) / u du
    integral = mpmath.quad(lambda w: _psi_ft_mp(mo, w) / w, _breaks(mo))
    cd = float(mpmath.sqrt(mpmath.pi / 2) / (mpmath.log(2) * mo._psi0) * integral)
    assert abs(mo.cdelta - cd) <= 1e-10 * cd
    assert mo.dofmin == 2 and mo.gamma == -1 and mo.deltaj0 == -1


def test_published_values():
    mo = Morse()
    assert (mo.ga, mo.be) == (3.0, 20.0)
    assert abs(mo.cdelta - 2.44895) < 1e-5 and abs(mo.flambda() - 3.31107) < 1e-5
    p = Morse(1, 4)
    assert abs(p.cdelta - 1.13309) < 1e-5
    assert abs(p.flambda() - Paul(4).flambda()) < 1e-14
    assert abs(p.coi() - 1 / np.sqrt(np.exp(2 / 5) - 1)) < 1e-10      # 1.426, not Paul's tabulated sqrt(2)
    w = np.linspace(0.01, 30, 1000)
    assert np.abs(p.psi_ft(w) - Paul(4).psi_ft(w)).max() < 1e-14
    assert Morse(2, 3, gamma=1.2, deltaj0=0.7).gamma == 1.2


def _cdelta_identity(wavelet):
    """sqrt(pi/2) / (ln 2 psi(0)) int_0^inf psi_ft(u) / u du, numerically (real part of psi(0))."""
    integral = mpmath.quad(lambda w: float(np.real(wavelet.psi_ft(np.array([float(w)]))[0])) / w,
                           [1e-12, 1, 5, 10, 20, 40, 80])
    return float(np.sqrt(np.pi / 2) / (np.log(2) * abs(wavelet.psi(0.0))) * integral)


def test_cdelta_identity_on_tc98_families():
    """The closed form's identity applied to Morlet(6) and to Paul(4) with the correct psi(0) (Morse(1, 4))
    lands within 1 % of Torrence & Compo's 0.776 and 1.132."""
    assert abs(_cdelta_identity(Morlet(6)) / 0.776 - 1) < 0.01
    assert abs(_cdelta_identity(Morse(1, 4)) / 1.132 - 1) < 0.01


def test_large_be_has_no_nan():
    for mo in (Morse(1, 256), Morse(12, 256), Morse(3, 256)):
        f = np.concatenate([[0.0, 1e-300, 1e-30], np.geomspace(1e-3, 1e3, 500), [1e30, 1e300, np.inf]])
        v = mo.psi_ft(f)
        assert np.isfinite(v).all() and (v >= 0).all()
        sj = 0.25 * 2 ** (np.arange(0, 120) / 4)
        assert not _nan_rows(mo, sj, 2 ** 16, 0.25).any()


def test_parameters():
    for ga, be in ((0.5, 20), (13, 20), (3, 0.5), (3, 257)):
        with pytest.raises(ValueError):
            Morse(ga, be)
    mo = _check_parameter_wavelet('morse')
    assert isinstance(mo, Morse) and (mo.ga, mo.be) == (3.0, 20.0)
    assert pycwt.Morse is Morse and 'Morse' not in pycwt.__all__
    assert mo._engine_spec() == (_engine.MORSE, (20.0, 3.0))

    class Custom(Morse):
        def psi_ft(self, f):
            return Morse.psi_ft(self, f)
    assert Custom()._engine_spec() is None


def test_time_filter_table_speed():
    """psi is fast enough for the smoothing filter of coherence: the table at 145 scales x 65536 points
    within twice DOG's time (best of three each, a fresh object per Morse run)."""
    sj = 0.5 * 2 ** (np.arange(145) / 12)

    def best(make):
        out = []
        for _ in range(3):
            t0 = time.perf_counter()
            time_filter_table(make(), sj, 0.25, 65536)
            out.append(time.perf_counter() - t0)
        return min(out)
    t_dog, t_morse = best(lambda: DOG(2)), best(lambda: Morse())
    print("time_filter_table: DOG(2) %.3f s, Morse(3, 20) %.3f s" % (t_dog, t_morse))
    assert t_morse <= 2 * t_dog
