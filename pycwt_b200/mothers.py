"""Mother-wavelet objects with the interface of pycwt/mothers.py (reference
file:line cited per method).  They are parameter carriers for the CUDA engine plus the
small closed-form host formulas user code calls directly (flambda, coi, psi, psi_ft)."""
import numpy as np
from numpy.polynomial import hermite_e as _hermite_e
from scipy.special import gamma as _gamma
from scipy.special import gammaln as _gammaln

from . import _engine


#: Opt-in (SURVEY 8f rank 4): a smoothing operator for Paul and DOG.  The reference defines
#: `smooth` for Morlet only (mothers.py:61-104; `wct` with Paul/DOG raises AttributeError there,
#: and here while this is off).  When on, Paul/DOG objects expose `smooth` with the general
#: definition of Torrence & Webster (1999) / TC98 sec. 6 that Morlet's Gaussian is the special
#: case of: in time a filter given by the absolute value of the wavelet function at each scale,
#: normalised to unit weight; in scale a boxcar of width deltaj0 (TC98 table 2).
_GENERIC_SMOOTHING = False


def enable_generic_smoothing(on=True):
    """Give Paul and DOG a `smooth` method (see `_GENERIC_SMOOTHING`); returns the old setting."""
    global _GENERIC_SMOOTHING
    old, _GENERIC_SMOOTHING = _GENERIC_SMOOTHING, bool(on)
    return old


def time_filter_table(wavelet, scales, dt, npad):
    """Real frequency responses [S, npad] of the time smoothing |psi0(t/s)| / sum: the DFT of the
    wavelet modulus sampled on the circular grid of `npad` points (for Morlet this is the sampled
    counterpart of the Gaussian exp(-0.5 (s/dt)^2 k^2) of mothers.py:83-91)."""
    n = np.arange(npad)
    t = dt * np.where(n <= npad // 2, n, n - npad)
    out = np.empty((len(scales), npad))
    for j, s in enumerate(np.asarray(scales, dtype=float)):
        k = np.abs(wavelet.psi(t / s))
        out[j] = np.fft.fft(k / k.sum()).real
    return out


class _Base(object):
    #: engine family id and the attribute holding its parameter
    _family = None
    cdelta = -1
    gamma = -1
    deltaj0 = -1

    @property
    def smooth(self):
        """Only with `enable_generic_smoothing()`: see `_GENERIC_SMOOTHING`."""
        if not _GENERIC_SMOOTHING:
            raise AttributeError("'{}' object has no attribute 'smooth'".format(type(self).__name__))
        return self._smooth_generic

    def _smooth_generic(self, W, dt, dj, scales):
        from .wavelet import _smooth_device
        return _smooth_device(W, dt, dj, scales, self.deltaj0, wavelet=self)

    def _engine_spec(self):
        """(family, param) if the engine evaluates this wavelet analytically, else None."""
        return None

    def sup(self):
        """Wavelet support defined by the e-folding time (reference mothers.py:42-44
        divides by the bound method and raises TypeError; here it is evaluated)."""
        return 1.0 / self.coi()


class Morlet(_Base):
    """Morlet wavelet, angular wavenumber f0 (reference mothers.py:13-104)."""

    def __init__(self, f0=6):
        self._set_f0(f0)
        self.name = 'Morlet'

    def psi_ft(self, f):
        # mothers.py:26-28: two-sided, no Heaviside step
        return np.pi ** -0.25 * np.exp(-0.5 * (f - self.f0) ** 2)

    def psi(self, t):
        # mothers.py:30-32
        return np.pi ** -0.25 * np.exp(1j * self.f0 * t - t ** 2 / 2)

    def flambda(self):
        # mothers.py:34-36
        return (4 * np.pi) / (self.f0 + np.sqrt(2 + self.f0 ** 2))

    def coi(self):
        # mothers.py:38-40
        return 1. / np.sqrt(2)

    def _set_f0(self, f0):
        # Torrence & Compo (1998) table 2; mothers.py:46-59
        self.f0 = f0
        self.dofmin = 2
        if self.f0 == 6:
            self.cdelta, self.gamma, self.deltaj0 = 0.776, 2.32, 0.60
        else:
            self.cdelta = self.gamma = self.deltaj0 = -1

    def _engine_spec(self):
        if type(self).psi_ft is not Morlet.psi_ft:
            return None
        return _engine.MORLET, float(self.f0)

    def smooth(self, W, dt, dj, scales):
        """Coherence smoothing operator (mothers.py:61-104): Gaussian in time per scale
        (FFT, zero-padded to the next power of two) then a boxcar of width
        2*deltaj0/dj with half-weight end taps along the scale axis.  Runs on the GPU."""
        from .wavelet import _smooth_device
        return _smooth_device(W, dt, dj, scales, self.deltaj0)


class Paul(_Base):
    """Paul wavelet of order m (reference mothers.py:107-155)."""

    def __init__(self, m=4):
        self._set_m(m)
        self.name = 'Paul'

    def psi_ft(self, f):
        # mothers.py:118-122; for f < -709.78 exp overflows and inf*0 gives NaN
        m = self.m
        return (2 ** m / np.sqrt(m * np.prod(range(2, 2 * m))) *
                f ** m * np.exp(-f) * (f > 0))

    def psi(self, t):
        # mothers.py:124-128 (keeps the reference's prod(range(2, m-1)) factor)
        m = self.m
        return (2 ** m * 1j ** m * np.prod(range(2, m - 1)) /
                np.sqrt(np.pi * np.prod(range(2, 2 * m + 1))) *
                (1 - 1j * t) ** (-(m + 1)))

    def flambda(self):
        # mothers.py:130-132
        return 4 * np.pi / (2 * self.m + 1)

    def coi(self):
        # mothers.py:134-136
        return np.sqrt(2)

    def _set_m(self, m):
        # mothers.py:142-155
        self.m = m
        self.dofmin = 2
        if self.m == 4:
            self.cdelta, self.gamma, self.deltaj0 = 1.132, 1.17, 1.50
        else:
            self.cdelta = self.gamma = self.deltaj0 = -1

    def _engine_spec(self):
        if type(self).psi_ft is not Paul.psi_ft or int(self.m) != self.m or not 1 <= self.m <= 64:
            return None
        return _engine.PAUL, float(self.m)


class DOG(_Base):
    """m-th derivative of a Gaussian (reference mothers.py:158-222)."""

    def __init__(self, m=2):
        self._set_m(m)
        self.name = 'DOG'

    def psi_ft(self, f):
        # mothers.py:170-173; note -(1j**m): the minus applies after the power
        return (- 1j ** self.m / np.sqrt(_gamma(self.m + 0.5)) * f ** self.m *
                np.exp(- 0.5 * f ** 2))

    def psi(self, t):
        # mothers.py:175-191: probabilists' Hermite polynomial He_m
        he = _hermite_e.hermeval(t, [0] * int(self.m) + [1])
        return ((-1) ** (self.m + 1) * he * np.exp(-t ** 2 / 2) /
                np.sqrt(_gamma(self.m + 0.5)))

    def flambda(self):
        # mothers.py:193-195
        return 2 * np.pi / np.sqrt(self.m + 0.5)

    def coi(self):
        # mothers.py:197-199
        return 1 / np.sqrt(2)

    def _set_m(self, m):
        # mothers.py:205-222
        self.m = m
        self.dofmin = 1
        if self.m == 2:
            self.cdelta, self.gamma, self.deltaj0 = 3.541, 1.43, 1.40
        elif self.m == 6:
            self.cdelta, self.gamma, self.deltaj0 = 1.966, 1.37, 0.97
        else:
            self.cdelta = self.gamma = self.deltaj0 = -1

    def _engine_spec(self):
        if type(self).psi_ft is not DOG.psi_ft or int(self.m) != self.m or not 1 <= self.m <= 64:
            return None
        return _engine.DOG, float(self.m)


class Morse(_Base):
    """Generalized Morse wavelet (Olhede & Walden 2002; Lilly & Olhede 2009, 2012), zero order:
    psi_ft(w) = A w^be exp(-w^ga) for w > 0 and 0 otherwise, unit energy
    (A = sqrt(ga 2^((2be+1)/ga) / Gamma((2be+1)/ga))).  ga sets the shape, be the time-frequency
    trade-off; Morse(3, 20) (time-bandwidth product ga*be = 60) is the default wavelet of MATLAB's
    cwt, and Morse(1, m) is Paul(m).  Accepts 1 <= ga <= 12 and 1 <= be <= 256.

    Torrence & Compo's empirical `gamma` and `deltaj0` have no closed form here: they are -1 unless
    given, so coherence needs `enable_generic_smoothing()` and a `deltaj0`."""

    def __init__(self, ga=3, be=20, gamma=None, deltaj0=None):
        if not (1 <= ga <= 12 and 1 <= be <= 256):
            raise ValueError('Morse needs 1 <= ga <= 12 and 1 <= be <= 256, got ga=%r, be=%r' % (ga, be))
        self.ga, self.be = float(ga), float(be)
        self.name = 'Morse'
        self.dofmin = 2
        self.gamma = -1 if gamma is None else gamma
        self.deltaj0 = -1 if deltaj0 is None else deltaj0
        ga, be = self.ga, self.be
        r = (2 * be + 1) / ga
        self._lnA = 0.5 * (np.log(ga) + r * np.log(2.0) - _gammaln(r))
        self._bg = be / ga                          # f_p^ga
        self._lnfp = np.log(self._bg) / ga          # ln f_p, f_p = (be/ga)^(1/ga) the peak
        self._lnpk = self._lnA + be * self._lnfp - self._bg   # ln psi_ft(f_p)
        # psi(0) = A Gamma((be+1)/ga) / (ga sqrt(2 pi)); cdelta = (pi / ln 2) Gamma(be/ga) / Gamma((be+1)/ga),
        # the reconstruction constant of icwt for an analytic wavelet:
        # sqrt(pi/2) / (ln 2 psi(0)) * int_0^inf psi_ft(u) / u du in closed form
        self._psi0 = np.exp(self._lnA + _gammaln((be + 1) / ga)) / (ga * np.sqrt(2 * np.pi))
        self.cdelta = np.pi / np.log(2) * np.exp(_gammaln(be / ga) - _gammaln((be + 1) / ga))
        self._table = None
        self._te = self._efold_time()

    def psi_ft(self, f):
        # peak-relative log form: f^be and exp(-f^ga) are never formed apart, so no inf * 0
        f = np.asarray(f, dtype=float)
        with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
            u = np.log(np.where(f > 0, f, 1.0)) - self._lnfp
            v = np.exp(self._lnpk + self.be * u - self._bg * np.expm1(self.ga * u))
        return np.where((f > 0) & (f < np.inf), v, 0.0)

    def flambda(self):
        # the scale maximising s^(1/2) psi_ft(s w): w s = ((be + 1/2) / ga)^(1/ga)
        return 2 * np.pi / ((self.be + 0.5) / self.ga) ** (1 / self.ga)

    def coi(self):
        # Torrence & Compo's e-folding time: |psi(t_e)|^2 / |psi(0)|^2 = e^-2 (Morlet's 1/sqrt(2)
        # follows from it exactly; for ga = 1 it is 1/sqrt(e^(2/(be+1)) - 1), not Paul's tabulated sqrt(2))
        return 1.0 / self._te

    def psi(self, t):
        """psi(t) = (2 pi)^-1/2 int_0^inf psi_ft(w) e^(iwt) dw: quintic Hermite interpolation of psi,
        psi' and psi'' tabulated by quadrature on |t| <= 20 t_e (within 1e-10 |psi(0)|), the
        three-term asymptotic series of the small-w behaviour of psi_ft beyond."""
        if self._table is None:
            self._table = self._build_table()
        h, tmax, cr, ci = self._table
        t = np.asarray(t, dtype=float)
        a = np.abs(t)
        inside = a < tmax
        v = np.empty(a.shape, dtype=complex)
        if inside.all():
            v[...] = self._interp(a, h, cr, ci)
        else:
            v[inside] = self._interp(a[inside], h, cr, ci)
            v[~inside] = self._psi_tail(a[~inside])
        np.conjugate(v, out=v, where=t < 0)     # psi_ft is real: psi(-t) = conj(psi(t))
        return v

    @staticmethod
    def _interp(a, h, cr, ci):
        x = a * (1.0 / h)
        i = x.astype(np.intp)
        s = x - i
        vr, vi = cr[5].take(i), ci[5].take(i)
        for k in range(4, -1, -1):
            vr *= s
            vr += cr[k].take(i)
            vi *= s
            vi += ci[k].take(i)
        return vr + 1j * vi

    # ---- numerics of psi ---------------------------------------------------------------
    def _band(self, lneps):
        """The two roots in f of ln(psi_ft(f) / psi_ft(f_p)) = lneps (bisection in u = ln(f/f_p))."""
        be, ga, bg = self.be, self.ga, self._bg

        def g(u):
            with np.errstate(over='ignore'):
                return be * u - bg * np.expm1(ga * u)
        lo, hi = (lneps - bg) / be, 0.0
        for _ in range(200):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if g(mid) < lneps else (lo, mid)
        ulo, lo, hi = lo, 0.0, 1.0
        while g(hi) > lneps:
            hi *= 2
        for _ in range(200):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if g(mid) > lneps else (lo, mid)
        return np.exp(ulo + self._lnfp), np.exp(hi + self._lnfp)

    def _nodes(self, tmax):
        """Gauss-Legendre nodes and weights of int_0^inf dw for |t| <= tmax: panels of at most
        12 / tmax (24 nodes resolve e^(iwt) over 6 rad either side to rounding) on the band above 1e-20 of the
        peak, graded geometrically towards w = 0 where w^be is not smooth for fractional be."""
        flo, fhi = self._band(np.log(1e-20))
        width = min(12.0 / max(tmax, 1e-300), (fhi - flo) / 8)
        edges = [np.arange(flo, fhi, width), [fhi]]
        if flo < width:     # psi_ft reaches 1e-20 only within the first panel: grade it towards 0
            first = min(width, fhi)
            edges = [first * 2.0 ** -np.arange(40, 0, -1), np.arange(first, fhi, width), [fhi]]
        e = np.unique(np.concatenate(edges))
        x, w = np.polynomial.legendre.leggauss(24)
        a, b = e[:-1, None], e[1:, None]
        nodes = (0.5 * (b - a) * x + 0.5 * (b + a)).ravel()
        weights = (0.5 * (b - a) * w).ravel()
        return nodes, weights * self.psi_ft(nodes) / np.sqrt(2 * np.pi)

    def _psi_quad(self, t, orders=(0,), step=None):
        """psi^(q)(t) for q in `orders` by direct quadrature, t >= 0, [len(orders), len(t)].  With
        `step` the t are step * (0, 1, 2, ...): e^(iwt) of a block of 64 rows is then one row's
        exponential times a table shared by every block, not 64 rows of exponentials."""
        t = np.atleast_1d(np.asarray(t, dtype=float))
        w, c = self._nodes(np.abs(t).max())
        rhs = np.stack([c * (1j * w) ** q for q in orders], axis=1)
        out = np.empty((len(orders), t.size), dtype=complex)
        B = 64
        steps = None if step is None else np.exp(1j * np.outer(np.arange(B) * step, w))
        for j in range(0, t.size, B):
            if steps is None:
                e = np.exp(1j * np.outer(t[j:j + B], w))
            else:
                e = steps[:t.size - j] * np.exp(1j * t[j] * w)
            out[:, j:j + B] = (e @ rhs).T
        return out

    def _efold_time(self):
        """t_e with |psi(t_e)|^2 / |psi(0)|^2 = e^-2: the first crossing, bracketed on a doubling grid
        and refined by bisection."""
        ratio = lambda t: abs(self._psi_quad([t])[0, 0]) / self._psi0 - np.exp(-1)  # noqa: E731
        lo, hi = 0.0, 0.25 / np.exp(self._lnfp)
        while ratio(hi) > 0:
            lo, hi = hi, 2 * hi
        for _ in range(60):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if ratio(mid) > 0 else (lo, mid)
        return 0.5 * (lo + hi)

    def _build_table(self):
        # step 0.08 / f_hi: the quintic Hermite error is below (f_hi h)^6 / 46080 |psi(0)| ~ 6e-12 |psi(0)|
        _, fhi = self._band(np.log(1e-20))
        h = 0.08 / fhi
        tmax = 20 * self._te
        t = np.arange(int(np.ceil(tmax / h)) + 2) * h
        P = self._psi_quad(t, orders=(0, 1, 2), step=h)
        # per interval the quintic Hermite polynomial in s = t/h - i through psi, h psi', h^2 psi'' at
        # both ends, as coefficients of s^0 .. s^5 (real and imaginary parts apart)
        p0, p1 = P[0, :-1], P[0, 1:]
        d0, d1 = h * P[1, :-1], h * P[1, 1:]
        e0, e1 = h * h * P[2, :-1], h * h * P[2, 1:]
        dp = p1 - p0
        c = np.stack([p0, d0, 0.5 * e0,
                      10 * dp - 6 * d0 - 4 * d1 - 1.5 * e0 + 0.5 * e1,
                      -15 * dp + 8 * d0 + 7 * d1 + 1.5 * e0 - e1,
                      6 * dp - 3 * d0 - 3 * d1 - 0.5 * e0 + 0.5 * e1])
        return h, t[-2], np.ascontiguousarray(c.real), np.ascontiguousarray(c.imag)

    def _psi_tail(self, a):
        # psi(t) ~ (2 pi)^-1/2 A sum_k (-1)^k / k! Gamma(p_k) (-i t)^-p_k, p_k = be + 1 + k ga, t > 0
        out = np.zeros(np.shape(a), dtype=complex)
        la = np.log(a)    # (a > 20 t_e > 0)
        for k in range(3):
            p = self.be + 1 + k * self.ga
            mag = np.exp(self._lnA + _gammaln(p) - _gammaln(k + 1) - p * la) / np.sqrt(2 * np.pi)
            out += (-1) ** k * mag * np.exp(0.5j * np.pi * p)
        return out

    def _engine_spec(self):
        if type(self).psi_ft is not Morse.psi_ft:
            return None
        return _engine.MORSE, (self.be, self.ga)


class MexicanHat(DOG):
    """DOG with m = 2 (reference mothers.py:225-233)."""

    def __init__(self):
        self.name = 'Mexican Hat'
        self._set_m(2)
