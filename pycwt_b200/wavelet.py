"""Continuous wavelet transform API with the signatures of pycwt/wavelet.py, executed by
the H100 CUDA engine (pycwt_b200/csrc, C ABI in include/cwt_b200.h).

Division of labour (SURVEY 8a):
  * O(S) scalar work -- scale resolution, cone of influence, chi-square significance,
    NaN-row bookkeeping -- stays in NumPy on the host, written so that `sj`, `freqs` and
    `coi` are bit-identical to the reference's;
  * everything that touches an [S, N] array -- forward FFT, analytic wavelet response,
    per-scale inverse transforms, cross products, smoothing, coherence, Monte-Carlo
    histograms, the icwt reduction -- runs on the GPU.
There is no CPU fallback: without the CUDA library or a device, calls raise EngineError.
"""
import os
import threading as _threading

import numpy as np
from scipy.stats import chi2
from tqdm import tqdm

from . import _engine
from . import helpers as _helpers
from .helpers import (ar1, ar1_spectrum, fft, fft_kwargs, find, get_cache_dir,
                      rednoise)
from .mothers import Morlet, Paul, DOG, MexicanHat, Morse

_PRECISIONS = {'fp64': _engine.F64, 'f64': _engine.F64, 'float64': _engine.F64,
               'fp32': _engine.F32, 'f32': _engine.F32, 'float32': _engine.F32}


def _precision():
    """Arithmetic of the engine: fp64 (default, matches the reference) or fp32 via the
    CWTB_PRECISION environment variable."""
    return _PRECISIONS[os.environ.get('CWTB_PRECISION', 'fp64').lower()]


def _coherence_precision(precision):
    """Engine precision of the coherence paths from a spelling of `_PRECISIONS`
    (CWTB_PRECISION governs cwt only)."""
    try:
        return _PRECISIONS[str(precision).lower()]
    except KeyError:
        raise ValueError("precision must be one of %s, got %r"
                         % (", ".join(sorted(_PRECISIONS)), precision))


def _resolve_scales(n0, dt, dj, s0, J, wavelet, freqs):
    """Scale vector exactly as the reference builds it (wavelet.py:75-88)."""
    if freqs is None:
        if s0 == -1:
            s0 = 2 * dt / wavelet.flambda()
        if J == -1:
            J = int(np.round(np.log2(n0 * dt / s0) / dj))
        sj = s0 * 2 ** (np.arange(0, J + 1) * dj)
        freqs = 1 / (wavelet.flambda() * sj)
    else:
        sj = 1 / (wavelet.flambda() * freqs)
    return sj, freqs


def _nan_rows(wavelet, sj, npad, dt):
    """Rows the reference would find all-NaN and drop (wavelet.py:111-115), for the analytic
    families, in O(S) host work:
      * psi_ft evaluates to NaN at some bin -- Paul: inf*0 once s*pi/dt > 709.78.  Overflow
        happens first at the two extreme bins, which are the ones evaluated here;
      * the scale itself is unusable: a custom `freqs` entry of 0 gives s = inf (inf*0 at bin 0),
        a negative one gives the square root of a negative normalisation (wavelet.py:103), NaN
        stays NaN.
    Duck-typed wavelets do not come here: their rows are classified from the host-evaluated
    response table (`_response_table`)."""
    # the entries of fft.fftfreq(npad, dt) at the most negative and the most positive bin
    # (k / (npad*dt) with the signed bin number k, computed like numpy does:
    # k * (1.0 / (npad * dt))) without building the array.  Any npad: for an odd length the
    # most negative bin is -(npad-1)/2 at index (npad+1)/2.
    k = np.array([-(npad // 2), (npad - 1) // 2])
    edge = 2 * np.pi * (k * (1.0 / (npad * dt)))
    sj = np.asarray(sj, dtype=float)
    with np.errstate(all='ignore'):
        resp = wavelet.psi_ft(sj[:, None] * edge[None, :])
        unusable = ~np.isfinite(sj) | (sj < 0)
        if npad == 2:
            # fftfreq(2)[1] is negative: the reference's normalisation is NaN for every s > 0
            unusable = unusable | (sj > 0)
    return np.isnan(resp).any(axis=1) | unusable


def _response_table(wavelet, sj, npad, dt):
    """sqrt(s*w1*N) * conj(psi_ft(s*w)) on the [S, Np] grid, exactly as wavelet.py:102-104
    forms it: the host-evaluated path of duck-typed wavelets (SURVEY 8b)."""
    ftfreqs = 2 * np.pi * fft.fftfreq(npad, dt)
    col = np.asarray(sj)[:, np.newaxis]
    with np.errstate(all='ignore'):
        return ((col * ftfreqs[1] * npad) ** .5 *
                np.conjugate(wavelet.psi_ft(col * ftfreqs))).astype(np.complex128)


def _engine_family(wavelet):
    """(family, param) when the engine evaluates this wavelet analytically, else None."""
    return wavelet._engine_spec() if hasattr(wavelet, '_engine_spec') else None


def _sync_padding(eng, n0):
    """Hand the transform-length policy of helpers.fft_kwargs to the engine.  True if this
    transform runs un-padded (policy off and n0 not a power of two)."""
    eng.set_padding(_helpers._FFT_NEXT_POW2)
    return (not _helpers._FFT_NEXT_POW2) and (n0 & (n0 - 1)) != 0


def _transform(signal, dt, sj, wavelet, precision=None, engine=None, table=None):
    """W[S, n0] (complex128) for the given scales; rows are NOT yet NaN-filtered.  `table`:
    rows of `_response_table` for `sj` (duck-typed wavelets).  The caller holds the engine lock."""
    eng = engine or _engine.default_engine()
    precision = _precision() if precision is None else precision
    if _sync_padding(eng, len(signal)):
        precision = _engine.F64      # un-padded transforms run in fp64
    spec = _engine_family(wavelet)
    sig = np.asarray(signal)
    if sig.dtype != np.float32:
        sig = np.asarray(sig, dtype=np.float64)
    if spec is not None:
        family, param = spec
        W = eng.cwt(sig, dt, sj, family, param, precision)
    else:
        # duck-typed wavelet: the host evaluates psi_ft on the [S, Np] grid exactly as
        # wavelet.py:102-104 does; the device multiplies and inverse-transforms.
        if table is None:
            table = _response_table(wavelet, sj, fft_kwargs(sig)['n'], dt)
        W = eng.cwt(sig, dt, sj, _engine.TABLE, 0.0, precision, table=table)
    return W, eng


def cwt(signal, dt, dj=1/12, s0=-1, J=-1, wavelet='morlet', freqs=None):
    """Continuous wavelet transform of `signal` (reference wavelet.py:13-124).

    Returns (W, sj, freqs, coi, fft, fftfreqs) exactly like the reference: W is
    complex128 of shape (len(sj), len(signal)); scales whose transform is all-NaN
    (Paul at very large scales, unusable custom frequencies) are removed from W, sj and
    freqs.  A complex signal is transformed like the reference does (its FFT is linear):
    real and imaginary parts go through the engine separately."""
    wavelet = _check_parameter_wavelet(wavelet)
    n0 = len(signal)
    sj, freqs = _resolve_scales(n0, dt, dj, s0, J, wavelet, freqs)
    npad = fft_kwargs(signal)['n']

    table = None
    if _engine_family(wavelet) is None:
        table = _response_table(wavelet, np.asarray(sj, dtype=float), npad, dt)
        bad = np.isnan(table).any(axis=1)
    else:
        bad = _nan_rows(wavelet, np.asarray(sj, dtype=float), npad, dt)
    keep = ~bad

    # O(n0) host-side outputs (cone of influence, Fourier frequencies): for long signals they
    # are computed on a helper thread while the engine call (which releases the GIL) copies W
    # back from the device.
    side = {}

    def host_side():
        coi = (n0 / 2 - np.abs(np.arange(0, n0) - (n0 - 1) / 2))
        side['coi'] = wavelet.flambda() * wavelet.coi() * dt * coi
        ftfreqs = 2 * np.pi * fft.fftfreq(npad, dt)
        side['fftfreqs'] = ftfreqs[1:npad // 2] / (2 * np.pi)

    helper = None
    if n0 >= (1 << 16):
        helper = _threading.Thread(target=host_side)
        helper.start()
    sig = np.asarray(signal)
    parts = [sig.real, sig.imag] if np.iscomplexobj(sig) else [sig]
    eng = _engine.default_engine()
    try:
        Ws, spectra = [], []
        for part in parts:
            # one engine transaction per transform: length policy, transform, coefficients and
            # the spectrum of the SAME resident job (the default engine is shared by all threads)
            with eng.lock:
                if keep.any():
                    Wp, _ = _transform(part, dt, np.asarray(sj)[keep], wavelet, engine=eng,
                                       table=None if table is None else table[keep])
                else:
                    # every row NaN: the reference keeps them all (np.any(sel) is False)
                    _transform(part, dt, np.asarray(sj)[:1], wavelet, engine=eng,
                               table=None if table is None else np.zeros_like(table[:1]))
                    Wp = np.full((len(sj), n0), np.nan + 1j * np.nan)
                Ws.append(Wp)
                spectra.append(eng.signal_fft())
        if keep.any():
            sj, freqs = sj[keep], freqs[keep]
        if len(parts) == 2:
            W = Ws[0] + 1j * Ws[1]
            spectrum = spectra[0] + 1j * spectra[1]
        else:
            W, spectrum = Ws[0], spectra[0]
    finally:
        if helper is not None:
            helper.join()
    if helper is None:
        host_side()
    return (W, sj, freqs, side['coi'], spectrum, side['fftfreqs'])


def icwt(W, sj, dt, dj=1/12, wavelet='morlet'):
    """Inverse continuous wavelet transform (reference wavelet.py:127-171).

    The sum over scales of Re(W)/sqrt(s) runs on the GPU; W may be (S, N) or (N, S)
    as in the reference (which always reduces axis 0)."""
    wavelet = _check_parameter_wavelet(wavelet)
    W = np.asarray(W)
    sj = np.asarray(sj, dtype=float)
    a, b = W.shape
    c = sj.size
    if a == c:
        red = _engine.default_engine().icwt_sum(W, sj)
    elif b == c:
        # scales vary along axis 1 but the reference still sums axis 0
        red = _engine.default_engine().icwt_sum(W / np.sqrt(sj)[None, :], np.ones(a))
    else:
        raise Warning('Input array dimensions do not match.')
    return dj * np.sqrt(dt) / (wavelet.cdelta * wavelet.psi(0)) * red


def significance(signal, dt, scales, sigma_test=0, alpha=None,
                 significance_level=0.95, dof=-1, wavelet='morlet'):
    """Chi-square significance levels of the wavelet power spectrum against a red-noise
    background (reference wavelet.py:174-313; Torrence & Compo 1998 sec. 4-5).
    O(S) host arithmetic."""
    wavelet = _check_parameter_wavelet(wavelet)
    try:
        n0 = len(signal)
    except TypeError:
        n0 = 1
    scales = np.asarray(scales)
    J = len(scales) - 1
    dj = np.log2(scales[1] / scales[0])
    variance = signal if n0 == 1 else signal.std() ** 2
    if alpha is None:
        alpha, _, _ = ar1(signal)

    period = scales * wavelet.flambda()
    freq = dt / period
    dofmin = wavelet.dofmin
    # discrete red-noise spectrum, TC98 eq. 16 (evaluated at k/N = freq, N = n0)
    k_over = 2 * np.pi * freq / n0
    fft_theor = variance * (1 - alpha ** 2) / (1 + alpha ** 2 - 2 * alpha * np.cos(k_over))
    signif = fft_theor
    try:
        if dof == -1:
            dof = dofmin
    except ValueError:
        pass

    if sigma_test == 0:  # TC98 eq. 18
        dof = dofmin
        signif = fft_theor * (chi2.ppf(significance_level, dof) / dof)
    elif sigma_test == 1:  # time-averaged, TC98 eq. 23
        if len(dof) == 1:
            dof = np.zeros(1, J + 1) + dof  # TypeError as in the reference
        dof[find(dof < 1)] = 1
        dof = dofmin * (1 + (dof * dt / wavelet.gamma / scales) ** 2) ** 0.5
        dof[find(dof < dofmin)] = dofmin
        for n, d in enumerate(dof):
            signif[n] = fft_theor[n] * (chi2.ppf(significance_level, d) / d)
    elif sigma_test == 2:  # scale-averaged, TC98 eq. 25-28
        if len(dof) != 2:
            raise Exception('DOF must be set to [s1, s2], '
                            'the range of scale-averages')
        if wavelet.cdelta == -1:
            raise ValueError('Cdelta and dj0 not defined '
                             'for {} with f0={}'.format(wavelet.name, wavelet.f0))
        s1, s2 = dof
        sel = find((scales >= s1) & (scales <= s2))
        navg = sel.size
        if navg == 0:
            raise ValueError('No valid scales between {} and {}.'.format(s1, s2))
        Savg = 1 / sum(1. / scales[sel])
        Smid = np.exp((np.log(s1) + np.log(s2)) / 2.)
        dof = (dofmin * navg * Savg / Smid) * ((1 + (navg * dj / wavelet.deltaj0) ** 2) ** 0.5)
        fft_theor = Savg * sum(fft_theor[sel] / scales[sel])
        chisquare = chi2.ppf(significance_level, dof) / dof
        signif = (dj * dt / wavelet.cdelta / Savg) * fft_theor * chisquare
    else:
        raise ValueError('sigma_test must be either 0, 1, or 2.')
    return signif, fft_theor


def _standardise(y, normalize):
    y = np.asarray(y)
    std = y.std()
    return y, ((y - y.mean()) / std if normalize else y), std


def _unit_binade(y):
    """y times the power of two that brings max|y| into [1/2, 1): exact, so the coherence of the
    result is that of y.  The coherence pipeline smooths the auto-spectra of two series as the real
    and imaginary parts of one complex field, and an FFT's twiddle products mix the rounding of the
    two parts: a series whose amplitude is 2^d times the other's would see the rounding of the
    larger enlarged by about 2^(2d) in its own field.  y is returned as is when it is all zero or
    not finite."""
    m = np.max(np.abs(y)) if y.size else 0.0
    if not (np.isfinite(m) and m > 0):
        return y
    return np.ldexp(y, -int(np.frexp(m)[1]))


def xwt(y1, y2, dt, dj=1/12, s0=-1, J=-1, significance_level=0.95,
        wavelet='morlet', normalize=True, precision='fp64'):
    """Cross wavelet transform W1 * conj(W2) (reference wavelet.py:316-419).

    Both transforms and the conjugate product (fused into the second transform's output
    pass) run on the GPU.  Returns (W12, coi, freq, signif).  `precision` (an extension of
    the reference signature): 'fp64' (default) or 'fp32', the arithmetic of the transforms;
    W12 is complex128 either way.  Un-padded transforms run in fp64 whatever is asked."""
    p = _xwt_problem(y1, y2, dt, dj, s0, J, wavelet, normalize, precision)
    eng = _engine.default_engine()
    W12 = _xwt_on_device(eng, p, eng.xwt)
    coi = _coi(p.wavelet, dt, p.n0)
    return W12, coi, p.freq, _xwt_signif(p, significance_level)


def _xwt_problem(y1, y2, dt, dj, s0, J, wavelet, normalize, precision):
    """What `xwt` resolves on the host before the device call (reference wavelet.py:370-394): the
    wavelet, the raw and standardised series, the scales without the reference's all-NaN rows
    and the requested engine precision."""
    prec = _coherence_precision(precision)
    wavelet = _check_parameter_wavelet(wavelet)
    y1, y1n, std1 = _standardise(y1, normalize)
    y2, y2n, std2 = _standardise(y2, normalize)
    n0 = len(y1n)
    sj, freq = _resolve_scales(n0, dt, dj, s0, J, wavelet, None)
    npad = fft_kwargs(y1n)['n']
    keep = ~_nan_rows(wavelet, sj, npad, dt)
    if not keep.any():
        keep[:] = True
    sj, freq = sj[keep], freq[keep]
    return _Problem(y1=y1, y2=y2, y1n=y1n, y2n=y2n, std1=std1, std2=std2, n0=n0, dt=dt, dj=dj,
                    wavelet=wavelet, sj=sj, freq=freq, normalize=normalize, prec=prec)


def _xwt_on_device(eng, p, call):
    """One engine transaction of the cross transform: length policy (un-padded transforms run in
    fp64), then call(y1n, y2n, dt, scales, family, param, precision=).  Returns the call's result;
    `p.prec` becomes the precision used."""
    with eng.lock:
        if _sync_padding(eng, p.n0):
            p.prec = _engine.F64      # un-padded transforms run in fp64
        return call(p.y1n, p.y2n, p.dt, p.sj, *_family_of(p.wavelet), precision=p.prec)


def _xwt_signif(p, significance_level):
    """Significance level of |W12| per scale against the two series' red-noise spectra (reference
    wavelet.py:404-418): the fourth return value of `xwt`."""
    std1, std2 = (1., 1.) if p.normalize else (p.std1, p.std2)
    a1, _, _ = ar1(p.y1)
    a2, _, _ = ar1(p.y2)
    Pk1 = ar1_spectrum(p.freq * p.dt, a1)
    Pk2 = ar1_spectrum(p.freq * p.dt, a2)
    dof = p.wavelet.dofmin
    PPF = chi2.ppf(significance_level, dof)
    return (std1 * std2 * (Pk1 * Pk2) ** 0.5 * PPF / dof)


def _family_of(wavelet):
    spec = _engine_family(wavelet)
    if spec is None:
        raise NotImplementedError(
            'xwt/wct on the GPU need a Morlet, Paul, DOG or Morse mother wavelet')
    return spec


class _smoothing_filter(object):
    """Within the engine lock: install the time-smoothing responses of a non-Morlet wavelet
    (mothers.time_filter_table) for the calls inside the block, restore Morlet's Gaussian after."""

    def __init__(self, eng, wavelet, scales, dt, n):
        self.eng = eng
        self.table = None
        if not isinstance(wavelet, Morlet):
            from .mothers import time_filter_table
            self.table = time_filter_table(wavelet, scales, dt, fft_kwargs(range(n))['n'])

    def __enter__(self):
        if self.table is not None:
            self.eng.set_smooth_filter(self.table)
        return self

    def __exit__(self, *exc):
        if self.table is not None:
            self.eng.set_smooth_filter(None)
        return False


def _boxcar_len(wavelet, dj):
    """Number of taps of the scale-axis boxcar, int(round(2*deltaj0/dj)) (mothers.py:100)."""
    return int(np.round(wavelet.deltaj0 / dj * 2))


def _coi(wavelet, dt, n0):
    """Cone of influence of an n0-point series (reference wavelet.py:118-120)."""
    coi = (n0 / 2 - np.abs(np.arange(0, n0) - (n0 - 1) / 2))
    return wavelet.flambda() * wavelet.coi() * dt * coi


class _Problem(object):
    """What `xwt` / `wct` resolve on the host before the device call (see `_xwt_problem` and
    `_wct_problem`)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _wct_problem(series, dt, dj, s0, J, wavelet, normalize, precision):
    """What `wct` (two series) and `partial_wct` / `multiple_wct` (three) resolve on the host before
    the device pipeline (reference wavelet.py:461-497): the wavelet, s0 and J, the raw and
    standardised series (`ys`, `yns`), the scales, the boxcar length and the requested engine
    precision."""
    prec = _coherence_precision(precision)
    wavelet = _check_parameter_wavelet(wavelet)
    if not hasattr(wavelet, 'smooth'):
        # same failure mode as the reference for Paul / DOG (no smoothing operator)
        raise AttributeError("'{}' object has no attribute 'smooth'".format(
            type(wavelet).__name__))
    if s0 == -1:
        s0 = 2 * dt / wavelet.flambda()
    if J == -1:
        J = int(np.round(np.log2(series[0].size * dt / s0) / dj))  # .size: ndarray required, as in the reference
    ys, yns = zip(*[_standardise(y, normalize)[:2] for y in series])
    if not normalize:
        # series in their own units: the same binade for all, so that none drowns in the rounding of
        # another (`_unit_binade`).  WCT, aWCT, RP2, RM2 and their significance do not depend on it
        yns = tuple(_unit_binade(y) for y in yns)
    n0 = yns[0].size
    sj, freq = _resolve_scales(n0, dt, dj, s0, J, wavelet, None)
    klen = _boxcar_len(wavelet, dj)
    if klen < 1:
        raise ValueError('smoothing window undefined for this wavelet (deltaj0 = -1)')
    return _Problem(ys=ys, yns=yns, n0=n0, dt=dt, dj=dj, s0=s0, J=J,
                    wavelet=wavelet, sj=sj, freq=freq, klen=klen, prec=prec)


def _wct_on_device(eng, p, call, **kw):
    """One engine transaction of the coherence pipeline: length policy (un-padded transforms run
    in fp64), the Paul / DOG smoothing filter, then call(*yns, dt, dj, scales, family, param,
    boxcar_len=, precision=, **kw).  Returns the call's result; `p.prec` becomes the precision
    used."""
    with eng.lock:
        if _sync_padding(eng, len(p.yns[0])):
            p.prec = _engine.F64      # un-padded transforms run in fp64
        with _smoothing_filter(eng, p.wavelet, p.sj, p.dt, len(p.yns[0])):
            return call(*p.yns, p.dt, p.dj, p.sj, *_family_of(p.wavelet), boxcar_len=p.klen,
                        precision=p.prec, **kw)


def wct(y1, y2, dt, dj=1/12, s0=-1, J=-1, sig=True,
        significance_level=0.95, wavelet='morlet', normalize=True, precision='fp64',
        **kwargs):
    """Wavelet coherence (reference wavelet.py:422-528).

    Returns (WCT, aWCT, coi, freq, sig).  The two transforms, the |W|^2/s and W12/s
    products, the Gaussian time smoothing, the scale boxcar and the coherence ratio run
    on the GPU; `sig` comes from wct_significance (GPU Monte-Carlo) when sig=True.
    `precision` (an extension of the reference signature): 'fp64' (default) or 'fp32', the
    arithmetic of the device pipeline, also that of the significance test; WCT and aWCT are
    float64 either way and fp32 WCT is within 1e-3 of fp64 (DESIGN.md section 6).  With
    `normalize=False` each series is first scaled by the power of two that brings its largest
    magnitude into [1/2, 1): exact, so WCT and aWCT are those of the series as given, whatever
    their amplitudes and units."""
    p = _wct_problem((y1, y2), dt, dj, s0, J, wavelet, normalize, precision)
    (y1, y2), wavelet, s0, J, freq = p.ys, p.wavelet, p.s0, p.J, p.freq
    eng = _engine.default_engine()
    WCT, aWCT = _wct_on_device(eng, p, eng.wct)
    coi = _coi(wavelet, dt, p.n0)
    if sig:
        a1, b1, c1 = ar1(y1)
        a2, b2, c2 = ar1(y2)
        sig = _wct_significance(a1, a2, dt=dt, dj=dj, s0=s0, J=J,
                               significance_level=significance_level,
                               wavelet=wavelet, precision=precision, **kwargs)
    else:
        sig = np.asarray([0])
    return WCT, aWCT, coi, freq, sig


def partial_wct(y, x1, x2, dt, dj=1/12, s0=-1, J=-1, wavelet='morlet', normalize=True,
                precision='fp64'):
    """Partial wavelet coherence of `y` with `x1` once `x2` is accounted for (Mihanovic et al.
    2009; Ng & Chan 2012).  An extension: the reference has no three-series coherence.

    With S the smoothing operator of `wct`, S_a = S(|W_a|^2 / s), S_ab = S(W_a conj(W_b) / s):
        RP2 = |S_y1 S_2 - S_y2 S_21|^2 / ((S_y S_2 - |S_y2|^2) (S_1 S_2 - |S_12|^2))
            = |g_y1 - g_y2 g_21|^2 / ((1 - R2_y2) (1 - R2_12)),   g_ab = S_ab / sqrt(S_a S_b).
    Returns (RP2, coi, freq); RP2 is float64 [S, n0] in either `precision` ('fp64' default, or
    'fp32': the arithmetic of the transforms and smoothing; the smoothed fields are combined in
    double either way).  Scales, boxcar, un-padded fallback to fp64 and the Paul / DOG smoothing
    filter are resolved as in `wct`, with the same errors.  RP2 lies in [0, 1] up to rounding and
    is not clamped: where a denominator is zero or rounds to <= 0 it is inf or NaN.  Where x1 and
    x2 are nearly coherent (R2_12 -> 1) the measure is ill-conditioned: its rounding error grows
    like 1 / ((1 - R2_y2) (1 - R2_12)).  Significance levels: `wct3_significance`."""
    return _wct3(y, x1, x2, dt, dj, s0, J, wavelet, normalize, precision, partial=True)


def multiple_wct(y, x1, x2, dt, dj=1/12, s0=-1, J=-1, wavelet='morlet', normalize=True,
                 precision='fp64'):
    """Multiple wavelet coherence: how much of `y` the series `x1` and `x2` explain together
    (Ng & Chan 2012).  An extension: the reference has no three-series coherence.

    With the smoothed fields of `partial_wct`:
        RM2 = (R2_y1 + R2_y2 - 2 Re(g_y1 g_12 g_2y)) / (1 - R2_12)
            = 1 - det G3 / (S_y (S_1 S_2 - |S_12|^2)),   G3 the 3 x 3 smoothed spectral matrix.
    Returns (RM2, coi, freq), RM2 float64 [S, n0]; `precision`, scales, errors and the absence of
    clamping as in `partial_wct`.  RM2 >= max(R2_y1, R2_y2) up to rounding, and
    1 - RM2 = (1 - R2_y2) (1 - RP2).  Ill-conditioned where x1 and x2 are nearly coherent: the
    rounding error grows like 1 / (1 - R2_12).  Significance levels: `wct3_significance` (RM2 has a
    higher null level than the two-series coherence, since RM2 >= R2_y1 at every point)."""
    return _wct3(y, x1, x2, dt, dj, s0, J, wavelet, normalize, precision, partial=False)


def _wct3(y, x1, x2, dt, dj, s0, J, wavelet, normalize, precision, partial):
    p = _wct_problem((y, x1, x2), dt, dj, s0, J, wavelet, normalize, precision)
    eng = _engine.default_engine()
    RP2, RM2 = _wct_on_device(eng, p, eng.wct3, want_partial=partial, want_multiple=not partial)
    return (RP2 if partial else RM2), _coi(p.wavelet, dt, p.n0), p.freq


def _mc_problem(dt, dj, s0, J, wavelet, N=None):
    """Geometry of the Monte-Carlo coherence problem (reference wavelet.py:588-607): surrogate
    length, scales, cone-of-influence mask, last valid scale and the sig95 template.  `N`: the
    surrogate length; by default the reference's, derived from the largest scale."""
    if N is None:
        ms = s0 * (2 ** (J * dj)) / dt
        N = int(np.ceil(ms * 6))
    sj = s0 * 2 ** (np.arange(0, J + 1) * dj)
    freq = 1 / (wavelet.flambda() * sj)
    coi = (N / 2 - np.abs(np.arange(0, N) - (N - 1) / 2))
    coi = wavelet.flambda() * wavelet.coi() * dt * coi
    period = np.ones([1, N]) / freq[:, None]
    outsidecoi = (period <= (np.ones([J + 1, 1]) * coi[None, :]))
    sig95 = np.zeros(J + 1)
    maxscale = find(outsidecoi.any(axis=1))[-1]
    sig95[outsidecoi.any(axis=1)] = np.nan
    return dict(N=N, sj=sj, nbins=1000, maxscale=int(maxscale), sig95=sig95,
                mask=np.ascontiguousarray(outsidecoi, dtype=np.uint8))


def _mc_histogram(prob, dt, dj, wavelet, draw, indices, progress=False, engine=None,
                  precision=_engine.F64, nser=2):
    """1000-bin histograms of the coherence of the surrogate units draw(i), i in `indices`
    (reference wavelet.py:609-630), accumulated on the GPU.  `nser` = 2: draw(i) is a pair, the
    result the coherence histogram int64 [S, nbins].  `nser` = 3: draw(i) is a triple (y, x1, x2),
    the result int64 [2, S, nbins], the histograms of the partial and of the multiple coherence.
    `precision`: engine precision of the coherence."""
    N, sj, nbins = prob['N'], prob['sj'], prob['nbins']
    hist = np.zeros((nser - 1, sj.size, nbins), dtype=np.int64)
    eng = engine or _engine.default_engine()
    fam = _family_of(wavelet)
    indices = list(indices)
    batch = max(1, min(len(indices), int((256 << 20) // (8 * nser * N)) or 1))
    bar = tqdm(total=len(indices), disable=not progress)
    for b0 in range(0, len(indices), batch):
        idx = indices[b0:b0 + batch]
        noise = np.empty((len(idx), nser, N))
        for k, i in enumerate(idx):
            noise[k] = draw(i)
        with eng.lock:
            prec = _engine.F64 if _sync_padding(eng, N) else precision
            with _smoothing_filter(eng, wavelet, sj, dt, N):
                if nser == 2:
                    eng.wct_mc(noise, dt, dj, sj, fam[0], fam[1], _boxcar_len(wavelet, dj), prob['mask'],
                               prob['maxscale'], nbins, hist[0], precision=prec)
                else:
                    eng.wct3_mc(noise, dt, sj, fam[0], fam[1], _boxcar_len(wavelet, dj), prob['mask'],
                                prob['maxscale'], nbins, hist[0], hist[1], precision=prec)
        bar.update(len(idx))
    bar.close()
    return hist[0] if nser == 2 else hist


def _mc_levels(prob, hist, significance_level):
    """Percentile of every scale's histogram (reference wavelet.py:632-640)."""
    nbins = prob['nbins']
    sig95 = prob['sig95'].copy()
    R2y = (np.arange(nbins) + 0.5) / nbins
    for s in range(prob['maxscale']):
        sel = hist[s] != 0
        P = hist[s, sel].astype(float).cumsum()
        P = (P - 0.5) / P[-1]
        sig95[s] = np.interp(significance_level, P, R2y[sel])
    return sig95


def _mc_histogram_seeded(prob, dt, dj, wavelet, seed, first, count, engine=None,
                         precision=_engine.F64, nser=2):
    """The same histograms with the surrogates drawn on the device (Philox stream keyed by
    (seed, pair or triple number)): no host RNG, no noise H2D."""
    sj, nbins = prob['sj'], prob['nbins']
    hist = np.zeros((nser - 1, sj.size, nbins), dtype=np.int64)
    eng = engine or _engine.default_engine()
    fam = _family_of(wavelet)
    args = (prob['N'], dt, sj, fam[0], fam[1], _boxcar_len(wavelet, dj), prob['mask'], prob['maxscale'], nbins)
    with eng.lock:
        prec = _engine.F64 if _sync_padding(eng, prob['N']) else precision
        with _smoothing_filter(eng, wavelet, sj, dt, prob['N']):
            if nser == 2:
                eng.wct_mc_seeded(seed, first, count, *args, hist[0], precision=prec)
            else:
                eng.wct3_mc_seeded(seed, first, count, *args, hist[0], hist[1], precision=prec)
    return hist[0] if nser == 2 else hist


def wct_significance(al1, al2, dt, dj, s0, J, significance_level=0.95,
                     wavelet='morlet', mc_count=300, progress=True,
                     cache=True, seed=None):
    """Monte-Carlo significance level of the wavelet coherence per scale (reference
    wavelet.py:531-647).

    Default (`seed=None`): surrogates are drawn on the host with numpy's global RNG in exactly
    the reference's order (one set-up draw, then noise1, noise2 per iteration), so a seeded
    run reproduces the reference's numbers; transforms, smoothing, coherence and the
    1000-bin histograms are accumulated on the GPU.  With an integer `seed` (an extension of
    the reference signature) the surrogates are drawn on the device from a counter-based
    Philox stream: statistically equivalent white noise, no host RNG or upload, about twice
    as fast; the result then depends on `seed` only, not on numpy's global state.  The
    on-disk cache keeps the reference's key and format (~/.cache/pycwt/<key>.gz).
    The parameter list stays the reference's (plus `seed`): the fp32 coherence of the surrogates
    is reached through `wct(..., sig=True, precision='fp32')`."""
    return _wct_significance(al1, al2, dt, dj, s0, J, significance_level, wavelet, mc_count,
                             progress, cache, seed)


def _wct_significance(al1, al2, dt, dj, s0, J, significance_level=0.95, wavelet='morlet',
                      mc_count=300, progress=True, cache=True, seed=None, precision='fp64'):
    """wct_significance with `precision`: 'fp64' (default) or 'fp32', the arithmetic of the
    device coherence.  The surrogates, ar1 and the levels stay float64 on the host; the fp32
    levels agree with fp64 within a histogram bin, so the cache key does not include it."""
    prec = _coherence_precision(precision)
    wavelet = _check_parameter_wavelet(wavelet)
    if cache:
        aa = np.round(np.arctanh(np.array([al1, al2]) * 4))
        aa = np.abs(aa) + 0.5 * (aa < 0)
        cache_file = 'wct_sig_{:0.5f}_{:0.5f}_{:0.5f}_{:0.5f}_{:d}_{}'\
            .format(aa[0], aa[1], dj, s0 / dt, J, wavelet.name)
        cache_dir = get_cache_dir()
        try:
            dat = np.loadtxt('{}/{}.gz'.format(cache_dir, cache_file), unpack=True)
            print('NOTE: WCT significance loaded from cache.\n')
            return dat
        except IOError:
            pass
    print('Calculating wavelet coherence significance')

    prob = _mc_problem(dt, dj, s0, J, wavelet)
    N = prob['N']
    if seed is None:
        rednoise(N, al1, 1)  # the reference's set-up draw (its transform only yields sj/freq/coi)

        def draw(i):
            return rednoise(N, al1, 1), rednoise(N, al2, 1)

        hist = _mc_histogram(prob, dt, dj, wavelet, draw, range(mc_count), progress, precision=prec)
    else:
        hist = _mc_histogram_seeded(prob, dt, dj, wavelet, seed, 0, mc_count, precision=prec)
    sig95 = _mc_levels(prob, hist, significance_level)

    if cache:
        np.savetxt('{}/{}.gz'.format(cache_dir, cache_file), sig95)
    return sig95


def _wct3_mc_setup(wavelet, dj, precision):
    """(wavelet, engine precision) of a three-series Monte-Carlo run, with the errors of
    `partial_wct` / `multiple_wct`."""
    prec = _coherence_precision(precision)
    wavelet = _check_parameter_wavelet(wavelet)
    if not hasattr(wavelet, 'smooth'):
        raise AttributeError("'{}' object has no attribute 'smooth'".format(type(wavelet).__name__))
    if _boxcar_len(wavelet, dj) < 1:
        raise ValueError('smoothing window undefined for this wavelet (deltaj0 = -1)')
    _family_of(wavelet)
    return wavelet, prec


def wct3_significance(al_y, al1, al2, dt, dj, s0, J, significance_level=0.95, wavelet='morlet',
                      mc_count=300, progress=True, seed=None, precision='fp64'):
    """Monte-Carlo significance levels of `partial_wct` and `multiple_wct` per scale.  An
    extension: the reference has no three-series coherence.

    Returns (sig_partial, sig_multiple), float64 [J + 1] each, with the conventions of
    `wct_significance`: the `significance_level` quantile of the 1000-bin histogram of every row
    with points outside the cone of influence of the surrogates, 0 for a row without any.

    Null: three mutually independent white-noise series of N = ceil(6 s0 2^(J dj) / dt) samples
    per triple (`rednoise`, which is white noise as in the reference; `al_y`, `al1`, `al2` only
    set how many draws it discards), not standardised, each triple through the whole pipeline of
    `partial_wct` / `multiple_wct`.  This null does not keep a coherence between x1 and x2.  A
    point whose RP2 or RM2 is not finite (a zero denominator) is not counted.

    Default (`seed=None`): the triples are drawn on the host with numpy's global RNG, one set-up
    draw rednoise(N, al_y, 1), then rednoise(N, al_y), rednoise(N, al1), rednoise(N, al2) per
    triple, so a run seeded through np.random is reproducible.  With an integer `seed` the triples
    come from the device's counter-based Philox stream, keyed by (seed, triple number) and disjoint
    from the pairs of `wct_significance(seed=)`.  `precision`: 'fp64' (default) or 'fp32', the
    arithmetic of the surrogates' transforms and smoothing; the levels are float64 either way.
    Errors as in `partial_wct`.  No on-disk cache."""
    wavelet, prec = _wct3_mc_setup(wavelet, dj, precision)
    prob = _mc_problem(dt, dj, s0, J, wavelet)
    N = prob['N']
    if seed is None:
        rednoise(N, al_y, 1)  # set-up draw, as in wct_significance

        def draw(i):
            return rednoise(N, al_y, 1), rednoise(N, al1, 1), rednoise(N, al2, 1)

        hist = _mc_histogram(prob, dt, dj, wavelet, draw, range(mc_count), progress, precision=prec,
                             nser=3)
    else:
        hist = _mc_histogram_seeded(prob, dt, dj, wavelet, seed, 0, mc_count, precision=prec, nser=3)
    return _mc_levels(prob, hist[0], significance_level), _mc_levels(prob, hist[1], significance_level)


def _surrogate_problem(series, dt, dj, s0, J, wavelet, normalize, precision):
    """(p, prob) of a Monte-Carlo run against phase-randomised surrogates of `series`: the
    `_wct_problem` of the data and the Monte-Carlo geometry of their own length and cone of
    influence."""
    p = _wct_problem(series, dt, dj, s0, J, wavelet, normalize, precision)
    if any(y.size != p.n0 for y in p.yns):
        raise ValueError('the series must have the same length')
    if not all(np.isfinite(y).all() for y in p.yns):
        raise ValueError('the series must be finite: phase randomisation transforms every sample')
    _family_of(p.wavelet)
    return p, _mc_problem(dt, dj, p.s0, p.J, p.wavelet, N=p.n0)


_NULLS = {'ar1': _engine.NULL_AR1, 'phase': _engine.NULL_PHASE}


def _null_kind(null):
    """The engine's null of a null's name."""
    if null not in _NULLS:
        raise ValueError("null must be 'ar1' or 'phase', got %r" % (null,))
    return _NULLS[null]


def _ar1_params(ys, normalize, fit):
    """Lists g, m, sigma of the AR(1) null of the raw series `ys`: g = ar1(y)[0] where `fit` (a flag
    per series) is set, else 0; m = 0 and sigma = 1 with `normalize` (the units are standardised as
    the data are), else y's mean and standard deviation (ddof 0)."""
    g = [ar1(y)[0] if f else 0.0 for y, f in zip(ys, fit)]
    if normalize:
        return g, [0.0] * len(ys), [1.0] * len(ys)
    return g, [float(y.mean()) for y in ys], [float(y.std()) for y in ys]


def _coherence_null(null, p, normalize, conditional=True):
    """The engine's null (`_engine.CoherenceNull`) of a coherence test of the series of `p` (a
    `_wct_problem`): 'phase' puts the series in the phase groups (0, 1), or (0, 1, 1) for a
    conditional triple and (0, 1, 2) otherwise; 'ar1' draws every series, except x1 and x2 of a
    conditional triple, which are held at the data as transformed (`p.yns`).  With normalize=False
    the AR(1) m and sigma are the mean and standard deviation of `p.yns`.  ValueError for an
    unknown name and for a drawn series whose g is not finite or has |g| >= 1."""
    kind = _null_kind(null)
    nser = len(p.ys)
    if kind == _engine.NULL_PHASE:
        return _engine.CoherenceNull(kind, (0, 1) if nser == 2 else (0, 1, 1) if conditional else (0, 1, 2))
    held = (0, 1, 1) if nser == 3 and conditional else (0,) * nser
    # normalize=False: the series as transformed, in the binade `_unit_binade` gives them, so that the
    # drawn series share the binade of the held ones (g, and the coherence, are the same either way)
    g, m, sigma = _ar1_params(p.ys if normalize else p.yns, normalize, [not h for h in held])
    for s, (gs, h) in enumerate(zip(g, held)):
        if not h and not (np.isfinite(gs) and abs(gs) < 1):
            raise ValueError("the AR(1) null needs a finite lag-1 autocorrelation with |g| < 1; series %d "
                             "has g = %r" % (s, gs))
    return _engine.CoherenceNull(kind, None, g, m, sigma, held)


def _surrogate_histogram(p, prob, null, seed, first, count, engine=None, serial=None):
    """Histograms int64 [nser - 1, S, nbins] of the coherence (two series) or of the partial and
    multiple coherence (three) of the surrogate units first .. first + count - 1 of `null` (a
    `_coherence_null` of `p`) for the standardised data `p.yns`, drawn and accumulated on the device
    in one transaction.  With the `serial` of the resident product of the same data, the same run
    also counts, per point, the units that reach the product's value (`Engine.surrogate_counts`,
    counters reset first)."""
    nser = len(p.yns)
    hist = np.zeros((nser - 1, p.sj.size, prob['nbins']), dtype=np.int64)
    eng = engine or _engine.default_engine()

    def call(*a, boxcar_len, precision):
        dt, _, sj, family, param = a[nser:]
        args = (np.stack(a[:nser]), null, seed, first, count, dt, sj, family, param, boxcar_len,
                prob['mask'], prob['maxscale'], prob['nbins'], *hist)
        if serial is None:
            eng.wct_mc_phase(*args, precision=precision)
        else:
            eng.surrogate_counts(*args, serial=serial, reset=True, precision=precision)

    _wct_on_device(eng, p, call)
    return hist


def _surrogate_seed(seed):
    """`seed`, or one draw from numpy's global RNG (so np.random.seed makes a run repeatable)."""
    return int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed)


def wct_surrogate_significance(y1, y2, dt, dj=1/12, s0=-1, J=-1, significance_level=0.95,
                               wavelet='morlet', normalize=True, mc_count=300, seed=None,
                               precision='fp64', null='phase'):
    """Monte-Carlo significance level of the wavelet coherence of `y1` and `y2` per scale, against
    surrogates of the data's length drawn on the device.  An extension: the reference tests against
    white noise only (`wct_significance`).

    Null `null='phase'` (default): each surrogate pair is the two standardised series with the
    Fourier phases of each replaced by independent uniform random phases (Theiler et al. 1992), at
    the series' own length n0: X'_k = X_k e^{i phi_k} for 1 <= k < n0/2, Hermitian completion, mean
    and Nyquist bin kept.  Every surrogate keeps the power spectrum, mean and variance of its series
    exactly; the two are independent of each other.

    `null='ar1'`: red noise (Grinsted et al. 2004), two independent AR(1) series per pair, series s
    x = m + sigma z, z[0] = e[0], z[n] = g z[n-1] + sqrt(1 - g^2) e[n], with g = ar1(y_s)[0] of the
    raw series, m = 0 and sigma = 1 with normalize=True, else the mean and standard deviation (ddof
    0) of y_s as the coherence transforms it (scaled by the power of two that brings max|y_s| into
    [1/2, 1)): the pairs of `ResidentCrossWavelet.surrogate_test(null='ar1')` for the same seed and
    parameters.  It makes no assumption of a circular record.  ValueError where a g is not finite or
    |g| >= 1.

    Each pair goes through the whole pipeline of `wct` at the data's length.

    The arguments are those of `wct`, resolved the same way (scales, boxcar, standardisation,
    `precision`, errors), so the result, float64 [J + 1], lines up row for row with the WCT of the
    same arguments: `WCT > sig[:, None]`.  The geometry is the data's: the histograms count the
    points inside the cone of influence of an n0-point record.  Conventions of `wct_significance`:
    the `significance_level` quantile of the 1000-bin histogram, NaN from the last row with such
    points on, 0 for a row without any.

    The surrogates are drawn on the device from a counter-based Philox stream keyed by (`seed`,
    pair number), in one device transaction (no progress bar); `seed=None` takes one draw from
    numpy's global RNG as the seed, so `np.random.seed` makes a run repeatable.  Transforms of the
    surrogate generator run in fp64 whatever `precision`.  A non-finite sample or series of unequal
    lengths raise ValueError.  No on-disk cache (the key would have to hash the data).

    Phase randomisation assumes a stationary record and treats it as circular: a strong trend or a
    mismatch between the two ends is spread over all frequencies of the surrogates and biases the
    level, so detrend the series first (as the samples do).  The surrogates are Gaussian-like
    whatever the data's amplitude distribution (no amplitude adjustment)."""
    p, prob = _surrogate_problem((y1, y2), dt, dj, s0, J, wavelet, normalize, precision)
    hist = _surrogate_histogram(p, prob, _coherence_null(null, p, normalize), _surrogate_seed(seed), 0, mc_count)
    return _mc_levels(prob, hist[0], significance_level)


def wct3_surrogate_significance(y, x1, x2, dt, dj=1/12, s0=-1, J=-1, significance_level=0.95,
                                wavelet='morlet', normalize=True, mc_count=300, seed=None,
                                precision='fp64', conditional=True, null='phase'):
    """Monte-Carlo significance levels of `partial_wct` and `multiple_wct` per scale, against
    phase-randomised surrogates of the data themselves (`null='phase'`, the default) or red noise
    (`null='ar1'`).  Returns (sig_partial, sig_multiple), float64 [J + 1] each, row for row with the
    RP2 / RM2 of the same arguments.

    Null, `conditional=True` (default): in every surrogate triple x1 and x2 are rotated by the SAME
    random phases and y by phases of its own (Prichard & Theiler 1994).  x1 and x2 keep their power
    spectra and their cross spectrum, hence their coherence and phase relation, exactly; y keeps
    its power spectrum and is independent of both.  This is the null of "y is unrelated to x1 and
    x2, which are related to each other as in the data", the one RP2 and RM2 need where x1 and x2
    share a driver.  `conditional=False`: three independent sets of phases, the data-coloured
    counterpart of `wct3_significance`'s null (no coherence between x1 and x2 is kept).

    Null `null='ar1'`, `conditional=True`: y is red noise, the AR(1) series of
    `wct_surrogate_significance(null='ar1')` with y's own g, m and sigma, and x1 and x2 are held at
    the data in every triple: the standardised series exactly as `partial_wct` transforms them.  The
    null is "y is red noise unrelated to x1 and x2, and x1 and x2 are as observed": the relation
    between x1 and x2 is kept exactly, not just their cross spectrum, and no model of the drivers is
    needed (which is why it is preferred here to a fitted VAR(1) pair).  `conditional=False`: three
    independent AR(1) series, each with its own g, m and sigma (x2 under a counter stream of its
    own).  ValueError where a drawn series' g is not finite or |g| >= 1.

    Everything else as `wct_surrogate_significance`: arguments and errors of `partial_wct`, the
    data's length and cone of influence, the conventions of `wct_significance` for the levels, a
    point whose RP2 or RM2 is not finite is not counted, Philox stream keyed by (`seed`, triple
    number), `seed=None` draws the seed from numpy's global RNG, no cache, no progress bar.

    Phase randomisation assumes a stationary record and treats it as circular: a strong trend or a
    mismatch between the two ends is spread over all frequencies of the surrogates and biases the
    level, so detrend the series first (as the samples do).  The surrogates are Gaussian-like
    whatever the data's amplitude distribution (no amplitude adjustment)."""
    p, prob = _surrogate_problem((y, x1, x2), dt, dj, s0, J, wavelet, normalize, precision)
    hist = _surrogate_histogram(p, prob, _coherence_null(null, p, normalize, conditional), _surrogate_seed(seed),
                                0, mc_count)
    return _mc_levels(prob, hist[0], significance_level), _mc_levels(prob, hist[1], significance_level)


def _smooth_device(W, dt, dj, scales, deltaj0, wavelet=None):
    """Morlet.smooth on the GPU (reference mothers.py:61-104); with `wavelet` (Paul / DOG, opt-in)
    the same operator with that wavelet's time filter."""
    W = np.asarray(W)
    scales = np.asarray(scales, dtype=float)
    klen = int(np.round(deltaj0 / dj * 2))
    if klen < 1:
        # deltaj0 = -1 (f0 != 6): the reference fails inside rect()
        raise ValueError('smoothing window undefined for this wavelet (deltaj0 = -1)')
    eng = _engine.default_engine()
    with eng.lock:
        _sync_padding(eng, W.shape[1])
        with _smoothing_filter(eng, wavelet if wavelet is not None else Morlet(6), scales, dt, W.shape[1]):
            if np.isreal(W).all():
                return eng.smooth(np.ascontiguousarray(W.real, dtype=np.float64), dt, scales, klen)
            return eng.smooth(np.ascontiguousarray(W, dtype=np.complex128), dt, scales, klen)


def _check_parameter_wavelet(wavelet):
    """Strings map to default-constructed mother wavelets, anything else is returned as
    is (reference wavelet.py:650-663); unknown names raise KeyError."""
    mothers = {'morlet': Morlet, 'paul': Paul, 'dog': DOG, 'mexicanhat': MexicanHat, 'morse': Morse}
    if isinstance(wavelet, str):
        return mothers[wavelet]()
    return wavelet
