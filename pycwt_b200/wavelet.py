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
from .mothers import Morlet, Paul, DOG, MexicanHat

_PRECISIONS = {'fp64': _engine.F64, 'f64': _engine.F64, 'float64': _engine.F64,
               'fp32': _engine.F32, 'f32': _engine.F32, 'float32': _engine.F32}


def _precision():
    """Arithmetic of the engine: fp64 (default, matches the reference) or fp32 via the
    CWTB_PRECISION environment variable."""
    return _PRECISIONS[os.environ.get('CWTB_PRECISION', 'fp64').lower()]


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


def xwt(y1, y2, dt, dj=1/12, s0=-1, J=-1, significance_level=0.95,
        wavelet='morlet', normalize=True):
    """Cross wavelet transform W1 * conj(W2) (reference wavelet.py:316-419).

    Both transforms and the conjugate product (fused into the second transform's output
    pass) run on the GPU.  Returns (W12, coi, freq, signif)."""
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
    eng = _engine.default_engine()
    with eng.lock:
        _sync_padding(eng, n0)
        W12 = eng.xwt(y1n, y2n, dt, sj, *_family_of(wavelet))
    coi = (n0 / 2 - np.abs(np.arange(0, n0) - (n0 - 1) / 2))
    coi = wavelet.flambda() * wavelet.coi() * dt * coi

    if normalize:
        std1 = std2 = 1.
    a1, _, _ = ar1(y1)
    a2, _, _ = ar1(y2)
    Pk1 = ar1_spectrum(freq * dt, a1)
    Pk2 = ar1_spectrum(freq * dt, a2)
    dof = wavelet.dofmin
    PPF = chi2.ppf(significance_level, dof)
    signif = (std1 * std2 * (Pk1 * Pk2) ** 0.5 * PPF / dof)
    return W12, coi, freq, signif


def _family_of(wavelet):
    spec = _engine_family(wavelet)
    if spec is None:
        raise NotImplementedError(
            'xwt/wct on the GPU need a Morlet, Paul or DOG mother wavelet')
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


def wct(y1, y2, dt, dj=1/12, s0=-1, J=-1, sig=True,
        significance_level=0.95, wavelet='morlet', normalize=True, **kwargs):
    """Wavelet coherence (reference wavelet.py:422-528).

    Returns (WCT, aWCT, coi, freq, sig).  The two transforms, the |W|^2/s and W12/s
    products, the Gaussian time smoothing, the scale boxcar and the coherence ratio run
    on the GPU; `sig` comes from wct_significance (GPU Monte-Carlo) when sig=True."""
    wavelet = _check_parameter_wavelet(wavelet)
    if not hasattr(wavelet, 'smooth'):
        # same failure mode as the reference for Paul / DOG (no smoothing operator)
        raise AttributeError("'{}' object has no attribute 'smooth'".format(
            type(wavelet).__name__))
    if s0 == -1:
        s0 = 2 * dt / wavelet.flambda()
    if J == -1:
        J = int(np.round(np.log2(y1.size * dt / s0) / dj))  # y1.size: ndarray required, as in the reference
    y1, y1n, _ = _standardise(y1, normalize)
    y2, y2n, _ = _standardise(y2, normalize)
    n0 = y1n.size
    sj, freq = _resolve_scales(n0, dt, dj, s0, J, wavelet, None)
    eng = _engine.default_engine()
    klen = _boxcar_len(wavelet, dj)
    if klen < 1:
        raise ValueError('smoothing window undefined for this wavelet (deltaj0 = -1)')
    with eng.lock:
        _sync_padding(eng, len(y1n))
        with _smoothing_filter(eng, wavelet, sj, dt, len(y1n)):
            WCT, aWCT = eng.wct(y1n, y2n, dt, dj, sj, *_family_of(wavelet), boxcar_len=klen)
    coi = (n0 / 2 - np.abs(np.arange(0, n0) - (n0 - 1) / 2))
    coi = wavelet.flambda() * wavelet.coi() * dt * coi
    if sig:
        a1, b1, c1 = ar1(y1)
        a2, b2, c2 = ar1(y2)
        sig = wct_significance(a1, a2, dt=dt, dj=dj, s0=s0, J=J,
                               significance_level=significance_level,
                               wavelet=wavelet, **kwargs)
    else:
        sig = np.asarray([0])
    return WCT, aWCT, coi, freq, sig


def _mc_problem(dt, dj, s0, J, wavelet):
    """Geometry of the Monte-Carlo coherence problem (reference wavelet.py:588-607): surrogate
    length, scales, cone-of-influence mask, last valid scale and the sig95 template."""
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


def _mc_histogram(prob, dt, dj, wavelet, draw, indices, progress=False, engine=None):
    """1000-bin histograms of the coherence of the surrogate pairs draw(i), i in `indices`
    (reference wavelet.py:609-630), accumulated on the GPU: int64 [S, nbins]."""
    N, sj, nbins = prob['N'], prob['sj'], prob['nbins']
    hist = np.zeros((sj.size, nbins), dtype=np.int64)
    eng = engine or _engine.default_engine()
    fam = _family_of(wavelet)
    indices = list(indices)
    batch = max(1, min(len(indices), int((256 << 20) // (16 * N)) or 1))
    bar = tqdm(total=len(indices), disable=not progress)
    for b0 in range(0, len(indices), batch):
        idx = indices[b0:b0 + batch]
        noise = np.empty((len(idx), 2, N))
        for k, i in enumerate(idx):
            noise[k, 0], noise[k, 1] = draw(i)
        with eng.lock:
            _sync_padding(eng, N)
            with _smoothing_filter(eng, wavelet, sj, dt, N):
                eng.wct_mc(noise, dt, dj, sj, fam[0], fam[1], _boxcar_len(wavelet, dj), prob['mask'],
                           prob['maxscale'], nbins, hist)
        bar.update(len(idx))
    bar.close()
    return hist


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


def _mc_histogram_seeded(prob, dt, dj, wavelet, seed, first, count, engine=None):
    """The same histograms with the surrogates drawn on the device (Philox stream keyed by
    (seed, pair number)): no host RNG, no noise H2D."""
    sj, nbins = prob['sj'], prob['nbins']
    hist = np.zeros((sj.size, nbins), dtype=np.int64)
    eng = engine or _engine.default_engine()
    fam = _family_of(wavelet)
    with eng.lock:
        _sync_padding(eng, prob['N'])
        with _smoothing_filter(eng, wavelet, sj, dt, prob['N']):
            eng.wct_mc_seeded(seed, first, count, prob['N'], dt, sj, fam[0], fam[1], _boxcar_len(wavelet, dj),
                              prob['mask'], prob['maxscale'], nbins, hist)
    return hist


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
    on-disk cache keeps the reference's key and format (~/.cache/pycwt/<key>.gz)."""
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

        hist = _mc_histogram(prob, dt, dj, wavelet, draw, range(mc_count), progress)
    else:
        hist = _mc_histogram_seeded(prob, dt, dj, wavelet, seed, 0, mc_count)
    sig95 = _mc_levels(prob, hist, significance_level)

    if cache:
        np.savetxt('{}/{}.gz'.format(cache_dir, cache_file), sig95)
    return sig95


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
    mothers = {'morlet': Morlet, 'paul': Paul, 'dog': DOG, 'mexicanhat': MexicanHat}
    if isinstance(wavelet, str):
        return mothers[wavelet]()
    return wavelet
