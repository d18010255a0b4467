"""Device-resident transform and its derived products (SURVEY 8f rank 2).

`pycwt.cwt` has to hand the caller a complex128 array of S x N coefficients; at the north-star
size that is 4.3 GB over PCIe for a few ms of GPU work.  What the reference's sample scripts
then do with W (pycwt/sample/simple_sample.py:64-96) are reductions of |W|^2:

    power        = |W|^2                      (optionally rectified: / s_j, Liu et al. 2007,
                                               docs/tutorial/cwt.md:49-53)
    glbl_power   = power.mean(axis=1)         (simple_sample.py:79)
    scale_avg    = dj*dt/Cdelta * sum_{j in band} power[j] / s_j      (:88-91, TC98 eq. 24)
    iwave        = icwt(W, ...)               (:60)

`cwt_resident` runs the same transform as `cwt` but keeps W in HBM and returns a handle whose
methods evaluate those products on the device, so only O(S) or O(N) numbers cross the bus.
The handle is valid until the next transform on the same engine.

`wct_resident` does the same for the wavelet coherence, `xwt_resident` for the cross-wavelet
transform, `wct3_resident` for the partial and multiple coherence of three series and
`power_resident` for the wavelet power of one series with its tests against surrogates (see the
second half of this module).
"""
import collections

import numpy as np

from . import _engine
from . import helpers as _helpers
from .helpers import ar1, fft, fft_kwargs
from .wavelet import (_ar1_params, _check_parameter_wavelet, _coherence_null, _coherence_precision, _coi,
                      _mc_levels, _nan_rows, _null_kind, _precision, _resolve_scales, _standardise,
                      _surrogate_histogram, _surrogate_problem, _surrogate_seed,
                      _sync_padding, _wct_on_device, _wct_problem, _wct_significance,
                      _xwt_on_device, _xwt_problem, _xwt_signif, wct3_significance,
                      wct3_surrogate_significance, wct_surrogate_significance)

__all__ = ['cwt_resident', 'ResidentTransform', 'wct_resident', 'ResidentCoherence',
           'xwt_resident', 'ResidentCrossWavelet', 'wct3_resident', 'ResidentCoherence3',
           'power_resident', 'ResidentPower', 'FdrResult', 'ClusterResult']


def _coi_ranges(wavelet, dt, n0, period):
    """Columns inside the cone of influence, per scale: period_j <= coi[n] holds on one centred
    range [lo_j, hi_j)."""
    c = wavelet.flambda() * wavelet.coi() * dt
    # coi[n] = c * (n0/2 - |n - (n0-1)/2|) >= period  <=>  |n - (n0-1)/2| <= n0/2 - period/c
    half = n0 / 2 - period / c
    mid = (n0 - 1) / 2
    lo = np.ceil(mid - half - 1e-12).astype(np.int64)
    hi = np.floor(mid + half + 1e-12).astype(np.int64) + 1
    empty = half < 0
    lo = np.clip(lo, 0, n0)
    hi = np.clip(hi, 0, n0)
    hi[empty] = lo[empty]
    return lo, hi


def _live(method):
    """Product methods run as one engine transaction: check that this transform is still the
    resident one and evaluate, under the engine lock."""
    import functools

    @functools.wraps(method)
    def wrapper(self, *args, **kwargs):
        with self.engine.lock:
            self._check_live()
            return method(self, *args, **kwargs)
    return wrapper


class _Resident(object):
    """What the handles of one resident [S, n0] product share.  A subclass names its frequency
    attribute (`_FREQ`), the engine method that returns its product's serial (`_SERIAL`) and the
    message once that serial has moved on (`_GONE`)."""

    def __init__(self, engine, wavelet, n0, dt, dj, sj, precision, serial):
        self.engine = engine
        self.wavelet = wavelet
        self.n0 = int(n0)
        self.dt = float(dt)
        self.dj = dj
        self.scales = sj
        self.precision = precision
        self._serial = serial
        self._coi = None

    # O(n0) host array of the `cwt` return tuple, built on first use
    @property
    def coi(self):
        if self._coi is None:
            self._coi = _coi(self.wavelet, self.dt, self.n0)
        return self._coi

    @property
    def shape(self):
        return (len(self.scales), self.n0)

    @property
    def period(self):
        return 1.0 / np.asarray(getattr(self, self._FREQ))

    def coi_ranges(self):
        """Columns inside the cone of influence, per scale (see `_coi_ranges`)."""
        return _coi_ranges(self.wavelet, self.dt, self.n0, self.period)

    def _check_live(self):
        if getattr(self.engine, self._SERIAL)() != self._serial:
            raise _engine.EngineError(self._GONE)

    def _band(self, period_min, period_max):
        """The scales with period_min <= period < period_max."""
        per = self.period
        return (per >= period_min) & (per < period_max)

    def _band_weights(self, period_min, period_max, factor=1.0):
        """(band, factor * dj * dt / Cdelta / s_j on the band and 0 elsewhere): the weights of
        TC98 eq. 24 (simple_sample.py:87-91)."""
        if self.wavelet.cdelta == -1:
            raise ValueError('Cdelta not defined for this wavelet')
        sel = self._band(period_min, period_max)
        w = np.where(sel, 1.0 / np.asarray(self.scales, dtype=float), 0.0)
        return sel, w * (factor * self.dj * self.dt / self.wavelet.cdelta)


class _ResidentSlot(_Resident):
    """A product in a device buffer of its own, freed by the engine method `_RELEASE`."""

    def release(self):
        """Free the device buffer (16 bytes per scale and time point for a coherence, 24 for a
        partial and multiple coherence, 16 or 8 for a cross spectrum or a power, whose tests add 4
        for the counts and 4 for the cluster labels).  The handle is invalid afterwards; releasing
        an invalid handle does nothing."""
        with self.engine.lock:
            if getattr(self.engine, self._SERIAL)() == self._serial:
                getattr(self.engine, self._RELEASE)()


class ResidentTransform(_Resident):
    """W[S, n0] of one `cwt_resident` call, resident on the device."""

    _FREQ, _SERIAL = 'freqs', 'job_serial'
    _GONE = "this transform is no longer resident: another transform has run on the same engine"

    def __init__(self, engine, wavelet, n0, dt, dj, sj, freqs, precision, serial):
        super(ResidentTransform, self).__init__(engine, wavelet, n0, dt, dj, sj, precision, serial)
        self.freqs = freqs
        self.npad = fft_kwargs(range(self.n0))['n']       # transform length (helpers.py:15-30)
        self._fftfreqs = None

    @property
    def fftfreqs(self):
        if self._fftfreqs is None:
            npad = self.npad
            self._fftfreqs = (2 * np.pi * fft.fftfreq(npad, self.dt))[1:npad // 2] / (2 * np.pi)
        return self._fftfreqs

    # -- the products --------------------------------------------------------------------
    @_live
    def wave(self):
        """The coefficients themselves (complex128, S x n0): the expensive fetch."""
        return self.engine.get_w(len(self.scales), self.n0, self.precision)

    @_live
    def fft(self):
        """Normalised signal spectrum, as returned by `cwt` (wavelet.py:123)."""
        return self.engine.signal_fft()

    @_live
    def power(self, rectify=False, variance=None):
        """|W|^2, divided by the scale if `rectify` and by `variance` if given."""
        rs = None
        if rectify or variance is not None:
            rs = np.ones(len(self.scales))
            if rectify:
                rs = rs / np.asarray(self.scales, dtype=float)
            if variance is not None:
                rs = rs / float(variance)
        return self.engine.power(len(self.scales), self.n0, rs)

    @_live
    def window(self, rows=slice(None), cols=slice(None)):
        """W[rows, cols] (complex128) for two slices with steps >= 1, gathered on the device: only
        the sub-grid crosses the bus."""
        return _field_window(self.engine, _engine.FIELD_W, self.shape, rows, cols)

    @_live
    def global_power(self, inside_coi=False, signif=None):
        """Time mean of |W|^2 per scale (`power.mean(axis=1)`); with `inside_coi` only over
        the columns where the period is inside the cone of influence, with `signif` (power units,
        as `significance()` returns it) only over the points where |W|^2 > signif[j] (none where
        signif[j] is NaN).  NaN for a scale without points."""
        if signif is None:
            if not inside_coi:
                return self.engine.global_power(len(self.scales))
            lo, hi = self.coi_ranges()
            return self.engine.global_power_ranges(lo, hi)
        lo, hi = _column_ranges(self, inside_coi)
        st = self.engine.field_row_stats(_engine.FIELD_W, lo, hi, _power_threshold(self, signif))
        return _ratio(st[:, 1], st[:, 0])

    @_live
    def significant_fraction(self, signif):
        """Per scale, the fraction of the points inside the cone of influence where
        |W|^2 > signif[j] (power units); NaN for a scale without such points."""
        lo, hi = self.coi_ranges()
        st = self.engine.field_row_stats(_engine.FIELD_W, lo, hi, _power_threshold(self, signif))
        return _ratio(st[:, 0], hi - lo)

    @_live
    def scale_avg_power(self, period_min, period_max, variance=1.0):
        """Scale-averaged power over period_min <= period < period_max (TC98 eq. 24 as in
        simple_sample.py:87-91): variance * dj * dt / Cdelta * sum_j |W_j|^2 / s_j."""
        _, w = self._band_weights(period_min, period_max, variance)
        return self.engine.scale_avg_power(w)

    @_live
    def icwt(self):
        """Inverse transform of the resident coefficients (wavelet.py:169-170)."""
        return _inverse(self, self.engine.icwt_sum())

    @_live
    def reconstruct(self, period_min=-np.inf, period_max=np.inf, inside_coi=False, signif=None):
        """The inverse transform summed over the selected points only (wavelet filtering, TC98 §5
        eq. 29): x[n] = dj sqrt(dt) / (Cdelta psi(0)) * sum over the selected (j, n) of
        Re W[j, n] / sqrt(s_j), length n0, with the factor and the dtype of `icwt()`.  A point is
        selected where every condition given holds: period_min <= period_j < period_max (ValueError
        when no scale is in the band), inside the cone of influence if `inside_coi`, |W|^2 > signif[j]
        if `signif` is given (power units; a NaN entry selects none of its scale).  A column without a
        selected point is 0.  With everything selected it equals `icwt()` to rounding: the sums run in
        another order.  W is read on the device; n0 numbers cross the bus."""
        thr = None if signif is None else _power_threshold(self, signif)
        w, lo, hi = _reconstruct_rows(self, period_min, period_max, inside_coi)
        return _inverse(self, self.engine.field_reconstruct(_engine.FIELD_W, w, lo, hi, thr))


def _inverse(h, red):
    """dj sqrt(dt) / (Cdelta psi(0)) * red: the inverse transform of a sum of Re W / sqrt(s_j)."""
    fac = h.dj * np.sqrt(h.dt) / (h.wavelet.cdelta * h.wavelet.psi(0))
    if not np.iscomplexobj(fac):
        return fac * red
    # complex factor (Morlet / Paul: psi(0) is complex in the reference, so is its icwt): one pass per
    # component instead of NumPy's promote-then-multiply over N points
    out = h.engine.result_array(red.shape, np.complex128)   # pooled: no first-touch page faults per call
    np.multiply(red, np.real(fac), out=out.real)
    np.multiply(red, np.imag(fac), out=out.imag)
    return out


def _reconstruct_rows(h, period_min, period_max, inside_coi):
    """(weights, lo, hi) of a reconstruction: 1 / sqrt(s_j) on the band and 0 elsewhere, and the
    columns of each row."""
    if h.wavelet.cdelta == -1:
        raise ValueError('Cdelta not defined for this wavelet')
    sel = h._band(period_min, period_max)
    if not sel.any():
        raise ValueError("no scale with %r <= period < %r" % (period_min, period_max))
    w = np.where(sel, 1.0 / np.sqrt(np.asarray(h.scales, dtype=float)), 0.0)
    lo, hi = _column_ranges(h, inside_coi)
    return w, lo, hi


def _engine_wavelet(wavelet, name):
    """(wavelet, (family, param)) of a resident transform: TypeError for a wavelet the engine does
    not evaluate itself."""
    wavelet = _check_parameter_wavelet(wavelet)
    spec = wavelet._engine_spec() if hasattr(wavelet, '_engine_spec') else None
    if spec is None:
        # duck-typed objects, subclasses that override psi_ft, non-integer or out-of-range orders
        raise TypeError("%s needs one of the analytic families the engine evaluates "
                        "itself: Morlet(f0), Paul(m) or DOG(m) with an integer order in [1, 64], "
                        "or Morse(ga, be), with the stock psi_ft" % name)
    return wavelet, spec


def _kept_scales(n0, dt, dj, s0, J, wavelet, freqs):
    """(scales, freqs) of `cwt` for an n0-point series: without the rows the reference drops as
    all-NaN (Paul at very large scales)."""
    sj, freqs = _resolve_scales(n0, dt, dj, s0, J, wavelet, freqs)
    npad = fft_kwargs(range(n0))['n']
    keep = ~_nan_rows(wavelet, np.asarray(sj, dtype=float), npad, dt)
    if not keep.any():
        raise ValueError("every scale of this transform is NaN in the reference")
    return sj[keep], freqs[keep]


def cwt_resident(signal, dt, dj=1/12, s0=-1, J=-1, wavelet='morlet', freqs=None, engine=None):
    """Same transform as `cwt` (reference wavelet.py:13-124), W kept on the device.

    Returns a `ResidentTransform`.  Scales whose row the reference would drop as all-NaN
    (Paul at very large scales) are dropped here as well, so `.scales` / `.freqs` equal the
    ones `cwt` returns."""
    wavelet, spec = _engine_wavelet(wavelet, "cwt_resident")
    n0 = len(signal)
    sj, freqs = _kept_scales(n0, dt, dj, s0, J, wavelet, freqs)
    eng = engine or _engine.default_engine()
    sig = np.asarray(signal)
    if sig.dtype != np.float32:
        sig = np.asarray(sig, dtype=np.float64)
    family, param = spec
    precision = _precision()
    with eng.lock:
        if _sync_padding(eng, n0):
            precision = _engine.F64
        eng.cwt(sig, dt, sj, family, param, precision, fetch=False)
        serial = eng.job_serial()
    return ResidentTransform(eng, wavelet, n0, dt, dj, sj, freqs, precision, serial)


# ---- resident coherence ------------------------------------------------------------------------
# `wct` hands the caller two float64 [S, n0] fields; at config 4 that is 600 MB over PCIe for a few
# ms of GPU work.  What the reference's sample script (pycwt/sample/sample_xwt.py) and Grinsted et
# al. (2004) then do with them are contours of WCT / sig95, phase arrows on a sub-grid and
# reductions over regions of the (scale, time) plane.  `wct_resident` runs the same pipeline as
# `wct(sig=False)` and keeps WCT and aWCT on the device, in a buffer of their own: the handle stays
# valid across later cwt / xwt / wct / Monte-Carlo calls, until the next `wct_resident` on the same
# engine or `release()`.

MeanPhase = collections.namedtuple('MeanPhase', 'angle strength count')


def _slice_range(s, n, name):
    """(start, count, step) of a slice with step >= 1 over range(n)."""
    if not isinstance(s, slice):
        raise ValueError("%s must be a slice, got %r" % (name, s))
    if s.step is not None and (not isinstance(s.step, (int, np.integer)) or isinstance(s.step, bool)
                               or s.step < 1):
        raise ValueError("%s: the step must be an integer >= 1, got %r" % (name, s.step))
    try:
        start, stop, step = s.indices(n)
    except TypeError as exc:
        raise ValueError("%s: %s" % (name, exc))
    return start, len(range(start, stop, step)), step


def _field_window(engine, field, shape, rows, cols):
    """field[rows, cols] of a resident complex field, complex128, gathered on the device."""
    S, n0 = shape
    r0, nr, rs = _slice_range(rows, S, 'rows')
    c0, nc, cs = _slice_range(cols, n0, 'cols')
    if nr == 0 or nc == 0:
        return np.empty((nr, nc), dtype=np.complex128)
    return engine.field_window(field, r0, nr, rs, c0, nc, cs)


def _column_ranges(h, inside_coi):
    """Per scale, the columns inside the cone of influence, or every column."""
    if inside_coi:
        return h.coi_ranges()
    S = len(h.scales)
    return np.zeros(S, dtype=np.int64), np.full(S, h.n0, dtype=np.int64)


def _power_threshold(h, signif):
    """A per-scale threshold on |F|^2: one entry per scale, none negative (NaN selects no point)."""
    thr = np.asarray(signif, dtype=float)
    if thr.shape != (len(h.scales),):
        raise ValueError("signif must have one entry per scale (%d), got shape %s"
                         % (len(h.scales), thr.shape))
    if (thr < 0).any():
        raise ValueError("signif must not be negative")
    return thr


def _mean_phase(cnt, c, s, per_scale):
    """MeanPhase of per-scale point counts and sums of cos / sin of the phase."""
    if not per_scale:
        cnt, c, s = cnt.sum(), c.sum(), s.sum()
    angle = np.where(cnt > 0, np.arctan2(s, c), np.nan)
    strength = _ratio(np.hypot(c, s), cnt)
    if per_scale:
        return MeanPhase(angle, strength, cnt.astype(np.int64))
    return MeanPhase(float(angle), float(strength), int(cnt))


def _ratio(num, den):
    """num / den, NaN where den == 0."""
    num = np.asarray(num, dtype=float)
    den = np.asarray(den, dtype=float)
    with np.errstate(divide='ignore', invalid='ignore'):
        return np.where(den > 0, num / np.where(den > 0, den, 1.0), np.nan)


# ---- point-wise tests against phase-randomised surrogates --------------------------------------
# `surrogate_test` runs the M surrogate units 0 .. M - 1 of `wct_surrogate_significance` /
# `wct3_surrogate_significance` (same seed, same units) and, in the same device run, counts per
# point k[s, n] = #{i : R2_i[s, n] >= R2_obs[s, n]} (a non-finite R2_i counts) into counters that
# live with the resident product.  p = (1 + k) / (1 + M); NaN where R2_obs is not finite.

FdrResult = collections.namedtuple('FdrResult', 'alpha rejected tested')

_MAX_UNITS = 2 ** 31 - 1    # units of one counting call (a C int); the counters are uint32


def _kmax(alpha, M):
    """The largest k with (1 + k) / (1 + M) <= alpha (-1: none), evaluated in double."""
    if isinstance(alpha, bool) or not np.isscalar(alpha) or not 0 < alpha <= 1:
        raise ValueError("alpha must lie in (0, 1], got %r" % (alpha,))
    k = min(M, max(-1, int(np.floor(alpha * (1 + M))) - 1))
    while k < M and (1 + (k + 1)) / (1 + M) <= alpha:
        k += 1
    while k >= 0 and (1 + k) / (1 + M) > alpha:
        k -= 1
    return k


def _fdr(hist, M, q, method):
    """Benjamini-Hochberg / -Yekutieli step-up test of the p-values (1 + k) / (1 + M) from their
    histogram over k.  At the value of k the rank is the cumulative count H(k) (ties), and the
    adjusted p-values are formed as scipy.stats.false_discovery_control forms them."""
    m = int(hist.sum())
    if m == 0:
        return FdrResult(0.0, 0, 0)
    k = np.flatnonzero(hist)
    rank = np.cumsum(hist)[k].astype(float)
    p = (1 + k) / (1 + M)
    adj = p * (m / rank)
    if method == 'by':
        adj = adj * np.sum(1 / np.arange(1, m + 1, dtype=float))
    ok = np.flatnonzero(adj <= q)
    if ok.size == 0:
        return FdrResult(0.0, 0, m)
    top = ok[-1]
    return FdrResult(float(p[top]), int(rank[top]), m)


# ---- cluster tests against phase-randomised surrogates -------------------------------------------
# `cluster_test(sig, mc_count=M, seed=s)` selects the points with a finite R > sig[j] (inside the
# cone of influence by default) in the resident map and in the map of each surrogate unit 0 .. M - 1
# of `surrogate_significance(mc_count=M, seed=s)`, labels the 8-connected clusters of each on the
# device and weighs a cluster by its area normalised by the reproducing kernel's width,
# A = sum dj dt / s_j over its points.  Exactly: a point of row j weighs the integer
# q_j = floor(2^32 s_min / s_j + 1/2) (double arithmetic), Q = sum q_j in uint64, and
# A = (dj dt / s_min) Q / 2^32.  p_c = (1 + #{u : Qmax_u >= Q_c}) / (1 + M), Qmax_u the largest Q of
# unit u (0 without clusters): the max-statistic test, which controls the family-wise error over
# the clusters (Nichols & Holmes 2002; Maris & Oostenveld 2007).

ClusterResult = collections.namedtuple('ClusterResult', 'area points rows cols pvalue null_max')


def _cluster_weights(h):
    """(q uint64 [S], the area of one unit of Q)."""
    sj = np.asarray(h.scales, dtype=float)
    smin = sj.min()
    q = np.floor(2.0 ** 32 * smin / sj + 0.5).astype(np.uint64)
    return q, h.dj * h.dt / smin / 2.0 ** 32


class _SurrogateTest(object):
    """The point-wise and cluster tests of a resident product: the counts of its last
    `surrogate_test`, the clusters of its last `cluster_test`, and what is read from them.  A
    subclass names the engine's clusters of its product (`_CLUSTERS`: False for the coherence, True
    for the partial and multiple coherence, `_engine.POWER` for the power, `_engine.CROSS` for the
    cross spectrum), passes its measure to the readers (None for the coherence, `_engine.POWER` /
    `_engine.CROSS` for the power / the cross spectrum) and runs its units on the device
    (`_count_units`, `_cluster_units`)."""

    _UNTESTED = ("no surrogate test has counted for this product: call surrogate_test first")
    surrogate_seed = None     # seed, M and null of the last surrogate_test
    surrogate_units = None
    surrogate_null = None

    def _seed_of_run(self, mc_count, seed):
        """The checks of a surrogate run of units 0 .. mc_count - 1, and its seed."""
        if isinstance(mc_count, bool) or not isinstance(mc_count, (int, np.integer)) \
                or not 1 <= mc_count <= _MAX_UNITS:
            raise ValueError("mc_count must be an integer in [1, %d], got %r" % (_MAX_UNITS, mc_count))
        if bool(_helpers._FFT_NEXT_POW2) != self._padding:
            raise ValueError("the FFT padding mode has changed since this product was computed: its "
                             "counts would not compare like with like")
        return _surrogate_seed(seed)

    def _cluster(self, sig, mc_count, seed, inside_coi, *args):
        """ClusterResult of a cluster test of units 0 .. mc_count - 1 (the caller holds the lock);
        `args` go to `_cluster_units`."""
        thr = self._threshold(sig)
        if thr is None:
            raise ValueError("cluster_test needs a per-scale threshold sig")
        seed = self._seed_of_run(mc_count, seed)
        lo, hi = _column_ranges(self, inside_coi)
        q, unit_area = _cluster_weights(self)
        qmax = self._cluster_units(seed, int(mc_count), thr, lo, hi, q, *args)
        Q, pts, box = self.engine.cluster_table(self._CLUSTERS)
        M = int(mc_count)
        reached = M - np.searchsorted(np.sort(qmax), Q, side='left')
        return ClusterResult(Q.astype(float) * unit_area, pts, box[:, 0:2], box[:, 2:4],
                             (1.0 + reached) / (1.0 + M), qmax.astype(float) * unit_area)

    def _cluster_labels(self, rows, cols):
        S, n0 = self.shape
        r0, nr, rs = _slice_range(rows, S, 'rows')
        c0, nc, cs = _slice_range(cols, n0, 'cols')
        if nr == 0 or nc == 0:
            return np.empty((nr, nc), dtype=np.int32)
        return self.engine.cluster_labels(self._CLUSTERS, r0, nr, rs, c0, nc, cs)

    def _count(self, mc_count, seed, null, *args):
        """What `_count_units` returns for a counting run of units 0 .. mc_count - 1 of `null` (the
        caller holds the lock)."""
        seed = self._seed_of_run(mc_count, seed)
        self.surrogate_seed = self.surrogate_units = self.surrogate_null = None
        out = self._count_units(seed, int(mc_count), null, *args)
        self.surrogate_seed, self.surrogate_units, self.surrogate_null = seed, int(mc_count), null
        return out

    def _units(self):
        if self.surrogate_units is None:
            raise _engine.EngineError(self._UNTESTED)
        return self.surrogate_units

    def _pvalues(self, measure, rows, cols):
        self._units()
        S, n0 = self.shape
        r0, nr, rs = _slice_range(rows, S, 'rows')
        c0, nc, cs = _slice_range(cols, n0, 'cols')
        if nr == 0 or nc == 0:
            return np.empty((nr, nc))
        return self.engine.pvalue_window(measure, r0, nr, rs, c0, nc, cs)

    def _cut_stats(self, measure, lo, hi, thr, alpha, want_phase=False):
        """Row stats over the points with p <= alpha (and R > thr where given)."""
        kmax = _kmax(alpha, self._units())
        return self.engine.pvalue_row_stats(measure, lo, hi, kmax, thr, want_phase)

    def _pvalue_fraction(self, measure, alpha):
        M = self._units()
        lo, hi = self.coi_ranges()
        sel = self.engine.pvalue_row_stats(measure, lo, hi, _kmax(alpha, M))[:, 0]
        tested = self.engine.pvalue_row_stats(measure, lo, hi, M)[:, 0]
        return _ratio(sel, tested)

    def _fdr_threshold(self, measure, q, method, inside_coi):
        if isinstance(q, bool) or not np.isscalar(q) or not 0 < q < 1:
            raise ValueError("q must lie in (0, 1), got %r" % (q,))
        if method not in ('bh', 'by'):
            raise ValueError("method must be 'bh' or 'by', got %r" % (method,))
        M = self._units()
        lo, hi = _column_ranges(self, inside_coi)
        return _fdr(self.engine.count_hist(measure, lo, hi, M + 1), M, q, method)


class _CoherenceTest(_SurrogateTest):
    """The units of the coherence products' tests: the surrogates of `_coherence_null` ('phase' or
    'ar1', conditional or not for three series) through the whole coherence pipeline, with the
    Monte-Carlo histograms of `_surrogate_problem`."""

    def _problem(self, null, conditional):
        """(p, prob, the engine's null) of a run."""
        _null_kind(null)
        p, prob = _surrogate_problem(self._y, self.dt, self.dj, self.s0, self.J, self.wavelet,
                                     self.normalize, self.precision)
        return p, prob, _coherence_null(null, p, self.normalize, conditional)

    def _count_units(self, seed, M, null, conditional=True):
        """(prob, hist) of a counting run."""
        p, prob, cnull = self._problem(null, conditional)
        hist = _surrogate_histogram(p, prob, cnull, seed, 0, M, engine=self.engine,
                                    serial=self._serial)
        return prob, hist

    def _cluster_units(self, seed, M, thr, lo, hi, q, null, conditional, measure):
        """The units' largest cluster sums, uint64 [M]."""
        p, prob, cnull = self._problem(null, conditional)
        nser = len(p.yns)
        hist = np.zeros((nser - 1, p.sj.size, prob['nbins']), dtype=np.int64)
        eng = self.engine

        def call(*a, boxcar_len, precision):
            dt, _, sj, family, param = a[nser:]
            return eng.cluster_test(np.stack(a[:nser]), cnull, seed, 0, M, dt, sj, family,
                                    param, boxcar_len, prob['mask'], prob['maxscale'], prob['nbins'],
                                    *hist, serial=self._serial, thr=thr, lo=lo, hi=hi, q=q,
                                    measure=measure, precision=precision)

        return _wct_on_device(eng, p, call)


class ResidentCoherence(_CoherenceTest, _ResidentSlot):
    """WCT and aWCT [S, n0] of one `wct_resident` call, resident on the device.

    Point-wise test: `surrogate_test(mc_count=M, seed=seed)` runs the surrogate pairs 0 .. M - 1 of
    `wct_surrogate_significance(..., mc_count=M, seed=seed)` and counts, per point, the pairs whose
    coherence reaches the observed one, k[s, n] = #{i : WCT_i[s, n] >= WCT[s, n]} (a non-finite
    WCT_i counts: the conservative choice), on every row and column, the cone of influence included
    (the surrogates have the data's length and the same edge effects).  p = (1 + k) / (1 + M)
    (Davison & Hinkley 1997; North et al. 2002), so the smallest p is 1 / (M + 1); NaN where WCT is
    not finite, and such points are left out of every fraction and count.  A selection p <= alpha is
    the integer cut k <= kmax, kmax the largest k with (1 + k) / (1 + M) <= alpha in double.  The
    counts take 4 bytes per scale-point on the device and live until the next `surrogate_test`,
    `release()` or `wct_resident` on the same engine."""

    _FREQ, _SERIAL, _RELEASE = 'freq', 'coherence_serial', 'coherence_release'
    _CLUSTERS = False
    _GONE = ("this coherence is no longer resident: it was released or another wct_resident has "
             "run on the same engine")

    def __init__(self, engine, problem, normalize, precision, serial):
        p = problem
        super(ResidentCoherence, self).__init__(engine, p.wavelet, p.n0, p.dt, p.dj, p.sj,
                                                precision, serial)
        self.s0 = p.s0
        self.J = p.J
        self.freq = p.freq
        self.normalize = normalize
        self._y = tuple(np.array(y, copy=True) for y in p.ys)   # raw series, for ar1 and surrogates
        self._padding = bool(_helpers._FFT_NEXT_POW2)

    def _threshold(self, sig95):
        if sig95 is None:
            return None
        thr = np.asarray(sig95, dtype=float)
        if thr.shape != (len(self.scales),):
            raise ValueError("sig95 must have one entry per scale (%d), got shape %s"
                             % (len(self.scales), thr.shape))
        return thr

    # -- the products --------------------------------------------------------------------
    @_live
    def coherence(self):
        """WCT (float64, S x n0), as returned by `wct(..., sig=False)`: the expensive fetch."""
        S, n0 = self.shape
        return self.engine.coherence_window(0, S, 1, 0, n0, 1, want_angle=False)[0]

    @_live
    def phase(self):
        """aWCT (float64, S x n0), as returned by `wct(..., sig=False)`."""
        S, n0 = self.shape
        return self.engine.coherence_window(0, S, 1, 0, n0, 1, want_wct=False)[1]

    @_live
    def window(self, rows=slice(None), cols=slice(None)):
        """(WCT[rows, cols], aWCT[rows, cols]) for two slices with steps >= 1, gathered on the
        device: only the sub-grid crosses the bus (contour and phase-arrow plots)."""
        S, n0 = self.shape
        r0, nr, rs = _slice_range(rows, S, 'rows')
        c0, nc, cs = _slice_range(cols, n0, 'cols')
        if nr == 0 or nc == 0:
            return np.empty((nr, nc)), np.empty((nr, nc))
        return self.engine.coherence_window(r0, nr, rs, c0, nc, cs)

    @_live
    def significance(self, significance_level=0.95, mc_count=300, progress=True, cache=True,
                     seed=None):
        """Monte-Carlo significance level per scale, as `wct(..., sig=True)` computes it (lag-1
        autocorrelations of the raw series, this coherence's dt, dj, s0, J, wavelet and
        precision).  The coherence stays resident."""
        a1, _, _ = ar1(self._y[0])
        a2, _, _ = ar1(self._y[1])
        return _wct_significance(a1, a2, dt=self.dt, dj=self.dj, s0=self.s0, J=self.J,
                                 significance_level=significance_level, wavelet=self.wavelet,
                                 mc_count=mc_count, progress=progress, cache=cache, seed=seed,
                                 precision=self.precision)

    @_live
    def global_coherence(self, inside_coi=False, sig95=None, alpha=None):
        """Mean WCT per scale over the selected points: inside the cone of influence
        (period_j <= coi[n]) if `inside_coi`, where WCT[j, n] > sig95[j] if `sig95` is given
        (false where sig95[j] is NaN), where the p-value of the last `surrogate_test` is <= alpha if
        `alpha` is given (both: logical AND).  NaN for a scale without points."""
        lo, hi = _column_ranges(self, inside_coi)
        if alpha is not None:
            st = self._cut_stats(None, lo, hi, self._threshold(sig95), alpha)
        else:
            st = self.engine.coherence_row_stats(lo, hi, self._threshold(sig95))
        return _ratio(st[:, 1], st[:, 0])

    @_live
    def significant_fraction(self, sig95):
        """Per scale, the fraction of the points inside the cone of influence where
        WCT > sig95[j]; NaN for a scale without such points."""
        lo, hi = self.coi_ranges()
        st = self.engine.coherence_row_stats(lo, hi, self._threshold(sig95))
        return _ratio(st[:, 0], hi - lo)

    @_live
    def mean_phase(self, period_min=-np.inf, period_max=np.inf, inside_coi=True, sig95=None,
                   per_scale=False, alpha=None):
        """Circular mean of aWCT over the points of the scales with period_min <= period <
        period_max, inside the cone of influence if `inside_coi`, where WCT > sig95 if given and
        where the p-value of the last `surrogate_test` is <= alpha if given (Grinsted et al. 2004):
        MeanPhase(angle = atan2(sum sin, sum cos), strength = |sum e^{i aWCT}| / count, count), for
        the whole band or, with `per_scale`, per scale (arrays; NaN angle and strength where the
        count is 0)."""
        sel = self._band(period_min, period_max)
        lo, hi = _column_ranges(self, inside_coi)
        lo, hi = np.where(sel, lo, 0), np.where(sel, hi, 0)
        if alpha is not None:
            st = self._cut_stats(None, lo, hi, self._threshold(sig95), alpha, want_phase=True)
        else:
            st = self.engine.coherence_row_stats(lo, hi, self._threshold(sig95), want_phase=True)
        return _mean_phase(st[:, 0], st[:, 2], st[:, 3], per_scale)

    @_live
    def scale_avg(self, period_min, period_max):
        """Two length-n0 series over the scales with period_min <= period < period_max: the mean
        WCT and the circular mean phase atan2(sum sin aWCT, sum cos aWCT)."""
        sel = self._band(period_min, period_max)
        if not sel.any():
            raise ValueError("no scale with %r <= period < %r" % (period_min, period_max))
        out = self.engine.coherence_scale_avg(sel.astype(float))
        return out[0] / float(sel.sum()), np.arctan2(out[2], out[1])

    @_live
    def surrogate_significance(self, significance_level=0.95, mc_count=300, seed=None, null='phase'):
        """`wct_surrogate_significance` on this handle's series and arguments, against `null`
        ('phase' or 'ar1').  The coherence stays resident."""
        return wct_surrogate_significance(*self._y, dt=self.dt, dj=self.dj, s0=self.s0, J=self.J,
                                          significance_level=significance_level,
                                          wavelet=self.wavelet, normalize=self.normalize,
                                          mc_count=mc_count, seed=seed, precision=self.precision,
                                          null=null)

    @_live
    def surrogate_test(self, mc_count=300, seed=None, significance_level=0.95, null='phase'):
        """Run the surrogate pairs 0 .. mc_count - 1 of `null` once ('phase': phase-randomised
        surrogates of the two series, 'ar1': two independent red-noise series with the data's lag-1
        autocorrelations; see `wct_surrogate_significance`): count per point the pairs whose
        coherence reaches this one (kept on the device, replacing the counts of an earlier test) and
        return the per-scale levels, bit-identical to `surrogate_significance` with the same `seed`,
        `mc_count` and `null`.  `seed=None` draws the seed from numpy's global RNG; the seed, M and
        null are kept as `surrogate_seed`, `surrogate_units` and `surrogate_null`.  ValueError for
        mc_count outside [1, 2^31 - 1], an unknown null, an AR(1) null whose g is not finite or has
        |g| >= 1, or when the FFT padding mode differs from the one this coherence was computed
        with."""
        _null_kind(null)
        prob, hist = self._count(mc_count, seed, null)
        return _mc_levels(prob, hist[0], significance_level)

    @_live
    def pvalues(self, rows=slice(None), cols=slice(None)):
        """p[rows, cols] = (1 + k) / (1 + M) (float64) of the last `surrogate_test`, with the slicing
        of `window`; NaN where WCT is not finite."""
        return self._pvalues(None, rows, cols)

    @_live
    def pvalue_fraction(self, alpha):
        """Per scale, the fraction of the points inside the cone of influence (with a finite p) whose
        p <= alpha; NaN for a scale without such points."""
        return self._pvalue_fraction(None, alpha)

    @_live
    def fdr_threshold(self, q=0.05, method='bh', inside_coi=True):
        """False-discovery-rate control of the p-values of the last `surrogate_test`, over the points
        with a finite p inside the cone of influence (every such point with `inside_coi=False`):
        Benjamini & Hochberg (1995), `method='bh'`, or Benjamini & Yekutieli (2001), `'by'`.
        Returns FdrResult(alpha, rejected, tested): the largest p-value the step-up procedure rejects
        (0.0 if none; select with `pvalues() <= alpha`), the points rejected and the points tested.
        p takes only the values (1 + k) / (1 + M), so the procedure is decided exactly from a
        histogram of k (tied p-values take the rank of the last of them) and equals
        scipy.stats.false_discovery_control on the same p-values.  The points of a map are strongly
        dependent: BH controls the FDR under positive regression dependence (Benjamini &
        Yekutieli 2001), BY under any dependence, at the price of power."""
        return self._fdr_threshold(None, q, method, inside_coi)

    @_live
    def cluster_test(self, sig, mc_count=300, seed=None, inside_coi=True, null='phase'):
        """Cluster (areawise) test of this coherence against the surrogate pairs 0 .. mc_count - 1 of
        `surrogate_significance(mc_count=mc_count, seed=seed, null=null)` (Maraun et al. 2007; Schulte et
        al. 2015).  A point is selected where WCT is finite and > sig[j] (a NaN selects nothing),
        inside the cone of influence if `inside_coi`; clusters are the 8-connected patches of the
        selection, in this map and in every surrogate pair's, labelled on the device.  A cluster's
        area is A = sum dj dt / s_j over its points (the module notes give the exact integer
        weights), and its p-value is (1 + #{pairs whose largest cluster is at least as large}) /
        (1 + M): rejecting p <= alpha controls the family-wise error over clusters at alpha.

        `sig` should not come from the same surrogates as the null: take
        `surrogate_significance(mc_count=M, seed=s1)` and test with a seed s2 != s1, or take the
        white-noise levels of `significance()`.  Returns ClusterResult(area, points, rows, cols,
        pvalue, null_max): per cluster of this map, ordered by area descending (ties by the
        row-major index of the first point), its area, point count, row range [first, last + 1),
        column range and p-value, and the M pairs' largest areas in pair order.  The labels stay on
        the device (`cluster_labels`, 4 bytes per scale-point) until the next `cluster_test`,
        `release()` or `wct_resident`.  ValueError for a `sig` without one entry per scale and for
        the checks of `surrogate_test`; the counts of an earlier `surrogate_test` are kept."""
        _null_kind(null)
        return self._cluster(sig, mc_count, seed, inside_coi, null, True, None)

    @_live
    def cluster_labels(self, rows=slice(None), cols=slice(None)):
        """int32 labels[rows, cols] of the last `cluster_test`, with the slicing of `window`: 0 off
        the clusters, c + 1 on cluster c of its result."""
        return self._cluster_labels(rows, cols)


def wct_resident(y1, y2, dt, dj=1/12, s0=-1, J=-1, wavelet='morlet', normalize=True,
                 precision='fp64', engine=None):
    """Same coherence as `wct(y1, y2, dt, dj, s0, J, sig=False, wavelet=wavelet,
    normalize=normalize, precision=precision)`, WCT and aWCT kept on the device.

    Returns a `ResidentCoherence`.  Scales, boxcar, un-padded fallback to fp64 and the Paul / DOG
    smoothing filter are resolved by the same code as `wct`'s."""
    p = _wct_problem((y1, y2), dt, dj, s0, J, wavelet, normalize, precision)
    eng = engine or _engine.default_engine()
    serial = _wct_on_device(eng, p, eng.wct_resident)
    return ResidentCoherence(eng, p, normalize, precision, serial)


# ---- resident cross spectrum -------------------------------------------------------------------
# `xwt` hands the caller a complex128 [S, n0] field; at config 4 that is 608 MB over PCIe for about
# 1.5 ms of GPU work.  What the reference's sample script (pycwt/sample/sample_xwt.py) and Grinsted
# et al. (2004) do with it are |W12| against `signif`, phase arrows on a sub-grid and the circular
# mean phase over the region where |W12| is significant.  `xwt_resident` runs the same transforms
# as `xwt` and keeps W12 on the device, in a buffer of its own: the handle stays valid across later
# cwt / xwt / wct / wct_resident / Monte-Carlo calls, until the next `xwt_resident` on the same
# engine or `release()`.
# `xwt`'s `signif` is a per-scale chi-squared level built from two fitted AR(1) spectra; applied point
# by point it paints spurious patches, as the power's does.  The handle tests |W12|^2 point by point
# and patch by patch against pairs of surrogates drawn on the device, with the definitions of
# `ResidentPower`:
#   'ar1'    two independent AR(1) series per pair, series s with g_s = ar1(y_s)[0] and, with
#            normalize=True, m = 0 and sigma = 1, else y_s's mean and standard deviation (ddof 0);
#   'phase'  the phase-randomised surrogates of the two transformed series with independent phases:
#            each keeps its own periodogram and is independent of the other.
# Each pair is transformed exactly as `xwt` of it would be.  |W12|^2 is common power: a burst in one
# series alone reaches it (Maraun & Kurths 2004), so these test common power, not association.

class ResidentCrossWavelet(_SurrogateTest, _ResidentSlot):
    """W12 = W1 conj(W2) [S, n0] of one `xwt_resident` call, resident on the device.

    `signif` arguments of the methods are in |W12| units, as `xwt` returns them (`.signif`); a
    point is selected where |W12| > signif[j], i.e. re^2 + im^2 > signif[j]^2.  The sample
    script's `|W12|^2 / signif > 1` convention is `signif=np.sqrt(h.signif)`.  A negative entry
    raises ValueError, a NaN entry selects no point of its scale.

    Tests against surrogate pairs (see the notes above `xwt_resident`): `surrogate_test`, `pvalues`,
    `pvalue_fraction`, `fdr_threshold`, `cluster_test` and `cluster_labels` are those of
    `ResidentPower` with |W12|^2 in place of |W|^2; `sig` / `signif` stay in |W12| units.  They test
    common power, not association: a burst in one series alone can be significant (Maraun & Kurths
    2004).  The coherence tests are the tests of association."""

    _FREQ, _SERIAL, _RELEASE = 'freq', 'cross_serial', 'cross_release'
    _CLUSTERS = _engine.CROSS
    _GONE = ("this cross spectrum is no longer resident: it was released or another xwt_resident "
             "has run on the same engine")

    def __init__(self, engine, problem, signif, precision, serial):
        p = problem
        super(ResidentCrossWavelet, self).__init__(engine, p.wavelet, p.n0, p.dt, p.dj, p.sj,
                                                   precision, serial)
        self.freq = p.freq
        self.signif = signif
        self.normalize = p.normalize
        # raw series (ar1, mean and std) and the transformed ones (the phase null)
        self._y = tuple(np.array(y, dtype=np.float64, copy=True) for y in (p.y1, p.y2))
        self._yn = np.array(np.stack([p.y1n, p.y2n]), dtype=np.float64, copy=True)
        self._padding = bool(_helpers._FFT_NEXT_POW2)

    def _threshold(self, signif):
        """A |W12| threshold per scale, squared: the device compares re^2 + im^2."""
        return None if signif is None else _power_threshold(self, signif) ** 2

    def _stats(self, lo, hi, signif):
        return self.engine.field_row_stats(_engine.FIELD_CROSS, lo, hi, self._threshold(signif))

    def _null(self, null):
        """(engine null, g [2], m [2], sigma [2]) of a null's name."""
        kind = _null_kind(null)
        return (kind,) + _ar1_params(self._y, self.normalize, [null == 'ar1'] * 2)

    def _on_device(self, call, null, seed, M, *args):
        kind, g, m, sigma = self._null(null)
        _sync_padding(self.engine, self.n0)
        return call(self._yn, kind, g, m, sigma, seed, 0, M, self.dt, self.scales,
                    *self.wavelet._engine_spec(), self._serial, *args)

    def _count_units(self, seed, M, null):
        self._on_device(self.engine.cross_surrogate_counts, null, seed, M)

    def _cluster_units(self, seed, M, thr, lo, hi, q, null):
        return self._on_device(self.engine.cross_cluster_test, null, seed, M, thr, lo, hi, q)

    def _selected(self, lo, hi, signif, alpha, cluster):
        """The five row stats of `field_row_stats` over the columns [lo, hi) and the selection of
        `signif`, `alpha` or `cluster`."""
        if cluster is None:
            if alpha is not None:
                return self._cut_stats(_engine.CROSS, lo, hi, self._threshold(signif), alpha)
            return self._stats(lo, hi, signif)
        if signif is not None or alpha is not None:
            raise ValueError("cluster selects the points of one cluster: it takes no signif or alpha")
        _, _, box = self.engine.cluster_table(_engine.CROSS)
        if isinstance(cluster, bool) or not isinstance(cluster, (int, np.integer)) \
                or not 0 <= cluster < len(box):
            raise ValueError("cluster must be a row of the last cluster_test's result (0 .. %d), got %r"
                             % (len(box) - 1, cluster))
        r0, r1, c0, c1 = (int(v) for v in box[cluster])
        rows = np.arange(len(self.scales))
        inside = (rows >= r0) & (rows < r1)
        lo = np.where(inside, np.maximum(lo, c0), 0)
        hi = np.where(inside, np.maximum(np.minimum(hi, c1), lo), 0)
        return self.engine.cross_cluster_row_stats(int(cluster), lo, hi)

    # -- the products --------------------------------------------------------------------
    @_live
    def cross_spectrum(self):
        """W12 (complex128, S x n0), as returned by `xwt`: the expensive fetch."""
        return self.engine.field_get(_engine.FIELD_CROSS)

    @_live
    def window(self, rows=slice(None), cols=slice(None)):
        """W12[rows, cols] (complex128) for two slices with steps >= 1, gathered on the device
        (phase arrows, a down-sampled |W12| image)."""
        return _field_window(self.engine, _engine.FIELD_CROSS, self.shape, rows, cols)

    @_live
    def global_power(self, inside_coi=False, signif=None, alpha=None, cluster=None):
        """Mean |W12| per scale over the selected points: inside the cone of influence if
        `inside_coi`, where |W12| > signif[j] if `signif` is given, where the p-value of the last
        `surrogate_test` is <= alpha if `alpha` is given (all: logical AND), or, with `cluster`, on
        the points of row `cluster` of the last `cluster_test`'s result (and inside the cone if
        `inside_coi`; no `signif` or `alpha`).  NaN for a scale without points."""
        st = self._selected(*_column_ranges(self, inside_coi), signif, alpha, cluster)
        return _ratio(st[:, 2], st[:, 0])

    @_live
    def significant_fraction(self, signif):
        """Per scale, the fraction of the points inside the cone of influence where
        |W12| > signif[j]; NaN for a scale without points inside the cone."""
        lo, hi = self.coi_ranges()
        st = self._stats(lo, hi, signif)
        return _ratio(st[:, 0], hi - lo)

    @_live
    def mean_phase(self, period_min=-np.inf, period_max=np.inf, inside_coi=True, signif=None,
                   per_scale=False, alpha=None, cluster=None):
        """Circular mean of angle(W12) over the points of the scales with period_min <= period <
        period_max, inside the cone of influence if `inside_coi`, where |W12| > signif if given and
        where the p-value of the last `surrogate_test` is <= alpha if given (Grinsted et al. 2004),
        or, with `cluster`, on the points of row `cluster` of the last `cluster_test`'s result (the
        lead or lag inside one significant patch; no `signif` or `alpha`): MeanPhase(angle =
        atan2(sum sin, sum cos), strength = |sum e^{i angle}| / count, count), for the whole band
        or, with `per_scale`, per scale (NaN angle and strength where the count is 0).  A zero
        coefficient has phase 0."""
        sel = self._band(period_min, period_max)
        lo, hi = _column_ranges(self, inside_coi)
        lo, hi = np.where(sel, lo, 0), np.where(sel, hi, 0)
        st = self._selected(lo, hi, signif, alpha, cluster)
        return _mean_phase(st[:, 0], st[:, 3], st[:, 4], per_scale)

    @_live
    def scale_avg(self, period_min, period_max):
        """Scale-averaged cross spectrum over period_min <= period < period_max (complex128,
        length n0): dj * dt / Cdelta * sum_j W12[j] / s_j, Torrence & Compo (1998) eq. 24 with
        W12 in place of |W|^2."""
        sel, w = self._band_weights(period_min, period_max)
        if not sel.any():
            raise ValueError("no scale with %r <= period < %r" % (period_min, period_max))
        return self.engine.cross_scale_avg(w)

    @_live
    def surrogate_test(self, mc_count=300, seed=None, null='ar1'):
        """Run the pairs 0 .. mc_count - 1 of `null` ('ar1' or 'phase') once and count per point the
        pairs whose |W12|^2 reaches this one (kept on the device, replacing the counts of an earlier
        test).  Seed, records and errors as `ResidentPower.surrogate_test`."""
        self._null(null)
        self._count(mc_count, seed, null)

    @_live
    def pvalues(self, rows=slice(None), cols=slice(None)):
        """p[rows, cols] = (1 + k) / (1 + M) (float64) of the last `surrogate_test`, with the slicing
        of `window`; NaN where |W12| is not finite."""
        return self._pvalues(_engine.CROSS, rows, cols)

    @_live
    def pvalue_fraction(self, alpha):
        """Per scale, the fraction of the points inside the cone of influence (with a finite p) whose
        p <= alpha; NaN for a scale without such points."""
        return self._pvalue_fraction(_engine.CROSS, alpha)

    @_live
    def fdr_threshold(self, q=0.05, method='bh', inside_coi=True):
        """`ResidentCoherence.fdr_threshold` over the p-values of the last `surrogate_test`."""
        return self._fdr_threshold(_engine.CROSS, q, method, inside_coi)

    @_live
    def cluster_test(self, sig, mc_count=300, seed=None, null='ar1', inside_coi=True):
        """Cluster (areawise) test of this cross spectrum against the pairs 0 .. mc_count - 1 of
        `null`: `ResidentCoherence.cluster_test` with a point selected where |W12| is finite and
        > sig[j] (|W12| units: `h.cluster_test(h.signif, ...)` is the natural call).  Returns
        ClusterResult; the counts of an earlier `surrogate_test` are kept."""
        self._null(null)
        return self._cluster(sig, mc_count, seed, inside_coi, null)

    @_live
    def cluster_labels(self, rows=slice(None), cols=slice(None)):
        """`ResidentCoherence.cluster_labels` of the last `cluster_test`."""
        return self._cluster_labels(rows, cols)


def xwt_resident(y1, y2, dt, dj=1/12, s0=-1, J=-1, significance_level=0.95, wavelet='morlet',
                 normalize=True, precision='fp64', engine=None):
    """Same cross-wavelet transform as `xwt(y1, y2, dt, dj, s0, J, significance_level, wavelet,
    normalize, precision)`, W12 kept on the device.

    Returns a `ResidentCrossWavelet`; its `signif` is `xwt`'s fourth return value.  Scales,
    standardisation, the un-padded fallback to fp64 and `signif` are resolved by the same code
    as `xwt`'s.  No transform stays resident afterwards (handles of `cwt_resident` die)."""
    p = _xwt_problem(y1, y2, dt, dj, s0, J, wavelet, normalize, precision)
    eng = engine or _engine.default_engine()
    serial = _xwt_on_device(eng, p, eng.xwt_resident)
    return ResidentCrossWavelet(eng, p, _xwt_signif(p, significance_level), precision, serial)


# ---- resident partial and multiple coherence ---------------------------------------------------
# `partial_wct` and `multiple_wct` each hand the caller one float64 [S, n0] field and run the whole
# three-series pipeline for it; at config 4 that is two pipelines and 608 MB over PCIe.
# `wct3_resident` runs the pipeline once and keeps RP2, the partial phase and RM2 on the device, in
# a buffer of their own: the handle stays valid across later cwt / xwt / wct / wct_resident /
# xwt_resident / partial_wct / Monte-Carlo calls, until the next `wct3_resident` on the same engine
# or `release()`.

_MEASURES = {'partial': _engine.MEASURE_PARTIAL, 'multiple': _engine.MEASURE_MULTIPLE}


class ResidentCoherence3(_CoherenceTest, _ResidentSlot):
    """RP2, the partial phase and RM2 [S, n0] of one `wct3_resident` call, resident on the device.

    The partial phase is the angle of the smoothed partial cross spectrum of y and x1 with x2
    removed, u = S_y1 S_2 - S_y2 conj(S_12) (the numerator of RP2 = |u|^2 / (D_y D_12)), in the sign
    convention of `wct`'s aWCT: the angle of W_y conj(W_x1).  aWCT is the angle of the *unsmoothed*
    cross spectrum (reference wavelet.py:514); an unsmoothed partial spectrum does not exist, so the
    partial phase is the angle of a smoothed quantity and differs from aWCT even where x2 plays no
    role.  A zero u has phase 0.  RM2 has no phase.

    `measure` arguments are 'partial' (RP2) or 'multiple' (RM2).  `sig` arguments take one entry
    per scale in the units of the measure (as `wct3_significance` returns them); a point is
    selected where R > sig[j], and a NaN entry selects no point of its scale.

    Point-wise test: `surrogate_test` counts, per point and measure, the surrogate triples of
    `wct3_surrogate_significance` that reach the observed RP2 / RM2, with the definitions of
    `ResidentCoherence` (8 bytes per scale-point on the device for the two measures)."""

    _FREQ, _SERIAL, _RELEASE = 'freq', 'coherence3_serial', 'coherence3_release'
    _CLUSTERS = True
    _GONE = ("this partial / multiple coherence is no longer resident: it was released or another "
             "wct3_resident has run on the same engine")

    def __init__(self, engine, problem, normalize, precision, serial):
        p = problem
        super(ResidentCoherence3, self).__init__(engine, p.wavelet, p.n0, p.dt, p.dj, p.sj,
                                                 precision, serial)
        self.s0 = p.s0
        self.J = p.J
        self.freq = p.freq
        self.normalize = normalize
        self._y = tuple(np.array(y, copy=True) for y in p.ys)   # raw series, for ar1 and surrogates
        self._padding = bool(_helpers._FFT_NEXT_POW2)

    def _measure(self, measure):
        try:
            return _MEASURES[measure]
        except (KeyError, TypeError):
            raise ValueError("measure must be 'partial' or 'multiple', got %r" % (measure,))

    def _threshold(self, sig):
        if sig is None:
            return None
        thr = np.asarray(sig, dtype=float)
        if thr.shape != (len(self.scales),):
            raise ValueError("sig must have one entry per scale (%d), got shape %s"
                             % (len(self.scales), thr.shape))
        return thr

    def _field(self, measure, want_value=True, want_phase=False):
        S, n0 = self.shape
        return self.engine.coherence3_window(measure, 0, S, 1, 0, n0, 1, want_value, want_phase)

    # -- the products --------------------------------------------------------------------
    @_live
    def partial(self):
        """RP2 (float64, S x n0), as returned by `partial_wct`: the expensive fetch."""
        return self._field(_engine.MEASURE_PARTIAL)[0]

    @_live
    def multiple(self):
        """RM2 (float64, S x n0), as returned by `multiple_wct`: the expensive fetch."""
        return self._field(_engine.MEASURE_MULTIPLE)[0]

    @_live
    def phase(self):
        """The partial phase (float64, S x n0, radians in [-pi, pi])."""
        return self._field(_engine.MEASURE_PARTIAL, want_value=False, want_phase=True)[1]

    @_live
    def window(self, rows=slice(None), cols=slice(None)):
        """(RP2[rows, cols], phase[rows, cols], RM2[rows, cols]) for two slices with steps >= 1,
        gathered on the device: only the sub-grid crosses the bus (contour and phase-arrow plots)."""
        S, n0 = self.shape
        r0, nr, rs = _slice_range(rows, S, 'rows')
        c0, nc, cs = _slice_range(cols, n0, 'cols')
        if nr == 0 or nc == 0:
            return np.empty((nr, nc)), np.empty((nr, nc)), np.empty((nr, nc))
        rp, ph = self.engine.coherence3_window(_engine.MEASURE_PARTIAL, r0, nr, rs, c0, nc, cs,
                                               want_phase=True)
        rm = self.engine.coherence3_window(_engine.MEASURE_MULTIPLE, r0, nr, rs, c0, nc, cs)[0]
        return rp, ph, rm

    @_live
    def global_coherence(self, measure='partial', inside_coi=False, sig=None, alpha=None):
        """Mean of the measure per scale over the selected points: inside the cone of influence
        (period_j <= coi[n]) if `inside_coi`, where R[j, n] > sig[j] if `sig` is given, where the
        measure's p-value of the last `surrogate_test` is <= alpha if `alpha` is given.  NaN for a
        scale without points."""
        m = self._measure(measure)
        lo, hi = _column_ranges(self, inside_coi)
        if alpha is not None:
            st = self._cut_stats(m, lo, hi, self._threshold(sig), alpha)
        else:
            st = self.engine.coherence3_row_stats(m, lo, hi, self._threshold(sig))
        return _ratio(st[:, 1], st[:, 0])

    @_live
    def significant_fraction(self, sig, measure='partial'):
        """Per scale, the fraction of the points inside the cone of influence where R > sig[j];
        NaN for a scale without points inside the cone."""
        m = self._measure(measure)
        lo, hi = self.coi_ranges()
        st = self.engine.coherence3_row_stats(m, lo, hi, self._threshold(sig))
        return _ratio(st[:, 0], hi - lo)

    @_live
    def mean_phase(self, period_min=-np.inf, period_max=np.inf, inside_coi=True, sig=None,
                   per_scale=False, alpha=None):
        """Circular mean of the partial phase over the points of the scales with period_min <=
        period < period_max, inside the cone of influence if `inside_coi`, where RP2 > sig if given
        and where RP2's p-value of the last `surrogate_test` is <= alpha if given: MeanPhase(angle =
        atan2(sum sin, sum cos), strength = |sum e^{i phase}| / count, count), for the whole band
        or, with `per_scale`, per scale (NaN angle and strength where the count is 0)."""
        sel = self._band(period_min, period_max)
        lo, hi = _column_ranges(self, inside_coi)
        lo, hi = np.where(sel, lo, 0), np.where(sel, hi, 0)
        if alpha is not None:
            st = self._cut_stats(_engine.MEASURE_PARTIAL, lo, hi, self._threshold(sig), alpha,
                                 want_phase=True)
        else:
            st = self.engine.coherence3_row_stats(_engine.MEASURE_PARTIAL, lo, hi,
                                                  self._threshold(sig), want_phase=True)
        return _mean_phase(st[:, 0], st[:, 2], st[:, 3], per_scale)

    @_live
    def scale_avg(self, period_min, period_max):
        """Three length-n0 series over the scales with period_min <= period < period_max: the mean
        RP2, the circular mean partial phase atan2(sum sin, sum cos) and the mean RM2."""
        sel = self._band(period_min, period_max)
        if not sel.any():
            raise ValueError("no scale with %r <= period < %r" % (period_min, period_max))
        w = sel.astype(float)
        k = float(sel.sum())
        p = self.engine.coherence3_scale_avg(_engine.MEASURE_PARTIAL, w)
        rp, ph = p[0] / k, np.arctan2(p[2], p[1])
        rm = self.engine.coherence3_scale_avg(_engine.MEASURE_MULTIPLE, w)[0] / k
        return rp, ph, rm

    @_live
    def significance(self, significance_level=0.95, mc_count=300, progress=True, seed=None):
        """(sig_partial, sig_multiple) of `wct3_significance` with the lag-1 autocorrelations of the
        raw series and this handle's dt, dj, s0, J, wavelet and precision.  The fields stay
        resident."""
        al = [ar1(y)[0] for y in self._y]
        return wct3_significance(*al, dt=self.dt, dj=self.dj, s0=self.s0, J=self.J,
                                 significance_level=significance_level, wavelet=self.wavelet,
                                 mc_count=mc_count, progress=progress, seed=seed,
                                 precision=self.precision)

    @_live
    def surrogate_significance(self, significance_level=0.95, mc_count=300, seed=None,
                               conditional=True, null='phase'):
        """(sig_partial, sig_multiple) of `wct3_surrogate_significance` on this handle's series and
        arguments, against `null` ('phase' or 'ar1').  The fields stay resident."""
        return wct3_surrogate_significance(*self._y, dt=self.dt, dj=self.dj, s0=self.s0, J=self.J,
                                           significance_level=significance_level,
                                           wavelet=self.wavelet, normalize=self.normalize,
                                           mc_count=mc_count, seed=seed, precision=self.precision,
                                           conditional=conditional, null=null)

    @_live
    def surrogate_test(self, mc_count=300, seed=None, significance_level=0.95, conditional=True,
                       null='phase'):
        """Run the surrogate triples 0 .. mc_count - 1 of `null` once ('phase' or 'ar1'; with
        `conditional=True` and 'ar1', y is red noise and x1, x2 are held at the data in every triple,
        see `wct3_surrogate_significance`): count per point the triples whose RP2 and RM2 reach this
        handle's (one count field per measure, kept on the device, replacing the counts of an
        earlier test) and return (sig_partial, sig_multiple), bit-identical to
        `surrogate_significance` with the same `seed`, `mc_count`, `conditional` and `null`.  Seed,
        errors and records as `ResidentCoherence.surrogate_test`."""
        _null_kind(null)
        prob, hist = self._count(mc_count, seed, null, conditional)
        return _mc_levels(prob, hist[0], significance_level), _mc_levels(prob, hist[1], significance_level)

    @_live
    def pvalues(self, rows=slice(None), cols=slice(None), measure='partial'):
        """The measure's p[rows, cols] = (1 + k) / (1 + M) (float64) of the last `surrogate_test`,
        with the slicing of `window`; NaN where the measure is not finite."""
        return self._pvalues(self._measure(measure), rows, cols)

    @_live
    def pvalue_fraction(self, alpha, measure='partial'):
        """Per scale, the fraction of the points inside the cone of influence (with a finite p) whose
        p <= alpha; NaN for a scale without such points."""
        return self._pvalue_fraction(self._measure(measure), alpha)

    @_live
    def fdr_threshold(self, q=0.05, method='bh', inside_coi=True, measure='partial'):
        """`ResidentCoherence.fdr_threshold` over the measure's p-values."""
        return self._fdr_threshold(self._measure(measure), q, method, inside_coi)

    @_live
    def cluster_test(self, sig, mc_count=300, seed=None, inside_coi=True, measure='partial',
                     conditional=True, null='phase'):
        """`ResidentCoherence.cluster_test` of the measure against the surrogate triples
        0 .. mc_count - 1 of `surrogate_significance(mc_count=mc_count, seed=seed,
        conditional=conditional, null=null)`; `sig` in the units of the measure."""
        m = self._measure(measure)
        _null_kind(null)
        return self._cluster(sig, mc_count, seed, inside_coi, null, conditional, m)

    @_live
    def cluster_labels(self, rows=slice(None), cols=slice(None)):
        """`ResidentCoherence.cluster_labels` of the last `cluster_test`."""
        return self._cluster_labels(rows, cols)


def wct3_resident(y, x1, x2, dt, dj=1/12, s0=-1, J=-1, wavelet='morlet', normalize=True,
                  precision='fp64', engine=None):
    """Same partial and multiple coherence as `partial_wct(y, x1, x2, dt, dj, s0, J, wavelet,
    normalize, precision)` and `multiple_wct(...)`, from one run of the pipeline, kept on the device
    with the partial phase.

    Returns a `ResidentCoherence3`.  Scales, boxcar, standardisation, the un-padded fallback to fp64,
    the Paul / DOG smoothing filter and the errors are resolved by the same code as `partial_wct`'s.
    No transform stays resident afterwards (handles of `cwt_resident` die); the handles of
    `wct_resident` and `xwt_resident` survive."""
    p = _wct_problem((y, x1, x2), dt, dj, s0, J, wavelet, normalize, precision)
    eng = engine or _engine.default_engine()
    serial = _wct_on_device(eng, p, eng.wct3_resident)
    return ResidentCoherence3(eng, p, normalize, precision, serial)


# ---- resident wavelet power and its tests against surrogates --------------------------------------
# The wavelet power |W|^2 of one series is the map a user draws most; its classic test is the
# per-scale chi-squared level of `significance()` (TC98 eq. 18), which, applied point by point, paints
# many spurious patches (Maraun et al. 2007).  `power_resident` keeps W in a device buffer of its own
# (the handle survives later cwt / xwt / wct / Monte-Carlo calls, until the next `power_resident` or
# `release()`) and tests it point by point and patch by patch against surrogates drawn on the device:
#   'ar1'    red noise x = m + sigma z, z[0] = e[0], z[n] = g z[n-1] + sqrt(1 - g^2) e[n], with
#            g = ar1(series)[0] (the background `significance()` assumes), m = 0 and sigma = 1 for
#            normalize=True, else the series' mean and standard deviation (ddof 0);
#   'phase'  the phase-randomised surrogates of the transformed series (the periodogram kept
#            exactly): is the *local* power larger than a stationary process with the data's own
#            spectrum would give?
# Each unit is transformed with the handle's plan, exactly as `cwt` of it would be, and its power is
# compared with the resident one on every point (`surrogate_test`) or labelled into clusters
# (`cluster_test`), with the definitions of `ResidentCoherence`.

class ResidentPower(_SurrogateTest, _ResidentSlot):
    """W[S, n0] of one `power_resident` call, resident on the device, and the tests of its power
    P = |W|^2.

    `signif` arguments are per-scale thresholds in power units, as `significance()` returns them:
    with normalize=True, `significance(1.0, dt, scales, 0, g)[0]` (g = ar1(series)[0]); with
    normalize=False, `significance(series, dt, scales, 0)[0]`.  A point is selected where
    P > signif[j]; a negative entry raises ValueError, a NaN entry selects no point of its scale.

    Point-wise test: `surrogate_test(mc_count=M, seed=s, null=...)` counts, per point, the units
    0 .. M - 1 of the null whose power reaches this one, k[s, n] = #{i : P_i[s, n] >= P[s, n]} (a
    non-finite P_i counts), p = (1 + k) / (1 + M), NaN where P is not finite; the counts take 4 bytes
    per scale-point on the device.  The readers, FDR control and the cluster test are those of
    `ResidentCoherence` with P in place of the coherence.  There are no per-scale Monte-Carlo levels:
    the cluster-forming threshold is the caller's, typically the chi-squared level of
    `significance()`."""

    _FREQ, _SERIAL, _RELEASE = 'freqs', 'power_serial', 'power_release'
    _CLUSTERS = _engine.POWER
    _GONE = ("this power is no longer resident: it was released or another power_resident has run "
             "on the same engine")

    def __init__(self, engine, wavelet, y, yn, dt, dj, sj, freqs, normalize, precision, serial):
        super(ResidentPower, self).__init__(engine, wavelet, len(yn), dt, dj, sj, precision, serial)
        self.freqs = freqs
        self.normalize = normalize
        self._y = np.array(y, dtype=np.float64, copy=True)     # raw series: ar1, mean and std
        self._yn = np.array(yn, dtype=np.float64, copy=True)   # the transformed series: phase null
        self._padding = bool(_helpers._FFT_NEXT_POW2)

    def _threshold(self, signif):
        return None if signif is None else _power_threshold(self, signif)

    def _null(self, null):
        """(engine null, g, m, sigma) of a null's name."""
        kind = _null_kind(null)
        g, m, sigma = _ar1_params([self._y], self.normalize, [null == 'ar1'])
        return kind, g[0], m[0], sigma[0]

    def _on_device(self, call, null, seed, M, *args):
        kind, g, m, sigma = self._null(null)
        eng = self.engine
        _sync_padding(eng, self.n0)
        return call(self._yn, kind, g, m, sigma, seed, 0, M, self.dt, self.scales,
                    *self.wavelet._engine_spec(), self._serial, *args)

    def _count_units(self, seed, M, null):
        self._on_device(self.engine.power_surrogate_counts, null, seed, M)

    def _cluster_units(self, seed, M, thr, lo, hi, q, null):
        return self._on_device(self.engine.power_cluster_test, null, seed, M, thr, lo, hi, q)

    # -- the products --------------------------------------------------------------------
    @_live
    def wave(self):
        """The coefficients themselves (complex128, S x n0): the expensive fetch."""
        return self.engine.field_get(_engine.FIELD_POWER)

    @_live
    def power(self, rows=slice(None), cols=slice(None)):
        """|W|^2[rows, cols] (float64) for two slices with steps >= 1, formed on the device exactly as
        the tests form it (re^2 + im^2 in double): 8 bytes per point cross the bus.  The whole map
        is the expensive fetch."""
        S, n0 = self.shape
        r0, nr, rs = _slice_range(rows, S, 'rows')
        c0, nc, cs = _slice_range(cols, n0, 'cols')
        out = np.empty((nr, nc))
        # in blocks of rows, so that the device staging stays below 2^25 points
        step = max(1, (1 << 25) // max(nc, 1))
        for b in range(0, nr, step):
            k = min(step, nr - b)
            out[b:b + k] = self.engine.power_window(r0 + b * rs, k, rs, c0, nc, cs)
        return out

    @_live
    def window(self, rows=slice(None), cols=slice(None)):
        """W[rows, cols] (complex128) for two slices with steps >= 1, gathered on the device."""
        return _field_window(self.engine, _engine.FIELD_POWER, self.shape, rows, cols)

    @_live
    def global_power(self, inside_coi=False, signif=None, alpha=None):
        """Time mean of |W|^2 per scale over the selected points: inside the cone of influence if
        `inside_coi`, where |W|^2 > signif[j] if `signif` is given, where the p-value of the last
        `surrogate_test` is <= alpha if `alpha` is given (all: logical AND).  NaN for a scale
        without points."""
        lo, hi = _column_ranges(self, inside_coi)
        thr = self._threshold(signif)
        if alpha is not None:
            st = self._cut_stats(_engine.POWER, lo, hi, thr, alpha)
        else:
            st = self.engine.field_row_stats(_engine.FIELD_POWER, lo, hi, thr)
        return _ratio(st[:, 1], st[:, 0])

    @_live
    def significant_fraction(self, signif):
        """Per scale, the fraction of the points inside the cone of influence where
        |W|^2 > signif[j]; NaN for a scale without such points."""
        lo, hi = self.coi_ranges()
        st = self.engine.field_row_stats(_engine.FIELD_POWER, lo, hi, _power_threshold(self, signif))
        return _ratio(st[:, 0], hi - lo)

    @_live
    def scale_avg_power(self, period_min, period_max, variance=1.0):
        """Scale-averaged power over period_min <= period < period_max (TC98 eq. 24), as
        `ResidentTransform.scale_avg_power`."""
        _, w = self._band_weights(period_min, period_max, variance)
        return self.engine.power_scale_avg(w)

    @_live
    def reconstruct(self, period_min=-np.inf, period_max=np.inf, inside_coi=False, signif=None, alpha=None,
                    cluster=None):
        """The series behind a band, the significant points or the significant clusters of this power:
        `ResidentTransform.reconstruct` on this handle's W, x[n] = dj sqrt(dt) / (Cdelta psi(0)) * sum
        over the selected (j, n) of Re W[j, n] / sqrt(s_j).  A point is selected where every condition
        given holds: the band and `inside_coi` as there; P > signif[j] if `signif` is given; a finite P
        whose p-value of the last `surrogate_test` is <= alpha if `alpha` is given (EngineError without
        a test); or, with `cluster` (an int or a sequence of ints, rows of the last `cluster_test`'s
        ClusterResult, e.g. `np.flatnonzero(res.pvalue <= 0.05)`; a repeated row counts once, an empty
        one gives zeros), on the points of those clusters, with no `signif` or `alpha`.

        W is the W of the transformed series: with normalize=True the result is in standardised units;
        multiply it by the series' standard deviation (`y.std()`) for data units."""
        thr = self._threshold(signif)
        w, lo, hi = _reconstruct_rows(self, period_min, period_max, inside_coi)
        if cluster is not None:
            if signif is not None or alpha is not None:
                raise ValueError("cluster selects the points of clusters: it takes no signif or alpha")
            rows = self._cluster_rows(cluster)
            red = self.engine.power_cluster_reconstruct(w, lo, hi, rows)
        elif alpha is not None:
            red = self.engine.power_pvalue_reconstruct(w, lo, hi, _kmax(alpha, self._units()), thr)
        else:
            red = self.engine.field_reconstruct(_engine.FIELD_POWER, w, lo, hi, thr)
        return _inverse(self, red)

    def _cluster_rows(self, cluster):
        """int64 rows of the last cluster_test's table: an int or a sequence of ints."""
        Q, _, _ = self.engine.cluster_table(_engine.POWER)
        rows = np.asarray(cluster)
        if rows.ndim > 1 or rows.dtype == bool or (rows.size and not np.issubdtype(rows.dtype, np.integer)):
            raise ValueError("cluster must be an int or a sequence of ints, got %r" % (cluster,))
        rows = rows.astype(np.int64).reshape(-1)
        if ((rows < 0) | (rows >= len(Q))).any():
            raise ValueError("cluster must hold rows of the last cluster_test's result (0 .. %d), got %r"
                             % (len(Q) - 1, cluster))
        return rows

    @_live
    def surrogate_test(self, mc_count=300, seed=None, null='ar1'):
        """Run the units 0 .. mc_count - 1 of `null` ('ar1' or 'phase') once and count per point the
        units whose power reaches this one (kept on the device, replacing the counts of an earlier
        test).  `seed=None` draws the seed from numpy's global RNG; the seed and M are kept as
        `surrogate_seed` and `surrogate_units`.  ValueError for mc_count outside [1, 2^31 - 1], an
        unknown null, or when the FFT padding mode differs from the one this power was computed
        with."""
        self._null(null)
        self._count(mc_count, seed, null)

    @_live
    def pvalues(self, rows=slice(None), cols=slice(None)):
        """p[rows, cols] = (1 + k) / (1 + M) (float64) of the last `surrogate_test`, with the slicing
        of `window`; NaN where the power is not finite."""
        return self._pvalues(_engine.POWER, rows, cols)

    @_live
    def pvalue_fraction(self, alpha):
        """Per scale, the fraction of the points inside the cone of influence (with a finite p) whose
        p <= alpha; NaN for a scale without such points."""
        return self._pvalue_fraction(_engine.POWER, alpha)

    @_live
    def fdr_threshold(self, q=0.05, method='bh', inside_coi=True):
        """`ResidentCoherence.fdr_threshold` over the p-values of the last `surrogate_test`."""
        return self._fdr_threshold(_engine.POWER, q, method, inside_coi)

    @_live
    def cluster_test(self, sig, mc_count=300, seed=None, null='ar1', inside_coi=True):
        """Cluster (areawise) test of this power against the units 0 .. mc_count - 1 of `null`
        (Maraun et al. 2007): `ResidentCoherence.cluster_test` with a point selected where |W|^2 is
        finite and > sig[j] (power units, typically the chi-squared level of `significance()`).
        Returns ClusterResult; the counts of an earlier `surrogate_test` are kept."""
        self._null(null)
        return self._cluster(sig, mc_count, seed, inside_coi, null)

    @_live
    def cluster_labels(self, rows=slice(None), cols=slice(None)):
        """`ResidentCoherence.cluster_labels` of the last `cluster_test`."""
        return self._cluster_labels(rows, cols)


def power_resident(signal, dt, dj=1/12, s0=-1, J=-1, wavelet='morlet', freqs=None, normalize=True,
                   precision='fp64', engine=None):
    """The transform of `cwt` of the series (standardised first with `normalize`, as `xwt` and
    `wct` do), in `precision` ('fp64' or 'fp32'), W kept on the device for the power tests.

    Returns a `ResidentPower`.  Scales, the dropped Paul rows and the un-padded fallback to fp64
    are resolved by the same code as `cwt_resident` and `wct`; wavelets the engine does not evaluate
    itself raise TypeError.  No transform stays resident afterwards (handles of `cwt_resident`
    die); the other resident products survive."""
    wavelet, spec = _engine_wavelet(wavelet, "power_resident")
    prec = _coherence_precision(precision)
    y, yn, _ = _standardise(np.asarray(signal, dtype=np.float64), normalize)
    n0 = len(yn)
    sj, freqs = _kept_scales(n0, dt, dj, s0, J, wavelet, freqs)
    eng = engine or _engine.default_engine()
    with eng.lock:
        if _sync_padding(eng, n0):
            prec = _engine.F64      # un-padded transforms run in fp64
        serial = eng.power_resident(yn, dt, sj, *spec, precision=prec)
    return ResidentPower(eng, wavelet, y, yn, dt, dj, sj, freqs, normalize, precision, serial)
