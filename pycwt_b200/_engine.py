"""ctypes binding of the C-ABI engine (include/cwt_b200.h).  No PyTorch, no CPU
fallback: if the CUDA library or a device is missing, calls raise EngineError."""
import collections
import ctypes
import os
import threading
import weakref

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcwtb200.so")

MORLET, PAUL, DOG, TABLE, MORSE = 0, 1, 2, 3, 4
#: Morse's shape parameter ga when `param` gives be alone
MORSE_GA = 3.0
F64, F32 = 0, 1
# complex fields of the cwtb_field_* calls, each with the id of its product below
FIELD_W, FIELD_CROSS, FIELD_POWER = 0, 1, 5
MEASURE_PARTIAL, MEASURE_MULTIPLE = 0, 1   # the measures of the cwtb_coherence3_* calls
# the resident products of cwtb_resident_shape: the two fields, the coherence (cwtb_coherence_*), the
# partial and multiple coherence (cwtb_coherence3_*) and the power (cwtb_power_*)
PRODUCT_W, PRODUCT_CROSS, PRODUCT_COHERENCE, PRODUCT_COHERENCE3, PRODUCT_POWER = 0, 1, 2, 3, 5   # 4: none
NULL_AR1, NULL_PHASE = 0, 1      # the nulls of the tests against surrogates (enum cwtb_null)


class CoherenceNull(collections.namedtuple('CoherenceNull', 'kind groups g m sigma held')):
    """The null of a coherence Monte-Carlo call (cwtb_wct_mc_null): NULL_PHASE with the phase group of
    each series (`groups`), or NULL_AR1 with each series' AR(1) parameters g, m, sigma and held flag
    (1: the data's row in every unit, None: every series drawn)."""
    __slots__ = ()

    def __new__(cls, kind, groups=None, g=None, m=None, sigma=None, held=None):
        return super(CoherenceNull, cls).__new__(cls, kind, groups, g, m, sigma, held)
# the `measure` of the surrogate-test readers below that names the resident power, and the one that
# names the resident cross spectrum
POWER = 'power'
CROSS = 'cross'
_COMPLEX = {POWER: PRODUCT_POWER, CROSS: PRODUCT_CROSS}   # their products; each is the prefix of its C calls

_P = ctypes.c_void_p
_I64 = ctypes.c_int64
_D = ctypes.c_double
_I = ctypes.c_int


class EngineError(RuntimeError):
    pass


_SIGNATURES = {
    "cwtb_device_count": (_I, []),
    "cwtb_create": (_I, [_I, ctypes.POINTER(_P)]),
    "cwtb_destroy": (None, [_P]),
    "cwtb_last_error": (ctypes.c_char_p, [_P]),
    "cwtb_version": (ctypes.c_char_p, []),
    "cwtb_set_band_eps": (_I, [_P, _D]),
    "cwtb_set_expand_eps": (_I, [_P, _D, _D]),
    "cwtb_set_padding": (_I, [_P, _I]),
    "cwtb_set_coherence_precision": (_I, [_P, _I]),
    "cwtb_set_smooth_filter": (_I, [_P, _P, _I, _I64]),
    "cwtb_set_morse_ga": (_I, [_P, _D]),
    "cwtb_host_alloc": (_I, [_P, ctypes.c_size_t, ctypes.POINTER(_P)]),
    "cwtb_host_free": (_I, [_P, _P]),
    "cwtb_cwt": (_I, [_P, _P, _I, _I64, _D, _P, _I, _I, _D, _I, _P]),
    "cwtb_cwt_dev": (_I, [_P, _P, _I, _I64, _D, _P, _I, _I, _D, _I]),
    "cwtb_get_w": (_I, [_P, _P, _I, _I, _I]),
    "cwtb_get_signal_fft": (_I, [_P, _P]),
    "cwtb_padded_length": (_I64, [_P]),
    "cwtb_job_serial": (_I64, [_P]),
    "cwtb_w_device_ptr": (_P, [_P]),
    "cwtb_resident_shape": (_I, [_P, _I, ctypes.POINTER(_I), ctypes.POINTER(_I64), ctypes.POINTER(_I)]),
    "cwtb_last_kernel_ms": (_D, [_P]),
    "cwtb_last_launch_count": (_I, [_P]),
    "cwtb_last_plan": (_I, [_P, _P, _I]),
    "cwtb_bench_last": (_I, [_P, _I, ctypes.POINTER(_D)]),
    "cwtb_profile_last": (_I, [_P, ctypes.c_char_p, ctypes.c_size_t]),
    "cwtb_profile_begin": (_I, [_P]),
    "cwtb_profile_end": (_I, [_P, ctypes.c_char_p, ctypes.c_size_t]),
    "cwtb_dev_alloc": (_I, [_P, ctypes.c_size_t, ctypes.POINTER(_P)]),
    "cwtb_dev_free": (_I, [_P, _P]),
    "cwtb_memcpy_h2d": (_I, [_P, _P, _P, ctypes.c_size_t]),
    "cwtb_memcpy_d2h": (_I, [_P, _P, _P, ctypes.c_size_t]),
    "cwtb_sync": (_I, [_P]),
    "cwtb_fft_c2c": (_I, [_P, _P, _P, _I64, _I, _I, _I]),
    "cwtb_cwt_to_host": (_I, [_P, _P, _I, _I64, _D, _P, _I, _I, _D, _I, _P, _I]),
    "cwtb_icwt_sum": (_I, [_P, _P]),
    "cwtb_icwt_sum_host": (_I, [_P, _P, _P, _I, _I64, _P]),
    "cwtb_get_power": (_I, [_P, _P]),
    "cwtb_global_power": (_I, [_P, _P]),
    "cwtb_get_power_scaled": (_I, [_P, _P, _P]),
    "cwtb_global_power_ranges": (_I, [_P, _P, _P, _P]),
    "cwtb_scale_avg_power": (_I, [_P, _P, _P]),
    "cwtb_xwt": (_I, [_P, _P, _P, _I64, _D, _P, _I, _I, _D, _P]),
    "cwtb_wct": (_I, [_P, _P, _P, _I64, _D, _D, _P, _I, _I, _D, _I, _P, _P]),
    "cwtb_wct_resident": (_I, [_P, _P, _P, _I64, _D, _D, _P, _I, _I, _D, _I]),
    "cwtb_wct3": (_I, [_P, _P, _P, _P, _I64, _D, _D, _P, _I, _I, _D, _I, _P, _P]),
    "cwtb_coherence_serial": (_I64, [_P]),
    "cwtb_coherence_release": (_I, [_P]),
    "cwtb_coherence_window": (_I, [_P, _I, _I, _I, _I64, _I64, _I64, _P, _P]),
    "cwtb_coherence_row_stats": (_I, [_P, _P, _P, _P, _I, _P]),
    "cwtb_coherence_scale_avg": (_I, [_P, _P, _P]),
    "cwtb_wct3_resident": (_I, [_P, _P, _P, _P, _I64, _D, _D, _P, _I, _I, _D, _I]),
    "cwtb_coherence3_serial": (_I64, [_P]),
    "cwtb_coherence3_release": (_I, [_P]),
    "cwtb_coherence3_window": (_I, [_P, _I, _I, _I, _I, _I64, _I64, _I64, _P, _P]),
    "cwtb_coherence3_row_stats": (_I, [_P, _I, _P, _P, _P, _I, _P]),
    "cwtb_coherence3_scale_avg": (_I, [_P, _I, _P, _P]),
    "cwtb_xwt_resident": (_I, [_P, _P, _P, _I64, _D, _P, _I, _I, _D]),
    "cwtb_cross_serial": (_I64, [_P]),
    "cwtb_cross_release": (_I, [_P]),
    "cwtb_field_get": (_I, [_P, _I, _I, _I, _P]),
    "cwtb_field_window": (_I, [_P, _I, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_field_row_stats": (_I, [_P, _I, _P, _P, _P, _P]),
    "cwtb_field_reconstruct": (_I, [_P, _I, _P, _P, _P, _P, _P]),
    "cwtb_cross_scale_avg": (_I, [_P, _P, _P]),
    "cwtb_smooth": (_I, [_P, _P, _I, _I, _I64, _D, _P, _I, _P]),
    "cwtb_wct_mc": (_I, [_P, _P, _I, _I64, _D, _D, _P, _I, _I, _D, _I, _P, _I, _I, _P]),
    "cwtb_wct_mc_seeded": (_I, [_P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I, _D, _I, _P, _I, _I, _P]),
    "cwtb_mc_surrogates": (_I, [_P, ctypes.c_uint64, _I64, _I, _I64, _P]),
    "cwtb_wct3_mc": (_I, [_P, _P, _I, _I64, _D, _P, _I, _I, _D, _I, _P, _I, _I, _P, _P]),
    "cwtb_wct3_mc_seeded": (_I, [_P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I, _D, _I, _P, _I, _I,
                                 _P, _P]),
    "cwtb_mc_surrogates3": (_I, [_P, ctypes.c_uint64, _I64, _I, _I64, _P]),
    "cwtb_wct_mc_phase": (_I, [_P, _P, _I, _P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I, _D, _I, _P, _I, _I,
                                _P, _P]),
    "cwtb_mc_phase_surrogates": (_I, [_P, _P, _I, _P, ctypes.c_uint64, _I64, _I, _I64, _P]),
    "cwtb_coherence_surrogate_counts": (_I, [_P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I, _D, _I,
                                             _P, _I, _I, _P, _I64, _I]),
    "cwtb_coherence3_surrogate_counts": (_I, [_P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I, _D, _I,
                                              _P, _I, _I, _P, _P, _I64, _I]),
    "cwtb_coherence_pvalue_window": (_I, [_P, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_coherence3_pvalue_window": (_I, [_P, _I, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_coherence_pvalue_row_stats": (_I, [_P, _P, _P, _P, _I64, _I, _P]),
    "cwtb_coherence3_pvalue_row_stats": (_I, [_P, _I, _P, _P, _P, _I64, _I, _P]),
    "cwtb_coherence_count_hist": (_I, [_P, _P, _P, _I64, _P]),
    "cwtb_coherence3_count_hist": (_I, [_P, _I, _P, _P, _I64, _P]),
    "cwtb_coherence_cluster_test": (_I, [_P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I, _D, _I,
                                         _P, _I, _I, _P, _I64, _P, _P, _P, _P, _P]),
    "cwtb_coherence3_cluster_test": (_I, [_P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I, _D, _I,
                                          _P, _I, _I, _P, _P, _I64, _P, _P, _P, _P, _I, _P]),
    "cwtb_coherence_cluster_table": (_I, [_P, _I64, _P, _P, _P, _P]),
    "cwtb_coherence3_cluster_table": (_I, [_P, _I64, _P, _P, _P, _P]),
    # the coherence Monte-Carlo calls with the null of choice: (series, nser,) null, group, g, m, sigma,
    # held in place of group
    "cwtb_wct_mc_null": (_I, [_P, _P, _I, _I, _P, _P, _P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I,
                              _D, _I, _P, _I, _I, _P, _P]),
    "cwtb_mc_ar1_series_surrogates": (_I, [_P, _I, _P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _P]),
    "cwtb_coherence_surrogate_counts_null": (_I, [_P, _P, _I, _P, _P, _P, _P, _P, ctypes.c_uint64, _I64, _I, _I64,
                                                  _D, _P, _I, _I, _D, _I, _P, _I, _I, _P, _I64, _I]),
    "cwtb_coherence3_surrogate_counts_null": (_I, [_P, _P, _I, _P, _P, _P, _P, _P, ctypes.c_uint64, _I64, _I, _I64,
                                                   _D, _P, _I, _I, _D, _I, _P, _I, _I, _P, _P, _I64, _I]),
    "cwtb_coherence_cluster_test_null": (_I, [_P, _P, _I, _P, _P, _P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _D,
                                              _P, _I, _I, _D, _I, _P, _I, _I, _P, _I64, _P, _P, _P, _P, _P]),
    "cwtb_coherence3_cluster_test_null": (_I, [_P, _P, _I, _P, _P, _P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _D,
                                               _P, _I, _I, _D, _I, _P, _I, _I, _P, _P, _I64, _P, _P, _P, _P, _I, _P]),
    "cwtb_coherence_cluster_labels": (_I, [_P, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_coherence3_cluster_labels": (_I, [_P, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_cluster_label_bits": (_I, [_P, _P, _I, _I64, _P, _I64, _P, _P, _P, _P, _P, _P]),
    "cwtb_power_resident": (_I, [_P, _P, _I64, _D, _P, _I, _I, _D]),
    "cwtb_power_serial": (_I64, [_P]),
    "cwtb_power_release": (_I, [_P]),
    "cwtb_power_scale_avg": (_I, [_P, _P, _P]),
    "cwtb_mc_ar1_surrogates": (_I, [_P, _D, _D, _D, ctypes.c_uint64, _I64, _I, _I64, _P]),
    "cwtb_power_surrogate_counts": (_I, [_P, _P, _I, _D, _D, _D, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I,
                                         _D, _I64, _I]),
    "cwtb_power_cluster_test": (_I, [_P, _P, _I, _D, _D, _D, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I, _D,
                                     _I64, _P, _P, _P, _P, _P]),
    "cwtb_power_window": (_I, [_P, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_power_pvalue_window": (_I, [_P, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_power_pvalue_row_stats": (_I, [_P, _P, _P, _P, _I64, _P]),
    "cwtb_power_count_hist": (_I, [_P, _P, _P, _I64, _P]),
    "cwtb_power_cluster_table": (_I, [_P, _I64, _P, _P, _P, _P]),
    "cwtb_power_cluster_labels": (_I, [_P, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_power_pvalue_reconstruct": (_I, [_P, _P, _P, _P, _P, _I64, _P]),
    "cwtb_power_cluster_reconstruct": (_I, [_P, _P, _P, _P, _P, _I64, _P]),
    "cwtb_mc_ar1_pair_surrogates": (_I, [_P, _P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _P]),
    "cwtb_cross_surrogate_counts": (_I, [_P, _P, _I, _P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I,
                                         _D, _I64, _I]),
    "cwtb_cross_cluster_test": (_I, [_P, _P, _I, _P, _P, _P, ctypes.c_uint64, _I64, _I, _I64, _D, _P, _I, _I, _D,
                                     _I64, _P, _P, _P, _P, _P]),
    "cwtb_cross_pvalue_window": (_I, [_P, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_cross_pvalue_row_stats": (_I, [_P, _P, _P, _P, _I64, _P]),
    "cwtb_cross_count_hist": (_I, [_P, _P, _P, _I64, _P]),
    "cwtb_cross_cluster_table": (_I, [_P, _I64, _P, _P, _P, _P]),
    "cwtb_cross_cluster_labels": (_I, [_P, _I, _I, _I, _I64, _I64, _I64, _P]),
    "cwtb_cross_cluster_row_stats": (_I, [_P, _I64, _P, _P, _P]),
    "cwtb_cwt_batch": (_I, [_P, _P, _I, _I, _I64, _D, _P, _I, _I, _D, _I, _P, _P]),
    "cwtb_cwt_batch_dev": (_I, [_P, _P, _I, _I64, _D, _P, _I, _I, _D, _I, _P]),
    "cwtb_comm_unique_id": (_I, [_P]),
    "cwtb_comm_init": (_I, [_P, _I, _I, _P]),
    "cwtb_comm_destroy": (_I, [_P]),
    "cwtb_comm_world": (_I, [_P]),
    "cwtb_comm_rank": (_I, [_P]),
    "cwtb_comm_allgather": (_I, [_P, _P, _P, ctypes.c_size_t]),
    "cwtb_comm_allreduce_sum_i64": (_I, [_P, _P, ctypes.c_size_t]),
    "cwtb_comm_allreduce_max_f64": (_I, [_P, _P, ctypes.c_size_t]),
    "cwtb_comm_broadcast": (_I, [_P, _P, ctypes.c_size_t, _I]),
}


def load_library(path=None):
    """dlopen the engine and declare the prototypes of every exported symbol."""
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise EngineError(
            "CUDA engine not built: %s is missing (run `python -m pycwt_b200.build`)" % path)
    lib = ctypes.CDLL(path)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    return lib


def _ptr(a):
    return a.ctypes.data_as(_P)


def _locked(method):
    """Run an Engine method under the engine's (re-entrant) lock."""
    import functools

    @functools.wraps(method)
    def wrapper(self, *args, **kwargs):
        with self.lock:
            return method(self, *args, **kwargs)
    return wrapper


def _row_args(name, rows, lo, hi, thr):
    """lo, hi (and thr, if given) of a per-row reduction, checked for one entry per row."""
    lo = np.ascontiguousarray(lo, dtype=np.int64)
    hi = np.ascontiguousarray(hi, dtype=np.int64)
    if lo.shape != (rows,) or hi.shape != (rows,):
        raise ValueError("%s: one column range per row expected" % name)
    if thr is not None:
        thr = np.ascontiguousarray(thr, dtype=np.float64)
        if thr.shape != (rows,):
            raise ValueError("%s: one threshold per row expected" % name)
    return lo, hi, thr


def _weights(name, rows, weights):
    """Per-row weights of a scale average, checked for one entry per row."""
    w = np.ascontiguousarray(weights, dtype=np.float64)
    if w.shape != (rows,):
        raise ValueError("%s: one weight per row expected" % name)
    return w


class Engine(object):
    """One context = one device + one stream.  Every call into the C library is made under
    `self.lock`, a re-entrant lock: compound operations of the Python surface (set the length
    policy, transform, fetch the coefficients, fetch the spectrum) hold it across all their
    steps, so concurrent callers of the shared default engine cannot interleave inside one
    another's transform (the C side keeps ONE resident job per context)."""

    def __init__(self, device=0, lib_path=None):
        self.lib = load_library(lib_path)
        if self.lib.cwtb_device_count() <= 0:
            raise EngineError("no CUDA device visible: the CUDA engine has no CPU fallback")
        h = _P()
        rc = self.lib.cwtb_create(int(device), ctypes.byref(h))
        if rc != 0:
            raise EngineError("cwtb_create(device=%d) failed with status %d" % (device, rc))
        self.h = h
        self.device = device
        self.lock = threading.RLock()
        # pinned result buffers: bookkeeping has its own small lock because buffers come back
        # from weakref finalizers on arbitrary threads (re-entrant: a finalizer may run at any
        # allocation point of the thread that already holds it)
        self._pool_lock = threading.RLock()
        self._pool = []          # idle pinned buffers, least recently released first: (nbytes, addr)
        self._pool_bytes = 0
        self._dead = []          # retired pinned buffers waiting for _reap()
        self._outstanding = 0    # result arrays still alive that alias pinned memory

    def _reap(self):
        """Free the pinned buffers the finalizers retired.  Finalizers never call into the
        library themselves (they can fire at any allocation point of any thread, also inside
        this class's critical sections); the frees happen here, under the engine lock."""
        with self._pool_lock:
            dead, self._dead = self._dead, []
        if dead and getattr(self, "h", None):
            with self.lock:
                for addr in dead:
                    self.lib.cwtb_host_free(self.h, _P(addr))

    def trim(self, keep_bytes=0):
        """Release idle pinned result buffers until at most `keep_bytes` stay pooled."""
        with self._pool_lock:
            while self._pool and self._pool_bytes > keep_bytes:
                nbytes, addr = self._pool.pop(0)
                self._pool_bytes -= nbytes
                self._dead.append(addr)
        self._reap()

    def close(self):
        """Destroy the context.  While result arrays that alias its pinned memory are alive
        only the idle pooled buffers are released; the context goes with the last array."""
        if not getattr(self, "h", None):
            return
        with self.lock:
            self._closing = True
            self.trim(0)
            if self._outstanding == 0:
                self.lib.cwtb_destroy(self.h)
                self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            msg = self.lib.cwtb_last_error(self.h)
            raise EngineError("engine status %d: %s" % (rc, (msg or b"").decode()))

    def version(self):
        return self.lib.cwtb_version().decode()

    # ---- what is resident: the engine's record (cwtb_resident_shape) -------------------------
    # The library sizes every copy from what is resident, not from the caller's arrays, so every
    # method that hands it an output array sizes that array from the same record.
    def _shape(self, product):
        """(rows, n0, precision) of the resident product; EngineError when there is none."""
        rows, n0, prec = _I(), _I64(), _I()
        self._check(self.lib.cwtb_resident_shape(self.h, int(product), ctypes.byref(rows), ctypes.byref(n0),
                                                 ctypes.byref(prec)))
        if rows.value <= 0:
            raise EngineError("no %s resident" % {PRODUCT_W: "single transform", PRODUCT_CROSS: "cross spectrum",
                                                  PRODUCT_COHERENCE: "coherence",
                                                  PRODUCT_COHERENCE3: "partial / multiple coherence",
                                                  PRODUCT_POWER: "power"}[product])
        return rows.value, n0.value, prec.value

    def _transform(self, rows=None, n0=None):
        """(rows, n0, precision) of the resident transform, which a caller's rows and n0 must match."""
        r, n, prec = self._shape(PRODUCT_W)
        if (rows is not None and rows != r) or (n0 is not None and n0 != n):
            raise ValueError("the resident transform is %d x %d, the call asks for %s x %s"
                             % (r, n, "?" if rows is None else rows, "?" if n0 is None else n0))
        return r, n, prec

    def _fam(self, family, param):
        """(family, param) of the C calls.  Morse's `param` is be or (be, ga) (ga = MORSE_GA with be
        alone); its ga goes to the context here, so every call sets it inside the same locked call as
        the transform that reads it."""
        family = int(family)
        if family != MORSE:
            return family, float(param)
        be, ga = (param, MORSE_GA) if np.ndim(param) == 0 else param
        self._check(self.lib.cwtb_set_morse_ga(self.h, float(ga)))
        return family, float(be)

    @_locked
    def set_band_eps(self, eps):
        self._check(self.lib.cwtb_set_band_eps(self.h, float(eps)))

    @_locked
    def set_expand_eps(self, eps64=5e-13, eps32=2e-7):
        """Tolerance of the band-limited expansion path (include/cwt_b200.h); 0 switches it off
        (every scale through the exact pruned transforms)."""
        self._check(self.lib.cwtb_set_expand_eps(self.h, float(eps64), float(eps32)))

    @_locked
    def set_smooth_filter(self, table=None):
        """Real frequency responses [rows, n] of the time smoothing used by smooth / wct / wct_mc
        instead of Morlet's Gaussian; None restores the Gaussian."""
        if table is None:
            self._check(self.lib.cwtb_set_smooth_filter(self.h, None, 0, 0))
            return
        t = np.ascontiguousarray(table, dtype=np.float64)
        self._check(self.lib.cwtb_set_smooth_filter(self.h, _ptr(t), t.shape[0], t.shape[1]))

    @_locked
    def set_padding(self, pad_to_pow2):
        """True (default): pad to the next power of two like the reference's scipy branch;
        False: transform at the signal's own length (the reference's pyfftw policy)."""
        self._check(self.lib.cwtb_set_padding(self.h, 1 if pad_to_pow2 else 0))
        self._pad_pow2 = bool(pad_to_pow2)

    # ---- pinned host arrays -------------------------------------------------------
    @_locked
    def pinned_empty(self, shape, dtype):
        """numpy array backed by page-locked memory owned by the engine context."""
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        p = _P()
        self._check(self.lib.cwtb_host_alloc(self.h, max(n, 1), ctypes.byref(p)))
        buf = (ctypes.c_char * max(n, 1)).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
        return arr, p

    @_locked
    def pinned_free(self, p):
        self.lib.cwtb_host_free(self.h, p)

    #: results at least this large are returned in page-locked memory (D2H at PCIe speed)
    PINNED_MIN_BYTES = 1 << 20
    #: idle pinned memory kept for reuse (env CWTB_POOL_MB).  Default: room for one result of
    #: the north-star size (4.3 GB) so that steady-state calls neither allocate nor pin; least
    #: recently released buffers of any size are evicted first.
    POOL_MAX_BYTES = int(os.environ.get("CWTB_POOL_MB", "4608")) << 20
    _closing = False

    def result_array(self, shape, dtype):
        """Array for a transform result.  Large results alias pinned host memory taken
        from a per-engine pool; the buffer returns to the pool when the array (and every
        view of it) is garbage-collected, so steady-state calls neither allocate nor pin."""
        dtype = np.dtype(dtype)
        count = int(np.prod(shape))
        nbytes = count * dtype.itemsize
        if nbytes < self.PINNED_MIN_BYTES:
            return np.empty(shape, dtype=dtype)
        self._reap()
        addr = None
        with self._pool_lock:
            for i in range(len(self._pool) - 1, -1, -1):     # most recently released first
                if self._pool[i][0] == nbytes:
                    addr = self._pool.pop(i)[1]
                    self._pool_bytes -= nbytes
                    break
        if addr is None:
            p = _P()
            with self.lock:
                rc = self.lib.cwtb_host_alloc(self.h, nbytes, ctypes.byref(p))
            if rc != 0 or not p.value:
                self.trim(0)      # give pooled buffers of other sizes back and retry once
                with self.lock:
                    rc = self.lib.cwtb_host_alloc(self.h, nbytes, ctypes.byref(p))
            if rc != 0 or not p.value:
                # page-locked memory exhausted: an ordinary array still works, the copy is slower
                return np.empty(shape, dtype=dtype)
            addr = p.value
        buf = (ctypes.c_char * nbytes).from_address(addr)
        with self._pool_lock:
            self._outstanding += 1
        fin = weakref.finalize(buf, self._release, nbytes, addr)
        fin.atexit = False
        return np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)

    def _release(self, nbytes, addr):
        """Finalizer of a pinned result array (any thread, any time): pool the buffer and
        retire the least recently released ones beyond POOL_MAX_BYTES.  No library calls."""
        with self._pool_lock:
            self._outstanding -= 1
            last = self._outstanding == 0
            if self.h is None:
                return
            if self._closing or nbytes > self.POOL_MAX_BYTES:
                self._dead.append(addr)
            else:
                self._pool.append((nbytes, addr))
                self._pool_bytes += nbytes
                while self._pool_bytes > self.POOL_MAX_BYTES and len(self._pool) > 1:
                    nb, ad = self._pool.pop(0)
                    self._pool_bytes -= nb
                    self._dead.append(ad)
        if self._closing and last and self.lock.acquire(blocking=False):
            try:
                self.close()
            finally:
                self.lock.release()

    # ---- transform ------------------------------------------------------------------
    @_locked
    def cwt(self, signal, dt, scales, family, param, precision=F64, table=None,
            fetch=True, out_f64=True):
        sig = np.ascontiguousarray(signal)
        if sig.dtype == np.float32:
            is32 = 1
        else:
            sig = np.ascontiguousarray(sig, dtype=np.float64)
            is32 = 0
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        tptr = None
        if table is not None:
            table = np.ascontiguousarray(table, dtype=np.complex128)
            tptr = _ptr(table)
        with self.lock:
            if fetch and table is None:
                # transform and copy back in one call: the engine starts the device->host copy
                # of the rows that are finished first while the remaining kernels still run
                dtype = np.complex128 if (precision == F64 or out_f64) else np.complex64
                W = self.result_array((sj.size, sig.size), dtype)
                self._check(self.lib.cwtb_cwt_to_host(self.h, _ptr(sig), is32, sig.size, float(dt),
                                                      _ptr(sj), sj.size, *self._fam(family, param),
                                                      int(precision), _ptr(W), 1 if out_f64 else 0))
                return W
            self._check(self.lib.cwtb_cwt(self.h, _ptr(sig), is32, sig.size, float(dt),
                                          _ptr(sj), sj.size, *self._fam(family, param),
                                          int(precision), tptr))
            if not fetch:
                return None
            return self.get_w(sj.size, sig.size, precision, out_f64)

    @_locked
    def get_w(self, nrows, n0, precision=F64, out_f64=True):
        """The first `nrows` rows of the resident transform: complex128, or complex64 for an fp32
        transform with out_f64 False.  The element type is the transform's; `precision` is not
        read."""
        rows, _, prec = self._transform(None, n0)
        if nrows > rows:
            raise ValueError("get_w: %d rows requested, %d resident" % (nrows, rows))
        dtype = np.complex128 if (prec == F64 or out_f64) else np.complex64
        W = self.result_array((nrows, n0), dtype)
        self._check(self.lib.cwtb_get_w(self.h, _ptr(W), 1 if out_f64 else 0, 0, nrows))
        return W

    @_locked
    def signal_fft(self):
        npad = int(self.lib.cwtb_padded_length(self.h))
        out = np.empty(max(npad // 2 - 1, 0), dtype=np.complex128)
        if out.size:
            self._check(self.lib.cwtb_get_signal_fft(self.h, _ptr(out)))
        return out

    @_locked
    def job_serial(self):
        return int(self.lib.cwtb_job_serial(self.h))

    @_locked
    def padded_length(self):
        return int(self.lib.cwtb_padded_length(self.h))

    @_locked
    def last_plan(self, n):
        out = (ctypes.c_int * n)()
        m = self.lib.cwtb_last_plan(self.h, out, n)
        return list(out)[:max(m, 0)]

    @_locked
    def last_kernel_ms(self):
        return float(self.lib.cwtb_last_kernel_ms(self.h))

    @_locked
    def last_launch_count(self):
        return int(self.lib.cwtb_last_launch_count(self.h))

    @_locked
    def fft_c2c(self, x, sign, precision=F64):
        x = np.ascontiguousarray(x, dtype=np.complex128)
        if x.ndim == 1:
            x = x[None, :]
        out = np.empty_like(x)
        self._check(self.lib.cwtb_fft_c2c(self.h, _ptr(x), _ptr(out), x.shape[1],
                                          x.shape[0], int(sign), int(precision)))
        return out

    # ---- reductions / derived products of the resident transform ------------------------
    @_locked
    def icwt_sum(self, W=None, scales=None):
        """sum_j Re(W[j, :]) / sqrt(s_j): of the resident transform (W is None) or of a host
        array W[S, n]."""
        with self.lock:
            if W is None:
                _, n0, _ = self._shape(PRODUCT_W)
                out = self.result_array((n0,), np.float64)     # pinned when large: D2H at PCIe speed
                self._check(self.lib.cwtb_icwt_sum(self.h, _ptr(out)))
                return out
            W = np.ascontiguousarray(W, dtype=np.complex128)
            sj = np.ascontiguousarray(scales, dtype=np.float64)
            out = np.empty(W.shape[1], dtype=np.float64)
            self._check(self.lib.cwtb_icwt_sum_host(self.h, _ptr(W), _ptr(sj), W.shape[0],
                                                    W.shape[1], _ptr(out)))
            return out

    @_locked
    def global_power(self, nrows):
        self._transform(nrows)
        out = np.empty(nrows, dtype=np.float64)
        self._check(self.lib.cwtb_global_power(self.h, _ptr(out)))
        return out

    @_locked
    def global_power_ranges(self, lo, hi):
        """Row means of |W|^2 over the column ranges [lo[j], hi[j]) (NaN where empty)."""
        lo = np.ascontiguousarray(lo, dtype=np.int64)
        hi = np.ascontiguousarray(hi, dtype=np.int64)
        if lo.shape != hi.shape:
            raise ValueError("global_power_ranges: lo and hi must have one entry per row")
        self._transform(lo.size)
        out = np.empty(lo.size, dtype=np.float64)
        with self.lock:
            self._check(self.lib.cwtb_global_power_ranges(self.h, _ptr(lo), _ptr(hi), _ptr(out)))
        return out

    @_locked
    def power(self, nrows, n0, row_scale=None):
        """|W|^2 of the resident transform, optionally times one factor per row."""
        self._transform(nrows, n0)
        out = self.result_array((nrows, n0), np.float64)
        with self.lock:
            if row_scale is None:
                self._check(self.lib.cwtb_get_power(self.h, _ptr(out)))
            else:
                rs = np.ascontiguousarray(row_scale, dtype=np.float64)
                if rs.size != nrows:
                    raise ValueError("power: one factor per row expected")
                self._check(self.lib.cwtb_get_power_scaled(self.h, _ptr(rs), _ptr(out)))
        return out

    @_locked
    def scale_avg_power(self, weights):
        """sum_j weights[j] |W[j, :]|^2 of the resident transform (TC98 eq. 24)."""
        w = np.ascontiguousarray(weights, dtype=np.float64)
        _, n0, _ = self._transform(w.size)
        out = self.result_array((n0,), np.float64)
        with self.lock:
            self._check(self.lib.cwtb_scale_avg_power(self.h, _ptr(w), _ptr(out)))
        return out

    # ---- cross wavelet / coherence ------------------------------------------------------
    @_locked
    def xwt(self, y1, y2, dt, scales, family, param, precision=F64):
        """W12 = W1 conj(W2) (complex128 whatever `precision`, the arithmetic of the call)."""
        y1 = np.ascontiguousarray(y1, dtype=np.float64)
        y2 = np.ascontiguousarray(y2, dtype=np.float64)
        if y1.shape != y2.shape or y1.ndim != 1:
            raise ValueError("xwt: the two series must be 1-D and of equal length")
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        out = self.result_array((sj.size, y1.size), np.complex128)
        with self.lock:
            self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
            self._check(self.lib.cwtb_xwt(self.h, _ptr(y1), _ptr(y2), y1.size, float(dt), _ptr(sj),
                                          sj.size, *self._fam(family, param), _ptr(out)))
        return out

    @_locked
    def wct(self, y1, y2, dt, dj, scales, family, param, boxcar_len, want_angle=True, precision=F64):
        y1 = np.ascontiguousarray(y1, dtype=np.float64)
        y2 = np.ascontiguousarray(y2, dtype=np.float64)
        if y1.shape != y2.shape or y1.ndim != 1:
            raise ValueError("wct: the two series must be 1-D and of equal length")
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        WCT = self.result_array((sj.size, y1.size), np.float64)
        aWCT = self.result_array((sj.size, y1.size), np.float64) if want_angle else None
        with self.lock:
            self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
            self._check(self.lib.cwtb_wct(self.h, _ptr(y1), _ptr(y2), y1.size, float(dt), float(dj),
                                          _ptr(sj), sj.size, *self._fam(family, param),
                                          int(boxcar_len), _ptr(WCT),
                                          _ptr(aWCT) if want_angle else None))
        return WCT, aWCT

    @_locked
    def wct3(self, y, x1, x2, dt, dj, scales, family, param, boxcar_len, want_partial=True,
             want_multiple=True, precision=F64):
        """(RP2, RM2): partial coherence of y with x1 (x2 removed) and multiple coherence of y on
        x1 and x2, float64 [S, n0]; a measure not asked for is None.  No transform is resident
        afterwards; the resident coherence and cross spectrum are left alone."""
        ys = [np.ascontiguousarray(v, dtype=np.float64) for v in (y, x1, x2)]
        if any(v.ndim != 1 or v.shape != ys[0].shape for v in ys):
            raise ValueError("wct3: the three series must be 1-D and of equal length")
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        RP2 = self.result_array((sj.size, ys[0].size), np.float64) if want_partial else None
        RM2 = self.result_array((sj.size, ys[0].size), np.float64) if want_multiple else None
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        self._check(self.lib.cwtb_wct3(self.h, _ptr(ys[0]), _ptr(ys[1]), _ptr(ys[2]), ys[0].size,
                                       float(dt), float(dj), _ptr(sj), sj.size,
                                       *self._fam(family, param), int(boxcar_len),
                                       _ptr(RP2) if want_partial else None,
                                       _ptr(RM2) if want_multiple else None))
        return RP2, RM2

    # ---- resident coherence and cross spectrum (device buffers of their own, see
    # include/cwt_b200.h) and the reads of a resident field ------------------------------------

    @_locked
    def wct_resident(self, y1, y2, dt, dj, scales, family, param, boxcar_len, precision=F64):
        """`wct` with WCT and aWCT kept on the device; returns the coherence serial that
        identifies them."""
        y1 = np.ascontiguousarray(y1, dtype=np.float64)
        y2 = np.ascontiguousarray(y2, dtype=np.float64)
        if y1.shape != y2.shape or y1.ndim != 1:
            raise ValueError("wct_resident: the two series must be 1-D and of equal length")
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        self._check(self.lib.cwtb_wct_resident(self.h, _ptr(y1), _ptr(y2), y1.size, float(dt), float(dj),
                                               _ptr(sj), sj.size, *self._fam(family, param),
                                               int(boxcar_len)))
        return self.coherence_serial()

    @_locked
    def coherence_serial(self):
        return int(self.lib.cwtb_coherence_serial(self.h))

    @_locked
    def coherence_release(self):
        self._check(self.lib.cwtb_coherence_release(self.h))

    @_locked
    def coherence_window(self, row0, nrows, row_step, col0, ncols, col_step, want_wct=True,
                         want_angle=True):
        """(WCT, aWCT)[row0::row_step][:nrows, col0::col_step][:, :ncols] of the resident
        coherence; a field not asked for is None."""
        self._shape(PRODUCT_COHERENCE)
        WCT = self.result_array((nrows, ncols), np.float64) if want_wct else None
        aWCT = self.result_array((nrows, ncols), np.float64) if want_angle else None
        self._check(self.lib.cwtb_coherence_window(
            self.h, int(row0), int(nrows), int(row_step), int(col0), int(ncols), int(col_step),
            _ptr(WCT) if want_wct else None, _ptr(aWCT) if want_angle else None))
        return WCT, aWCT

    @_locked
    def coherence_row_stats(self, lo, hi, thr=None, want_phase=False):
        """[rows, 4]: count, sum WCT, sum cos aWCT, sum sin aWCT over the columns [lo[j], hi[j])
        where thr is None or WCT > thr[j]."""
        rows, _, _ = self._shape(PRODUCT_COHERENCE)
        lo, hi, thr = _row_args("coherence_row_stats", rows, lo, hi, thr)
        out = np.empty((rows, 4), dtype=np.float64)
        self._check(self.lib.cwtb_coherence_row_stats(self.h, _ptr(lo), _ptr(hi),
                                                      None if thr is None else _ptr(thr),
                                                      1 if want_phase else 0, _ptr(out)))
        return out

    @_locked
    def coherence_scale_avg(self, weights):
        """[3, n0]: sum_j w_j WCT[j], sum_j w_j cos aWCT[j], sum_j w_j sin aWCT[j]."""
        rows, n0, _ = self._shape(PRODUCT_COHERENCE)
        w = _weights("coherence_scale_avg", rows, weights)
        out = self.result_array((3, n0), np.float64)
        self._check(self.lib.cwtb_coherence_scale_avg(self.h, _ptr(w), _ptr(out)))
        return out

    @_locked
    def wct3_resident(self, y, x1, x2, dt, dj, scales, family, param, boxcar_len, precision=F64):
        """`wct3` with RP2, the partial phase and RM2 kept on the device; returns the serial
        that identifies them.  No transform is resident afterwards."""
        ys = [np.ascontiguousarray(v, dtype=np.float64) for v in (y, x1, x2)]
        if any(v.ndim != 1 or v.shape != ys[0].shape for v in ys):
            raise ValueError("wct3_resident: the three series must be 1-D and of equal length")
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        self._check(self.lib.cwtb_wct3_resident(self.h, _ptr(ys[0]), _ptr(ys[1]), _ptr(ys[2]),
                                                ys[0].size, float(dt), float(dj), _ptr(sj), sj.size,
                                                *self._fam(family, param), int(boxcar_len)))
        return self.coherence3_serial()

    @_locked
    def coherence3_serial(self):
        return int(self.lib.cwtb_coherence3_serial(self.h))

    @_locked
    def coherence3_release(self):
        self._check(self.lib.cwtb_coherence3_release(self.h))

    @_locked
    def coherence3_window(self, measure, row0, nrows, row_step, col0, ncols, col_step,
                          want_value=True, want_phase=False):
        """(R, phase)[row0::row_step][:nrows, col0::col_step][:, :ncols] of the resident measure
        (MEASURE_PARTIAL: RP2 and the partial phase; MEASURE_MULTIPLE: RM2, no phase); a field
        not asked for is None."""
        self._shape(PRODUCT_COHERENCE3)
        R = self.result_array((nrows, ncols), np.float64) if want_value else None
        ph = self.result_array((nrows, ncols), np.float64) if want_phase else None
        self._check(self.lib.cwtb_coherence3_window(
            self.h, int(measure), int(row0), int(nrows), int(row_step), int(col0), int(ncols),
            int(col_step), _ptr(R) if want_value else None, _ptr(ph) if want_phase else None))
        return R, ph

    @_locked
    def coherence3_row_stats(self, measure, lo, hi, thr=None, want_phase=False):
        """[rows, 4]: count, sum R, sum cos phase, sum sin phase over the columns [lo[j], hi[j])
        where thr is None or R > thr[j]."""
        rows, _, _ = self._shape(PRODUCT_COHERENCE3)
        lo, hi, thr = _row_args("coherence3_row_stats", rows, lo, hi, thr)
        out = np.empty((rows, 4), dtype=np.float64)
        self._check(self.lib.cwtb_coherence3_row_stats(self.h, int(measure), _ptr(lo), _ptr(hi),
                                                       None if thr is None else _ptr(thr),
                                                       1 if want_phase else 0, _ptr(out)))
        return out

    @_locked
    def coherence3_scale_avg(self, measure, weights):
        """[3, n0]: sum_j w_j R[j], sum_j w_j cos phase[j], sum_j w_j sin phase[j] (the last two
        0 for MEASURE_MULTIPLE)."""
        rows, n0, _ = self._shape(PRODUCT_COHERENCE3)
        w = _weights("coherence3_scale_avg", rows, weights)
        out = self.result_array((3, n0), np.float64)
        self._check(self.lib.cwtb_coherence3_scale_avg(self.h, int(measure), _ptr(w), _ptr(out)))
        return out

    @_locked
    def xwt_resident(self, y1, y2, dt, scales, family, param, precision=F64):
        """`xwt` with W12 kept on the device; returns the cross serial that identifies it.  No
        transform is resident afterwards."""
        y1 = np.ascontiguousarray(y1, dtype=np.float64)
        y2 = np.ascontiguousarray(y2, dtype=np.float64)
        if y1.shape != y2.shape or y1.ndim != 1:
            raise ValueError("xwt_resident: the two series must be 1-D and of equal length")
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        self._check(self.lib.cwtb_xwt_resident(self.h, _ptr(y1), _ptr(y2), y1.size, float(dt),
                                               _ptr(sj), sj.size, *self._fam(family, param)))
        return self.cross_serial()

    @_locked
    def cross_serial(self):
        return int(self.lib.cwtb_cross_serial(self.h))

    @_locked
    def cross_release(self):
        self._check(self.lib.cwtb_cross_release(self.h))

    @_locked
    def field_get(self, field):
        """The whole field, complex128 [rows, n0]."""
        rows, n0, _ = self._shape(field)
        out = self.result_array((rows, n0), np.complex128)
        self._check(self.lib.cwtb_field_get(self.h, int(field), 0, rows, _ptr(out)))
        return out

    @_locked
    def field_window(self, field, row0, nrows, row_step, col0, ncols, col_step):
        """F[row0::row_step][:nrows, col0::col_step][:, :ncols] as complex128."""
        self._shape(field)
        out = self.result_array((nrows, ncols), np.complex128)
        self._check(self.lib.cwtb_field_window(self.h, int(field), int(row0), int(nrows), int(row_step),
                                               int(col0), int(ncols), int(col_step), _ptr(out)))
        return out

    @_locked
    def field_row_stats(self, field, lo, hi, thr=None):
        """[rows, 5]: count, sum |F|^2, sum |F|, sum cos arg F, sum sin arg F over the columns
        [lo[j], hi[j]) where thr is None or |F|^2 > thr[j]."""
        rows, _, _ = self._shape(field)
        lo, hi, thr = _row_args("field_row_stats", rows, lo, hi, thr)
        out = np.empty((rows, 5), dtype=np.float64)
        self._check(self.lib.cwtb_field_row_stats(self.h, int(field), _ptr(lo), _ptr(hi),
                                                  None if thr is None else _ptr(thr), _ptr(out)))
        return out

    def _reconstruct(self, name, product, weights, lo, hi, thr, call):
        """float64 [n0] of a cwtb_*_reconstruct `call(w, lo, hi, thr, out)` on the resident product."""
        rows, n0, _ = self._shape(product)
        w = _weights(name, rows, weights)
        lo, hi, thr = _row_args(name, rows, lo, hi, thr)
        out = self.result_array((n0,), np.float64)
        self._check(call(_ptr(w), _ptr(lo), _ptr(hi), None if thr is None else _ptr(thr), _ptr(out)))
        return out

    @_locked
    def field_reconstruct(self, field, weights, lo, hi, thr=None):
        """sum_j weights[j] Re F[j, n] (float64, n0) over the columns [lo[j], hi[j]) where thr is None
        or |F|^2 > thr[j] (cwtb_field_reconstruct: W or the power's W)."""
        return self._reconstruct("field_reconstruct", field, weights, lo, hi, thr,
                                 lambda *a: self.lib.cwtb_field_reconstruct(self.h, int(field), *a))

    @_locked
    def cross_scale_avg(self, weights):
        """sum_j w_j W12[j, :] (complex128, n0)."""
        rows, n0, _ = self._shape(PRODUCT_CROSS)
        w = _weights("cross_scale_avg", rows, weights)
        out = self.result_array((n0,), np.complex128)
        self._check(self.lib.cwtb_cross_scale_avg(self.h, _ptr(w), _ptr(out)))
        return out

    @_locked
    def smooth(self, W, dt, scales, boxcar_len):
        W = np.ascontiguousarray(W)
        is_c = np.iscomplexobj(W)
        W = np.ascontiguousarray(W, dtype=np.complex128 if is_c else np.float64)
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        if W.ndim != 2 or sj.ndim != 1 or sj.size != W.shape[0]:
            # the reference fails here too (broadcast of the [S, 1] filter against W, mothers.py:87)
            raise ValueError("smooth: W must be [scales, time] with one scale per row "
                             "(got W %s, %d scales)" % (W.shape, sj.size))
        out = np.empty_like(W)
        with self.lock:
            self._check(self.lib.cwtb_smooth(self.h, _ptr(W), int(is_c), W.shape[0], W.shape[1],
                                             float(dt), _ptr(sj), int(boxcar_len), _ptr(out)))
        return out

    @_locked
    def wct_mc(self, noise, dt, dj, scales, family, param, boxcar_len, mask, maxscale, nbins,
               hist, precision=F64):
        noise = np.ascontiguousarray(noise, dtype=np.float64)
        if noise.ndim != 3 or noise.shape[1] != 2:
            raise ValueError("wct_mc: surrogates must be [pairs, 2, n0]")
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        if mask.shape != (sj.size, noise.shape[2]):
            raise ValueError("wct_mc: mask must be [scales, n0]")
        h, _ = self._mc_hists("wct_mc", sj.size, nbins, hist, None)
        with self.lock:
            self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
            self._check(self.lib.cwtb_wct_mc(self.h, _ptr(noise), noise.shape[0], noise.shape[2],
                                             float(dt), float(dj), _ptr(sj), sj.size,
                                             *self._fam(family, param), int(boxcar_len), _ptr(mask),
                                             int(maxscale), int(nbins), h))
        return hist

    @_locked
    def wct_mc_seeded(self, seed, first_pair, n_pairs, n0, dt, scales, family, param, boxcar_len, mask,
                      maxscale, nbins, hist, precision=F64):
        """Monte-Carlo coherence histograms of `n_pairs` surrogate pairs drawn on the device
        (Philox stream keyed by (seed, pair number)); accumulated into `hist`."""
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        if mask.shape != (sj.size, int(n0)):
            raise ValueError("wct_mc_seeded: mask must be [scales, n0]")
        h, _ = self._mc_hists("wct_mc_seeded", sj.size, nbins, hist, None)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        self._check(self.lib.cwtb_wct_mc_seeded(self.h, int(seed) & (2 ** 64 - 1), int(first_pair), int(n_pairs),
                                                int(n0), float(dt), _ptr(sj), sj.size,
                                                *self._fam(family, param), int(boxcar_len), _ptr(mask), int(maxscale),
                                                int(nbins), h))
        return hist

    @_locked
    def mc_surrogates(self, seed, first_pair, n_pairs, n0):
        out = np.empty((int(n_pairs), 2, int(n0)), dtype=np.float64)
        self._check(self.lib.cwtb_mc_surrogates(self.h, int(seed) & (2 ** 64 - 1), int(first_pair),
                                                int(n_pairs), int(n0), _ptr(out)))
        return out

    @staticmethod
    def _mc_hists(name, S, nbins, hist_a, hist_b):
        """The histograms of a Monte-Carlo call (two series: hist_b None; three: the partial and
        the multiple coherence), checked; at least one given."""
        if hist_a is None and hist_b is None:
            raise ValueError("%s: no histogram given" % name)
        for h in (hist_a, hist_b):
            if h is not None and not (h.dtype == np.int64 and h.flags.c_contiguous and h.shape == (S, nbins)):
                raise ValueError("%s: histograms must be C-contiguous int64 [%d, %d]" % (name, S, nbins))
        return [None if h is None else _ptr(h) for h in (hist_a, hist_b)]

    @_locked
    def wct3_mc(self, noise, dt, scales, family, param, boxcar_len, mask, maxscale, nbins,
                hist_partial, hist_multiple, precision=F64):
        """Monte-Carlo histograms of the partial (RP2) and multiple (RM2) coherence of the
        surrogate triples noise[n_triples, 3, n0] (y, x1, x2), accumulated into the given
        histograms [S, nbins] (either may be None)."""
        noise = np.ascontiguousarray(noise, dtype=np.float64)
        if noise.ndim != 3 or noise.shape[1] != 3:
            raise ValueError("wct3_mc: surrogates must be [triples, 3, n0]")
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        if mask.shape != (sj.size, noise.shape[2]):
            raise ValueError("wct3_mc: mask must be [scales, n0]")
        hp, hm = self._mc_hists("wct3_mc", sj.size, nbins, hist_partial, hist_multiple)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        self._check(self.lib.cwtb_wct3_mc(self.h, _ptr(noise), noise.shape[0], noise.shape[2], float(dt),
                                          _ptr(sj), sj.size, *self._fam(family, param), int(boxcar_len),
                                          _ptr(mask), int(maxscale), int(nbins), hp, hm))
        return hist_partial, hist_multiple

    @_locked
    def wct3_mc_seeded(self, seed, first_triple, n_triples, n0, dt, scales, family, param, boxcar_len,
                       mask, maxscale, nbins, hist_partial, hist_multiple, precision=F64):
        """`wct3_mc` with the triples drawn on the device (Philox stream keyed by (seed, triple
        number), disjoint from the pairs of `wct_mc_seeded`)."""
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        if mask.shape != (sj.size, int(n0)):
            raise ValueError("wct3_mc_seeded: mask must be [scales, n0]")
        hp, hm = self._mc_hists("wct3_mc_seeded", sj.size, nbins, hist_partial, hist_multiple)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        self._check(self.lib.cwtb_wct3_mc_seeded(self.h, int(seed) & (2 ** 64 - 1), int(first_triple),
                                                 int(n_triples), int(n0), float(dt), _ptr(sj), sj.size,
                                                 *self._fam(family, param), int(boxcar_len), _ptr(mask),
                                                 int(maxscale), int(nbins), hp, hm))
        return hist_partial, hist_multiple

    @_locked
    def mc_surrogates3(self, seed, first_triple, n_triples, n0):
        """The triples of the seeded mode, float64 [n_triples, 3, n0]."""
        out = np.empty((int(n_triples), 3, int(n0)), dtype=np.float64)
        self._check(self.lib.cwtb_mc_surrogates3(self.h, int(seed) & (2 ** 64 - 1), int(first_triple),
                                                 int(n_triples), int(n0), _ptr(out)))
        return out

    @staticmethod
    def _phase_inputs(name, series, groups):
        """The data [nser, n0] and the phase groups of a phase-randomised Monte-Carlo call."""
        series = np.ascontiguousarray(series, dtype=np.float64)
        groups = np.ascontiguousarray(groups, dtype=np.int32)
        if series.ndim != 2 or series.shape[0] not in (2, 3) or groups.shape != (series.shape[0],):
            raise ValueError("%s: series must be [2 or 3, n0] with one phase group each" % name)
        if not np.isfinite(series).all():
            raise ValueError("%s: non-finite sample" % name)
        return series, groups

    @classmethod
    def _null_inputs(cls, name, series, null):
        """The data [nser, n0], the C arguments null, group, g, m, sigma, held of a coherence
        Monte-Carlo call (cwtb_wct_mc_null) and the arrays behind them, which the caller keeps alive
        across the call.  `null` is a CoherenceNull, or the phase groups of the phase null."""
        if not isinstance(null, CoherenceNull):
            null = CoherenceNull(NULL_PHASE, null)
        if null.kind != NULL_AR1:   # the phase null, or an unknown one for the engine to refuse
            series, groups = cls._phase_inputs(name, series, null.groups)
            return series, (int(null.kind), _ptr(groups), None, None, None, None), groups
        series = np.ascontiguousarray(series, dtype=np.float64)
        if series.ndim != 2 or series.shape[0] not in (2, 3):
            raise ValueError("%s: series must be [2 or 3, n0]" % name)
        nser = series.shape[0]
        held = np.zeros(nser) if null.held is None else null.held
        arrays = tuple(np.ascontiguousarray(v, dtype=t) for v, t in ((null.g, np.float64), (null.m, np.float64),
                                                                     (null.sigma, np.float64), (held, np.int32)))
        if any(v.shape != (nser,) for v in arrays):
            raise ValueError("%s: g, m, sigma and held take one entry per series (%d)" % (name, nser))
        if not np.isfinite(series[arrays[3] != 0]).all():
            raise ValueError("%s: non-finite sample in a held series" % name)
        return series, (NULL_AR1, None) + tuple(_ptr(v) for v in arrays), arrays

    @_locked
    def wct_mc_phase(self, series, null, seed, first_unit, n_units, dt, scales, family, param, boxcar_len,
                     mask, maxscale, nbins, hist_a, hist_b=None, precision=F64):
        """Monte-Carlo histograms of `n_units` surrogate units of `series` [nser, n0]
        (cwtb_wct_mc_null): `null` the phase groups of phase-randomised units (series of equal group
        number share the random phases and keep their coherence) or a CoherenceNull.  Two series:
        `hist_a` the coherence histogram.  Three (y, x1, x2): `hist_a` the partial, `hist_b` the
        multiple coherence, either may be None.  Accumulated into the histograms [S, nbins]."""
        series, nargs, _keep = self._null_inputs("wct_mc_phase", series, null)
        nser, n0 = series.shape
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        if mask.shape != (sj.size, n0):
            raise ValueError("wct_mc_phase: mask must be [scales, n0]")
        if nser == 2 and hist_b is not None:
            raise ValueError("wct_mc_phase: two series have one histogram")
        ha, hb = self._mc_hists("wct_mc_phase", sj.size, nbins, hist_a, hist_b)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        self._check(self.lib.cwtb_wct_mc_null(self.h, _ptr(series), nser, *nargs, int(seed) & (2 ** 64 - 1),
                                              int(first_unit), int(n_units), n0, float(dt), _ptr(sj), sj.size,
                                              *self._fam(family, param), int(boxcar_len), _ptr(mask),
                                              int(maxscale), int(nbins), ha, hb))
        return hist_a, hist_b

    @_locked
    def mc_phase_surrogates(self, series, groups, seed, first_unit, n_units):
        """The surrogate units of `wct_mc_phase`, float64 [n_units, nser, n0]."""
        series, groups = self._phase_inputs("mc_phase_surrogates", series, groups)
        out = np.empty((int(n_units),) + series.shape, dtype=np.float64)
        self._check(self.lib.cwtb_mc_phase_surrogates(self.h, _ptr(series), series.shape[0], _ptr(groups),
                                                      int(seed) & (2 ** 64 - 1), int(first_unit), int(n_units),
                                                      series.shape[1], _ptr(out)))
        return out

    # ---- point-wise tests of a resident coherence against phase-randomised surrogates ----------
    # `measure` None: the resident coherence (cwtb_coherence_*); MEASURE_PARTIAL / _MULTIPLE: the
    # resident partial / multiple coherence (cwtb_coherence3_*).
    @_locked
    def surrogate_counts(self, series, null, seed, first_unit, n_units, dt, scales, family, param, boxcar_len,
                         mask, maxscale, nbins, hist_a, hist_b=None, serial=None, reset=True, precision=F64):
        """`wct_mc_phase` that also counts, per point, the units whose coherence (two series) or
        partial and multiple coherence (three) reach the resident product's, into that product's
        counters (cwtb_coherence*_surrogate_counts_null); `serial` is the product's serial.  `reset`
        zeroes the counters first, otherwise the units are added (to counts of the same null)."""
        series, nargs, _keep = self._null_inputs("surrogate_counts", series, null)
        nser, n0 = series.shape
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        if mask.shape != (sj.size, n0):
            raise ValueError("surrogate_counts: mask must be [scales, n0]")
        if nser == 2 and hist_b is not None:
            raise ValueError("surrogate_counts: two series have one histogram")
        ha, hb = self._mc_hists("surrogate_counts", sj.size, nbins, hist_a, hist_b)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        args = (self.h, _ptr(series), *nargs, int(seed) & (2 ** 64 - 1), int(first_unit), int(n_units), n0,
                float(dt), _ptr(sj), sj.size, *self._fam(family, param), int(boxcar_len), _ptr(mask), int(maxscale),
                int(nbins))
        if nser == 2:
            self._check(self.lib.cwtb_coherence_surrogate_counts_null(*args, ha, int(serial), 1 if reset else 0))
        else:
            self._check(self.lib.cwtb_coherence3_surrogate_counts_null(*args, ha, hb, int(serial), 1 if reset else 0))
        return hist_a, hist_b

    @_locked
    def pvalue_window(self, measure, row0, nrows, row_step, col0, ncols, col_step):
        """p = (1 + k) / (1 + M) [row0::row_step][:nrows, col0::col_step][:, :ncols] of the counts
        of the resident product, NaN where its value is not finite."""
        P = self.result_array((nrows, ncols), np.float64)
        w = (int(row0), int(nrows), int(row_step), int(col0), int(ncols), int(col_step), _ptr(P))
        if measure is None:
            self._shape(PRODUCT_COHERENCE)
            self._check(self.lib.cwtb_coherence_pvalue_window(self.h, *w))
        elif measure in _COMPLEX:
            self._shape(_COMPLEX[measure])
            self._check(getattr(self.lib, "cwtb_%s_pvalue_window" % measure)(self.h, *w))
        else:
            self._shape(PRODUCT_COHERENCE3)
            self._check(self.lib.cwtb_coherence3_pvalue_window(self.h, int(measure), *w))
        return P

    @_locked
    def pvalue_row_stats(self, measure, lo, hi, kmax, thr=None, want_phase=False):
        """[rows, 4] of `coherence_row_stats` / `coherence3_row_stats` ([rows, 5] of
        `field_row_stats` for the power and the cross spectrum) over the points with a finite value and
        a count k <= kmax."""
        if measure in _COMPLEX:
            rows, _, _ = self._shape(_COMPLEX[measure])
            lo, hi, thr = _row_args("pvalue_row_stats", rows, lo, hi, thr)
            out = np.empty((rows, 5), dtype=np.float64)
            fn = getattr(self.lib, "cwtb_%s_pvalue_row_stats" % measure)
            self._check(fn(self.h, _ptr(lo), _ptr(hi), None if thr is None else _ptr(thr), int(kmax), _ptr(out)))
            return out
        rows, _, _ = self._shape(PRODUCT_COHERENCE if measure is None else PRODUCT_COHERENCE3)
        lo, hi, thr = _row_args("pvalue_row_stats", rows, lo, hi, thr)
        out = np.empty((rows, 4), dtype=np.float64)
        a = (_ptr(lo), _ptr(hi), None if thr is None else _ptr(thr), int(kmax), 1 if want_phase else 0, _ptr(out))
        if measure is None:
            self._check(self.lib.cwtb_coherence_pvalue_row_stats(self.h, *a))
        else:
            self._check(self.lib.cwtb_coherence3_pvalue_row_stats(self.h, int(measure), *a))
        return out

    @_locked
    def count_hist(self, measure, lo, hi, nbins):
        """int64 [nbins]: the number of points with count k over the columns [lo[j], hi[j]) whose
        value is finite; nbins must be M + 1."""
        rows, _, _ = self._shape(PRODUCT_COHERENCE if measure is None else
                                 _COMPLEX[measure] if measure in _COMPLEX else PRODUCT_COHERENCE3)
        lo, hi, _ = _row_args("count_hist", rows, lo, hi, None)
        out = np.empty(int(nbins), dtype=np.int64)
        if measure in _COMPLEX:
            fn = getattr(self.lib, "cwtb_%s_count_hist" % measure)
            self._check(fn(self.h, _ptr(lo), _ptr(hi), int(nbins), _ptr(out)))
        elif measure is None:
            self._check(self.lib.cwtb_coherence_count_hist(self.h, _ptr(lo), _ptr(hi), int(nbins), _ptr(out)))
        else:
            self._check(self.lib.cwtb_coherence3_count_hist(self.h, int(measure), _ptr(lo), _ptr(hi), int(nbins),
                                                            _ptr(out)))
        return out

    # ---- cluster tests of a resident coherence against phase-randomised surrogates ------------
    # `measure` None: the resident coherence; MEASURE_PARTIAL / _MULTIPLE: the resident partial /
    # multiple coherence.
    @_locked
    def cluster_test(self, series, null, seed, first_unit, n_units, dt, scales, family, param, boxcar_len,
                     mask, maxscale, nbins, hist_a, hist_b=None, serial=None, thr=None, lo=None, hi=None, q=None,
                     measure=None, precision=F64):
        """`wct_mc_phase` that also labels the clusters of the resident product's map and of every
        unit's (cwtb_coherence*_cluster_test_null): uint64 [n_units], the largest cluster sum Q of
        each unit.  The resident map's clusters stay with the product (`cluster_table`,
        `cluster_labels`)."""
        series, nargs, _keep = self._null_inputs("cluster_test", series, null)
        nser, n0 = series.shape
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        if mask.shape != (sj.size, n0):
            raise ValueError("cluster_test: mask must be [scales, n0]")
        if nser == 2 and (hist_b is not None or measure is not None):
            raise ValueError("cluster_test: two series have one histogram and one measure")
        ha, hb = self._mc_hists("cluster_test", sj.size, nbins, hist_a, hist_b)
        lo, hi, thr = _row_args("cluster_test", sj.size, lo, hi, thr)
        q = np.ascontiguousarray(q, dtype=np.uint64)
        if q.shape != (sj.size,):
            raise ValueError("cluster_test: q must have one entry per scale")
        qmax = np.zeros(int(n_units), dtype=np.uint64)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        args = (self.h, _ptr(series), *nargs, int(seed) & (2 ** 64 - 1), int(first_unit), int(n_units), n0,
                float(dt), _ptr(sj), sj.size, *self._fam(family, param), int(boxcar_len), _ptr(mask), int(maxscale),
                int(nbins))
        rows = (_ptr(thr), _ptr(lo), _ptr(hi), _ptr(q))
        if nser == 2:
            self._check(self.lib.cwtb_coherence_cluster_test_null(*args, ha, int(serial), *rows, _ptr(qmax)))
        else:
            self._check(self.lib.cwtb_coherence3_cluster_test_null(*args, ha, hb, int(serial), *rows, int(measure),
                                                                   _ptr(qmax)))
        return qmax

    @staticmethod
    def _table(call):
        """(Q uint64, points int64, box int64 [count, 4]) of a table call(cap, count, Q, points, box)."""
        count = _I64()
        call(0, ctypes.byref(count), None, None, None)
        m = count.value
        Q = np.empty(m, dtype=np.uint64)
        pts = np.empty(m, dtype=np.int64)
        box = np.empty((m, 4), dtype=np.int64)
        call(m, ctypes.byref(count), _ptr(Q), _ptr(pts), _ptr(box))
        return Q, pts, box

    def _cluster_call(self, triple, what):
        """cwtb_{coherence, coherence3, power, cross}_cluster_<what> for `triple` False, True, POWER or
        CROSS."""
        name = triple if triple in _COMPLEX else "coherence3" if triple else "coherence"
        return getattr(self.lib, "cwtb_%s_cluster_%s" % (name, what))

    @_locked
    def cluster_table(self, triple=False):
        """The resident map's clusters of the last cluster test of the coherence (`triple` False),
        of the partial / multiple coherence (True), of the power (POWER) or of the cross spectrum
        (CROSS): (Q, points, box [:, 4] =
        first row, last row + 1, first column, last column + 1), in table order."""
        fn = self._cluster_call(triple, "table")
        return self._table(lambda *a: self._check(fn(self.h, *a)))

    @_locked
    def cluster_labels(self, triple, row0, nrows, row_step, col0, ncols, col_step):
        """int32 labels [row0::row_step][:nrows, col0::col_step][:, :ncols] of the last cluster
        test of the coherence (`triple` False), of the partial / multiple coherence (True), of the
        power (POWER) or of the cross spectrum (CROSS): 0 off the clusters, c + 1 on table row c."""
        out = np.empty((int(nrows), int(ncols)), dtype=np.int32)
        w = (int(row0), int(nrows), int(row_step), int(col0), int(ncols), int(col_step), _ptr(out))
        self._check(self._cluster_call(triple, "labels")(self.h, *w))
        return out

    # ---- the resident power and its tests against AR(1) or phase-randomised surrogates ---------
    @_locked
    def power_resident(self, y, dt, scales, family, param, precision=F64):
        """`cwt` of `y` in `precision` with W kept on the device as the resident power; returns the
        power serial that identifies it.  No transform is resident afterwards."""
        y = np.ascontiguousarray(y, dtype=np.float64)
        if y.ndim != 1:
            raise ValueError("power_resident: the series must be 1-D")
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        self._check(self.lib.cwtb_set_coherence_precision(self.h, int(precision)))
        self._check(self.lib.cwtb_power_resident(self.h, _ptr(y), y.size, float(dt), _ptr(sj), sj.size,
                                                 *self._fam(family, param)))
        return self.power_serial()

    @_locked
    def power_serial(self):
        return int(self.lib.cwtb_power_serial(self.h))

    @_locked
    def power_release(self):
        self._check(self.lib.cwtb_power_release(self.h))

    @_locked
    def power_window(self, row0, nrows, row_step, col0, ncols, col_step):
        """P = |W|^2 [row0::row_step][:nrows, col0::col_step][:, :ncols] (float64) of the resident
        power, formed on the device as its tests form it."""
        self._shape(PRODUCT_POWER)
        out = self.result_array((nrows, ncols), np.float64)
        self._check(self.lib.cwtb_power_window(self.h, int(row0), int(nrows), int(row_step), int(col0), int(ncols),
                                               int(col_step), _ptr(out)))
        return out

    @_locked
    def power_scale_avg(self, weights):
        """sum_j w_j |W[j, :]|^2 (float64, n0) of the resident power."""
        rows, n0, _ = self._shape(PRODUCT_POWER)
        w = _weights("power_scale_avg", rows, weights)
        out = self.result_array((n0,), np.float64)
        self._check(self.lib.cwtb_power_scale_avg(self.h, _ptr(w), _ptr(out)))
        return out

    @_locked
    def power_pvalue_reconstruct(self, weights, lo, hi, kmax, thr=None):
        """`field_reconstruct` of the resident power over the points with a finite |W|^2 and k <= kmax
        of its counts (cwtb_power_pvalue_reconstruct)."""
        return self._reconstruct("power_pvalue_reconstruct", PRODUCT_POWER, weights, lo, hi, thr,
                                 lambda w, lo, hi, thr, out: self.lib.cwtb_power_pvalue_reconstruct(
                                     self.h, w, lo, hi, thr, int(kmax), out))

    @_locked
    def power_cluster_reconstruct(self, weights, lo, hi, clusters):
        """`field_reconstruct` of the resident power over the points of the clusters `clusters` (rows of
        the table) of its last cluster test (cwtb_power_cluster_reconstruct)."""
        cl = np.ascontiguousarray(clusters, dtype=np.int64).reshape(-1)
        return self._reconstruct("power_cluster_reconstruct", PRODUCT_POWER, weights, lo, hi, None,
                                 lambda w, lo, hi, thr, out: self.lib.cwtb_power_cluster_reconstruct(
                                     self.h, w, lo, hi, _ptr(cl), cl.size, out))

    @_locked
    def mc_ar1_surrogates(self, g, m, sigma, seed, first_unit, n_units, n0):
        """The AR(1) units of the power tests, float64 [n_units, n0]."""
        out = np.empty((int(n_units), int(n0)), dtype=np.float64)
        self._check(self.lib.cwtb_mc_ar1_surrogates(self.h, float(g), float(m), float(sigma),
                                                    int(seed) & (2 ** 64 - 1), int(first_unit), int(n_units),
                                                    int(n0), _ptr(out)))
        return out

    def _power_args(self, name, series, null, g, m, sigma, seed, first_unit, n_units, dt, sj, family, param, serial):
        """The arguments of a power test up to `serial` (the series: the phase null's data, 1-D).  The
        caller keeps `series` and `sj` alive across the call."""
        if series.ndim != 1:
            raise ValueError("%s: the series must be 1-D" % name)
        if null == NULL_PHASE and not np.isfinite(series).all():
            raise ValueError("%s: non-finite sample" % name)
        return (_ptr(series), int(null), float(g), float(m), float(sigma), int(seed) & (2 ** 64 - 1),
                int(first_unit), int(n_units), series.size, float(dt), _ptr(sj), sj.size,
                *self._fam(family, param), int(serial))

    @_locked
    def power_surrogate_counts(self, series, null, g, m, sigma, seed, first_unit, n_units, dt, scales, family,
                               param, serial, reset=True):
        """Count, per point, the units of the null whose power reaches the resident power's, into its
        counters (cwtb_power_surrogate_counts); `serial` is the power's serial.  `reset` zeroes the
        counters first, otherwise the units are added."""
        series = np.ascontiguousarray(series, dtype=np.float64)
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        a = self._power_args("power_surrogate_counts", series, null, g, m, sigma, seed, first_unit, n_units, dt, sj,
                             family, param, serial)
        self._check(self.lib.cwtb_power_surrogate_counts(self.h, *a, 1 if reset else 0))

    @_locked
    def power_cluster_test(self, series, null, g, m, sigma, seed, first_unit, n_units, dt, scales, family, param,
                           serial, thr, lo, hi, q):
        """Label the clusters of the resident power's map and of every unit's
        (cwtb_power_cluster_test): uint64 [n_units], the largest cluster sum Q of each unit."""
        series = np.ascontiguousarray(series, dtype=np.float64)
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        a = self._power_args("power_cluster_test", series, null, g, m, sigma, seed, first_unit, n_units, dt, sj,
                             family, param, serial)
        lo, hi, thr = _row_args("power_cluster_test", sj.size, lo, hi, thr)
        q = np.ascontiguousarray(q, dtype=np.uint64)
        if q.shape != (sj.size,):
            raise ValueError("power_cluster_test: q must have one entry per scale")
        qmax = np.zeros(int(n_units), dtype=np.uint64)
        self._check(self.lib.cwtb_power_cluster_test(self.h, *a, _ptr(thr), _ptr(lo), _ptr(hi), _ptr(q),
                                                     _ptr(qmax)))
        return qmax

    # ---- tests of the resident cross spectrum against AR(1) or phase-randomised surrogate pairs --
    @staticmethod
    def _pair_params(name, g, m, sigma):
        """The AR(1) parameters of the two series, float64 [2] each."""
        out = tuple(np.ascontiguousarray(v, dtype=np.float64) for v in (g, m, sigma))
        if any(v.shape != (2,) for v in out):
            raise ValueError("%s: g, m and sigma take one entry per series (2)" % name)
        return out

    @_locked
    def mc_ar1_pair_surrogates(self, g, m, sigma, seed, first_unit, n_units, n0):
        """The AR(1) pairs of the cross-spectrum tests, float64 [n_units, 2, n0]: series s with
        (g[s], m[s], sigma[s]) under the series tag s (series 0 is `mc_ar1_surrogates`' unit)."""
        g, m, sigma = self._pair_params("mc_ar1_pair_surrogates", g, m, sigma)
        out = np.empty((int(n_units), 2, int(n0)), dtype=np.float64)
        self._check(self.lib.cwtb_mc_ar1_pair_surrogates(self.h, _ptr(g), _ptr(m), _ptr(sigma),
                                                         int(seed) & (2 ** 64 - 1), int(first_unit), int(n_units),
                                                         int(n0), _ptr(out)))
        return out

    @_locked
    def mc_ar1_series_surrogates(self, g, m, sigma, seed, first_unit, n_units, n0):
        """The AR(1) units of len(g) = 1, 2 or 3 series, float64 [n_units, nser, n0]: series s with
        (g[s], m[s], sigma[s]) under the series tag s (two series: `mc_ar1_pair_surrogates`)."""
        g, m, sigma = (np.ascontiguousarray(v, dtype=np.float64).reshape(-1) for v in (g, m, sigma))
        if not g.shape == m.shape == sigma.shape:
            raise ValueError("mc_ar1_series_surrogates: g, m and sigma take one entry per series")
        out = np.empty((int(n_units), g.size, int(n0)), dtype=np.float64)
        self._check(self.lib.cwtb_mc_ar1_series_surrogates(self.h, g.size, _ptr(g), _ptr(m), _ptr(sigma),
                                                           int(seed) & (2 ** 64 - 1), int(first_unit), int(n_units),
                                                           int(n0), _ptr(out)))
        return out

    def _cross_args(self, name, series, null, g, m, sigma, seed, first_unit, n_units, dt, sj, family, param, serial):
        """The arguments of a cross-spectrum test up to `serial` (series [2, n0]: the phase null's
        data), and the arrays the caller keeps alive across the call."""
        series = np.ascontiguousarray(series, dtype=np.float64)
        if series.ndim != 2 or series.shape[0] != 2:
            raise ValueError("%s: the series must be [2, n0]" % name)
        if null == NULL_PHASE and not np.isfinite(series).all():
            raise ValueError("%s: non-finite sample" % name)
        g, m, sigma = self._pair_params(name, g, m, sigma)
        keep = (series, g, m, sigma)
        return (_ptr(series), int(null), _ptr(g), _ptr(m), _ptr(sigma), int(seed) & (2 ** 64 - 1), int(first_unit),
                int(n_units), series.shape[1], float(dt), _ptr(sj), sj.size, *self._fam(family, param),
                int(serial)), keep

    @_locked
    def cross_surrogate_counts(self, series, null, g, m, sigma, seed, first_unit, n_units, dt, scales, family,
                               param, serial, reset=True):
        """Count, per point, the pairs of the null whose |W12|^2 reaches the resident cross spectrum's,
        into its counters (cwtb_cross_surrogate_counts); `serial` is the cross spectrum's serial.
        `reset` zeroes the counters first, otherwise the units are added."""
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        a, _keep = self._cross_args("cross_surrogate_counts", series, null, g, m, sigma, seed, first_unit, n_units,
                                    dt, sj, family, param, serial)
        self._check(self.lib.cwtb_cross_surrogate_counts(self.h, *a, 1 if reset else 0))

    @_locked
    def cross_cluster_test(self, series, null, g, m, sigma, seed, first_unit, n_units, dt, scales, family, param,
                           serial, thr, lo, hi, q):
        """Label the clusters of the resident cross spectrum's |W12|^2 and of every pair's
        (cwtb_cross_cluster_test): uint64 [n_units], the largest cluster sum Q of each pair."""
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        a, _keep = self._cross_args("cross_cluster_test", series, null, g, m, sigma, seed, first_unit, n_units, dt,
                                    sj, family, param, serial)
        lo, hi, thr = _row_args("cross_cluster_test", sj.size, lo, hi, thr)
        q = np.ascontiguousarray(q, dtype=np.uint64)
        if q.shape != (sj.size,):
            raise ValueError("cross_cluster_test: q must have one entry per scale")
        qmax = np.zeros(int(n_units), dtype=np.uint64)
        self._check(self.lib.cwtb_cross_cluster_test(self.h, *a, _ptr(thr), _ptr(lo), _ptr(hi), _ptr(q),
                                                     _ptr(qmax)))
        return qmax

    @_locked
    def cross_cluster_row_stats(self, cluster, lo, hi):
        """[rows, 5] of `field_row_stats` over the points of cluster `cluster` (row of the table) of the
        last cross-spectrum cluster test, on the columns [lo[j], hi[j]) of each row."""
        rows, _, _ = self._shape(PRODUCT_CROSS)
        lo, hi, _ = _row_args("cross_cluster_row_stats", rows, lo, hi, None)
        out = np.empty((rows, 5), dtype=np.float64)
        self._check(self.lib.cwtb_cross_cluster_row_stats(self.h, int(cluster), _ptr(lo), _ptr(hi), _ptr(out)))
        return out

    @_locked
    def cluster_label_bits(self, bits, n0, q, want_labels=True):
        """Test hook: the cluster tests' labeller on a host bitmask uint32 [S, ceil(n0 / 32)] with the
        weights q [S]: (Q, points, box, labels int32 [S, n0] or None, qmax)."""
        bits = np.ascontiguousarray(bits, dtype=np.uint32)
        q = np.ascontiguousarray(q, dtype=np.uint64)
        if bits.ndim != 2 or bits.shape[1] != (int(n0) + 31) // 32:
            raise ValueError("cluster_label_bits: bits must be [scales, ceil(n0 / 32)]")
        S = int(bits.shape[0])
        if q.shape != (S,):
            raise ValueError("cluster_label_bits: q must have one entry per scale")
        labels = np.empty((S, int(n0)), dtype=np.int32) if want_labels else None
        qmax = np.zeros(1, dtype=np.uint64)
        lab = None if labels is None else _ptr(labels)

        def call(cap, count, Q, pts, box):
            self._check(self.lib.cwtb_cluster_label_bits(self.h, _ptr(bits), S, int(n0), _ptr(q), cap, count,
                                                         Q, pts, box, lab, _ptr(qmax)))
        Q, pts, box = self._table(call)
        return Q, pts, box, labels, int(qmax[0])

    @_locked
    def cwt_batch(self, X, dt, scales, family, param, precision=F64, want_power=True,
                  want_w=False):
        X = np.ascontiguousarray(X)
        if X.dtype != np.float32:
            X = np.ascontiguousarray(X, dtype=np.float64)
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        nch, n0 = X.shape
        power = np.empty((nch, sj.size), dtype=np.float64) if want_power else None
        W = None
        if want_w:
            W = np.empty((nch, sj.size, n0), dtype=np.complex128 if precision == F64 else np.complex64)
        with self.lock:
            self._check(self.lib.cwtb_cwt_batch(self.h, _ptr(X), int(X.dtype == np.float32), nch, n0,
                                                float(dt), _ptr(sj), sj.size,
                                                *self._fam(family, param), int(precision),
                                                _ptr(power) if want_power else None,
                                                _ptr(W) if want_w else None))
        return power, W

    # ---- device-resident benchmarking helpers -------------------------------------
    @_locked
    def dev_alloc(self, nbytes):
        p = _P()
        self._check(self.lib.cwtb_dev_alloc(self.h, nbytes, ctypes.byref(p)))
        return p

    @_locked
    def dev_free(self, p):
        self.lib.cwtb_dev_free(self.h, p)

    @_locked
    def h2d(self, dptr, arr):
        arr = np.ascontiguousarray(arr)
        self._check(self.lib.cwtb_memcpy_h2d(self.h, dptr, _ptr(arr), arr.nbytes))

    @_locked
    def cwt_dev(self, dptr, is_f32, n0, dt, scales, family, param, precision=F64):
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        self._check(self.lib.cwtb_cwt_dev(self.h, dptr, int(is_f32), int(n0), float(dt),
                                          _ptr(sj), sj.size, *self._fam(family, param),
                                          int(precision)))

    @_locked
    def cwt_batch_dev(self, dptr, n_chan, n0, dt, scales, family, param, precision=F64,
                      want_power=False):
        sj = np.ascontiguousarray(scales, dtype=np.float64)
        power = np.empty((n_chan, sj.size), dtype=np.float64) if want_power else None
        self._check(self.lib.cwtb_cwt_batch_dev(self.h, dptr, int(n_chan), int(n0), float(dt),
                                                _ptr(sj), sj.size, *self._fam(family, param),
                                                int(precision), _ptr(power) if want_power else None))
        return power

    @_locked
    def bench_last(self, iters):
        ms = _D()
        self._check(self.lib.cwtb_bench_last(self.h, int(iters), ctypes.byref(ms)))
        return ms.value

    @_locked
    def profile_last(self):
        """Per-kernel-type device times of one pass of the last cwt_dev transform:
        list of dicts {name, launches, ms, rows}."""
        buf = ctypes.create_string_buffer(1 << 16)
        n = self.lib.cwtb_profile_last(self.h, buf, len(buf))
        if n < 0:
            self._check(n)
        out = []
        for line in buf.value.decode().splitlines():
            name, nl, ms, rows = line.rsplit("|", 3)
            out.append({"name": name, "launches": int(nl), "ms": float(ms), "rows": int(rows)})
        return out

    @staticmethod
    def _parse_profile(text):
        out = []
        for line in text.splitlines():
            name, nl, ms, rows = line.rsplit("|", 3)
            out.append({"name": name, "launches": int(nl), "ms": float(ms), "rows": int(rows)})
        return out

    @_locked
    def profile_begin(self):
        """Start recording per-kernel device times of every following call (serialised streams)."""
        self._check(self.lib.cwtb_profile_begin(self.h))

    @_locked
    def profile_end(self):
        buf = ctypes.create_string_buffer(1 << 16)
        n = self.lib.cwtb_profile_end(self.h, buf, len(buf))
        if n < 0:
            self._check(n)
        return self._parse_profile(buf.value.decode())

    @_locked
    def sync(self):
        self._check(self.lib.cwtb_sync(self.h))

    # ---- multi-GPU collectives (NCCL behind the C ABI; no torch) --------------------
    def comm_unique_id(self):
        """128-byte NCCL id (rank 0 creates it, the host program distributes it)."""
        buf = ctypes.create_string_buffer(128)
        rc = self.lib.cwtb_comm_unique_id(buf)
        if rc != 0:
            raise EngineError("cwtb_comm_unique_id failed with status %d (libnccl not loadable?)" % rc)
        return buf.raw

    @_locked
    def comm_init(self, world, rank, uid):
        buf = ctypes.create_string_buffer(bytes(uid), 128)
        self._check(self.lib.cwtb_comm_init(self.h, int(world), int(rank), buf))

    @_locked
    def comm_destroy(self):
        self.lib.cwtb_comm_destroy(self.h)

    def comm_world(self):
        return int(self.lib.cwtb_comm_world(self.h))

    def comm_rank(self):
        return int(self.lib.cwtb_comm_rank(self.h))

    @_locked
    def comm_allgather(self, local):
        """Every rank contributes an equal-shape array; returns the [world, ...] stack."""
        local = np.ascontiguousarray(local)
        out = np.empty((self.comm_world(),) + local.shape, dtype=local.dtype)
        self._check(self.lib.cwtb_comm_allgather(self.h, _ptr(local), _ptr(out), local.nbytes))
        return out

    @_locked
    def comm_allreduce_sum(self, array):
        a = np.ascontiguousarray(array, dtype=np.int64).copy()
        self._check(self.lib.cwtb_comm_allreduce_sum_i64(self.h, _ptr(a), a.size))
        return a

    @_locked
    def comm_allreduce_max(self, array):
        a = np.atleast_1d(np.ascontiguousarray(array, dtype=np.float64)).copy()
        self._check(self.lib.cwtb_comm_allreduce_max_f64(self.h, _ptr(a), a.size))
        return a

    @_locked
    def comm_broadcast(self, array, root=0):
        a = np.ascontiguousarray(array).copy()
        self._check(self.lib.cwtb_comm_broadcast(self.h, _ptr(a), a.nbytes, int(root)))
        return a


_default = {}
_default_lock = threading.Lock()


def device_count():
    return int(load_library().cwtb_device_count())


def default_engine(device=None):
    """Process-wide engine per device (device from CWTB_DEVICE / LOCAL_RANK, default 0)."""
    if device is None:
        device = int(os.environ.get("CWTB_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    with _default_lock:
        if device not in _default:
            _default[device] = Engine(device)
        return _default[device]
