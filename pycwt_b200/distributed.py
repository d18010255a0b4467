"""Multi-GPU plumbing (SURVEY 8e): one process per GPU, independent units block-partitioned over
the ranks -- channels of a batched transform, scales of one long signal, surrogate pairs of the
Monte-Carlo coherence significance -- with NO collective on the data path.  What crosses the
interconnect are the reduced products: per-channel spectra [channels, scales] (all-gather),
surrogate histograms [scales, 1000] (one all-reduce), timings (max).

Two communicators with the same three methods (`allgather_rows`, `allreduce_sum`, `max`):

  * `NcclComm(engine)`  -- the product path: NCCL behind the engine's C ABI
    (include/cwt_b200.h `cwtb_comm_*`, libnccl bound at run time); no PyTorch.  The 128-byte
    NCCL id travels from rank 0 to the others through a caller-supplied exchange or, by default,
    a rendezvous file next to MASTER_PORT (ranks of one box).
  * `TorchComm(dist)`   -- torch.distributed (gloo in the CPU tests of the host logic, where no
    NCCL exists; any initialised process group works).

Every function below takes `comm=None` for the single-process case.
"""
import os
import time

import numpy as np


def shard_range(n_items, rank, world):
    """Contiguous block [lo, hi) of `n_items` owned by `rank` (sizes differ by at most 1)."""
    base, rem = divmod(int(n_items), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


# ---- communicators -----------------------------------------------------------------------
class _CommBase(object):
    rank = 0
    world = 1

    def allgather_rows(self, local, n_total):
        """All ranks contribute their block of rows (as produced by shard_range); every rank gets
        the full [n_total, ...] array back."""
        local = np.ascontiguousarray(local)
        if self.world == 1:
            return local
        sizes = [shard_range(n_total, r, self.world) for r in range(self.world)]
        maxrows = max(hi - lo for lo, hi in sizes)
        buf = np.zeros((maxrows,) + local.shape[1:], dtype=local.dtype)
        buf[:local.shape[0]] = local
        stack = self._allgather_equal(buf)
        return np.concatenate([stack[r][:hi - lo] for r, (lo, hi) in enumerate(sizes)], axis=0)


class NcclComm(_CommBase):
    """NCCL through the engine's C ABI.  `exchange(uid_or_None) -> uid` hands rank 0's id to
    every rank (rank 0 passes the id in, the others pass None); default: a rendezvous file."""

    def __init__(self, engine, rank=None, world=None, exchange=None):
        self.engine = engine
        self.rank = int(os.environ.get("RANK", "0")) if rank is None else int(rank)
        self.world = int(os.environ.get("WORLD_SIZE", "1")) if world is None else int(world)
        if self.world > 1:
            uid = engine.comm_unique_id() if self.rank == 0 else None
            uid = (exchange or self._file_exchange)(uid)
            engine.comm_init(self.world, self.rank, uid)

    def _file_exchange(self, uid):
        # one file per launch: under torchrun every rank has the launcher as its parent, so its pid
        # separates two launches that reuse a port within minutes (a stale id of the previous launch
        # made the second of two back-to-back runs fail); rank 0 removes the file in close()
        tag = "%s_%s" % (os.environ.get("MASTER_PORT", "0"), os.environ.get("TORCHELASTIC_RUN_ID", "run"))
        if "TORCHELASTIC_RUN_ID" in os.environ:
            tag += "_%d" % os.getppid()
        path = os.path.join(os.environ.get("CWTB_COMM_DIR", "/tmp"), "cwtb_comm_%s.id" % tag)
        self._id_path = path
        if self.rank == 0:
            tmp = path + ".tmp%d" % os.getpid()
            with open(tmp, "wb") as f:
                f.write(uid)
            os.replace(tmp, path)
            return uid
        t0 = time.time()
        while True:
            try:
                with open(path, "rb") as f:
                    data = f.read()
                if len(data) == 128 and time.time() - os.path.getmtime(path) < 600:
                    return data
            except OSError:
                pass
            if time.time() - t0 > 120:
                raise RuntimeError("NCCL id of rank 0 did not appear at %s" % path)
            time.sleep(0.01)

    def _allgather_equal(self, buf):
        return self.engine.comm_allgather(buf)

    def allreduce_sum(self, array):
        array = np.ascontiguousarray(array)
        if self.world == 1:
            return array
        return self.engine.comm_allreduce_sum(array).reshape(array.shape)

    def max(self, value):
        if self.world == 1:
            return float(value)
        return float(self.engine.comm_allreduce_max([float(value)])[0])

    def close(self):
        if self.world > 1:
            self.engine.comm_destroy()
            if self.rank == 0 and getattr(self, "_id_path", None):
                try:
                    os.remove(self._id_path)
                except OSError:
                    pass


class TorchComm(_CommBase):
    """torch.distributed process group (gloo on CPU, nccl on GPUs)."""

    def __init__(self, dist, device=None):
        self.dist = dist
        self.device = device
        self.rank = dist.get_rank()
        self.world = dist.get_world_size()

    def _tensor(self, array):
        import torch
        t = torch.from_numpy(np.ascontiguousarray(array).copy())
        return t.to(self.device) if self.device is not None else t

    def _allgather_equal(self, buf):
        import torch
        t = self._tensor(buf)
        outs = [torch.empty_like(t) for _ in range(self.world)]
        self.dist.all_gather(outs, t)
        return [o.cpu().numpy() for o in outs]

    def allreduce_sum(self, array):
        if self.world == 1:
            return np.ascontiguousarray(array)
        t = self._tensor(array)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM)
        return t.cpu().numpy()

    def max(self, value):
        if self.world == 1:
            return float(value)
        t = self._tensor(np.array([float(value)]))
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return float(t.cpu().numpy()[0])

    def close(self):
        pass


def _as_comm(comm):
    """Accept a communicator, a torch.distributed module (legacy callers) or None."""
    if comm is None or isinstance(comm, _CommBase):
        return comm
    return TorchComm(comm)


def _rank_world(comm):
    return (0, 1) if comm is None else (comm.rank, comm.world)


# ---- sharded operations --------------------------------------------------------------------
def gather_rows(local, n_total, comm=None, device=None):
    comm = _as_comm(comm)
    if comm is None:
        return np.ascontiguousarray(local)
    if device is not None and isinstance(comm, TorchComm):
        comm.device = device
    return comm.allgather_rows(local, n_total)


def max_over_ranks(value, comm=None, device=None):
    """Maximum of a python float over all ranks (timings are max-over-ranks)."""
    comm = _as_comm(comm)
    if comm is None:
        return float(value)
    if device is not None and isinstance(comm, TorchComm):
        comm.device = device
    return comm.max(value)


def sum_over_ranks(array, comm=None, device=None):
    """Element-wise sum of an integer array over all ranks (every rank gets the total)."""
    comm = _as_comm(comm)
    if comm is None:
        return np.ascontiguousarray(array)
    if device is not None and isinstance(comm, TorchComm):
        comm.device = device
    return comm.allreduce_sum(array)


def cwt_batch_sharded(X, dt, scales, family, param, precision, engine, comm=None, device=None):
    """Global wavelet spectra of every channel of X[channels, n0], computed by the rank that
    owns the channel and gathered on all ranks.  X may be the full array (each rank slices
    its block) -- only the [channels, scales] result crosses the interconnect."""
    comm = _as_comm(comm)
    rank, world = _rank_world(comm)
    lo, hi = shard_range(X.shape[0], rank, world)
    power, _ = engine.cwt_batch(X[lo:hi], dt, scales, family, param, precision, want_power=True)
    return gather_rows(power, X.shape[0], comm, device)


def surrogate_pair(seed, index, N, *als):
    """Surrogate unit number `index` of a sharded Monte-Carlo run, one series per coefficient in
    `als` (a pair for the coherence, a triple for the partial / multiple coherence): white noise
    like the reference's `rednoise` output (helpers.py:146-173 filters a length-1 axis, SURVEY 8a
    row 10), from an RNG stream keyed by (seed, index) so that the unit does not depend on which
    rank draws it."""
    rs = np.random.RandomState([int(seed) & 0x7fffffff, int(index)])

    def white(al):
        tau = 0 if al == 0 else int(np.ceil(-2 / np.log(np.abs(al))))
        return rs.randn(N + tau)[tau:]
    return tuple(white(al) for al in als)


def wct_significance_sharded(al1, al2, dt, dj, s0, J, significance_level=0.95, wavelet='morlet',
                             mc_count=300, seed=0, engine=None, comm=None, device=None, device_rng=False,
                             precision='fp64'):
    """Monte-Carlo coherence significance (reference wavelet.py:531-647) with the surrogate
    pairs block-partitioned over the ranks (SURVEY 8e): every rank accumulates the [S, 1000]
    int64 histograms of its pairs on its GPU, ONE all-reduce (sum, ~1 MB) combines them and
    every rank evaluates the percentiles.  The result is independent of the world size.
    `precision`: 'fp64' (default) or 'fp32', as in wavelet.wct_significance."""
    from . import wavelet as wv
    prec = wv._coherence_precision(precision)
    comm = _as_comm(comm)
    mother = wv._check_parameter_wavelet(wavelet)
    rank, world = _rank_world(comm)
    prob = wv._mc_problem(dt, dj, s0, J, mother)
    lo, hi = shard_range(mc_count, rank, world)
    if device_rng:
        # surrogates drawn on each rank's GPU from the Philox stream keyed by (seed, pair number)
        hist = wv._mc_histogram_seeded(prob, dt, dj, mother, seed, lo, hi - lo, engine=engine,
                                       precision=prec)
    else:
        hist = wv._mc_histogram(prob, dt, dj, mother,
                                lambda i: surrogate_pair(seed, i, prob['N'], al1, al2),
                                range(lo, hi), progress=False, engine=engine, precision=prec)
    hist = sum_over_ranks(hist, comm, device)
    return wv._mc_levels(prob, hist, significance_level)


def wct3_significance_sharded(al_y, al1, al2, dt, dj, s0, J, significance_level=0.95, wavelet='morlet',
                              mc_count=300, seed=0, engine=None, comm=None, device=None, device_rng=False,
                              precision='fp64'):
    """`wavelet.wct3_significance` with the surrogate triples block-partitioned over the ranks:
    every rank accumulates the histograms of the partial and of the multiple coherence of its
    triples, ONE all-reduce of both ([2, S, 1000] int64) combines them and every rank evaluates
    the levels.  The result is independent of the world size.  Host RNG (`device_rng=False`):
    triple i is `surrogate_pair(seed, i, N, al_y, al1, al2)`; device RNG: the Philox triples of
    (seed, i).  Returns (sig_partial, sig_multiple)."""
    from . import wavelet as wv
    mother, prec = wv._wct3_mc_setup(wavelet, dj, precision)
    comm = _as_comm(comm)
    rank, world = _rank_world(comm)
    prob = wv._mc_problem(dt, dj, s0, J, mother)
    lo, hi = shard_range(mc_count, rank, world)
    if device_rng:
        hist = wv._mc_histogram_seeded(prob, dt, dj, mother, seed, lo, hi - lo, engine=engine,
                                       precision=prec, nser=3)
    else:
        hist = wv._mc_histogram(prob, dt, dj, mother,
                                lambda i: surrogate_pair(seed, i, prob['N'], al_y, al1, al2),
                                range(lo, hi), progress=False, engine=engine, precision=prec, nser=3)
    hist = sum_over_ranks(hist, comm, device)
    return (wv._mc_levels(prob, hist[0], significance_level),
            wv._mc_levels(prob, hist[1], significance_level))


def _surrogate_significance_sharded(series, groups, dt, dj, s0, J, significance_level, wavelet, normalize,
                                    mc_count, seed, engine, comm, device, precision):
    from . import wavelet as wv
    p, prob = wv._surrogate_problem(series, dt, dj, s0, J, wavelet, normalize, precision)
    comm = _as_comm(comm)
    rank, world = _rank_world(comm)
    lo, hi = shard_range(mc_count, rank, world)
    hist = wv._surrogate_histogram(p, prob, groups, seed, lo, hi - lo, engine=engine)
    hist = sum_over_ranks(hist, comm, device)
    return [wv._mc_levels(prob, h, significance_level) for h in hist]


def wct_surrogate_significance_sharded(y1, y2, dt, dj=1/12, s0=-1, J=-1, significance_level=0.95,
                                       wavelet='morlet', normalize=True, mc_count=300, seed=0, engine=None,
                                       comm=None, device=None, precision='fp64'):
    """`wavelet.wct_surrogate_significance` with the phase-randomised surrogate pairs
    block-partitioned over the ranks: every rank holds the data, draws pairs (seed, i) of its block
    on its GPU and accumulates their histogram, ONE all-reduce combines them and every rank
    evaluates the levels.  The result is independent of the world size."""
    return _surrogate_significance_sharded((y1, y2), (0, 1), dt, dj, s0, J, significance_level, wavelet,
                                           normalize, mc_count, seed, engine, comm, device, precision)[0]


def wct3_surrogate_significance_sharded(y, x1, x2, dt, dj=1/12, s0=-1, J=-1, significance_level=0.95,
                                        wavelet='morlet', normalize=True, mc_count=300, seed=0, engine=None,
                                        comm=None, device=None, precision='fp64', conditional=True):
    """`wavelet.wct3_surrogate_significance` with the surrogate triples block-partitioned over the
    ranks, as `wct_surrogate_significance_sharded`; one all-reduce of both histograms.  Returns
    (sig_partial, sig_multiple), independent of the world size."""
    return tuple(_surrogate_significance_sharded((y, x1, x2), (0, 1, 1) if conditional else (0, 1, 2), dt, dj,
                                                 s0, J, significance_level, wavelet, normalize, mc_count,
                                                 seed, engine, comm, device, precision))


def scale_rows(n_scales, rank, world, layout='cyclic'):
    """Scales owned by `rank`: 'cyclic' (j = rank, rank + world, ...) balances the cost -- the small
    scales (wide bands, two-kernel transforms) cost 4x the large ones, a contiguous block would give
    them all to rank 0; 'block' = contiguous shard_range."""
    if layout == 'block':
        lo, hi = shard_range(n_scales, rank, world)
        return np.arange(lo, hi)
    return np.arange(rank, n_scales, world)


def cwt_scale_sharded(signal, dt, scales, family, param, precision, engine, comm=None, device=None,
                      fetch=False, layout='cyclic'):
    """One long signal, scales partitioned over the ranks (SURVEY 8e row 2).  Every rank
    holds the signal and runs its own forward transform (cheaper than broadcasting the 16 MiB
    spectrum), then transforms only its scales (`scale_rows`), which stay
    resident in that GPU's HBM.  No collective on the data path; the per-scale global power
    (mean_n |W|^2, [S]) is all-gathered so that every rank sees the whole spectrum.

    Returns (rows, global_power[S], W_rows or None): `rows` are the indices of this rank's scales."""
    comm = _as_comm(comm)
    rank, world = _rank_world(comm)
    scales = np.ascontiguousarray(scales, dtype=np.float64)
    rows = scale_rows(scales.size, rank, world, layout)
    W = None
    if rows.size:
        W = engine.cwt(signal, dt, scales[rows], family, param, precision, fetch=fetch)
        local = engine.global_power(rows.size)
    else:
        local = np.zeros(0)
    # equal-length contributions: pad to the largest share, then scatter to the global order
    per = -(-scales.size // world)
    buf = np.full(per, np.nan)
    buf[:rows.size] = local
    if comm is None or world == 1:
        stack = [buf]
    else:
        stack = comm._allgather_equal(buf)
    power = np.empty(scales.size)
    for r in range(world):
        rr = scale_rows(scales.size, r, world, layout)
        power[rr] = np.asarray(stack[r])[:rr.size]
    return rows, power, W


def wct_halo(boxcar_len):
    """Scale rows below / above a block that its coherence needs: the scale boxcar of
    `Morlet.smooth` (reference mothers.py:96-102, convolve2d 'same' with zero fill) makes output row
    i depend on the time-smoothed rows q with i + (K-1)//2 - (K-1) <= q <= i + (K-1)//2."""
    K = int(boxcar_len)
    return K - 1 - (K - 1) // 2, (K - 1) // 2


def wct_scale_sharded(y1, y2, dt, dj=1 / 12, s0=-1, J=-1, wavelet='morlet', normalize=True,
                      engine=None, comm=None, device=None, precision='fp64'):
    """Deterministic part of the wavelet coherence (reference wavelet.py:422-516) with the SCALES
    block-partitioned over the ranks (SURVEY 8e row 4).  The transforms and the time smoothing are
    per scale; only the scale boxcar couples neighbouring rows, so every rank computes its block
    plus a halo of `wct_halo` rows on either side (redundant work of at most K-1 scales per rank
    instead of a halo exchange of S x n0 fields) and keeps the interior.  At the ends of the scale
    ladder the block ends where the reference's zero fill starts, so the result equals the
    single-GPU one row for row.  No collective on the data path: the coherence slabs stay with
    their rank; the per-scale mean coherence [S] is all-gathered.

    `precision`: 'fp64' (default) or 'fp32', as in wavelet.wct.

    Returns (lo, hi, WCT[lo:hi], aWCT[lo:hi], mean_wct[S], freq[S])."""
    from . import wavelet as wv
    from . import _engine
    prec = wv._coherence_precision(precision)
    comm = _as_comm(comm)
    rank, world = _rank_world(comm)
    mother = wv._check_parameter_wavelet(wavelet)
    if not hasattr(mother, 'smooth'):
        raise AttributeError("'{}' object has no attribute 'smooth'".format(type(mother).__name__))
    y1 = np.asarray(y1)
    y2 = np.asarray(y2)
    if s0 == -1:
        s0 = 2 * dt / mother.flambda()
    if J == -1:
        J = int(np.round(np.log2(y1.size * dt / s0) / dj))
    _, y1n, _ = wv._standardise(y1, normalize)
    _, y2n, _ = wv._standardise(y2, normalize)
    n0 = y1n.size
    sj, freq = wv._resolve_scales(n0, dt, dj, s0, J, mother, None)
    klen = wv._boxcar_len(mother, dj)
    if klen < 1:
        raise ValueError('smoothing window undefined for this wavelet (deltaj0 = -1)')
    S = sj.size
    lo, hi = shard_range(S, rank, world)
    below, above = wct_halo(klen)
    a, b = max(0, lo - below), min(S, hi + above)
    eng = engine or _engine.default_engine()
    if hi > lo:
        with eng.lock:
            if wv._sync_padding(eng, n0):
                prec = _engine.F64      # un-padded transforms run in fp64
            with wv._smoothing_filter(eng, mother, sj[a:b], dt, n0):
                WCT, aWCT = eng.wct(y1n, y2n, dt, dj, sj[a:b], *wv._family_of(mother), boxcar_len=klen,
                                    precision=prec)
        WCT, aWCT = WCT[lo - a:hi - a], aWCT[lo - a:hi - a]
        local = WCT.mean(axis=1)
    else:
        WCT = np.zeros((0, n0))
        aWCT = np.zeros((0, n0))
        local = np.zeros(0)
    mean = gather_rows(local, S, comm, device)
    return lo, hi, WCT, aWCT, mean, freq
