"""Host-side mirror (pycwt_b200/{helpers,mothers,wavelet.significance}) and the CPU oracle against
the reference's own results on randomised inputs.  The inputs are drawn here from fixed seeds; what
the unmodified reference returned for them is stored in tests/golden/host_reference.npz (written by
tests/golden/make_host_reference.py, which draws the same inputs through the generators below).
Results of length n are stored as per-row digests (`digest`), and a few of them also as exact samples."""
import builtins
import warnings

import numpy as np
import pytest

from conftest import load_golden

SUB = 8           # exact samples kept of the 1-D results compared element by element
REDNOISE_STRIDE = 64


class Packed(object):
    """The arrays of a fixture packed by `pack`, by name; `files` lists the names."""

    def __init__(self, z):
        self.arrays = {}
        for k, v in zip(z["str_keys"], z["str_vals"]):
            self.arrays[str(k)] = np.asarray(str(v))
        keys = str(z["keys"]).split("\n")
        for k, pool, start, nd, d0, d1 in zip(keys, z["pool"], z["start"], z["ndim"], z["d0"], z["d1"]):
            shape = (int(d0), int(d1))[:nd]
            a = z[("real", "cplx")[int(pool)]][start:start + int(np.prod(shape, dtype=np.int64))]
            self.arrays[str(k)] = a.reshape(shape)
        self.files = list(self.arrays)

    def __getitem__(self, key):
        return self.arrays[key]


def pack(out):
    """Many small arrays as a few flat ones (one zip member per array would cost more than the data):
    float64 and complex128 pools, strings apart, and per name its pool, offset and shape."""
    pools = {"real": [], "cplx": []}
    size = {"real": 0, "cplx": 0}
    meta = {"keys": [], "pool": [], "start": [], "ndim": [], "d0": [], "d1": []}
    skeys, svals = [], []
    for k in sorted(out):
        a = np.asarray(out[k])
        if a.dtype.kind == "U":
            skeys.append(k)
            svals.append(str(a))
            continue
        assert a.ndim <= 2, k
        pool = "cplx" if a.dtype.kind == "c" else "real"
        flat = a.astype(np.complex128 if pool == "cplx" else np.float64).ravel()
        shape = a.shape + (0, 0)
        for f, v in zip(("keys", "pool", "start", "ndim", "d0", "d1"), (k, pool, size[pool], a.ndim) + shape[:2]):
            meta[f].append(v)
        pools[pool].append(flat)
        size[pool] += flat.size
    arrays = {p: (np.concatenate(v) if v else np.zeros(0)) for p, v in pools.items()}
    arrays.update({f: np.asarray(v, dtype=np.int32) for f, v in meta.items() if f not in ("keys", "pool")})
    arrays.update(keys=np.asarray("\n".join(meta["keys"])), pool=np.asarray(meta["pool"]) == "cplx")
    arrays.update(str_keys=np.asarray(skeys), str_vals=np.asarray(svals))
    return arrays


@pytest.fixture(scope="module")
def ref():
    return Packed(load_golden("host_reference"))


def same(a, b, tol=0.0):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if tol == 0:
        return np.array_equal(a, b, equal_nan=True)
    return np.allclose(a, b, rtol=tol, atol=0, equal_nan=True)


def col_stride(n):
    return max(1, n // SUB)


def digest(a):
    """Per-row fingerprint of an array whose rows have length n: the projection of each row on a
    fixed, seeded random vector, and the row's L1 norm.  Two arrays that agree element by element to a
    relative `tol` have projections and L1 norms within `tol * L1` of each other.  A difference
    spread over a row is caught at that level, one in a single element of a row of n once it exceeds
    about `tol * n` of that element."""
    a = np.asarray(a)
    v = np.random.RandomState(a.shape[-1]).uniform(-1, 1, a.shape[-1])
    return a @ v, np.abs(a).sum(axis=-1)


def matches(ref, key, a, tol):
    """`a` agrees with the reference result stored under `key` (see `digest`) to a relative `tol`;
    tol is at least 1e-12, above the rounding of the projection itself (n eps L1, n <= 2^11)."""
    p, l1 = digest(a)
    rp, rl = ref[key + "_proj"], ref[key + "_l1"]
    if np.shape(p) != rp.shape:
        return False
    bad = ~np.isfinite(rp)
    if not np.array_equal(bad, ~np.isfinite(p)):
        return False
    ok = ~bad & np.isfinite(rl)
    return bool(np.all(np.abs(p - rp)[~bad] <= tol * rl[~bad]) and np.all(np.abs(l1 - rl)[ok] <= tol * rl[ok]))


def check_raises(name, fn):
    """fn raises what the reference raised (recorded by class name): that class or one derived from it."""
    cls = getattr(builtins, name, Exception)
    with pytest.raises(cls) as ei:
        fn()
    assert name in [k.__name__ for k in type(ei.value).__mro__], (name, type(ei.value))


# ---- input generators, shared with tests/golden/make_host_reference.py ------------------------
MOTHER_FREQS = np.r_[np.linspace(-30, 30, 241), [0.0, 1e-3, 800.0, -800.0]]
MOTHER_CASES = (("Morlet", [6, 4.5, 8, 12, 20]), ("Paul", [4, 1, 2, 6, 10]), ("DOG", [2, 1, 3, 6, 9]))
MOTHER_ATTRS = ("name", "dofmin", "cdelta", "gamma", "deltaj0")


def helper_cases():
    rs = np.random.RandomState(3)
    for it in range(120):
        n = int(rs.randint(8, 3000))
        x = np.cumsum(rs.randn(n)) * rs.uniform(0.1, 10) if rs.rand() < 0.5 else rs.randn(n)
        fr, al = rs.uniform(0, 0.5, size=rs.randint(1, 50)), rs.uniform(-0.95, 0.95)
        k = int(rs.randint(1, 40))
        seed, g = int(rs.randint(1e6)), float(rs.uniform(0.01, 0.95) * rs.choice([-1, 1]))
        c = rs.rand(30) > 0.5
        yield dict(it=it, n=n, x=x, fr=fr, al=al, k=k, norm=bool(it % 2), seed=seed, g=g, c=c)


def significance_cases():
    rs = np.random.RandomState(4)
    for it in range(120):
        n, dt = int(rs.randint(32, 2000)), float(10 ** rs.uniform(-1, 1))
        x = rs.randn(n)
        fam = rs.randint(3)
        S = int(rs.randint(3, 40))
        sj = 2 * dt * 2 ** (np.arange(S) * 0.25)
        st = int(rs.randint(3))
        kw = dict(sigma_test=st, alpha=float(rs.uniform(0, 0.9)),
                  significance_level=float(rs.choice([0.9, 0.95, 0.99])))
        sig = x if rs.rand() < 0.5 else float(x.var())
        if st == 1:
            kw["dof"] = (n - sj).copy()
        if st == 2:
            kw["dof"] = [sj[1], sj[min(S - 1, 5)]]
        yield dict(it=it, fam=int(fam), sig=sig, dt=dt, sj=sj, kw=kw)


def significance_mother(module, fam):
    return [module.Morlet(6), module.Paul(4), module.DOG(2)][fam]


def oracle_cases():
    """Random cwt calls, then random xwt / wct calls (one random stream, as the test always drew)."""
    from scipy.signal import lfilter
    rs = np.random.RandomState(6)
    for it in range(60):
        n, dt = int(2 ** rs.uniform(2.2, 11)), float(10 ** rs.uniform(-1, 1))
        x = rs.randn(n)
        fam = rs.randint(3)
        order = [rs.choice([6, 8]), rs.choice([4, 2, 6]), rs.choice([2, 3, 6])][fam]
        dj = float(rs.choice([0.5, 0.25, 0.125]))
        yield dict(kind="cwt", it=it, x=x, dt=dt, fam=int(fam), order=order, dj=dj)
    for it in range(10):
        n, dt = int(2 ** rs.uniform(5, 9)), float(10 ** rs.uniform(-1, 1))
        y1 = lfilter([1], [1, -0.5], rs.randn(n))
        y2 = np.roll(y1, 2) + 0.7 * rs.randn(n)
        dj = float(rs.choice([0.5, 0.25, 1 / 6]))
        yield dict(kind="coherence", it=it, y1=y1, y2=y2, dt=dt, dj=dj)


def oracle_mother(module, fam, order):
    return [module.Morlet, module.Paul, module.DOG][fam](order)


# ---- the comparisons ---------------------------------------------------------------------------
def test_mother_wavelets_match(ref):
    from pycwt_b200 import mothers as om
    f = MOTHER_FREQS
    for cls, params in MOTHER_CASES:
        for p in params:
            b = getattr(om, cls)(p)
            key = "m_%s_%g_" % (cls, p)
            with np.errstate(all="ignore"):
                assert same(ref[key + "psi_ft"], b.psi_ft(f)), (cls, p)          # bit-identical
                r0 = ref[key + "psi0"]
                assert np.abs(r0 - b.psi(0)) <= 4e-16 * abs(r0), (cls, p)
            assert ref[key + "flambda"] == b.flambda() and ref[key + "coi"] == b.coi()
            for attr in MOTHER_ATTRS:
                assert ref[key + attr] == getattr(b, attr), (cls, p, attr)
    assert str(ref["mexicanhat_name"]) == om.MexicanHat().name


def test_helpers_match(ref):
    from pycwt_b200 import helpers as oh
    for case in helper_cases():
        it, n, x = case["it"], case["n"], case["x"]
        key = "h%d_" % it
        if key + "ar1_warning" in ref.files:
            with pytest.raises(Warning):
                oh.ar1(x)
        else:
            assert same(ref[key + "ar1"], oh.ar1(x), 1e-13), it
        assert same(ref[key + "ar1_spectrum"], oh.ar1_spectrum(case["fr"], case["al"]))
        assert same(ref[key + "rect"], oh.rect(case["k"], normalize=case["norm"]))
        np.random.seed(case["seed"])
        r = oh.rednoise(n, case["g"], 2.0)
        assert r.shape == (n,) and same(ref[key + "rednoise"], r[::REDNOISE_STRIDE])   # same draws
        assert matches(ref, key + "rednoise", r, 1e-12)
        assert same(ref[key + "find"], oh.find(case["c"]))
    assert oh.fft_kwargs(np.zeros(300)) == {"n": 512}


def test_significance_matches(ref):
    import pycwt_b200 as our
    from pycwt_b200 import mothers as om
    for case in significance_cases():
        key = "s%d_" % case["it"]
        kw = dict(case["kw"])
        call = lambda: our.significance(case["sig"], case["dt"], case["sj"].copy(),  # noqa: E731
                                        wavelet=significance_mother(om, case["fam"]), **kw)
        if key + "raises" in ref.files:
            check_raises(str(ref[key + "raises"]), call)
            continue
        o = call()
        assert same(ref[key + "signif"], o[0], 1e-13) and same(ref[key + "fft_theor"], o[1], 1e-13), case["it"]


def test_oracle_matches_reference_on_random_inputs(ref):
    """The oracle is pinned by the committed fixtures of the fixed cases too; here it is compared on
    random lengths, sampling steps, families, orders and call variants."""
    from oracle import cwt_oracle as orc
    warnings.filterwarnings("ignore")
    names = ("W", "sj", "freqs", "coi", "fft", "fftfreqs")
    for case in oracle_cases():
        it = case["it"]
        if case["kind"] == "cwt":
            key = "c%d_" % it
            mo = oracle_mother(orc, case["fam"], case["order"])
            with np.errstate(all="ignore"):
                if key + "raises" in ref.files:
                    check_raises(str(ref[key + "raises"]), lambda: orc.cwt(case["x"], case["dt"], dj=case["dj"], wavelet=mo))
                    continue
                o = orc.cwt(case["x"], case["dt"], dj=case["dj"], wavelet=mo)
            assert tuple(ref[key + "W_shape"]) == o[0].shape, it
            for nm, b in zip(names, o):
                if nm in ("sj", "freqs"):
                    assert same(ref[key + nm], b, 1e-12), (it, nm)
                else:
                    assert matches(ref, key + nm, b, 1e-12), (it, nm)
            if key + "iW_proj" in ref.files:
                iw = orc.icwt(o[0], o[1], case["dt"], case["dj"], mo)
                assert matches(ref, key + "iW", iw, 1e-12), it
        else:
            key = "x%d_" % it
            m_o = orc.Morlet(6)
            y1, y2, dt, dj = case["y1"], case["y2"], case["dt"], case["dj"]
            st = col_stride(y1.size)
            b = orc.xwt(y1, y2, dt, dj=dj, wavelet=m_o)
            assert matches(ref, key + "W12", b[0], 1e-11), it
            assert same(ref[key + "coi"], b[1][::st], 1e-11) and matches(ref, key + "coi", b[1], 1e-11), it
            assert same(ref[key + "freq"], b[2], 1e-11) and same(ref[key + "signif"], b[3], 1e-11), it
            b = orc.wct(y1, y2, dt, dj=dj, sig=False, wavelet=m_o)
            assert matches(ref, key + "WCT", b[0], 1e-10), it
            assert matches(ref, key + "angle", np.exp(1j * b[1]), 1e-9), it     # on the unit circle
            assert same(ref[key + "wct_coi"], b[2][::st], 1e-14) and matches(ref, key + "wct_coi", b[2], 1e-12)
            assert same(ref[key + "wct_freq"], b[3])
