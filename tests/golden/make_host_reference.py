#!/usr/bin/env python
"""Write tests/golden/host_reference.npz: what the UNMODIFIED reference package (regeirk/pycwt)
returns on the randomised inputs of tests/test_host_vs_reference.py.

    python tests/golden/make_host_reference.py <checkout of the reference>

The inputs come from the test module's own generators, so the fixture and the test draw the same
numbers; only the reference's results are stored (results of length n as the test's `digest`).
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))        # tests/: the test module and its conftest
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import test_host_vs_reference as T  # noqa: E402


def put(out, key, a):
    out[key + "_proj"], out[key + "_l1"] = (np.asarray(d) for d in T.digest(a))


def main(ref_root):
    sys.path.insert(0, ref_root)
    warnings.filterwarnings("ignore")
    import pycwt as rp  # noqa: E402  (the reference)
    from pycwt import helpers as rh, mothers as rm  # noqa: E402
    out = {}

    for cls, params in T.MOTHER_CASES:
        for p in params:
            a = getattr(rm, cls)(p)
            key = "m_%s_%g_" % (cls, p)
            with np.errstate(all="ignore"):
                out[key + "psi_ft"] = a.psi_ft(T.MOTHER_FREQS)
                out[key + "psi0"] = np.asarray(a.psi(0))
            out[key + "flambda"] = np.asarray(a.flambda())
            out[key + "coi"] = np.asarray(a.coi())
            for attr in T.MOTHER_ATTRS:
                out[key + attr] = np.asarray(getattr(a, attr))
    out["mexicanhat_name"] = np.asarray(rm.MexicanHat().name)

    for case in T.helper_cases():
        key = "h%d_" % case["it"]
        try:
            out[key + "ar1"] = np.asarray(rh.ar1(case["x"]))
        except Warning:
            out[key + "ar1_warning"] = np.asarray(True)
        out[key + "ar1_spectrum"] = np.asarray(rh.ar1_spectrum(case["fr"], case["al"]))
        out[key + "rect"] = np.asarray(rh.rect(case["k"], normalize=case["norm"]))
        np.random.seed(case["seed"])
        rn = np.asarray(rh.rednoise(case["n"], case["g"], 2.0))
        out[key + "rednoise"] = rn[::T.REDNOISE_STRIDE]
        put(out, key + "rednoise", rn)
        out[key + "find"] = np.asarray(rh.find(case["c"]))

    for case in T.significance_cases():
        key = "s%d_" % case["it"]
        try:
            r = rp.significance(case["sig"], case["dt"], case["sj"].copy(),
                                wavelet=T.significance_mother(rm, case["fam"]), **dict(case["kw"]))
        except Exception as e:
            out[key + "raises"] = np.asarray(type(e).__name__)
            continue
        out[key + "signif"], out[key + "fft_theor"] = np.asarray(r[0]), np.asarray(r[1])

    names = ("W", "sj", "freqs", "coi", "fft", "fftfreqs")
    for case in T.oracle_cases():
        if case["kind"] == "cwt":
            key = "c%d_" % case["it"]
            mr = T.oracle_mother(rm, case["fam"], case["order"])
            with np.errstate(all="ignore"):
                try:
                    r = rp.cwt(case["x"], case["dt"], dj=case["dj"], wavelet=mr)
                except Exception as e:
                    out[key + "raises"] = np.asarray(type(e).__name__)
                    continue
                out[key + "W_shape"] = np.asarray(r[0].shape)
                for nm, a in zip(names, r):
                    if nm in ("sj", "freqs"):
                        out[key + nm] = np.asarray(a)
                    else:
                        put(out, key + nm, a)
                if mr.cdelta != -1 and r[0].size and np.isfinite(r[0]).all():
                    put(out, key + "iW", rp.icwt(r[0], r[1], case["dt"], case["dj"], mr))
        else:
            key = "x%d_" % case["it"]
            m_r = rm.Morlet(6)
            y1, y2, dt, dj = case["y1"], case["y2"], case["dt"], case["dj"]
            st = T.col_stride(y1.size)
            a = rp.xwt(y1, y2, dt, dj=dj, wavelet=m_r)
            put(out, key + "W12", a[0])
            out[key + "coi"], out[key + "freq"], out[key + "signif"] = a[1][::st], np.asarray(a[2]), np.asarray(a[3])
            put(out, key + "coi", a[1])
            a = rp.wct(y1, y2, dt, dj=dj, sig=False, wavelet=m_r)
            put(out, key + "WCT", a[0])
            put(out, key + "angle", np.exp(1j * a[1]))
            out[key + "wct_coi"], out[key + "wct_freq"] = a[2][::st], np.asarray(a[3])
            put(out, key + "wct_coi", a[2])

    path = os.path.join(HERE, "host_reference.npz")
    np.savez_compressed(path, **T.pack(out))
    print("%s: %d arrays, %.1f KB" % (path, len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
