"""`partial_wct` + `multiple_wct` against `wct3_resident` and its device-side products at config 4's
triple (three 2^18-point series, s0 = 2, dj = 1/12, J = 144, boxcar K = 14), in fp64 and fp32.

Per precision three legs run alternately, `--reps` times:
  * two calls: `partial_wct` then `multiple_wct` (one pipeline each, 2 x 304 MB float64 fetched);
  * resident: `wct3_resident` alone (one pipeline, RP2, the partial phase and RM2 stay on the device);
  * resident + products: `wct3_resident`, then `global_coherence(inside_coi=True)`,
    `mean_phase(sig=...)`, `scale_avg` over one octave and `window` (every 3rd row and column).
For every leg the script records the end-to-end time of the Python calls and the device time of
the engine's kernels (last_kernel_ms of each pipeline call, summed), and reports their median and
min-max.  A separate pass records every kernel of each leg with cwtb_profile_begin / end (launches
serialised on one stream, bracketed by events), and the time of `Wct3FinalBody` with the phase
store (`wct3_resident`) and without it (`Engine.wct3`, both measures, the kernel `partial_wct`
runs).  The sig of mean_phase comes from an 8-triple seeded `wct3_significance` run.  The card's
name, power limit and maximum SM clock go into the output.  Needs a GPU: without one it fails.
The summary goes to stdout; `--out FILE` also writes the full record as JSON.

    python profiles/coherence3_resident.py --out /tmp/coherence3_resident.json
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import workloads  # noqa: E402
import pycwt_b200 as pycwt  # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from pycwt_b200.wavelet import _family_of, _wct_problem  # noqa: E402
from coherence_fp32 import card, stats  # noqa: E402

DT, DJ, S0, J = 1.0, 1 / 12, 2.0, 144


def config4_triple():
    """config 4's two series and a third chirp with another phase and noise of its own (the triple
    of tests/test_gpu_partial_coherence.py)."""
    y, x1 = workloads.config4_signals()
    n = y.size
    return y, x1, workloads.chirp(n, phase=2.1) + 0.5 * np.random.RandomState(2).randn(n)


def final_ms(rec):
    return sum(r["ms"] for r in rec if "Wct3FinalBody" in r["name"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("coherence3_resident: no CUDA device")
    eng = pycwt.default_engine()
    y, x1, x2 = config4_triple()
    kw = dict(dj=DJ, s0=S0, J=J)
    h = pycwt.wct3_resident(y, x1, x2, DT, **kw)
    sig_p, _ = h.significance(mc_count=8, seed=3, progress=False)
    per = h.period
    band = (per[48], per[60])        # one octave
    products = {
        "global_coherence": lambda h: h.global_coherence(inside_coi=True),
        "mean_phase": lambda h: h.mean_phase(sig=sig_p),
        "scale_avg": lambda h: h.scale_avg(*band),
        "window": lambda h: h.window(slice(None, None, 3), slice(None, None, 3)),
    }
    h.release()
    res = {"card": card(), "config": {"n": int(y.size), "scales": J + 1, "boxcar": 14,
                                      "slot_bytes": int(3 * (J + 1) * y.size * 8)},
           "timing": {}, "device_profile": {}, "final_kernel": {}}
    for p in ("fp64", "fp32"):
        def two_calls():
            a = pycwt.partial_wct(y, x1, x2, DT, precision=p, **kw)
            d = eng.last_kernel_ms()
            b = pycwt.multiple_wct(y, x1, x2, DT, precision=p, **kw)
            return (a, b), d + eng.last_kernel_ms()

        def resident():
            h = pycwt.wct3_resident(y, x1, x2, DT, precision=p, **kw)
            return h, eng.last_kernel_ms()

        def resident_products():
            h, d = resident()
            for f in products.values():
                f(h)
            return h, d

        legs = {"two_calls": two_calls, "resident": resident, "resident_products": resident_products}
        for f in legs.values():      # warm-up: module load, plans, buffers
            f()
        t = {k + s: [] for k in legs for s in ("_call_ms", "_device_ms")}
        for _ in range(args.reps):
            for k, f in legs.items():
                t0 = time.perf_counter()
                out, d = f()
                t[k + "_call_ms"].append((time.perf_counter() - t0) * 1e3)
                t[k + "_device_ms"].append(d)
                del out
        res["timing"][p] = {k: stats(v) for k, v in t.items()}
        print(p, json.dumps({k: round(v["median"], 3) for k, v in res["timing"][p].items()}), flush=True)

        # every kernel of each leg, launches serialised and bracketed by events (separate pass)
        res["device_profile"][p] = {}
        for k, f in legs.items():
            eng.profile_begin()
            out = f()
            rec = eng.profile_end()
            del out
            res["device_profile"][p][k] = {"device_ms": sum(r["ms"] for r in rec), "launches": len(rec),
                                           "Wct3FinalBody_ms": final_ms(rec)}
        print(p, "profiled device ms", json.dumps({k: round(v["device_ms"], 3)
                                                   for k, v in res["device_profile"][p].items()}), flush=True)

        # Wct3FinalBody with the phase store (wct3_resident) and without it (both measures, no phase)
        prob = _wct_problem((y, x1, x2), DT, DJ, S0, J, "morlet", True, p)
        fam = _family_of(prob.wavelet)
        with_ph, without = [], []
        for _ in range(args.reps):
            eng.profile_begin()
            eng.wct3_resident(*prob.yns, DT, DJ, prob.sj, *fam, prob.klen, precision=prob.prec)
            with_ph.append(final_ms(eng.profile_end()))
            eng.profile_begin()
            out = eng.wct3(*prob.yns, DT, DJ, prob.sj, *fam, prob.klen, precision=prob.prec)
            without.append(final_ms(eng.profile_end()))
            del out
        eng.coherence3_release()
        res["final_kernel"][p] = {"with_phase_ms": stats(with_ph), "without_phase_ms": stats(without)}
        print(p, "Wct3FinalBody ms with / without the phase store: %.4f / %.4f"
              % (np.median(with_ph), np.median(without)), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
