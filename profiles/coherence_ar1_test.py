"""Cost of the coherence tests against AR(1) surrogates (`surrogate_test(null='ar1')`) per unit, beside
the phase null: config 4's data sizes (n0 = 2^18, s0 = 2, dj = 1/12, J = 144: 145 scales), fp64 and
fp32, the pair (`wct_resident`) and the triple (`wct3_resident`, `conditional` True and False).

Per case, `--reps` times, one `surrogate_test(mc_count=--units)`, every launch between an event pair
(cwtb_profile_begin / end, launches serialised on one stream).  Reported per unit: the device time
of the generation (kernels tagged "ar1:" or "phase:") and of the coherence pipeline (every other
kernel: the transforms, smoothing, final kernel with its counting, and for the phase null the data's
spectra once per call), median and min-max of the reps.  The card's name, power limit and maximum SM
clock go into the output.  Needs a GPU: without one it fails.

    python profiles/coherence_ar1_test.py --out /tmp/coherence_ar1_test.json
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import pycwt_b200 as pycwt  # noqa: E402
import workloads  # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from coherence_fp32 import card, stats  # noqa: E402
from power_surrogate_test import split  # noqa: E402
from surrogate_pvalues import profiled  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--units", type=int, default=8)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("coherence_ar1_test: no CUDA device")
    c = workloads.C4
    y = list(workloads.config4_signals())
    x2 = np.random.RandomState(4).randn(y[0].size) + 0.3 * y[1]
    record = {"card": card(), "units": args.units, "reps": args.reps, "cases": []}
    print("card:", record["card"])
    eng = pycwt.default_engine()
    geo = dict(dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=pycwt.Morlet(c["f0"]))
    for prec in ("fp64", "fp32"):
        pair = pycwt.wct_resident(y[0], y[1], c["dt"], precision=prec, **geo)
        triple = pycwt.wct3_resident(y[0], y[1], x2, c["dt"], precision=prec, **geo)
        cases = [("pair", pair, {})] + [("triple" + ("" if cond else " unconditional"), triple,
                                        dict(conditional=cond)) for cond in (True, False)]
        for name, h, kw in cases:
            for null in ("ar1", "phase"):
                h.surrogate_test(mc_count=2, seed=1, null=null, **kw)     # warm-up: plans, buffers, modules
                legs = []
                for r in range(args.reps):
                    _, rec = profiled(eng, lambda: h.surrogate_test(mc_count=args.units, seed=10 + r, null=null, **kw))
                    legs.append(split(rec, args.units))
                out = {"case": name, "precision": prec, "null": null, "shape": list(h.shape),
                       "generation": stats([x["generation"] for x in legs]),
                       "pipeline": stats([x["transform"] + x["count"] for x in legs])}
                g, p = out["generation"]["median"], out["pipeline"]["median"]
                out["generation_share"] = g / (g + p)
                record["cases"].append(out)
                print("config4 %-20s %s %-5s  ms/unit: generation %.4f  pipeline %.3f  (generation %.2f %% of the unit)"
                      % (name, prec, null, g, p, 100 * out["generation_share"]))
        pair.release()
        triple.release()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(record, f, indent=1)


if __name__ == "__main__":
    main()
