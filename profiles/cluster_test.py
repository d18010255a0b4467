"""Cost of the cluster test at config 4's data sizes (n0 = 2^18, s0 = 2, dj = 1/12, J = 144: 145
scales, boxcar K = 14), pairs (`wct_resident`) and triples (`wct3_resident`, conditional null, the
partial coherence), fp64 and fp32.

Per case, `--reps` times and alternating, one `cluster_test(sig, mc_count=--units, seed)` and one
`surrogate_significance` with the same seed (histograms only), every launch between an event pair
(cwtb_profile_begin / end, launches serialised on one stream).  `sig` is the 95 % level of
`surrogate_significance` with another seed.  Reported per surrogate unit: the device time of all
kernels, of the final coherence kernel and of the labelling kernels (`Cluster*Body`), as the median
and min-max of the reps, and the wall time per unit of both calls.  The card's name, power limit and
maximum SM clock go into the output.  Needs a GPU: without one it fails.

    python profiles/cluster_test.py --out /tmp/cluster_test.json
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

import pycwt_b200 as pycwt  # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from coherence_fp32 import card, stats  # noqa: E402
from surrogate_pvalues import DT, DJ, S0, J, series, profiled  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--units", type=int, default=32)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("cluster_test: no CUDA device")
    eng = pycwt.default_engine()
    y, x1, x2 = series()
    kw = dict(dj=DJ, s0=S0, J=J)
    record = {"card": card(), "units": args.units, "reps": args.reps, "cases": []}
    print("card:", record["card"])
    for nser in (2, 3):
        for prec in ("fp64", "fp32"):
            h = (pycwt.wct_resident(y, x1, DT, precision=prec, **kw) if nser == 2
                 else pycwt.wct3_resident(y, x1, x2, DT, precision=prec, **kw))
            final = "WctFinalBody" if nser == 2 else "Wct3FinalBody"
            sig = h.surrogate_significance(mc_count=args.units, seed=1)
            sig = sig if nser == 2 else sig[0]
            h.cluster_test(sig, mc_count=2, seed=1)          # warm-up: plans, buffers, module loads
            legs = {"cluster": [], "significance": []}
            for r in range(args.reps):
                for leg in ("cluster", "significance"):
                    fn = ((lambda s: h.cluster_test(sig, mc_count=args.units, seed=s)) if leg == "cluster"
                          else (lambda s: h.surrogate_significance(mc_count=args.units, seed=s)))
                    t0 = time.perf_counter()
                    res, rec = profiled(eng, lambda: fn(100 + r))
                    wall = 1e3 * (time.perf_counter() - t0) / args.units
                    legs[leg].append({"total": sum(x["ms"] for x in rec) / args.units,
                                      "final": sum(x["ms"] for x in rec if final in x["name"]) / args.units,
                                      "label": sum(x["ms"] for x in rec if "Cluster" in x["name"]) / args.units,
                                      "wall": wall,
                                      "clusters": int(res.area.size) if leg == "cluster" else None})
            case = {"nser": nser, "precision": prec}
            for leg, v in legs.items():
                case[leg] = {k: stats([x[k] for x in v]) for k in ("total", "final", "label", "wall")}
            case["clusters"] = legs["cluster"][0]["clusters"]
            t, s = case["cluster"], case["significance"]
            case["added_unit_ms"] = t["total"]["median"] - s["total"]["median"]
            case["added_wall_ms"] = t["wall"]["median"] - s["wall"]["median"]
            record["cases"].append(case)
            print("%d series %s: device per unit %.3f ms (cluster test) vs %.3f ms (significance), +%.3f ms "
                  "(%.1f %%); labelling %.3f ms, final kernel %.3f vs %.3f ms; wall per unit %.3f vs %.3f ms; "
                  "%d observed clusters"
                  % (nser, prec, t["total"]["median"], s["total"]["median"], case["added_unit_ms"],
                     100 * case["added_unit_ms"] / s["total"]["median"], t["label"]["median"],
                     t["final"]["median"], s["final"]["median"], t["wall"]["median"], s["wall"]["median"],
                     case["clusters"]))
            h.release()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(record, f, indent=1)


if __name__ == "__main__":
    main()
