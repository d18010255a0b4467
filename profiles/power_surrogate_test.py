"""Cost of the power tests (`power_resident` -> `surrogate_test`, `cluster_test`) per surrogate unit:
config 4's first series (n0 = 2^18, s0 = 2, dj = 1/12, J = 144: 145 scales) in fp64 and fp32, and
config 2's geometry (n0 = 2^20, 256 scales) in fp64, both nulls.

Per case, `--reps` times, one `surrogate_test(mc_count=--units)` and one `cluster_test` at the 95 %
chi-squared level of `significance()`, every launch between an event pair (cwtb_profile_begin /
end, launches serialised on one stream).  Reported per unit: the device time of the generation
(kernels tagged "ar1:" or "phase:"), of the transform (the untagged kernels but the comparison and
the labelling), of the comparison kernel (`PowerCountBody`) and of the labelling (`Cluster*Body`),
median and min-max of the reps; and the comparison's bytes over its time against 3.35 TB/s (the
counting pass reads the unit's W and the resident W and reads and writes the uint32 counters: 2 x 16
+ 8 B per scale-point in fp64, 2 x 8 + 8 in fp32).  The card's name, power limit and maximum SM
clock go into the output.  Needs a GPU: without one it fails.

    python profiles/power_surrogate_test.py --out /tmp/power_surrogate_test.json
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
from surrogate_pvalues import profiled  # noqa: E402

HBM = 3.35e12


def split(rec, units):
    """ms per unit of the generation, transform, comparison and labelling kernels."""
    out = {"generation": 0.0, "transform": 0.0, "count": 0.0, "label": 0.0}
    for r in rec:
        n = r["name"]
        if n.startswith("ar1:") or n.startswith("phase:"):
            out["generation"] += r["ms"]
        elif "PowerCountBody" in n:
            out["count"] += r["ms"]
        elif "Cluster" in n:
            out["label"] += r["ms"]
        else:
            out["transform"] += r["ms"]
    return {k: v / units for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--units", type=int, default=16)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("power_surrogate_test: no CUDA device")
    c4, c2 = workloads.C4, workloads.C2
    cases = [("config4", workloads.config4_signals()[0], c4, "fp64"),
             ("config4", workloads.config4_signals()[0], c4, "fp32"),
             ("config2", workloads.config2_signal(), c2, "fp64")]
    record = {"card": card(), "units": args.units, "reps": args.reps, "cases": []}
    print("card:", record["card"])
    eng = pycwt.default_engine()
    for name, y, c, prec in cases:
        h = pycwt.power_resident(y, c["dt"], dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=pycwt.Morlet(c["f0"]),
                                 precision=prec)
        S, n0 = h.shape
        sig = pycwt.significance(1.0, h.dt, h.scales, 0, pycwt.ar1(y)[0])[0]
        for null in ("ar1", "phase"):
            h.surrogate_test(mc_count=2, seed=1, null=null)     # warm-up: plans, buffers, module loads
            h.cluster_test(sig, mc_count=2, seed=1, null=null)
            legs = {"test": [], "cluster": []}
            for r in range(args.reps):
                _, rec = profiled(eng, lambda: h.surrogate_test(mc_count=args.units, seed=10 + r, null=null))
                legs["test"].append(split(rec, args.units))
                _, rec = profiled(eng, lambda: h.cluster_test(sig, mc_count=args.units, seed=10 + r, null=null))
                legs["cluster"].append(split(rec, args.units))
            esz = 16 if prec == "fp64" else 8
            count_bytes = S * n0 * (2 * esz + 8)
            out = {"case": name, "precision": prec, "null": null, "shape": [S, n0]}
            for leg, v in legs.items():
                out[leg] = {k: stats([x[k] for x in v]) for k in v[0]}
            tc = out["test"]["count"]["median"] * 1e-3
            out["count_bytes"] = count_bytes
            out["count_rate_TBps"] = count_bytes / tc / 1e12 if tc > 0 else None
            out["count_share_of_3.35TBps"] = count_bytes / tc / HBM if tc > 0 else None
            record["cases"].append(out)
            t = out["test"]
            print("%s %s %-5s  ms/unit: generation %.3f  transform %.3f  count %.3f (%.2f TB/s, %.0f %% of 3.35)"
                  "  | cluster test: count+select %.3f  label %.3f"
                  % (name, prec, null, t["generation"]["median"], t["transform"]["median"], t["count"]["median"],
                     out["count_rate_TBps"] or 0, 100 * (out["count_share_of_3.35TBps"] or 0),
                     out["cluster"]["count"]["median"], out["cluster"]["label"]["median"]))
        h.release()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(record, f, indent=1)


if __name__ == "__main__":
    main()
