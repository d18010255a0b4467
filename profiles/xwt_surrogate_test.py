"""Cost of the cross-wavelet tests (`xwt_resident` -> `surrogate_test`, `cluster_test`) per surrogate
pair: config 4's pair (n0 = 2^18, s0 = 2, dj = 1/12, J = 144: 145 scales) in fp64 and fp32, both
nulls.

Per case, `--reps` times, one `surrogate_test(mc_count=--units)` and one `cluster_test` at
`h.signif`, every launch between an event pair (cwtb_profile_begin / end, launches serialised on
one stream).  Reported per pair: the device time of the generation (kernels tagged "ar1:" or
"phase:"), of the two transforms (the untagged kernels but the comparison and the labelling), of
the comparison kernel (`PowerCountBody`) and of the labelling (`Cluster*Body`), median and min-max
of the reps; and the comparison's bytes over its time against 3.35 TB/s (the counting pass reads
the pair's W12 and the resident W12 and reads and writes the uint32 counters: 2 x 16 + 8 B per
scale-point in fp64, 2 x 8 + 8 in fp32).  The card's name, power limit and maximum SM clock go into
the output.  Needs a GPU: without one it fails.

    python profiles/xwt_surrogate_test.py --out /tmp/xwt_surrogate_test.json
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import pycwt_b200 as pycwt  # noqa: E402
import workloads  # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from coherence_fp32 import card, stats  # noqa: E402
from power_surrogate_test import HBM, split  # noqa: E402
from surrogate_pvalues import profiled  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--units", type=int, default=16)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("xwt_surrogate_test: no CUDA device")
    c = workloads.C4
    y = workloads.config4_signals()
    record = {"card": card(), "units": args.units, "reps": args.reps, "cases": []}
    print("card:", record["card"])
    eng = pycwt.default_engine()
    for prec in ("fp64", "fp32"):
        h = pycwt.xwt_resident(y[0], y[1], c["dt"], dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=pycwt.Morlet(c["f0"]),
                               precision=prec)
        S, n0 = h.shape
        for null in ("ar1", "phase"):
            h.surrogate_test(mc_count=2, seed=1, null=null)     # warm-up: plans, buffers, module loads
            h.cluster_test(h.signif, mc_count=2, seed=1, null=null)
            legs = {"test": [], "cluster": []}
            for r in range(args.reps):
                _, rec = profiled(eng, lambda: h.surrogate_test(mc_count=args.units, seed=10 + r, null=null))
                legs["test"].append(split(rec, args.units))
                _, rec = profiled(eng, lambda: h.cluster_test(h.signif, mc_count=args.units, seed=10 + r, null=null))
                legs["cluster"].append(split(rec, args.units))
            esz = 16 if prec == "fp64" else 8
            count_bytes = S * n0 * (2 * esz + 8)
            out = {"case": "config4", "precision": prec, "null": null, "shape": [S, n0]}
            for leg, v in legs.items():
                out[leg] = {k: stats([x[k] for x in v]) for k in v[0]}
            tc = out["test"]["count"]["median"] * 1e-3
            out["count_bytes"] = count_bytes
            out["count_rate_TBps"] = count_bytes / tc / 1e12 if tc > 0 else None
            out["count_share_of_3.35TBps"] = count_bytes / tc / HBM if tc > 0 else None
            record["cases"].append(out)
            t = out["test"]
            print("config4 %s %-5s  ms/pair: generation %.3f  transforms %.3f  count %.3f (%.2f TB/s, %.0f %% of "
                  "3.35)  | cluster test: count+select %.3f  label %.3f"
                  % (prec, null, t["generation"]["median"], t["transform"]["median"], t["count"]["median"],
                     out["count_rate_TBps"] or 0, 100 * (out["count_share_of_3.35TBps"] or 0),
                     out["cluster"]["count"]["median"], out["cluster"]["label"]["median"]))
        h.release()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(record, f, indent=1)


if __name__ == "__main__":
    main()
