"""Cost of the point-wise surrogate test at config 4's data sizes (n0 = 2^18, s0 = 2, dj = 1/12,
J = 144: 145 scales, boxcar K = 14), pairs (`wct_resident`) and triples (`wct3_resident`, conditional
null), fp64 and fp32.

Per case, `--reps` times and alternating, one `surrogate_test(mc_count=--units, seed)` (counts
every point) and one `surrogate_significance` with the same seed (histograms only), every launch
between an event pair (cwtb_profile_begin / end, launches serialised on one stream).  Reported per
surrogate unit: the device time of all kernels and of the final coherence kernel (`WctFinalBody` /
`Wct3FinalBody`) with and without counting, as the median and min-max of the reps; the levels of
the two calls are checked to be bit-identical.  Then the wall time of the reads of the counts:
`pvalues()` (the full map) and a window of every 8th row and column, `fdr_threshold` (the count
histogram plus the host step-up test) and `pvalue_fraction`.  The card's name, power limit and
maximum SM clock go into the output.  Needs a GPU: without one it fails.

    python profiles/surrogate_pvalues.py --out /tmp/surrogate_pvalues.json
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
from coherence_fp32 import card, stats  # noqa: E402

DT, DJ, S0, J = 1.0, 1 / 12, 2.0, 144


def series():
    y, x1 = workloads.config4_signals()
    n = y.size
    return y, x1, 0.6 * x1 + workloads.chirp(n, phase=2.1) + 0.5 * np.random.RandomState(2).randn(n)


def profiled(eng, call):
    eng.profile_begin()
    out = call()
    rec = eng.profile_end()
    return out, rec


def wall(call, reps=3):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        t.append(1e3 * (time.perf_counter() - t0))
    return stats(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--units", type=int, default=32)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("surrogate_pvalues: no CUDA device")
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
            h.surrogate_test(mc_count=2, seed=1)          # warm-up: plans, buffers, module loads
            h.surrogate_significance(mc_count=2, seed=1)
            legs = {"test": [], "significance": []}
            for r in range(args.reps):
                for leg in ("test", "significance"):
                    fn = h.surrogate_test if leg == "test" else h.surrogate_significance
                    lev, rec = profiled(eng, lambda: fn(mc_count=args.units, seed=100 + r))
                    legs[leg].append({"levels": lev, "total": sum(x["ms"] for x in rec) / args.units,
                                      "final": sum(x["ms"] for x in rec if final in x["name"]) / args.units})
            same = all(np.array_equal(np.asarray(a["levels"]), np.asarray(b["levels"]), equal_nan=True)
                       for a, b in zip(legs["test"], legs["significance"]))
            S, n0 = h.shape
            mkw = {} if nser == 2 else {"measure": "partial"}
            case = {"nser": nser, "precision": prec, "levels_bit_identical": bool(same)}
            for leg, v in legs.items():
                case[leg] = {"unit_ms": stats([x["total"] for x in v]), "final_ms": stats([x["final"] for x in v])}
            case["added_unit_ms"] = case["test"]["unit_ms"]["median"] - case["significance"]["unit_ms"]["median"]
            case["added_final_ms"] = case["test"]["final_ms"]["median"] - case["significance"]["final_ms"]["median"]
            case["reads_ms"] = {
                "pvalues_full": wall(lambda: h.pvalues(**mkw)),
                "pvalues_8th": wall(lambda: h.pvalues(slice(None, None, 8), slice(None, None, 8), **mkw)),
                "count_hist": wall(lambda: eng.count_hist(None if nser == 2 else 0, *h.coi_ranges(),
                                                          h.surrogate_units + 1)),
                "fdr_threshold": wall(lambda: h.fdr_threshold(0.05, **mkw)),
                "pvalue_fraction": wall(lambda: h.pvalue_fraction(0.05, **mkw)),
            }
            case["fdr"] = list(h.fdr_threshold(0.05, **mkw))
            record["cases"].append(case)
            print("%d series %s: unit %.3f ms (test) vs %.3f ms (significance), +%.3f ms; final kernel "
                  "%.3f vs %.3f ms (+%.3f); levels identical: %s"
                  % (nser, prec, case["test"]["unit_ms"]["median"], case["significance"]["unit_ms"]["median"],
                     case["added_unit_ms"], case["test"]["final_ms"]["median"],
                     case["significance"]["final_ms"]["median"], case["added_final_ms"], same))
            print("   reads (ms, median): " + ", ".join("%s %.2f" % (k, v["median"])
                                                        for k, v in case["reads_ms"].items()))
            h.release()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(record, f, indent=1)


if __name__ == "__main__":
    main()
