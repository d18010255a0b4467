"""Morse(3, 20) against Morlet(6) on the device, at config 2's geometry (one 2^20-point series, 256
scales, fp64) and config 3's (one 2^18-point series, 128 scales, fp32).

Per configuration the two wavelets run alternately in one process, `--reps` times after one warm-up
call each: `cwt_dev` on a device-resident signal, timed by the device events of the engine's kernels
(last_kernel_ms).  The script reports the median and min-max per wavelet, the class of every row
(last_plan: dense, pruned, overlap-save, expansion by R), and the card's name, power limit and maximum
SM clock.  Needs a GPU: without one it fails.  `--out FILE` also writes the record as JSON.

    python profiles/morse.py --out /tmp/morse.json
"""
import argparse
import collections
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import workloads  # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from coherence_fp32 import card, stats  # noqa: E402

WAVELETS = {"Morse(3, 20)": (_engine.MORSE, (20.0, 3.0)), "Morlet(6)": (_engine.MORLET, 6.0)}


def classes(plan, log2N):
    """Row counts per class of last_plan."""
    out = collections.Counter()
    for p in plan:
        if p == -2:
            out["overlap-save"] += 1
        elif p < 0:
            out["expansion R=%d" % 2 ** (log2N + p)] += 1
        elif p == log2N:
            out["dense"] += 1
        else:
            out["pruned K'=2^%d" % p] += 1
    return dict(sorted(out.items()))


def configs():
    c3 = workloads.C3["paul"]
    return [("config 2 (2^20 x 256, fp64)", workloads.config2_signal(), workloads.config2_scales(),
             _engine.F64, 20),
            ("config 3 (2^18 x 128, fp32)", workloads.config3_signal(),
             workloads.geometric_scales(c3["s0"], c3["dj"], c3["J"]), _engine.F32, 18)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("morse: no CUDA device")
    eng = _engine.Engine(0)
    res = {"card": card(), "configs": {}}
    for name, x, sj, prec, log2N in configs():
        is32 = x.dtype == np.float32
        d = eng.dev_alloc(x.nbytes)
        eng.h2d(d, x)
        times = {w: [] for w in WAVELETS}
        plans = {}
        for w, (fam, par) in WAVELETS.items():      # warm-up and plan
            eng.cwt_dev(d, is32, x.size, 1.0, sj, fam, par, prec)
            plans[w] = classes(eng.last_plan(len(sj)), log2N)
        for _ in range(args.reps):
            for w, (fam, par) in WAVELETS.items():
                eng.cwt_dev(d, is32, x.size, 1.0, sj, fam, par, prec)
                times[w].append(eng.last_kernel_ms())
        eng.dev_free(d)
        res["configs"][name] = {w: {"kernel_ms": stats(times[w]), "rows": plans[w]} for w in WAVELETS}
    print("card: %(name)s, power limit %(power_limit)s, max SM clock %(max_sm_clock)s" % res["card"])
    for name, per in res["configs"].items():
        print(name)
        for w, r in per.items():
            k = r["kernel_ms"]
            print("  %-13s kernels %.3f ms (min %.3f, max %.3f, n %d)  rows %s"
                  % (w, k["median"], k["min"], k["max"], k["n"], r["rows"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
