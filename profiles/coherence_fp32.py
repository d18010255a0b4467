"""fp32 against fp64 coherence at config 4 (two 2^18-point series, s0 = 2, dj = 1/12, J = 144):
xwt, wct(sig=False) and 200 Monte-Carlo surrogate pairs (host-RNG and seeded mode).

The two precisions run alternately, `--reps` times per leg.  For every call the script records the
device time of the engine's kernels (last_kernel_ms) and the end-to-end time of the Python call,
and reports their median and spread.  A separate pass records the per-kernel device times of one
surrogate pair in each precision (cwtb_profile_begin / end).  The fp32-versus-fp64 errors are
taken at the timed sizes.  The card's name, power limit and maximum SM clock go into the output.
Needs a GPU: without one it fails.  The summary goes to stdout; `--out FILE` also writes the full
record, per-kernel tables included, as JSON.

    python profiles/coherence_fp32.py --out /tmp/coherence_fp32.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import workloads  # noqa: E402
import pycwt_b200 as pycwt  # noqa: E402
from pycwt_b200 import _engine, wavelet as wv  # noqa: E402

DT, DJ, S0, J = 1.0, 1 / 12, 2.0, 144
PREC = {"fp64": _engine.F64, "fp32": _engine.F32}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, power, clock = [s.strip() for s in out.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def stats(v):
    v = np.asarray(v, dtype=float)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max()), "n": int(v.size)}


def hist_checks(h32, h64, prob):
    """Counts per row, 'every sample moves at most one bin', and the levels."""
    nxt = np.concatenate([h64[:, 1:], np.zeros((h64.shape[0], 1), h64.dtype)], axis=1)
    moved = np.abs(np.cumsum(h32, axis=1) - np.cumsum(h64, axis=1))
    s32, s64 = wv._mc_levels(prob, h32, 0.95), wv._mc_levels(prob, h64, 0.95)
    ok = np.isfinite(s64)
    return {"row_counts_equal": bool((h32.sum(axis=1) == h64.sum(axis=1)).all()),
            "at_most_one_bin": bool((moved <= h64 + nxt).all()),
            "samples_moved_upper_bound": int(moved.sum()),
            "sig95_finite_pattern_equal": bool((np.isfinite(s32) == ok).all()),
            "sig95_max_abs_diff": float(np.abs(s32[ok] - s64[ok]).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pairs", type=int, default=200)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("coherence_fp32: no CUDA device")
    eng = pycwt.default_engine()
    y1, y2 = workloads.config4_signals()
    mother = pycwt.Morlet(6)
    prob = wv._mc_problem(DT, DJ, S0, J, mother)
    N = prob["N"]

    def draw_factory():
        rs = np.random.RandomState(2024)
        return lambda i: (rs.randn(N), rs.randn(N))

    legs = {
        "xwt": lambda p: pycwt.xwt(y1, y2, DT, dj=DJ, s0=S0, J=J, precision=p),
        "wct": lambda p: pycwt.wct(y1, y2, DT, dj=DJ, s0=S0, J=J, sig=False, precision=p),
        "mc_host": lambda p: wv._mc_histogram(prob, DT, DJ, mother, draw_factory(), range(args.pairs),
                                              precision=PREC[p]),
        "mc_seeded": lambda p: wv._mc_histogram_seeded(prob, DT, DJ, mother, 7, 0, args.pairs,
                                                       precision=PREC[p]),
    }
    res = {"card": card(), "config": {"n": int(y1.size), "scales": J + 1, "mc_N": N, "mc_pairs": args.pairs},
           "timing": {}, "errors": {}}
    outputs = {}
    for leg, fn in legs.items():
        for p in ("fp64", "fp32"):       # warm-up: module load, plans, buffers
            fn(p)
        dev = {"fp64": [], "fp32": []}
        e2e = {"fp64": [], "fp32": []}
        for _ in range(args.reps):
            for p in ("fp64", "fp32"):
                t0 = time.perf_counter()
                out = fn(p)
                e2e[p].append((time.perf_counter() - t0) * 1e3)
                dev[p].append(eng.last_kernel_ms())
                outputs[(leg, p)] = out
        res["timing"][leg] = {p: {"device_ms": stats(dev[p]), "call_ms": stats(e2e[p])} for p in dev}
        print(leg, json.dumps(res["timing"][leg]), flush=True)

    W64, W32 = outputs[("xwt", "fp64")][0], outputs[("xwt", "fp32")][0]
    rowmax = np.abs(W64).max(axis=1)
    row_rel = np.abs(W32 - W64).max(axis=1) / rowmax
    c64, c32 = outputs[("wct", "fp64")], outputs[("wct", "fp32")]
    dW = np.abs(c32[0] - c64[0])
    ang = np.abs(W64) * np.abs(np.exp(1j * c32[1]) - np.exp(1j * c64[1]))
    res["errors"]["xwt_relerr"] = float(np.abs(W32 - W64).max() / rowmax.max())
    res["errors"]["xwt_relerr_worst_row"] = float(row_rel.max())
    res["errors"]["angle_metric_worst_row"] = float((ang.max(axis=1) / rowmax).max())
    res["errors"]["wct_max_abs"] = float(dW.max())
    res["errors"]["wct_p999_abs"] = float(np.percentile(dW, 99.9))
    res["errors"]["wct_worst_row"] = int(dW.max(axis=1).argmax())
    for leg in ("mc_host", "mc_seeded"):
        res["errors"][leg] = hist_checks(outputs[(leg, "fp32")], outputs[(leg, "fp64")], prob)
    print("errors", json.dumps(res["errors"]), flush=True)

    # per-kernel device times of one surrogate pair, kernels serialised (separate pass)
    res["kernels_one_pair"] = {}
    for p in ("fp64", "fp32"):
        wv._mc_histogram_seeded(prob, DT, DJ, mother, 7, 0, 1, precision=PREC[p])
        eng.profile_begin()
        wv._mc_histogram_seeded(prob, DT, DJ, mother, 7, 0, 1, precision=PREC[p])
        res["kernels_one_pair"][p] = sorted(eng.profile_end(), key=lambda r: -r["ms"])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
        print(json.dumps({k: res[k] for k in ("card", "config", "timing", "errors")}))
    else:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
