"""`xwt` against `xwt_resident` and its device-side products at config 4 (two 2^18-point series,
s0 = 2, dj = 1/12, J = 144), in fp64 and fp32.

Per precision the two paths run alternately, `--reps` times:
  * xwt: `xwt(...)`, which returns W12 (complex128, 608 MB);
  * resident: `xwt_resident`, then `global_power(inside_coi=True)`, `mean_phase(signif=h.signif)`,
    `scale_avg` over one octave band and `window(slice(None, None, 3), slice(None, None, 3))`.
For every call the script records the end-to-end time of the Python call and, for the two
cross-transform calls, the device time of the engine's kernels (last_kernel_ms); it reports their
median and min-max.  A separate pass records the device time of each product's kernels
(cwtb_profile_begin / end), and the rate at which `RowStatsBody<CxView>` reads W12 in
`global_power(inside_coi=True)`: S x (columns inside the cone) x (bytes per coefficient: 16 in
fp64, 8 in fp32) over its time, against the data sheet's 3.35 TB/s.  The card's name, power limit
and maximum SM clock go into the output.  Needs a GPU: without one it fails.  The summary goes to
stdout; `--out FILE` also writes the full record as JSON.

    python profiles/xwt_resident.py --out /tmp/xwt_resident.json
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
HBM_TBS = 3.35      # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("xwt_resident: no CUDA device")
    eng = pycwt.default_engine()
    y1, y2 = workloads.config4_signals()
    kw = dict(dj=DJ, s0=S0, J=J)
    res = {"card": card(), "config": {"n": int(y1.size), "scales": J + 1,
                                      "field_bytes": int((J + 1) * y1.size * 16)},
           "timing": {}, "product_kernels": {}, "row_stats_rate": {}}
    for p in ("fp64", "fp32"):
        h = pycwt.xwt_resident(y1, y2, DT, precision=p, **kw)
        per = h.period
        band = (per[48], per[60])        # one octave
        products = {
            "global_power": lambda h: h.global_power(inside_coi=True),
            "mean_phase": lambda h: h.mean_phase(signif=h.signif),
            "scale_avg": lambda h: h.scale_avg(*band),
            "window": lambda h: h.window(slice(None, None, 3), slice(None, None, 3)),
        }

        def xwt_call():
            return pycwt.xwt(y1, y2, DT, precision=p, **kw)

        def resident_call():
            return pycwt.xwt_resident(y1, y2, DT, precision=p, **kw)
        xwt_call()                                 # warm-up: module load, plans, buffers
        h = resident_call()
        for f in products.values():
            f(h)
        t = {"xwt_call_ms": [], "xwt_device_ms": [], "resident_call_ms": [], "resident_device_ms": [],
             "resident_total_ms": []}
        t.update({k + "_call_ms": [] for k in products})
        for _ in range(args.reps):
            t0 = time.perf_counter()
            out = xwt_call()
            t["xwt_call_ms"].append((time.perf_counter() - t0) * 1e3)
            t["xwt_device_ms"].append(eng.last_kernel_ms())
            del out
            t0 = time.perf_counter()
            h = resident_call()
            t1 = time.perf_counter()
            t["resident_device_ms"].append(eng.last_kernel_ms())
            t["resident_call_ms"].append((t1 - t0) * 1e3)
            for k, f in products.items():
                ta = time.perf_counter()
                f(h)
                t[k + "_call_ms"].append((time.perf_counter() - ta) * 1e3)
            t["resident_total_ms"].append((time.perf_counter() - t0) * 1e3)
        res["timing"][p] = {k: stats(v) for k, v in t.items()}
        print(p, json.dumps({k: round(v["median"], 3) for k, v in res["timing"][p].items()}), flush=True)

        # device time of each product's kernels, launches bracketed by events (separate pass)
        res["product_kernels"][p] = {}
        for k, f in products.items():
            eng.profile_begin()
            f(h)
            rec = eng.profile_end()
            res["product_kernels"][p][k] = {"device_ms": sum(r["ms"] for r in rec), "kernels": rec}
        print(p, "product device ms",
              json.dumps({k: round(v["device_ms"], 4) for k, v in res["product_kernels"][p].items()}),
              flush=True)

        # read rate of the row-statistics kernel over the inside-COI columns
        lo, hi = h.coi_ranges()
        nbytes = int((hi - lo).sum()) * (16 if p == "fp64" else 8)
        ms = []
        for _ in range(5):
            eng.profile_begin()
            h.global_power(inside_coi=True)
            ms.append(sum(r["ms"] for r in eng.profile_end() if "RowStatsBody" in r["name"]))
        kms = float(np.median(ms))
        rate = nbytes / (kms * 1e-3) / 1e12
        res["row_stats_rate"][p] = {"bytes": nbytes, "kernel_ms": kms, "kernel_ms_all": ms, "TB_s": rate,
                                    "of_data_sheet": rate / HBM_TBS}
        print(p, "RowStatsBody<CxView> %.1f MB in %.4f ms: %.2f TB/s, %.2f of %.2f TB/s"
              % (nbytes / 1e6, kms, rate, rate / HBM_TBS, HBM_TBS), flush=True)
        h.release()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
