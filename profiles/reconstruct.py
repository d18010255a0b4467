"""Cost of the reconstruction over a selection (`reconstruct`) against `icwt()` on the same W: config
2's geometry (n0 = 2^20, 256 scales) and config 4's first series (n0 = 2^18, 145 scales), fp64, and a
short series with many scales (n0 = 2^14, 256 scales), fp64, where the column pass has few CTAs.

Per case, after a warm-up call of each, `--reps` calls of each mode, every launch between an event
pair (cwtb_profile_begin / end, launches serialised on one stream): `reconstruct()` with every point
selected, with a quarter of the scales, with `alpha` (the counts of a 3-unit `surrogate_test`) and with
`cluster` (every cluster of a 3-unit `cluster_test`), all on `power_resident`'s W, and `icwt()` and
`reconstruct()` on `cwt_resident`'s W of the same series.  Reported: the kernel time of the column
pass (`SelScaleAvgBody` / `IcwtBody`, median and min-max of the reps), its algorithmic bytes (selected
rows x n0 x 16 B, plus 4 B per point read for counts or labels, plus 8 B x n0 out) over that time
against 3.35 TB/s, and reconstruct over icwt.  The card's name, power limit and maximum SM clock go
into the output.  Needs a GPU: without one it fails.

    python profiles/reconstruct.py --out /tmp/reconstruct.json
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
from surrogate_pvalues import profiled  # noqa: E402

HBM = 3.35e12


def kernel_ms(eng, call, key, reps):
    """Per rep, the summed device time of the launches whose name contains `key`."""
    call()
    out = []
    for _ in range(reps):
        _, rec = profiled(eng, call)
        out.append(sum(r["ms"] for r in rec if key in r["name"]))
    return stats(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("reconstruct: no CUDA device")
    c2, c4 = workloads.C2, workloads.C4
    short = dict(c2, n=2 ** 14)
    cases = [("config2", workloads.config2_signal(), c2),
             ("config4", workloads.config4_signals()[0], c4),
             ("short", workloads.chirp(2 ** 14), short)]
    record = {"card": card(), "reps": args.reps, "cases": []}
    print("card:", record["card"])
    eng = pycwt.default_engine()
    for name, y, c in cases:
        kw = dict(dj=c["dj"], s0=c["s0"], J=c["J"], wavelet=pycwt.Morlet(c["f0"]))
        h = pycwt.power_resident(y, c["dt"], **kw)
        S, n0 = h.shape
        sig = pycwt.significance(1.0, h.dt, h.scales, 0, pycwt.ar1(y)[0])[0]
        h.surrogate_test(mc_count=3, seed=1)
        res = h.cluster_test(sig, mc_count=3, seed=2)
        per = h.period
        band = (float(per[3 * S // 8]), float(per[5 * S // 8]))
        nband = int(h._band(*band).sum())
        rows = list(range(len(res.area)))
        modes = [("all", lambda: h.reconstruct(), S, 0),
                 ("quarter", lambda: h.reconstruct(*band), nband, 0),
                 ("alpha", lambda: h.reconstruct(alpha=0.5), S, 4),
                 ("cluster", lambda: h.reconstruct(cluster=rows), S, 4)]
        out = {"case": name, "shape": [S, n0], "clusters": len(rows), "quarter_rows": nband, "modes": {}}
        for mode, call, nrows, extra in modes:
            t = kernel_ms(eng, call, "SelScaleAvgBody", args.reps)
            out["modes"][mode] = dict(ms=t, bytes=nrows * n0 * (16 + extra) + 8 * n0)
        ht = pycwt.cwt_resident(y, c["dt"], **kw)
        out["modes"]["icwt"] = dict(ms=kernel_ms(eng, ht.icwt, "IcwtBody", args.reps), bytes=S * n0 * 16 + 8 * n0)
        out["modes"]["transform_all"] = dict(ms=kernel_ms(eng, ht.reconstruct, "SelScaleAvgBody", args.reps),
                                             bytes=S * n0 * 16 + 8 * n0)
        for mode, v in out["modes"].items():
            sec = v["ms"]["median"] * 1e-3
            v["TBps"] = v["bytes"] / sec / 1e12 if sec > 0 else None
            v["share_of_3.35TBps"] = v["bytes"] / sec / HBM if sec > 0 else None
            print("%-8s %-14s %-13s %8.3f ms (%.3f-%.3f)  %5.2f TB/s  %3.0f %% of 3.35"
                  % (name, str((S, n0)), mode, v["ms"]["median"], v["ms"]["min"], v["ms"]["max"],
                     v["TBps"] or 0, 100 * (v["share_of_3.35TBps"] or 0)))
        out["all_over_icwt"] = out["modes"]["all"]["ms"]["median"] / out["modes"]["icwt"]["ms"]["median"]
        print("%-8s reconstruct() / icwt() = %.3f" % (name, out["all_over_icwt"]))
        record["cases"].append(out)
        h.release()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(record, f, indent=1)


if __name__ == "__main__":
    main()
