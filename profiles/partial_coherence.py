"""Partial and multiple wavelet coherence at config 4's geometry (three 2^18-point series, s0 = 2,
dj = 1/12, J = 144, K = 14), in fp64 and fp32.

Per precision four paths run alternately, `--reps` times:
  * multiple: `multiple_wct(y, x1, x2)`;
  * partial: `partial_wct(y, x1, x2)`;
  * wct: `wct(y, x1, sig=False)`, the two-series pipeline, for scale;
  * composed (fp64 only, the public calls' arithmetic): what a user writes without these calls,
    3 x `cwt` + 6 x `Morlet.smooth` on host arrays + the formula of RM2 in numpy.
For every call the script records the end-to-end time of the Python call and, for the device calls,
the device time of the engine's kernels (last_kernel_ms); it reports their median and min-max.  A
separate pass records the per-kernel device times of one `multiple_wct` (cwtb_profile_begin / end),
grouped into the three transforms, Wct3PrepBody, the five smoothing passes and Wct3FinalBody, and
gives the final kernel's HBM rate from the bytes it must move (five fields read once, one float64
output written) against the data sheet's 3.35 TB/s.  The results of the paths are compared at the
timed size.  The card's name, power limit and maximum SM clock go into the output, with the SM
clock read right after the timed loop.

Monte-Carlo leg, at config 4's Monte-Carlo geometry (surrogates of 49152 samples padded to 65536,
145 scales, K = 14): per precision, `--mc-count` triples of `wct3_significance` in seeded and in
host-RNG mode, alternating with as many pairs of the two-series `wct_significance` in the same two
modes, `--mc-reps` times; call time and the device time of the engine's Monte-Carlo call.  Then the
per-kernel device times of one seeded triple (noise, three transforms, prep, five smoothings, the
final kernel with both histograms), and the final kernel of the output path (`Engine.wct3` with both
outputs) at the same geometry, per row, to show what the histograms' atomics cost against the
stores of the output path.

Needs a GPU: without one it fails.  The summary goes to stdout; `--out FILE` also writes the full
record as JSON.

    python profiles/partial_coherence.py --out /tmp/partial_coherence.json
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
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import workloads  # noqa: E402
import pycwt_b200 as pycwt  # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from coherence_fp32 import card, stats  # noqa: E402

DT, DJ, S0, J = 1.0, 1 / 12, 2.0, 144
HBM_PEAK = 3.35e12       # bytes/s, H100 SXM data sheet


def triple():
    y, x1 = workloads.config4_signals()
    n = y.size
    return y, x1, workloads.chirp(n, phase=2.1) + 0.5 * np.random.RandomState(2).randn(n)


def composed(y, x1, x2, mother):
    """RM2 from public calls only: three transforms to the host, six smoothings, numpy."""
    Ws = []
    for v in (y, x1, x2):
        W, sj = pycwt.cwt((v - v.mean()) / v.std(), DT, DJ, S0, J, mother)[:2]
        Ws.append(W)
    inv = 1.0 / sj[:, None]
    Sy, S1, S2 = (mother.smooth(np.abs(W) ** 2 * inv, DT, DJ, sj) for W in Ws)
    Wy, W1, W2 = Ws
    Sy1, Sy2, S12 = (mother.smooth(a * b.conj() * inv, DT, DJ, sj) for a, b in ((Wy, W1), (Wy, W2), (W1, W2)))
    N = S2 * np.abs(Sy1) ** 2 + S1 * np.abs(Sy2) ** 2 - 2 * (Sy1 * S12 * Sy2.conj()).real
    return N / (Sy * (S1 * S2 - np.abs(S12) ** 2))


def sm_clock():
    out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout
    return out.splitlines()[0].strip()


def kernel_groups(rec, S, n0, esize):
    """Device ms of the transforms, the prep, the smoothing and the final kernel of one call."""
    names = [r["name"] for r in rec]
    ip = next(i for i, s in enumerate(names) if s.startswith("Wct3PrepBody"))
    iF = next(i for i, s in enumerate(names) if s.startswith("Wct3FinalBody"))
    ms = lambda rs: float(sum(r["ms"] for r in rs))        # noqa: E731
    final_ms = ms(rec[iF:iF + 1])
    final_bytes = S * n0 * (5 * 2 * esize + 8)
    return {"transforms_ms": ms(rec[:ip]), "prep_ms": ms(rec[ip:ip + 1]),
            "smoothing_ms": ms(rec[ip + 1:iF]), "smoothing_per_field_ms": ms(rec[ip + 1:iF]) / 5,
            "final_ms": final_ms, "final_name": names[iF], "final_bytes": int(final_bytes),
            "final_hbm_TBps": final_bytes / (final_ms * 1e-3) / 1e12,
            "final_share_of_hbm_peak": final_bytes / (final_ms * 1e-3) / HBM_PEAK,
            "sum_ms": ms(rec), "launches": len(rec)}


def mc_groups(rec):
    """Device ms of one Monte-Carlo triple by stage; the final kernel's ms per output row."""
    names = [r["name"] for r in rec]
    ms = lambda rs: float(sum(r["ms"] for r in rs))        # noqa: E731
    ip = next(i for i, s in enumerate(names) if s.startswith("Wct3PrepBody"))
    iF = next(i for i, s in enumerate(names) if s.startswith("Wct3FinalBody"))
    noise = [r for r in rec[:ip] if r["name"].startswith("NoiseBody")]
    return {"noise_ms": ms(noise), "transforms_ms": ms(rec[:ip]) - ms(noise), "prep_ms": ms(rec[ip:ip + 1]),
            "smoothing_ms": ms(rec[ip + 1:iF]), "final_ms": ms(rec[iF:iF + 1]), "final_name": names[iF],
            "final_rows": int(rec[iF].get("rows", 0)), "sum_ms": ms(rec), "launches": len(rec)}


def mc_leg(eng, count, reps, res):
    from pycwt_b200 import wavelet as wv
    c4 = workloads.C4
    dt, dj, s0, J = c4["dt"], c4["dj"], c4["s0"], c4["J"]
    mother = pycwt.Morlet(6)
    prob = wv._mc_problem(dt, dj, s0, J, mother)
    res["mc"] = {"config": {"N": prob["N"], "scales": int(prob["sj"].size), "maxscale": prob["maxscale"],
                            "count": count}, "timing": {}, "kernels": {}}
    for p in ("fp64", "fp32"):
        paths = {
            "triples_seeded": lambda s: pycwt.wct3_significance(0.3, 0.5, 0.2, dt, dj, s0, J, mc_count=count,
                                                                progress=False, seed=s, precision=p),
            "triples_host": lambda s: pycwt.wct3_significance(0.3, 0.5, 0.2, dt, dj, s0, J, mc_count=count,
                                                              progress=False, precision=p),
            "pairs_seeded": lambda s: wv._wct_significance(0.3, 0.5, dt, dj, s0, J, mc_count=count, progress=False,
                                                           cache=False, seed=s, precision=p),
            "pairs_host": lambda s: wv._wct_significance(0.3, 0.5, dt, dj, s0, J, mc_count=count, progress=False,
                                                         cache=False, precision=p),
        }
        for f in paths.values():                          # warm-up
            f(1)
        t = {}
        for rep in range(reps):
            np.random.seed(rep)
            for k, f in paths.items():
                t0 = time.perf_counter()
                f(100 + rep)
                t.setdefault(k + "_call_s", []).append(time.perf_counter() - t0)
                t.setdefault(k + "_device_s", []).append(eng.last_kernel_ms() * 1e-3)
        res["mc"]["timing"][p] = {k: stats(v) for k, v in t.items()}
        res["mc"]["timing"][p]["sm_clock_after"] = sm_clock()
        print("mc", p, json.dumps({k: round(v["median"], 4) for k, v in res["mc"]["timing"][p].items()
                                   if isinstance(v, dict)}), flush=True)

        eng.profile_begin()
        pycwt.wct3_significance(0.3, 0.5, 0.2, dt, dj, s0, J, mc_count=1, progress=False, seed=7, precision=p)
        mc = mc_groups(eng.profile_end())
        # the output path's final kernel at the same geometry (both outputs), for its per-row cost
        noise = eng.mc_surrogates3(7, 0, 1, prob["N"])[0]
        eng.profile_begin()
        eng.wct3(*noise, dt, dj, prob["sj"], _engine.MORLET, 6.0, 14, precision=_engine.F64 if p == "fp64" else _engine.F32)
        out = mc_groups(eng.profile_end())
        res["mc"]["kernels"][p] = {"mc_triple": mc, "output_path": out,
                                   "final_ms_per_row_mc": mc["final_ms"] / prob["maxscale"],
                                   "final_ms_per_row_output": out["final_ms"] / prob["sj"].size}
        print("mc", p, "kernels", json.dumps({k: (round(v, 5) if isinstance(v, float) else v)
                                              for k, v in res["mc"]["kernels"][p].items()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mc-count", type=int, default=200, help="triples (and pairs) per Monte-Carlo call")
    ap.add_argument("--mc-reps", type=int, default=3)
    ap.add_argument("--mc-only", action="store_true", help="only the Monte-Carlo leg")
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if _engine.device_count() <= 0:
        raise SystemExit("partial_coherence: no CUDA device")
    eng = pycwt.default_engine()
    y, x1, x2 = triple()
    mother = pycwt.Morlet(6)
    kw = dict(dj=DJ, s0=S0, J=J)
    S, n0 = J + 1, y.size
    res = {"card": card(), "config": {"n": int(n0), "scales": S, "boxcar": 14}, "timing": {},
           "kernels": {}, "checks": {}}
    out64 = {}
    for p in (() if args.mc_only else ("fp64", "fp32")):
        paths = {
            "multiple": lambda: pycwt.multiple_wct(y, x1, x2, DT, precision=p, **kw)[0],
            "partial": lambda: pycwt.partial_wct(y, x1, x2, DT, precision=p, **kw)[0],
            "wct": lambda: pycwt.wct(y, x1, DT, sig=False, precision=p, **kw)[0],
        }
        if p == "fp64":
            paths["composed"] = lambda: composed(y, x1, x2, mother)
        outs = {k: f() for k, f in paths.items()}        # warm-up: module load, plans, buffers
        t = {}
        for _ in range(args.reps):
            for k, f in paths.items():
                t0 = time.perf_counter()
                r = f()
                t.setdefault(k + "_call_ms", []).append((time.perf_counter() - t0) * 1e3)
                if k != "composed":
                    t.setdefault(k + "_device_ms", []).append(eng.last_kernel_ms())
                del r
        res["timing"][p] = {k: stats(v) for k, v in t.items()}
        res["timing"][p]["sm_clock_after"] = sm_clock()
        print(p, json.dumps({k: round(v["median"], 3) for k, v in res["timing"][p].items()
                             if isinstance(v, dict)}), flush=True)

        eng.profile_begin()
        pycwt.multiple_wct(y, x1, x2, DT, precision=p, **kw)
        rec = eng.profile_end()
        res["kernels"][p] = kernel_groups(rec, S, n0, 8 if p == "fp64" else 4)
        res["kernels"][p]["records"] = rec
        print(p, "kernels", json.dumps({k: (round(v, 4) if isinstance(v, float) else v)
                                        for k, v in res["kernels"][p].items() if k != "records"}), flush=True)

        D12 = 1 - pycwt.wct(x1, x2, DT, sig=False, precision="fp64", **kw)[0]
        if p == "fp64":
            out64 = outs
            res["checks"]["multiple_vs_composed_scaled"] = float((np.abs(outs["multiple"] - outs["composed"]) * D12).max())
        else:
            res["checks"]["fp32_vs_fp64_multiple_scaled"] = float((np.abs(outs["multiple"] - out64["multiple"]) * D12).max())
        res["checks"]["%s_identity_1-RM2=(1-R2y2)(1-RP2)" % p] = float(
            (np.abs((1 - outs["multiple"])
                    - (1 - pycwt.wct(y, x2, DT, sig=False, precision=p, **kw)[0]) * (1 - outs["partial"])) * D12).max())
    print("checks", json.dumps(res["checks"]), flush=True)
    if args.mc_count > 0:
        mc_leg(eng, args.mc_count, args.mc_reps, res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
