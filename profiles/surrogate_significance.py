"""What the phase-randomised surrogates cost beside the coherence pipeline they feed, at config 4's
data sizes (series of 2^18 samples, s0 = 2, dj = 1/12, J = 144, K = 14), for two and three series,
in fp64 and fp32.

After a warm-up call, `--reps` calls of `Engine.wct_mc_phase` with `--units` surrogate units each
run between `profile_begin` / `profile_end` (a CUDA event pair around every kernel launch), and as
many calls of the white-noise `wct_mc_seeded` / `wct3_mc_seeded` at the same length.  Per unit:
  (a) generation: PhaseRotBody, the inverse row transforms and RealPartBody (the kernels recorded
      under "phase:"), plus once per call the forward transform of the data ("data:");
  (b) pipeline: every other kernel of the call (transforms, products, smoothing, final kernel);
  (c) the white-noise call: NoiseBody and its pipeline.
Medians over the calls, with the bytes the rotation and the store move against the data sheet's
3.35 TB/s.  The card's name and power limit are printed with the numbers.

Needs a GPU: without one it fails.  `--out FILE` also writes the record as JSON.

    python profiles/surrogate_significance.py --out /tmp/surrogate_significance.json
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import workloads  # noqa: E402
import pycwt_b200 as pycwt  # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from coherence_fp32 import card  # noqa: E402

HBM_PEAK = 3.35e12       # bytes/s, H100 SXM data sheet


def split(rec, *prefixes):
    """ms of the records whose kernel name starts with each prefix, then ms of all the others."""
    ms = [float(sum(r["ms"] for r in rec if r["name"].startswith(p))) for p in prefixes]
    return ms + [float(sum(r["ms"] for r in rec)) - sum(ms)]


def data(n):
    y, x1 = workloads.config4_signals(n)
    x2 = 0.6 * x1 + workloads.chirp(n, phase=2.1) + 0.5 * np.random.RandomState(2).randn(n)
    return np.stack([(v - v.mean()) / v.std() for v in (y, x1, x2)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=workloads.C4["n"], help="samples per series")
    ap.add_argument("--units", type=int, default=8, help="surrogate units per call")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="JSON file for the full record (default: stdout only)")
    args = ap.parse_args()
    if args.n < 4 or args.units < 1 or args.reps < 1:
        ap.error("--n >= 4, --units >= 1, --reps >= 1")
    from pycwt_b200 import wavelet as wv
    c4 = workloads.C4
    dt, dj, s0, J = c4["dt"], c4["dj"], c4["s0"], c4["J"]
    mother = pycwt.Morlet(c4["f0"])
    prob = wv._mc_problem(dt, dj, s0, J, mother, N=args.n)
    K = wv._boxcar_len(mother, dj)
    x = data(args.n)
    print("geometry: n0 = %d, %d scales, maxscale %d, K = %d, %d units per call"
          % (args.n, prob["sj"].size, prob["maxscale"], K, args.units), flush=True)
    if _engine.device_count() <= 0:
        raise SystemExit("surrogate_significance: no CUDA device")
    eng = pycwt.default_engine()
    res = {"card": card(), "config": {"n": args.n, "scales": int(prob["sj"].size), "boxcar": K,
                                      "units": args.units, "reps": args.reps}, "runs": {}}
    print("card", json.dumps(res["card"]), flush=True)
    tail = (dt, prob["sj"], _engine.MORLET, c4["f0"], K, prob["mask"], prob["maxscale"], prob["nbins"])
    for nser, groups in ((2, (0, 1)), (3, (0, 1, 1))):
        for p, prec in (("fp64", _engine.F64), ("fp32", _engine.F32)):
            def hists():
                return [np.zeros((prob["sj"].size, prob["nbins"]), dtype=np.int64) for _ in range(nser - 1)]

            def phase():
                eng.wct_mc_phase(x[:nser], groups, 7, 0, args.units, *tail, *hists(), precision=prec)

            def white():
                f = eng.wct_mc_seeded if nser == 2 else eng.wct3_mc_seeded
                f(7, 0, args.units, args.n, *tail, *hists(), precision=prec)

            phase()
            white()                                          # warm-up: modules, plans, buffers
            t = {k: [] for k in ("gen", "fwd", "pipe", "noise", "white_pipe")}
            for _ in range(args.reps):
                eng.profile_begin()
                phase()
                gen, fwd, pipe = split(eng.profile_end(), "phase:", "data:")
                eng.profile_begin()
                white()
                noise, wpipe = split(eng.profile_end(), "NoiseBody")
                for k, v in zip(t, (gen, fwd, pipe, noise, wpipe)):
                    t[k].append(v)
            m = {k: float(np.median(v)) for k, v in t.items()}
            u = args.units
            samples = nser * args.n
            r = {"generation_ms_per_unit": m["gen"] / u, "data_spectra_ms_per_call": m["fwd"],
                 "pipeline_ms_per_unit": m["pipe"] / u, "generation_over_pipeline": m["gen"] / m["pipe"],
                 "white_noise_ms_per_unit": m["noise"] / u, "white_pipeline_ms_per_unit": m["white_pipe"] / u,
                 # rotation: read the data spectra (cached after the first unit), write 16 B per sample;
                 # store: read 16 B, write the engine's real type
                 "rotate_plus_store_bytes_per_unit": samples * (16 + 16 + (8 if p == "fp64" else 4)),
                 "all": t}
            r["rotate_plus_store_floor_ms_per_unit"] = r["rotate_plus_store_bytes_per_unit"] / HBM_PEAK * 1e3
            res["runs"]["%d series %s" % (nser, p)] = r
            print("%d series %s:" % (nser, p),
                  json.dumps({k: (round(v, 5) if isinstance(v, float) else v) for k, v in r.items() if k != "all"}),
                  flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
