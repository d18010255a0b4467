"""The register-resident 1024-point core (fft_tile.cuh: x32_first / x32_last) against a library
built without it, side by side in one process, alternating:

    python profiles/micro/x32_ab.py PARENT_LIB [NEW_LIB] [rounds]

PARENT_LIB is a library built from the parent commit (for instance with build_variant.py in a
checkout of it), NEW_LIB defaults to the in-tree pycwt_b200/libcwtb200.so.  Config 2 (Morlet(6),
N = 2^20, 256 scales, fp64): each round times `bench_last(20)` on each library (default 8 rounds).
Prints the card, its power limit and max SM clock, the median and min-max step time of each arm,
the serialised time and us per row of the three kernels that run the core (OsBody, the dense first
kernel PassABody<double, 1024, 0, 1> and the second kernel PassBBody<double, 1, 1024>), the full
per-kernel table of each arm (`profile_last`), the overlap-save rows of each plan, and the largest
per-row difference of W between the arms, relative to the row's maximum."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import workloads as wl          # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from bench import pin_to_gpu_numa_node  # noqa: E402

CORE = (("OsBody", "OsBody<4>"), ("dense first", "PassABody<double, 1024, 0, 1>"),
        ("second", "PassBBody<double, 1, 1024"))


def main():
    args = sys.argv[1:]
    parent = args[0]
    new = args[1] if len(args) > 1 and not args[1].isdigit() else os.path.join(ROOT, "pycwt_b200", "libcwtb200.so")
    rounds = int(args[-1]) if args[-1].isdigit() else 8
    pin_to_gpu_numa_node(0)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip())
    c = wl.C2
    x = wl.config2_signal()
    sj = wl.config2_scales()
    arms = {"parent": _engine.Engine(0, lib_path=parent), "new": _engine.Engine(0, lib_path=new)}
    dev = {}
    for name, eng in arms.items():
        d = eng.dev_alloc(x.nbytes)
        eng.h2d(d, x)
        eng.cwt_dev(d, 0, c["n"], c["dt"], sj, _engine.MORLET, c["f0"], _engine.F64)
        eng.bench_last(10)
        dev[name] = d
        plan = eng.last_plan(len(sj))
        os_rows = [j for j, p in enumerate(plan) if p == -2]
        print("%-6s plan: %d overlap-save rows (%s), %d expansion, %d exact" % (
            name, len(os_rows), "%d..%d" % (os_rows[0], os_rows[-1]) if os_rows else "-",
            sum(p < -2 for p in plan), sum(p >= 0 for p in plan)))
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for name, eng in arms.items():
            times[name].append(eng.bench_last(20))
    for name, t in times.items():
        print("%-6s config 2 step %.4f ms (min %.4f, max %.4f) over %d runs of 20 steps" % (
            name, float(np.median(t)), min(t), max(t), len(t)))
    print("median difference parent - new: %.4f ms" % (float(np.median(times["parent"])) - float(np.median(times["new"]))))
    prof = {name: eng.profile_last() for name, eng in arms.items()}
    for label, key in CORE:
        for name in arms:
            ks = [k for k in prof[name] if k["name"].startswith(key)]
            ms = sum(k["ms"] for k in ks)
            rows = sum(k["rows"] for k in ks)
            print("%-11s %-6s %7.4f ms serialised, %3d rows, %5.1f us per row" % (
                label, name, ms, rows, 1e3 * ms / rows if rows else float("nan")))
    for name in arms:
        print(name + ": serialised kernels of one step")
        for k in sorted(prof[name], key=lambda k: -k["ms"]):
            print("      %-52s %3d x  %7.4f ms  rows %d" % (k["name"], k["launches"], k["ms"], k["rows"]))
    err = []
    for r0 in range(0, len(sj), 32):   # W in 512 MiB pieces
        rows = []
        for eng in arms.values():
            out = np.empty((32, c["n"]), np.complex128)
            eng._check(eng.lib.cwtb_get_w(eng.h, _engine._ptr(out), 1, r0, 32))
            rows.append(out)
        for i in range(32):
            err.append(float(np.abs(rows[1][i] - rows[0][i]).max() / np.abs(rows[0][i]).max()))
    err = np.array(err)
    print("per row max|W_new - W_parent| / max|W_parent| of the row: worst %.2e (row %d); rows 0..63 worst %.2e, "
          "rows 64.. worst %.2e, rows bit-identical %d of %d" % (
              err.max(), int(err.argmax()), err[:64].max(), err[64:].max(), int((err == 0).sum()), len(err)))
    print("per row, rows 0..63: " + " ".join("%.1e" % e for e in err[:64]))
    for name, eng in arms.items():
        eng.dev_free(dev[name])
        eng.close()


if __name__ == "__main__":
    main()
