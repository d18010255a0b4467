"""Config 2 with and without the overlap-save rows (CWTB_OS), alternating in one process:

    python profiles/micro/os_ab.py [rounds]

Each round times `bench_last` on a context with the class on and on one with it off (the switch is
read when a context is created).  Prints the card, the median and min-max step time of each arm,
the serialised per-kernel table of each (`profile_last`) and the largest per-row difference of W
between the arms, relative to the row's maximum."""
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import workloads as wl          # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from bench import pin_to_gpu_numa_node  # noqa: E402


def engine(os_on):
    os.environ["CWTB_OS"] = "1" if os_on else "0"
    try:
        return _engine.Engine(0)
    finally:
        del os.environ["CWTB_OS"]


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    pin_to_gpu_numa_node(0)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip())
    c = wl.C2
    x = wl.config2_signal()
    sj = wl.config2_scales()
    arms = {"os on": engine(True), "os off": engine(False)}
    dev = {}
    for name, eng in arms.items():
        d = eng.dev_alloc(x.nbytes)
        eng.h2d(d, x)
        eng.cwt_dev(d, 0, c["n"], c["dt"], sj, _engine.MORLET, c["f0"], _engine.F64)
        eng.bench_last(5)
        dev[name] = d
        plan = eng.last_plan(len(sj))
        print("%-7s plan: %d overlap-save rows %s, %d expansion, %d exact" % (
            name, sum(p == -2 for p in plan), [j for j, p in enumerate(plan) if p == -2],
            sum(p < -2 for p in plan), sum(p >= 0 for p in plan)))
    # planning cost: a call whose scales differ in the last bits must plan again (host clock around
    # the synchronous call, one step included)
    for name, eng in arms.items():
        t = []
        for i in range(4):
            s = sj * (1.0 + 1e-15 * (i % 2 + 1))
            t0 = time.perf_counter()
            eng.cwt_dev(dev[name], 0, c["n"], c["dt"], s, _engine.MORLET, c["f0"], _engine.F64)
            t.append((time.perf_counter() - t0) * 1e3)
        eng.cwt_dev(dev[name], 0, c["n"], c["dt"], sj, _engine.MORLET, c["f0"], _engine.F64)
        print("%-7s call that plans again: median %.1f ms (min %.1f, max %.1f)" % (
            name, float(np.median(t)), min(t), max(t)))
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for name, eng in arms.items():
            times[name].append(eng.bench_last(20))
    for name, t in times.items():
        print("%-7s step %.4f ms (min %.4f, max %.4f) over %d runs of 20 steps" % (
            name, float(np.median(t)), min(t), max(t), len(t)))
    for name, eng in arms.items():
        print(name + ": serialised kernels of one step")
        for k in sorted(eng.profile_last(), key=lambda k: -k["ms"]):
            print("      %-46s %3d x  %7.4f ms  rows %d" % (k["name"], k["launches"], k["ms"], k["rows"]))
    rows = 72   # every row the class can take at this geometry (j < 64), and some beyond
    a = arms["os on"].get_w(rows, c["n"])
    b = arms["os off"].get_w(rows, c["n"])
    err = [float(np.abs(a[i] - b[i]).max() / np.abs(b[i]).max()) for i in range(rows)]
    print("per row max|W_on - W_off| / max|W_off| of the row: worst %.2e (row %d)" % (max(err), int(np.argmax(err))))
    del a, b
    for name, eng in arms.items():
        eng.dev_free(dev[name])
        eng.close()


if __name__ == "__main__":
    main()
