"""Two builds of the engine side by side in one process, alternating:

    python profiles/micro/coarse_ab.py PARENT_LIB [NEW_LIB] [rounds]

PARENT_LIB is a library built from the parent commit (for instance with build_variant.py in a
checkout of it), NEW_LIB defaults to the in-tree pycwt_b200/libcwtb200.so.  Config 2 (Morlet(6),
N = 2^20, 256 scales, fp64): each round times `bench_last(20)` on each library.  Prints the card,
its power limit and max SM clock, the median and min-max step time of each arm, the launches per
step, the serialised per-kernel table of each (`profile_last`), and whether W is bit-identical
between the arms: config 2 (fp64), config 3's Paul(4) transform (fp32), and xwt and wct at config 4
in fp64 and fp32."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import workloads as wl          # noqa: E402
import pycwt_b200 as pycwt      # noqa: E402
from pycwt_b200 import _engine  # noqa: E402
from pycwt_b200.wavelet import _boxcar_len  # noqa: E402
from bench import pin_to_gpu_numa_node  # noqa: E402


def identical(arms, fn):
    a, b = (fn(e) for e in arms.values())
    if isinstance(a, tuple):
        return all(np.array_equal(x, y) for x, y in zip(a, b) if x is not None)
    return np.array_equal(a, b)


def main():
    args = sys.argv[1:]
    parent = args[0]
    new = args[1] if len(args) > 1 and not args[1].isdigit() else os.path.join(ROOT, "pycwt_b200", "libcwtb200.so")
    rounds = int(args[-1]) if args[-1].isdigit() else 6
    pin_to_gpu_numa_node(0)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip())
    c = wl.C2
    x = wl.config2_signal()
    sj = wl.config2_scales()
    arms = {"parent": _engine.Engine(0, lib_path=parent), "new": _engine.Engine(0, lib_path=new)}
    dev = {}
    launches = {}
    for name, eng in arms.items():
        d = eng.dev_alloc(x.nbytes)
        eng.h2d(d, x)
        eng.cwt_dev(d, 0, c["n"], c["dt"], sj, _engine.MORLET, c["f0"], _engine.F64)
        eng.bench_last(10)
        launches[name] = eng.last_launch_count()
        dev[name] = d
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for name, eng in arms.items():
            times[name].append(eng.bench_last(20))
    for name, t in times.items():
        print("%-6s config 2 step %.4f ms (min %.4f, max %.4f) over %d runs of 20 steps, %d launches per step" % (
            name, float(np.median(t)), min(t), max(t), len(t), launches[name]))
    print("median difference parent - new: %.4f ms" % (float(np.median(times["parent"])) - float(np.median(times["new"]))))
    for name, eng in arms.items():
        print(name + ": serialised kernels of one step")
        for k in sorted(eng.profile_last(), key=lambda k: -k["ms"]):
            print("      %-52s %3d x  %7.4f ms  rows %d" % (k["name"], k["launches"], k["ms"], k["rows"]))
    same = True
    for r0 in range(0, len(sj), 32):   # W of config 2 in 512 MiB pieces

        rows = []
        for eng in arms.values():
            out = np.empty((32, c["n"]), np.complex128)
            eng._check(eng.lib.cwtb_get_w(eng.h, _engine._ptr(out), 1, r0, 32))
            rows.append(out)
        same = same and np.array_equal(rows[0], rows[1])
    print("config 2 W (fp64, 256 rows): %s" % ("bit-identical" if same else "DIFFERENT"))
    for name, eng in arms.items():
        eng.dev_free(dev[name])
    # config 3 (fp32, N = 2^18): the coarse chain is its critical path.  Step times alternating like
    # config 2's, then W of the Paul(4) transform
    c3 = wl.C3
    x3 = wl.config3_signal()
    for fam, code in (("dog", _engine.DOG), ("paul", _engine.PAUL)):
        p = c3[fam]
        s3 = wl.geometric_scales(p["s0"], p["dj"], p["J"])
        for name, eng in arms.items():
            d = eng.dev_alloc(x3.nbytes)
            eng.h2d(d, x3)
            eng.cwt_dev(d, 1, c3["n"], c3["dt"], s3, code, float(p["m"]), _engine.F32)
            eng.bench_last(10)
            launches[name] = eng.last_launch_count()
            dev[name] = d
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for name, eng in arms.items():
                times[name].append(eng.bench_last(20))
        for name, t in times.items():
            print("%-6s config 3 %-4s step %.4f ms (min %.4f, max %.4f), %d launches per step" % (
                name, fam, float(np.median(t)), min(t), max(t), launches[name]))
        for name, eng in arms.items():
            print("%s: serialised kernels of one config 3 %s step" % (name, fam))
            for k in sorted(eng.profile_last(), key=lambda k: -k["ms"]):
                print("      %-52s %3d x  %7.4f ms  rows %d" % (k["name"], k["launches"], k["ms"], k["rows"]))
            eng.dev_free(dev[name])
    print("config 3 Paul(4) W (fp32): %s" % ("bit-identical" if identical(
        arms, lambda e: e.cwt(x3, c3["dt"], s3, _engine.PAUL, float(p["m"]), _engine.F32)) else "DIFFERENT"))
    # config 4: xwt and wct, fp64 and fp32
    c4 = wl.C4
    y1, y2 = wl.config4_signals()
    s4 = wl.geometric_scales(c4["s0"], c4["dj"], c4["J"])
    klen = _boxcar_len(pycwt.Morlet(c4["f0"]), c4["dj"])
    for prec, pname in ((_engine.F64, "fp64"), (_engine.F32, "fp32")):
        ok_x = identical(arms, lambda e: e.xwt(y1, y2, c4["dt"], s4, _engine.MORLET, c4["f0"], prec))
        ok_w = identical(arms, lambda e: e.wct(y1, y2, c4["dt"], c4["dj"], s4, _engine.MORLET, c4["f0"], klen,
                                               True, prec))
        print("config 4 %s: xwt %s, wct %s" % (pname, "bit-identical" if ok_x else "DIFFERENT",
                                               "bit-identical" if ok_w else "DIFFERENT"))
    for eng in arms.values():
        eng.close()


if __name__ == "__main__":
    main()
