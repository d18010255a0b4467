"""Timeline of one config 2 step: when the coarse chain of the expansion rows runs, and when the
expansion kernels start.

    python profiles/micro/coarse_timeline.py [OUT_DIR] [--lib PATH]

Runs config 2 (Morlet(6), N = 2^20, 256 scales, fp64) with warm-up, then captures one step
(`bench_last(1)`) under torch.profiler with CUDA activities: CUPTI records the kernels the engine
library launches through ctypes like any other.  Writes the Chrome trace to OUT_DIR (default: a
coarse_timeline directory under the system's temporary directory) and prints the card, its power
limit and max SM clock, then per stream: the span of its kernels, the coarse-chain kernels on it,
the idle gaps; and for the step: the
start and end of the coarse chain, the start of the first expansion launch, and how long the
coarse kernels overlap the overlap-save and dense launches.  Times are in ms from the first kernel
of the step."""
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import workloads as wl          # noqa: E402
from pycwt_b200 import _engine  # noqa: E402


def kind(name):
    """coarse | expand | os | dense | fwd | other, from the kernel's (demangled) name."""
    n = name.replace("cwtb::", "")
    if re.search(r"ExpandBandBody|RowsBody|Coarse", n):
        return "coarse"
    if re.search(r"Expand(Mma)?Body", n):
        return "expand"
    if "OsBody" in n:
        return "os"
    if re.search(r"PassABody<double, \d+, 3, 1>|PassABody<float, \d+, 3, 1>", n):
        return "coarse"
    if re.search(r"PassABody<\w+, \d+, 2, -1>|PassBBody<\w+, -1", n):
        return "fwd"
    if re.search(r"PassABody|PassBBody|BandBody", n):
        return "dense"
    return "other"


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    lib = None
    if "--lib" in sys.argv:
        lib = sys.argv[sys.argv.index("--lib") + 1]
        args = [a for a in args if a != lib]
    out_dir = args[0] if args else os.path.join(tempfile.gettempdir(), "coarse_timeline")
    os.makedirs(out_dir, exist_ok=True)
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.zeros(1, device="cuda")
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip())
    c = wl.C2
    x = wl.config2_signal()
    sj = wl.config2_scales()
    eng = _engine.Engine(0, lib_path=lib)
    d = eng.dev_alloc(x.nbytes)
    eng.h2d(d, x)
    eng.cwt_dev(d, 0, c["n"], c["dt"], sj, _engine.MORLET, c["f0"], _engine.F64)
    eng.bench_last(10)
    print("step %.4f ms (bench_last(20), profiler off), %d launches per step"
          % (eng.bench_last(20), eng.last_launch_count()))
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.bench_last(1)
        eng.sync()
    path = os.path.join(out_dir, "coarse_timeline.pt.trace.json")
    prof.export_chrome_trace(path)
    eng.dev_free(d)
    eng.close()

    with open(path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    t0 = ev[0]["ts"]
    k = [(kind(e["name"]), e["args"].get("stream"), (e["ts"] - t0) / 1e3, (e["ts"] + e["dur"] - t0) / 1e3,
          e["name"]) for e in ev]
    end = max(e for _, _, _, e, _ in k)
    print("step span in the trace: %.3f ms, %d kernels" % (end, len(k)))
    coarse_streams = sorted({s for kd, s, _, _, _ in k if kd == "coarse"})
    for s in sorted({s for _, s, _, _, _ in k}):
        ks = [r for r in k if r[1] == s]
        gaps = [b[2] - a[3] for a, b in zip(ks, ks[1:]) if b[2] > a[3]]
        kinds = {}
        for r in ks:
            kinds[r[0]] = kinds.get(r[0], 0) + 1
        print("stream %-4s %3d kernels %-40s %.3f .. %.3f ms, busy %.3f ms, idle gaps %d totalling %.3f ms "
              "(largest %.3f)" % (s, len(ks), kinds, ks[0][2], ks[-1][3], sum(r[3] - r[2] for r in ks),
                                  len(gaps), sum(gaps), max(gaps) if gaps else 0.0))
        if s in coarse_streams:
            for r in ks:
                print("      %-7s %.3f .. %.3f  %s" % (r[0], r[2], r[3], r[4][:110]))
    co = [r for r in k if r[0] == "coarse"]
    # coarse PassB launches share the dense kernels' name: those on the coarse streams belong to it
    co += [r for r in k if r[0] == "dense" and r[1] in coarse_streams and "PassBBody" in r[4]]
    ex = [r for r in k if r[0] == "expand"]
    if co:
        print("coarse chain: %d kernels, %.3f .. %.3f ms, %.3f ms of kernel time"
              % (len(co), min(r[2] for r in co), max(r[3] for r in co), sum(r[3] - r[2] for r in co)))
    if ex:
        print("first expansion launch starts at %.3f ms; expansion launches end at %.3f ms"
              % (min(r[2] for r in ex), max(r[3] for r in ex)))
    other = [r for r in k if r[0] in ("os", "dense") and r[1] not in coarse_streams]

    def overlap(a, b):
        return max(0.0, min(a[3], b[3]) - max(a[2], b[2]))
    print("coarse kernels overlapping overlap-save / dense launches: %.3f ms (sum over pairs)"
          % sum(overlap(a, b) for a in co for b in other))


if __name__ == "__main__":
    main()
