"""Per-kernel device times of the paths bench.py's headline does not cover: wct / xwt / Monte-Carlo
pair (config 4 geometry), resident reductions (config 2), fp32 configs.  One H100."""
import os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import workloads as wl
import pycwt_b200 as pycwt
from pycwt_b200 import _engine, wavelet as wv

eng = pycwt.default_engine()


def show(title, prof, note=""):
    tot = sum(k["ms"] for k in prof)
    print("== %s: %.3f ms in %d launches %s" % (title, tot, sum(k["launches"] for k in prof), note))
    for k in sorted(prof, key=lambda k: -k["ms"])[:14]:
        print("   %-46s %3d x %8.4f ms  rows %d" % (k["name"], k["launches"], k["ms"], k["rows"]))


c = wl.C4
y1, y2 = wl.config4_signals()
m = pycwt.Morlet(c["f0"])
pycwt.wct(y1, y2, c["dt"], c["dj"], c["s0"], c["J"], sig=False, wavelet=m)
eng.profile_begin()
pycwt.wct(y1, y2, c["dt"], c["dj"], c["s0"], c["J"], sig=False, wavelet=m)
show("wct(sig=False) N=2^18 S=145", eng.profile_end())
eng.profile_begin()
pycwt.xwt(y1, y2, c["dt"], c["dj"], c["s0"], c["J"], wavelet=m)
show("xwt N=2^18 S=145", eng.profile_end())
prob = wv._mc_problem(c["dt"], c["dj"], c["s0"], c["J"], m)
wv._mc_histogram_seeded(prob, c["dt"], c["dj"], m, 1, 0, 4)
eng.profile_begin()
wv._mc_histogram_seeded(prob, c["dt"], c["dj"], m, 1, 0, 8)
show("Monte-Carlo, 8 seeded pairs N=49152 S=145", eng.profile_end(), "(per pair: /8)")
t0 = time.perf_counter()
wv._mc_histogram_seeded(prob, c["dt"], c["dj"], m, 1, 0, 200)
t1 = time.perf_counter() - t0
np.random.seed(0)
t0 = time.perf_counter()
pycwt.wct_significance(0.3, 0.5, c["dt"], c["dj"], c["s0"], c["J"], wavelet=m, mc_count=200, progress=False, cache=False)
t2 = time.perf_counter() - t0
print("200 pairs: device RNG %.3f s, host RNG (reference order) %.3f s" % (t1, t2))

c2 = wl.C2
x = wl.config2_signal()
r = pycwt.cwt_resident(x, c2["dt"], c2["dj"], c2["s0"], c2["J"], pycwt.Morlet(6))
r.global_power(), r.scale_avg_power(2, 8), r.icwt()
for name, fn in (("global_power", r.global_power), ("scale_avg_power(2,8)", lambda: r.scale_avg_power(2, 8)),
                 ("scale_avg_power(all)", lambda: r.scale_avg_power(0, 1e9)), ("icwt", r.icwt)):
    eng.profile_begin()
    fn()
    p = eng.profile_end()
    t0 = time.perf_counter()
    fn()
    dt = time.perf_counter() - t0
    ms = sum(k["ms"] for k in p)
    print("resident %-22s kernels %.3f ms (%.0f GB/s of the 4.29 GB read), call %.3f ms" % (name, ms, 4.295 / ms * 1e3 if ms else 0, dt * 1e3))
