"""Config 2: step time and error for pruning / expansion tolerances.  The error is
max|W - W_default| / max|W_default| against the default tolerances (1e-16, 5e-13), whose result
agrees with the oracle to 4.7e-14 on every row (tests/test_gpu_fullsize.py); the widest-band
mode (band_eps = 0, expansion off) is listed with its worst rows."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import workloads as wl          # noqa: E402
from pycwt_b200 import _engine  # noqa: E402


def main():
    c = wl.C2
    sj = wl.config2_scales()
    x = wl.config2_signal()
    eng = _engine.Engine(0)
    dsig = eng.dev_alloc(x.nbytes)
    eng.h2d(dsig, x)

    def run(beps, xeps):
        eng.set_band_eps(beps)
        eng.set_expand_eps(xeps, 2e-7)
        eng.cwt_dev(dsig, 0, c["n"], c["dt"], sj, _engine.MORLET, c["f0"], _engine.F64)
        eng.bench_last(3)
        ms = eng.bench_last(20)
        return ms, eng.get_w(len(sj), c["n"])

    ms0, W0 = run(1e-16, 5e-13)
    W0 = W0.copy()
    scale = np.abs(W0).max()
    msx, Wx = run(0.0, 0.0)
    rows = np.array([float(np.abs(Wx[r] - W0[r]).max()) for r in range(len(sj))]) / scale
    worst = np.argsort(rows)[::-1][:6]
    print("band_eps 0, expansion off: %.3f ms; worst rows vs default: %s" % (
        msx, ", ".join("%d: %.2e" % (r, rows[r]) for r in worst)))
    print("plan of those rows:", [eng.last_plan(len(sj))[r] for r in worst])
    del Wx
    for beps, xeps in ((1e-15, 5e-13), (1e-14, 5e-13), (1e-14, 5e-12), (1e-13, 5e-12),
                       (1e-13, 5e-11), (1e-12, 5e-11)):
        ms, W = run(beps, xeps)
        err = 0.0
        for r0 in range(0, len(sj), 32):
            err = max(err, float(np.abs(W[r0:r0 + 32] - W0[r0:r0 + 32]).max()))
        plan = eng.last_plan(len(sj))
        nexp = int((np.asarray(plan) < 0).sum())
        ndense = int((np.asarray(plan) == 20).sum())
        print("band_eps %.0e expand_eps %.0e: %.4f ms  err %.2e  (expansion rows %d, dense rows %d)"
              % (beps, xeps, ms, err / scale, nexp, ndense))
        del W
    eng.dev_free(dsig)


if __name__ == "__main__":
    main()
