#!/usr/bin/env python
"""The NINO3 sea-surface-temperature analysis of Torrence & Compo (1998) with the H100
engine: the call sequence a pycwt user writes (cf. docs/tutorial of the reference), minus the
plotting.  Needs a CUDA device.

    python examples/nino3_tutorial.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pycwt_b200 as wavelet  # noqa: E402  (drop-in for `import pycwt as wavelet`)

dat = np.load(os.path.join(ROOT, "tests", "golden", "nino3_morlet_tutorial.npz"))["x"]
dt = 0.25                                   # years (seasonal data)
N = dat.size
p = np.polyfit(np.arange(N) * dt, dat, 1)   # detrend and normalise
dat_norm = (dat - np.polyval(p, np.arange(N) * dt))
std = dat_norm.std()
dat_norm = dat_norm / std

mother = wavelet.Morlet(6)
s0, dj, J = 2 * dt, 1 / 12, int(7 / (1 / 12))
alpha, _, _ = wavelet.ar1(dat)              # red-noise lag-1 autocorrelation

wave, scales, freqs, coi, fft, fftfreqs = wavelet.cwt(dat_norm, dt, dj, s0, J, mother)
iwave = wavelet.icwt(wave, scales, dt, dj, mother) * std
power = np.abs(wave) ** 2
period = 1 / freqs

signif, fft_theor = wavelet.significance(1.0, dt, scales, 0, alpha, significance_level=0.95,
                                         wavelet=mother)
sig95 = power / (np.ones([1, N]) * signif[:, None])

glbl_power = power.mean(axis=1)             # also available on the device: engine.global_power
dof = N - scales
glbl_signif, tmp = wavelet.significance(std ** 2, dt, scales, 1, alpha, significance_level=0.95,
                                        dof=dof, wavelet=mother)
sel = np.nonzero((period >= 2) & (period < 8))[0]
Cdelta = mother.cdelta
scale_avg = dj * dt / Cdelta * (power / scales[:, None])[sel, :].sum(axis=0)
scale_avg_signif, tmp = wavelet.significance(std ** 2, dt, scales, 2, alpha, significance_level=0.95,
                                             dof=[scales[sel[0]], scales[sel[-1]]], wavelet=mother)

print("NINO3 SST: N=%d, dt=%.2f yr, AR(1) alpha=%.3f" % (N, dt, alpha))
print("transform %s scales x %d points; period range %.2f .. %.1f yr" % (wave.shape[0], N, period[0], period[-1]))
print("reconstruction rms error / std: %.3f" % (np.sqrt(np.mean((np.real(iwave) - dat_norm * std) ** 2)) / std))
print("fraction of the scalogram above the 95%% red-noise level: %.3f" % (sig95 > 1).mean())
print("peak of the global wavelet spectrum at period %.2f yr" % period[np.argmax(glbl_power)])
print("2-8 yr scale-averaged variance: max %.3f degC^2, 95%% level %.3f" % (std ** 2 * scale_avg.max(), scale_avg_signif))
eng = wavelet.default_engine()
print("engine: %s, kernels of the cwt call above: %d launches" % (eng.version(), eng.last_launch_count()))

# The same products without moving the coefficient array to the host (an extension of this engine):
r = wavelet.cwt_resident(dat_norm, dt, dj, s0, J, mother)
assert np.allclose(r.global_power(), glbl_power, rtol=1e-12)
assert np.allclose(r.scale_avg_power(2, 8), scale_avg, rtol=1e-12)
assert np.allclose(r.icwt() * std, iwave, rtol=1e-12, atol=1e-12)
print("device-resident handle: global spectrum, 2-8 yr average and reconstruction agree with the "
      "host arithmetic; inside-COI global spectrum peak at %.2f yr"
      % period[np.nanargmax(r.global_power(inside_coi=True))])
