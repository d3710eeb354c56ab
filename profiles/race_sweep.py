"""Small eta sweep through the two eigen solvers (tensor-core default, fp32):
run under `compute-sanitizer --tool racecheck|memcheck`."""
import os
import sys
sys.path.insert(0, ".")
import numpy as np
from scintools_b200 import ththmod as thth
rng = np.random.default_rng(0)
nf, nt, npad = 32, 64, 1
d0 = rng.normal(size=(nf, nt)); d0 -= d0.mean()
t = np.arange(nt) * 10.0; f = 1400.0 + np.arange(nf) * 0.05
fd = thth.fft_axis(t, "mHz", npad); tau = thth.fft_axis(f, "us", npad)
edges = np.linspace(-20, 20, 96); etas = np.linspace(0.002, 0.02, 4)
cs = thth.conjugate_spectrum(d0, npad, 0.0)
print("tensor-core", thth.eta_sweep(cs, tau, fd, etas, edges))
os.environ["SB_EIG_FP32"] = "1"
print("fp32       ", thth.eta_sweep(cs, tau, fd, etas, edges))
