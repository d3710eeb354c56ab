"""Error of the default (fp16-iterate on the tensor cores + fp32 Rayleigh quotient) eigen
solver against the fp32 solver (SB_EIG_FP32=1, itself within 6e-7 of ARPACK) on all 1024
curvatures of the bench workload, with the iteration counts.  Run on the GPU box."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import bench
from scintools_b200 import ththmod as thth

dyn, freq, t = bench.make_dynspec()
fd = np.asarray(thth.fft_axis(t, "mHz", bench.NPAD)); tau = np.asarray(thth.fft_axis(freq, "us", bench.NPAD))
edges = np.linspace(-bench.EDGE_LIM, bench.EDGE_LIM, bench.NEDGE)
etas = bench.eta_grid(bench.NETA)
cs = thth.conjugate_spectrum(dyn, bench.NPAD, 0.0, ncols_keep=thth.needed_fd_columns(fd, edges))
os.environ["SB_EIG_FP32"] = "1"
ref, iref = thth.eta_sweep(cs, tau, fd, etas, edges, return_info=True)
del os.environ["SB_EIG_FP32"]
out = {"fp32_iters_mean": float(iref["iters"].mean())}
for label, env in (("default", {}), ("rtol5e4", {"SB_EIG_RTOL_R": "5e-4"}),
                   ("etol5e7", {"SB_EIG_ETOL_B": "5e-7"})):
    os.environ.update(env)
    got, info = thth.eta_sweep(cs, tau, fd, etas, edges, return_info=True)
    for k in env: del os.environ[k]
    rel = np.abs(got - ref) / ref
    it = info["iters"]
    w = np.argsort(rel)[-5:][::-1]
    out[label] = {"max": float(rel.max()), "p99": float(np.percentile(rel, 99)), "median": float(np.median(rel)),
                  "iters_mean": float(it.mean()), "iters_gt24": int((it > 24).sum()),
                  "worst": [(int(i), float(rel[i]), int(it[i]), int(iref["iters"][i])) for i in w]}
print(json.dumps(out))
