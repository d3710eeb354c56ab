"""Time of the theoretical intensity ACF (scint_sim.ACF, sb_acf_model_f64), with the card
read in the same run.

    python profiles/probe_acf_model.py [out.json]

Three cases: the example notebook's call (ar=2, psi=30, phasegrad=0.2), ar=4 with the same
angles, and ar=8 with nt = nf = 101.  For each, after one warm-up call:
  device   sb_acf_model_f64 alone on uploaded axes, CUDA events, median of 5
  call     ACF(...) end to end (host axes, uploads, the device call, downloads), host clock
           around a synchronised call, median of 5
and the float64 operations of the bilinear form from the shapes: per frequency column on
an n-point grid, 4 n^2 flops per lag for G ex (a real times a complex) and 8 n for ey^T.
The reference's times in the table are CPU times measured on a different machine (the
unmodified reference, numpy, one call per case)."""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CASES = [
    ("notebook", dict(psi=30, phasegrad=0.2, theta=0, ar=2, taumax=4, dnumax=4, nt=51, nf=51),
     2.0),
    ("ar4", dict(ar=4, psi=30, phasegrad=0.2), 14.6),
    ("ar8_101", dict(ar=8, psi=30, phasegrad=0.2, nt=101, nf=101), None),
]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def flops(n1, n2, nsn, ndnun):
    cols = [n2] + [n1] * (ndnun - 2)
    return sum(4.0 * n * n * nsn + 8.0 * n * nsn for n in cols)


def main():
    import torch
    from scintools_b200 import _device as D
    from scintools_b200 import _lib
    from scintools_b200.scint_sim import ACF
    out = {"card": card(), "cases": []}
    print("card:", out["card"])
    for name, kw, ref_s in CASES:
        a = ACF(**kw)                                   # warm-up, and the object for the axes
        h = a._axes()
        d = [D.upload(np.ascontiguousarray(h[k], dtype=np.float64))
             for k in ("snp", "snp2", "dnun", "snx", "sny")]
        n1, n2, nd, nsn = len(h["snp"]), len(h["snp2"]), len(h["dnun"]), len(h["snx"])
        m = _lib.AcfModel(*[t.data_ptr() for t in d], n1, n2, nd, nsn, int(h["quadrant"]),
                          h["sigxn"], h["sigyn"], h["sqrtar"], float(h["alph2"]),
                          float(h["step1"]), float(h["step2"]), h["wn_amp"], h["amp"])
        acf = D.empty(a.acf.shape, torch.float64)
        ef = D.empty((n1, n1), torch.float64)
        dev = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(_lib.lib.sb_acf_model_f64(m, acf.data_ptr(), ef.data_ptr(),
                                                  D.stream_ptr()))
            e1.record()
            torch.cuda.synchronize()
            dev.append(e0.elapsed_time(e1) / 1e3)
        assert np.array_equal(acf.cpu().numpy(), a.acf)
        call = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ACF(**kw)
            torch.cuda.synchronize()
            call.append(time.perf_counter() - t0)
        f = flops(n1, n2, nsn, nd)
        r = dict(name=name, kwargs=kw, grid_main=n1, grid_core=n2, lags=nsn, columns=nd,
                 acf_shape=list(a.acf.shape), flops=f, device_s=float(np.median(dev)),
                 call_s=float(np.median(call)), gflops=f / float(np.median(dev)) / 1e9,
                 reference_cpu_s_other_machine=ref_s)
        out["cases"].append(r)
        print("%-9s grid %5d / %5d  lags %3d x %3d  %.2e flop  device %.4f s (%.0f GFLOP/s)  "
              "call %.4f s  reference CPU (other machine) %s s" % (
                  name, n1, n2, nsn, nd, f, r["device_s"], r["gflops"], r["call_s"], ref_s))
    fn = sys.argv[1] if len(sys.argv) > 1 else None
    if fn:
        os.makedirs(os.path.dirname(os.path.abspath(fn)), exist_ok=True)
        with open(fn, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
