"""Chi-square curvature search (ththmod.chisq_sweep / chisq_calc): device time of
one chisq_sweep (CUDA events, after warm-up), the per-curvature chisq_calc loop
end to end, and one CPU core running the numpy oracle (oracle/chisq_oracle.py),
on two workloads:
  a     THTHSample.ipynb cell 40: 64 x 150 tutorial chunk, CS 256 x 600 (chirp-z),
        511 theta centres, 100 curvatures (tests/golden/thth_sample_64x150.npz);
  large 256 x 1024 synthetic chunk, CS 1024 x 4096 (radix), 1023 theta centres,
        8 curvatures (the large case of tests/test_gpu_chisq.py).
The oracle is timed on a subset of the curvatures and reported per curvature.
Prints the card's name and power limit and one JSON line."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from threadpoolctl import threadpool_limits  # noqa: E402

from oracle import chisq_oracle as CO  # noqa: E402
from oracle import thth_oracle as TO  # noqa: E402
from scintools_b200 import _device as D, ththmod as thth  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def case_a():
    g = np.load(os.path.join(ROOT, "tests", "golden", "thth_sample_64x150.npz"))
    d2 = g["dspec2"]
    CS = TO.conjugate_spectrum(d2 - d2.mean(), 3, 0.0)
    return d2, CS, g["tau"], g["fd"], np.linspace(12.5, 100.0, 100), np.linspace(-0.4, 0.4, 512)


def case_large():
    rng = np.random.default_rng(2024)
    nf, nt, npad = 256, 1024, 3
    t = np.arange(nt) * 10.0
    f = 1400.0 + np.arange(nf) * 0.05
    fdk = rng.uniform(-20, 20, 60)
    ak = (rng.normal(size=60) + 1j * rng.normal(size=60)) * np.exp(-(fdk / 10) ** 2)
    E = sum(a * np.exp(2j * np.pi * (fd_ * 1e-3 * t[None, :] - 0.01 * fd_ ** 2 * (f[:, None] - f[0])))
            for a, fd_ in zip(ak, fdk))
    dyn = np.abs(E) ** 2 + rng.normal(0, 0.05, (nf, nt))
    CS = TO.conjugate_spectrum(dyn - dyn.mean(), npad, 0.0)
    return (dyn, CS, TO.fft_axis(f, "us", npad), TO.fft_axis(t, "mHz", npad),
            np.linspace(0.006, 0.014, 8), np.linspace(-20.0, 20.0, 1024))


def measure(name, dspec, CS, tau, fd, etas, edges, n_oracle, reps=5):
    cs = thth.DeviceCS.from_numpy(CS)             # resident: the CS upload is not timed
    run = lambda: thth.chisq_sweep(dspec, cs, tau, fd, etas, edges, 1.0)   # noqa: E731
    run()
    run()
    torch.cuda.synchronize()
    # device time: events around the library call on the current stream (the host-side
    # rev_map centres and uploads happen before the first event is waited on)
    ev = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        orig = thth._lib.lib.sb_chisq_sweep

        def timed(*args, _o=orig, _a=a, _b=b):
            _a.record()
            rc = _o(*args)
            _b.record()
            return rc
        thth._lib.lib.sb_chisq_sweep = timed
        try:
            run()
        finally:
            thth._lib.lib.sb_chisq_sweep = orig
        ev.append((a, b))
    torch.cuda.synchronize()
    dev_ms = sorted(a.elapsed_time(b) for a, b in ev)
    t0 = time.perf_counter()
    for _ in range(reps):
        run()
    torch.cuda.synchronize()
    sweep_wall = (time.perf_counter() - t0) * 1e3 / reps
    t0 = time.perf_counter()
    for e in etas:
        thth.chisq_calc(dspec, cs, tau, fd, e, edges, 1.0)
    torch.cuda.synchronize()
    loop_ms = (time.perf_counter() - t0) * 1e3
    sub = etas[:: max(1, len(etas) // n_oracle)][:n_oracle]
    with threadpool_limits(limits=1):
        t0 = time.perf_counter()
        for e in sub:
            CO.chisq_calc(dspec, CS, tau, fd, e, edges, 1.0)
        cpu_per = (time.perf_counter() - t0) * 1e3 / len(sub)
    return {"case": name, "neta": int(len(etas)), "cs": list(CS.shape),
            "n_th": int(len(edges) - 1),
            "sweep_device_ms_min": dev_ms[0], "sweep_device_ms_median": dev_ms[len(dev_ms) // 2],
            "sweep_wall_ms": sweep_wall, "chisq_calc_loop_ms": loop_ms,
            "oracle_1core_ms_per_eta": cpu_per,
            "oracle_1core_ms_est": cpu_per * len(etas)}


def main():
    D.device()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q, flush=True)
    out = {"gpu": q, "results": [measure("a", *case_a(), n_oracle=10),
                                 measure("large", *case_large(), n_oracle=2)]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
