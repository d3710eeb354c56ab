"""Time of the brightness model (scint_sim.Brightness, sb_brightness_f64) at its default
size (600^2 lattice, 2000 x 1000 secondary spectrum), with the card read in the same run.

    python profiles/probe_brightness.py [out.json]

  device   sb_brightness_f64 for one set and for a batch of 64, CUDA events around each
           library call (after a warm-up), summed over the batch's memory groups, median of
           3; per set = time / sets
  dft      the float64 matrix-product kernels (br_gemm_kernel) of the batch of 64, summed
           from torch.profiler in a separate run, and their FLOP/s from the shapes: per set
           12 n^3 for B (a complex times a real, then a complex times a complex, real
           multiply-adds counted as 2) and 4 ntd^2 nfd + 4 ntd nfd^2 for the ACF
  call     Brightness(...) and brightness_batch end to end, host clock, once each
The first brightness_batch of a lattice also triangulates it on the host (seconds); the
warm-up call pays that."""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def main(out_path):
    import torch
    from scintools_b200 import _lib
    from scintools_b200 import scint_sim as S
    rng = np.random.default_rng(0)
    sets = [dict(ar=float(rng.uniform(1, 4)), psi=float(rng.uniform(-90, 90)))
            for _ in range(64)]
    times = []
    lib = _lib.lib
    real = lib.sb_brightness_f64

    class Timed:
        def sb_brightness_f64(self, m, stream):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            rc = real(m, stream)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
            return rc

        def __getattr__(self, name):
            return getattr(lib, name)
    S._lib.lib = Timed()
    res = {"card": card()}
    try:
        S.brightness_batch(sets[:2])                       # warm-up, triangulation
        for label, batch in (("one", sets[:1]), ("batch64", sets)):
            per_call = []
            for _ in range(3):
                times.clear()
                S.brightness_batch(batch)              # groups of at most 4 GiB: summed
                per_call.append(sum(times))
            ms = float(np.median(per_call))
            res[label] = dict(sets=len(batch), device_ms=ms, per_set_ms=ms / len(batch))
            print(label, res[label], flush=True)
    finally:
        S._lib.lib = lib
    t0 = time.perf_counter()
    S.Brightness()
    res["call_one_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    S.brightness_batch(sets)
    res["call_batch64_s"] = time.perf_counter() - t0
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        S.brightness_batch(sets)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "br_gemm_kernel" in e.key)
    n, ntd, nfd = 600, 2000, 1000
    flop = 64 * (12 * n ** 3 + 4 * ntd ** 2 * nfd + 4 * ntd * nfd ** 2)
    res["dft"] = dict(kernel_ms=us / 1e3, flop=flop, tflops=flop / (us * 1e-6) / 1e12)
    res["kernels_us"] = {e.key: e.device_time_total for e in prof.key_averages()
                         if e.key.startswith("void sb::br_")}
    print(json.dumps(res, indent=1))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
