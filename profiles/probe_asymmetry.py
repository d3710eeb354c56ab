"""Arc asymmetry (Dynspec.calc_asymmetry): device time (CUDA events from the first
conjugate spectrum to the end of the last sb_asymmetry_batch, after warm-up) and call wall
time of the batched call, the same for a Python loop of ththmod.calc_asymmetry over the
same chunks, and library launches per chunk, on two workloads:
  a      the tutorial field of tests/golden/asymmetry_sample.npz (1024 x 128), cwf = 64,
         cwt = 32: 16 x 4 chunks of widths 32 / 48 / 64 / 80;
  large  that field tiled to 8192 x 600, cwf = 64, cwt = 100: 128 x 6 chunks of widths
         100 .. 350 (the reference's growing time slice).
Both use 302 edges out to 0.3 mHz, npad = 3 and ththeta = 40 s^3.  Prints the card's name
and power limit and one JSON line."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from scintools_b200 import _device as D, _lib, ththmod as thth  # noqa: E402
from scintools_b200.dynspec import BasicDyn, Dynspec  # noqa: E402


def dynspec(dyn, freqs, times, cwf, cwt, edges, ththeta=40.0, npad=3):
    ds = Dynspec(dyn=BasicDyn(dyn, times=times, freqs=freqs), verbose=False)
    ds.cwf, ds.cwt, ds.npad = cwf, cwt, npad
    ds.ncf_fit, ds.nct_fit = dyn.shape[0] // cwf, dyn.shape[1] // cwt
    ds.fref, ds.edges, ds.ththeta = float(freqs.mean()), edges, ththeta
    return ds


def case_a(f):
    return dynspec(f["dyn"].astype(np.float64), f["freqs"], f["times"], 64, 32, f["edges"])


def case_large(f):
    dyn = np.tile(f["dyn"].astype(np.float64), (8, 5))[:, :600]
    freqs = f["freqs"][0] + (f["freqs"][1] - f["freqs"][0]) * np.arange(dyn.shape[0])
    times = (f["times"][1] - f["times"][0]) * np.arange(dyn.shape[1])
    return dynspec(dyn, freqs, times, 64, 100, f["edges"])


def device_span(run):
    """Milliseconds between events recorded before the first sb_cs_f32 and after the last
    sb_asymmetry_batch of run()."""
    lib = _lib.lib
    cs_orig, ab_orig = lib.sb_cs_f32, lib.sb_asymmetry_batch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    first = [True]

    def cs(*args):
        if first[0]:
            a.record()
            first[0] = False
        return cs_orig(*args)

    def ab(*args):
        rc = ab_orig(*args)
        b.record()
        return rc
    lib.sb_cs_f32, lib.sb_asymmetry_batch = cs, ab
    try:
        run()
    finally:
        lib.sb_cs_f32, lib.sb_asymmetry_batch = cs_orig, ab_orig
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def measure(name, ds, reps=5):
    pars = ds._asymmetry_params()
    nchunk = len(pars)
    runs = {"batched": lambda: ds.calc_asymmetry(),
            "loop": lambda: [thth.calc_asymmetry(p) for p in pars]}
    out = {"case": name, "chunks": [ds.ncf_fit, ds.nct_fit], "n_th": int(len(ds.edges) - 1),
           "widths": sorted({p[0].shape[1] for p in pars})}
    for key, run in runs.items():
        run()
        torch.cuda.synchronize()
        n0 = _lib.lib.sb_launch_count()
        run()
        torch.cuda.synchronize()
        out[key + "_launches_per_chunk"] = (_lib.lib.sb_launch_count() - n0) / nchunk
        dev = sorted(device_span(run) for _ in range(reps))
        t0 = time.perf_counter()
        for _ in range(reps):
            run()
        torch.cuda.synchronize()
        out[key + "_device_ms_min"] = dev[0]
        out[key + "_device_ms_median"] = dev[len(dev) // 2]
        out[key + "_call_wall_ms"] = (time.perf_counter() - t0) * 1e3 / reps
    a = np.array([r[0] for r in thth.asymmetry_batch(pars)])
    b = np.array([thth.calc_asymmetry(p)[0] for p in pars])
    out["loop_equals_batched"] = bool(np.array_equal(a, b, equal_nan=True))
    return out


def main():
    D.device()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q, flush=True)
    f = np.load(os.path.join(ROOT, "tests", "golden", "asymmetry_sample.npz"))
    out = {"gpu": q, "results": [measure("a", case_a(f)), measure("large", case_large(f))]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
