"""Time of the biharmonic gap fill (dynspec.inpaint_biharmonic, sb_inpaint_biharmonic_f64)
and of the masked median, with the card read in the same run, against the oracle's
spsolve on the CPU.

    python profiles/probe_refill.py [--no-oracle]

Cases (seeded):
  1024 x 2048  5 % random pixels, 16 zapped channels, a 64 x 256 block
  4096 x 8192  5 % random pixels, 4 channels, 4 sub-integrations, a 64 x 256 block
               (about 1.7 M unknowns)
Data: a smooth field sin(i / 150) cos(j / 230) plus 1e-3 noise.  One warm-up call, then 3
timed calls (CUDA events around the whole solve, including the host reads every 32
steps); the iteration count, restarts and final relative residual of each; the masked
median (5 x 5) at the same pixels.  The oracle's spsolve (SuperLU, one process) runs once
at 1024 x 2048, and the two results are compared, also for tol 1e-12 and 1e-13."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    """Name, power limit and SM clocks of GPU 0, read in the same run (read-only query)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def case(nf, nt, frac, chans, subints, block, seed):
    rng = np.random.default_rng(seed)
    i = np.arange(nf)[:, None]
    j = np.arange(nt)[None, :]
    img = np.sin(i / 150.0) * np.cos(j / 230.0) + 1e-3 * rng.normal(size=(nf, nt))
    mask = rng.random((nf, nt)) < frac
    mask[chans, :] = True
    mask[:, subints] = True
    r0, c0 = block
    mask[r0:r0 + 64, c0:c0 + 256] = True
    img[mask] = np.nan
    return img, mask


def main():
    import torch
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import dynspec
    print("card: %s" % card(), flush=True)
    rng = np.random.default_rng(1)
    cases = {
        "1024 x 2048": case(1024, 2048, 0.05, np.sort(rng.choice(1024, 16, replace=False)), [],
                            (400, 900), 2),
        "4096 x 8192": case(4096, 8192, 0.05, [100, 101, 2000, 4095], [0, 3000, 3001, 6000],
                            (1000, 5000), 3),
    }
    got = {}
    for name, (img, mask) in cases.items():
        dynspec.inpaint_biharmonic(img, mask)
        rows = []
        for _ in range(3):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            out, info = dynspec.inpaint_biharmonic(img, mask, return_info=True)
            b.record()
            torch.cuda.synchronize()
            rows.append(a.elapsed_time(b))
        got[name] = out
        meanval = float(np.mean(img[np.isfinite(img)]))
        dynspec._median_values(img, mask, (5, 5), meanval)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dynspec._median_values(img, mask, (5, 5), meanval)
        torch.cuda.synchronize()
        tm = (time.perf_counter() - t0) * 1e3
        print("%s: %d unknowns; biharmonic min %.1f / median %.1f ms (call incl. upload), "
              "%d iterations, %d restarts, residual %.2e; median 5x5 %.1f ms"
              % (name, mask.sum(), min(rows), float(np.median(rows)), info["iterations"],
                 info["restarts"], info["residual"], tm), flush=True)
    if "--no-oracle" not in sys.argv:
        from oracle import refill_oracle as O
        img, mask = cases["1024 x 2048"]
        t0 = time.perf_counter()
        ref = O.biharmonic(img, mask)
        ts = time.perf_counter() - t0
        known = img[~mask]
        err = np.max(np.abs(got["1024 x 2048"] - ref)) / (known.max() - known.min())
        print("1024 x 2048: oracle (assembly + spsolve, CPU) %.1f s; max |gpu - oracle| "
              "%.2e of the known range" % (ts, err), flush=True)
        for tol in (1e-12, 1e-13):
            out, info = dynspec.inpaint_biharmonic(img, mask, return_info=True, tol=tol)
            err = np.max(np.abs(out - ref)) / (known.max() - known.min())
            print("1024 x 2048, tol %.0e: %d iterations, %d restarts, residual %.2e, converged "
                  "%s; max |gpu - oracle| %.2e of the known range"
                  % (tol, info["iterations"], info["restarts"], info["residual"],
                     info["converged"], err), flush=True)


if __name__ == "__main__":
    main()
