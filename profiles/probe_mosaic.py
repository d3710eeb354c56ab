"""Device time of the wavefield mosaic passes (sb_mosaic_*) per kernel slot and the GB/s each
pass achieves against the bytes it must move (chunks once, plus W, dspec, N where read).

    python profiles/probe_mosaic.py

Sizes: 16 x 16 chunks of 64 x 64 (the reference's unmodified fullMosHess took 1.1 s and
rotInit 66 ms on the CPU at this size, one run on the build host) and 127 x 127 chunks of
64 x 128 (a 4096 x 8192 spectrum in half-overlapping chunks).  One warm-up call, then the
minimum of 5 timed calls."""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


# the unmodified reference on the build host's CPU, one run each (see the docstring)
REF_CPU_MS = {(16, 16, 64, 64): dict(overlap=66.0, fit=99.0, hess=1100.0)}


def card():
    """Name, power limit and SM clocks of GPU 0, read in the same run (read-only query)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def main():
    import torch
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _lib
    from scintools_b200 import ththmod as T
    print("card: %s" % card(), flush=True)
    for ncf, nct, cwf, cwt in ((16, 16, 64, 64), (127, 127, 64, 128)):
        torch.cuda.empty_cache()
        rng = np.random.default_rng(0)
        ch = (rng.normal(size=(ncf, nct, cwf, cwt)).astype(np.float32) +
              1j * rng.normal(size=(ncf, nct, cwf, cwt)).astype(np.float32)).astype(np.complex64)
        P = ncf * nct
        nF, nT = (ncf - 1) * (cwf // 2) + cwf, (nct - 1) * (cwt // 2) + cwt
        D = rng.uniform(0, 4, (nF, nT)).astype(np.float32)
        m = T.MosaicModel(ch, D, np.ones_like(D))
        p = np.concatenate([rng.uniform(-3, 3, P - 1), np.ones(P)])
        chunk_b, w_b, d_b = ch.nbytes, nF * nT * 8, nF * nT * 4
        passes = dict(overlap=(lambda q: m.rot_init(), chunk_b),
                      build=(lambda q: m.full_mos(q), chunk_b + w_b),
                      fit=(lambda q: m.grad(q), chunk_b + w_b + 2 * d_b),
                      hess=(lambda q: m.hess(q, sparse=True), chunk_b + w_b + 2 * d_b))
        for name, (fn, nbytes) in passes.items():
            best = None
            for it in range(6):
                q = p + 1e-3 * it
                if name in ("fit", "hess"):
                    m.full_mos(q)           # W is built outside the timed pass
                torch.cuda.synchronize()
                _lib.lib.sb_profile_enable(1)
                fn(q)
                ms = np.zeros(16)
                cnt = np.zeros(16, np.int32)
                _lib.lib.sb_profile_collect(ms.ctypes.data, cnt.ctypes.data, 16)
                _lib.lib.sb_profile_enable(0)
                if it and (best is None or ms[10] + ms[11] < best[0] + best[1]):
                    best = (ms[10], ms[11])
            ref = REF_CPU_MS.get((ncf, nct, cwf, cwt), {}).get(name)
            print("%d x %d x %d x %d %-7s tile %.3f ms (%.0f GB/s)  reduce %.3f ms%s" %
                  (ncf, nct, cwf, cwt, name, best[0], nbytes / best[0] / 1e6, best[1],
                   "  (reference CPU %.0f ms)" % ref if ref else ""), flush=True)


if __name__ == "__main__":
    main()
