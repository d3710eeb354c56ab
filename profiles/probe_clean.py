"""Time of Dynspec.zap and Dynspec.trim_edges (csrc/clean.cu) at 4096 x 8192, with the card
read in the same run, against the reference's numpy statements on the CPU.

    python profiles/probe_clean.py [--reps N]

Data (seeded): an exponential spectrum with two zero bands (300 and 170 channels), five
NaN sub-integrations, 1 % NaN and 20 % zero pixels, and 0.1 % pixels 100 times brighter.
Each call is timed end to end with a host clock and a device synchronise, transfers
included (upload, the kernels, the download), after one warm-up call; the device part of
zap alone (sb_zap_f64 on a resident copy) with CUDA events.  The numpy restatements are the
reference's own statements (dynspec.py:3867-3870 for zap; for trim_edges the NaN fill and
its one-row-at-a-time np.delete loops, dynspec.py:271-328).  Every result is compared
with numpy's, bit for bit."""
import argparse
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


def spectrum(nf=4096, nt=8192):
    rng = np.random.default_rng(2024)
    dyn = rng.exponential(1.0, (nf, nt))
    dyn[:300] = 0.0
    dyn[-170:] = 0.0
    dyn[:, :5] = np.nan
    dyn[rng.random((nf, nt)) < 0.01] = np.nan
    dyn[rng.random((nf, nt)) < 0.2] = 0.0
    hot = rng.random((nf, nt)) < 1e-3
    dyn[hot] *= 100.0
    return dyn


def np_zap(x, sigma):
    with np.errstate(all="ignore"):
        d = np.abs(x - np.median(x[~np.isnan(x)]))
        mdev = np.median(d[~np.isnan(d)])
        x[d / mdev > sigma] = np.nan


def np_trim(dyn, frac=0.5):
    """dynspec.py:271-318, the array part (freqs / times deletions left out)"""
    dyn[np.isnan(dyn)] = 0
    nc, nr = dyn.shape[1], dyn.shape[0]
    while len(np.argwhere(dyn[0, :] == 0)) > frac * nc or sum(abs(dyn[0, :])) == 0:
        dyn = np.delete(dyn, 0, axis=0)
    while len(np.argwhere(dyn[-1, :] == 0)) > frac * nc or sum(abs(dyn[-1, :])) == 0:
        dyn = np.delete(dyn, -1, axis=0)
    while len(np.argwhere(dyn[:, 0] == 0)) > frac * nr or sum(abs(dyn[:, 0])) == 0:
        dyn = np.delete(dyn, 0, axis=1)
    while len(np.argwhere(dyn[:, -1] == 0)) > frac * nr or sum(abs(dyn[:, -1])) == 0:
        dyn = np.delete(dyn, -1, axis=1)
    return dyn


def timed(fn, reps):
    import torch
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _device as D
    from scintools_b200 import _lib
    from scintools_b200.dynspec import BasicDyn, Dynspec
    print("card: %s" % card(), flush=True)
    dyn = spectrum()
    nf, nt = dyn.shape

    def ds_of(a):
        return Dynspec(dyn=BasicDyn(a, times=10.0 * np.arange(nt),
                                    freqs=1000.0 + 0.1 * np.arange(nf)), verbose=False)

    # zap, end to end
    ds = ds_of(dyn.copy())
    ds.zap()                                   # warm-up
    copies = [dyn.copy() for _ in range(args.reps)]
    objs = [ds_of(c) for c in copies]
    it = iter(objs)
    t_zap = timed(lambda: next(it).zap(), args.reps)
    ref = dyn.copy()
    t0 = time.perf_counter()
    np_zap(ref, 7)
    t_np_zap = time.perf_counter() - t0
    same = np.array_equal(objs[0].dyn, ref, equal_nan=True)
    print("zap 4096 x 8192, end to end: median %.2f ms (min %.2f) over %d; numpy %.0f ms; "
          "equal: %s" % (1e3 * np.median(t_zap), 1e3 * min(t_zap), args.reps, 1e3 * t_np_zap,
                         same), flush=True)
    # zap, device only (the mask of a repeated call is the same, the work is the same)
    d = D.upload(dyn)
    st = D.empty((2,), torch.float64)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    dev = []
    for _ in range(args.reps + 1):
        x = d.clone()
        ev[0].record()
        _lib.check(_lib.lib.sb_zap_f64(x.data_ptr(), x.numel(), 7.0, st.data_ptr(),
                                       D.stream_ptr()))
        ev[1].record()
        torch.cuda.synchronize()
        dev.append(ev[0].elapsed_time(ev[1]))
    dev = dev[1:]
    print("sb_zap_f64 device time: median %.3f ms (min %.3f); one read of the %.2f GB array "
          "takes %.3f ms at the data sheet's 3.35 TB/s" % (np.median(dev), min(dev),
                                                          dyn.nbytes / 1e9,
                                                          dyn.nbytes / 3.35e12 * 1e3),
          flush=True)
    # trim_edges, end to end
    ds = ds_of(dyn.copy())
    ds.trim_edges()
    objs = [ds_of(dyn.copy()) for _ in range(args.reps)]
    it = iter(objs)
    t_trim = timed(lambda: next(it).trim_edges(), args.reps)
    a = dyn.copy()
    t0 = time.perf_counter()
    ref = np_trim(a)
    t_np_trim = time.perf_counter() - t0
    same = np.array_equal(objs[0].dyn, ref)
    print("trim_edges 4096 x 8192, end to end: median %.2f ms (min %.2f) over %d; numpy %.0f "
          "ms; kept %s; equal: %s" % (1e3 * np.median(t_trim), 1e3 * min(t_trim), args.reps,
                                      1e3 * t_np_trim, ref.shape, same), flush=True)


if __name__ == "__main__":
    main()
