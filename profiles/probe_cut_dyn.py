"""Dynspec.cut_dyn (one batched pass: sb_sspec_tiles_f32 + sb_acf_tiles_f32) against the
per-tile loop it replaces (calc_sspec(input_dyn=tile) + calc_acf(input_dyn=tile) for every
tile), with the card read in the same run.

    python profiles/probe_cut_dyn.py [--out DIR]

Cases (seeded exponential fields, float32 on the host, dtype=np.float32 outputs):
  4096 x 8192    8 x 8 tiles of 512 x 1024   (tcuts = fcuts = 7)
  1024 x 2048   32 x 32 tiles of 32 x 64     (tcuts = fcuts = 31)
  16384 x 32768  2 x 2 tiles of 8192 x 16384 (tcuts = fcuts = 1; large tiles)
Both ways are first checked against each other on every tile (secondary spectra: linear
relative error < 1e-5 and < 2e-4 dB on bins above 1e-3 of the maximum; ACFs: < 1e-5), then
timed end to end (host clock around calls that end in a device synchronise, downloads
included) after one warm-up call each: best of 3 (1 for the large case).  One JSON line
per case and a summary line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CASES = [((4096, 8192), 7, 3), ((1024, 2048), 31, 3), ((16384, 32768), 1, 1)]


def card():
    """Name, power limit and SM clocks of GPU 0, read in the same run (read-only query)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def maxrel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def check_db(got, ref):
    lin_g, lin_r = 10 ** (got.astype(np.float64) / 10), 10 ** (ref.astype(np.float64) / 10)
    big = lin_r > 1e-3 * lin_r.max()
    return maxrel(lin_g, lin_r), float(np.max(np.abs(got[big] - ref[big])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from scintools_b200 import _device
    from scintools_b200.dynspec import BasicDyn, Dynspec
    _device.device()
    sync = torch.cuda.synchronize
    rows = []
    for (nf, nt), cuts, reps in CASES:
        dyn = np.random.default_rng(nf + nt).exponential(1.0, (nf, nt)).astype(np.float32)
        ds = Dynspec(dyn=BasicDyn(dyn, times=10.0 * np.arange(nt),
                                  freqs=1400.0 + 0.1 * np.arange(nf), dt=10.0, df=0.1),
                     verbose=False)
        fnum, tnum = nf // (cuts + 1), nt // (cuts + 1)

        def batched():
            ds.cut_dyn(tcuts=cuts, fcuts=cuts, dtype=np.float32)
            sync()

        def loop(check=False):
            worst = [0.0, 0.0, 0.0]
            for ii in range(cuts + 1):
                for jj in range(cuts + 1):
                    tile = dyn[ii * fnum:(ii + 1) * fnum, jj * tnum:(jj + 1) * tnum]
                    _, _, sec = ds.calc_sspec(input_dyn=tile, dtype=np.float32)
                    acf = ds.calc_acf(input_dyn=tile, dtype=np.float32)
                    if check:
                        r, db = check_db(ds.cutsspec[ii, jj], sec)
                        worst = [max(worst[0], r), max(worst[1], db),
                                 max(worst[2], maxrel(ds.cutacf[ii, jj], acf))]
                    del sec, acf
            sync()
            return worst

        batched()
        worst = loop(check=True)
        ok = worst[0] < 1e-5 and worst[1] < 2e-4 and worst[2] < 1e-5
        tb, tl = [], []
        for _ in range(reps):
            t0 = time.perf_counter()
            batched()
            tb.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            loop()
            tl.append(time.perf_counter() - t0)
        row = dict(case="%dx%d cut %dx%d" % (nf, nt, cuts + 1, cuts + 1), tile=[fnum, tnum],
                   tiles=(cuts + 1) ** 2, sspec_rel=worst[0], sspec_db=worst[1],
                   acf_rel=worst[2], match=ok, cut_dyn_s=min(tb), loop_s=min(tl),
                   speedup=min(tl) / min(tb))
        print(json.dumps(row), flush=True)
        rows.append(row)
        del ds
    summary = dict(card=card(), cases=rows)
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "probe_cut_dyn.json"), "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
