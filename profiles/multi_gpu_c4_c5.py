"""BASELINE.json configs 4 and 5 on N GPUs of one node (one process per GPU):

  C4  256 phase-screen realisations Simulation(ns=8192, nf=NF) -- seeds block-
      partitioned over the ranks (sharding.sharded_items), no data-path collective,
      one all-gather of a per-realisation checksum (reference: scint_sim.py:23-311)
  C5  1024 dynamic spectra (1024 x 2048, 1-D-screen recipe, seeds 1000+i) through
      the whole pipeline calc_sspec + calc_acf + single_search
      (pipeline.batch_arc_pipeline: the reference's pool.map mode, dynspec.py:1715-1719),
      dynspecs block-partitioned, one all-gather of (eta_fit, eta_sig)

  torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 profiles/multi_gpu_c4_c5.py \
      [--nreal 256] [--nf 256] [--ndyn 1024] [--out c4c5_N.json]

Rank 0 also RECOMPUTES a few items that other ranks own and asserts bit-equality
with the gathered results (same seed, same kernels -> same bits on any GPU), and
writes every per-item result so that runs at different N can be diffed offline.
Timing: barrier + synchronize on both sides, max over ranks."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def dynspec_1024(seed, nf=1024, nt=2048):
    import bench
    rng = np.random.default_rng(seed)
    nimg = 64
    fdk = rng.uniform(-8.0, 8.0, nimg)
    ak = (rng.normal(size=nimg) + 1j * rng.normal(size=nimg)) / np.sqrt(2)
    ak = ak * np.exp(-(fdk / 4.0) ** 2)
    tauk = bench.ETA_TRUE * fdk ** 2
    t = bench.DT * np.arange(nt)
    f = 0.125 * np.arange(nf)                      # 128 MHz band like C3
    U = np.exp(2j * np.pi * 1e-3 * fdk[:, None] * t[None, :])
    V = np.exp(-2j * np.pi * tauk[None, :] * f[:, None]) * ak[None, :]
    E = V.astype(np.complex64) @ U.astype(np.complex64)
    dyn = (E.real ** 2 + E.imag ** 2).astype(np.float32)
    dyn += rng.normal(0.0, 0.2 * dyn.mean(), dyn.shape).astype(np.float32)
    return dyn, 1400.0 + f, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nreal", type=int, default=256)
    ap.add_argument("--ns", type=int, default=8192)
    ap.add_argument("--nf", type=int, default=256)
    ap.add_argument("--ndyn", type=int, default=1024)
    ap.add_argument("--neta", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    import bench
    from scintools_b200 import _device as D
    from scintools_b200 import pipeline, sharding
    from scintools_b200.scint_sim import Simulation

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = D.device()
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)

    def sync():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def tmax(seconds):
        tt = torch.tensor([seconds], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        return float(tt.item())

    out = {"n_gpus": world}

    # ---------------- C4 ----------------
    def realise(seed):
        s = Simulation(mb2=2, ns=args.ns, nf=args.nf, dlam=0.25, seed=int(seed), device_rng=True,
                       lazy=True)       # w / xyp / xyi stay on the device unless asked for
        d = np.asarray(s.dyn, dtype=np.float64)
        return np.array([d.sum(), (d * d).sum(), float(d[d.shape[0] // 3, d.shape[1] // 5])])

    seeds = list(range(args.nreal))
    realise(10 ** 6)                                  # warm-up (tables, workspaces)
    sync()
    t0 = time.perf_counter()
    mine = sharding.sharded_items(seeds)
    local = np.array([realise(s) for s in mine]).reshape(len(mine), 3)
    cols = [sharding.all_gather_blocks(local[:, k] if len(mine) else np.zeros(0), len(seeds))
            for k in range(3)]
    sync()
    c4_s = tmax(time.perf_counter() - t0)
    chk = np.stack(cols, axis=1)
    out["c4"] = {"realisations": args.nreal, "ns": args.ns, "nf": args.nf, "seconds": c4_s,
                 "realisations_per_s": args.nreal / c4_s,
                 "screen_frequency_planes_per_s": args.nreal * args.nf / c4_s,
                 "checksums": chk.tolist()}
    if rank == 0:
        others = [s for s in (seeds[-1], seeds[len(seeds) // 2], seeds[len(seeds) // 3])
                  if s not in mine] or seeds[:1]
        for s in others:
            assert np.array_equal(realise(s), chk[s]), "C4 realisation %d differs across ranks" % s
        out["c4"]["cross_rank_equal"] = [int(s) for s in others]

    # ---------------- C5 ----------------
    etas = np.logspace(np.log10(bench.ETA_TRUE / 2), np.log10(2 * bench.ETA_TRUE), args.neta)
    edges = np.linspace(-bench.EDGE_LIM, bench.EDGE_LIM, 256)
    lo, hi = sharding.block_range(args.ndyn, rank, world)
    d0, freqs, times = dynspec_1024(999)
    pipeline.arc_pipeline(d0, freqs, times, etas, edges)          # warm-up
    host = [dynspec_1024(1000 + i)[0] for i in range(lo, hi)]     # synthetic inputs, not timed
    dyns = [None] * args.ndyn
    dyns[lo:hi] = host
    sync()
    t0 = time.perf_counter()
    fit, sig = pipeline.batch_arc_pipeline(dyns, freqs, times, etas, edges)
    sync()
    c5_s = tmax(time.perf_counter() - t0)
    out["c5"] = {"dynspecs": args.ndyn, "shape": [1024, 2048], "netas": args.neta,
                 "seconds": c5_s, "dynspecs_per_s": args.ndyn / c5_s,
                 "eta_fit": fit.tolist(), "eta_sig": sig.tolist()}
    if rank == 0:
        picks = [i for i in (args.ndyn - 1, args.ndyn // 2) if not (lo <= i < hi)] or [0]
        for i in picks:
            r = pipeline.arc_pipeline(dynspec_1024(1000 + i)[0], freqs, times, etas, edges)
            assert r["eta_fit"] == fit[i] or (np.isnan(r["eta_fit"]) and np.isnan(fit[i])), \
                "C5 dynspec %d differs across ranks" % i
        out["c5"]["cross_rank_equal"] = [int(i) for i in picks]
        line = json.dumps(out)
        if args.out:
            with open(args.out, "w") as fh:
                fh.write(line)
        short = {k: ({kk: vv for kk, vv in v.items() if kk not in ("checksums", "eta_fit", "eta_sig")}
                     if isinstance(v, dict) else v) for k, v in out.items()}
        print(json.dumps(short), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
