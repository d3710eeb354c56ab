"""A/B of the curvature-sweep gather between builds of libscint_b200, loaded side by side
by path and ALTERNATED on the benchmark's own inputs (bench.py: make_dynspec, eta_grid,
the same sb_cs_f32 / sb_cs_bound_f32 / sb_eta_sweep step).

    python profiles/probe_build_gather.py parent=/path/libparent.so new=scintools_b200/lib/libscint_b200.so

Per build: CUDA-event time of the step and the per-kernel times of sb_profile over
--rounds alternations of --steps steps (min / median / max over the rounds), and whether
eigs / status / nred / iters are bit-equal to the first build's.  Then sb_eta_sweep alone
(the spectrum is not recomputed) on three more workloads: the bench grid with 16
curvatures, a NON-UNIFORM 512-edge grid with 1024 and with 16 curvatures.
Prints the card's name, power limit and max SM clock, and one JSON line; --out also
writes the JSON to a file."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench as B  # noqa: E402
from scintools_b200 import _device as D, _lib, ththmod as thth  # noqa: E402


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    for name in ("sb_init", "sb_last_error", "sb_profile_enable", "sb_profile_collect",
                 "sb_eta_sweep", "sb_cs_f32", "sb_cs_bound_f32", "sb_release"):
        fn, ref = getattr(lib, name), getattr(_lib.lib, name)
        fn.restype, fn.argtypes = ref.restype, ref.argtypes
    if lib.sb_init(torch.cuda.current_device()) != 0:
        raise RuntimeError(lib.sb_last_error().decode())
    return lib


def check(lib, rc):
    if rc != 0:
        raise RuntimeError("error %d: %s" % (rc, lib.sb_last_error().decode()))


def stats(v):
    v = np.asarray(v, float)
    return {"min": float(v.min()), "median": float(np.median(v)), "max": float(v.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+", help="name=path, the first one is the reference")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", card)
    D.device()
    libs = [(s.split("=", 1)[0], load(s.split("=", 1)[1])) for s in a.libs]

    dyn, freq, t = B.make_dynspec()
    fd = np.asarray(thth.fft_axis(t, "mHz", B.NPAD))
    tau = np.asarray(thth.fft_axis(freq, "us", B.NPAD))
    edges = np.linspace(-B.EDGE_LIM, B.EDGE_LIM, B.NEDGE)
    rng = np.random.default_rng(11)
    # irregular edges inside the uniform grid's outermost centres: the same fd columns suffice
    lim_nu = B.EDGE_LIM * (1.0 - 1.0 / (B.NEDGE - 1))
    edges_nu = np.sort(rng.uniform(-lim_nu, lim_nu, B.NEDGE))
    d_dyn = D.upload(dyn)
    ntau, nfd = (B.NPAD + 1) * B.NF, (B.NPAD + 1) * B.NT
    pitch = nfd // 2 + 16
    d_cs = D.empty((ntau, pitch, 2), torch.float32)
    keep = thth.needed_fd_columns(fd, edges) or 0
    d_bound = D.empty((1,), torch.float32)
    cs = thth.DeviceCS(d_cs, nfd=nfd, ncols_valid=keep or None, bound=d_bound)
    stream = D.stream_ptr()

    def buffers(etas):
        n = len(etas)
        return dict(n=n, etas=D.upload(np.ascontiguousarray(etas)),
                    eigs=D.empty((n,), torch.float64), stat=D.empty((n,), torch.int32),
                    nred=D.empty((n,), torch.int32), iters=D.empty((n,), torch.int32))

    def sweep(lib, geom, buf):
        check(lib, lib.sb_eta_sweep(geom.ref, buf["etas"].data_ptr(), buf["n"], thth.DEFAULT_TOL, 0,
                                    buf["eigs"].data_ptr(), buf["stat"].data_ptr(),
                                    buf["nred"].data_ptr(), buf["iters"].data_ptr(), stream))

    def spectrum(lib):
        check(lib, lib.sb_cs_f32(d_dyn.data_ptr(), B.NF, B.NT, B.NPAD, 0.0, 0, 1, pitch, keep,
                                 d_cs.data_ptr(), stream))
        check(lib, lib.sb_cs_bound_f32(d_dyn.data_ptr(), B.NF, B.NT, B.NPAD, 0.0,
                                       d_bound.data_ptr(), stream))

    def timed(lib, step, steps):
        lib.sb_profile_enable(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            step()
        e1.record()
        torch.cuda.synchronize()
        ms = np.zeros(16)
        cnt = np.zeros(16, dtype=np.int32)
        check(lib, lib.sb_profile_collect(ms.ctypes.data, cnt.ctypes.data, 16))
        lib.sb_profile_enable(0)
        kern = {n_: ms[i] / steps for i, n_ in enumerate(B.PROF_NAMES) if cnt[i]}
        return e0.elapsed_time(e1) / steps, kern

    def ab(label, geom, etas, with_cs, rounds, steps):
        buf = buffers(etas)
        res = {name: {"step_ms": [], "kernel_ms": {}} for name, _ in libs}
        outs = {}
        for name, lib in libs:
            def step(lib=lib):
                if with_cs:
                    spectrum(lib)
                sweep(lib, geom, buf)
            for _ in range(a.warmup):
                step()
            torch.cuda.synchronize()
            outs[name] = {k: buf[k].cpu().numpy().copy() for k in ("eigs", "stat", "nred", "iters")}
            res[name]["step"] = step
        for _ in range(rounds):
            for name, lib in libs:
                ms, kern = timed(lib, res[name]["step"], steps)
                res[name]["step_ms"].append(ms)
                for k, v in kern.items():
                    res[name]["kernel_ms"].setdefault(k, []).append(v)
        ref = outs[libs[0][0]]
        out = {}
        for name, _ in libs:
            o = outs[name]
            same = all(np.array_equal(o[k], ref[k], equal_nan=(k == "eigs")) for k in o)
            out[name] = {"step_ms": stats(res[name]["step_ms"]),
                         "kernel_ms": {k: stats(v) for k, v in res[name]["kernel_ms"].items()},
                         "bit_equal_to_" + libs[0][0]: bool(same)}
            print(label, name, json.dumps(out[name]))
        return out

    geom = thth._Geom(cs, tau, fd, edges, True)
    geom_nu = thth._Geom(cs, tau, fd, edges_nu, True)
    report = {"card": card, "rounds": a.rounds, "steps": a.steps}
    report["bench_step_1024_uniform"] = ab("bench_step_1024_uniform", geom, B.eta_grid(B.NETA), True,
                                           a.rounds, a.steps)
    spectrum(libs[0][1])
    torch.cuda.synchronize()
    short = max(3, a.rounds // 2)
    report["sweep_16_uniform"] = ab("sweep_16_uniform", geom, B.eta_grid(16), False, short, a.steps)
    report["sweep_1024_nonuniform"] = ab("sweep_1024_nonuniform", geom_nu, B.eta_grid(B.NETA), False,
                                         short, max(2, a.steps // 4))
    report["sweep_16_nonuniform"] = ab("sweep_16_nonuniform", geom_nu, B.eta_grid(16), False, short,
                                       a.steps)
    for _, lib in libs:
        lib.sb_release()
    line = json.dumps(report)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
