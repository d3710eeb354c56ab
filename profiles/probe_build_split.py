"""Where the time of the curvature-sweep gather goes: per-kernel device times of one benchmark
step (bench.py: make_dynspec, eta_grid, the same sb_cs_f32 / sb_cs_bound_f32 / sb_eta_sweep
calls) for the library as shipped and for two diagnostic builds of the gather kernels
(thth_build_copy_kernel, thth_build_kernel in thth.cu, compile-time SB_BUILD_PROBE):

    stores_only   every gathered value is a constant: index math and stores, no gathers
    gathers_only  the stores sit behind a predicate that is never true: index math and
                  gathers, no triangle written

    python profiles/probe_build_split.py [--lib LIB] [--variants DIR] [--steps 20] [--out F]

The diagnostic libraries are DIR/libscint_b200_stores_only.so and
DIR/libscint_b200_gathers_only.so; missing ones are compiled there from this tree's sources
(default DIR: a new temporary directory).  Kernel times come from torch.profiler (CUDA
activities), min / median / max over the steps, per launch: the copy kernels
(thth_colmark, thth_colslots, cs_compact), the gather (thth_build_copy_kernel /
thth_build_kernel) and the eigen solver.  The diagnostic builds compute wrong triangles, so
their eigen-solver times are not meaningful.  Prints the card's name, power limit and max SM
clock, and one JSON line; --out also writes the JSON to a file."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__ as G  # noqa: E402
import bench as B  # noqa: E402
from scintools_b200 import _device as D, _lib, ththmod as thth  # noqa: E402

VARIANTS = {"stores_only": 1, "gathers_only": 2}
KERNELS = ("thth_colmark_kernel", "thth_colslots_kernel", "cs_compact_kernel",
           "thth_build_copy_kernel", "thth_build_kernel", "eig_half")


def compile_variant(path, probe):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + G.NVCC_FLAGS + ["-DSB_BUILD_PROBE=%d" % probe, "-o", path] + G.SOURCES
    subprocess.run(cmd, cwd=G.CSRC, check=True)


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    for name in ("sb_init", "sb_last_error", "sb_eta_sweep", "sb_cs_f32", "sb_cs_bound_f32",
                 "sb_release"):
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
    return {"min": float(v.min()), "median": float(np.median(v)), "max": float(v.max()),
            "n": int(v.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=G.LIB, help="the library as shipped")
    ap.add_argument("--variants", default=None, help="directory of the diagnostic builds")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    vdir = a.variants or tempfile.mkdtemp(prefix="sb_split_")
    os.makedirs(vdir, exist_ok=True)
    paths = [("shipped", a.lib)]
    for name, probe in VARIANTS.items():
        p = os.path.join(vdir, "libscint_b200_%s.so" % name)
        if not os.path.exists(p):
            compile_variant(p, probe)
        paths.append((name, p))

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", card)
    D.device()
    libs = [(name, load(p)) for name, p in paths]

    dyn, freq, t = B.make_dynspec()
    fd = np.asarray(thth.fft_axis(t, "mHz", B.NPAD))
    tau = np.asarray(thth.fft_axis(freq, "us", B.NPAD))
    edges = np.linspace(-B.EDGE_LIM, B.EDGE_LIM, B.NEDGE)
    d_dyn = D.upload(dyn)
    ntau, nfd = (B.NPAD + 1) * B.NF, (B.NPAD + 1) * B.NT
    pitch = nfd // 2 + 16
    d_cs = D.empty((ntau, pitch, 2), torch.float32)
    keep = thth.needed_fd_columns(fd, edges) or 0
    d_bound = D.empty((1,), torch.float32)
    cs = thth.DeviceCS(d_cs, nfd=nfd, ncols_valid=keep or None, bound=d_bound)
    geom = thth._Geom(cs, tau, fd, edges, True)
    etas = np.ascontiguousarray(B.eta_grid(B.NETA))
    n = len(etas)
    d_etas = D.upload(etas)
    eigs = D.empty((n,), torch.float64)
    stat, nred, iters = (D.empty((n,), torch.int32) for _ in range(3))
    stream = D.stream_ptr()

    def step(lib):
        check(lib, lib.sb_cs_f32(d_dyn.data_ptr(), B.NF, B.NT, B.NPAD, 0.0, 0, 1, pitch, keep,
                                 d_cs.data_ptr(), stream))
        check(lib, lib.sb_cs_bound_f32(d_dyn.data_ptr(), B.NF, B.NT, B.NPAD, 0.0,
                                       d_bound.data_ptr(), stream))
        check(lib, lib.sb_eta_sweep(geom.ref, d_etas.data_ptr(), n, thth.DEFAULT_TOL, 0,
                                    eigs.data_ptr(), stat.data_ptr(), nred.data_ptr(),
                                    iters.data_ptr(), stream))

    report = {"card": card, "steps": a.steps, "etas": n}
    for name, lib in libs:
        for _ in range(a.warmup):
            step(lib)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            step(lib)
        e1.record()
        torch.cuda.synchronize()
        step_ms = e0.elapsed_time(e1) / a.steps
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                step(lib)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            for k in KERNELS:
                if k in ev.name:
                    per.setdefault(k, []).append(ev.time_range.elapsed_us() / 1000.0)
        report[name] = {"step_ms": step_ms, "kernel_ms": {k: stats(v) for k, v in per.items()}}
        print(name, json.dumps(report[name]))
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
