"""GPU: every curvature of the benchmark's full-size sweeps against float64 eigenvalues.

The workload is bench.py's: a 4096 x 8192 dynamic spectrum (64 images on a 1-D
screen, eta_true = 0.08 s^3), npad = 3 -> a 16384 x 32768 conjugate spectrum kept
as its fd >= 0 half, with only the fd columns the 511-centre theta grid reaches
computed (needed_fd_columns) and the L1 bound of sb_cs_bound_f32 as the scale of
the default solver's fp16 copy.  Checked here:

  grid A     the 1024 headline curvatures, default solver and SB_EIG_FP32=1;
  grid B     the 8192 curvatures of the strong-scaling leg (the same range eight
             times denser), default solver, several launches of the batch slab;
  e2e        search_batch over five chunks from pinned float32 and float64 host
             memory, against single_search and the grid A references.

On EVERY curvature: |rel| <= 1e-5 against the reference, status 0, and the
cropped size nred bit-exact against the oracle's th_points.

Reference.  For each curvature the oracle's thth_redmap crop (the reference's
numpy gather, complex128) of the SAME fp32 spectrum the device made: whole.numpy(),
the whole fd >= 0 half plane expanded on the host (a column-limited plane cannot be
expanded; test_column_limited_plane ties the two planes together bit for bit), and
its largest algebraic eigenvalue from a dense LAPACK solve
(scipy.linalg.eigh, subset_by_index=[n-1, n-1]).  That is what the reference's
Eval_calc computes with ARPACK (eigsh(..., which="LA")); on the 77 curvatures that
test_gpu_fullsize.py checks with ARPACK, the two must agree to 1e-9.  The 9216
dense solves run in a fork pool with one BLAS thread per worker, bench.CpuSweep's
set-up (bench._G, bench._pool_init, bench._eval_one = Eval_calc); the workers share
the 4.3 GB host spectrum copy-on-write and never touch the GPU.

The run prints, per grid and solver, the worst error as a fraction of the bar and
the histogram of Lanczos iterations; neither the iteration counts nor which path
of the solver a curvature took are asserted."""
import math
import multiprocessing as mp
import os
import resource
import time

import numpy as np
import pytest
import scipy.linalg

import bench
from oracle import thth_oracle as TO

pytestmark = pytest.mark.gpu

REL = 1e-5
ETAS_A = bench.eta_grid(bench.NETA)
ETAS_B = bench.eta_grid(bench.NETA_STRONG)
EDGES = np.linspace(-bench.EDGE_LIM, bench.EDGE_LIM, bench.NEDGE)
# the curvatures of grid A that test_gpu_fullsize.py::test_c3_cs_and_sweep checks with
# ARPACK, the slowly converging ones of the round-1 stopping-rule bug among them
ARPACK_PICK = sorted(set(list(range(0, bench.NETA, 16)) +
                         [400, 700, 1023, 95, 118, 119, 120, 121, 162, 174, 325, 784, 809,
                          810, 905]))
# Copies of thth.cu: the per-launch budget of the sweep's fp32 matrix slab (sweep_batch)
# and the slab row length ld = 32 ceil(n / 32) of the 511-centre grid.  With them grid B
# must take ceil(8192 / 1536) = 6 launches; test_grid_b_every_curvature asserts that
# count so that it fails when the budget changes -- update these two constants with
# thth.cu, and keep grid B larger than one launch.
SLAB_BYTES = 3 << 30
LD = 512
# the float64 references of the whole module must come back within this many seconds
# (about 200 s on 8 cores); past it the pool is terminated and the fixture fails
REF_TIMEOUT = 600


@pytest.fixture(scope="module")
def sb():
    import scintools_b200
    from scintools_b200 import _device
    _device.device()
    return scintools_b200


@pytest.fixture(scope="module")
def full(sb):
    """The benchmark's spectrum as the benchmark builds it (column-limited half plane),
    the whole half plane, and the full fftshifted plane on the host (complex64)."""
    thth = sb.ththmod
    t0 = time.perf_counter()
    dyn, freq, t = bench.make_dynspec()
    tau = TO.fft_axis(freq, "us", bench.NPAD)
    fd = TO.fft_axis(t, "mHz", bench.NPAD)
    keep = thth.needed_fd_columns(fd, EDGES)
    assert keep is not None and keep < fd.shape[0] // 2 + 1
    cs = thth.conjugate_spectrum(dyn, bench.NPAD, 0.0, half=True, ncols_keep=keep)
    whole = thth.conjugate_spectrum(dyn, bench.NPAD, 0.0, half=True)
    assert cs.shape == whole.shape == (16384, 32768)
    CS = whole.numpy().astype(np.complex64)
    return dict(dyn=dyn, freq=freq, t=t, tau=tau, fd=fd, keep=keep, cs=cs, whole=whole,
                CS=CS, t0=t0)


# ---- float64 references in a fork pool (bench.CpuSweep's globals and initializer) ----
def _dense_top(eta):
    """Largest algebraic eigenvalue of the reference's crop, dense float64 LAPACK."""
    g = bench._G
    red, _ = TO.thth_redmap(g["CS"], g["tau"], g["fd"], eta, g["edges"])
    n = red.shape[0]
    w = scipy.linalg.eigh(red, eigvals_only=True, subset_by_index=[n - 1, n - 1])
    return abs(float(w[0]))         # Eval_calc returns |w|


def _nred(full, etas):
    return np.array([TO.th_points(full["tau"], full["fd"], e, EDGES).sum() for e in etas])


@pytest.fixture(scope="module")
def refs(full):
    etas = np.concatenate([ETAS_A, ETAS_B])
    procs = max(1, min(len(os.sched_getaffinity(0)), 64))
    bench._G.update(CS=full["CS"], tau=full["tau"], fd=full["fd"], edges=EDGES)
    t0 = time.perf_counter()
    # The references need the device-made spectrum, so the fork comes after the CUDA
    # context and torch's threads exist.  That is safe because the workers run numpy /
    # scipy only, never CUDA, and leave through os._exit.  bench._pool_init limits BLAS
    # to one thread where threadpoolctl is installed and is a no-op elsewhere, so a
    # worker's initializer cannot fail (a failing one is respawned without end).
    pool = mp.get_context("fork").Pool(procs, initializer=bench._pool_init)
    try:
        dense = np.array(pool.map_async(_dense_top, list(etas), chunksize=4).get(REF_TIMEOUT))
        t_dense = time.perf_counter() - t0
        arpack = np.array(pool.map_async(bench._eval_one, list(ETAS_A[ARPACK_PICK]),
                                         chunksize=1).get(max(1.0, REF_TIMEOUT - t_dense)))
    finally:
        pool.terminate()
        pool.join()
        bench._G.clear()
    t_all = time.perf_counter() - t0
    kb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    print("\nfloat64 references: %d dense solves in %.1f s, %d ARPACK solves, %.1f s in all, "
          "on %d processes; peak RSS of the test process %.1f GB"
          % (len(etas), t_dense, len(ARPACK_PICK), t_all, procs, kb / 2**20))
    return dict(a=dense[:ETAS_A.size], b=dense[ETAS_A.size:], arpack=arpack,
                nred_a=_nred(full, ETAS_A), nred_b=_nred(full, ETAS_B))


def _check_every_curvature(label, etas, eigs, info, ref, nred):
    """|rel| <= REL, status 0 and nred bit-exact on every curvature; prints the worst
    error (as a fraction of the bar) and the iteration histogram."""
    rel = np.abs(eigs - ref) / ref
    i = int(np.argmax(np.where(np.isfinite(rel), rel, np.inf)))
    vals, counts = np.unique(info["iters"], return_counts=True)
    print("\n%s: %d curvatures, worst |rel| %.2e = %.3f of the bar at eta[%d] = %.6f "
          "(nred %d); iters {%s}"
          % (label, etas.size, rel[i], rel[i] / REL, i, etas[i], info["nred"][i],
             ", ".join("%d: %d" % (v, c) for v, c in zip(vals, counts))))
    bad = np.flatnonzero(info["status"] != 0)
    assert bad.size == 0, "status != 0 at %s: %s" % (bad[:20], info["status"][bad[:20]])
    assert np.array_equal(info["nred"], nred), np.flatnonzero(info["nred"] != nred)[:20]
    bad = np.flatnonzero(~(rel <= REL))
    assert bad.size == 0, "|rel| > %g at %d curvatures: %s" % (
        REL, bad.size, [(int(k), float(rel[k])) for k in bad[:20]])


def test_column_limited_plane(sb, full):
    """The plane the benchmark sweeps (only the fd columns the grid reaches) gives
    bit-identically the sweep of the whole half plane: on a handful of curvatures
    (direct gathers from the spectrum) and on all of grid A (gathers from the compact
    copy of the reached columns)."""
    thth = sb.ththmod
    few = ETAS_A[[0, 95, 120, 400, 512, 809, 1023]]
    for etas in (few, ETAS_A):
        a, ia = thth.eta_sweep(full["whole"], full["tau"], full["fd"], etas, EDGES,
                               return_info=True)
        b, ib = thth.eta_sweep(full["cs"], full["tau"], full["fd"], etas, EDGES,
                               return_info=True)
        assert np.array_equal(a, b)
        for k in ("status", "nred", "iters"):
            assert np.array_equal(ia[k], ib[k]), k


def test_dense_reference_matches_arpack(refs):
    """The dense float64 reference is the reference's own eigenvalue (ARPACK eigsh on
    the same crop) on the curvatures test_gpu_fullsize.py checks that way."""
    dense = refs["a"][ARPACK_PICK]
    rel = np.abs(dense - refs["arpack"]) / refs["arpack"]
    print("\ndense vs ARPACK over %d curvatures: max |rel| %.2e" % (len(ARPACK_PICK), rel.max()))
    assert rel.max() <= 1e-9


@pytest.mark.parametrize("solver", ["default", "fp32"])
def test_grid_a_every_curvature(sb, full, refs, monkeypatch, solver):
    """The 1024 headline curvatures with the default solver (fp16 tensor-core
    Lanczos + fp32 Rayleigh quotient) and the fp32 solver (SB_EIG_FP32=1)."""
    if solver == "fp32":
        monkeypatch.setenv("SB_EIG_FP32", "1")
    eigs, info = sb.ththmod.eta_sweep(full["cs"], full["tau"], full["fd"], ETAS_A, EDGES,
                                      return_info=True)
    _check_every_curvature("grid A, %s solver" % solver, ETAS_A, eigs, info, refs["a"],
                           refs["nred_a"])
    assert abs(ETAS_A[np.argmax(eigs)] / bench.ETA_TRUE - 1) < 0.02


def test_grid_b_every_curvature(sb, full, refs, monkeypatch):
    """The 8192 curvatures of the strong-scaling leg, default solver.  Their matrices
    do not fit one launch's slab, so this is the multi-launch path at full size."""
    from scintools_b200 import _lib
    monkeypatch.delenv("SB_SWEEP_SLAB_MB", raising=False)
    monkeypatch.delenv("SB_EIG_FP32", raising=False)
    L = _lib.lib
    per_launch = SLAB_BYTES // (LD * LD * 8)
    want = math.ceil(ETAS_B.size / per_launch)
    bench.collect_prof(L, _lib)                 # drop events of earlier profiled calls
    L.sb_profile_enable(1)
    try:
        n0 = L.sb_launch_count()
        eigs, info = sb.ththmod.eta_sweep(full["cs"], full["tau"], full["fd"], ETAS_B, EDGES,
                                          return_info=True)
        launches = L.sb_launch_count() - n0
        _, cnt = bench.collect_prof(L, _lib)
    finally:
        L.sb_profile_enable(0)
    eig_launches = int(cnt[bench.PROF_NAMES.index("thth_eig")])
    print("\ngrid B: %d kernel launches, %d eigen-solver launches of at most %d curvatures"
          % (launches, eig_launches, per_launch))
    assert eig_launches == want > 1
    _check_every_curvature("grid B, default solver", ETAS_B, eigs, info, refs["b"],
                           refs["nred_b"])
    assert abs(ETAS_B[np.argmax(eigs)] / bench.ETA_TRUE - 1) < 0.02


def test_search_batch_end_to_end(sb, full, refs):
    """The benchmark's end-to-end call: search_batch over five chunks from pinned
    float32 and float64 host memory.  single_search pads with the chunk's mean where
    the grids above pad with 0.0; the bench spectrum has had its mean subtracted, so
    the two differ only by the fp32 rounding of that mean."""
    import torch
    thth = sb.ththmod
    dyn = full["dyn"]
    out = {}
    for name, host in (("float32", dyn), ("float64", dyn.astype(np.float64))):
        h = torch.from_numpy(host).pin_memory()
        params = [h.numpy(), full["freq"], full["t"], ETAS_A, EDGES, None, False, bench.FW,
                  bench.NPAD, True, 0.0, False]
        out[name] = thth.search_batch([params] * 5) + [thth.single_search(params)]
        del h, params
    eigs = out["float32"][-1][4]
    for name, res in out.items():
        for k, r in enumerate(res):
            assert np.array_equal(r[4], eigs), (name, k)
            assert r[0] == thth.peak_fit(ETAS_A, r[4], bench.FW)[0], (name, k)
    grid_a = thth.eta_sweep(full["cs"], full["tau"], full["fd"], ETAS_A, EDGES)
    pad = np.abs(eigs - grid_a) / grid_a
    rel = np.abs(eigs - refs["a"]) / refs["a"]
    eta_fit = out["float32"][0][0]
    eta_ref = TO.peak_fit(ETAS_A, refs["a"], bench.FW)[0]
    print("\nsearch_batch: mean vs 0.0 padding max |rel| %.2e; vs float64 max |rel| %.2e = "
          "%.3f of the bar; eta_fit %.7f, on the float64 curve %.7f (rel %.2e)"
          % (pad.max(), rel.max(), rel.max() / REL, eta_fit, eta_ref, eta_fit / eta_ref - 1))
    assert (rel <= REL).all(), np.flatnonzero(~(rel <= REL))[:20]
    assert abs(eta_fit / eta_ref - 1) <= 1e-3
    assert abs(ETAS_A[np.argmax(eigs)] / bench.ETA_TRUE - 1) < 0.02
    print("module wall time so far %.1f s, peak RSS of the test process %.1f GB"
          % (time.perf_counter() - full["t0"],
             resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20))
