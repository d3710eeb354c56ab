"""Multi-station theta-theta retrieval on the CPU: the numpy oracle's
VLBI_chunk_retrieval against the reference's wavefields
(tests/golden/vlbi_sample_*.npz), the device code of sb::vlbi_retrieval around the
eigenpair (composite gather, per-station scatter) under the SIMT emulator
(tests/host_emu/vlbi_emu.cpp) against the oracle, and the new C symbols."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import thth_oracle as TO
from oracle import vlbi_oracle as VO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")


def _inputs(f):
    """The fixture's list, station spectra as real arrays like the reference got them."""
    n_dish = int(f["n_dish"])
    autos = set(VO.auto_indices(n_dish))
    return [f["dspec"][k].real if k in autos else f["dspec"][k] for k in range(len(f["dspec"]))]


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_oracle_vlbi_matches_reference(golden_dir, tag):
    """Same eigenvalue; same eigenvector and wavefields after ONE global phase shared by
    every station (a: 3 stations radix sizes, b: 2 stations chirp-z sizes with a tau mask,
    c: one station)."""
    f = np.load(os.path.join(golden_dir, "vlbi_sample_%s.npz" % tag))
    n_dish = int(f["n_dish"])
    models, x = VO.VLBI_chunk_retrieval(_inputs(f), f["edges"], f["time"], f["freq"],
                                        float(f["eta"]), int(f["npad"]), n_dish,
                                        float(f["tau_mask"]), return_all=True)
    assert abs(x["w"] - float(f["w"])) <= 1e-12 * abs(float(f["w"]))
    assert np.linalg.norm(x["composite"]) == pytest.approx(float(f["fro"]), rel=1e-12)
    ph = np.vdot(f["V"], x["V"])
    ph /= abs(ph)
    assert np.linalg.norm(x["V"] - ph * f["V"]) < 1e-12
    for d in range(n_dish):
        ref = f["model_E"][d]
        assert np.linalg.norm(models[d] - np.conj(ph) * ref) <= 1e-12 * np.linalg.norm(ref), d


def test_oracle_vlbi_composite_layout(golden_dir):
    """Hermitian composite with zero trace; diagonal blocks are the station maps."""
    f = np.load(os.path.join(golden_dir, "vlbi_sample_a.npz"))
    cs, tau, fd = VO.spectra(_inputs(f), f["time"], f["freq"], int(f["npad"]), 3)
    comp, _ = VO.composite(cs, tau, fd, float(f["eta"]), f["edges"], 3)
    n = int(f["nred"])
    assert comp.shape == (3 * n, 3 * n)
    assert np.array_equal(comp, np.conjugate(comp.T))
    assert np.trace(comp) == 0
    assert np.abs(comp[n:2 * n, :n]).max() > 0


def _emu_lib():
    src = os.path.join(EMU, "vlbi_emu.cpp")
    out = os.path.join(EMU, "_build", "vlbi_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    csrc = os.path.join(ROOT, "scintools_b200", "csrc")
    newest = max([os.path.getmtime(os.path.join(csrc, f)) for f in os.listdir(csrc)] +
                 [os.path.getmtime(src), os.path.getmtime(os.path.join(EMU, "simt.h"))])
    if not os.path.exists(out) or os.path.getmtime(out) < newest:
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                        "-x", "c++", src, "-o", out], check=True)
    return ctypes.CDLL(out)


@pytest.mark.parametrize("tag", ["a", "b"])
def test_vlbi_kernels_on_host(golden_dir, tag):
    """The composite gather and the per-station scatter under the SIMT emulator against
    the oracle, on the fp32-rounded spectra the device sees (a: 3 stations, 256 x 512;
    b: 2 stations, 256 x 568 with a tau mask).  Composite: identical zero pattern (crop,
    diagonal, the full grid's anti-diagonal on the station blocks only, points outside the
    spectrum), every block in its place with its conjugation, values to fp32 rounding.
    Scatter: bin counts exact, every station's bin means to 1e-5 of the oracle's rev_map of
    its single row conj(V_d) sqrt(w)."""
    f = np.load(os.path.join(golden_dir, "vlbi_sample_%s.npz" % tag))
    n_dish, eta, edges = int(f["n_dish"]), float(f["eta"]), f["edges"]
    cs, tau, fd = VO.spectra(_inputs(f), f["time"], f["freq"], int(f["npad"]), n_dish,
                             float(f["tau_mask"]))
    cs32 = [np.ascontiguousarray(c.astype(np.complex64)) for c in cs]
    comp, edges_red = VO.composite([c.astype(np.complex128) for c in cs32], tau, fd, eta, edges,
                                   n_dish)
    n = comp.shape[0] // n_dish
    w_all, V_all = np.linalg.eigh(comp)
    w = float(w_all[-1])
    V32 = np.ascontiguousarray(V_all[:, -1].astype(np.complex64))
    th = TO.theta_centres(edges)
    th_red = TO.theta_centres(edges_red)
    ntau, nfd = cs[0].shape
    N = n_dish * len(th)
    A = np.zeros(N * N, np.complex64)
    recov = np.zeros((n_dish, ntau, nfd), np.complex64)
    cnt = np.zeros((ntau, nfd), np.int32)
    nred = np.zeros(1, np.int32)
    ptrs = (ctypes.c_void_p * len(cs32))(*[c.ctypes.data for c in cs32])
    lib = _emu_lib()
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
    c_ll, c_d, c_i, vp = ctypes.c_longlong, ctypes.c_double, ctypes.c_int, ctypes.c_void_p
    lib.emu_vlbi_stages.argtypes = [vp, c_i, c_ll, c_ll, c_d, c_d, c_d, c_d, c_d, c_d, vp, c_i,
                                    c_d, vp, c_d, c_d, vp, c_d, vp, vp, vp, vp]
    lib.emu_vlbi_stages(ptrs, n_dish, ntau, nfd, float(tau[0]), float(np.diff(tau).mean()),
                        float(abs(tau.max())), float(fd[0]), float(np.diff(fd).mean()),
                        float(abs(fd.max()) / 2), P(th), len(th), eta, P(th_red),
                        float(tau[1] - tau[0]), float(fd[1] - fd[0]), P(V32), w, P(nred), P(A),
                        P(recov), P(cnt))
    assert int(nred[0]) == n
    got = A[:(n_dish * n) ** 2].reshape(n_dish * n, n_dish * n).astype(np.complex128)
    assert np.array_equal(got == 0, comp == 0)
    eps = np.finfo(np.float32).eps
    assert (np.abs(got - comp) <= 4 * eps * np.abs(comp)).all()
    # the full grid's anti-diagonal is zero in the station blocks only
    sel = TO.th_points(tau, fd, eta, edges)
    full = np.flatnonzero(sel)
    anti = full[:, None] + full[None, :] == len(th) - 1
    assert anti.any()
    blk = lambda r, c: got[r * n:(r + 1) * n, c * n:(c + 1) * n]   # noqa: E731
    for d1 in range(n_dish):
        for d2 in range(n_dish - d1):
            # the map of spectrum (d1, d1 + d2), straight from the oracle's gather
            k = VO.pair_index(n_dish, d1, d2)
            t, _ = TO.thth_redmap(cs32[k].astype(np.complex128), tau, fd, eta, edges,
                                  hermetian=d2 == 0)
            lower, upper = blk(d1 + d2, d1), blk(d1, d1 + d2)
            assert (np.abs(lower - t) <= 4 * eps * np.abs(t)).all(), (d1, d2)
            assert np.array_equal(upper, np.conjugate(lower.T)), (d1, d2)
            if d2 == 0:
                assert (lower[anti] == 0).all() and (np.diag(lower) == 0).all()
            elif float(f["tau_mask"]) == 0:
                # the anti-diagonal gathers the tau = 0 row, which case b masks
                assert (lower[anti] != 0).any()
    # scatter: counts of all off-diagonal points, one half plane; bin means per station
    fd_edges = (np.linspace(0, nfd, nfd + 1) - .5) * (fd[1] - fd[0]) + fd[0]
    tau_edges = (np.linspace(0, ntau, ntau + 1) - .5) * (tau[1] - tau[0]) + tau[0]
    off = ~np.eye(n, dtype=bool)
    x = (th_red[np.newaxis, :] - th_red[:, np.newaxis])[off]
    y = (eta * (th_red[np.newaxis, :] ** 2 - th_red[:, np.newaxis] ** 2))[off]
    count = np.histogram2d(x, y, bins=(fd_edges, tau_edges))[0].T
    assert np.array_equal(cnt, count.astype(np.int32))
    V = V32.astype(np.complex128)
    for d in range(n_dish):
        m = np.zeros((n, n), complex)
        m[n // 2, :] = np.conjugate(V[d * n:(d + 1) * n]) * np.sqrt(w)
        ref = TO.rev_map(m, tau, fd, eta, edges_red, hermetian=False)
        assert np.abs(ref).max() > 0
        assert np.abs(recov[d] - ref).max() <= 1e-5 * np.abs(ref).max(), d


def test_vlbi_failures_recorded(golden_dir):
    f = np.load(os.path.join(golden_dir, "vlbi_sample_d.npz"))
    assert str(f["zero_error"]) == "ArpackError"
    assert str(f["wide_error"]) == "IndexError"
    assert str(f["one_error"]) == "IndexError"


def test_small_crop_raises_like_reference(golden_dir):
    """Host side: a crop of one centre gives the reference's exception type."""
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import ththmod
    f = np.load(os.path.join(golden_dir, "vlbi_sample_d.npz"))
    npad = int(f["npad"])
    tau, fd = TO.fft_axis(f["freq"], "us", npad), TO.fft_axis(f["time"], "mHz", npad)
    th = TO.theta_centres(f["edges"])
    _, errs = ththmod._rev_centres(th, tau, fd, np.array([float(f["one_eta"])]), min_crop=0)
    assert type(errs[0]).__name__ == str(f["one_error"])


def test_library_exports_vlbi_symbols():
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _lib, ththmod
    for name in ("sb_cs_c2c_f32", "sb_vlbi_retrieval"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib, name)
    assert _lib.lib.sb_abi_version() >= 4
    assert callable(ththmod.VLBI_chunk_retrieval)
