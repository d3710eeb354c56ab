"""Chi-square search on the CPU: the numpy oracle's chisq_calc against the reference's
values (tests/golden/chisq_sample_64x150.npz), and the device code of sb::chisq_sweep
up to the inverse FFT (crop, gather, batched eigenpair, rank-1 scatter) under the SIMT
emulator (tests/host_emu/chisq_emu.cpp) against the oracle."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import chisq_oracle as CO
from oracle import thth_oracle as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")


@pytest.fixture(scope="module")
def fx(golden_dir):
    return (np.load(os.path.join(golden_dir, "chisq_sample_64x150.npz")),
            np.load(os.path.join(golden_dir, "thth_sample_64x150.npz")))


def _case(fx, tag):
    c, g = fx
    npad = int(c["npad"])
    if tag == "a":
        d2 = g["dspec2"]
        return d2, TO.conjugate_spectrum(d2 - d2.mean(), npad, 0.0), g["tau"], g["fd"], \
            np.ones(d2.shape, bool)
    db = g["dspec2"][:, :128]
    return c["b_dspec"], TO.conjugate_spectrum(db, npad, None), c["b_tau"], c["b_fd"], c["b_mask"]


@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_chisq_matches_reference(fx, tag):
    """Every fifth curvature of cases a (chirp-z sizes) and b (mask, NaN outside it)."""
    c, _ = fx
    dspec, CS, tau, fd, mask = _case(fx, tag)
    for k in range(0, len(c["etas"]), 5):
        got = CO.chisq_calc(dspec, CS, tau, fd, c["etas"][k], c["edges"], float(c["N"]), mask)
        ref = c[tag + "_chisq"][k]
        assert abs(got - ref) <= 1e-9 * ref, (k, got, ref)


def test_oracle_chisq_zero_spectrum_raises(fx):
    """Case c: the reference raises on an all-zero conjugate spectrum; so does the oracle."""
    c, g = fx
    db = g["dspec2"][:, :128]
    zeros = np.zeros((len(c["b_tau"]), len(c["b_fd"])), complex)
    for e, name in zip(c["c_etas"], c["c_error"]):
        assert name
        with pytest.raises(Exception) as ex:
            CO.chisq_calc(db, zeros, c["b_tau"], c["b_fd"], e, c["edges"], float(c["N"]))
        assert type(ex.value).__name__ == name


def _emu_lib():
    src = os.path.join(EMU, "chisq_emu.cpp")
    out = os.path.join(EMU, "_build", "chisq_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    csrc = os.path.join(ROOT, "scintools_b200", "csrc")
    newest = max([os.path.getmtime(os.path.join(csrc, f)) for f in os.listdir(csrc)] +
                 [os.path.getmtime(src), os.path.getmtime(os.path.join(EMU, "simt.h"))])
    if not os.path.exists(out) or os.path.getmtime(out) < newest:
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                        "-x", "c++", src, "-o", out], check=True)
    return ctypes.CDLL(out)


def test_chisq_kernels_on_host(fx):
    """Case b, three curvatures: cropped sizes and occupied bins (counts) bit-exact, top
    eigenvalue and bin means to 1e-5 against the oracle's thth_redmap, dense eigh and
    rev_map of |w| V V^H on the reference's edges_red."""
    c, _ = fx
    dspec, CS, tau, fd, mask = _case(fx, "b")
    edges = c["edges"]
    th = TO.theta_centres(edges)
    n_th = len(th)
    sel = [10, 45, 80]
    etas = np.ascontiguousarray(c["etas"][sel])
    neta, ld = len(sel), 32 * ((n_th + 31) // 32)
    # per-curvature rev_map centres, as the host layer computes them
    th_red = np.zeros((neta, n_th))
    refs = []
    for k, e in enumerate(etas):
        red, edges_red = TO.thth_redmap(CS, tau, fd, e, edges)
        cents = TO.theta_centres(edges_red)
        th_red[k, :len(cents)] = cents
        refs.append((red, edges_red))
    ntau, nfd = CS.shape
    cs32 = np.ascontiguousarray(CS.astype(np.complex64))
    nred = np.zeros(neta, np.int32)
    status = np.zeros(neta, np.int32)
    iters = np.zeros(neta, np.int32)
    w = np.zeros(neta)
    V = np.zeros((neta, ld), np.complex64)
    recov = np.zeros((neta, ntau, nfd), np.complex64)
    cnt = np.zeros((neta, ntau, nfd), np.int32)
    lib = _emu_lib()
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    c_ll, c_d, c_i, vp = ctypes.c_longlong, ctypes.c_double, ctypes.c_int, ctypes.c_void_p
    lib.emu_chisq_stages.argtypes = [vp, c_ll, c_ll, c_d, c_d, c_d, c_d, c_d, c_d, vp, c_i, vp,
                                     c_i, vp, c_d, c_d, c_d, c_i, vp, vp, vp, vp, vp, vp, vp]
    lib.emu_chisq_stages(P(cs32), ntau, nfd, float(tau[0]), float(np.diff(tau).mean()),
                         float(abs(tau.max())), float(fd[0]), float(np.diff(fd).mean()),
                         float(abs(fd.max()) / 2), P(th), n_th, P(etas), neta, P(th_red),
                         float(tau[1] - tau[0]), float(fd[1] - fd[0]), 1e-7, 96, P(nred),
                         P(status), P(w), P(iters), P(V), P(recov), P(cnt))
    assert (status == 0).all(), status
    fd_edges = (np.linspace(0, nfd, nfd + 1) - .5) * (fd[1] - fd[0]) + fd[0]
    tau_edges = (np.linspace(0, ntau, ntau + 1) - .5) * (tau[1] - tau[0]) + tau[0]
    for k, e in enumerate(etas):
        red, edges_red = refs[k]
        n = red.shape[0]
        assert nred[k] == n == int(TO.th_points(tau, fd, e, edges).sum())
        wv, Vv = np.linalg.eigh(red)
        assert abs(w[k] - wv[-1]) <= 1e-5 * abs(wv[-1])
        rank1 = np.abs(wv[-1]) * np.outer(Vv[:, -1], np.conj(Vv[:, -1]))
        ref = TO.rev_map(rank1, tau, fd, e, edges_red)
        # histogram2d counts of rev_map (both half planes), diagonal points excluded
        tc = TO.theta_centres(edges_red)
        x = (tc[np.newaxis, :] - tc[:, np.newaxis])[~np.eye(n, dtype=bool)]
        y = (e * (tc[np.newaxis, :] ** 2 - tc[:, np.newaxis] ** 2))[~np.eye(n, dtype=bool)]
        count = (np.histogram2d(x, y, bins=(fd_edges, tau_edges))[0] +
                 np.histogram2d(-x, -y, bins=(fd_edges, tau_edges))[0]).T
        assert np.array_equal(cnt[k], count.astype(np.int32))
        assert np.abs(recov[k] - ref).max() <= 1e-5 * np.abs(ref).max()
