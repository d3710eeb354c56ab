"""The curvature-sweep gather from the compact, delay-contiguous copy of the spectrum
columns a theta grid reaches (csrc/thth.cu: thth_colmark_kernel, thth_colslots_kernel,
cs_compact_kernel, thth_build_copy_kernel) on the CPU under the SIMT emulator
(tests/host_emu/compact_gather_emu.cpp).  Every buffer the kernels get has the size the
library allocates and sits between inaccessible pages, so an index outside it kills the
process: each case therefore runs in a child process, which also makes the comparisons."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")


def _lib():
    src = os.path.join(EMU, "compact_gather_emu.cpp")
    out = os.path.join(EMU, "_build", "compact_gather_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    csrc = os.path.join(ROOT, "scintools_b200", "csrc")
    newest = max([os.path.getmtime(os.path.join(csrc, f)) for f in os.listdir(csrc)] +
                 [os.path.getmtime(os.path.join(EMU, f)) for f in os.listdir(EMU)
                  if f.endswith((".cpp", ".h"))])
    if not os.path.exists(out) or os.path.getmtime(out) < newest:
        subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                        "-x", "c++", src, "-o", out], check=True)
    return ctypes.CDLL(out)


def _axes(ntau, nfd, dtau=0.25, dfd=0.05):
    return (np.arange(ntau) - ntau // 2) * dtau, (np.arange(nfd) - nfd // 2) * dfd


def _centres(edges):
    return np.ascontiguousarray((edges[1:] + edges[:-1]) / 2)


def _case(name):
    """-> dict(ntau, nfd, half, pitch, th, etas, coherent, pack, expect)"""
    rng = np.random.default_rng(sum(map(ord, name)))
    c = dict(ntau=32, nfd=128, half=0, pitch=0, coherent=1, pack=2, expect={})
    tau, fd = _axes(c["ntau"], c["nfd"])
    lim = 0.45 * fd.max()                       # |theta_j - theta_i| stays on the fd axis
    if name == "uniform_511_half":
        c.update(ntau=32, nfd=2048, half=1, pitch=2048 // 2 + 16)
        tau, fd = _axes(c["ntau"], c["nfd"])
        c["th"] = _centres(np.linspace(-0.45 * fd.max(), 0.45 * fd.max(), 512))
        c["etas"] = tau.max() / c["th"].max() ** 2 * np.array([0.3, 0.31, 0.9, 1.5])
        c["expect"] = dict(max_slots=2 * 511)
    elif name == "uniform_small_full":
        c["th"] = _centres(np.linspace(-lim, lim, 42))
        c["etas"] = tau.max() / lim ** 2 * np.array([0.2, 0.5, 0.95, 1.0, 1.05, 2.0, 3.0, 4.0, 6.0])
    elif name == "nonuniform_edges":
        c.update(nfd=16384)
        tau, fd = _axes(c["ntau"], c["nfd"])
        lim = 0.45 * fd.max()
        c["th"] = _centres(np.sort(rng.uniform(-lim, lim, 70)))
        c["etas"] = tau.max() / lim ** 2 * np.array([0.3, 0.8, 1.7])
        c["expect"] = dict(min_slots=69 * 68 // 4)     # most pairs on a column of their own
    elif name == "half_narrow":
        c.update(half=1, pitch=128 // 2 + 16)
        c["th"] = _centres(np.linspace(-0.2 * fd.max(), 0.2 * fd.max(), 50))
        c["etas"] = tau.max() / (0.2 * fd.max()) ** 2 * np.array([0.4, 0.9, 1.3])
        c["expect"] = dict(max_col=int(0.4 * fd.max() / 0.05) + 2)
    elif name == "span_past_fd_axis":
        # theta differences up to 3.2 fd.max: bins beyond the axis (masked) ...
        c["th"] = _centres(np.linspace(-1.6 * fd.max(), 1.6 * fd.max(), 40))
        c["etas"] = tau.max() / fd.max() ** 2 * np.array([0.5, 2.0, 8.0])
    elif name == "wrap_negative":
        # ... and, on a descending grid, negative bins: python's wrap down to -nfd, then
        # the IndexError status
        c["th"] = _centres(np.linspace(1.6 * fd.max(), -1.6 * fd.max(), 40))
        c["etas"] = tau.max() / fd.max() ** 2 * np.array([0.5, 2.0, 8.0])
        c["expect"] = dict(index_error=True)
    elif name == "incoherent":
        c.update(coherent=0, half=1, pitch=128 // 2 + 1)
        c["th"] = _centres(np.linspace(-lim, lim, 37))
        c["etas"] = tau.max() / lim ** 2 * np.array([0.5, 1.5])
    elif name == "crop_moves_pairs":
        # eight curvatures of one CTA, each cropping a different number of centres
        c.update(pack=0)
        c["th"] = _centres(np.linspace(-lim, lim, 75))
        c["etas"] = tau.max() / lim ** 2 * np.linspace(0.9, 6.0, 8)
        c["expect"] = dict(distinct_nred=6)
    elif name == "mirrored_rows_1_and_last":
        # descending grid in the half layout: every pair lies in the mirrored half (row
        # ntau - tq).  For the pair (i, j) with the largest |theta1^2 - theta2^2| that survives
        # the crop, eta puts eta d at tau[ntau - 1] - 0.4 dtau (tq = ntau - 1, row 1); its
        # mirror image (-d) then has tq = 1, row ntau - 1.
        c.update(half=1, pitch=128 // 2 + 4)
        th = _centres(np.linspace(lim, -lim, 41))
        c["th"] = th
        i, j = 19, 39                          # theta_i next to zero, theta_j at the far end
        d = abs(th[j] ** 2 - th[i] ** 2)
        c["etas"] = np.array([(tau[-1] - 0.4 * 0.25) / d, 0.5 * (tau[-1] - 0.4 * 0.25) / d])
        c["expect"] = dict(rows={1, c["ntau"] - 1})
    else:
        raise KeyError(name)
    c["th"] = np.ascontiguousarray(c["th"], dtype=np.float64)
    c["etas"] = np.ascontiguousarray(c["etas"], dtype=np.float64)
    return c


CASES = ["uniform_511_half", "uniform_small_full", "nonuniform_edges", "half_narrow",
         "span_past_fd_axis", "wrap_negative", "incoherent", "crop_moves_pairs",
         "mirrored_rows_1_and_last"]


def _run(name):
    c = _case(name)
    lib = _lib()
    ntau, nfd, half = c["ntau"], c["nfd"], c["half"]
    tau, fd = _axes(ntau, nfd)
    pitch = c["pitch"] if half else nfd
    ncols = nfd // 2 + 1 if half else nfd
    rng = np.random.default_rng(7)
    cs = (rng.normal(size=(ntau, pitch)) + 1j * rng.normal(size=(ntau, pitch))).astype(np.complex64)
    # every element distinct, so that a gather from a wrong bin cannot go unnoticed
    cs += (np.arange(ntau * pitch).reshape(ntau, pitch) * 1e-3).astype(np.complex64)
    th, etas = c["th"], c["etas"]
    n, neta = len(th), len(etas)
    ld = 32 * ((n + 31) // 32)
    Mc = np.zeros((neta, ld, ld), np.complex64)
    Md = np.zeros_like(Mc)
    Mr = np.zeros_like(Mc)
    Bc = np.zeros((neta, ld * ld), np.uint32)
    Bd = np.zeros_like(Bc)
    nred = np.zeros(neta, np.int32)
    status = np.zeros(neta, np.int32)
    soc = np.zeros(ncols, np.int32)
    cos = np.zeros(ncols, np.int32)
    info = np.zeros(4, np.int32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    c_ll, c_d, c_i, vp = ctypes.c_longlong, ctypes.c_double, ctypes.c_int, ctypes.c_void_p
    lib.emu_compact_gather.argtypes = [vp, c_ll, c_ll, c_ll, c_i, c_d, c_d, c_d, c_d, c_d, c_d, vp,
                                       c_i, c_i, vp, c_i, c_i] + [vp] * 10
    rc = lib.emu_compact_gather(P(cs), ntau, nfd, pitch, half, float(tau[0]),
                                float(np.diff(tau).mean()), float(abs(tau.max())), float(fd[0]),
                                float(np.diff(fd).mean()), float(abs(fd.max()) / 2), P(th), n,
                                c["coherent"], P(etas), neta, c["pack"], P(Mc), P(Md), P(Mr),
                                P(Bc), P(Bd), P(nred), P(status), P(soc), P(cos), P(info))
    assert rc == 0, rc
    nslots, nslots_host, err, ncols_dev = (int(v) for v in info)
    assert ncols_dev == ncols
    assert err == 0
    assert nslots == nslots_host
    # slot_of_col / col_of_slot are inverses of each other; slots are dense
    mapped = np.flatnonzero(soc >= 0)
    assert len(mapped) == nslots and (soc[soc < 0] == -1).all()
    assert np.array_equal(np.sort(soc[mapped]), np.arange(nslots))
    assert np.array_equal(cos[soc[mapped]], mapped)
    assert np.array_equal(soc[cos[:nslots]], np.arange(nslots))
    # the whole slabs, junk included, are the same bytes from either source
    assert np.array_equal(Mc.view(np.uint32), Md.view(np.uint32))
    if c["pack"]:
        assert np.array_equal(Bc, Bd)
    # against thth_herm_upper on the cropped grid: same bins (distinct CS elements), the
    # Jacobian is a product of two fp32 roots here and one root there
    gathered = 0
    for e in range(neta):
        k = int(nred[e])
        up = np.triu(np.ones((k, k), bool), 1)
        got, ref = Mc[e, :k, :k][up], Mr[e, :k, :k][up]
        assert np.array_equal(got == 0, ref == 0)
        assert (np.abs(got - ref) <= 1e-6 * np.abs(ref)).all()
        assert (Mc[e, :k, :k][np.diag_indices(k)] == 0).all()
        gathered += int((got != 0).sum())
    ex = c["expect"]
    if not ex.get("index_error"):
        assert gathered > 0
    else:
        assert (status & 1).any()
    if "max_slots" in ex:
        assert nslots <= ex["max_slots"]
    if "min_slots" in ex:
        assert nslots >= ex["min_slots"]
    if "max_col" in ex:
        assert mapped.max() <= ex["max_col"]
    if "distinct_nred" in ex:
        assert len(set(nred.tolist())) >= ex["distinct_nred"], nred
    if "rows" in ex:
        # rows the kept pairs of the first curvature gather from, by the kernel's formula
        k = int(nred[0])
        assert k == n, (k, n)
        dtau = float(np.diff(tau).mean())
        d = th[None, :] ** 2 - th[:, None] ** 2            # [row i][column j]
        tq = np.floor((etas[0] * d - tau[0] + dtau / 2) / dtau).astype(int)
        iu = np.triu_indices(n, 1)
        keep = (iu[0] + iu[1] != n - 1) & (tq[iu] > 0) & (tq[iu] < ntau)
        rows = set((ntau - tq[iu][keep]).tolist())
        assert ex["rows"] <= rows, sorted(rows)
    print("ok", name, "nslots", nslots, "of", ncols, "gathered", gathered)


@pytest.mark.parametrize("name", CASES)
def test_compact_gather_matches_direct(name):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), name], capture_output=True,
                       text=True, cwd=ROOT)
    assert r.returncode == 0, "child exit %d\n%s\n%s" % (r.returncode, r.stdout, r.stderr)
    assert r.stdout.startswith("ok " + name)


if __name__ == "__main__":
    _run(sys.argv[1])
