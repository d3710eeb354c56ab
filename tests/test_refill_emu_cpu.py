"""The device code of the gap fills (csrc/inpaint.cu) on the CPU under the SIMT emulator
(tests/host_emu/inpaint_emu.cpp): the BiCGSTAB kernels, launched as the driver launches
them, against the oracle's spsolve on a 24 x 40 image, with several blocks per launch run
one after another; and the masked median against scipy.signal.medfilt."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import refill_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")
NF, NT = 24, 40


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(EMU, "inpaint_emu.cpp")
    out = os.path.join(EMU, "_build", "inpaint_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-x",
                    "c++", src, "-o", out], check=True)
    return ctypes.CDLL(out)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _run(emu, img, mask, threads, G, tol=1e-10, maxit=5000):
    from scintools_b200.dynspec import _stencil_tables
    nf, nt = img.shape
    pix = np.flatnonzero(mask).astype(np.int32)
    rcls, ccls, tables = _stencil_tables(nf, nt)
    known = img[~mask]
    img = np.ascontiguousarray(img, dtype=np.float64)
    out = np.zeros(pix.size)
    info = np.zeros(4, np.int32)
    resid = np.zeros(1)
    d = ctypes.c_double
    assert emu.emu_inpaint(_p(img), nf, nt, _p(pix), pix.size, _p(tables), _p(rcls),
                           tables.shape[0], _p(ccls), tables.shape[1], d(known.min()),
                           d(known.max()), d(tol), maxit, threads, G, _p(out), _p(info),
                           _p(resid)) == 0
    return out, info, resid[0]


def _masks():
    rng = np.random.default_rng(21)
    out = {"random15": rng.random((NF, NT)) < 0.15}
    m = np.zeros((NF, NT), bool)
    m[6:14, 10:22] = True
    m[0, :] = m[:, NT - 1] = True
    m[NF - 2:, :3] = True
    out["block_edges"] = m
    # isolated pixels (no masked pixel within two of another): A D^-1 is the identity, so
    # the first half step meets the rule -- kernel C's stop path, in every block
    m = np.zeros((NF, NT), bool)
    m[::3, ::3] = True
    out["isolated"] = m
    return out


MASKS = _masks()


@pytest.mark.parametrize("name", sorted(MASKS))
@pytest.mark.parametrize("threads,G", [(32, 2), (32, 5), (64, 64)])
def test_solver_kernels_match_spsolve(emu, name, threads, G):
    mask = MASKS[name]
    img = np.random.default_rng(len(name)).exponential(1.0, mask.shape)
    img[mask] = np.nan
    ref = O.biharmonic(img, mask)[mask]
    got, info, resid = _run(emu, img, mask, threads, G)
    known = img[~mask]
    err = np.max(np.abs(got - ref)) / (known.max() - known.min())
    print("%s, %d x %d: %d steps, %d restarts, stop launch %d, residual %.2e, err %.2e"
          % (name, G, threads, info[0], info[2], info[3], resid, err))
    assert info[1] == 1 and resid <= 1e-10
    assert err <= 1e-7
    if name == "isolated":
        assert info[0] == 1 and info[3] == 2 and info[2] == 0     # kernel C of step 0


def test_grids_agree_and_repeat(emu):
    """The result depends on the grid only through the partial sums' order: all grids agree
    to the tolerance, and each grid repeats bit for bit."""
    mask = MASKS["random15"] | MASKS["block_edges"]
    img = np.random.default_rng(5).exponential(1.0, mask.shape)
    a, ia, _ = _run(emu, img, mask, 32, 3)
    b, ib, _ = _run(emu, img, mask, 32, 3)
    c, _, _ = _run(emu, img, mask, 64, 1)
    assert np.array_equal(a, b) and np.array_equal(ia, ib)
    assert np.max(np.abs(a - c)) <= 1e-7 * (img[~mask].max() - img[~mask].min())


def test_cap_stops_every_run(emu):
    mask = MASKS["block_edges"]
    img = np.random.default_rng(6).exponential(1.0, mask.shape)
    got, info, resid = _run(emu, img, mask, 32, 4, maxit=7)
    assert info[0] == 7 and info[1] == 0 and np.all(np.isfinite(got))


@pytest.mark.parametrize("ks", [(3, 3), (5, 5), (3, 7), (11, 11), (31, 31)])
def test_median_kernel(emu, ks):
    rng = np.random.default_rng(8)
    img = rng.exponential(1.0, (NF, NT))
    mask = rng.random((NF, NT)) < 0.2
    img[mask] = np.nan
    fill = float(np.mean(img[~mask]))
    pix = np.flatnonzero(mask).astype(np.int32)
    out = np.zeros(pix.size)
    assert emu.emu_medfilt(_p(img), NF, NT, _p(pix), pix.size, ks[0], ks[1],
                           ctypes.c_double(fill), _p(out)) == 0
    from scipy.signal import medfilt
    ref = medfilt(np.where(mask, fill, img), ks)[mask]
    assert np.array_equal(out, ref)
