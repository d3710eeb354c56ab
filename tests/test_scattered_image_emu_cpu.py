"""The device code of Dynspec.calc_scattered_image (csrc/scatim.cu) on the CPU under the SIMT
emulator (tests/host_emu/scatim_emu.cpp): the unchanged kernels, launched as the driver
launches them, on small crops through the port's host steps, against scipy's
RectBivariateSpline (oracle/scattered_image_oracle.py).  The cases put query points exactly
on knots and data points and beyond both ends of the delay axis, take the flim == 0 crop,
sampling 0 and 1, several items in one launch, and the shift."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import scattered_image_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")
BAR = 1e-10


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(EMU, "scatim_emu.cpp")
    out = os.path.join(EMU, "_build", "scatim_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-x",
                    "c++", src, "-o", out], check=True)
    lib = ctypes.CDLL(out)
    lib.emu_scattered_image.restype = None
    return lib


def run(lib, sspecs, fdop, tdel, etas, sampling, shift):
    """Images of the spectra [k][ntdel][nfdop] (one crop) through the port's host steps."""
    from scintools_b200 import _lib
    from scintools_b200 import dynspec as DS
    S = np.ascontiguousarray(sspecs, dtype=np.float64)
    K, nr, nc = S.shape
    plan = DS._scatim_plan((nr, nc), fdop, tdel, etas[0], sampling)
    for e in etas[1:]:
        p = DS._scatim_plan((nr, nc), fdop, tdel, e, sampling)
        assert (p["rows"], p["cols"]) == (plan["rows"], plan["cols"])
    (r0, _), (c0, _) = plan["rows"], plan["cols"]
    tx, fx = DS.spline_tables(plan["x"])
    ty, fy = DS.spline_tables(plan["y"])
    keep = [np.ascontiguousarray(a, dtype=np.float64)
            for a in (tx, fx, ty, fy, plan["fdop_x"], plan["fdop_y"], etas)]
    off = np.array([k * nr * nc + r0 * nc + c0 for k in range(K)], dtype=np.int64)
    nx, ny = len(plan["fdop_x"]), len(plan["fdop_y"])
    img = np.full((K, nx, nx), np.nan)
    s = _lib.ScatIm()
    s.nitem, s.mx, s.my, s.nx, s.ny, s.shift = K, len(plan["x"]), len(plan["y"]), nx, ny, shift
    s.pitch, s.sspec, s.offset, s.eta = nc, S.ctypes.data, off.ctypes.data, keep[6].ctypes.data
    s.tx, s.fx, s.ty, s.fy, s.ax, s.ay = (a.ctypes.data for a in keep[:6])
    s.image = img.ctypes.data
    lib.emu_scattered_image(ctypes.byref(s))
    return img, plan["fdop_x"]


def check(lib, sspecs, fdop, tdel, etas, sampling, shift=0):
    got, ax = run(lib, sspecs, fdop, tdel, etas, sampling, shift)
    for k, e in enumerate(etas):
        ref, rax = SO.scattered_image(sspecs[k], fdop, tdel, e, sampling, plot_log=bool(shift))
        assert np.array_equal(ax, rax)
        assert np.max(np.abs(got[k] - ref)) <= BAR * np.max(np.abs(ref)), k
    return got


def spectra(rng, k, nr, nc):
    return 10 * np.log10(rng.uniform(0.1, 10.0, (k, nr, nc)))


def test_small_7x9(emu):
    rng = np.random.default_rng(1)
    fdop = np.linspace(-4.0, 4.0, 9)
    tdel = np.linspace(0.0, 3.0, 7)
    for sampling in (0, 1, 5, 16):
        check(emu, spectra(rng, 1, 7, 9), fdop, tdel, [0.12], sampling)


def test_64x150_items_and_shift(emu):
    rng = np.random.default_rng(2)
    fdop = (np.arange(150) - 75) * 0.37
    tdel = np.arange(64) * 0.21
    got = check(emu, spectra(rng, 3, 64, 150), fdop, tdel, [0.1, 0.1001, 0.1002], 21, shift=1)
    assert np.all(got.min(axis=(1, 2)) == 1e-10)


def test_knots_and_both_ends(emu):
    """Integer axes and eta = 1: every query sits on a data point or knot of both axes; the
    delay queries run past the last delay, and below the first one (tdel starts at 5)."""
    rng = np.random.default_rng(3)
    fdop = np.arange(-10.0, 11.0)
    tdel = np.arange(5.0, 45.0)
    # the row of fdop_y = 6 queries delays 36..72, clamped to 44 past the last delay
    check(emu, spectra(rng, 1, 40, 21), fdop, tdel, [1.0], 6)


def test_flim0_crop(emu):
    """eta * fdop[0]**2 below the last delay: rows [:tlim] and the delay axis fdop[:tlim]."""
    rng = np.random.default_rng(4)
    fdop = np.linspace(-1.0, 1.0, 12)
    tdel = np.linspace(0.0, 5.0, 30)
    check(emu, spectra(rng, 2, 30, 12), fdop, tdel, [1.5, 1.5], 0)
    check(emu, spectra(rng, 1, 30, 12), fdop, tdel, [1.5], 1)
    check(emu, spectra(rng, 1, 30, 12), fdop, tdel, [1.5], 7, shift=1)


def test_minus_inf_and_nan(emu):
    """-inf dB is zero power; a NaN spreads to every pixel through the solves."""
    rng = np.random.default_rng(5)
    fdop = np.linspace(-4.0, 4.0, 17)
    tdel = np.linspace(0.0, 3.0, 11)
    s = spectra(rng, 1, 11, 17)
    s[0, 3, 5] = -np.inf
    check(emu, s, fdop, tdel, [0.1], 8)
    s[0, 2, 9] = np.nan
    got, _ = run(emu, s, fdop, tdel, [0.1], 8, 0)
    assert np.isnan(got).all()
