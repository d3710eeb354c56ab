"""The device code of the theoretical intensity ACF (csrc/acf_model.cu) on the CPU under the
SIMT emulator (tests/host_emu/acf_model_emu.cpp): the unchanged kernels, launched as the
driver launches them, on small grids with several row tiles, lag tiles and blocks per
column.  The ACF is within 1e-12 amp of the float64 direct-sum oracle
(oracle/acf_model_oracle.py), the e-field table within 1e-14, and both mirrorings and the
wn rows land where the oracle puts them."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import acf_model_oracle as AO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")
D = ctypes.c_double
P = ctypes.POINTER(ctypes.c_double)
I = ctypes.c_int


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(EMU, "acf_model_emu.cpp")
    out = os.path.join(EMU, "_build", "acf_model_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-x",
                    "c++", src, "-o", out], check=True)
    lib = ctypes.CDLL(out)
    lib.emu_acf_model.restype = I
    lib.emu_acf_model.argtypes = [P, I, P, I, P, I, P, P, I, I] + [D] * 8 + [P, P]
    return lib


def _p(a):
    return a.ctypes.data_as(P)


def run(lib, kw):
    from scintools_b200.scint_sim import ACF
    a = ACF.__new__(ACF)
    a.calc_acf = lambda: None
    ACF.__init__(a, **kw)
    h = a._axes()
    arrs = [np.ascontiguousarray(h[k], dtype=np.float64)
            for k in ("snp", "snp2", "dnun", "snx", "sny")]
    nsn, nd, n1 = len(arrs[3]), len(arrs[2]), len(arrs[0])
    nt = 2 * nsn - 1 if h["quadrant"] else nsn
    acf = np.full((2 * nd - 1, nt), np.nan)
    ef = np.full((n1, n1), np.nan)
    nb = lib.emu_acf_model(_p(arrs[0]), n1, _p(arrs[1]), len(arrs[1]), _p(arrs[2]), nd,
                           _p(arrs[3]), _p(arrs[4]), nsn, int(h["quadrant"]), h["sigxn"],
                           h["sigyn"], h["sqrtar"], h["alph2"], h["step1"], h["step2"],
                           h["wn_amp"], h["amp"], _p(acf), _p(ef))
    return acf, ef, nb, h


CASES = {
    # half plane: 79 lags (3 lag tiles), grids 79 / 157 (2 and 3 row tiles)
    "half_plane": dict(nt=79, nf=7, phasegrad=0.2, theta=20, psi=35, wn=0.1, amp=0.7,
                       taumax=4, auto_sampling=False, spatial_factor=1, resolution_factor=2,
                       core_factor=2),
    # quadrant: 26 lags, grids 51 / 204
    "quadrant": dict(nt=51, nf=5, psi=70, wn=0.05),
    # alpha 1.2, ar 2, lags with no exact zero (wn dropped)
    "no_zero_lag": dict(nt=21, nf=9, ar=2, alpha=1.2, phasegrad=0.1, theta=-40, wn=0.3,
                        taumax=3.7, auto_sampling=False, spatial_factor=1.5,
                        resolution_factor=1, core_factor=3),
}


@pytest.mark.parametrize("name", list(CASES))
def test_emulated_kernels_match_oracle(emu, name):
    kw = CASES[name]
    acf, ef, nb, h = run(emu, kw)
    _, ref, ref_ef = AO.model(**kw)
    assert acf.shape == ref.shape
    assert np.all(np.isfinite(acf))
    err = np.max(np.abs(acf - ref))
    print("%s: %d blocks, max |acf - oracle| = %.2e" % (name, nb, err))
    assert err <= 1e-12 * kw.get("amp", 1)
    assert np.max(np.abs(ef - ref_ef)) <= 1e-14
    if name == "half_plane":            # row tiles split over several blocks per column
        assert nb > 3 * (len(h["dnun"]) - 1)


def test_emulated_plan_is_deterministic(emu):
    kw = CASES["half_plane"]
    a1 = run(emu, kw)[0]
    a2 = run(emu, kw)[0]
    assert np.array_equal(a1, a2)
