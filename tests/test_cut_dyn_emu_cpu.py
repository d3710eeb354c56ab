"""The tiled transforms of Dynspec.cut_dyn (csrc/tiles.cuh) on the CPU under the SIMT
emulator (tests/host_emu/cut_dyn_emu.cpp): per-tile statistics kernels as written, the tile
load / store functors around plain DFTs, on groups of three tiles, against
oracle/dynspec_oracle.py tile by tile.  This checks the tile index maps (parent slicing,
side-by-side half spectra, column-to-tile stores, per-tile planes and factors) without a
GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import dynspec_oracle as DO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(EMU, "cut_dyn_emu.cpp")
    out = os.path.join(EMU, "_build", "cut_dyn_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-x",
                    "c++", src, "-o", out], check=True)
    lib = ctypes.CDLL(out)
    vp, ci, cd = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    lib.emu_cut_dyn.argtypes = [vp, ci, ci, ci, ci, ci, ci, vp, vp, cd, cd, vp, vp]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _maxrel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


# (parent nf, nt, fnum, tnum, nfc, ntc, first tile of the group of three): a 2 x 2 grid
# whose group starts at tile 1 (so it spans two tile rows), a 1 x 3 grid with a dropped
# column, and a 3 x 1 grid of the smallest tiles
CASES = [(11, 17, 5, 7, 2, 2, 1), (6, 20, 6, 6, 1, 3, 0), (7, 5, 2, 5, 3, 1, 0)]


@pytest.mark.parametrize("nf,nt,fnum,tnum,nfc,ntc,tile0", CASES)
def test_tile_passes_match_oracle(emu, nf, nt, fnum, tnum, nfc, ntc, tile0):
    rng = np.random.default_rng(nf * 100 + nt)
    dyn = rng.exponential(1.0, (nf, nt)).astype(np.float32)
    ntile = 3
    nrfft, ncfft = DO.fft_lengths(fnum, tnum)
    cw, sw = DO.get_window(tnum, fnum)
    wt, wf = cw.astype(np.float32), sw.astype(np.float32)
    sec = np.full((ntile, nrfft // 2, ncfft), np.nan, np.float32)
    acf = np.full((ntile, 2 * fnum, 2 * tnum), np.nan, np.float32)
    assert emu.emu_cut_dyn(_p(dyn), nt, fnum, tnum, ntc, tile0, ntile, _p(wt), _p(wf),
                           float(cw.sum()), float(sw.sum()), _p(sec), _p(acf)) == 0
    for tl in range(ntile):
        ii, jj = divmod(tile0 + tl, ntc)
        tile = dyn[ii * fnum:(ii + 1) * fnum, jj * tnum:(jj + 1) * tnum].astype(np.float64)
        _, _, ref = DO.calc_sspec(tile, 1.0, 1.0, db=False)
        assert _maxrel(10 ** (sec[tl] / 10), ref) < 1e-5, tl
        ref = DO.calc_acf(tile, normalise=True, subtract_mean=False)
        assert _maxrel(acf[tl], ref) < 1e-5, tl
