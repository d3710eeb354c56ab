"""The device code of scint_sim.Brightness (csrc/brightness.cu) on the CPU under the SIMT
emulator (tests/host_emu/brightness_emu.cpp): the unchanged kernels, launched as the driver
launches them, on small batches whose matrix products span several output tiles and
partial edge tiles, against the float64 oracle (oracle/brightness_oracle.py).  thetax,
thetay and the Jacobian are bit-equal; the rest are held to the GPU test's bars."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import brightness_oracle as BO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")
EPS = np.finfo(np.float64).eps


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(EMU, "brightness_emu.cpp")
    out = os.path.join(EMU, "_build", "brightness_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-x",
                    "c++", src, "-o", out], check=True)
    lib = ctypes.CDLL(out)
    lib.emu_brightness.restype = None
    return lib


def run(lib, sets, grid):
    """Every stage for the parameter sets on one grid, through the port's host halves."""
    from scintools_b200 import _lib
    from scintools_b200 import scint_sim as S
    objs = []
    for p in sets:
        o = S.Brightness.__new__(S.Brightness)
        o.__dict__.update(dict(ar=1.0, psi=0, alpha=1.67, thetagx=0, thetagy=0, thetarx=0,
                               thetary=0), **grid)
        o.__dict__.update(p)
        objs.append(o)
    ns = len(objs)
    par = np.zeros((ns, S._BRIGHT_NPAR))
    hs = [S._sspec_host(o) for o in objs]
    for k, o in enumerate(objs):
        x, _, _, par[k, :4] = S._efield_host(o)
        par[k, 4:] = hs[k][4]
    fd, td = hs[0][0], hs[0][1]
    n, ntd, nfd = len(x), len(td), len(fd)
    bits = S.lattice_diagonals(x)
    keep = dict(x=x, bits=bits, td=td, par=par, colx=np.stack([h[2] for h in hs]),
                colq=np.stack([h[3] for h in hs]))
    out = {k: np.full((ns, n, n), np.nan) for k in ("acf_efield", "B")}
    out.update({k: np.full((ns, ntd, nfd), np.nan)
                for k in ("thetax", "thetay", "jacobian", "SS", "LSS", "acf")})
    m = _lib.Brightness()
    m.nset, m.n, m.ntd, m.nfd, m.stages = ns, n, ntd, nfd, 7
    for f, k in (("x", "x"), ("diag", "bits"), ("td", "td"), ("par", "par"), ("colx", "colx"),
                 ("colq", "colq")):
        setattr(m, f, keep[k].ctypes.data)
    for f, k in (("rho", "acf_efield"), ("B", "B"), ("thetax", "thetax"), ("thetay", "thetay"),
                 ("jac", "jacobian"), ("ss", "SS"), ("lss", "LSS"), ("acf", "acf")):
        setattr(m, f, out[k].ctypes.data)
    sc = hs[0][5]
    m.half_df, m.jac_cap, m.jac_out = sc["half_df"], sc["jac_cap"], sc["jac_out"]
    lib.emu_brightness(ctypes.byref(m))
    return out


def check(got, ref):
    for k in ("thetax", "thetay", "jacobian"):
        assert np.array_equal(got[k], ref[k]), k
    assert np.max(np.abs(got["acf_efield"] - ref["acf_efield"])) <= 4 * EPS
    mb = ref["B"].max()
    assert np.max(np.abs(got["B"] - ref["B"])) <= 1e-12 * mb
    fin = np.isfinite(ref["SS"])
    assert np.array_equal(np.isfinite(got["SS"]), fin)
    scale = 2e-12 * mb * ref["jacobian"].max()
    assert np.max(np.abs(got["SS"] - ref["SS"])[fin], initial=0) <= scale
    pos = fin & (ref["SS"] > 0)
    assert np.max(np.abs(got["LSS"] - ref["LSS"])[pos], initial=0) <= 1e-9
    if fin.all():
        assert np.max(np.abs(got["acf"] - ref["acf"])) <= 1e-12
    else:
        assert np.isnan(got["acf"]).all() and np.isnan(ref["acf"]).all()


CASES = {
    # 70^2 lattice and 70 delays: 2 x 2 output tiles in every product, two sets
    "two_tiles": ([dict(ar=2.0, psi=30), dict(ar=1.2, psi=-70, alpha=1.3, thetagx=0.05,
                                              thetagy=0.1, thetarx=0.02, thetary=-0.03)],
                  dict(nx=3.5, dx=0.1, nf=0.45, df=0.05, nt=5.6, dt=0.16)),
    # odd lattice (19) and odd query grid (9 x 13); thetay leaves the lattice: NaN
    "odd_hull": ([dict(ar=3, psi=10, alpha=2)], dict(nx=0.95, dx=0.1, nf=0.09, df=0.02,
                                                     nt=1.04, dt=0.16)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_emulated_kernels_match_oracle(emu, name):
    sets, grid = CASES[name]
    got = run(emu, sets, grid)
    for k, p in enumerate(sets):
        ref = BO.model(**dict(grid, **p))
        check({a: v[k] for a, v in got.items()}, ref)
    if name == "odd_hull":
        assert np.isnan(got["SS"]).any()
