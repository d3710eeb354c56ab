"""Dynspec.cut_dyn without a GPU: argument errors come before any device work, and the
tile shapes, the slicing and cutdyn match the reference's fixtures bit for bit with the
device call replaced by the CPU oracle (which must then reproduce cutsspec and the
per-tile ACFs to the float32 rounding of the fixtures)."""
import glob
import os

import numpy as np
import pytest

from oracle import dynspec_oracle as DO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "cut_dyn_*.npz")))


def _ds(dyn, dt=10.0, df=0.1):
    from scintools_b200.dynspec import BasicDyn, Dynspec
    nf, nt = dyn.shape
    bd = BasicDyn(dyn, times=dt * np.arange(nt), freqs=1400.0 + df * np.arange(nf), dt=dt,
                  df=df)
    return Dynspec(dyn=bd, verbose=False)


def _no_device(monkeypatch):
    from scintools_b200 import _device
    monkeypatch.setattr(_device, "device", lambda: pytest.fail("device touched"))


@pytest.mark.parametrize("shape,kw,exc", [
    ((16, 40), dict(plot=True), NotImplementedError),
    ((16, 40), dict(lamsteps=True), AttributeError),
    ((16, 40), dict(fcuts=8), ValueError),        # fnum = 1
    ((16, 40), dict(fcuts=16), ValueError),       # fnum = 0
    ((16, 40), dict(tcuts=8), ValueError),        # tnum = 4
    ((32769, 5), {}, ValueError),                 # fnum above 32768
    ((2, 16385), {}, ValueError),                 # tnum above 16384
])
def test_argument_errors_before_device(shape, kw, exc, monkeypatch):
    _no_device(monkeypatch)
    ds = _ds(np.ones(shape, np.float32))
    with pytest.raises(exc):
        ds.cut_dyn(**kw)
    assert not hasattr(ds, "cutdyn")


def _oracle_device(dyn, fnum, tnum, nfc, ntc, dtype):
    """Stand-in for dynspec._cut_dyn_device: the oracle's calc_sspec / calc_acf per tile."""
    sec, acf = [], []
    for ii in range(nfc):
        for jj in range(ntc):
            tile = np.asarray(dyn[ii * fnum:(ii + 1) * fnum, jj * tnum:(jj + 1) * tnum],
                              dtype=np.float64)
            sec.append(DO.calc_sspec(tile, 1.0, 1.0)[2])
            acf.append(DO.calc_acf(tile, normalise=True, subtract_mean=False))
    shape = lambda a: np.array(a).reshape((nfc, ntc) + a[0].shape).astype(dtype)
    return shape(sec), shape(acf)


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_slicing_matches_reference(path, monkeypatch):
    from scintools_b200 import dynspec
    _no_device(monkeypatch)
    monkeypatch.setattr(dynspec, "_cut_dyn_device", _oracle_device)
    g = np.load(path)
    ds = _ds(g["dyn"].copy(), float(g["dt"]), float(g["df"]))
    ds.cut_dyn(tcuts=int(g["tcuts"]), fcuts=int(g["fcuts"]))
    assert ds.cutdyn.dtype == np.float64
    assert ds.cutdyn.shape == g["cutdyn"].shape
    assert np.array_equal(ds.cutdyn, g["cutdyn"], equal_nan=True)
    assert ds.cutsspec.shape == g["cutsspec"].shape
    assert ds.cutacf.shape == g["cutacf"].shape
    # the fixtures hold the reference's outputs rounded to float32
    fin = np.isfinite(g["cutsspec"])
    assert np.array_equal(fin, np.isfinite(ds.cutsspec))
    assert np.allclose(ds.cutsspec[fin], g["cutsspec"][fin], rtol=1e-6, atol=1e-5)
    fin = np.isfinite(g["cutacf"])
    assert np.array_equal(fin, np.isfinite(ds.cutacf))
    assert np.allclose(ds.cutacf[fin], g["cutacf"][fin], rtol=0, atol=1e-7)


def test_exports_present():
    from scintools_b200 import _lib
    for name in ("sb_sspec_tiles_f32", "sb_acf_tiles_f32"):
        assert name in _lib.EXPORTS
        assert hasattr(_lib.lib, name)
    header = open(os.path.join(ROOT, "include", "scint_b200.h")).read()
    assert "int sb_sspec_tiles_f32(" in header and "int sb_acf_tiles_f32(" in header
