"""Dynspec.cut_dyn on the GPU (sb_sspec_tiles_f32, sb_acf_tiles_f32): every tile against the
reference's fixtures, against the single-spectrum drivers (calc_sspec / calc_acf with
input_dyn=tile) and against the CPU oracle, past 65,535 tiles, across workspace groups,
and at the tile size limits."""
import glob
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import dynspec_oracle as DO   # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "cut_dyn_*.npz")))
RTOL = 1e-5


def maxrel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def _check_db(got_db, ref_db, rtol=RTOL, db_tol=2e-4):
    """The rule of test_gpu_parity.py: linear relative error and dB error on strong bins."""
    lin_g, lin_r = 10 ** (got_db / 10), 10 ** (ref_db / 10)
    assert maxrel(lin_g, lin_r) < rtol
    big = lin_r > 1e-3 * lin_r.max()
    assert np.max(np.abs(got_db[big] - ref_db[big])) < db_tol


@pytest.fixture(scope="module")
def sb():
    import scintools_b200
    from scintools_b200 import _device
    _device.device()
    return scintools_b200


def _ds(sb, dyn, dt=10.0, df=0.1):
    nf, nt = dyn.shape
    bd = sb.dynspec.BasicDyn(dyn, times=dt * np.arange(nt), freqs=1400.0 + df * np.arange(nf),
                             dt=dt, df=df)
    return sb.dynspec.Dynspec(dyn=bd, verbose=False)


def _tiles(ds):
    nfc, ntc = ds.cutdyn.shape[:2]
    return [(ii, jj) for ii in range(nfc) for jj in range(ntc)]


def _check_tiles_vs_drivers(ds, f32=False):
    """Every tile against calc_sspec / calc_acf(input_dyn=tile) of the existing drivers."""
    dt = np.float32 if f32 else np.float64
    for ii, jj in _tiles(ds):
        tile = ds.cutdyn[ii, jj]
        _, _, sec = ds.calc_sspec(input_dyn=tile, dtype=dt)
        _check_db(ds.cutsspec[ii, jj].astype(np.float64), sec.astype(np.float64))
        acf = ds.calc_acf(input_dyn=tile, dtype=dt)
        assert maxrel(ds.cutacf[ii, jj], acf) < RTOL, (ii, jj)


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_fixtures(sb, path):
    g = np.load(path)
    ds = _ds(sb, g["dyn"].copy(), float(g["dt"]), float(g["df"]))
    ds.cut_dyn(tcuts=int(g["tcuts"]), fcuts=int(g["fcuts"]))
    assert np.array_equal(ds.cutdyn, g["cutdyn"], equal_nan=True)
    assert ds.cutsspec.shape == g["cutsspec"].shape and ds.cutsspec.dtype == np.float64
    assert ds.cutacf.shape == g["cutacf"].shape and ds.cutacf.dtype == np.float64
    for ii, jj in _tiles(ds):
        # stored as float32 (6e-8 relative): widen before the 1e-5 checks
        ref_s = g["cutsspec"][ii, jj].astype(np.float64)
        ref_a = g["cutacf"][ii, jj].astype(np.float64)
        if np.isnan(g["cutdyn"][ii, jj]).any():      # a NaN makes its own tile NaN
            assert np.isnan(ref_s).all() and np.isnan(ref_a).all()
            assert np.isnan(ds.cutsspec[ii, jj]).all() and np.isnan(ds.cutacf[ii, jj]).all()
            continue
        _check_db(ds.cutsspec[ii, jj], ref_s)
        assert maxrel(ds.cutacf[ii, jj], ref_a) < RTOL, (ii, jj)
    finite = [t for t in _tiles(ds) if not np.isnan(ds.cutdyn[t]).any()]
    assert finite, "every tile is NaN"
    for t in finite:                                  # neighbours of a NaN tile are whole
        assert np.isfinite(ds.cutacf[t]).all()


def test_nan_tile_only(sb):
    path = os.path.join(ROOT, "tests", "golden", "cut_dyn_nan_64x96_t2_f1.npz")
    g = np.load(path)
    ds = _ds(sb, g["dyn"].copy())
    ds.cut_dyn(tcuts=2, fcuts=1)
    nan = [(ii, jj) for ii, jj in _tiles(ds) if np.isnan(ds.cutsspec[ii, jj]).any()]
    assert nan == [(1, 0)]
    assert np.isnan(ds.cutsspec[1, 0]).all() and np.isnan(ds.cutacf[1, 0]).all()


@pytest.mark.parametrize("shape,tcuts,fcuts", [((101, 152), 2, 1), ((128, 256), 3, 1),
                                               ((200, 300), 4, 2), ((97, 61), 1, 3)])
def test_tiles_match_single_drivers(sb, shape, tcuts, fcuts):
    dyn = np.random.default_rng(sum(shape)).exponential(1.0, shape)
    ds = _ds(sb, dyn)
    ds.cut_dyn(tcuts=tcuts, fcuts=fcuts)
    _check_tiles_vs_drivers(ds)


def test_whole_spectrum(sb):
    dyn = np.random.default_rng(5).exponential(1.0, (48, 80))
    ds = _ds(sb, dyn)
    ds.cut_dyn()
    _, _, sec = ds.calc_sspec(input_dyn=dyn)
    _check_db(ds.cutsspec[0, 0], sec)
    assert maxrel(ds.cutacf[0, 0], ds.calc_acf(input_dyn=dyn)) < RTOL


def test_float32(sb):
    dyn = np.random.default_rng(6).exponential(1.0, (100, 150))
    a, b = _ds(sb, dyn), _ds(sb, dyn)
    a.cut_dyn(tcuts=2, fcuts=1)
    b.cut_dyn(tcuts=2, fcuts=1, dtype=np.float32)
    assert b.cutsspec.dtype == np.float32 and b.cutacf.dtype == np.float32
    assert b.cutdyn.dtype == np.float64
    assert np.array_equal(a.cutsspec, b.cutsspec.astype(np.float64))
    assert np.array_equal(a.cutacf, b.cutacf.astype(np.float64))


def test_65536_tiles(sb):
    """256 x 256 tiles of 2 x 5 (a 512 x 1280 parent), each against the oracle."""
    dyn = np.random.default_rng(7).exponential(1.0, (512, 1280))
    ds = _ds(sb, dyn)
    ds.cut_dyn(tcuts=255, fcuts=255)
    assert ds.cutsspec.shape == (256, 256, 2, 16) and ds.cutacf.shape == (256, 256, 4, 10)
    for ii, jj in _tiles(ds):
        tile = ds.cutdyn[ii, jj]
        _, _, lin = DO.calc_sspec(tile, 10.0, 0.1, db=False)
        got = 10 ** (ds.cutsspec[ii, jj] / 10)
        assert maxrel(got, lin) < RTOL, (ii, jj)
        assert maxrel(ds.cutacf[ii, jj], DO.calc_acf(tile, subtract_mean=False)) < RTOL, (ii, jj)


def _launches(sb, fn):
    L = sb._lib
    n0 = L.lib.sb_launch_count()
    fn()
    return L.lib.sb_launch_count() - n0


def test_workspace_groups(sb):
    """4096 x 4096 tiles of an 8192 x 8192 parent: the secondary spectra run in two groups
    of two tiles and the ACFs in four groups of one (fixed 1 GiB workspace budget); every
    tile against the single-spectrum drivers."""
    import torch
    from scintools_b200 import _device as D
    L = sb._lib
    dyn = np.random.default_rng(8).exponential(1.0, (8192, 8192)).astype(np.float32)
    fnum = tnum = 4096
    d = D.upload(dyn)
    cw, sw = sb.dynspec.get_window(tnum, fnum)
    wt, wf = D.upload(cw.astype(np.float32)), D.upload(sw.astype(np.float32))
    sec = D.empty((2, 2, 4096, 8192), torch.float32)
    acf = D.empty((2, 2, 8192, 8192), torch.float32)
    n_s = _launches(sb, lambda: L.check(L.lib.sb_sspec_tiles_f32(
        d.data_ptr(), 8192, 8192, fnum, tnum, 2, 2, wt.data_ptr(), wf.data_ptr(),
        float(cw.sum()), float(sw.sum()), sec.data_ptr(), D.stream_ptr())))
    n_a = _launches(sb, lambda: L.check(L.lib.sb_acf_tiles_f32(
        d.data_ptr(), 8192, 8192, fnum, tnum, 2, 2, acf.data_ptr(), D.stream_ptr())))
    # per group: statistics (2) + rows (1) + columns (2); ACF: 2 + 1 + 3 + 1
    assert (n_s, n_a) == (2 * 5, 4 * 7)
    ds = _ds(sb, dyn)
    for ii in range(2):
        for jj in range(2):
            tile = dyn[ii * fnum:(ii + 1) * fnum, jj * tnum:(jj + 1) * tnum]
            _, _, ref = ds.calc_sspec(input_dyn=tile, dtype=np.float32)
            _check_db(D.download(sec[ii, jj]).astype(np.float64), ref.astype(np.float64))
            ref = ds.calc_acf(input_dyn=tile, dtype=np.float32)
            assert maxrel(D.download(acf[ii, jj]), ref) < RTOL


@pytest.mark.parametrize("shape", [(2, 5), (2, 16384), (32768, 5)])
def test_size_limits_inside(sb, shape):
    dyn = np.random.default_rng(9).exponential(1.0, shape)
    ds = _ds(sb, dyn)
    ds.cut_dyn(dtype=np.float32)
    _check_tiles_vs_drivers(ds, f32=True)


@pytest.mark.parametrize("fnum,tnum", [(1, 5), (2, 4), (32769, 5), (2, 16385)])
def test_size_limits_outside(sb, fnum, tnum):
    import torch
    from scintools_b200 import _device as D
    L = sb._lib
    d = D.zeros((fnum, tnum), torch.float32)
    out = D.zeros((1,), torch.float32)
    for fn in (lambda: L.lib.sb_acf_tiles_f32(d.data_ptr(), fnum, tnum, fnum, tnum, 1, 1,
                                              out.data_ptr(), D.stream_ptr()),
               lambda: L.lib.sb_sspec_tiles_f32(d.data_ptr(), fnum, tnum, fnum, tnum, 1, 1,
                                                None, None, 0.0, 0.0, out.data_ptr(),
                                                D.stream_ptr())):
        with pytest.raises(L.SbError, match="outside the supported sizes"):
            L.check(fn())
    ds = _ds(sb, np.ones((fnum, tnum)))
    with pytest.raises(ValueError):
        ds.cut_dyn()
