"""The device code of the cleaning passes (csrc/clean.cu) on the CPU under the SIMT emulator
(tests/host_emu/clean_emu.cpp): the zero counts of trim_edges over row ranges, with several
blocks in both grid directions, against numpy; and zap's two radix selects and its mask
against numpy's medians, with several blocks, sizes that are not a multiple of the block,
and candidate buffers that fill after the first digit, after a later one or never."""
import ctypes
import os
import subprocess
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(EMU, "clean_emu.cpp")
    out = os.path.join(EMU, "_build", "clean_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-x",
                    "c++", src, "-o", out], check=True)
    lib = ctypes.CDLL(out)
    lib.emu_zap.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p,
                            ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _np_zap(x, sigma):
    """Dynspec.zap's statements (reference dynspec.py:3867-3870) on a copy."""
    x = x.copy()
    with np.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        med = np.median(x[~np.isnan(x)])
        d = np.abs(x - med)
        mdev = np.median(d[~np.isnan(d)])
        x[d / mdev > sigma] = np.nan
    return x, med, mdev


def _zap(emu, x, sigma, threads=64, G=3, cap=0):
    y = np.ascontiguousarray(x, dtype=np.float64).copy()
    stats = np.zeros(2)
    info = np.zeros(4, np.int64)
    assert emu.emu_zap(_p(y), y.size, float(sigma), _p(stats), threads, G, cap, _p(info)) == 0
    return y, stats, info


def _same(a, b):
    return a == b or (np.isnan(a) and np.isnan(b))


def _arrays():
    rng = np.random.default_rng(5)
    out = {}
    out["exp_odd"] = rng.exponential(1.0, 1001)
    out["exp_even"] = rng.exponential(1.0, 1000)
    x = rng.normal(0.0, 1.0, 777)
    x[rng.random(777) < 0.1] = np.nan
    x[::50] *= 40.0
    out["normal_nan_outliers"] = x
    x = rng.exponential(1.0, 640)
    x[:3] = np.inf
    x[3:5] = -np.inf
    out["inf"] = x
    x = np.full(300, np.inf)
    x[:100] = rng.random(100)
    out["inf_median"] = x                  # med = inf, so inf - inf gives NaN deviations
    out["all_nan"] = np.full(129, np.nan)
    out["one"] = np.array([2.5])
    out["two"] = np.array([-1.0, 3.0])
    x = np.ones(513)
    x[::7] = 5.0
    out["mdev_zero"] = x                   # more than half equal the median: mdev = 0
    x = np.zeros(256)
    x[:100] = -0.0
    x[200:] = rng.random(56)
    out["signed_zeros"] = x
    x = rng.integers(-3, 4, 999).astype(np.float64)
    out["ties"] = x                        # the two middle ranks in one bucket or in two
    out["halves"] = np.concatenate([np.full(500, 1.0), np.full(500, 2.0)])
    out["tiny_and_huge"] = np.array([5e-324, 1e308, -1e308, 1.7e308, 1.7e308, 0.0])
    return out


ARRAYS = _arrays()


@pytest.mark.parametrize("name", sorted(ARRAYS))
@pytest.mark.parametrize("sigma", [0.5, 3.0, 7.0])
def test_zap_matches_numpy(emu, name, sigma):
    x = ARRAYS[name]
    ref, med, mdev = _np_zap(x, sigma)
    got, stats, info = _zap(emu, x, sigma)
    assert _same(stats[0], med) and _same(stats[1], mdev), (stats, med, mdev)
    assert np.array_equal(got, ref, equal_nan=True)


@pytest.mark.parametrize("threads,G", [(32, 1), (64, 5), (96, 7)])
@pytest.mark.parametrize("cap", [0, 1, 40, 2000])
def test_zap_blocks_and_buffers(emu, threads, G, cap):
    """The same results for every grid and for buffers that fill at any digit or never."""
    x = np.random.default_rng(threads + G).exponential(1.0, 1237)
    x[::13] = np.nan
    ref, med, mdev = _np_zap(x, 2.0)
    got, stats, info = _zap(emu, x, 2.0, threads, G, cap)
    assert stats[0] == med and stats[1] == mdev
    assert np.array_equal(got, ref, equal_nan=True)
    if cap == 1:
        assert info[1] == -1 or info[0] <= 1
    if cap == 2000:
        assert info[1] == 0        # every candidate fits after the first digit


def test_zap_compacts_after_first_digit(emu):
    """A spread of values: the buffer of n/8 keys fills after digit 0, so each median reads
    the array twice plus the compaction."""
    x = np.random.default_rng(1).exponential(1.0, 20000)
    _, _, info = _zap(emu, x, 7.0, 128, 4)
    assert info[1] == 0 and info[3] == 0
    assert 0 < info[0] <= 20000 // 8 and 0 < info[2] <= 20000 // 8


@pytest.mark.parametrize("shape,rows", [((70, 300), (0, 70)), ((70, 300), (5, 66)),
                                        ((200, 37), (64, 129)), ((3, 600), (1, 1)),
                                        ((129, 257), (0, 129))])
def test_zero_counts(emu, shape, rows):
    rng = np.random.default_rng(sum(shape))
    x = rng.normal(size=shape)
    x[rng.random(shape) < 0.3] = 0.0
    x[rng.random(shape) < 0.1] = np.nan
    x[rng.random(shape) < 0.05] = -0.0
    x[2, :] = 0.0
    x[:, 3] = np.nan
    r0, r1 = rows
    rc = np.full(r1 - r0, -1, np.int32)
    cc = np.full(shape[1], -1, np.int32)
    assert emu.emu_zero_counts(_p(x), shape[0], shape[1], r0, r1, _p(rc), _p(cc)) == 0
    z = (x == 0) | np.isnan(x)
    assert np.array_equal(rc, z[r0:r1].sum(axis=1))
    assert np.array_equal(cc, z[r0:r1].sum(axis=0))
