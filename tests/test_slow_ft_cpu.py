"""CPU tests of scint_utils.slow_FT: the float64 oracles against the reference's fixtures
(tests/golden/slow_ft_*.npz, made by oracle/make_golden_slow_ft.py), the device functors
of csrc/slow_ft.cu under the host emulator, the argument errors of the port raised before
any device call, and the new C symbol."""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest

from oracle import slow_ft_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "slow_ft_*.npz")))


@pytest.mark.parametrize("fn", FIXTURES, ids=[os.path.basename(f)[8:-4] for f in FIXTURES])
@pytest.mark.parametrize("method", ["direct", "bluestein"])
def test_oracle_matches_reference(fn, method):
    z = np.load(fn)
    got = getattr(O, method)(z["dynspec"], z["freqs"])
    ref = z["out"]
    assert got.shape == ref.shape and got.dtype == np.complex128
    if not np.all(np.isfinite(z["dynspec"])):
        assert not np.any(np.isfinite(ref))
        assert not np.any(np.isfinite(got))
        return
    assert np.max(np.abs(got - ref)) <= 1e-12 * np.max(np.abs(ref))


def test_fixtures_cover_the_cases():
    names = {os.path.basename(f)[8:-4] for f in FIXTURES}
    assert names == {"64x48", "75x37_desc", "150x64_wide", "1x5", "5x1", "2x2", "nan"}
    assert sum(os.path.getsize(f) for f in FIXTURES) < 500_000
    z = np.load(os.path.join(ROOT, "tests", "golden", "slow_ft_75x37_desc.npz"))
    assert np.all(np.diff(z["freqs"]) < 0)
    z = np.load(os.path.join(ROOT, "tests", "golden", "slow_ft_150x64_wide.npz"))
    s = z["freqs"] / z["freqs"][32]
    assert s.min() < 0.7 and s.max() > 1.3


def test_oracles_agree_on_odd_shapes():
    rng = np.random.default_rng(3)
    for nt, nf in [(1, 1), (3, 7), (300, 50), (257, 3)]:
        x = rng.normal(size=(nt, nf))
        f = np.linspace(400.0, 800.0, nf)[::-1]
        d, b = O.direct(x, f), O.bluestein(x, f)
        assert np.max(np.abs(d - b)) <= 1e-12 * np.max(np.abs(d))


# ---- device code under the host emulator -------------------------------------------------
def _emu():
    src = os.path.join(EMU, "slow_ft_emu.cpp")
    out = os.path.join(EMU, "_build", "slow_ft_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-o", out],
                   check=True)
    return ctypes.CDLL(out)


@pytest.fixture(scope="module")
def emu():
    return _emu()


@pytest.mark.parametrize("nt", [1, 2, 3, 8, 75])
@pytest.mark.parametrize("nf", [1, 2, 3, 8, 75])
def test_slow_ft_functors_on_host(emu, nt, nf):
    """csrc/slow_ft.cu's functors (per-channel chirps with float64 phases, the kernel
    transforms b_f, the in-place multiply, the output chirp and both delay-row stores) around
    a reference DFT, against the float64 direct sum.  The kernel transform always runs as a
    column pass, so every shape here covers it; nf 8 takes the radix rows, every other nf the
    row chirp-z.  Bounds: those of the GPU tests."""
    rng = np.random.default_rng(nt * 100 + nf)
    x = rng.normal(size=(nt, nf)).astype(np.float32)
    f = np.linspace(400.0, 800.0, nf) if nf > 1 else np.array([600.0])
    rng.shuffle(f)
    s = f / f[nf // 2]
    out = np.zeros((nt, nf), np.complex64)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert emu.emu_slow_ft(P(x), nt, nf, P(s), P(out)) == 0
    ref = O.direct(x.astype(np.float64), f)
    assert np.linalg.norm(out - ref) <= 1e-6 * np.linalg.norm(ref)
    assert np.max(np.abs(out - ref)) <= 1e-5 * np.max(np.abs(ref))


def test_nonfinite_on_host(emu):
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    for nf in (8, 9):
        f = np.linspace(400.0, 800.0, nf)
        for bad in ("nan", "inf", "fref0"):
            x = np.random.default_rng(1).normal(size=(20, nf)).astype(np.float32)
            s = f / f[nf // 2]
            if bad == "nan":
                x[3, 2] = np.nan
            elif bad == "inf":
                x[3, 2] = np.inf
            else:
                with np.errstate(divide="ignore"):
                    s = f / 0.0
            out = np.zeros((20, nf), np.complex64)
            emu.emu_slow_ft(P(x), 20, nf, P(s), P(out))
            assert not np.any(np.isfinite(out)), (nf, bad)


# ---- Python layer -------------------------------------------------------------------------
def test_argument_errors_before_device(monkeypatch):
    """Every ValueError of slow_FT is raised before any device call, and the input array is
    not modified."""
    from scintools_b200 import _device, scint_utils

    def no_device(*a, **k):
        raise AssertionError("device touched")

    monkeypatch.setattr(_device, "device", no_device)
    f = np.linspace(400.0, 800.0, 16)
    cases = [
        (np.zeros(16), f),                                   # 1-D
        (np.zeros((2, 4, 16)), f),                           # 3-D
        (np.zeros((8, 16)), f[:15]),                         # len(freqs) != nfreq
        (np.zeros((8, 16)), f.reshape(4, 4)),                # freqs not 1-D
        (np.zeros((8, 16)), np.where(np.arange(16) == 3, np.nan, f)),
        (np.zeros((8, 16)), np.where(np.arange(16) == 3, np.inf, f)),
        (np.zeros((0, 16)), f),
        (np.zeros((8, 0)), f[:0]),
        (np.zeros((32769, 1), np.float32), f[:1]),
        (np.zeros((1, 8193), np.float32), np.linspace(400.0, 800.0, 8193)),
    ]
    for dyn, fr in cases:
        before = dyn.copy()
        with pytest.raises(ValueError):
            scint_utils.slow_FT(dyn, fr)
        assert np.array_equal(dyn, before)


def test_library_exports_slow_ft_symbol():
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _lib
    assert "sb_slow_ft_f32" in _lib.EXPORTS
    assert _lib.lib.sb_abi_version() == 8
