"""GPU tests of scint_utils.slow_FT (csrc/slow_ft.cu, sb_slow_ft_f32).

Bounds, for the complex64 result against a float64 reference:
    ||got - ref||_2 / ||ref||_2 <= 1e-6,     max|got - ref| / max|ref| <= 1e-5,
those of tests/test_gpu_fft_lengths.py for float32 complex outputs.  The arithmetic behind
them: every output is a float32 sum formed by radix passes whose rounding grows as
u sqrt(log2 n) in the 2-norm (u = 2^-24): the Doppler axis is three transforms of length
M <= 65536 (the kernels b_f, the chirped data, the inverse) and the delay axis one of
length nfreq, or three of length MT <= 16384 for the row chirp-z, plus one float32 rounding
per chirp factor (their phases are reduced mod 2 in float64, so they carry no phase error
that grows with t^2).  That is about sqrt(6 * 16 + 4) u ~ 6e-7 relative in the 2-norm for
the longest chain; the element-wise bound leaves a further factor 10 for the largest
deviations.

References: the reference's fixtures (tests/golden/slow_ft_*.npz); the float64 Bluestein
restatement (oracle/slow_ft_oracle.py) at sizes the direct sum cannot reach; numpy's
fft2 when every channel has the same frequency (independent of Bluestein); and the closed
form of a single impulse, up to the 32768 x 8192 corner.
"""
import glob
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "slow_ft_*.npz")))

L2_BOUND = 1e-6
MAX_BOUND = 1e-5


def _errors(got, ref):
    return (np.linalg.norm(got - ref) / np.linalg.norm(ref),
            np.max(np.abs(got - ref)) / np.max(np.abs(ref)))


def _check(got, ref, what):
    e2, em = _errors(got, ref)
    print("%s: l2 %.2e, max %.2e" % (what, e2, em))
    assert e2 <= L2_BOUND and em <= MAX_BOUND, (what, e2, em)


def _slow_ft(*a, **k):
    from scintools_b200 import scint_utils
    return scint_utils.slow_FT(*a, **k)


@pytest.mark.parametrize("fn", FIXTURES, ids=[os.path.basename(f)[8:-4] for f in FIXTURES])
def test_fixture_parity(fn):
    z = np.load(fn)
    got = _slow_ft(z["dynspec"], z["freqs"])
    ref = z["out"]
    assert got.shape == ref.shape and got.dtype == np.complex128
    if not np.all(np.isfinite(z["dynspec"])):
        assert not np.any(np.isfinite(got))
    else:
        _check(got, ref, os.path.basename(fn))


# ntime: M = 16384 is the longest kernel that fits one row FFT and 32768 needs a column
# pass; the driver uses the column pass for every M, so both sides run the same code, and
# these shapes pin the lengths around that size.  nfreq: powers of two (radix rows),
# chirp-z rows (odd, even non-power-of-two, 2 and 4) and 1.
@pytest.mark.parametrize("nt,nf", [(8192, 16), (8193, 17), (8191, 64), (12000, 3), (1025, 1),
                                   (2, 100), (777, 4), (333, 2), (64, 8192), (31, 8191),
                                   (1000, 1000)])
def test_against_float64_bluestein(nt, nf):
    from oracle import slow_ft_oracle as O
    rng = np.random.default_rng(nt + 7 * nf)
    x = rng.normal(size=(nt, nf))
    f = np.linspace(400.0, 800.0, nf) if nf > 1 else np.array([700.0])
    rng.shuffle(f)
    _check(_slow_ft(x, f), O.bluestein(x, f), "%d x %d" % (nt, nf))


@pytest.mark.parametrize("nt,nf", [(256, 100), (75, 64), (1000, 8), (4097, 1), (1, 37)])
def test_equal_freqs_is_fft2(nt, nf):
    """With every channel at one frequency (s = 1) the transform is an ordinary 2-D FFT:
    numpy's float64 fftshift(fft2(x)), independent of the Bluestein restatement."""
    x = np.random.default_rng(nt * nf).normal(size=(nt, nf))
    ref = np.fft.fftshift(np.fft.fft2(x))
    _check(_slow_ft(x, np.full(nf, 1400.0)), ref, "%d x %d, s = 1" % (nt, nf))


def _impulse_check(nt, nf, t0, f0, block=1024):
    """x[t0, f0] = 1: out[m, j] = exp(-2 pi i s_f0 t0 (m - c) / nt)
    exp(-2 pi i f0 (j - nf//2) / nf), checked at every element, in row blocks."""
    freqs = np.linspace(400.0, 800.0, nf) if nf > 1 else np.array([650.0])
    x = np.zeros((nt, nf), np.float32)
    x[t0, f0] = 1.0
    got = _slow_ft(x, freqs, dtype=np.float32)
    assert got.dtype == np.complex64 and got.shape == (nt, nf)
    s = freqs[f0] / freqs[nf // 2]
    m = np.arange(nt, dtype=np.float64) - nt // 2
    pm = np.mod(s * t0 * m / nt, 1.0)                    # turns, reduced in float64
    j = np.arange(nf, dtype=np.float64) - nf // 2
    pj = np.mod(f0 * j / nf, 1.0)
    row = np.exp(-2j * np.pi * pj)
    se2, sr2, emax = 0.0, 0.0, 0.0
    for r0 in range(0, nt, block):
        ref = np.exp(-2j * np.pi * pm[r0:r0 + block])[:, None] * row[None, :]
        d = got[r0:r0 + block] - ref
        se2 += float(np.sum(d.real ** 2 + d.imag ** 2))
        sr2 += float(ref.size)
        emax = max(emax, float(np.max(np.abs(d))))
    e2 = np.sqrt(se2 / sr2)
    print("impulse %d x %d at (%d, %d): l2 %.2e, max %.2e" % (nt, nf, t0, f0, e2, emax))
    assert e2 <= L2_BOUND and emax <= MAX_BOUND, (nt, nf, e2, emax)


def test_impulse_corner():
    _impulse_check(32768, 8192, 12345, 3001)


@pytest.mark.parametrize("nt,nf,t0,f0", [(32768, 1, 29999, 0), (1, 8192, 0, 5001),
                                         (4097, 8191, 4000, 6007), (30000, 77, 17, 60),
                                         (5, 5, 3, 4)])
def test_impulse_shapes(nt, nf, t0, f0):
    _impulse_check(nt, nf, t0, f0)


def test_limits_both_sides():
    from scintools_b200 import _device as D, _lib
    import torch
    f = np.array([1400.0])
    for shape in [(32769, 1), (1, 8193), (0, 1), (1, 0)]:
        with pytest.raises(ValueError):
            _slow_ft(np.zeros(shape, np.float32), np.linspace(400, 800, shape[1]))
    # the C ABI refuses the same shapes before touching its buffers
    x = D.upload(np.zeros(8, np.float32))
    s = D.upload(np.ones(8))
    out = D.empty((8, 2), torch.float32)
    for nt, nf in [(32769, 1), (1, 8193), (0, 1), (1, 0)]:
        rc = _lib.lib.sb_slow_ft_f32(x.data_ptr(), nt, nf, s.data_ptr(), out.data_ptr(),
                                     D.stream_ptr())
        assert rc == -4, (nt, nf, rc)         # SB_ERR_UNSUPPORTED
    # 32768 and 8192 run: test_impulse_corner / test_impulse_shapes
    assert _slow_ft(np.ones((1, 1)), f).shape == (1, 1)


@pytest.mark.parametrize("nf", [64, 50])
@pytest.mark.parametrize("bad", ["nan", "inf", "fref0"])
def test_nonfinite_everywhere(nf, bad):
    nt = 300
    x = np.random.default_rng(5).normal(size=(nt, nf))
    freqs = np.linspace(400.0, 800.0, nf)
    if bad == "nan":
        x[123, 7] = np.nan
    elif bad == "inf":
        x[123, 7] = np.inf
    else:
        freqs[nf // 2] = 0.0
    out = _slow_ft(x, freqs)
    assert not np.any(np.isfinite(out))


def test_deterministic_dtypes_and_input_unchanged():
    rng = np.random.default_rng(11)
    x = rng.normal(size=(4097, 100))
    f = np.linspace(1200.0, 1600.0, 100)
    x0, f0 = x.copy(), f.copy()
    a = _slow_ft(x, f)
    b = _slow_ft(x, f)
    assert a.dtype == np.complex128
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    c = _slow_ft(x, f, dtype=np.float32)
    assert c.dtype == np.complex64
    assert np.array_equal(c.astype(np.complex128), a)
    assert np.array_equal(x, x0) and np.array_equal(f, f0)
