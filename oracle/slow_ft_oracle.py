"""Float64 restatements of scint_utils.slow_FT (reference scint_utils.py:655-702, with its
``fftshift(..., axis=0)`` read as ``axes=0``).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Written from the semantics: with
c = ntime // 2, s_f = freqs[f] / freqs[nfreq // 2] and a_f = s_f / ntime,

    Y[m, f]   = sum_t x[t, f] exp(-2 pi i a_f t (m - c))            (fftshifted Doppler axis)
    out[m, j] = sum_f Y[m, f] exp(-2 pi i f (j - nfreq//2) / nfreq)  (fftshifted delay axis)

``direct`` forms the ntime x ntime phase matrix of each channel (small sizes only);
``bluestein`` computes the Doppler axis as a chirp, a cyclic convolution of length
M >= 2 ntime - 1 by FFT, and a chirp, which is fast enough for the GPU tests' large cases.
"""
import numpy as np


def _scale(freqs):
    f = np.asarray(freqs, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return f / f[len(f) // 2]


def _delay(Y):
    return np.fft.fftshift(np.fft.fft(Y, axis=1), axes=1)


def direct(dynspec, freqs):
    x = np.real(np.asarray(dynspec)).astype(np.float64)
    ntime, nfreq = x.shape
    s = _scale(freqs)
    t = np.arange(ntime, dtype=np.float64)
    m = t - ntime // 2
    Y = np.empty((ntime, nfreq), np.complex128)
    with np.errstate(invalid="ignore", over="ignore"):
        for f in range(nfreq):
            Y[:, f] = np.exp(-2j * np.pi * s[f] * np.outer(m, t) / ntime) @ x[:, f]
    return _delay(Y)


def bluestein(dynspec, freqs):
    x = np.real(np.asarray(dynspec)).astype(np.float64)
    ntime, nfreq = x.shape
    s = _scale(freqs)
    c = ntime // 2
    M = 8
    while M < 2 * ntime - 1:
        M *= 2
    t = np.arange(ntime, dtype=np.float64)
    n = np.arange(M)
    n = np.where(n < ntime, n, n - M).astype(np.float64)        # |n| < ntime live
    with np.errstate(invalid="ignore", over="ignore"):
        a = s[None, :] / ntime
        # phases reduced mod 2 in float64 before the exponential, like the device code
        ph = lambda q: np.exp(1j * np.pi * np.mod(q, 2.0))
        b = ph(a * (n * n)[:, None])
        b[np.abs(n) >= ntime] = 0.0
        A = np.zeros((M, nfreq), np.complex128)
        A[:ntime] = x * ph(-a * (t * t - 2 * c * t)[:, None])
        conv = np.fft.ifft(np.fft.fft(A, axis=0) * np.fft.fft(b, axis=0), axis=0)[:ntime]
        Y = ph(-a * (t * t)[:, None]) * conv
    return _delay(Y)
