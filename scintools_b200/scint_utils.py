"""CUDA-native mirror of scintools.scint_utils.

  slow_FT   scint_utils.py:655-702 -> sb_slow_ft_f32 (per-channel chirp-z transform)

There is no CPU fallback.
"""
import numpy as np

from . import _device as D
from . import _lib

SLOW_FT_MAX_NTIME = 32768
SLOW_FT_MAX_NFREQ = 8192


def _slow_ft_check(dynspec, freqs):
    """Argument checks of slow_FT, raised before any device call.  Returns the real part
    of dynspec and freqs as float64."""
    a = np.asarray(dynspec)
    if a.ndim != 2:
        raise ValueError("slow_FT takes a 2-D [time, frequency] array, got shape %s"
                         % (a.shape,))
    ntime, nfreq = a.shape
    f = np.asarray(freqs, dtype=np.float64)
    if f.ndim != 1 or f.shape[0] != nfreq:
        raise ValueError("slow_FT: freqs has shape %s, the dynamic spectrum has %d channels"
                         % (f.shape, nfreq))
    if not np.all(np.isfinite(f)):
        raise ValueError("slow_FT: freqs must be finite")
    if not (1 <= ntime <= SLOW_FT_MAX_NTIME and 1 <= nfreq <= SLOW_FT_MAX_NFREQ):
        raise ValueError("slow_FT: shape %d x %d is outside 1..%d x 1..%d (ntime x nfreq)"
                         % (ntime, nfreq, SLOW_FT_MAX_NTIME, SLOW_FT_MAX_NFREQ))
    return np.real(a), f


def slow_FT(dynspec, freqs, dtype=np.float64):
    """scint_utils.slow_FT: Fourier transform of a dynamic spectrum along t * f / fref in
    each channel, which removes the frequency scaling of the Doppler frequency, then
    along frequency.

    ``dynspec`` is [time, frequency] (the transpose of ``Dynspec.dyn``); its real part is
    used.  ``freqs`` holds the ``nfreq`` channel frequencies, in any order, and
    fref = freqs[nfreq // 2].  With c = ntime // 2 and s_f = freqs[f] / fref the result is

        out[m, j] = sum_f sum_t x[t, f] exp(-2 pi i s_f t (m - c) / ntime)
                                        exp(-2 pi i f (j - nfreq//2) / nfreq),

    both axes fftshifted, with no mean subtraction, window or padding.  This is the
    reference's arithmetic with one deliberate deviation: the reference calls
    ``np.fft.fftshift(SS, axis=0)``, a keyword numpy does not have, so it always raises
    TypeError; here that shift is the intended ``axes=0``.

    The Doppler axis is a chirp-z transform per channel and the delay axis an FFT, in
    float32 on the device (csrc/slow_ft.cu), so the cost is O(ntime log ntime) per channel
    rather than the reference's ntime^2.  Returns complex128 for ``dtype=np.float64`` and
    complex64 for ``np.float32``.  A NaN or inf in ``dynspec``, or fref = 0, makes every
    output non-finite, as in the reference.

    Raises ValueError, before any device work, when ``dynspec`` is not 2-D, ``freqs`` is
    not a 1-D array of ``nfreq`` finite values, or the shape is outside
    1..32768 x 1..8192 (ntime x nfreq)."""
    import torch
    a, f = _slow_ft_check(dynspec, freqs)
    ntime, nfreq = a.shape
    with np.errstate(divide="ignore", invalid="ignore"):
        fscale = f / f[nfreq // 2]
    x = D.upload_f32(a)
    s = D.upload(fscale)
    out = D.empty((ntime, nfreq, 2), torch.float32)
    _lib.check(_lib.lib.sb_slow_ft_f32(x.data_ptr(), ntime, nfreq, s.data_ptr(), out.data_ptr(),
                                       D.stream_ptr()))
    res = D.download(out).view(np.complex64)[..., 0]
    cdt = np.complex64 if np.dtype(dtype) == np.float32 else np.complex128
    return res.astype(cdt, copy=False)
