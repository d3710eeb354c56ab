"""Generate tests/golden/slow_ft_*.npz by running the UNMODIFIED reference's
scint_utils.slow_FT (via oracle/ref_loader.py).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python oracle/make_golden_slow_ft.py

As written the reference always raises TypeError: it calls
``np.fft.fftshift(SS, axis=0)``, and numpy's keyword is ``axes``.  This script checks
that, then calls it again with ``np.fft.fftshift`` wrapped for the duration of the call
only, mapping ``axis=`` to ``axes=``; every other operation is the reference's own.

One file per case, keys ``dynspec`` ([time, frequency] float64), ``freqs`` and ``out``
(complex128):
  64x48        random, 1400 MHz + 0.1 MHz channels
  75x37_desc   odd ntime, descending freqs
  150x64_wide  400-800 MHz band (s from 0.67 to 1.33)
  1x5, 5x1, 2x2
  nan          24x16 with one NaN pixel
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_loader  # noqa: E402


def reference_slow_ft(su, dynspec, freqs):
    try:
        su.slow_FT(dynspec, freqs)
    except TypeError:
        pass
    else:
        raise AssertionError("the reference slow_FT no longer raises TypeError")
    orig = np.fft.fftshift

    def fftshift(x, axes=None, axis=None):
        return orig(x, axes=axis if axis is not None else axes)

    np.fft.fftshift = fftshift
    try:
        return su.slow_FT(dynspec, freqs)
    finally:
        np.fft.fftshift = orig


def main():
    su = ref_loader.load().scint_utils
    rng = np.random.default_rng(20261017)
    cases = {
        "64x48": (rng.normal(size=(64, 48)), 1400.0 + 0.1 * np.arange(48)),
        "75x37_desc": (rng.exponential(1.0, (75, 37)), 1500.0 - 0.25 * np.arange(37)),
        "150x64_wide": (rng.normal(size=(150, 64)), np.linspace(400.0, 800.0, 64)),
        "1x5": (rng.normal(size=(1, 5)), 1400.0 + np.arange(5.0)),
        "5x1": (rng.normal(size=(5, 1)), np.array([1400.0])),
        "2x2": (rng.normal(size=(2, 2)), np.array([1400.0, 1410.0])),
    }
    x = rng.normal(size=(24, 16))
    x[7, 5] = np.nan
    cases["nan"] = (x, 1300.0 + 2.0 * np.arange(16))
    total = 0
    for name, (dyn, freqs) in cases.items():
        out = reference_slow_ft(su, dyn.copy(), freqs.copy())
        fn = os.path.join(GOLD, "slow_ft_%s.npz" % name)
        np.savez_compressed(fn, dynspec=dyn, freqs=freqs, out=out)
        total += os.path.getsize(fn)
        print("  %-12s %s %s" % (name, out.shape, out.dtype))
    print("total %d bytes" % total)


if __name__ == "__main__":
    main()
