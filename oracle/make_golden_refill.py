"""Generate tests/golden/refill_*.npz: Dynspec.refill of the UNMODIFIED reference (via
oracle/ref_loader.py) on the paths that need no scikit-image, and the biharmonic oracle
(oracle/refill_oracle.py) for the biharmonic cases.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python oracle/make_golden_refill.py

One file per case, keys ``dyn_in`` (float64 [nf][nt] with NaN gaps, a zapped channel, a
zapped sub-integration of zeros and a few isolated zeros), ``dyn_out`` (self.dyn after the
call), ``method``, ``zeros``, ``kernel_size`` and ``linear``, and ``source`` ('reference'
or 'oracle'):
  median_k3, median_k5, median_k3x7   method='median', zeros=True
  median_k5_nozeros                   method='median', zeros=False
  mean, mean_nozeros                  method='mean' (no method step: the mean fill only)
  linear_off                          method='linear', linear=False
  biharmonic, biharmonic_nozeros      the oracle's spsolve
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_loader  # noqa: E402
from oracle import refill_oracle as O  # noqa: E402


def gapped(rng, nf=40, nt=56):
    dyn = rng.exponential(1.0, (nf, nt)) + 0.5
    dyn[rng.random((nf, nt)) < 0.08] = np.nan
    dyn[17, :] = np.nan                  # a zapped channel
    dyn[:, 9] = 0.0                      # a zapped sub-integration
    dyn[3, 30] = dyn[33, 2] = dyn[0, 0] = 0.0
    dyn[-3:, -4:] = np.nan               # a hole in the corner
    return dyn


def reference_refill(ds_cls, dyn, **kw):
    ds = ds_cls.__new__(ds_cls)
    ds.dyn = dyn.copy()
    ds.refill(**kw)
    return ds.dyn


def main():
    ref = ref_loader.load().dynspec
    rng = np.random.default_rng(20261017)
    dyn = gapped(rng)
    cases = {
        "median_k3": dict(method="median", zeros=True, kernel_size=3),
        "median_k5": dict(method="median", zeros=True, kernel_size=5),
        "median_k3x7": dict(method="median", zeros=True, kernel_size=(3, 7)),
        "median_k5_nozeros": dict(method="median", zeros=False, kernel_size=5),
        "mean": dict(method="mean", zeros=True),
        "mean_nozeros": dict(method="mean", zeros=False),
        "linear_off": dict(method="linear", zeros=True, linear=False),
        "biharmonic": dict(method="biharmonic", zeros=True),
        "biharmonic_nozeros": dict(method="biharmonic", zeros=False),
    }
    total = 0
    for name, kw in cases.items():
        kw = dict(dict(kernel_size=5, linear=True), **kw)
        if kw["method"] == "biharmonic":
            out, source = O.refill(dyn, **kw), "oracle"
        else:
            out, source = reference_refill(ref.Dynspec, dyn, **kw), "reference"
        fn = os.path.join(GOLD, "refill_%s.npz" % name)
        np.savez_compressed(fn, dyn_in=dyn, dyn_out=out, method=kw["method"], zeros=kw["zeros"],
                            kernel_size=np.array(kw["kernel_size"]), linear=kw["linear"],
                            source=source)
        total += os.path.getsize(fn)
        print("  %-20s %-9s nan left %d" % (name, source, np.isnan(out).sum()))
    print("total %d bytes" % total)


if __name__ == "__main__":
    main()
