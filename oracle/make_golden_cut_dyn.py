"""Generate tests/golden/cut_dyn_*.npz by running the UNMODIFIED reference's
Dynspec.cut_dyn (dynspec.py:3158-3271) through oracle/ref_loader.py.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python -m oracle.make_golden_cut_dyn

Each fixture holds the input (dyn, dt, df, tcuts, fcuts), the reference's cutdyn and
cutsspec, and cutacf: every tile's calc_acf(input_dyn=tile) from the reference (cut_dyn
computes these and discards them).  To keep the files small, the inputs are multiples of
1/64 (they compress well and are exact in float32), and cutsspec and cutacf are stored
rounded to float32: 6e-8 relative, far below the 1e-5 the tests allow.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_loader  # noqa: E402
from oracle.make_golden import _ref_dynspec  # noqa: E402


def case(pkg, name, dyn, tcuts, fcuts, dt=10.0, df=0.1):
    ds = _ref_dynspec(pkg, dyn.copy(), dt, df)
    ds.cut_dyn(tcuts=tcuts, fcuts=fcuts)
    cutacf = np.empty(ds.cutdyn.shape[:2] + (2 * ds.cutdyn.shape[2], 2 * ds.cutdyn.shape[3]))
    for ii in range(fcuts + 1):
        for jj in range(tcuts + 1):
            cutacf[ii, jj] = ds.calc_acf(input_dyn=ds.cutdyn[ii, jj])
    np.savez_compressed(os.path.join(GOLD, "cut_dyn_%s.npz" % name), dyn=dyn, dt=dt, df=df,
                        tcuts=tcuts, fcuts=fcuts, cutdyn=ds.cutdyn,
                        cutsspec=ds.cutsspec.astype(np.float32),
                        cutacf=cutacf.astype(np.float32))


def field(rng, shape):
    """Exponential intensities rounded to multiples of 1/64."""
    return np.round(rng.exponential(1.0, shape) * 64) / 64


def main():
    pkg = ref_loader.load()
    rng = np.random.default_rng(3158)
    # fcuts=1, tcuts=2 make 50 x 50 tiles of both: 100 x 150 is covered exactly, 101 x 152
    # drops the last row and the last two columns
    case(pkg, "101x152_t2_f1", field(rng, (101, 152)), tcuts=2, fcuts=1)
    case(pkg, "100x150_t2_f1", field(rng, (100, 150)), tcuts=2, fcuts=1)
    case(pkg, "128x256_t3_f1", field(rng, (128, 256)), tcuts=3, fcuts=1)
    case(pkg, "48x80_t0_f0", field(rng, (48, 80)), tcuts=0, fcuts=0)
    dyn = field(rng, (64, 96))
    dyn[40, 10] = np.nan                 # tile (1, 0) of the 2 x 3 grid
    case(pkg, "nan_64x96_t2_f1", dyn, tcuts=2, fcuts=1)


if __name__ == "__main__":
    main()
