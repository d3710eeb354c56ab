"""Generate tests/golden/scale_dyn_wideband.npz by running the UNMODIFIED
reference's Dynspec.scale_dyn(scale='lambda', spacing='min') (via
oracle/ref_loader.py) on a 64-channel band from 704 to 4032 MHz, with the
frequencies ascending and descending.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python -m oracle.make_golden_lambda

The fixture is committed; the GPU box never needs the reference.  On this band
the wavelength steps vary by a factor of 33, so 'min' spacing gives about 5.7
output rows per channel, the ratio the large scale_dyn cases of
tests/test_gpu_item_counts.py rely on.  The fixture pins
oracle.dynspec_oracle.scale_dyn_lambda, which those GPU tests use as their
reference.
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

NF, NT, F_LO, F_HI, DT = 64, 5, 704.0, 4032.0, 10.0


def golden_lambda(pkg):
    rng = np.random.default_rng(31)
    dyn = rng.exponential(1.0, (NF, NT))
    df = (F_HI - F_LO) / (NF - 1)
    out = dict(dyn=dyn, dt=DT)
    for tag, sl in (("asc", slice(None)), ("desc", slice(None, None, -1))):
        ds = _ref_dynspec(pkg, dyn[sl].copy(), DT, df, f0=F_LO)
        ds.freqs = np.linspace(F_LO, F_HI, NF)[sl].copy()
        ds.scale_dyn(scale="lambda", spacing="min")
        out.update({tag + "_freqs": np.asarray(ds.freqs), tag + "_lamdyn": ds.lamdyn,
                    tag + "_lam": ds.lam, tag + "_dlam": ds.dlam})
        print("scale_dyn wideband %s: lamdyn %s, dlam %.4e" % (tag, ds.lamdyn.shape, ds.dlam))
    np.savez_compressed(os.path.join(GOLD, "scale_dyn_wideband.npz"), **out)


if __name__ == "__main__":
    golden_lambda(ref_loader.load())
