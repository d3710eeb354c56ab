"""Generate tests/golden/brightness_*.npz by running the UNMODIFIED reference's
scint_sim.Brightness (via oracle/ref_loader.py).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python oracle/make_golden_brightness.py [case ...]

One file per case.  Keys: ``kwargs`` (JSON of the constructor arguments), ``diag_sha256``
(the sha256 of the lattice's packed diagonal bits, oracle/brightness_oracle.py, so a qhull
that triangulates differently is reported as such) and:
* small cases (lattices of about 80^2, query grids of about 100 x 100): the full attributes
  ``x fd td acf_efield B thetax thetay jacobian SS LSS acf``;
* ``default`` (600^2, 2000 x 1000, several minutes): the sha256 of ``x fd td``, and for each
  of ``acf_efield B thetax thetay jacobian SS LSS acf`` the values at 4096 seeded flat
  positions (``<name>_idx``, ``<name>_val``).
"""
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import brightness_oracle as BO  # noqa: E402
from oracle import ref_loader  # noqa: E402

SMALL = dict(nx=4, dx=0.1, nf=1, df=0.02, nt=8, dt=0.16)        # 80^2 lattice, 100 x 100
CASES = {
    "angles": dict(SMALL, ar=2.0),
    "ar1": dict(SMALL, ar=1, psi=45, alpha=1.0),
    "ar3_psi30_alpha2": dict(SMALL, ar=3, psi=30, alpha=2),
    "thetag_thetar": dict(SMALL, ar=1.5, psi=60, thetagx=0.3, thetagy=-0.2, thetarx=0.25,
                          thetary=0.1),
    # x in [-2, 1.95]: thetay reaches 2.8, so part of the queries leave the lattice
    "hull": dict(SMALL, nx=2, dx=0.05, ar=1.3, psi=20),
    # 79^2 lattice, 99 x 99 queries
    "odd": dict(nx=3.95, dx=0.1, nf=0.99, df=0.02, nt=7.92, dt=0.16, ar=2.5, psi=-40,
                alpha=1.4, thetagx=0.1, thetarx=0.1),
    "default": {},
}
FULL = ("x", "fd", "td", "acf_efield", "B", "thetax", "thetay", "jacobian", "SS", "LSS", "acf")
SAMPLED = ("acf_efield", "B", "thetax", "thetay", "jacobian", "SS", "LSS", "acf")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


def main(names):
    ss = ref_loader.load().scint_sim
    for name in names or CASES:
        kwargs = CASES[name]
        t0 = time.perf_counter()
        b = ss.Brightness(**kwargs)
        dt = time.perf_counter() - t0
        out = dict(kwargs=np.array(json.dumps(kwargs)),
                   diag_sha256=np.array(BO.diag_sha256(BO.diagonals(b.x))))
        if name == "default":
            rng = np.random.default_rng(2020)
            for k in ("x", "fd", "td"):
                out[k + "_sha256"] = np.array(sha(getattr(b, k)))
            for k in SAMPLED:
                a = np.ravel(getattr(b, k))
                idx = np.sort(rng.choice(a.size, 4096, replace=False))
                out[k + "_idx"], out[k + "_val"] = idx, a[idx]
        else:
            for k in FULL:
                out[k] = np.asarray(getattr(b, k))
        fn = os.path.join(GOLD, "brightness_%s.npz" % name)
        np.savez_compressed(fn, **out)
        print("  %-18s lattice %d, SS %s  %.1f s  %d bytes" % (
            name, len(b.x), b.SS.shape, dt, os.path.getsize(fn)), flush=True)


if __name__ == "__main__":
    main(sys.argv[1:])
