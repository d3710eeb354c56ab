"""Generate tests/golden/acf_model_*.npz by running the UNMODIFIED reference's
scint_sim.ACF (via oracle/ref_loader.py).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python oracle/make_golden_acf_model.py [case ...]

Under numpy 2 the reference fails on ``np.complex_`` (removed from numpy); this script
sets ``np.complex_ = np.complex128`` for itself only.  Every other operation is the
reference's own.  The ar = 8 case takes a few minutes on a CPU.

One file per case.  Keys: ``kwargs`` (JSON of the constructor arguments), the attributes
``acf fn tn sn snp ddnun dsp sp_fac res_fac core_fac nf nt``, ``acf_efield`` only where
the main grid has at most 256 points per side (elsewhere the tests tabulate it from the
same expression), and ``sspec_<window>`` for each ``calc_sspec`` call in ``sspec``.
"""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_loader  # noqa: E402

NOTEBOOK = dict(psi=30, phasegrad=0.2, theta=0, ar=2, taumax=4, dnumax=4, nt=51, nf=51)
BOTH = (("hanning", 1), ("blackman", 1.0))

# name: (constructor kwargs, calc_sspec calls (window, window_frac))
CASES = {
    "default": ({}, BOTH),
    "notebook": (NOTEBOOK, BOTH),
    "pg05_theta45": (dict(nt=50, nf=20, phasegrad=0.5, theta=45, wn=0.1, amp=0.8),
                     (("hamming", 0.5),)),
    "wn_taumax4": (dict(phasegrad=0.3, wn=0.1, taumax=4, nt=51), ()),
    "wn_taumax3p7": (dict(phasegrad=0.3, wn=0.1, taumax=3.7, nt=51), ()),
    "psi0": (dict(psi=0, wn=0.2), ()),
    "psi90": (dict(psi=90, phasegrad=0.2, theta=60), ()),
    "alpha2": (dict(alpha=2, psi=45, nt=31, nf=21), ()),
    "alpha1p2": (dict(alpha=1.2, psi=10, phasegrad=0.1, nt=41, nf=31), ()),
    "manual": (dict(auto_sampling=False, spatial_factor=3, resolution_factor=1.5,
                    core_factor=3, ar=1.5, psi=60, phasegrad=0.15, theta=-30, nt=31, nf=25),
               (("bartlett", 0.7),)),
    "ar4": (dict(ar=4, psi=30, phasegrad=0.2), ()),
    "ar8": (dict(ar=8, psi=20, phasegrad=0.1, theta=10), ()),
}

ATTRS = ("acf", "fn", "tn", "sn", "snp", "ddnun", "dsp", "sp_fac", "res_fac", "core_fac",
         "nf", "nt")


def main(names):
    np.complex_ = np.complex128
    ss = ref_loader.load().scint_sim
    for name in names or CASES:
        kwargs, sspecs = CASES[name]
        t0 = time.perf_counter()
        a = ss.ACF(**kwargs)
        dt = time.perf_counter() - t0
        out = {k: np.asarray(getattr(a, k)) for k in ATTRS}
        if a.acf_efield.shape[0] <= 256:
            out["acf_efield"] = a.acf_efield
        for window, frac in sspecs:
            a.calc_sspec(window=window, window_frac=frac)
            out["sspec_%s" % window] = a.sspec
        out["sspec"] = np.array(json.dumps(sspecs))
        out["kwargs"] = np.array(json.dumps(kwargs))
        fn = os.path.join(GOLD, "acf_model_%s.npz" % name)
        np.savez_compressed(fn, **out)
        print("  %-14s acf %s grid %d  %.2f s  %d bytes" % (
            name, a.acf.shape, a.acf_efield.shape[0], dt, os.path.getsize(fn)), flush=True)


if __name__ == "__main__":
    main(sys.argv[1:])
