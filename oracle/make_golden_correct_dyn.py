"""Generate tests/golden/correct_dyn_*.npz by running the UNMODIFIED reference's
Dynspec.correct_dyn (via oracle/ref_loader.py).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python oracle/make_golden_correct_dyn.py

Every case starts from a fresh reference Dynspec; its keys are prefixed by the case name:
``args`` (svd, nmodes, frequency, time, lamsteps, nsmooth or -1), ``inputs`` (the names of
the shared input arrays ``in_<name>`` used as dyn and, with lamsteps, as lamdyn, which is
set on the object before the call so scale_dyn is not involved), the attributes after the
call (``dyn``, ``lamdyn``, ``svd_model``, ``bandpass`` where set) and ``dtypes``
(attribute=dtype, comma separated).  svd_model is stored as its real part: the reference's
is complex128 and its imaginary part is checked to be zero here.

correct_dyn_svd.npz: svd=True with nmodes 1, 2, 3 on a 32 x 96 dyn with band and gain
structure, scattered zeros and NaNs; a prescribed-spectrum 24 x 64 matrix (singular values
100, 30, 10, 3, 1, 0.3, ...) with nmodes 3; nmodes 8 >= min(6, 40); lamsteps=True.
correct_dyn_bandpass.npz: svd=False with frequency only, time only, both, both with
nsmooth=5 (the dyn has an all-zero channel and an all-zero sub-integration), and
lamsteps=True (lamdyn has zeros, NaNs and an all-zero row).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_loader  # noqa: E402


def _ref_dynspec(pkg, dyn, dt=8.0, df=0.25, f0=1400.0):
    nf, nt = dyn.shape
    freqs = f0 + df * np.arange(nf)
    times = dt * np.arange(nt)
    bd = pkg.dynspec.BasicDyn(dyn, name="golden", header=["golden"], times=times, freqs=freqs,
                              nchan=nf, nsub=nt, bw=df * nf, df=df, freq=float(np.mean(freqs)),
                              tobs=dt * nt, dt=dt, mjd=60000)
    return pkg.dynspec.Dynspec(dyn=bd, verbose=False, process=False)


def structured_dyn(rng, nf, nt, nzero=20, nnan=6):
    """Scintles (exponential) times a bandpass and a gain curve, with scattered zeros and
    NaNs."""
    f = np.linspace(0, 1, nf)
    t = np.linspace(0, 1, nt)
    band = 1.0 + 0.6 * np.sin(2 * np.pi * 1.3 * f) ** 2 + 0.3 * f
    gain = 0.7 + 0.3 * np.cos(2 * np.pi * 0.8 * t) + 0.1 * t
    dyn = band[:, None] * gain[None, :] * rng.exponential(1.0, (nf, nt))
    idx = rng.choice(nf * nt, nzero + nnan, replace=False)
    dyn.flat[idx[:nzero]] = 0.0
    dyn.flat[idx[nzero:]] = np.nan
    return dyn


def prescribed(rng, nf, nt, s):
    U, _ = np.linalg.qr(rng.normal(size=(nf, len(s))))
    V, _ = np.linalg.qr(rng.normal(size=(nt, len(s))))
    return (U * s) @ V.T


def run_case(pkg, out, name, dyn, svd=True, nmodes=1, frequency=True, time=True,
             lamsteps=False, nsmooth=None, lamdyn=None):
    ds = _ref_dynspec(pkg, out["in_" + dyn].copy())
    names = [dyn]
    if lamdyn is not None:
        ds.lamdyn = out["in_" + lamdyn].copy()
        names.append(lamdyn)
    out[name + "_inputs"] = np.array(",".join(names))
    ds.correct_dyn(svd=svd, nmodes=nmodes, frequency=frequency, time=time, lamsteps=lamsteps,
                   nsmooth=nsmooth)
    out[name + "_args"] = np.array([svd, nmodes, frequency, time, lamsteps,
                                    -1 if nsmooth is None else nsmooth], dtype=np.int64)
    dts = []
    for attr in ("dyn", "lamdyn", "svd_model", "bandpass"):
        if hasattr(ds, attr):
            v = np.asarray(getattr(ds, attr))
            dts.append("%s=%s" % (attr, v.dtype))
            if np.iscomplexobj(v):
                assert not np.any(v.imag)
                v = v.real.copy()
            out[name + "_" + attr] = v
    out[name + "_dtypes"] = np.array(",".join(dts))
    print("  %-8s %s" % (name, ", ".join(dts)))


def main():
    pkg = ref_loader.load()
    rng = np.random.default_rng(20261017)
    out = {"in_A": structured_dyn(rng, 32, 96, 12, 5)}
    for k in (1, 2, 3):
        run_case(pkg, out, "s%d" % k, "A", nmodes=k)
    s = np.array([100.0, 30.0, 10.0, 3.0, 1.0, 0.3, 0.1, 0.03])
    out["in_P"] = prescribed(rng, 24, 64, s)
    run_case(pkg, out, "p3", "P", nmodes=3)
    out["in_F"] = 1.0 + rng.exponential(1.0, (6, 40))
    run_case(pkg, out, "full", "F", nmodes=8)
    out["in_L"] = structured_dyn(rng, 30, 96, 10, 4)
    run_case(pkg, out, "lam", "A", nmodes=1, lamsteps=True, lamdyn="L")
    np.savez_compressed(os.path.join(GOLD, "correct_dyn_svd.npz"), **out)

    B = structured_dyn(rng, 32, 96, 12, 5)
    B[17, :] = 0.0
    B[:, 61] = 0.0
    L = structured_dyn(rng, 30, 96, 10, 4)
    L[23, :] = 0.0
    out = {"in_B": B, "in_L": L}
    run_case(pkg, out, "freq", "B", svd=False, time=False)
    run_case(pkg, out, "time", "B", svd=False, frequency=False)
    run_case(pkg, out, "both", "B", svd=False)
    run_case(pkg, out, "smooth", "B", svd=False, nsmooth=5)
    run_case(pkg, out, "lam", "B", svd=False, lamsteps=True, lamdyn="L")
    np.savez_compressed(os.path.join(GOLD, "correct_dyn_bandpass.npz"), **out)


if __name__ == "__main__":
    main()
