"""Generate tests/golden/arcfit_*.npz by running the UNMODIFIED reference's
Dynspec.norm_sspec and Dynspec.fit_arc (via oracle/ref_loader.py) on the CPU.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python oracle/make_golden_arcfit.py

Two dynamic spectra, one file each:
  arcfit_61x103.npz       an odd-shaped 1-D-screen arc (61 channels x 103 subints)
  arcfit_zeros_48x90.npz  an arc whose secondary spectra hold exact-zero power bins,
                          so their dB values are -inf

Each file stores the input (dyn as float32, dt, df, f0), both secondary spectra the
calls read (``sspec`` with ``tdel``, ``lamsspec`` with ``beta``, and ``fdop``) as
float32 (the reference is run on float64 copies of exactly those values, which are
what the device receives), then one group of keys per call, prefixed by the call's
name:

  <name>_kind       "norm_sspec" or "fit_arc"
  <name>_kwargs     the call's keyword arguments, as a JSON string
  <name>_raises     the exception type name if the reference raises, else ""

``freq`` is the centre frequency as the reference's Dynspec holds it, a Python float.
fit_arc(lamsteps=False) divides its default ``constraint`` list by it, so it raises
TypeError there; the ``_f64`` calls hold it as numpy.float64, which broadcasts.

norm_sspec calls add ``_normsspec`` (float32 of the reference's float64 samples,
NaN under the mask), ``_mask``, ``_normsspecavg``, ``_powerspectrum``, ``_fdop``,
``_tdel``; fit_arc calls add the curvature and its errors (``_eta``, ``_etaerr``,
``_etaerr2``, with ``_left`` / ``_right`` for asymm=True), ``_noise``, and the length
and end values of the curvature axis (``_eta_array_n``, ``_eta_array_ends``).
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_loader  # noqa: E402
from oracle.make_golden import _ref_dynspec  # noqa: E402

# (name, kwargs): norm_sspec calls without an eta get the spectrum's for their lamsteps
NORM_CALLS = [
    ("n_freq", dict(lamsteps=False, cutmid=0, startbin=1)),
    ("n_lam", dict(lamsteps=True, cutmid=3, startbin=1)),
    ("n_start0", dict(lamsteps=False, cutmid=0, startbin=0)),
    ("n_start0_unweighted", dict(lamsteps=False, cutmid=0, startbin=0, weighted=False)),
    ("n_cutwide", dict(lamsteps=False, cutmid=21, startbin=2)),
    ("n_unweighted", dict(lamsteps=True, cutmid=2, startbin=1, weighted=False)),
    ("n_pscut", dict(lamsteps=True, cutmid=0, startbin=1, powerspec_cut=True)),
    ("n_pscut_freq", dict(lamsteps=False, cutmid=0, startbin=1, powerspec_cut=True)),
    # the first row alone above the white-noise level on the 61 x 103 arc
    ("n_pscut_one", dict(lamsteps=True, cutmid=0, startbin=1, powerspec_cut=True, eta=1600.0)),
    ("n_numsteps", dict(lamsteps=False, cutmid=4, startbin=3, numsteps=777, maxnormfac=2)),
]
FIT_CALLS = [
    ("f_lam", dict(lamsteps=True)),
    ("f_freq", dict(lamsteps=False)),
    ("f_freq_f64", dict(lamsteps=False)),
    ("f_asymm", dict(lamsteps=True, asymm=True)),
    ("f_start0", dict(lamsteps=True, startbin=0)),
    ("f_cut0", dict(lamsteps=True, cutmid=0)),
    ("f_cutwide", dict(lamsteps=True, cutmid=15)),
    ("f_weighted", dict(lamsteps=True, weighted=True)),
    ("f_numsteps", dict(lamsteps=True, numsteps=3000)),
]


def arc_dyn(rng, nf, nt, dt, df, eta_true=0.35, nimg=200):
    """|sum of images on a parabola|^2 with 2 % noise (as in make_golden.golden_fit_arc)."""
    fdk = rng.uniform(-14.0, 14.0, nimg)
    ak = (rng.normal(size=nimg) + 1j * rng.normal(size=nimg)) * np.exp(-(fdk / 7.0) ** 2)
    ak[0] += 12.0
    fdk[0] = 0.0
    t = dt * np.arange(nt)
    f = df * np.arange(nf)
    E = sum(a * np.exp(2j * np.pi * (fd_ * 1e-3 * t[None, :] - eta_true * fd_ ** 2 * f[:, None]))
            for a, fd_ in zip(ak, fdk))
    dyn = np.abs(E) ** 2
    return dyn + rng.normal(0.0, 0.02 * dyn.mean(), dyn.shape)


def spectra(pkg, dyn, dt, df, f0, nzero=0, rng=None):
    """Both secondary spectra of the reference, rounded to float32; with nzero, that many
    linear power bins of each are set to exactly zero before the dB step."""
    ds = _ref_dynspec(pkg, dyn.copy(), dt, df, f0)
    out = {}
    for lam in (True, False):
        fd, yaxis, sec = ds.calc_sspec(lamsteps=lam, return_sspec=True)
        if nzero:
            lin = 10 ** (np.asarray(sec) / 10)
            lin.flat[rng.choice(lin.size, nzero, replace=False)] = 0.0
            with np.errstate(divide="ignore"):
                sec = 10 * np.log10(lin)
        out["lamsspec" if lam else "sspec"] = np.asarray(sec, dtype=np.float32)
        out["beta" if lam else "tdel"] = np.asarray(yaxis, dtype=np.float64)
        out["fdop"] = np.asarray(fd, dtype=np.float64)
    return out


def fresh(pkg, g, f64=False):
    """A reference Dynspec holding the stored (float32-valued) spectra and axes."""
    ds = _ref_dynspec(pkg, g["dyn"].copy(), g["dt"], g["df"], g["f0"])
    assert type(ds.freq) is float and ds.freq == g["freq"]
    if f64:
        ds.freq = np.float64(ds.freq)
    ds.sspec = g["sspec"].astype(np.float64)
    ds.lamsspec = g["lamsspec"].astype(np.float64)
    ds.tdel, ds.beta, ds.fdop = g["tdel"].copy(), g["beta"].copy(), g["fdop"].copy()
    return ds


def run_calls(pkg, g, eta_freq, eta_lam):
    out = {}
    calls = [(n, "norm_sspec", kw) for n, kw in NORM_CALLS] + \
        [(n, "fit_arc", kw) for n, kw in FIT_CALLS]
    for name, kind, kw in calls:
        kw = dict(kw)
        if kind == "norm_sspec" and "eta" not in kw:
            kw["eta"] = eta_lam if kw["lamsteps"] else eta_freq
        ds = fresh(pkg, g, name.endswith("_f64"))
        out[name + "_kind"] = kind
        out[name + "_kwargs"] = json.dumps(kw, sort_keys=True)
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                with np.errstate(all="ignore"):
                    getattr(ds, kind)(plot=False, **kw)
        except Exception as e:      # noqa: BLE001 -- the type is the fixture
            out[name + "_raises"] = type(e).__name__
            print("  %-22s raises %s: %s" % (name, type(e).__name__, e))
            continue
        out[name + "_raises"] = ""
        if kind == "norm_sspec":
            out.update({name + "_normsspec": np.ma.filled(ds.normsspec, np.nan).astype(np.float32),
                        name + "_mask": np.ma.getmaskarray(ds.normsspec),
                        name + "_normsspecavg": np.ma.filled(ds.normsspecavg, np.nan),
                        name + "_powerspectrum": np.ma.filled(ds.powerspectrum, np.nan),
                        name + "_fdop": np.asarray(ds.normsspec_fdop, dtype=np.float64),
                        name + "_tdel": np.asarray(ds.normsspec_tdel, dtype=np.float64)})
            print("  %-22s normsspec %s, %d masked" % (name, ds.normsspec.shape,
                                                       int(np.ma.getmaskarray(ds.normsspec).sum())))
        else:
            pre = "betaeta" if kw.get("lamsteps") else "eta"
            sufs = ("_left", "_right") if kw.get("asymm") else ("",)
            for suf in sufs:
                for q in ("", "err", "err2"):
                    out[name + "_eta" + q + suf] = float(getattr(ds, pre + q + suf))
            ea = np.asarray(ds.eta_array, dtype=np.float64)
            out.update({name + "_noise": float(ds.noise), name + "_eta_array_n": ea.size,
                        name + "_eta_array_ends": ea[[0, -1]]})
            print("  %-22s %s%s = %s" % (name, pre, sufs[0],
                                         out[name + "_eta" + sufs[0]]))
    return out


def make(pkg, fname, dyn, dt, df, f0, eta_freq, eta_lam, nzero=0, seed=0):
    rng = np.random.default_rng(seed)
    freq = float(np.mean(f0 + df * np.arange(dyn.shape[0])))
    g = dict(dyn=dyn.astype(np.float32), dt=dt, df=df, f0=f0, freq=freq)
    g.update(spectra(pkg, dyn, dt, df, f0, nzero, rng))
    g["ninf"] = int(np.isneginf(g["sspec"]).sum() + np.isneginf(g["lamsspec"]).sum())
    print(fname, "sspec", g["sspec"].shape, "lamsspec", g["lamsspec"].shape,
          "-inf bins", g["ninf"])
    g.update(run_calls(pkg, g, eta_freq, eta_lam))
    path = os.path.join(GOLD, fname)
    np.savez_compressed(path, **g)
    print("  %d KiB" % (os.path.getsize(path) // 1024))


def main():
    pkg = ref_loader.load()
    rng = np.random.default_rng(61103)
    make(pkg, "arcfit_61x103.npz", arc_dyn(rng, 61, 103, 8.0, 0.25), 8.0, 0.25, 1300.0,
         eta_freq=0.35, eta_lam=800.0)
    rng = np.random.default_rng(4890)
    make(pkg, "arcfit_zeros_48x90.npz", arc_dyn(rng, 48, 90, 8.0, 0.25), 8.0, 0.25, 1300.0,
         eta_freq=0.35, eta_lam=800.0, nzero=8, seed=3)


if __name__ == "__main__":
    main()
