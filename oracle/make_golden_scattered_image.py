"""Generate tests/golden/scatim_*.npz by running the UNMODIFIED reference's
Dynspec.calc_scattered_image (via oracle/ref_loader.py, matplotlib mocked) on the CPU.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python oracle/make_golden_scattered_image.py

One file, ``scatim_arc_48x80.npz``: a 1-D-screen arc (48 channels x 80 subints,
oracle/make_golden_arcfit.arc_dyn).  It stores the input (``dyn``, ``dt``, ``df``, ``f0``),
the reference's spectra and axes that the calls read (``sspec``, ``lamsspec``, ``fdop``,
``tdel``, ``beta``), a second spectrum on its own axes for ``input_sspec`` (``alt_sspec``,
``alt_fdop``, ``alt_tdel``), then per call, prefixed by its name:

  <name>_kwargs   the keyword arguments as JSON; "input_sspec": "sspec" / "alt" / "minf" /
                  "nan" names the array passed ("minf", "nan": copies of ``sspec`` with
                  ``minf_idx`` set to -inf or ``nan_idx`` set to NaN), with the axes that go
                  with it
  <name>_preset   JSON of attributes set on the object before the call (eta, betaeta;
                  "freq": "float64" holds freq as numpy.float64)
  <name>_raises   the exception type name, or "" when the call returns
  <name>_eta, <name>_betaeta   the object's curvatures after the call (NaN if unset): the
                  fit_arc cases record what the reference's fit found
  <name>_ax       scattered_image_ax
  <name>_image    scattered_image when it has at most 4096 pixels; larger images store
                  <name>_idx (2048 seeded flat positions), <name>_val and <name>_absmax
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
from oracle.make_golden_arcfit import arc_dyn  # noqa: E402

NF, NT, DT, DF, F0 = 48, 80, 8.0, 0.25, 1300.0


def calls(fdop, tdel):
    """(name, kwargs, preset); the etas that pick the crops are computed from the axes."""
    tmax = float(np.max(tdel))
    # flim == 1: the column slice starts at 1 - int(0.02 nf) < 0 and wraps to the last columns
    wrap1 = 0.5 * (tmax / fdop[0] ** 2 + tmax / fdop[1] ** 2)
    wrap2 = 0.5 * (tmax / fdop[1] ** 2 + tmax / fdop[2] ** 2)
    flim0 = 0.3 * tmax / fdop[0] ** 2
    return [
        ("eta", dict(input_eta=0.35), {}),
        ("eta_nolog", dict(input_eta=0.35, plot_log=False), {}),
        # fit_arc divides its default constraint list by a Python-float freq (TypeError)
        ("fit_freq", dict(), {}),
        ("fit_freq_f64", dict(), {"freq": "float64"}),
        ("fit_lam", dict(lamsteps=True), {}),
        ("fit_lam_ref", dict(lamsteps=True, ref_freq=1100), {"betaeta": 800.0}),
        ("preset_eta", dict(), {"eta": 0.5}),
        ("nofit", dict(fit_arc=False), {}),
        ("nofit_alt", dict(input_sspec="alt", fit_arc=False, sampling=12), {}),
        ("flim0", dict(input_eta=flim0), {}),
        ("flim0_s7", dict(input_eta=flim0, sampling=7, plot_log=False), {}),
        ("wrap", dict(input_eta=wrap1, sampling=9), {}),
        ("wrap_short", dict(input_eta=wrap2), {}),
        # plot_scattered_image's centres_to_edges needs two axis points (IndexError)
        ("s0", dict(input_eta=0.35, sampling=0), {}),
        ("s0_nolog", dict(input_eta=0.35, sampling=0, plot_log=False), {}),
        ("s1", dict(input_eta=0.35, sampling=1), {}),
        ("s1_nolog", dict(input_eta=0.35, sampling=1, plot_log=False), {}),
        ("s157", dict(input_eta=0.2, sampling=157), {}),
        ("minf", dict(input_sspec="minf", input_eta=0.35, sampling=20), {}),
        ("alt", dict(input_sspec="alt", input_eta=0.02, sampling=33), {}),
        ("alt_nolog", dict(input_sspec="alt", input_eta=0.02, plot_log=False), {}),
        ("stop", dict(input_eta=float("nan")), {}),
        ("attr", dict(), {"betaeta": 800.0}),
        ("nan", dict(input_sspec="nan", input_eta=0.35), {}),
        ("nan_nolog", dict(input_sspec="nan", input_eta=0.35, sampling=4, plot_log=False), {}),
        ("angle", dict(input_eta=0.35, use_angle=True), {}),
        ("spatial", dict(input_eta=0.35, use_spatial=True, s=0.5, veff=100.0), {}),
    ]


def main():
    pkg = ref_loader.load()
    rng = np.random.default_rng(4880)
    dyn = arc_dyn(rng, NF, NT, DT, DF)
    ds = _ref_dynspec(pkg, dyn.copy(), DT, DF, F0)
    g = dict(dyn=dyn, dt=DT, df=DF, f0=F0)
    fdop, tdel, sec = ds.calc_sspec(return_sspec=True)
    _, beta, lsec = ds.calc_sspec(lamsteps=True, return_sspec=True)
    g.update(sspec=np.asarray(sec, dtype=np.float64), lamsspec=np.asarray(lsec, dtype=np.float64),
             fdop=np.asarray(fdop, dtype=np.float64), tdel=np.asarray(tdel, dtype=np.float64),
             beta=np.asarray(beta, dtype=np.float64))
    adyn = arc_dyn(rng, 30, 40, 4.0, 0.5)
    afd, atd, asec = _ref_dynspec(pkg, adyn, 4.0, 0.5, 1500.0).calc_sspec(return_sspec=True)
    g.update(alt_sspec=np.asarray(asec, dtype=np.float64), alt_fdop=np.asarray(afd, np.float64),
             alt_tdel=np.asarray(atd, np.float64))
    n = g["sspec"].size
    g["minf_idx"] = rng.choice(n, 40, replace=False)
    g["nan_idx"] = np.array([g["sspec"].shape[1] * 3 + g["sspec"].shape[1] // 2 + 5])
    arrays = dict(sspec=(g["sspec"], g["fdop"], g["tdel"]),
                  alt=(g["alt_sspec"], g["alt_fdop"], g["alt_tdel"]))
    minf = g["sspec"].copy()
    minf.flat[g["minf_idx"]] = -np.inf
    nan = g["sspec"].copy()
    nan.flat[g["nan_idx"]] = np.nan
    arrays.update(minf=(minf, g["fdop"], g["tdel"]), nan=(nan, g["fdop"], g["tdel"]))
    pick = np.random.default_rng(7)
    for name, kw, preset in calls(g["fdop"], g["tdel"]):
        r = _ref_dynspec(pkg, dyn.copy(), DT, DF, F0)
        r.sspec, r.lamsspec = g["sspec"].copy(), g["lamsspec"].copy()
        r.fdop, r.tdel, r.beta = g["fdop"].copy(), g["tdel"].copy(), g["beta"].copy()
        for k, v in preset.items():
            setattr(r, k, np.float64(r.freq) if v == "float64" else v)
        args = dict(kw)
        if "input_sspec" in args:
            a = arrays[args["input_sspec"]]
            args.update(input_sspec=a[0].copy(), input_fdop=a[1].copy(), input_tdel=a[2].copy())
        g[name + "_kwargs"] = json.dumps(kw, sort_keys=True)
        g[name + "_preset"] = json.dumps(preset, sort_keys=True)
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                with np.errstate(all="ignore"):
                    r.calc_scattered_image(**args)
        except Exception as e:      # noqa: BLE001 -- the type is the fixture
            g[name + "_raises"] = type(e).__name__
            assert not hasattr(r, "scattered_image")
            print("  %-12s raises %s: %s" % (name, type(e).__name__, e))
            continue
        g[name + "_raises"] = ""
        for k in ("eta", "betaeta"):
            g[name + "_" + k] = float(getattr(r, k, np.nan))
        im = np.asarray(r.scattered_image, dtype=np.float64)
        g[name + "_ax"] = np.asarray(r.scattered_image_ax, dtype=np.float64)
        if im.size <= 4096:
            g[name + "_image"] = im
        else:
            idx = np.sort(pick.choice(im.size, 2048, replace=False))
            g[name + "_idx"], g[name + "_val"] = idx, im.flat[idx]
            g[name + "_shape"] = np.array(im.shape)
            g[name + "_absmax"] = float(np.nanmax(np.abs(im)))
        print("  %-12s image %s, eta %r betaeta %r" % (name, im.shape, g[name + "_eta"],
                                                       g[name + "_betaeta"]))
    path = os.path.join(GOLD, "scatim_arc_48x80.npz")
    np.savez_compressed(path, **g)
    print("%s: %d KiB" % (path, os.path.getsize(path) // 1024))


if __name__ == "__main__":
    main()
