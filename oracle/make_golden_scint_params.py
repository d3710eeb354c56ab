"""Generate tests/golden/scint_params_*.npz: the UNMODIFIED reference's
Dynspec.get_scint_params / get_acf_tilt (via oracle/ref_loader.py), with the lmfit stand-in
of oracle/scint_params_oracle.py installed first.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python oracle/make_golden_scint_params.py

One file per spectrum.  Keys: ``dyn`` (float64 input), ``acf_sha`` (sha256 of the
reference's float64 ACF, which oracle.dynspec_oracle.calc_acf reproduces; or ``acf`` itself
for the crafted ACFs, which no spectrum makes), the Dynspec attributes in ``meta`` (dt, df,
tobs, bw, nsub, nchan, freq) and ``name``, and per case ``<case>/...``:
  kwargs (repr of the call's keyword arguments), call ('scint' or 'tilt', or 'scint+tilt'),
  error (the exception type name, or '');
  fit<k>/model, fit<k>/p0_<name> / vary_<name>, fit<k>/arg<i> (the 1-D fcn_args) or
  fit<k>/box (row0, nrows, col0, ncols of the 2-D crop in the ACF), fit<k>/tdata,
  fit<k>/fdata, fit<k>/ydata_sha, fit<k>/weights_sha, fit<k>/weights_special (the
  positions of the weights that are not the formula's: value, row, col);
  fit<k>/value_<name>, fit<k>/stderr_<name> (NaN for None), fit<k>/chisqr, nfev, success;
  attr_<name> for every attribute the call set (scalars; None as NaN with attrnone_<name>).
Cases: three J0437-4715 observations (load_file: zapped channels, odd sub-integration
counts) with acf1d, acf2d_approx and nofit; on the second also free alpha, weighted=False,
bartlett=False, full_frame=True, tau_vary_2d=False with tau_input, a 'sim:mb2=' name, and
get_acf_tilt before and after a fit; a seeded synthetic spectrum with a prescribed ACF and
a phase-gradient shear; and crafted ACFs for the fallback guesses, the crop floor, the
frequency-range branch and the IndexError branch.
"""
import glob
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import scint_params_oracle as SO  # noqa: E402

SO.install()
from oracle import ref_loader  # noqa: E402
from oracle import dynspec_oracle as DO  # noqa: E402

META = ("dt", "df", "tobs", "bw", "nsub", "nchan", "freq")
ATTRS = ("tau", "dnu", "amp", "wn", "tauerr", "dnuerr", "amperr", "tscat", "nscint",
         "fse_tau", "fse_dnu", "talpha", "talphaerr", "scint_param_method", "dnu_est",
         "dnu_esterr", "tscat_est", "modulation_index", "wnerr", "phasegrad", "phasegraderr",
         "fse_phasegrad", "acf_tilt", "acf_tilt_err", "fse_tilt")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


def crop_box(acf, view):
    off = view.__array_interface__["data"][0] - acf.__array_interface__["data"][0]
    row, rem = divmod(off, acf.strides[0])      # the reference's ACF is a strided real view
    col = rem // acf.strides[1]
    return np.array([row, view.shape[0], col, view.shape[1]])


def specials(weights):
    """Entries of the 2-D fcn_args weights that the formula cannot give: 1e10."""
    pos = np.argwhere(weights == 1e10)
    return np.array([[1e10, r, c] for r, c in pos]).reshape(-1, 3)


def make_ds(R, dyn, meta, name, acf=None):
    ds = R.dynspec.Dynspec.__new__(R.dynspec.Dynspec)
    ds.dyn = np.array(dyn, dtype=np.float64)
    ds.name = name
    for k, v in meta.items():
        setattr(ds, k, v)
    if acf is not None:
        ds.acf = np.array(acf, dtype=np.float64)
    return ds


def run_case(R, out, case, dyn, meta, name, acf, call, kwargs, pre_attrs=None):
    ds = make_ds(R, dyn, meta, name, acf)
    for k, v in (pre_attrs or {}).items():
        setattr(ds, k, v)
    SO.CALLS.clear()
    before = set(vars(ds))
    err = ""
    try:
        if call in ("scint", "scint+tilt"):
            ds.get_scint_params(**kwargs)
        if call in ("tilt", "scint+tilt"):
            ds.get_acf_tilt()
    except Exception as e:  # the reference's own exception, recorded by type
        err = type(e).__name__
    p = case + "/"
    out[p + "kwargs"] = repr(kwargs)
    out[p + "call"] = call
    out[p + "error"] = err
    for k, rec in enumerate(SO.CALLS):
        q = p + "fit%d/" % k
        out[q + "model"] = rec["model"]
        for n, par in rec["params0"].items():
            out[q + "p0_" + n] = float(par.value)
            out[q + "vary_" + n] = bool(par.vary)
        args = rec["fcn_args"]
        if rec["model"] == "scint_acf_model":
            (xt, xf), (yt, yf), (wt, wf) = args
            ones_t = np.ones(np.shape(yt)) if wt is None else wt
            ones_f = np.ones(np.shape(yf)) if wf is None else wf
            for i, a in enumerate((xt, xf, yt, yf, ones_t, ones_f)):
                out[q + "arg%d" % i] = np.asarray(a, dtype=np.float64)
            out[q + "weighted"] = wt is not None
        else:
            tdata, fdata, y2, w2 = args
            out[q + "box"] = crop_box(ds.acf, y2)
            out[q + "tdata"] = tdata
            out[q + "fdata"] = fdata
            out[q + "ydata_sha"] = sha(y2)
            out[q + "weights_sha"] = sha(w2)
            out[q + "weights_special"] = specials(w2)
        res = rec.get("result")
        if res is not None:
            for n, par in res.params.items():
                out[q + "value_" + n] = float(par.value)
                out[q + "stderr_" + n] = np.nan if par.stderr is None else float(par.stderr)
            out[q + "chisqr"] = res.chisqr
            out[q + "nfev"] = res.nfev
            out[q + "success"] = res.success
    for n in set(vars(ds)) - before:
        if n not in ATTRS:
            continue
        v = getattr(ds, n)
        if v is None:
            out[p + "attrnone_" + n] = True
            v = np.nan
        out[p + "attr_" + n] = v
    return ds


def crafted_acf(nf, nt, dt, df, tau, dnu, spike=0.05, shear=0.0, seed=0, tri=True):
    """An ACF surface [2 nf][2 nt]: the 2-D approximate model (with the triangle if tri)
    plus a white-noise spike at the centre and a little noise, normalised to a peak of 1."""
    tl = (np.arange(2 * nt) - nt) * dt
    fl = (np.arange(2 * nf) - nf) * df
    T, F = np.meshgrid(tl, fl)
    m = np.exp(-(np.abs((T - shear * F) / tau) ** 2.5 +
                 np.abs(F / (dnu / np.log(2))) ** 1.5) ** (2 / 3))
    if tri:
        m *= (1 - np.abs(T) / (nt * dt)) * (1 - np.abs(F) / (nf * df))
    m += np.random.default_rng(seed).normal(0, 0.003, m.shape)
    m[nf, nt] += spike
    return m / m.max()


def synthetic(seed=3, nf=96, nt=128, dt=8.0, df=0.25, tau=120.0, dnu=1.5, grad=40.0):
    """A seeded dynamic spectrum with a Gaussian-correlated intensity field of scale tau in
    time and dnu in frequency, sheared by `grad` s/MHz (a phase gradient)."""
    rng = np.random.default_rng(seed)
    pad_t, pad_f = 3 * nt, 3 * nf
    kt = np.fft.fftfreq(pad_t, dt)
    kf = np.fft.fftfreq(pad_f, df)
    KT, KF = np.meshgrid(kt, kf)
    amp = np.exp(-(np.pi * tau * KT) ** 2 - (np.pi * dnu * (KF + grad * KT)) ** 2)
    z = np.fft.ifft2(amp * (rng.normal(size=amp.shape) + 1j * rng.normal(size=amp.shape)))
    I = np.abs(z[:nf, :nt]) ** 2
    return I / I.mean()


def main():
    R = ref_loader.load()
    files = sorted(glob.glob(os.path.join(ref_loader.REFERENCE_ROOT, "scintools", "examples",
                                          "data", "J0437-4715", "*.dynspec")))
    for idx in (0, 1, 2):
        ds0 = R.dynspec.Dynspec(filename=files[idx], verbose=False, process=False)
        meta = {k: getattr(ds0, k) for k in META}
        name = ds0.name
        dyn = np.array(ds0.dyn, dtype=np.float64)
        ds0.calc_acf()
        assert np.array_equal(ds0.acf, DO.calc_acf(dyn))
        out = {"dyn": dyn, "acf_sha": sha(ds0.acf), "name": name,
               "meta": np.array([float(meta[k]) for k in META])}
        cases = [("acf1d", "scint", dict(method="acf1d")),
                 ("acf2d", "scint", dict(method="acf2d_approx")),
                 ("nofit", "scint", dict(method="nofit"))]
        if idx == 1:
            cases += [("alpha_free", "scint", dict(method="acf1d", alpha=None)),
                      ("alpha_free_2d", "scint", dict(method="acf2d_approx", alpha=None)),
                      ("unweighted_2d", "scint", dict(method="acf2d_approx", weighted=False)),
                      ("nobartlett", "scint", dict(method="acf1d", bartlett=False)),
                      ("full_frame_1d", "scint", dict(method="acf1d", full_frame=True)),
                      ("full_frame_2d", "scint", dict(method="acf2d_approx", full_frame=True)),
                      ("tau_fixed_2d", "scint", dict(method="acf2d_approx", tau_vary_2d=False,
                                                    tau_input=3000.0)),
                      ("tilt_first", "tilt", {}),
                      ("tilt_then_2d", "scint+tilt", dict(method="acf1d"))]
        for case, call, kw in cases:
            run_case(R, out, case, dyn, meta, name, None, call, kw)
        if idx == 1:
            # the 2-D fit started from a measured tilt
            ds = make_ds(R, dyn, meta, name)
            ds.get_acf_tilt()
            run_case(R, out, "acf2d_from_tilt", dyn, meta, name, None, "scint",
                     dict(method="acf2d_approx"),
                     pre_attrs={"acf_tilt": ds.acf_tilt, "acf_tilt_err": ds.acf_tilt_err})
            run_case(R, out, "simname", dyn, meta, "sim:mb2=2.0,ar=1", None, "scint",
                     dict(method="acf1d"))
        np.savez_compressed(os.path.join(GOLD, "scint_params_j0437_%d.npz" % idx), **out)
        print("J0437 observation", idx, "done")

    # a seeded synthetic spectrum: 96 x 128, tau 120 s, dnu 1.5 MHz, shear 40 s/MHz
    dyn = synthetic()
    nf, nt = dyn.shape
    meta = dict(dt=8.0, df=0.25, tobs=nt * 8.0, bw=nf * 0.25, nsub=nt, nchan=nf, freq=1400.0)
    assert np.array_equal(DO.calc_acf(dyn), DO.calc_acf(dyn))
    out = {"dyn": dyn, "acf_sha": sha(DO.calc_acf(dyn)), "name": "synthetic",
           "meta": np.array([float(meta[k]) for k in META])}
    for case, call, kw in [("acf1d", "scint", dict(method="acf1d")),
                           ("acf2d", "scint", dict(method="acf2d_approx")),
                           ("alpha_free", "scint", dict(method="acf1d", alpha=None)),
                           ("nofit", "scint", dict(method="nofit"))]:
        run_case(R, out, case, dyn, meta, "synthetic", None, call, kw)
    np.savez_compressed(os.path.join(GOLD, "scint_params_synthetic.npz"), **out)

    # crafted ACFs for the branches real spectra rarely reach
    nf, nt, dt, df = 40, 48, 10.0, 0.5
    meta = dict(dt=dt, df=df, tobs=nt * dt, bw=nf * df, nsub=nt, nchan=nf, freq=1400.0)
    dyn = np.random.default_rng(9).exponential(1.0, (nf, nt))
    crafted = {
        # tau far beyond the span: no time lag under amp/e -> tau = tobs; dnu beyond bw:
        # dnu = bw, and nscale exceeds the frequency range (the tmin = 0, tmax = nf branch)
        "fallback": crafted_acf(nf, nt, dt, df, tau=1e4, dnu=1e3, tri=False),
        # scales under a sample: the 5-sample crop floor on both axes
        "floor": crafted_acf(nf, nt, dt, df, tau=4.0, dnu=0.2),
        # moderate scales with a shear: the ordinary crop
        "sheared": crafted_acf(nf, nt, dt, df, tau=60.0, dnu=3.0, shear=8.0),
    }
    # exactly one time lag under amp/e: the reference's squeeze()[0] raises IndexError
    a = crafted_acf(nf, nt, dt, df, tau=1e4, dnu=3.0, tri=False)
    a[nf, nt + 5] = -0.5
    crafted["indexerror"] = a
    out = {"dyn": dyn, "name": "crafted", "meta": np.array([float(meta[k]) for k in META])}
    for key, acf in crafted.items():
        out["acf_" + key] = acf
        for method in ("acf1d", "acf2d_approx"):
            run_case(R, out, "%s_%s" % (key, method), dyn, meta, "crafted", acf, "scint",
                     dict(method=method))
    np.savez_compressed(os.path.join(GOLD, "scint_params_crafted.npz"), **out)
    for fn in sorted(glob.glob(os.path.join(GOLD, "scint_params_*.npz"))):
        z = np.load(fn)
        print(os.path.basename(fn), os.path.getsize(fn),
              sorted(k.split("/")[0] + ":" + str(z[k]) for k in z.files if k.endswith("/error")))


if __name__ == "__main__":
    main()
