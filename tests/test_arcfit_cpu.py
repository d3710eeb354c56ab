"""Host glue of the classical arc fit (scintools_b200/arcfit.py: Dynspec.norm_sspec /
fit_arc) against outputs of the unmodified reference (tests/golden/fit_arc_128x160.npz,
norm_sspec_64x96.npz), with the device resampling replaced by a numpy stand-in that
follows the reference loop (np.interp per delay row) -- no GPU needed.  The CUDA
kernels themselves are checked in tests/test_gpu_arcfit.py."""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def numpy_norm_rows(sspec, fdop, tdel, eta, maxnormfac, fdopnew, weights_fn, want_2d=True):
    """dynspec.py:2076-2166 in numpy (oracle/dynspec_oracle.norm_sspec's loop).  avg is
    what the device returns: the weighted mean of the unmasked samples, +-inf where one
    of them is infinite (np.ma.average masks those), NaN where the weights sum to zero."""
    rows, mask = [], []
    for ii in range(len(tdel)):
        s = np.sqrt(tdel[ii] / eta)
        sel = abs(fdop) <= maxnormfac * s
        ifdop = fdop[sel] / s
        rows.append(np.interp(fdopnew, ifdop, sspec[ii, sel]))
        mask.append(np.abs(fdopnew) > np.max(np.abs(ifdop)))
    norm = np.array(rows).squeeze()
    mask = np.array(mask).squeeze() + np.isnan(norm)
    nm = nm_all = np.ma.array(norm, mask=mask)
    power = np.ma.filled(np.ma.mean(np.power(10, nm / 10), axis=1), np.nan)
    w = weights_fn(power)
    if isinstance(w, tuple):        # (weights, rows): only the selected rows are averaged
        w, rows = w
        nm, w = nm[np.asarray(rows, dtype=bool)], np.asarray(w)[np.asarray(rows, dtype=bool)]
    if np.ndim(nm) == 2 and nm.shape[0] == 0:
        return np.ma.filled(nm_all, np.nan), power, np.full(np.shape(fdopnew)[0], np.nan)
    a = np.ma.average(nm, axis=0, weights=w)
    avg = np.where(np.ma.getmaskarray(a) & ~np.isinf(np.ma.getdata(a)), np.nan, np.ma.getdata(a))
    return np.ma.filled(nm_all, np.nan), power, avg


@pytest.fixture()
def host_only(monkeypatch):
    from scintools_b200 import arcfit
    monkeypatch.setattr(arcfit, "_norm_rows", numpy_norm_rows)
    return arcfit


def _bare_dynspec(g):
    from scintools_b200.dynspec import BasicDyn, Dynspec
    dyn = g["dyn"]
    nf, nt = dyn.shape
    dt, df = float(g["dt"]), float(g["df"])
    f0 = float(g["f0"]) if "f0" in g.files else 1400.0
    return Dynspec(dyn=BasicDyn(dyn, times=dt * np.arange(nt), freqs=f0 + df * np.arange(nf),
                                dt=dt, df=df), verbose=False)


def test_fit_arc_host_logic_matches_reference(host_only, golden_dir):
    g = np.load(os.path.join(golden_dir, "fit_arc_128x160.npz"))
    ds = _bare_dynspec(g)
    # the reference's own secondary spectrum: this test is about the glue after it
    ds.lamsspec, ds.beta, ds.fdop, ds.tdel = g["lamsspec"], g["beta"], g["fdop"], g["tdel"]
    ds.fit_arc(lamsteps=True)
    assert ds.betaeta == pytest.approx(float(g["betaeta"]), rel=1e-9)
    assert ds.betaetaerr == pytest.approx(float(g["betaetaerr"]), rel=1e-9)
    assert ds.betaetaerr2 == pytest.approx(float(g["betaetaerr2"]), rel=1e-7)
    assert ds.noise == pytest.approx(float(g["noise"]), rel=1e-12)
    assert np.allclose(ds.eta_array, g["eta_array"], rtol=1e-12)
    assert np.allclose(np.ma.filled(ds.norm_sspec_avg, np.nan), g["norm_sspec_avg"],
                       rtol=1e-9, equal_nan=True)
    assert np.allclose(np.ma.filled(ds.prob_eta_peak, np.nan), g["prob_eta_peak"], rtol=1e-7,
                       equal_nan=True)
    assert np.allclose(ds.normsspec_fdop, g["nsf"]) and np.allclose(ds.normsspec_tdel, g["nst"])
    assert np.allclose(np.ma.filled(ds.normsspecavg, np.nan), g["nsa"], rtol=1e-9, equal_nan=True)
    assert np.allclose(np.ma.filled(ds.powerspectrum, np.nan), g["powerspectrum"], rtol=1e-9,
                       equal_nan=True)
    ds.fit_arc(lamsteps=True, asymm=True, nsmooth=7, low_power_diff=-2.0, high_power_diff=-1.0)
    assert ds.betaeta_left == pytest.approx(float(g["betaeta_left"]), rel=1e-9)
    assert ds.betaeta_right == pytest.approx(float(g["betaeta_right"]), rel=1e-9)
    assert ds.betaetaerr_left == pytest.approx(float(g["betaetaerr_left"]), rel=1e-9)
    assert ds.betaetaerr_right == pytest.approx(float(g["betaetaerr_right"]), rel=1e-9)
    ds.fit_arc(lamsteps=True, numsteps=4000, etamin=300.0, etamax=12000.0, log_parabola=True,
               weighted=True, cutmid=5, startbin=4)
    assert ds.betaeta == pytest.approx(float(g["betaeta_log"]), rel=1e-9)
    assert ds.betaetaerr == pytest.approx(float(g["betaetaerr_log"]), rel=1e-9)
    assert ds.betaetaerr2 == pytest.approx(float(g["betaetaerr2_log"]), rel=1e-7)


def test_norm_sspec_host_logic_matches_reference(host_only, golden_dir):
    g = np.load(os.path.join(golden_dir, "norm_sspec_64x96.npz"))
    ds = _bare_dynspec(g)
    ds.sspec, ds.fdop, ds.tdel = g["sspec"], g["fdop"], g["tdel"]
    ds.freq = float(g["freq"])
    ds.norm_sspec(eta=float(g["eta"]), lamsteps=False, cutmid=int(g["cutmid"]),
                  startbin=int(g["startbin"]))
    assert np.array_equal(np.ma.getmaskarray(ds.normsspec), g["mask"])
    assert np.allclose(np.ma.filled(ds.normsspec, np.nan), g["normsspec"], rtol=1e-12,
                       equal_nan=True)
    assert np.allclose(np.ma.filled(ds.normsspecavg, np.nan), g["normsspecavg"], rtol=1e-10,
                       equal_nan=True)
    assert np.allclose(ds.normsspec_fdop, g["normsspec_fdop"])
    assert np.allclose(np.ma.filled(ds.powerspectrum, np.nan), g["powerspectrum"], rtol=1e-10,
                       equal_nan=True)


def test_unsupported_modes_raise(host_only, golden_dir):
    g = np.load(os.path.join(golden_dir, "norm_sspec_64x96.npz"))
    ds = _bare_dynspec(g)
    ds.sspec, ds.fdop, ds.tdel = g["sspec"], g["fdop"], g["tdel"]
    for kw in (dict(plot=True), dict(logsteps=True), dict(fit_spectrum=True), dict(velocity=True)):
        with pytest.raises(NotImplementedError):
            ds.norm_sspec(eta=0.4, lamsteps=False, **kw)
    with pytest.raises(NotImplementedError):
        ds.fit_arc(plot=True)
