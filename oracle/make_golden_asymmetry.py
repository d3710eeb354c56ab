"""Generate tests/golden/asymmetry_sample.npz by running the UNMODIFIED reference's
Dynspec.calc_asymmetry / ththmod.calc_asymmetry (via oracle/ref_loader.py) on the tutorial
field.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python -m oracle.make_golden_asymmetry

Case a: Dynspec.calc_asymmetry on Sample_Data.npz (|E|^2 plus the seeded noise of
golden_thth in make_golden.py, the first 128 time bins, a few NaNs in one place), cwf=64,
cwt=32, npad=3, ththeta=40 s^3, 302 edges out to 0.3 mHz: 16 x 4 chunks of widths
32 / 48 / 64 / 80 (the reference's time slice ct*cwt//2 : (ct+1)*cwt), padded 256 x 128 /
192 / 256 / 320.  The field is stored as float16 and the reference runs on exactly those
values.  The reference's calc_asymmetry and eigsh are wrapped (not changed) so that each
chunk's arguments, its reduced theta-theta matrix and the (w, V) eigsh returned are
recorded next to the asymmetry: nred, the two largest eigenvalues, ||thth_red||_F,
S = sum|left|^2 + sum|right|^2 and |V|^2 (float32).

Case b: single chunks the reference cannot recover -- an all-zero chunk (ARPACK error), a
curvature whose crop keeps fewer than 3 centres, edges that reach past the fd axis
(IndexError).  The fixtures are committed; the GPU box never needs the reference.
"""
import contextlib
import io
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_loader  # noqa: E402

CWF, CWT, NPAD, THTHETA, NT = 64, 32, 3, 40.0, 128
EDGES = np.linspace(-0.3, 0.3, 302)
NANS = ((70, 20), (71, 40), (100, 41))      # (channel, time bin): chunk cf = 1, ct = 0..2


def field(arch):
    rng = np.random.default_rng(7)
    wf = arch["Espec"]
    dyn = (np.abs(wf) ** 2 + rng.normal(0, 20, wf.shape))[:, :NT].astype(np.float16)
    for f, t in NANS:
        dyn[f, t] = np.nan
    return dyn


def golden_asymmetry(pkg):
    u = sys.modules["astropy.units"]
    thth = pkg.ththmod
    arch = np.load(os.path.join(ref_loader.REFERENCE_ROOT, "scintools", "examples", "data",
                                "ththsims", "Sample_Data.npz"))
    dyn16 = field(arch)
    freqs, times = arch["f_MHz"], arch["t_s"][:NT]
    nf = dyn16.shape[0]
    df, dt = freqs[1] - freqs[0], times[1] - times[0]
    bd = pkg.dynspec.BasicDyn(dyn16.astype(np.float64), name="asym", header=["asym"],
                              times=times, freqs=freqs, nchan=nf, nsub=NT, bw=df * nf, df=df,
                              freq=float(np.mean(freqs)), tobs=dt * NT, dt=dt, mjd=60000)
    ds = pkg.dynspec.Dynspec(dyn=bd, verbose=False, process=False)
    ds.cwf, ds.cwt, ds.npad = CWF, CWT, NPAD
    ds.ncf_fit, ds.nct_fit = nf // CWF, NT // CWT
    ds.fref = freqs.mean() * u.MHz
    ds.edges = EDGES * u.mHz
    ds.ththeta = THTHETA * u.s ** 3
    calls, mats = [], []
    orig_calc, orig_eigsh = thth.calc_asymmetry, thth.eigsh

    def spy_calc(params):
        mats.append(None)
        calls.append(params)
        return orig_calc(params)

    def spy_eigsh(a, *args, **kw):
        mats[-1] = np.array(a)
        w, V = orig_eigsh(a, *args, **kw)
        mats[-1] = (np.array(a), w[0], V[:, 0])
        return w, V

    thth.calc_asymmetry, thth.eigsh = spy_calc, spy_eigsh
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ds.calc_asymmetry()
    finally:
        thth.calc_asymmetry, thth.eigsh = orig_calc, orig_eigsh
    asym = np.asarray(ds.asymmetry)
    nchunk = len(calls)
    nred = np.zeros(nchunk, np.int32)
    w1, w2, fro, S = (np.full(nchunk, np.nan) for _ in range(4))
    pad, eta, tslice = np.zeros(nchunk), np.zeros(nchunk), np.zeros((nchunk, 2), np.int32)
    for k, (p, m) in enumerate(zip(calls, mats)):
        dspec2, edges, time2, freq2, et, ct, cf, npad, _ = p
        pad[k] = dspec2.mean()
        eta[k] = float(et.value)
        t0 = int(np.flatnonzero(times == time2.value[0])[0])
        tslice[k] = (t0, t0 + time2.value.shape[0])
        if isinstance(m, tuple):
            a, _, V = m
            ev = np.linalg.eigvalsh(a)
            nred[k] = a.shape[0]
            w1[k], w2[k], fro[k] = ev[-1], ev[-2], np.linalg.norm(a)
            h = (nred[k] - 1) // 2
            S[k] = np.sum(np.abs(V[:h]) ** 2) + np.sum(np.abs(V[h + 1:]) ** 2)
    nmax = int(nred.max())
    V2 = np.zeros((nchunk, nmax), np.float32)
    for k, m in enumerate(mats):
        if isinstance(m, tuple):
            V2[k, :nred[k]] = np.abs(m[2]) ** 2
    ncf = ds.ncf_fit
    edges_cf = np.array([np.asarray(calls[k * ds.nct_fit][1].value) for k in range(ncf)])
    # case b: chunks the reference cannot recover
    d0 = np.nan_to_num(dyn16[CWF:2 * CWF, :CWT].astype(np.float64))
    d0 -= d0.mean()
    b_cases = dict(zero=(np.zeros((CWF, CWT)), EDGES, THTHETA),
                   small=(d0, EDGES, 1e9),
                   wide=(d0, np.linspace(-40.0, 40.0, 64), 0.01))
    b_out = {}
    for tag, (d, e, et) in b_cases.items():
        buf = io.StringIO()
        with warnings.catch_warnings(), contextlib.redirect_stdout(buf):
            warnings.simplefilter("ignore")
            res = thth.calc_asymmetry((d, e * u.mHz, times[:CWT] * u.s, freqs[CWF:2 * CWF] * u.MHz,
                                       et * u.s ** 3, 0, 1, NPAD, False))
        b_out["b_%s_asymm" % tag] = float(res[0])
        b_out["b_%s_printed" % tag] = buf.getvalue().strip()
        b_out["b_%s_edges" % tag] = e
        b_out["b_%s_eta" % tag] = et
        print("asymmetry b %s: %r, printed %r" % (tag, res[0], buf.getvalue().strip()))
    np.savez_compressed(
        os.path.join(GOLD, "asymmetry_sample.npz"), dyn=dyn16, freqs=freqs, times=times,
        cwf=CWF, cwt=CWT, npad=NPAD, ththeta=THTHETA, fref=float(freqs.mean()), edges=EDGES,
        asymmetry=asym, nred=nred, w1=w1, w2=w2, fro=fro, S=S, V2=V2, pad=pad, eta=eta,
        tslice=tslice, edges_cf=edges_cf, b_dspec=d0, **b_out)
    print("asymmetry a: %d chunks, %d NaN, nred %d..%d, min rel gap %.3g" %
          (nchunk, int(np.isnan(asym).sum()), nred.min(), nred.max(),
           np.nanmin((w1 - w2) / np.abs(w1))))


if __name__ == "__main__":
    golden_asymmetry(ref_loader.load())
