"""Generate tests/golden/mosaic_*.npz by running the UNMODIFIED reference's rotInit, rotMos,
rotFit, rotDer, fullMos, fullMosFit, fullMosGrad and fullMosHess (via oracle/ref_loader.py).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python -m oracle.make_golden_mosaic

Case a (mosaic_sample.npz): chunks from the reference's own Dynspec.thetatheta_chunks on
the tutorial Sample_Data.npz (|E|^2 of the first 140 time bins), 4 x 6 chunks of 64 x 40,
stored as complex64; the reference runs on exactly those values.  dspec = |E|^2 and
N = sqrt(dspec) + 1, cropped to the mosaic, float32; p = (rotInit, ones), so rotMos(x) is
stored once, as fullMos.
Case b (mosaic_synth.npz): chunks cut from one wavefield E with injected a_k e^{i psi_k},
one all-zero chunk, NaN pixels in dspec, p longer than 2P-1, N larger than the mosaic;
b2: a single-chunk frequency axis of odd width 7.
Case c (mosaic_errors.npz): the exception each reference function raises for an odd
width on a multi-chunk axis, a short x / p and a dspec of the wrong shape.
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_loader  # noqa: E402


def run_all(thth, ch, x, p, dspec, N):
    out = dict(chunks=ch, x=x, p=p, dspec=dspec, N=N)
    out["rotInit"] = thth.rotInit(ch)
    out["rotMos"] = thth.rotMos(ch, x)
    out["rotFit"] = thth.rotFit(x, ch)
    out["rotDer"] = thth.rotDer(x, ch)
    out["fullMos"] = thth.fullMos(ch, p)
    out["fullMosFit"] = thth.fullMosFit(p, ch, dspec, N)
    P = ch.shape[0] * ch.shape[1]
    nF, nT = out["fullMos"].shape
    out["fullMosGrad"] = thth.fullMosGrad(p, ch, dspec[:nF, :nT], N)
    out["fullMosHess"] = thth.fullMosHess(p, ch, dspec[:nF, :nT], N)
    if out["rotMos"].size < 20000:
        out["mosaic"] = thth.mosaic(ch)
    print("  P=%d mosaic %s fit %.6g |H| %.3g" % (P, (nF, nT), out["fullMosFit"],
                                                  np.abs(out["fullMosHess"]).max()))
    return out


def case_a(pkg):
    u = sys.modules["astropy.units"]
    thth = pkg.ththmod
    arch = np.load(os.path.join(ref_loader.REFERENCE_ROOT, "scintools", "examples", "data",
                                "ththsims", "Sample_Data.npz"))
    ncf, nct, cwf, cwt, npad = 4, 6, 64, 40, 3
    nf, nt = (ncf + 1) * cwf // 2, (nct + 1) * cwt // 2
    E = arch["Espec"][:nf, :nt]
    freqs, times = arch["f_MHz"][:nf], arch["t_s"][:nt]
    dyn = np.abs(E) ** 2
    df, dt = freqs[1] - freqs[0], times[1] - times[0]
    bd = pkg.dynspec.BasicDyn(dyn, name="mos", header=["mos"], times=times, freqs=freqs,
                              nchan=nf, nsub=nt, bw=df * nf, df=df, freq=float(np.mean(freqs)),
                              tobs=dt * nt, dt=dt, mjd=60000)
    ds = pkg.dynspec.Dynspec(dyn=bd, verbose=False, process=False)
    ds.cwf, ds.cwt, ds.npad = cwf, cwt, npad
    ds.ncf_ret, ds.nct_ret = ncf, nct
    ds.fref = freqs.mean() * u.MHz
    ds.edges = np.linspace(-0.3, 0.3, 128) * u.mHz
    ds.ththeta = 40.0 * u.s ** 3
    ds.thth_tau_mask = 0 * u.us
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ds.thetatheta_chunks()
    ch = np.asarray(ds.chunks).astype(np.complex64)
    P = ncf * nct
    x = thth.rotInit(ch)
    p = np.concatenate([x, np.ones(P)])
    dspec = dyn.astype(np.float32)
    N = (np.sqrt(dyn) + 1).astype(np.float32)
    out = run_all(thth, ch, x, p, dspec, N)
    # p = (x, ones): fullMos is rotMos(x); keep one copy so the fixture stays near 1 MB
    assert np.array_equal(out["rotMos"], out["fullMos"])
    del out["rotMos"]
    return out


def case_b(pkg, ncf, nct, cwf, cwt, seed, zero=None, nans=0, extra=0):
    thth = pkg.ththmod
    rng = np.random.default_rng(seed)
    nF = (ncf - 1) * (cwf // 2) + cwf
    nT = (nct - 1) * (cwt // 2) + cwt
    E = rng.normal(size=(nF, nT)) + 1j * rng.normal(size=(nF, nT))
    P = ncf * nct
    a = rng.uniform(0.5, 2.0, P)
    psi = rng.uniform(-np.pi, np.pi, P)
    ch = np.zeros((ncf, nct, cwf, cwt), complex)
    for cf in range(ncf):
        for ct in range(nct):
            k = cf * nct + ct
            ch[cf, ct] = E[cf * (cwf // 2):cf * (cwf // 2) + cwf,
                           ct * (cwt // 2):ct * (cwt // 2) + cwt] * a[k] * np.exp(1j * psi[k])
    if zero is not None:
        ch[zero] = 0
    ch = ch.astype(np.complex64)
    dspec = (np.abs(E) ** 2 + 0.1 * rng.normal(size=E.shape)).astype(np.float32)
    for _ in range(nans):
        dspec[rng.integers(nF), rng.integers(nT)] = np.nan
    N = rng.uniform(0.5, 1.5, (nF + 2, nT + 1)).astype(np.float32)
    x = rng.uniform(-np.pi, np.pi, P - 1 + extra)
    p = np.concatenate([rng.uniform(-np.pi, np.pi, P - 1), rng.uniform(0.5, 2, P),
                        rng.uniform(size=extra)])
    out = run_all(thth, ch, x, p, dspec, N)
    out.update(E=E.astype(np.complex64), a=a, psi=psi)
    return out


def case_c(pkg):
    thth = pkg.ththmod
    rng = np.random.default_rng(3)
    odd = (rng.normal(size=(2, 2, 7, 8)) + 0j).astype(np.complex64)
    ch = (rng.normal(size=(2, 3, 8, 8)) + 1j * rng.normal(size=(2, 3, 8, 8))).astype(np.complex64)
    P = 6
    good = np.ones((12, 16), np.float32)
    calls = dict(
        rotMos_odd=lambda: thth.rotMos(odd, np.zeros(3)),
        rotInit_odd=lambda: thth.rotInit(odd),
        fullMosFit_odd=lambda: thth.fullMosFit(np.ones(7), odd, good, good),
        rotMos_short=lambda: thth.rotMos(ch, np.zeros(P - 2)),
        rotDer_short=lambda: thth.rotDer(np.zeros(P - 2), ch),
        fullMos_short=lambda: thth.fullMos(ch, np.ones(2 * P - 2)),
        fullMosGrad_short=lambda: thth.fullMosGrad(np.ones(2 * P - 2), ch, good, good),
        fullMosHess_short=lambda: thth.fullMosHess(np.ones(2 * P - 2), ch, good, good),
        fullMosGrad_dspec=lambda: thth.fullMosGrad(np.ones(2 * P - 1), ch, np.ones((13, 16)), good),
        fullMosHess_dspec=lambda: thth.fullMosHess(np.ones(2 * P - 1), ch, np.ones((12, 15)), good),
        fullMosGrad_N=lambda: thth.fullMosGrad(np.ones(2 * P - 1), ch, good, np.ones((11, 16))),
        fullMosFit_small=lambda: thth.fullMosFit(np.ones(2 * P - 1), ch, np.ones((11, 16)), good),
    )
    out = {}
    for name, f in calls.items():
        try:
            f()
            out[name] = "none"
        except Exception as e:     # noqa: BLE001 -- recording what the reference raises
            out[name] = type(e).__name__
        print("  c %s: %s" % (name, out[name]))
    return out


if __name__ == "__main__":
    pkg = ref_loader.load()
    print("case a")
    np.savez_compressed(os.path.join(GOLD, "mosaic_sample.npz"), **case_a(pkg))
    print("case b")
    b = case_b(pkg, 3, 4, 16, 8, 11, zero=(1, 2), nans=5, extra=3)
    b2 = case_b(pkg, 1, 3, 7, 8, 12, extra=1)
    np.savez_compressed(os.path.join(GOLD, "mosaic_synth.npz"), **b,
                        **{"b2_" + k: v for k, v in b2.items()})
    print("case c")
    np.savez_compressed(os.path.join(GOLD, "mosaic_errors.npz"), **case_c(pkg))
