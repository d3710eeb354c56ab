"""Generate tests/golden/axes_geometry.npz by running the UNMODIFIED reference's ththmod
(via oracle/ref_loader.py and the units shim) on descending and offset axes and irregular
theta grids.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python -m oracle.make_golden_axes

One 32 x 75 dynamic spectrum (a 24-image arc at eta = 1/32 s^3 plus noise, in multiples
of 1/64) padded with npad = 1 gives a 64 x 150 conjugate spectrum: tau in steps of
0.25 us, fd in steps of 2/3 mHz (+-50 mHz).  Each case is an axis variant and a theta grid:

  axes   asc (control), desc_tau (descending frequencies), desc_fd (descending times),
         both; offset (the zero of each axis moved by a fraction of a bin) and jitter
         (diffs not exactly uniform, so the mean diff differs from the first) are given
         as tau / fd directly and so reach only the entry points that take CS, tau, fd
  grids  sym (31 centres, step 2: eta = 1/32 puts eta th^2 on delay-bin edges), asym,
         nozero (edges that do not cross zero), sinh (symmetric, non-uniform), even (30
         centres: the recentring of theta_centres ties), wide_neg / wide_pos (reaching
         past the fd axis on one side), wide_sym (+-1.7 max|fd|), short (span 150 mHz:
         one bin short of the IndexError threshold), past (span 150.5 mHz: one beyond)

Per case and curvature (ETAS) the fixture records, with the exception's type name where
the reference raises (key ``<case>/<what>_err``):
  ix       thth_map(hermetian=False) of a spectrum whose element (r, c) is
           r nfd + c + 1 + 1j: the flat index each point gathers (0: outside pnts),
           i.e. tau_inv, fd_inv (mod nfd) and pnts, at ETAS[1]
  red, edges_red   thth_redmap at ETAS[1]
  eigs     Eval_calc at every curvature, NaN where it raises (the eta loop)
  thin, sv two_curve_map and singularvalue_calc at ETAS[1] against the sym grid's
           first 16 edges
  chisq    chisq_calc at ETAS[1] (N = 1)
  w, recov modeler at ETAS[1]
  rev      rev_map of thth_map at ETAS[1]
and, for the axes made from frequencies and times: single_search's eigenvalues,
single_chunk_retrieval's wavefield, calc_asymmetry and VLBI_chunk_retrieval (two
stations) at ETAS[1].

The reference calls eigsh without a start vector in modeler and VLBI_chunk_retrieval, and
ARPACK then draws a random one, so the eigenvector's phase (and the last bits of the
eigenvalue) change from run to run.  To make the file reproducible the generator hands
those calls a fixed start vector (ones); everything else runs unmodified.
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

NF, NT, NPAD = 32, 75, 1
DT, DF, F0 = 10.0, 0.0625, 1400.0
ETA_ARC = 1.0 / 32
ETAS = np.array([1.0 / 4096, 1.0 / 32, 1.0 / 8])


def grids():
    s = 150.5 / 30
    return {
        "sym": np.linspace(-31, 31, 32),
        "asym": np.linspace(-15, 47, 32),
        "nozero": np.linspace(3, 65, 32),
        "sinh": 24 * np.sinh(np.linspace(-2.5, 2.5, 42)) / np.sinh(2.5),
        "even": np.linspace(-15, 15, 31),
        "wide_neg": np.linspace(-161, 11, 44),
        "wide_pos": np.linspace(-11, 161, 44),
        "wide_sym": np.linspace(-87.5, 87.5, 36),
        "short": np.linspace(-77.5, 77.5, 32),
        "past": np.linspace(-15.5 * s, 15.5 * s, 32),
    }


def axes(name, nf=NF, nt=NT, npad=NPAD):
    """-> (freq, time) or None, tau, fd of axis variant ``name`` for nf x nt padded by npad."""
    f = F0 + DF * np.arange(nf)
    t = DT * np.arange(nt)
    if name in ("asc", "desc_tau", "desc_fd", "both"):
        if name in ("desc_tau", "both"):
            f = f[::-1].copy()
        if name in ("desc_fd", "both"):
            t = t[::-1].copy()
        return (f, t), fft(f, "us", npad), fft(t, "mHz", npad)
    tau, fd = fft(f, "us", npad), fft(t, "mHz", npad)
    if name == "offset":
        return None, tau + 0.3 * (tau[1] - tau[0]), fd - 0.4 * (fd[1] - fd[0])
    assert name == "jitter"
    k = np.arange(fd.shape[0])
    return (None, tau + 0.01 * (tau[1] - tau[0]) * np.cos(np.arange(tau.shape[0])),
            fd + 0.01 * (fd[1] - fd[0]) * np.sin(k))


def fft(x, unit, npad):
    f = np.fft.fftfreq((npad + 1) * x.shape[0], x[1] - x[0])
    return np.fft.fftshift(f * 1e3 if unit == "mHz" else f)


CASES = ([(a, g) for g in grids() for a in ("asc", "desc_fd")] +
         [(a, g) for g in ("sym", "asym", "wide_sym") for a in ("desc_tau", "both")] +
         [(a, g) for g in ("sym", "sinh", "wide_neg") for a in ("offset", "jitter")])


def case_name(a, g):
    return "%s-%s" % (a, g)


def screen(seed=32, n_dish=1):
    """Wavefields of n_dish stations: 24 images on the arc tau = ETA_ARC fd^2."""
    rng = np.random.default_rng(seed)
    f = F0 + DF * np.arange(NF)
    t = DT * np.arange(NT)
    fdk = rng.uniform(-20.0, 20.0, 24)
    ak = (rng.normal(size=24) + 1j * rng.normal(size=24)) * np.exp(-(fdk / 12.0) ** 2)
    U = np.exp(2j * np.pi * 1e-3 * fdk[:, None] * t[None, :])
    out = []
    for d in range(n_dish):
        ph = np.exp(2j * np.pi * rng.uniform(size=24) * 0.2 * d)
        V = np.exp(-2j * np.pi * ETA_ARC * fdk[None, :] ** 2 * (f[:, None] - F0)) * (ak * ph)[None, :]
        out.append(V @ U)
    return out, rng


def q64(a):
    return np.round(np.asarray(a) * 64) / 64


def inputs():
    (E,), rng = screen()
    dyn = np.abs(E) ** 2
    dyn = q64(dyn + rng.normal(0.0, 0.2 * dyn.mean(), dyn.shape))
    (E1, E2), rng = screen(seed=33, n_dish=2)
    vis = [q64(np.abs(E1) ** 2), q64(E1 * np.conj(E2)), q64(np.abs(E2) ** 2)]
    return dyn, vis


def run(out, key, fn):
    """out[key] = fn(), or out[key + '_err'] = the exception's type name."""
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out[key] = fn()
    except Exception as e:  # noqa: BLE001  (recording what the reference raises)
        out[key + "_err"] = np.array(type(e).__name__)


def _eigsh_fixed_start(eigsh):
    def call(A, k=6, **kw):
        if kw.get("v0") is None:
            kw["v0"] = np.ones(A.shape[0], dtype=A.dtype)
        return eigsh(A, k, **kw)
    return call


def golden_axes(pkg):
    u = sys.modules["astropy.units"]
    T = pkg.ththmod
    T.eigsh = _eigsh_fixed_start(T.eigsh)
    dyn, vis = inputs()
    pad = np.pad(dyn, ((0, NPAD * NF), (0, NPAD * NT)), constant_values=dyn.mean())
    CS = np.fft.fftshift(np.fft.fft2(pad))
    ntau, nfd = CS.shape
    code = (np.arange(ntau)[:, None] * nfd + np.arange(nfd)[None, :] + 1) + 1j
    out = dict(dyn=dyn, vis=np.array(vis), etas=ETAS, npad=NPAD)
    eta = ETAS[1] * u.s ** 3
    e2 = grids()["sym"][:16] * u.mHz
    for a, g in CASES:
        c = case_name(a, g)
        ft, tau, fd = axes(a)
        edges = grids()[g]
        out[c + "/tau"], out[c + "/fd"], out[c + "/edges"] = tau, fd, edges
        tq, fq, eq = tau * u.us, fd * u.mHz, edges * u.mHz
        run(out, c + "/ix", lambda: T.thth_map(code, tq, fq, eta, eq, hermetian=False))
        if c + "/ix" in out:             # 0 where the weight is zero: outside pnts, or the diagonal
            m = out[c + "/ix"]
            hit = m.imag != 0
            out[c + "/ix"] = np.where(hit, np.rint(m.real / np.where(hit, m.imag, 1.0)), 0).astype(np.int32)

        def redmap():
            r, er = T.thth_redmap(CS, tq, fq, eta, eq)
            out[c + "/edges_red"] = np.asarray(er.value)
            return r
        run(out, c + "/red", redmap)
        eigs, errs = np.full(ETAS.shape[0], np.nan), []
        for k, e in enumerate(ETAS):
            try:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    eigs[k] = T.Eval_calc(CS, tq, fq, e * u.s ** 3, eq)
                errs.append("")
            except Exception as ex:  # noqa: BLE001  (the eta loop stores NaN)
                errs.append(type(ex).__name__)
        out[c + "/eigs"], out[c + "/eigs_errs"] = eigs, np.array(errs)

        def thin():
            r, _, _ = T.two_curve_map(CS, tq, fq, eta, eq, eta, e2)
            return np.asarray(r)
        run(out, c + "/thin", thin)
        run(out, c + "/sv", lambda: np.float64(T.singularvalue_calc(CS, tq, fq, eta, eq, eta, e2,
                                                                     0.0 * u.mHz)))
        run(out, c + "/chisq", lambda: np.float64(T.chisq_calc(dyn, CS, tq, fq, eta, eq, 1.0)))

        def modeler():
            m = T.modeler(CS, tq, fq, eta, eq)
            out[c + "/w"] = np.float64(m[5])
            return np.asarray(m[2]).astype(np.complex64)
        run(out, c + "/recov", modeler)

        def rev():
            m = T.thth_map(CS, tq, fq, eta, eq)
            return np.asarray(T.rev_map(m, tq, fq, eta, eq)).astype(np.complex64)
        run(out, c + "/rev", rev)
        if ft is None:
            continue
        f, t = ft
        fu, tu = f * u.MHz, t * u.s
        run(out, c + "/search", lambda: np.asarray(T.single_search(
            [dyn, fu, tu, ETAS * u.s ** 3, eq, "", False, 0.1, NPAD, True, 0.0 * u.us, False])[4]))
        run(out, c + "/wavefield", lambda: np.asarray(T.single_chunk_retrieval(
            (dyn, eq, tu, fu, eta, 0, 0, NPAD, 0.0 * u.us, False))[0]).astype(np.complex64))
        run(out, c + "/asym", lambda: np.float64(T.calc_asymmetry(
            (dyn, eq, tu, fu, eta, 0, 0, NPAD, False))[0]))
        run(out, c + "/vlbi", lambda: np.array(T.VLBI_chunk_retrieval(
            (vis, eq, tu, fu, eta, 0, 0, NPAD, 2, 0.0 * u.us, False))[0]).astype(np.complex64))
    out["cases"] = np.array([case_name(a, g) for a, g in CASES])
    path = os.path.join(GOLD, "axes_geometry.npz")
    np.savez_compressed(path, **out)
    print("axes_geometry: %d cases, %.0f kB" % (len(CASES), os.path.getsize(path) / 1e3))


if __name__ == "__main__":
    golden_axes(ref_loader.load())
