"""Chi-square curvature search (ththmod.chisq_calc / chisq_sweep, sb_chisq_sweep)
against the reference's own values (tests/golden/chisq_sample_64x150.npz, made by
oracle/make_golden_chisq.py from the unmodified reference) and the numpy oracle.

Per-curvature error bound: the model is the rank-1 projection onto the top
eigenvector, so to first order |d chisq| / chisq <= 2 rho (e_model + e_vec / relgap)
with rho = ||model|| / ||model - dspec|| over the mask and relgap = (w1 - w2) / |w1|
of the reference's theta-theta matrix.  e_model = 5e-5 is the model bar of
test_modeler (fp32 gather, scatter and transform), e_vec = 4e-6 twice the residual
the eigenpair kernel accepts (2e-6 |w|)."""
import os

import numpy as np
import pytest
from scipy.optimize import curve_fit

from oracle import chisq_oracle as CO
from oracle import thth_oracle as TO

pytestmark = pytest.mark.gpu

E_MODEL, E_VEC = 5e-5, 4e-6


@pytest.fixture(scope="module")
def sb():
    import scintools_b200
    return scintools_b200


@pytest.fixture(scope="module")
def fx(golden_dir):
    return (np.load(os.path.join(golden_dir, "chisq_sample_64x150.npz")),
            np.load(os.path.join(golden_dir, "thth_sample_64x150.npz")))


def case_a(fx):
    c, g = fx
    d2 = g["dspec2"]
    CS = TO.conjugate_spectrum(d2 - d2.mean(), int(c["npad"]), 0.0)
    return d2, CS, g["tau"], g["fd"], np.ones(d2.shape, bool)


def case_b(fx):
    c, g = fx
    db = g["dspec2"][:, :128]
    CS = TO.conjugate_spectrum(db, int(c["npad"]), None)        # padded with the mean
    return c["b_dspec"], CS, c["b_tau"], c["b_fd"], c["b_mask"]


def bound(c, tag):
    rho = c[tag + "_model_norm"] / c[tag + "_resid_norm"]
    relgap = (c[tag + "_w1"] - c[tag + "_w2"]) / np.abs(c[tag + "_w1"])
    return 2 * rho * (E_MODEL + E_VEC / relgap)


def notebook_fit(etas, chisq, fw=0.1):
    """The parabola fit of THTHSample.ipynb cell 40 around the chi-square minimum."""
    e_min = etas[chisq == chisq.min()][0]
    win = np.abs(etas - e_min) < fw * e_min
    ef, cf = etas[win], chisq[win]
    C = cf.min()
    x0 = ef[cf == C][0]
    A0 = (cf[0] - C) / ((ef[0] - x0) ** 2)
    popt, _ = curve_fit(TO.chi_par, ef, cf, p0=np.array([A0, x0, C]))
    return popt[1], np.sqrt((cf - TO.chi_par(ef, *popt)).std() / popt[0])


@pytest.mark.parametrize("tag", ["a", "b"])
def test_chisq_sweep_matches_reference(sb, fx, tag):
    """Every curvature within its first-order bound; same minimum; same fitted curvature."""
    c, _ = fx
    dspec, CS, tau, fd, mask = (case_a if tag == "a" else case_b)(fx)
    etas, edges, N = c["etas"], c["edges"], float(c["N"])
    got, info = sb.ththmod.chisq_sweep(dspec, CS, tau, fd, etas, edges, N, mask,
                                       return_info=True)
    ref = c[tag + "_chisq"]
    assert not np.isnan(got).any() and (info["status"] == 0).all()
    assert np.array_equal(info["nred"], c[tag + "_nred"])
    b = bound(c, tag)
    ratio = np.abs(got - ref) / ref / b
    print("case %s: worst error / bound %.3g (error %.3g)" %
          (tag, ratio.max(), (np.abs(got - ref) / ref).max()))
    assert ratio.max() <= 1.0
    kg, kr = int(np.argmin(got)), int(np.argmin(ref))
    assert kg == kr or ref[kg] - ref[kr] <= b[kg] * ref[kg]
    fit_g, _ = notebook_fit(etas, got)
    fit_r, sig_r = notebook_fit(etas, ref)
    assert abs(fit_g - fit_r) <= 1e-2 * sig_r


def test_chisq_paths_agree(sb, fx):
    """chisq_calc = chisq_sweep[k] = the sum over modeler()[3]; |w| = eta_sweep; nred =
    th_points; an array N broadcasts."""
    c, _ = fx
    th = sb.ththmod
    dspec, CS, tau, fd, mask = case_a(fx)
    etas, edges, N = c["etas"], c["edges"], float(c["N"])
    sweep, info = th.chisq_sweep(dspec, CS, tau, fd, etas, edges, N, mask, return_info=True)
    eig = th.eta_sweep(CS, tau, fd, etas, edges)
    assert (np.abs(np.abs(info["w"]) - eig) / eig).max() < 1e-5
    b = bound(c, "a")
    for k in (5, 40, 77):
        one = th.chisq_calc(dspec, CS, tau, fd, etas[k], edges, N, mask)
        assert abs(one - sweep[k]) <= 1e-6 * sweep[k]
        model = th.modeler(CS, tau, fd, etas[k], edges)[3][:dspec.shape[0], :dspec.shape[1]]
        host = np.sum((model - dspec)[mask] ** 2) / N
        assert abs(host - sweep[k]) <= b[k] * host
        assert info["nred"][k] == int(th.th_points(tau, fd, etas[k], edges).sum())
    Ns = np.array([N, 2 * N])
    both = th.chisq_calc(dspec, CS, tau, fd, etas[5], edges, Ns, mask)
    assert both.shape == (2,) and np.allclose(both, [sweep[5], sweep[5] / 2], rtol=1e-6)
    assert th.chisq_sweep(dspec, CS, tau, fd, etas[:3], edges, Ns, mask).shape == (3, 2)


def test_chisq_batching_and_layout(sb, fx, monkeypatch):
    """Several batches (small slab budget) and a half-plane DeviceCS give the results of
    one batch on the full numpy CS (fp32 scatter atomics: not bit-identical)."""
    c, _ = fx
    th = sb.ththmod
    db = fx[1]["dspec2"][:, :128]
    dspec, CS, tau, fd, mask = case_b(fx)
    etas, edges, N = c["etas"][::4], c["edges"], float(c["N"])
    ref = th.chisq_sweep(dspec, CS, tau, fd, etas, edges, N, mask)
    cs_half = th.conjugate_spectrum(db, int(c["npad"]), None)
    assert cs_half.half
    half = th.chisq_sweep(dspec, cs_half, tau, fd, etas, edges, N, mask)
    assert (np.abs(half - ref) / ref).max() < 1e-5
    monkeypatch.setenv("SB_SWEEP_SLAB_MB", "20")       # 2-3 curvatures per batch
    small = th.chisq_sweep(dspec, CS, tau, fd, etas, edges, N, mask)
    assert (np.abs(small - ref) / ref).max() < 1e-6


def test_chisq_failures(sb, fx):
    """Zero spectrum (the reference raises: ARPACK), crops below 3 x 3, grids past the fd
    axis; argument errors leave the library usable."""
    c, _ = fx
    th = sb.ththmod
    dspec, CS, tau, fd, mask = case_b(fx)
    edges, N = c["edges"], float(c["N"])
    db = fx[1]["dspec2"][:, :128]
    # (c): all-zero CS
    assert all(c["c_error"])
    z, info = th.chisq_sweep(db, np.zeros_like(CS), tau, fd, c["c_etas"], edges, N,
                             return_info=True)
    assert np.isnan(z).all() and ((info["status"] & 2) != 0).all()
    assert (info["w"] == 0).all()
    with pytest.raises(RuntimeError):
        th.chisq_calc(db, np.zeros_like(CS), tau, fd, c["c_etas"][0], edges, N)
    # a crop of one centre
    thc = TO.theta_centres(edges)
    eta1 = 2 * np.abs(tau.max()) / np.min(np.abs(thc[thc != 0])) ** 2
    assert TO.th_points(tau, fd, eta1, edges).sum() < 3
    got, info = th.chisq_sweep(dspec, CS, tau, fd, np.array([40.0, eta1]), edges, N, mask,
                               return_info=True)
    assert np.isfinite(got[0]) and np.isnan(got[1]) and info["status"][1] & 4
    with pytest.raises(TypeError):
        th.chisq_calc(dspec, CS, tau, fd, eta1, edges, N, mask)
    # edges far wider than the fd axis: IndexError in the reference's thth_map
    wide = np.linspace(-6.0, 6.0, 64)
    etas = np.array([0.5, 20.0])
    got, info = th.chisq_sweep(dspec, CS, tau, fd, etas, wide, N, mask, return_info=True)
    for k, e in enumerate(etas):
        try:
            TO.thth_map(CS, tau, fd, e, wide)
            raised = False
        except IndexError:
            raised = True
        assert bool(info["status"][k] & 1) == raised
        assert np.isnan(got[k]) == raised
    assert (info["status"] & 1).any()
    with pytest.raises(IndexError):
        th.chisq_calc(dspec, CS, tau, fd, etas[np.argmax(info["status"] & 1)], wide, N, mask)
    # argument errors, each followed by a good call
    good = th.chisq_calc(dspec, CS, tau, fd, 40.0, edges, N, mask)
    big = np.ones((CS.shape[0] + 1, 8))
    with pytest.raises(sb._lib.SbError, match="larger than the conjugate spectrum"):
        th.chisq_sweep(big, CS, tau, fd, np.array([40.0]), edges, N)
    assert th.chisq_calc(dspec, CS, tau, fd, 40.0, edges, N, mask) == pytest.approx(good, rel=1e-6)
    with pytest.raises(IndexError):
        th.chisq_sweep(dspec, CS, tau, fd, np.array([40.0]), edges, N, mask[:, :-1])
    assert th.chisq_calc(dspec, CS, tau, fd, 40.0, edges, N, mask) == pytest.approx(good, rel=1e-6)
    with pytest.raises(sb._lib.SbError, match="4096"):
        th.chisq_sweep(dspec, CS, tau, fd, np.array([40.0]), np.linspace(-0.4, 0.4, 4098), N,
                       mask)
    assert th.chisq_calc(dspec, CS, tau, fd, 40.0, edges, N, mask) == pytest.approx(good, rel=1e-6)


def test_chisq_large_against_oracle(sb):
    """256 x 1024 chunk, npad = 3 (CS 1024 x 4096), 1024 edges, 8 curvatures against the
    numpy oracle's chisq_calc, each within the bound computed from the oracle's matrix."""
    rng = np.random.default_rng(2024)
    nf, nt, npad = 256, 1024, 3
    dt, df = 10.0, 0.05
    t = np.arange(nt) * dt
    f = 1400.0 + np.arange(nf) * df
    fdk = rng.uniform(-20, 20, 60)
    ak = (rng.normal(size=60) + 1j * rng.normal(size=60)) * np.exp(-(fdk / 10) ** 2)
    E = sum(a * np.exp(2j * np.pi * (fd_ * 1e-3 * t[None, :] - 0.01 * fd_ ** 2 * (f[:, None] - f[0])))
            for a, fd_ in zip(ak, fdk))
    dyn = np.abs(E) ** 2 + rng.normal(0, 0.05, (nf, nt))
    fd, tau = TO.fft_axis(t, "mHz", npad), TO.fft_axis(f, "us", npad)
    CS = TO.conjugate_spectrum(dyn - dyn.mean(), npad, 0.0)
    edges = np.linspace(-20.0, 20.0, 1024)
    etas = np.linspace(0.006, 0.014, 8)
    N = 0.05
    got, info = sb.ththmod.chisq_sweep(dyn, CS, tau, fd, etas, edges, N, return_info=True)
    assert (info["status"] == 0).all() and np.isfinite(got).all()
    worst = 0.0
    for k, e in enumerate(etas):
        ref = CO.chisq_calc(dyn, CS, tau, fd, e, edges, N)
        out = TO.modeler(CS, tau, fd, e, edges)
        wv = np.linalg.eigvalsh(out[0])
        model = out[3][:nf, :nt]
        rho = np.sqrt(np.sum(model ** 2) / np.sum((model - dyn) ** 2))
        b = 2 * rho * (E_MODEL + E_VEC / ((wv[-1] - wv[-2]) / abs(wv[-1])))
        worst = max(worst, abs(got[k] - ref) / ref / b)
    print("large case: worst error / bound %.3g" % worst)
    assert worst <= 1.0
