"""The theta-theta entry points on descending and offset axes and irregular theta grids,
against the unmodified reference (tests/golden/axes_geometry.npz, oracle/make_golden_axes.py)
and the float64 oracle on the same fp32 spectrum the device holds (cs.numpy()).

The index math of the reference does not depend on the sign of the axes: it floor-divides
by the mean diff, wraps a negative fd index like python indexing and raises IndexError
when fd_inv < -nfd.  A BasicDyn keeps descending frequencies, so Dynspec reaches a
descending tau axis, and every ththmod function takes the axes its caller passes.  The
device has sign-specific branches: lower_check_needed (thth.cu) decides on the host
whether the IndexError scan runs, floor_div_fast sends a negative divisor to
floor_div_exact, needed_fd_columns gives up on a descending or offset fd axis (the sweep
then transforms and gathers the whole half plane), and rev_map's histogram bins must
ascend (the reference raises numpy's ValueError; so do the wrappers, before any launch).

The case table (AXIS_CASES) takes the fixture's geometries (a 64 x 150 spectrum, chirp-z
on the device) through four spectrum sources -- numpy full plane, device half plane (a
64 x 128 spectrum with the same axis variant and grid), chirp-z full plane and a complex
visibility (c2c) -- and three solvers: fp16, SB_EIG_FP32=1 and the direct kernel (a grid
of more than 512 centres).  test_case_table_coverage (no GPU) fails if an edit drops an
axis, grid, source or solver regime.

Bars as in test_gpu_cs_layouts.py: index arrays, crop sizes, status words, exception
types and NaN patterns bit-exact; eigenvalues and singular values |rel| <= 1e-5, a case
whose reference gap (w1 - w2) / w1 is below 1e-3 being a bad case; rev_map 1e-5 of its
largest bin; models, wavefields, chi-square and asymmetry within the first-order
eigenvector bound.  The run prints the worst error of each regime as a fraction of its
bar."""
import math
import os
import sys
from collections import namedtuple

import numpy as np
import pytest

from oracle import make_golden_axes as MG
from oracle import thth_oracle as TO

RTOL = 1e-5
GAP_MIN = 1e-3
TOL_ACCEPT = 2e-6
E_MODEL = 5e-5
U32 = 2.0 ** -24
ST_INDEX_ERROR = 1

Case = namedtuple("Case", "axes grid src solver")

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "axes_geometry.npz")
Z = np.load(GOLD)
FIXTURE_CASES = [str(c) for c in Z["cases"]]
ETAS = Z["etas"]
ETA = float(ETAS[1])
NPAD = int(Z["npad"])


def _table():
    out = [Case(*c.split("-"), "chirp", "fp16") for c in FIXTURE_CASES]
    for c in FIXTURE_CASES:
        a, g = c.split("-")
        if g in ("sym", "wide_neg", "wide_sym", "short", "past"):
            out.append(Case(a, g, "numpy", "fp16"))
            out.append(Case(a, g, "half", "fp16"))
    for a in ("asc", "desc_fd", "both", "offset"):
        out.append(Case(a, "sym", "c2c", "fp16"))
        out.append(Case(a, "sym", "numpy", "fp32"))
    for a in ("asc", "desc_fd", "desc_tau", "jitter"):
        out.append(Case(a, "dense", "chirp", "direct"))
    return out


AXIS_CASES = _table()


def case_id(c):
    return "%s-%s-%s-%s" % c


def has_fixture(c):
    return "%s-%s" % (c.axes, c.grid) in FIXTURE_CASES and c.src in ("numpy", "chirp")


def grid(name):
    if name == "dense":       # 545 centres over +-24 mHz: ld 576 > 512, the direct kernel
        return np.linspace(-24, 24, 546)
    return MG.grids()[name]


def geometry(c):
    """-> (freq, time) or None, tau, fd, edges, (nf, nt) of the dynamic spectrum."""
    nf, nt = (MG.NF, 64) if c.src == "half" else (MG.NF, MG.NT)
    ft, tau, fd = MG.axes(c.axes, nf, nt, NPAD)
    return ft, tau, fd, grid(c.grid), (nf, nt)


def fd_inv_extremes(th, fd):
    """The smallest fd_inv over all pairs, from the two ends of th1 - th2."""
    dfd = np.diff(fd).mean()
    span = th.max() - th.min()
    return min(math.floor(((-span) - fd[0] + dfd / 2) / dfd),
               math.floor((span - fd[0] + dfd / 2) / dfd))


def lower_check_needed(th, fd):
    """thth.cu lower_check_needed: can any pair reach fd_inv < -nfd?"""
    return not fd_inv_extremes(th, fd) - 2.0 >= -fd.shape[0]


def lower_check_needed_ascending_only(th, fd):
    """The rule before it looked at both ends (min(th) - max(th) only)."""
    dfd = np.diff(fd).mean()
    worst = math.floor(((th.min() - th.max()) - fd[0] + dfd / 2) / dfd) - 2.0
    return not worst >= -fd.shape[0]


def theta(edges):
    try:
        return TO.theta_centres(edges)
    except ValueError:
        return None


def regimes(c):
    _, tau, fd, edges, _ = geometry(c)
    th = theta(edges)
    return dict(axes=c.axes, grid=c.grid, src=c.src, solver=c.solver,
                fd_sign="desc" if np.diff(fd).mean() < 0 else "asc",
                tau_sign="desc" if np.diff(tau).mean() < 0 else "asc",
                index_error=th is not None and fd_inv_extremes(th, fd) < -fd.shape[0],
                gate_old_misses=(th is not None and lower_check_needed(th, fd) and
                                 not lower_check_needed_ascending_only(th, fd)))


# --------------------------------------------------------------------------
# tests without a GPU
# --------------------------------------------------------------------------
def missing_coverage():
    miss = []
    rs = [regimes(c) for c in AXIS_CASES]
    for key, want in (("axes", ("asc", "desc_tau", "desc_fd", "both", "offset", "jitter")),
                      ("grid", ("sym", "asym", "nozero", "sinh", "even", "wide_neg",
                                "wide_pos", "wide_sym", "short", "past", "dense")),
                      ("src", ("numpy", "half", "chirp", "c2c")),
                      ("solver", ("fp16", "fp32", "direct"))):
        for w in want:
            if not any(r[key] == w for r in rs):
                miss.append("%s %s" % (key, w))
    for s in ("asc", "desc"):
        for src in ("numpy", "half", "chirp", "c2c"):
            if not any(r["fd_sign"] == s and r["src"] == src for r in rs):
                miss.append("%s fd on %s" % (s, src))
        if not any(r["tau_sign"] == s and r["solver"] == "direct" for r in rs):
            miss.append("%s tau on the direct kernel" % s)
    for g in ("wide_neg", "wide_pos", "short", "past"):
        for s in ("asc", "desc"):
            if not any(r["grid"] == g and r["fd_sign"] == s for r in rs):
                miss.append("grid %s on %s fd" % (g, s))
    if not any(r["gate_old_misses"] for r in rs):
        miss.append("a geometry the ascending-only gate misses")
    if not any(r["src"] == "half" and r["index_error"] and r["fd_sign"] == "desc" for r in rs):
        miss.append("IndexError on the half plane with descending fd")
    return miss


def test_case_table_coverage():
    """Every axis variant, grid, spectrum source and solver is reached, both fd signs on
    every source, both edges of the IndexError threshold on both fd signs, and a geometry
    that the ascending-only gate let through."""
    assert missing_coverage() == []
    ids = [case_id(c) for c in AXIS_CASES]
    assert len(set(ids)) == len(ids)
    assert {"%s-%s" % (c.axes, c.grid) for c in AXIS_CASES} >= set(FIXTURE_CASES)


def test_threshold_grids():
    """short is one bin short of the IndexError threshold and past one bin beyond it, on
    both fd signs; the ascending-only gate skips the scan for desc_fd-wide_neg although
    the reference raises IndexError there."""
    for a in ("asc", "desc_fd"):
        _, _, fd = MG.axes(a)
        nfd = fd.shape[0]
        assert fd_inv_extremes(TO.theta_centres(grid("short")), fd) == -nfd
        assert fd_inv_extremes(TO.theta_centres(grid("past")), fd) == -nfd - 1
    _, _, fd = MG.axes("desc_fd")
    th = TO.theta_centres(grid("wide_neg"))
    assert lower_check_needed(th, fd) and not lower_check_needed_ascending_only(th, fd)
    assert str(Z["desc_fd-wide_neg/eigs_errs"][0]) == "IndexError"


def _exc_name(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        return type(e).__name__
    return None


@pytest.mark.parametrize("name", FIXTURE_CASES)
def test_oracle_against_reference(name):
    """The float64 oracle on the reference's own float64 spectrum: index arrays and
    exception types bit-exact, eigenvalues, maps and rev_map to 1e-9."""
    ft, tau, fd = MG.axes(name.split("-")[0])
    edges = Z[name + "/edges"]
    assert np.array_equal(tau, Z[name + "/tau"]) and np.array_equal(fd, Z[name + "/fd"])
    dyn = Z["dyn"]
    CS = TO.conjugate_spectrum(dyn, NPAD, None)
    ntau, nfd = CS.shape
    if name + "/ix_err" in Z.files:
        assert _exc_name(lambda: TO.thth_map(CS, tau, fd, ETA, edges)) == str(Z[name + "/ix_err"])
    else:
        assert np.array_equal(encoded_indices(*TO.thth_indices(tau, fd, ETA, edges)[1:], nfd),
                              Z[name + "/ix"])
        red, er = TO.thth_redmap(CS, tau, fd, ETA, edges)
        assert np.array_equal(er, Z[name + "/edges_red"])
        assert np.abs(red - Z[name + "/red"]).max() <= 1e-9 * np.abs(red).max()
    for k, e in enumerate(ETAS):
        err = str(Z[name + "/eigs_errs"][k])
        if err:
            assert _exc_name(lambda: TO.Eval_calc(CS, tau, fd, e, edges)) == err
        else:
            w = TO.Eval_calc(CS, tau, fd, e, edges)
            assert abs(w - Z[name + "/eigs"][k]) <= 1e-9 * w
    if name + "/rev_err" in Z.files:
        assert _exc_name(lambda: TO.rev_map(TO.thth_map(CS, tau, fd, ETA, edges), tau, fd, ETA,
                                            edges)) == str(Z[name + "/rev_err"])
    else:
        rv = TO.rev_map(TO.thth_map(CS, tau, fd, ETA, edges), tau, fd, ETA, edges)
        assert np.abs(rv - Z[name + "/rev"]).max() <= 1e-6 * np.abs(rv).max()


def encoded_indices(tau_inv, fd_inv, pnts, nfd):
    """What thth_map(hermetian=False) of the code spectrum r nfd + c + 1 + 1j decodes to:
    the flat gathered index + 1 on pnts off the diagonal, 0 elsewhere."""
    n = tau_inv.shape[0]
    ix = np.where(pnts, tau_inv * nfd + np.where(fd_inv < 0, fd_inv + nfd, fd_inv) + 1, 0)
    ix[np.arange(n), np.arange(n)] = 0
    return ix.astype(np.int32)


# --------------------------------------------------------------------------
# GPU
# --------------------------------------------------------------------------
WORST = {}


def report(regime, frac):
    WORST[regime] = max(WORST.get(regime, 0.0), float(frac))
    assert frac <= 1.0, (regime, frac)


@pytest.fixture(scope="module")
def sb():
    import scintools_b200
    from scintools_b200 import _device
    _device.device()
    yield scintools_b200
    if WORST:
        print("\naxis geometry: worst error per regime, as a fraction of its bar")
        for k in sorted(WORST):
            print("  %-44s %.3g" % (k, WORST[k]))
    sys.stdout.flush()


def make_cs(sb, c, nf, nt):
    """-> (what the entry points get, the float64 copy of the spectrum the device holds,
    the dynamic spectrum)"""
    th = sb.ththmod
    if c.src == "c2c":
        vis = Z["vis"][1]
        cs = th.conjugate_spectrum(vis, NPAD, None)
        return cs, cs.numpy(), vis
    dyn = Z["dyn"] if nt == MG.NT else Z["dyn"][:, :nt]
    if c.src == "numpy":
        CS = TO.conjugate_spectrum(dyn, NPAD, None).astype(np.complex64).astype(np.complex128)
        return CS, CS, dyn
    cs = th.conjugate_spectrum(dyn, NPAD, None)
    assert cs.half == (c.src == "half")
    return cs, cs.numpy(), dyn


def ref_eig(CS, tau, fd, eta, edges):
    red, edges_red = TO.thth_redmap(CS, tau, fd, eta, edges)
    w, V = np.linalg.eigh(red)
    k = np.argsort(w)[::-1]
    w1, w2 = w[k[0]], w[k[1]]
    assert (w1 - w2) / w1 > GAP_MIN, ("bad case: reference gap", eta, (w1 - w2) / w1)
    return dict(n=red.shape[0], w1=w1, w2=w2, V=V[:, k[0]], fro=np.linalg.norm(red),
                edges_red=edges_red)


def dV_bound(r):
    return np.sqrt(2) * ((2 + np.sqrt(r["n"])) * U32 * r["fro"] + TOL_ACCEPT * abs(r["w1"])) / \
        (r["w1"] - r["w2"])


def oracle_outcome(fn):
    """(value, None) or (None, exception type name)"""
    try:
        return fn(), None
    except Exception as e:  # noqa: BLE001
        return None, type(e).__name__


def raises_before_launch(sb, fn):
    """The exception fn raises, asserting that no kernel was launched first."""
    lib = sb._lib.lib
    n0 = lib.sb_launch_count()
    name = _exc_name(fn)
    assert lib.sb_launch_count() == n0, "launched before raising"
    return name


@pytest.mark.gpu
@pytest.mark.parametrize("case", AXIS_CASES, ids=case_id)
def test_maps_and_sweep(sb, case, monkeypatch):
    """thth_map (indices bit-exact), th_points, thth_redmap, eta_sweep (status and NaN
    pattern bit-exact), Eval_calc and thin_sweep / singularvalue_calc."""
    th = sb.ththmod
    ft, tau, fd, edges, (nf, nt) = geometry(case)
    if case.solver == "fp32":
        monkeypatch.setenv("SB_EIG_FP32", "1")
    cs, CS, _ = make_cs(sb, case, nf, nt)
    tag = "%s %s %s" % (case.src, case.solver, regimes(case)["fd_sign"])
    etas = ETAS if case.grid != "dense" else np.array([ETA / 4, ETA / 2])
    if theta(edges) is None:            # an even grid: the recentring ties, as the reference
        for fn in (lambda: th.thth_map(cs, tau, fd, ETA, edges),
                   lambda: th.eta_sweep(cs, tau, fd, etas, edges),
                   lambda: th.Eval_calc(cs, tau, fd, ETA, edges)):
            assert _exc_name(fn) == "ValueError"
        return
    # thth_map: indices against the oracle, and the reference's own gathers
    _, ti_r, fi_r, pn_r = TO.thth_indices(tau, fd, ETA, edges)
    ref_map, err = oracle_outcome(lambda: TO.thth_map(CS, tau, fd, ETA, edges))
    if err:
        assert _exc_name(lambda: th.thth_map(cs, tau, fd, ETA, edges, return_indices=True)) == err
    else:
        m, ti, fi, pn = th.thth_map(cs, tau, fd, ETA, edges, return_indices=True)
        assert np.array_equal(ti, ti_r.astype(np.int32))
        assert np.array_equal(fi, fi_r.astype(np.int32))
        assert np.array_equal(pn, pn_r)
        assert np.array_equal(m == 0, ref_map == 0)
        report("thth_map entries (1e-6) " + tag, np.abs(m - ref_map).max() / np.abs(ref_map).max() / 1e-6)
        if has_fixture(case):
            name = "%s-%s" % (case.axes, case.grid)
            assert np.array_equal(encoded_indices(ti, fi, pn, fd.shape[0]), Z[name + "/ix"])
        red, er = th.thth_redmap(cs, tau, fd, ETA, edges)
        rred, rer = TO.thth_redmap(CS, tau, fd, ETA, edges)
        assert red.shape == rred.shape and np.array_equal(er, rer)
        report("thth_redmap entries (1e-6) " + tag, np.abs(red - rred).max() / np.abs(rred).max() / 1e-6)
    for e in etas:
        assert np.array_equal(th.th_points(tau, fd, e, edges), TO.th_points(tau, fd, e, edges))
    # the sweep: the oracle's exception pattern, status bits and values
    got, info = th.eta_sweep(cs, tau, fd, etas, edges, return_info=True)
    outcomes = [oracle_outcome(lambda e=e: TO.Eval_calc(CS, tau, fd, e, edges)) for e in etas]
    assert list(np.isnan(got)) == [o[1] is not None for o in outcomes], (got, outcomes)
    for k, (e, (w_ref, err)) in enumerate(zip(etas, outcomes)):
        if err == "IndexError":
            assert info["status"][k] & ST_INDEX_ERROR
            assert _exc_name(lambda: th.Eval_calc(cs, tau, fd, e, edges)) == "IndexError"
            continue
        assert err is None and info["status"][k] == 0, (err, info["status"][k])
        assert info["nred"][k] == TO.th_points(tau, fd, e, edges).sum()
        r = ref_eig(CS, tau, fd, e, edges)
        report("sweep " + tag, abs(got[k] - r["w1"]) / r["w1"] / RTOL)
        if has_fixture(case):
            wz = Z["%s-%s/eigs" % (case.axes, case.grid)][k]
            report("sweep vs reference " + tag, abs(got[k] - wz) / wz / RTOL)
    if case.src == "c2c" or case.solver != "fp16":
        return
    # thin: n x 15 centres of the sym grid's first 16 edges
    e2 = MG.grids()["sym"][:16]
    sv, tinfo = th.thin_sweep(cs, tau, fd, np.array([ETA]), edges, e2, 0.0, return_info=True)
    red2, _, _ = TO.two_curve_map(CS, tau, fd, ETA, edges, ETA, e2)
    assert (tinfo["n1"][0], tinfo["n2"][0]) == red2.shape[::-1]
    s = np.linalg.svd(red2, compute_uv=False)[:2]
    if (s[0] ** 2 - s[1] ** 2) / s[0] ** 2 > GAP_MIN:
        report("thin " + tag, abs(sv[0] - s[0]) / s[0] / RTOL)
        assert th.singularvalue_calc(cs, tau, fd, ETA, edges, ETA, e2, 0.0) == sv[0]
    if has_fixture(case):
        name = "%s-%s" % (case.axes, case.grid)
        assert np.allclose(red2, Z[name + "/thin"], rtol=0, atol=1e-6 * np.abs(red2).max())


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURE_CASES)
def test_retrieval_entry_points(sb, name):
    """rev_map, modeler, chisq_calc / chisq_sweep, VLBI_chunk_retrieval and, for axes made
    from frequencies and times, single_search, search_batch, single_chunk_retrieval and
    calc_asymmetry / asymmetry_batch: the reference's exception types (raised before any
    launch where the wrapper can tell), NaN and zero patterns, and values."""
    th = sb.ththmod
    a, g = name.split("-")
    ft, tau, fd = MG.axes(a)
    edges = Z[name + "/edges"]
    dyn = Z["dyn"]
    cs = th.conjugate_spectrum(dyn, NPAD, None)
    CS = cs.numpy()
    desc = np.diff(tau).mean() < 0 or np.diff(fd).mean() < 0
    tag = "desc" if desc else "asc"
    # rev_map of the oracle's map (a plain array: no device work before the axis check)
    if name + "/rev_err" in Z.files:
        err = str(Z[name + "/rev_err"])
        if err == "ValueError" and theta(edges) is not None:
            m = TO.thth_map(CS, tau, fd, ETA, edges)
            assert raises_before_launch(sb, lambda: th.rev_map(m, tau, fd, ETA, edges)) == err
            assert raises_before_launch(
                sb, lambda: th.chisq_sweep(dyn, cs, tau, fd, ETAS, edges, 1.0)) == "ValueError"
        assert _exc_name(lambda: th.modeler(cs, tau, fd, ETA, edges)) == str(Z[name + "/recov_err"])
    else:
        m = TO.thth_map(CS, tau, fd, ETA, edges)
        got, ref = th.rev_map(m, tau, fd, ETA, edges), TO.rev_map(m, tau, fd, ETA, edges)
        assert np.array_equal(got == 0, ref == 0)
        report("rev_map (1e-5) " + tag, np.abs(got - ref).max() / np.abs(ref).max() / RTOL)
        r = ref_eig(CS, tau, fd, ETA, edges)
        _, _, recov, _, edges_red, w, _ = th.modeler(cs, tau, fd, ETA, edges)
        assert np.array_equal(edges_red, r["edges_red"])
        report("modeler w " + tag, abs(w - r["w1"]) / r["w1"] / RTOL)
        report("modeler w vs reference " + tag, abs(w - Z[name + "/w"]) / r["w1"] / RTOL)
        dV = dV_bound(r)
        rrecov = Z[name + "/recov"]
        report("modeler recov vs reference " + tag,
               np.linalg.norm(recov - rrecov) / np.linalg.norm(rrecov) / (2 * dV + RTOL + E_MODEL))
    # chisq_calc: the reference's exception or its value
    if name + "/chisq_err" in Z.files:
        err = str(Z[name + "/chisq_err"])
        got = raises_before_launch(sb, lambda: th.chisq_calc(dyn, cs, tau, fd, ETA, edges, 1.0)) \
            if desc or theta(edges) is None else \
            _exc_name(lambda: th.chisq_calc(dyn, cs, tau, fd, ETA, edges, 1.0))
        assert got == err
    else:
        ref = float(Z[name + "/chisq"])
        r = ref_eig(CS, tau, fd, ETA, edges)
        dm = (2 * dV_bound(r) + RTOL + E_MODEL) * np.sqrt(ref + np.linalg.norm(dyn) ** 2)
        resid = np.sqrt(ref)
        got = th.chisq_calc(dyn, cs, tau, fd, ETA, edges, 1.0)
        report("chisq vs reference " + tag, abs(got - ref) / (2 * resid * dm + dm ** 2))
        sweep = th.chisq_sweep(dyn, cs, tau, fd, np.array([ETA]), edges, 1.0)
        assert abs(sweep[0] - got) <= 1e-6 * got
    if ft is None:
        return
    f, t = ft
    _search_and_chunks(sb, name, f, t, edges, dyn, tag)


def _phase_err(got, ref):
    ph = np.vdot(got.ravel(), ref.ravel())
    ph = ph / abs(ph) if ph != 0 else 1.0
    return np.linalg.norm(got * ph - ref) / np.linalg.norm(ref)


def _search_and_chunks(sb, name, f, t, edges, dyn, tag):
    th = sb.ththmod
    params = [dyn, f, t, ETAS, edges, None, False, 0.1, NPAD, True, 0.0, False]
    if name + "/search_err" in Z.files:
        err = str(Z[name + "/search_err"])
        assert _exc_name(lambda: th.single_search(params)) == err
    else:
        # the reference returns the finite eigenvalues only; this port keeps NaN in place
        ref = Z[name + "/search"]
        failed = [str(x) != "" for x in Z[name + "/eigs_errs"]]
        for res in (th.single_search(params), th.search_batch([params, params])[1]):
            eigs = res[4]
            assert list(np.isnan(eigs)) == failed, (eigs, failed)
            fin = eigs[np.isfinite(eigs)]
            assert fin.shape == ref.shape
            report("single_search vs reference " + tag,
                   (np.abs(fin - ref) / ref).max() / RTOL if ref.size else 0.0)
    CS = th.conjugate_spectrum(dyn, NPAD, None).numpy()
    ft_tau, ft_fd = MG.axes(name.split("-")[0])[1:]
    # single_chunk_retrieval: zeros where the reference's try/except gave zeros
    wf_ref = Z[name + "/wavefield"]
    wf = th.single_chunk_retrieval((dyn, edges, t, f, ETA, 0, 0, NPAD, 0.0, False))[0]
    assert wf.shape == wf_ref.shape
    if not np.any(wf_ref):
        assert not np.any(wf)
    else:
        r = ref_eig(CS, ft_tau, ft_fd, ETA, edges)
        report("single_chunk_retrieval vs reference " + tag,
               _phase_err(wf, wf_ref) / (2 * dV_bound(r) + E_MODEL + 1e-6))
    # calc_asymmetry / asymmetry_batch: NaN where the reference gives NaN
    a_ref = float(Z[name + "/asym"])
    p = (dyn, edges, t, f, ETA, 0, 0, NPAD, False)
    a = th.calc_asymmetry(p)[0]
    assert th.asymmetry_batch([p, p])[1][0] == a or (np.isnan(a) and np.isnan(a_ref))
    assert np.isnan(a) == np.isnan(a_ref), (a, a_ref)
    if np.isfinite(a_ref):
        r = ref_eig(CS, ft_tau, ft_fd, ETA, edges)
        report("calc_asymmetry vs reference " + tag, abs(a - a_ref) / (4 * dV_bound(r) + 1e-6))
    # VLBI_chunk_retrieval (two stations): the reference's exception, or its wavefields
    vis = list(Z["vis"])
    vp = (vis, edges, t, f, ETA, 0, 0, NPAD, 2, 0.0, False)
    if name + "/vlbi_err" in Z.files:
        # the axis check runs before any launch; an IndexError on ascending axes comes
        # from the device
        check = raises_before_launch if tag == "desc" else (lambda _, fn: _exc_name(fn))
        assert check(sb, lambda: th.VLBI_chunk_retrieval(vp)) == str(Z[name + "/vlbi_err"])
    else:
        got = np.array(th.VLBI_chunk_retrieval(vp)[0])
        ref = Z[name + "/vlbi"]
        assert got.shape == ref.shape
        report("VLBI vs reference (1e-3) " + tag, _phase_err(got, ref) / 1e-3)


@pytest.mark.gpu
def test_dynspec_descending_frequencies(sb):
    """A Dynspec of a BasicDyn with descending frequencies: its delay axis descends.
    thetatheta_single and fit_thetatheta run the sweep on it (and agree with the same
    call's eta_sweep), while calc_wavefield and calc_asymmetry give what the reference's
    rev_map failure gives in every chunk: zero wavefields and NaN asymmetries."""
    from scintools_b200.dynspec import BasicDyn, Dynspec
    (f, t), _, _ = MG.axes("desc_tau")
    dyn = np.tile(Z["dyn"], (2, 2))
    f2 = MG.F0 + MG.DF * np.arange(2 * MG.NF)[::-1]
    t2 = MG.DT * np.arange(2 * MG.NT)
    ds = Dynspec(dyn=BasicDyn(dyn, times=t2, freqs=f2, dt=MG.DT, df=MG.DF), verbose=False)
    assert ds.freqs[0] > ds.freqs[-1]
    ds.prep_thetatheta(cwf=MG.NF, cwt=MG.NT, eta_min=ETA / 2, eta_max=ETA * 2, nedge=32,
                       edges_lim=12, npad=NPAD, verbose=False)
    etas, eigs, _ = ds.thetatheta_single(cf=0, ct=0, verbose=False)[:3]
    assert np.isfinite(eigs).any()
    ds.fit_thetatheta(verbose=False)
    ds.calc_wavefield(verbose=False)
    assert not np.any(ds.wavefield)
    ds.calc_asymmetry(verbose=False)
    assert np.isnan(ds.asymmetry).all()
