"""The theta-theta entry points over the shape and the device layout of the conjugate
spectrum (CS) they read, against float64 references; and the magnitude bound of a
device-made spectrum against the spectrum it bounds.

A sweep (eta_sweep / Eval_calc / single_search, thth.cu::eta_sweep) with the default
fp16 solver (ld <= 512, no SB_EIG_FP32) scales its fp16 copy by a bound on
max(|re|, |im|) of the CS: the L1 bound of the dynamic spectrum (sb_cs_bound_f32) when
the DeviceCS carries one, else a scan of the spectrum (cs_absmax_kernel).  The scan
reads rows at the spectrum's pitch, so an odd pitch starts every other row 8 bytes off
a 16-byte boundary.  CS_CASES restates how a CS reaches the device:
  numpy   a numpy array: full plane, pitch nfd, no bound (the scan)
  abs     the real incoherent |CS| as a numpy array: the same
  half    conjugate_spectrum on a power-of-two plane: half plane, pitch NT/2 + 16, bound
  keep    the same with ncols_keep (cs_valid_cols odd or even)
  chirp   conjugate_spectrum on other sizes (chirp-z): full plane, pitch NT, bound
  c2c     conjugate_spectrum of a complex visibility: full plane, pitch NT, no bound
and on which solver (fp16, SB_EIG_FP32=1, the direct kernel for ld > 512) and from
which gather source (the spectrum or the compact column copy, thth_gather_source) each
case runs.  test_case_table_coverage (no GPU) fails if an edit drops a regime.

Input: a synthetic arc (48 images on a 1-D screen, eta 0.02 s^3, 20 % noise), the
geometry of test_gpu_theta_grids.py at other sizes: tau_max = 16 us and fd_max = 50 mHz
at every size, so every grid spans +-24 mHz and curvatures below 0.0273 keep all its
centres.  References are the oracle in float64 on the SAME fp32 spectrum the device
holds (cs.numpy()).

Bars as in test_gpu_theta_grids.py: eigenvalues and singular values |rel| <= 1e-5;
cropped sizes, status words and index arrays bit-exact; a case whose reference
relative gap (w1 - w2) / w1 is below 1e-3 is a bad case, not a solver failure.  The
run prints the worst error of each regime as a fraction of its bar, and the ratio of
the bound to the spectrum maximum for each bound case."""
import math
import sys
from collections import namedtuple

import numpy as np
import pytest

from oracle import thth_oracle as TO

DT, DF, F0 = 10.0, 0.03125, 1400.0
ETA_ARC = 0.02
EDGE = 24.0
FULL = (0.016, 0.02, 0.024)

RTOL = 1e-5
GAP_MIN = 1e-3
TOL_ACCEPT = 2e-6
E_MODEL = 5e-5
U32 = 2.0 ** -24
BOUND_SLACK = 1e-5       # fp32 transform rounding above the float64 L1 norm

Case = namedtuple("Case", "src nf nt npad n neta extra")


def _c(src, nf, nt, npad, n, neta=3, **extra):
    return Case(src, nf, nt, npad, n, neta, tuple(sorted(extra.items())))


def cs_shape(c):
    return (c.npad + 1) * c.nf, (c.npad + 1) * c.nt


CS_CASES = [
    # numpy full plane (the scan): odd x odd, even x odd, odd x even, a minimal shape;
    # few curvatures gather from the spectrum, many from the compact copy
    _c("numpy", 127, 301, 0, 33),
    _c("numpy", 127, 301, 0, 129, 8),
    _c("numpy", 128, 301, 0, 65),
    _c("numpy", 128, 301, 0, 129, 8),
    _c("numpy", 127, 300, 0, 33),
    _c("numpy", 127, 300, 0, 129, 8),
    _c("numpy", 9, 13, 0, 15),
    _c("numpy", 127, 301, 0, 33, fp32=1),
    _c("abs", 127, 301, 0, 33),
    _c("abs", 127, 301, 0, 129, 8),
    # device half plane (the bound), whole and column-limited
    _c("half", 32, 128, 1, 65),
    _c("half", 32, 128, 1, 129, 8),
    _c("half", 32, 128, 1, 65, fp32=1),
    _c("keep", 32, 128, 1, 65, keep=0),
    _c("keep", 32, 128, 1, 65, keep=1),
    # chirp-z full plane from odd nt (the bound, odd pitch)
    _c("chirp", 43, 101, 0, 33),
    _c("chirp", 43, 101, 2, 33),
    _c("chirp", 43, 101, 2, 129, 8),
    _c("chirp", 43, 101, 2, 545, 2),
    # a complex visibility (the scan, odd pitch)
    _c("c2c", 127, 301, 0, 33),
    _c("c2c", 43, 101, 2, 129, 8),
]


def case_id(c):
    ntau, nfd = cs_shape(c)
    s = "%s-%dx%d-npad%d-n%d-neta%d" % (c.src, ntau, nfd, c.npad, c.n, c.neta)
    return s + "".join("-%s=%s" % kv for kv in c.extra)


# --------------------------------------------------------------------------
# geometry and dispatch (host only)
# --------------------------------------------------------------------------
def axes(nf, nt, npad):
    t = DT * np.arange(nt)
    f = F0 + DF * np.arange(nf)
    return t, f, TO.fft_axis(f, "us", npad), TO.fft_axis(t, "mHz", npad)


def grid(n):
    """n + 1 edges over -EDGE .. EDGE; an even count is shifted by a tenth of a step
    so that the smallest |centre| is unique (theta_centres needs one)."""
    e = np.linspace(-EDGE, EDGE, n + 1)
    return e + (0.1 * (e[1] - e[0]) if n % 2 == 0 else 0.0)


def etas_of(c):
    return np.linspace(FULL[0], FULL[-1], c.neta) if c.neta > 1 else np.array([ETA_ARC])


def is_half(c):
    NF, NT = cs_shape(c)
    return c.src in ("half", "keep") and not (NF & (NF - 1)) and not (NT & (NT - 1))


def layout(c):
    """(pitch, ncols the scan covers, bounded)"""
    ntau, nfd = cs_shape(c)
    if is_half(c):
        return nfd // 2 + 16, nfd // 2 + 1, True
    return nfd, nfd, c.src in ("chirp", "half", "keep")


def solver(c):
    ld = 32 * math.ceil(c.n / 32)
    if ld > 512:
        return "direct"
    return "fp32" if dict(c.extra).get("fp32") else "fp16"


def scale_source(c):
    """Where the fp16 solver takes its scale from (None: the solver has no fp16 copy)."""
    if solver(c) != "fp16":
        return None
    pitch, _, bounded = layout(c)
    if bounded:
        return "bound"
    return "scan float4" if pitch % 2 == 0 else "scan float2"


def reached_columns(c):
    """Stored spectrum columns that some pair (i, j), j > i, i + j != n - 1, of the
    grid maps to (thth_colmark_kernel with thth_pair_column, thth.cuh)."""
    _, _, tau, fd = axes(c.nf, c.nt, c.npad)
    th = TO.theta_centres(grid(c.n))
    n, nfd = th.shape[0], fd.shape[0]
    i, j = np.triu_indices(n, 1)
    keep = i + j != n - 1
    i, j = i[keep], j[keep]
    dfd = np.diff(fd).mean()
    fq = ((th[j] - th[i]) - fd[0] + dfd / 2) // dfd
    fq = fq[(fq < nfd) & ~(fq < -nfd)].astype(np.int64)
    fi = np.where(fq < 0, fq + nfd, fq)
    if is_half(c):
        h = nfd // 2
        fi = np.where(fi >= h, fi - h, np.where(fi == 0, h, h - fi))
    return np.unique(fi)


def gather_source(c):
    """thth_gather_source (thth.cu): the compact copy when the 32-byte sectors of the
    direct gather are at least twice the bytes of making the copy."""
    ntau, _ = cs_shape(c)
    nslots = reached_columns(c).shape[0]
    pairs = 0.5 * c.n * (c.n - 1)
    direct_bytes = 32.0 * c.neta * pairs
    copy_bytes = 40.0 * nslots * ntau
    return "spectrum" if (nslots == 0 or direct_bytes < 2.0 * copy_bytes) else "copy"


def keep_cols(c):
    """ncols_keep of a keep case: needed_fd_columns, or one more, whichever has the
    parity the case asks for (keep=0: even, 1: odd)."""
    from scintools_b200 import ththmod
    _, _, _, fd = axes(c.nf, c.nt, c.npad)
    need = ththmod.needed_fd_columns(fd, grid(c.n))
    want = dict(c.extra)["keep"]
    return need if need % 2 == want else need + 1


def regimes(c):
    ntau, nfd = cs_shape(c)
    par = "%s x %s" % ("odd" if ntau % 2 else "even", "odd" if nfd % 2 else "even")
    return dict(src=c.src, shape=par, solver=solver(c), scale=scale_source(c),
                gather=gather_source(c), pitch_odd=layout(c)[0] % 2 == 1)


def missing_coverage():
    miss = []
    rs = [regimes(c) for c in CS_CASES]
    for src in ("numpy", "abs", "half", "keep", "chirp", "c2c"):
        if not any(r["src"] == src for r in rs):
            miss.append("source " + src)
    for par in ("odd x odd", "even x odd", "odd x even", "even x even"):
        if not any(r["shape"] == par for r in rs):
            miss.append("shape " + par)
    pow2 = [c for c in CS_CASES if not any(x & (x - 1) for x in cs_shape(c))]
    if not pow2 or len(pow2) == len(CS_CASES):
        miss.append("power-of-two and other sizes")
    if not any(max(cs_shape(c)) < 16 for c in CS_CASES):
        miss.append("minimal shape")
    for s in ("fp16", "fp32", "direct"):
        if not any(r["solver"] == s for r in rs):
            miss.append("solver " + s)
    if not any(r["solver"] == "direct" and cs_shape(c)[1] % 2 for c, r in zip(CS_CASES, rs)):
        miss.append("direct solver at odd nfd")
    for s in ("bound", "scan float4", "scan float2"):
        if not any(r["scale"] == s for r in rs):
            miss.append("scale " + s)
    for src in ("numpy", "c2c", "abs"):          # the scan at an odd pitch
        if not any(r["src"] == src and r["scale"] == "scan float2" for r in rs):
            miss.append("odd-pitch scan " + src)
    if not any(r["src"] == "chirp" and r["scale"] == "bound" and r["pitch_odd"] for r in rs):
        miss.append("bound at odd pitch")
    for g in ("spectrum", "copy"):
        for axis in (0, 1):
            if not any(r["gather"] == g and cs_shape(c)[axis] % 2 for c, r in zip(CS_CASES, rs)):
                miss.append("gather %s at odd %s" % (g, ("ntau", "nfd")[axis]))
    if {dict(c.extra)["keep"] for c in CS_CASES if c.src == "keep"} != {0, 1}:
        miss.append("keep odd and even")
    if {c.npad for c in CS_CASES if c.src == "chirp" and c.nt % 2} < {0, 2}:
        miss.append("chirp odd nt npad 0 and 2")
    return miss


# --------------------------------------------------------------------------
# tests without a GPU
# --------------------------------------------------------------------------
def test_case_table_coverage():
    """Every source, shape parity, solver, scale source and gather source is reached:
    both gather sources at odd ntau and at odd nfd, the scan at an odd pitch for each
    source without a bound, the direct kernel at odd nfd."""
    assert missing_coverage() == []
    ids = [case_id(c) for c in CS_CASES]
    assert len(set(ids)) == len(ids)
    for c in CS_CASES:
        _, _, tau, fd = axes(c.nf, c.nt, c.npad)
        # the grid stays inside the fd axis and the crop
        assert 2 * EDGE < -fd[0] or max(cs_shape(c)) < 16, case_id(c)
        assert all(e * EDGE ** 2 < tau.max() for e in etas_of(c)), case_id(c)
        if c.src in ("half", "keep"):
            assert is_half(c), case_id(c)
        if c.src == "chirp":
            assert not is_half(c) and cs_shape(c)[1] % 2, case_id(c)


def test_gather_source_rule_against_theta_grids():
    """The restated rule picks the spectrum for a three-curvature sweep of 33 centres
    and the copy once the pairs far outnumber the reached columns."""
    c = _c("numpy", 127, 301, 0, 33)
    assert gather_source(c) == "spectrum"
    assert gather_source(c._replace(n=129, neta=8)) == "copy"
    assert 0 < reached_columns(c).shape[0] <= 32


# --------------------------------------------------------------------------
# GPU: inputs and references
# --------------------------------------------------------------------------
WORST = {}
RATIO = {}


def report(regime, frac):
    WORST[regime] = max(WORST.get(regime, 0.0), float(frac))
    assert frac <= 1.0, (regime, frac)


def screen(nf, nt, seed, n_dish=1):
    """Wavefields of n_dish stations seeing one 48-image screen on the arc tau =
    ETA_ARC fd^2 (test_gpu_theta_grids.py at nf x nt)."""
    rng = np.random.default_rng(seed)
    t, f, _, _ = axes(nf, nt, 0)
    k = 48
    fdk = rng.uniform(-22.0, 22.0, k)
    ak = (rng.normal(size=k) + 1j * rng.normal(size=k)) / np.sqrt(2) * np.exp(-(fdk / 12.0) ** 2)
    U = np.exp(2j * np.pi * 1e-3 * fdk[:, None] * t[None, :])
    out = []
    for d in range(n_dish):
        ph = np.exp(2j * np.pi * rng.uniform(size=k) * 0.2 * d)
        V = np.exp(-2j * np.pi * ETA_ARC * fdk[None, :] ** 2 * (f[:, None] - F0)) * (ak * ph)[None, :]
        out.append(V @ U)
    return out, rng


def arc_dynspec(nf, nt, seed=5, noise=0.2):
    (E,), rng = screen(nf, nt, seed)
    dyn = np.abs(E) ** 2
    dyn += rng.normal(0.0, noise * dyn.mean(), dyn.shape)
    return dyn - dyn.mean()


def visibility(nf, nt, seed=9):
    (E1, E2), rng = screen(nf, nt, seed, n_dish=2)
    sig = np.mean(np.abs(E1) ** 2)
    return E1 * np.conj(E2) + 0.05 * sig * (rng.normal(size=E1.shape) + 1j * rng.normal(size=E1.shape))


def f32(a):
    return np.asarray(a).astype(np.complex64).astype(np.complex128)


@pytest.fixture(scope="module")
def sb():
    import scintools_b200
    from scintools_b200 import _device
    _device.device()
    yield scintools_b200
    if WORST:
        print("\ncs layouts: worst error per regime, as a fraction of its bar")
        for k in sorted(WORST):
            print("  %-40s %.3g" % (k, WORST[k]))
    if RATIO:
        print("cs bound: bound / max(|re|, |im|) of the spectrum it bounds "
              "(pad 0, 2.5, -2.5, mean; clamp: 0, mean)")
        for k in sorted(RATIO):
            print("  %-36s %s" % (k, " ".join("%.7g" % r for r in RATIO[k])))
    sys.stdout.flush()


def make_cs(sb, c):
    """-> (what the entry points get, the float64 copy of the spectrum the device holds,
    the dynamic spectrum)"""
    th = sb.ththmod
    if c.src == "c2c":
        vis = visibility(c.nf, c.nt)
        cs = th.conjugate_spectrum(vis, c.npad, None)
        assert cs.bound is None and cs.pitch == cs_shape(c)[1]
        return cs, cs.numpy(), vis
    dyn = arc_dynspec(c.nf, c.nt)
    if c.src in ("numpy", "abs"):
        CS = f32(TO.conjugate_spectrum(dyn, c.npad, None))
        if c.src == "abs":
            CS = np.abs(CS).astype(np.float32).astype(np.float64)
        return CS, CS.astype(np.complex128), dyn
    if c.src == "keep":
        cs = th.conjugate_spectrum(dyn, c.npad, None, ncols_keep=keep_cols(c))
        assert cs.ncols_valid == keep_cols(c) and cs.ncols_valid % 2 == dict(c.extra)["keep"]
        CS = th.conjugate_spectrum(dyn, c.npad, None).numpy()
    else:
        cs = th.conjugate_spectrum(dyn, c.npad, None)
        CS = cs.numpy()
    pitch, _, bounded = layout(c)
    assert cs.pitch == pitch and (cs.bound is not None) == bounded and cs.half == is_half(c)
    return cs, CS, dyn


def ref_eig(CS, tau, fd, eta, edges):
    red, edges_red = TO.thth_redmap(CS, tau, fd, eta, edges)
    w, V = np.linalg.eigh(red)
    k = np.argsort(w)[::-1]
    w1, w2 = w[k[0]], w[k[1]]
    assert (w1 - w2) / w1 > GAP_MIN, ("bad case: reference gap", eta, (w1 - w2) / w1)
    return dict(n=red.shape[0], w1=w1, w2=w2, V=V[:, k[0]], fro=np.linalg.norm(red),
                edges_red=edges_red, red=red)


def dV_bound(n, w1, w2, fro):
    return np.sqrt(2) * ((2 + np.sqrt(n)) * U32 * fro + TOL_ACCEPT * abs(w1)) / (w1 - w2)


@pytest.fixture(scope="module")
def made(sb):
    cache = {}

    def get(c):
        key = (c.src, c.nf, c.nt, c.npad, dict(c.extra).get("keep"))
        if key not in cache:
            cache.clear()
            cache[key] = make_cs(sb, c)
        return cache[key]
    return get


# --------------------------------------------------------------------------
# a. eta_sweep, Eval_calc, thth_map, thth_redmap over the case table
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CS_CASES, ids=case_id)
def test_sweep_and_maps(sb, made, case, monkeypatch):
    th = sb.ththmod
    cs, CS, _ = made(case)
    _, _, tau, fd = axes(case.nf, case.nt, case.npad)
    edges, etas = grid(case.n), etas_of(case)
    r = regimes(case)
    tag = "%s %s %s" % (case.src, r["solver"], r["gather"])
    if r["solver"] == "fp32":
        monkeypatch.setenv("SB_EIG_FP32", "1")
    got, info = th.eta_sweep(cs, tau, fd, etas, edges, return_info=True)
    nred = [int(TO.th_points(tau, fd, e, edges).sum()) for e in etas]
    assert list(info["status"]) == [0] * len(etas), info["status"]
    assert list(info["nred"]) == nred
    refs = [ref_eig(CS, tau, fd, e, edges) for e in etas]
    for g, ref, n in zip(got, refs, nred):
        assert ref["n"] == n
        report("sweep " + tag, abs(g - ref["w1"]) / ref["w1"] / RTOL)
    w = th.Eval_calc(cs, tau, fd, etas[0], edges)
    report("Eval_calc " + case.src, abs(w - refs[0]["w1"]) / refs[0]["w1"] / RTOL)
    # index arrays bit-exact, map entries against the oracle's on the same spectrum
    m, ti, fi, pn = th.thth_map(cs, tau, fd, etas[-1], edges, return_indices=True)
    _, rti, rfi, rpn = TO.thth_indices(tau, fd, etas[-1], edges)
    assert np.array_equal(ti, rti.astype(np.int32))
    assert np.array_equal(fi, rfi.astype(np.int32))
    assert np.array_equal(pn, rpn)
    rm = TO.thth_map(CS, tau, fd, etas[-1], edges)
    assert np.array_equal(m == 0, rm == 0)
    report("thth_map entries (1e-6) " + case.src, np.abs(m - rm).max() / np.abs(rm).max() / 1e-6)
    red, er = th.thth_redmap(cs, tau, fd, etas[0], edges)
    rred, rer = TO.thth_redmap(CS, tau, fd, etas[0], edges)
    assert red.shape == rred.shape and np.array_equal(er, rer)
    assert np.array_equal(red == 0, rred == 0)
    report("thth_redmap entries (1e-6) " + case.src,
           np.abs(red - rred).max() / np.abs(rred).max() / 1e-6)


# --------------------------------------------------------------------------
# b. thin_sweep, modeler, rev_map, chisq_sweep on the coherent spectra
# --------------------------------------------------------------------------
MODEL_CASES = [c for c in CS_CASES if c.src in ("numpy", "half", "chirp", "c2c") and
               c.neta == 3 and not c.extra and c.n < 512]


def test_model_cases_cover_odd_axes():
    shapes = {tuple(x % 2 for x in cs_shape(c)) for c in MODEL_CASES}
    assert {(1, 1), (0, 1), (1, 0), (0, 0)} <= shapes


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODEL_CASES, ids=case_id)
def test_thin_modeler_rev_map_chisq(sb, made, case):
    th = sb.ththmod
    cs, CS, dyn = made(case)
    _, _, tau, fd = axes(case.nf, case.nt, case.npad)
    ntau, nfd = cs_shape(case)
    edges, eta = grid(case.n), ETA_ARC
    # thin_sweep / singularvalue_calc: n x (n // 2 + 1) centres
    e2 = grid(case.n // 2 + 1)
    sv, info = th.thin_sweep(cs, tau, fd, np.array([eta]), edges, e2, 0.0, return_info=True)
    red2, _, _ = TO.two_curve_map(CS, tau, fd, eta, edges, eta, e2)
    s = np.linalg.svd(red2, compute_uv=False)[:2]
    assert (s[0] ** 2 - s[1] ** 2) / s[0] ** 2 > GAP_MIN, ("bad case: reference gap", s)
    assert info["status"][0] == 0 and (info["n1"][0], info["n2"][0]) == red2.shape[::-1]
    report("thin " + case.src, abs(sv[0] - s[0]) / s[0] / RTOL)
    assert th.singularvalue_calc(cs, tau, fd, eta, edges, eta, e2, 0.0) == sv[0]
    # rev_map of the reference's full map: occupied bins bit-exact
    rm = TO.thth_map(CS, tau, fd, eta, edges)
    got = th.rev_map(rm, tau, fd, eta, edges)
    ref = TO.rev_map(rm, tau, fd, eta, edges)
    assert got.shape == (ntau, nfd)
    assert np.array_equal(got == 0, ref == 0)
    report("rev_map (1e-5) " + case.src, np.abs(got - ref).max() / np.abs(ref).max() / RTOL)
    # modeler: w and the occupied bins of its recovered spectrum
    r = ref_eig(CS, tau, fd, eta, edges)
    _, _, recov, model, edges_red, w, V = th.modeler(cs, tau, fd, eta, edges)
    assert np.array_equal(edges_red, r["edges_red"]) and V.shape == (r["n"],)
    report("modeler w " + case.src, abs(w - r["w1"]) / r["w1"] / RTOL)
    rrecov = TO.rev_map(np.outer(r["V"], np.conj(r["V"])) * abs(r["w1"]), tau, fd, eta,
                        r["edges_red"], True)
    assert np.array_equal(recov == 0, rrecov == 0)
    rmodel = np.fft.ifft2(np.fft.ifftshift(rrecov)).real
    dV = dV_bound(r["n"], r["w1"], r["w2"], r["fro"])
    err = np.linalg.norm(model - rmodel) / np.linalg.norm(rmodel)
    report("modeler model " + case.src, err / (2 * dV + RTOL + E_MODEL))
    if case.src == "c2c":
        return
    # chisq_sweep: the model against the dynamic spectrum it came from
    chisq, info = th.chisq_sweep(dyn, cs, tau, fd, np.array([eta]), edges, 1.0, return_info=True)
    assert info["status"][0] == 0 and info["nred"][0] == r["n"]
    report("chisq w " + case.src, abs(info["w"][0] - r["w1"]) / r["w1"] / RTOL)
    mod = rmodel[:case.nf, :case.nt]
    resid = np.linalg.norm(mod - dyn)
    dm = (2 * dV + RTOL + E_MODEL) * np.linalg.norm(rmodel)
    report("chisq value " + case.src, abs(chisq[0] - resid ** 2) / (2 * resid * dm + dm ** 2))


# --------------------------------------------------------------------------
# c. single_search on odd nt, npad 0 and 2
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nf,nt,npad", [(43, 101, 0), (43, 101, 2), (64, 75, 2)])
def test_single_search_odd_nt(sb, nf, nt, npad):
    th = sb.ththmod
    dyn = arc_dynspec(nf, nt, seed=11)
    t, f, tau, fd = axes(nf, nt, npad)
    edges, etas = grid(33), np.linspace(FULL[0], FULL[-1], 5)
    res = th.single_search([dyn, f, t, etas, edges, None, False, 0.1, npad, True, 0.0, False])
    CS = th.conjugate_spectrum(dyn, npad, None).numpy()
    for g, e in zip(res[4], etas):
        r = ref_eig(CS, tau, fd, e, edges)
        report("single_search odd nt", abs(g - r["w1"]) / r["w1"] / RTOL)


# --------------------------------------------------------------------------
# d. one spectrum as the numpy full plane and as its device half plane
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,neta", [(65, 3), (129, 8)])
def test_full_and_half_plane_agree(sb, n, neta):
    """thth_map of the two layouts is bit-identical.  The half plane scanned (its bound
    dropped) reaches the same elements and the same scale as the full plane, so its
    eigenvalues are bit-identical too; with its bound the fp16 copy is scaled by another
    power of two, and the sweep agrees to the bar."""
    from scintools_b200.ththmod import DeviceCS
    th = sb.ththmod
    nf, nt, npad = 32, 128, 1
    dyn = arc_dynspec(nf, nt)
    _, _, tau, fd = axes(nf, nt, npad)
    edges = grid(n)
    etas = np.linspace(FULL[0], FULL[-1], neta)
    half = th.conjugate_spectrum(dyn, npad, None)
    full = half.numpy()
    scanned = DeviceCS(half.t, nfd=half.shape[1], bound=None)
    for eta in (etas[0], etas[-1]):
        a = th.thth_map(full, tau, fd, eta, edges, return_indices=True)
        b = th.thth_map(half, tau, fd, eta, edges, return_indices=True)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
    ga, ia = th.eta_sweep(full, tau, fd, etas, edges, return_info=True)
    gb, ib = th.eta_sweep(half, tau, fd, etas, edges, return_info=True)
    gs, is_ = th.eta_sweep(scanned, tau, fd, etas, edges, return_info=True)
    for info in (ib, is_):
        assert np.array_equal(ia["status"], info["status"]) and (ia["status"] == 0).all()
        assert np.array_equal(ia["nred"], info["nred"])
    assert np.array_equal(ga.view(np.uint64), gs.view(np.uint64))
    report("full vs bounded half plane", (np.abs(gb - ga) / ga).max() / RTOL)
    for g, e in zip(ga, etas):
        r = ref_eig(full, tau, fd, e, edges)
        report("full plane sweep", abs(g - r["w1"]) / r["w1"] / RTOL)


# --------------------------------------------------------------------------
# e. sb_cs_bound_f32 against the spectrum it bounds
# --------------------------------------------------------------------------
# (nf, nt): power-of-two planes at npad 0, 1, 3; chirp-z at npad 2 and at odd sizes
BOUND_SHAPES = [(16, 16), (32, 64), (33, 64), (32, 65), (33, 65), (7, 9)]
BOUND_PADS = [0.0, 2.5, -2.5, None]
BOUND_INPUTS = ["arc", "pixel", "const", "zeros", "big", "clamp", "noise"]


def bound_input(kind, nf, nt):
    rng = np.random.default_rng(nf * 1000 + nt)
    if kind == "arc":
        return arc_dynspec(nf, nt)
    if kind == "pixel":         # |CS| equals the L1 norm at every bin (pad 0)
        d = np.zeros((nf, nt))
        d[nf // 3, nt // 2] = 3.75
        return d
    if kind == "const":
        return np.full((nf, nt), 1.5)
    if kind == "zeros":
        return np.zeros((nf, nt))
    if kind == "big":           # positive, near 1e30: the DC bin is the L1 norm
        a = arc_dynspec(nf, nt)
        return 1e30 * (1.0 + a / (4 * np.abs(a).max()))
    if kind == "clamp":         # L1 norm past the 3e38 clamp, the spectrum itself finite
        d = rng.normal(size=(nf, nt))
        d -= d.mean()
        return d * (1.2e38 / (nf * nt) ** 0.75)
    if kind == "noise":         # white noise: the bound ~sqrt(N) above the maximum
        return rng.normal(size=(nf, nt))
    raise ValueError(kind)


def test_bound_inputs_are_representable():
    """The float64 spectra of the bound inputs stay inside float32 (the clamp case has
    a margin of 2 below 3.4e38), and the clamp input's L1 norm exceeds 3e38 whenever
    nf nt >= 198."""
    for nf, nt in BOUND_SHAPES:
        for npad in range(4):
            for kind in BOUND_INPUTS:
                d = bound_input(kind, nf, nt)
                for pad in BOUND_PADS:
                    if kind == "clamp" and pad not in (0.0, None):
                        continue
                    CS = TO.conjugate_spectrum(d, npad, pad)
                    m = max(np.abs(CS.real).max(), np.abs(CS.imag).max())
                    assert m < 1.7e38, (kind, nf, nt, npad, pad)
            d = bound_input("clamp", nf, nt)
            if nf * nt >= 198:
                assert np.abs(d).sum() > 3e38


def _max_re_im(CS):
    return max(np.abs(CS.real).max(), np.abs(CS.imag).max())


@pytest.mark.gpu
@pytest.mark.parametrize("nf,nt", BOUND_SHAPES)
def test_cs_bound_bounds_the_spectrum(sb, nf, nt):
    """max(|re|, |im|) of the device spectrum <= bound (1 + 1e-5), for every pad mode,
    npad 0-3, both transform paths and the adversarial inputs; the clamp input's bound
    is 3e38 (power-of-two planes only)."""
    th = sb.ththmod
    for npad in range(4):
        NF, NT = (npad + 1) * nf, (npad + 1) * nt
        pow2 = not (NF & (NF - 1)) and not (NT & (NT - 1)) and NT >= 16 and NF >= 4
        for kind in BOUND_INPUTS:
            d = bound_input(kind, nf, nt)
            for pad in BOUND_PADS:
                # clamp: a constant pad makes |c| NF NT the whole story; and on the
                # chirp-z path the transform's float32 intermediates overflow (the device
                # spectrum comes out NaN) before a spectrum this large does
                if kind == "clamp" and (pad not in (0.0, None) or not pow2):
                    continue
                cs = th.conjugate_spectrum(d, npad, pad)
                CS = cs.numpy()
                assert np.isfinite(CS).all(), (kind, npad, pad)
                bound = float(cs.bound.cpu()[0])
                m = _max_re_im(CS)
                key = "%dx%d npad%d %s" % (nf, nt, npad, kind)
                assert m <= bound * (1 + BOUND_SLACK), (key, pad, m, bound)
                if kind == "clamp" and nf * nt >= 198:
                    assert bound == np.float32(3e38), key
                RATIO.setdefault(key, []).append(bound / m if m > 0 else float("inf"))


# (nf, nt, npad, noise): one sweep from the bounded spectrum, one from its re-upload
SWEEP_BOUND = [(32, 64, 1, 0.2), (33, 65, 0, 0.2), (33, 65, 2, 0.2), (32, 65, 1, 0.2),
               (33, 64, 3, 0.2), (128, 512, 1, 30.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("nf,nt,npad,noise", SWEEP_BOUND)
def test_sweep_bound_vs_scan(sb, nf, nt, npad, noise):
    """The sweep scaled by the L1 bound and the sweep of the same spectrum re-uploaded
    (scaled by the scan) agree with each other and with the oracle; none stops at the
    iteration cap.  noise = 30: white noise thirty times the arc, where the bound is
    about sqrt(N) / 4 (60) times the maximum."""
    th = sb.ththmod
    dyn = arc_dynspec(nf, nt, seed=13, noise=noise)
    _, _, tau, fd = axes(nf, nt, npad)
    edges, etas = grid(65), np.array(FULL)
    cs = th.conjugate_spectrum(dyn, npad, None)
    CS = cs.numpy()
    ga, ia = th.eta_sweep(cs, tau, fd, etas, edges, return_info=True)
    gb, ib = th.eta_sweep(CS, tau, fd, etas, edges, return_info=True)
    for info in (ia, ib):
        assert (info["status"] == 0).all(), info["status"]       # no iteration cap (bit 8)
    assert np.array_equal(ia["nred"], ib["nred"])
    bound, m = float(cs.bound.cpu()[0]), _max_re_im(CS)
    RATIO["sweep %dx%d npad%d noise=%g" % (nf, nt, npad, noise)] = [bound / m]
    report("bound vs scan sweep", (np.abs(ga - gb) / gb).max() / RTOL)
    for a, b, e in zip(ga, gb, etas):
        r = ref_eig(CS, tau, fd, e, edges)
        report("bound sweep", abs(a - r["w1"]) / r["w1"] / RTOL)
        report("scan sweep", abs(b - r["w1"]) / r["w1"] / RTOL)
