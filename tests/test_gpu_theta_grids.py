"""The theta-theta solvers at every grid-size regime up to their limits, against
float64 references, and every grid limit from both sides.

Besides the spectrum size, the theta-theta code is dispatched on the number of
theta centres N, padded to ld = 32 ceil(N / 32):
  sweep      eta_sweep / Eval_calc / single_search (thth.cu::eta_sweep):
             ld <= 512: the fp16 tensor-core solver (eig_half.cu), or with
             SB_EIG_FP32=1 the fp32 direct-load thth_eig_kernel; ld 544 .. 4096:
             thth_eig_kernel, which walks the cropped matrix in column chunks
             of 512 (nchunk = ceil(nred / 512) = 1 .. 8);
             ld > 4096 is refused before any launch.
  thin       thin_sweep / singularvalue_calc (thin.cu): columns in chunks of 512
             (nchunk = ceil(n1 / 512) = 1 .. 8), rows of any count; 4096 on
             either axis.
  eigvec     modeler / single_chunk_retrieval (herm_eigvec, n <= 8192),
             chisq_sweep / asymmetry_batch (herm_eigvec_batch, ld <= 4096),
             VLBI_chunk_retrieval (a composite of n_dish nred <= 8192).
SWEEP_CASES / THIN_CASES / EIGVEC_CASES restate that dispatch;
test_case_table_coverage (no GPU) fails if an edit drops a regime or a side of
a limit.

Input: one synthetic arc (48 images on a 1-D screen, eta 0.02 s^3, 20 % noise)
as a 64 x 4096 dynamic spectrum, npad = 1: a 128 x 8192 conjugate spectrum with
dfd = 0.0122 mHz.  Every grid spans +-24 mHz, so at 4096 centres the theta
spacing is 0.96 fd bins, and the largest |theta_i - theta_j| = 48 mHz stays
inside the fd axis (+-50 mHz).  Curvatures below tau_max / 24^2 = 0.0273 keep
every centre.  References are the oracle in float64 on the SAME fp32 spectrum
the device made (cs.numpy()); a case whose reference relative gap
(w1 - w2) / w1 is below 1e-3 is a bad case, not a solver failure.

Bars.  Eigenvalues and singular values: |rel| <= 1e-5, cropped sizes bit-exact.
Vectors, after one global phase (first-order Davis-Kahan: sin theta <=
(||E|| + ||r||) / (w1 - w2), |dV| <= sqrt(2) sin theta):

    |dV| <= sqrt(2) (c(n) 2^-24 ||A||_F + TOL_ACCEPT |w1|) / (w1 - w2)

where ||A||_F is the Frobenius norm of the reference matrix and c(n) counts the
fp32 perturbations of A relative to ||A||_F.  The reference shares the device's
spectrum, so the transform term of test_gpu_asymmetry.py (17) drops out.  That
leaves 1 for rounding each gathered entry to fp32, 1 for the fp32 Jacobian, and
sqrt(n) for the fp32 mat-vec of the Lanczos steps: each row sums n products, and
their rounding errors grow like sqrt(n) 2^-24.  So c(n) = 2 + sqrt(n): 36 at
n = 1024 and 66 at 4095.  The constant 17 = sqrt(301) of the asymmetry test is
this term at n = 301.  TOL_ACCEPT = 2e-6 is the residual the solver accepts at
its iteration cap.  A wavefield or model is linear (model_E) or quadratic
(modeler's model) in V, so its normwise relative error is at most |dV| (2 |dV|)
plus 1e-5 for w, plus E_MODEL = 5e-5 for the fp32 scatter and inverse transform,
the value test_gpu_vlbi.py uses.  The run prints the worst error of each regime
as a fraction of its bar."""
import math
import os
import sys
from collections import namedtuple

import numpy as np
import pytest

from oracle import thth_oracle as TO
from oracle import vlbi_oracle as VO

NF, NT, NPAD = 64, 4096, 1
DT, DF, F0 = 10.0, 0.03125, 1400.0
ETA_ARC = 0.02                   # s^3, curvature of the synthetic arc
EDGE = 24.0                      # mHz, every grid spans -EDGE .. EDGE
FULL = (0.016, 0.02, 0.024)      # curvatures that keep all centres (< 0.0273)
LIMIT = 4096                     # theta centres of the sweep, thin and batched eigvec paths

RTOL = 1e-5
GAP_MIN = 1e-3
TOL_ACCEPT = 2e-6
E_MODEL = 5e-5
U32 = 2.0 ** -24

Case = namedtuple("Case", "path n etas extra")


def _c(path, n, etas, **extra):
    return Case(path, n, tuple(etas), tuple(sorted(extra.items())))


def case_id(c):
    s = "%s-%s-%s" % (c.path, c.n if isinstance(c.n, int) else "x".join(map(str, c.n)),
                      ",".join("%g" % e for e in c.etas))
    return s + "".join("-%s=%s" % kv for kv in c.extra)


SWEEP_N = [31, 32, 33, 511, 512, 513, 1023, 1024, 1025, 1317, 1537, 2049, 3073, 4095, 4096]
# one launch whose curvatures crop 3073 centres down to ~480: one ld, nchunk 7 .. 1
CROP_ETAS = tuple(np.round(np.geomspace(0.02, 1.1, 8), 5))
SWEEP_CASES = [_c("sweep", n, FULL if n < 511 else FULL[1:]) for n in SWEEP_N] + \
    [_c("sweep", 3073, CROP_ETAS, crop=1)] + \
    [_c("sweep", n, FULL[1:2], fp32=1) for n in (511, 512)]

THIN_COLS = [511, 512, 513, 1025, 2049, 4095, 4096]
THIN_CASES = [_c("thin", (n1, n2), (ETA_ARC,)) for n1 in THIN_COLS
              for n2 in sorted({33, n1, LIMIT})] + \
    [_c("thin", (n1, 33), (ETA_ARC,)) for n1 in (1537, 2561, 3073)] + \
    [_c("thin", (33, LIMIT), (ETA_ARC,)),
     _c("thin", (1536, 513), (ETA_ARC,), cut=0.5 * EDGE),
     _c("thin", (LIMIT, 512), (ETA_ARC,), power=1)]

EIGVEC_CASES = [_c("retrieval", n, (ETA_ARC,)) for n in (513, 1317, 4095)] + \
    [_c("chisq", LIMIT, (ETA_ARC,)), _c("asymmetry", LIMIT, (ETA_ARC,)),
     _c("vlbi", (2, LIMIT), (ETA_ARC,))]

# (what, accepted case, refused size)
LIMITS = [
    ("sweep centres", _c("sweep", 4096, FULL[1:]), 4097),
    ("thin columns", _c("thin", (LIMIT, 33), (ETA_ARC,)), (4097, 33)),
    ("thin rows", _c("thin", (33, LIMIT), (ETA_ARC,)), (33, 4097)),
    ("chisq centres", _c("chisq", LIMIT, (ETA_ARC,)), 4097),
    ("asymmetry centres", _c("asymmetry", LIMIT, (ETA_ARC,)), 4097),
    ("vlbi composite", _c("vlbi", (2, LIMIT), (ETA_ARC,)), (2, 4097)),
]


# --------------------------------------------------------------------------
# geometry (host only)
# --------------------------------------------------------------------------
def axes():
    t = DT * np.arange(NT)
    f = F0 + DF * np.arange(NF)
    return t, f, TO.fft_axis(f, "us", NPAD), TO.fft_axis(t, "mHz", NPAD)


def grid(n):
    """n + 1 edges over -EDGE .. EDGE; an even count is shifted by a tenth of a step
    so that the smallest |centre| is unique (theta_centres needs one)."""
    e = np.linspace(-EDGE, EDGE, n + 1)
    return e + (0.1 * (e[1] - e[0]) if n % 2 == 0 else 0.0)


def nred(n, eta):
    _, _, tau, fd = axes()
    return int(TO.th_points(tau, fd, eta, grid(n)).sum())


def sweep_regimes(c):
    """The solver each curvature of a sweep case runs on."""
    ld = 32 * math.ceil(c.n / 32)
    out = []
    for eta in c.etas:
        if ld <= 512:
            out.append("fp32 direct ld<=512" if dict(c.extra).get("fp32") else "fp16")
        else:
            out.append("direct nchunk=%d" % math.ceil(nred(c.n, eta) / 512))
    return out


def thin_regime(c):
    return "thin nchunk=%d" % math.ceil(c.n[0] / 512)


def missing_coverage():
    miss = []
    sweep = {r for c in SWEEP_CASES for r in sweep_regimes(c)}
    for want in ["fp16", "fp32 direct ld<=512"] + ["direct nchunk=%d" % k for k in range(1, 9)]:
        if want not in sweep:
            miss.append("sweep " + want)
    lds = {32 * math.ceil(c.n / 32) for c in SWEEP_CASES}
    miss += ["sweep ld %d" % ld for ld in (512, 544, 4096) if ld not in lds]
    thin = {thin_regime(c) for c in THIN_CASES}
    miss += ["thin nchunk=%d" % k for k in range(1, 9) if "thin nchunk=%d" % k not in thin]
    sizes = {c.n for c in THIN_CASES}
    miss += ["thin %dx%d" % s for s in ((LIMIT, 33), (33, LIMIT), (LIMIT, LIMIT)) if s not in sizes]
    if not any(dict(c.extra).get("power") for c in THIN_CASES):
        miss.append("thin power")
    cut = [c for c in THIN_CASES if dict(c.extra).get("cut")]
    if not cut:
        miss.append("thin center_cut")
    for c in cut:       # zeroed columns in the first and in the last of >= 3 column chunks
        e = grid(c.n[0])
        z = np.flatnonzero(np.abs((e[1:] + e[:-1]) / 2) < dict(c.extra)["cut"])
        last = (c.n[0] - 1) // 512
        if not (last >= 2 and z.min() < 512 and z.max() >= 512 * last):
            miss.append("thin center_cut chunks")
    return miss


# --------------------------------------------------------------------------
# tests without a GPU
# --------------------------------------------------------------------------
def test_case_table_coverage():
    """Every sweep solver and direct-kernel chunk count 1 .. 8, both sides of the
    ld 512 / 544 switch, every thin column-chunk count 1 .. 8, both thin extremes,
    the incoherent and center-cut variants are reached by some case."""
    assert missing_coverage() == []
    ids = [case_id(c) for c in SWEEP_CASES + THIN_CASES + EIGVEC_CASES]
    assert len(set(ids)) == len(ids)
    # full-crop curvatures really keep every centre
    for c in SWEEP_CASES:
        if not dict(c.extra).get("crop"):
            assert all(nred(c.n, e) == c.n for e in c.etas), case_id(c)
    crop = [nred(3073, e) for e in CROP_ETAS]
    assert crop[0] == 3073 and crop[-1] < 512 and crop == sorted(crop, reverse=True)


def test_limits_both_sides_in_table():
    """The largest accepted size of each limit is a case; the refused size is one past it."""
    ids = {case_id(c) for c in SWEEP_CASES + THIN_CASES + EIGVEC_CASES}
    for what, ok, bad in LIMITS:
        assert case_id(ok) in ids, what
        n_ok = ok.n if isinstance(ok.n, int) else max(ok.n)
        n_bad = bad if isinstance(bad, int) else max(bad)
        assert n_bad == n_ok + 1 and 32 * math.ceil(n_bad / 32) > LIMIT, what


def test_grid_spacing_and_fd_axis():
    """At 4096 centres the theta spacing is about one fd bin, and 2 EDGE stays inside
    the fd axis, so no case becomes an IndexError by accident."""
    _, _, tau, fd = axes()
    dfd = np.diff(fd).mean()
    step = np.diff(TO.theta_centres(grid(LIMIT))).mean()
    assert 0.9 < step / dfd < 1.1
    assert 2 * EDGE < -fd[0] and EDGE < abs(fd.max()) / 2


# --------------------------------------------------------------------------
# GPU: shared input and references
# --------------------------------------------------------------------------
WORST = {}


def report(regime, frac):
    WORST[regime] = max(WORST.get(regime, 0.0), float(frac))
    assert frac <= 1.0, (regime, frac)


def screen(seed=5, n_dish=1):
    """Wavefields of n_dish stations seeing one 48-image screen on the arc tau =
    ETA_ARC fd^2, each image with a per-station phase."""
    rng = np.random.default_rng(seed)
    t, f, _, _ = axes()
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


def synthetic_dynspec():
    (E,), rng = screen()
    dyn = np.abs(E) ** 2
    dyn += rng.normal(0.0, 0.2 * dyn.mean(), dyn.shape)
    return dyn - dyn.mean()


@pytest.fixture(scope="module")
def sb():
    import scintools_b200
    from scintools_b200 import _device
    _device.device()
    return scintools_b200


@pytest.fixture(scope="module")
def data(sb):
    """The dynamic spectrum, its device spectrum (padded with its mean, half plane:
    what single_search, single_chunk_retrieval and asymmetry_batch make) and the
    float64 copy of that spectrum the references use."""
    dyn = synthetic_dynspec()
    cs = sb.ththmod.conjugate_spectrum(dyn, NPAD, None)
    t, f, tau, fd = axes()
    yield dict(dyn=dyn, cs=cs, CS=cs.numpy(), t=t, f=f, tau=tau, fd=fd, cache={})
    if WORST:
        print("\ntheta grids: worst error per regime, as a fraction of its bar")
        for k in sorted(WORST):
            print("  %-36s %.3g" % (k, WORST[k]))
        sys.stdout.flush()


def ref_eig(data, n, eta):
    """The oracle's cropped matrix and its two top eigenpairs, once per module."""
    from scipy.sparse.linalg import eigsh
    key = ("eig", n, eta)
    if key not in data["cache"]:
        red, edges_red = TO.thth_redmap(data["CS"], data["tau"], data["fd"], eta, grid(n))
        if red.shape[0] <= 1100:
            w, V = np.linalg.eigh(red)
        else:
            v0 = red[red.shape[0] // 2].copy()
            v0 /= np.linalg.norm(v0)
            w, V = eigsh(red, 2, v0=v0, which="LA", ncv=24)
        k = np.argsort(w)[::-1]
        w1, w2, V = w[k[0]], w[k[1]], V[:, k]
        assert (w1 - w2) / w1 > GAP_MIN, ("bad case: reference gap", n, eta, (w1 - w2) / w1)
        data["cache"][key] = dict(n=red.shape[0], w1=w1, w2=w2, V=V[:, 0],
                                  fro=np.linalg.norm(red), edges_red=edges_red)
    return data["cache"][key]


def dV_bound(n, w1, w2, fro):
    return np.sqrt(2) * ((2 + np.sqrt(n)) * U32 * fro + TOL_ACCEPT * abs(w1)) / (w1 - w2)


def align(V, Vr):
    ph = np.vdot(Vr, V)
    return ph / abs(ph)


# --------------------------------------------------------------------------
# a. eta_sweep, Eval_calc, single_search
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", SWEEP_CASES, ids=case_id)
def test_sweep(sb, data, case, monkeypatch):
    th = sb.ththmod
    edges = grid(case.n)
    etas = np.array(case.etas)
    if dict(case.extra).get("fp32"):
        monkeypatch.setenv("SB_EIG_FP32", "1")
    got, info = th.eta_sweep(data["cs"], data["tau"], data["fd"], etas, edges, return_info=True)
    assert (info["status"] == 0).all(), info["status"]
    assert list(info["nred"]) == [nred(case.n, e) for e in etas]
    refs = [ref_eig(data, case.n, e) for e in etas]
    for e, r, g, reg in zip(etas, refs, got, sweep_regimes(case)):
        assert r["n"] == nred(case.n, e)
        report("sweep " + reg, abs(g - r["w1"]) / r["w1"] / RTOL)
    if dict(case.extra):
        return
    # Eval_calc and single_search (its own spectrum, fd columns restricted to the grid)
    w = th.Eval_calc(data["cs"], data["tau"], data["fd"], etas[0], edges)
    report("sweep Eval_calc", abs(w - refs[0]["w1"]) / refs[0]["w1"] / RTOL)
    res = th.single_search([data["dyn"], data["f"], data["t"], etas, edges, None, False, 0.1,
                            NPAD, True, 0.0, False])
    for g, r in zip(res[4], refs):
        report("sweep single_search", abs(g - r["w1"]) / r["w1"] / RTOL)


@pytest.mark.gpu
def test_sweep_small_slab_bit_identical(sb, data, monkeypatch):
    """4095 centres (134 MB per matrix): one curvature per launch gives the bits of
    the default single launch."""
    th = sb.ththmod
    etas = np.array(FULL)
    whole = th.eta_sweep(data["cs"], data["tau"], data["fd"], etas, grid(4095))
    monkeypatch.setenv("SB_SWEEP_SLAB_MB", "1")
    sliced = th.eta_sweep(data["cs"], data["tau"], data["fd"], etas, grid(4095))
    assert np.array_equal(whole.view(np.uint64), sliced.view(np.uint64))


@pytest.mark.gpu
def test_sweep_limit_refused_before_any_launch(sb, data):
    """4097 centres: sb_eta_sweep refuses, naming 4096, before any launch; Eval_calc and
    single_search raise SbError; the library keeps working."""
    import torch
    from scintools_b200 import _device as D, _lib
    th = sb.ththmod
    edges = grid(4097)
    geom = th._Geom(data["cs"], data["tau"], data["fd"], edges, True)
    d_etas = D.upload(np.array(FULL))
    out = [D.empty((3,), torch.float64)] + [D.empty((3,), torch.int32) for _ in range(3)]
    n0 = _lib.lib.sb_launch_count()
    rc = _lib.lib.sb_eta_sweep(geom.ref, d_etas.data_ptr(), 3, th.DEFAULT_TOL, 0,
                               *[o.data_ptr() for o in out], D.stream_ptr())
    assert rc != 0 and b"4096" in _lib.lib.sb_last_error()
    assert _lib.lib.sb_launch_count() == n0
    with pytest.raises(_lib.SbError, match="4096"):
        th.eta_sweep(data["cs"], data["tau"], data["fd"], np.array(FULL), edges)
    with pytest.raises(_lib.SbError, match="4096"):
        th.Eval_calc(data["cs"], data["tau"], data["fd"], ETA_ARC, edges)
    with pytest.raises(_lib.SbError, match="4096"):
        th.single_search([data["dyn"], data["f"], data["t"], np.array(FULL), edges, None, False,
                          0.1, NPAD, True, 0.0, False])
    r = ref_eig(data, 33, ETA_ARC)
    w = th.Eval_calc(data["cs"], data["tau"], data["fd"], ETA_ARC, grid(33))
    assert abs(w - r["w1"]) <= RTOL * r["w1"]


# --------------------------------------------------------------------------
# b. thth_map and thth_redmap at 4095 centres
# --------------------------------------------------------------------------
@pytest.mark.gpu
def test_thth_map_indices_4095(sb, data):
    th = sb.ththmod
    edges = grid(4095)
    m, ti, fi, pn = th.thth_map(data["cs"], data["tau"], data["fd"], ETA_ARC, edges,
                                return_indices=True)
    _, rti, rfi, rpn = TO.thth_indices(data["tau"], data["fd"], ETA_ARC, edges)
    assert np.array_equal(ti, rti.astype(np.int32))
    assert np.array_equal(fi, rfi.astype(np.int32))
    assert np.array_equal(pn, rpn)
    del m, ti, fi, pn, rti, rfi, rpn
    eta = CROP_ETAS[3]
    red, er = th.thth_redmap(data["cs"], data["tau"], data["fd"], eta, edges)
    rred, rer = TO.thth_redmap(data["CS"], data["tau"], data["fd"], eta, edges)
    assert red.shape == rred.shape and red.shape[0] < 4095
    assert np.array_equal(er, rer)
    assert np.array_equal(red == 0, rred == 0)
    report("thth_redmap entries (1e-6)", np.abs(red - rred).max() / np.abs(rred).max() / 1e-6)


# --------------------------------------------------------------------------
# c. thin_sweep and singularvalue_calc
# --------------------------------------------------------------------------
def ref_thin(data, n1, n2, eta, cut, power):
    from scipy.sparse.linalg import LinearOperator, eigsh
    src = np.abs(data["CS"]) ** 2 if power else data["CS"]
    red, er1, _ = TO.two_curve_map(src, data["tau"], data["fd"], eta, grid(n1), eta, grid(n2))
    red[:, np.abs((er1[1:] + er1[:-1]) / 2) < cut] = 0
    assert red.shape == (n2, n1)
    if min(red.shape) <= 600:
        s = np.linalg.svd(red, compute_uv=False)[:2]
    else:
        op = LinearOperator((n1, n1), matvec=lambda x: red.conj().T @ (red @ x),
                            dtype=np.complex128)
        s = np.sqrt(np.sort(eigsh(op, 2, which="LA", ncv=24)[0])[::-1])
    assert (s[0] ** 2 - s[1] ** 2) / s[0] ** 2 > GAP_MIN, ("bad case: reference gap", n1, n2)
    return s[0]


@pytest.mark.gpu
@pytest.mark.parametrize("case", THIN_CASES, ids=case_id)
def test_thin(sb, data, case):
    th = sb.ththmod
    (n1, n2), eta = case.n, case.etas[0]
    x = dict(case.extra)
    cut, power = x.get("cut", 0.0), bool(x.get("power"))
    sv, info = th.thin_sweep(data["cs"], data["tau"], data["fd"], np.array([eta]), grid(n1),
                             grid(n2), cut, power=power, return_info=True)
    assert info["status"][0] == 0 and (info["n1"][0], info["n2"][0]) == (n1, n2)
    ref = ref_thin(data, n1, n2, eta, cut, power)
    tag = " power" if power else (" cut" if cut else "")
    report(thin_regime(case) + tag, abs(sv[0] - ref) / ref / RTOL)
    if not power:
        s = th.singularvalue_calc(data["cs"], data["tau"], data["fd"], eta, grid(n1), eta,
                                  grid(n2), cut)
        assert s == sv[0]


@pytest.mark.gpu
def test_thin_small_slab_bit_identical(sb, data, monkeypatch):
    """120 pairs on grids padded to 64 x 64 (32 KiB per matrix): SB_SWEEP_SLAB_MB=1 (32
    pairs per launch) gives the bits of the default single launch."""
    th = sb.ththmod
    etas = np.linspace(0.012, 0.03, 120)

    def run():
        sv, info = th.thin_sweep(data["cs"], data["tau"], data["fd"], etas, grid(63), grid(50),
                                 0.0, etasArclet=etas[::-1], return_info=True)
        return [sv] + [info[k] for k in ("status", "n1", "n2", "iters")]

    whole = run()
    assert np.isfinite(whole[0]).all() and (whole[1] == 0).any()
    monkeypatch.setenv("SB_SWEEP_SLAB_MB", "1")
    sliced = run()
    assert np.array_equal(whole[0].view(np.uint64), sliced[0].view(np.uint64))
    for a, b in zip(whole[1:], sliced[1:]):
        assert np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("n1,n2", [(4097, 33), (33, 4097)])
def test_thin_limit_refused_before_any_launch(sb, data, n1, n2):
    """4097 on either axis: sb_thin_sweep refuses, naming 4096, before any launch (the
    DeviceCS is already made, so the library's only call here is sb_thin_sweep)."""
    from scintools_b200 import _lib
    th = sb.ththmod
    n0 = _lib.lib.sb_launch_count()
    with pytest.raises(_lib.SbError, match="4096"):
        th.thin_sweep(data["cs"], data["tau"], data["fd"], np.array([ETA_ARC]), grid(n1),
                      grid(n2), 0.0)
    assert _lib.lib.sb_launch_count() == n0
    with pytest.raises(_lib.SbError, match="4096"):
        th.singularvalue_calc(data["cs"], data["tau"], data["fd"], ETA_ARC, grid(n1), ETA_ARC,
                              grid(n2), 0.0)


# --------------------------------------------------------------------------
# d. top eigenpairs at large n
# --------------------------------------------------------------------------
def ref_model(data, n, eta):
    """modeler's recov / model and single_chunk_retrieval's model_E from the oracle's
    pieces on the reference eigenpair."""
    key = ("model", n, eta)
    if key not in data["cache"]:
        r = ref_eig(data, n, eta)
        tau, fd, V, w = data["tau"], data["fd"], r["V"], r["w1"]
        recov = TO.rev_map(np.outer(V, np.conj(V)) * abs(w), tau, fd, eta, r["edges_red"], True)
        model = np.fft.ifft2(np.fft.ifftshift(recov)).real
        E = np.zeros((r["n"], r["n"]), dtype=complex)
        E[r["n"] // 2] = np.conj(V) * np.sqrt(w)
        recE = TO.rev_map(E, tau, fd, eta, r["edges_red"], hermetian=False)
        model_E = np.fft.ifft2(np.fft.ifftshift(recE))[:NF, :NT] * (NF * NT / 4)
        data["cache"][key] = dict(recov=recov, model=model, model_E=model_E)
    return data["cache"][key]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [c.n for c in EIGVEC_CASES if c.path == "retrieval"])
def test_modeler_and_retrieval(sb, data, n):
    th = sb.ththmod
    r = ref_eig(data, n, ETA_ARC)
    m = ref_model(data, n, ETA_ARC)
    dV = dV_bound(r["n"], r["w1"], r["w2"], r["fro"])
    _, _, recov, model, edges_red, w, V = th.modeler(data["cs"], data["tau"], data["fd"], ETA_ARC,
                                                     grid(n))
    assert np.array_equal(edges_red, r["edges_red"]) and V.shape == (n,)
    report("herm_eigvec w", abs(w - r["w1"]) / r["w1"] / RTOL)
    ev = np.linalg.norm(V - align(V, r["V"]) * r["V"])
    report("herm_eigvec V (Davis-Kahan)", ev / dV)
    assert np.array_equal(recov == 0, m["recov"] == 0)
    err = np.linalg.norm(model - m["model"]) / np.linalg.norm(m["model"])
    report("modeler model", err / (2 * dV + RTOL + E_MODEL))
    model_E = th.single_chunk_retrieval((data["dyn"], grid(n), data["t"], data["f"], ETA_ARC,
                                         0, 0, NPAD, 0.0, False))[0]
    ref_E = m["model_E"]
    err = np.linalg.norm(model_E - align(model_E, ref_E) * ref_E) / np.linalg.norm(ref_E)
    report("single_chunk_retrieval model_E", err / (dV + RTOL + E_MODEL))


@pytest.mark.gpu
def test_chisq_sweep_4096(sb, data):
    th = sb.ththmod
    r = ref_eig(data, LIMIT, ETA_ARC)
    m = ref_model(data, LIMIT, ETA_ARC)
    chisq, info = th.chisq_sweep(data["dyn"], data["cs"], data["tau"], data["fd"],
                                 np.array([ETA_ARC]), grid(LIMIT), 1.0, return_info=True)
    assert info["status"][0] == 0 and info["nred"][0] == LIMIT
    report("chisq w", abs(info["w"][0] - r["w1"]) / r["w1"] / RTOL)
    model = m["model"][:NF, :NT]
    resid = np.linalg.norm(model - data["dyn"])
    dm = (2 * dV_bound(LIMIT, r["w1"], r["w2"], r["fro"]) + RTOL + E_MODEL) * \
        np.linalg.norm(m["model"])
    ref = resid ** 2
    report("chisq value", abs(chisq[0] - ref) / (2 * resid * dm + dm ** 2))


@pytest.mark.gpu
def test_asymmetry_4096(sb, data):
    th = sb.ththmod
    r = ref_eig(data, LIMIT, ETA_ARC)
    res, info = th.asymmetry_batch([(data["dyn"], grid(LIMIT), data["t"], data["f"], ETA_ARC,
                                     0, 0, NPAD, False)], return_info=True)
    assert info["status"][0] == 0 and info["nred"][0] == LIMIT
    report("asymmetry w", abs(info["w"][0] - r["w1"]) / r["w1"] / RTOL)
    dV = dV_bound(LIMIT, r["w1"], r["w2"], r["fro"])
    V = info["V"][0]
    report("asymmetry V (Davis-Kahan)", np.linalg.norm(V - align(V, r["V"]) * r["V"]) / dV)
    p = np.abs(r["V"]) ** 2
    m = LIMIT
    L, R = p[:(m - 1) // 2].sum(), p[(m + 1) // 2:].sum()
    a = (L - R) / (L + R)
    report("asymmetry value", abs(res[0][0] - a) / (2 * (1 + abs(a)) / (L + R) * dV))


def stations():
    """[I1, V12, I2] of two stations, 64 x 4096 each, with 5 % noise."""
    (E1, E2), rng = screen(seed=9, n_dish=2)
    sig = np.mean(np.abs(E1) ** 2)
    out = []
    for d1, d2 in ((0, 0), (0, 1), (1, 1)):
        Ea, Eb = (E1, E2)[d1], (E1, E2)[d2]
        if d1 == d2:
            x = np.abs(Ea) ** 2 + rng.normal(0, 0.05 * sig, Ea.shape)
            out.append(x - x.mean())
        else:
            out.append(Ea * np.conj(Eb) + 0.05 * sig * (rng.normal(size=Ea.shape) +
                                                         1j * rng.normal(size=Ea.shape)))
    return out


@pytest.mark.gpu
def test_vlbi_composite_8192(sb, data):
    """2 stations x 4096 centres: a composite of exactly 8192 with non-zero
    visibilities.  The reference solves the composite as a LinearOperator over its
    three blocks, on the device's spectra."""
    from scipy.sparse.linalg import LinearOperator, eigsh
    th = sb.ththmod
    dl = stations()
    tau, fd, edges = data["tau"], data["fd"], grid(LIMIT)
    model, w, V, info, err = th._vlbi_run(dl, edges, data["t"], data["f"], ETA_ARC, NPAD, 2, 0.0)
    assert err is None and info["status"] == 0 and info["nred"] == LIMIT
    blocks, edges_red = [], None
    for k, d in enumerate(dl):
        cs = th.conjugate_spectrum(d, NPAD, None if k != 1 else 0.0, tau, 0.0, half=False)
        red, edges_red = TO.thth_redmap(cs.numpy(), tau, fd, ETA_ARC, edges, hermetian=k != 1)
        blocks.append(red)
        del cs
    A0, T, A1 = blocks
    n = A0.shape[0]

    def mv(x):
        x = np.ravel(x)
        return np.concatenate((A0 @ x[:n] + T.conj().T @ x[n:], T @ x[:n] + A1 @ x[n:]))

    op = LinearOperator((2 * n, 2 * n), matvec=mv, dtype=np.complex128)
    ww, VV = eigsh(op, 2, which="LA", ncv=24)
    k = np.argsort(ww)[::-1]
    w1, w2, Vr = ww[k[0]], ww[k[1]], VV[:, k[0]]
    assert (w1 - w2) / w1 > GAP_MIN, ("bad case: reference gap", (w1 - w2) / w1)
    fro = np.sqrt(np.linalg.norm(A0) ** 2 + np.linalg.norm(A1) ** 2 + 2 * np.linalg.norm(T) ** 2)
    del blocks, A0, T, A1
    report("vlbi w", abs(w - w1) / w1 / RTOL)
    dV = dV_bound(2 * n, w1, w2, fro)
    ph = align(V, Vr)
    report("vlbi V (Davis-Kahan)", np.linalg.norm(V - ph * Vr) / dV)
    refs = VO.station_models(w1, Vr, 2, tau, fd, ETA_ARC, edges_red, (NF, NT))
    for d in range(2):
        # model_E is linear in conj(V): the same phase, conjugated, for both stations
        e = np.linalg.norm(model[d] - np.conj(ph) * refs[d]) / np.linalg.norm(refs[d])
        report("vlbi wavefield", e / (dV + RTOL + E_MODEL))


@pytest.mark.gpu
def test_batched_eigvec_limits_refused(sb, data):
    """One centre past each batched limit: chisq_sweep and asymmetry_batch refuse 4097
    centres, VLBI refuses a composite of 2 x 4097, all naming the limit."""
    from scintools_b200 import _lib
    th = sb.ththmod
    edges = grid(4097)
    with pytest.raises(_lib.SbError, match="4096"):
        th.chisq_sweep(data["dyn"], data["cs"], data["tau"], data["fd"], np.array([ETA_ARC]),
                       edges, 1.0)
    with pytest.raises(_lib.SbError, match="4096"):
        th.asymmetry_batch([(data["dyn"], edges, data["t"], data["f"], ETA_ARC, 0, 0, NPAD,
                             False)])
    z = [np.zeros((16, 16))] * 3
    with pytest.raises(_lib.SbError, match="8192"):
        th._vlbi_run(z, np.linspace(-1.0, 1.0, 4098), 10.0 * np.arange(16),
                     1400.0 + 0.05 * np.arange(16), 1e-3, 0, 2, 0.0)


# --------------------------------------------------------------------------
# the reference notebook's grid: 1317 centres on a 128 x 150 chunk
# (tests/golden/thth_notebook_1317.npz, made by oracle/make_golden_grids.py)
# --------------------------------------------------------------------------
def _notebook(golden_dir):
    return np.load(os.path.join(golden_dir, "thth_notebook_1317.npz"))


def test_notebook_fixture_matches_oracle(golden_dir):
    """The oracle reproduces the unmodified reference at 1317 centres: Eval_calc on
    three of the stored curvatures, modeler's w and |V|^2."""
    g = _notebook(golden_dir)
    assert g["edges"].shape == (1318,) and g["chunk"].shape == (128, 150)
    npad = int(g["npad"])
    tau, fd = TO.fft_axis(g["freq"], "us", npad), TO.fft_axis(g["time"], "mHz", npad)
    assert np.array_equal(tau, g["tau"]) and np.array_equal(fd, g["fd"])
    CS = TO.conjugate_spectrum(g["chunk"], npad, None)
    assert CS.shape == (512, 600)
    for k in (0, int(np.argmax(g["eigs"])), len(g["etas"]) - 1):
        w = TO.Eval_calc(CS, tau, fd, g["etas"][k], g["edges"])
        assert w == pytest.approx(float(g["eigs"][k]), rel=1e-9), k
    red, _ = TO.thth_redmap(CS, tau, fd, float(g["eta_model"]), g["edges"])
    assert red.shape[0] == int(g["nred"])
    w, V = np.linalg.eigh(red)
    assert w[-1] == pytest.approx(float(g["w"]), rel=1e-9)
    assert np.abs(np.abs(V[:, -1]) ** 2 - g["V2"]).max() < 1e-9 * g["V2"].max()


@pytest.mark.gpu
def test_notebook_grid_on_gpu(sb, golden_dir):
    """eta_sweep and modeler on the notebook chunk (CS 512 x 600 on the chirp-z path,
    ld 1344: the direct kernel with 3 column chunks at the wide curvatures) against
    the reference.  The device spectrum is fp32 here, so the vector bound adds the
    transform term 17 of test_gpu_asymmetry.py: c(n) = 19 + sqrt(n)."""
    th = sb.ththmod
    g = _notebook(golden_dir)
    npad = int(g["npad"])
    cs = th.conjugate_spectrum(g["chunk"], npad, None)
    got, info = th.eta_sweep(cs, g["tau"], g["fd"], g["etas"], g["edges"], return_info=True)
    assert (info["status"] == 0).all() and info["nred"].max() > 1024
    report("notebook eta_sweep", (np.abs(got - g["eigs"]) / g["eigs"]).max() / RTOL)
    _, _, _, _, _, w, V = th.modeler(cs, g["tau"], g["fd"], float(g["eta_model"]), g["edges"])
    n = int(g["nred"])
    assert V.shape == (n,)
    report("notebook modeler w", abs(w - float(g["w"])) / float(g["w"]) / RTOL)
    w1, w2, fro = float(g["w1"]), float(g["w2"]), float(g["fro"])
    dV = np.sqrt(2) * ((19 + np.sqrt(n)) * U32 * fro + TOL_ACCEPT * w1) / (w1 - w2)
    r2 = g["V2"]
    bound = (2 * np.sqrt(r2) + dV) * dV
    report("notebook modeler |V|^2", (np.abs(np.abs(V) ** 2 - r2) / bound).max())
