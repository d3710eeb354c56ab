"""The batched entry points at item counts past 65,535: curvatures, curvature pairs,
chunks and output rows, against the same items sent in small calls and against
float64 references.

Each of these entry points handles a caller-supplied number of items in one call.
CUDA caps gridDim.y at 65535, so a launch that gives every item a row of the grid
has to be split (or loop) past that count:
  eta_sweep     sb_eta_sweep (eta_sweep, Eval_calc, single_search): the IndexError
                scan of thth_prep runs in launches of <= 65535 curvatures whenever
                the theta span reaches past the fd axis (lower_check_needed).
  chisq_sweep   sb_chisq_sweep: the same thth_prep, then batches of <= 65535
                curvatures.
  thin_sweep    sb_thin_sweep: the IndexError scan in launches of <= 65535
                (etas, etasArclet) pairs, always.
  asymmetry     sb_asymmetry_batch: thth_prep_table's scan in launches of <= 65535
                chunks, then batches of <= 65535.
  scale_dyn     Dynspec.scale_dyn: spline_eval_kernel walks the output rows in steps
                of gridDim.y <= 65535.
ITEM_CASES and SCALE_CASES restate those limits; the tests without a GPU fail if an
entry point loses its case on either side of 65,535.

Input: 31 theta centres (ld 32) on an 8 x 32 dynamic spectrum, npad = 1, so the
conjugate spectrum is 16 x 64 (8 KB in fp32) and the count is the only thing that
is large.  At this size a chi-square curvature needs 45 KB of workspace, so the
65535 cap, not the 3 GiB slab, sets its batch.  Two grids: WIDE spans 165 mHz, past
1.5 x the fd range, so numpy raises IndexError for the smaller curvatures and not
for the larger; ORDINARY stays inside the fd axis, so no scan runs (the control).
The curvatures are a shuffled geometric set over ETA_LO .. ETA_HI, and every
launch of <= 65535 holds both outcomes.

Checks, per entry point:
  * every item equals the same item sent in calls of at most SPLIT = 30000 items
    (a size that never needed more than one launch): bit-identical eigenvalues,
    singular values, asymmetries, status, sizes and iteration counts.  The
    chi-square sums are accumulated with fp32 atomics, so they are held to 1e-6
    (as test_gpu_chisq.py's batching test) and their eigenvalues bit-exactly;
  * the NaN / IndexError status pattern equals the oracle's IndexError pattern
    for every item (index_errors / thin_index_errors restate the oracle's test
    with the same float64 expressions, vectorised over curvatures; a CPU test
    checks them against the oracle's own try/except);
  * at least 200 sampled items, among them the four on each side of every
    65535 boundary, against float64 references: oracle Eval_calc and
    singularvalue_calc at 1e-5, oracle chisq_calc at test_gpu_chisq.py's
    first-order bar 2 rho (E_MODEL + E_VEC / relgap);
  * scale_dyn: every output row against oracle.dynspec_oracle.scale_dyn_lambda in
    float64 on the same fp32-rounded input, within 1e-6 of the column's max |y|.
The run prints each family's worst error as a fraction of its bar."""
import math
import os
import sys
from collections import namedtuple

import numpy as np
import pytest

from oracle import dynspec_oracle as DO
from oracle import thth_oracle as TO

NF, NT, NPAD = 8, 32, 1
DT, DF, F0 = 10.0, 0.1, 1400.0
WIDE = np.linspace(-70.0, 95.0, 32)          # 31 centres, reaches past the fd axis
ORDINARY = np.linspace(-20.0, 20.0, 32)      # 31 centres, inside it
ETA_LO, ETA_HI = 3e-4, 8e-3                  # s^3
LAUNCH = 65535                               # gridDim.y cap
SPLIT = 30000                                # items per call of the comparison runs
N_MAX = 2 * LAUNCH + 1                       # 131071: three launches of the scan
N_SAMPLE = 200

RTOL = 1e-5
E_MODEL, E_VEC = 5e-5, 4e-6                  # test_gpu_chisq.py
SCALE_TOL = 1e-6

ItemCase = namedtuple("ItemCase", "entry count grid")
ITEM_CASES = [ItemCase("eta_sweep", n, "wide") for n in (LAUNCH, LAUNCH + 1, N_MAX)] + \
    [ItemCase("eta_sweep", LAUNCH + 1, "ordinary"),
     ItemCase("chisq_sweep", LAUNCH + 1, "wide"),
     ItemCase("thin_sweep", 256 * 256, "wide grid"),
     ItemCase("thin_sweep", N_MAX, "wide"),
     ItemCase("asymmetry", LAUNCH + 1, "mixed")]

ScaleCase = namedtuple("ScaleCase", "nf nt f_lo f_hi spacing")
SCALE_CASES = [ScaleCase(LAUNCH, 3, 1200.0, 1600.0, "auto"),
               ScaleCase(LAUNCH + 1, 3, 1200.0, 1600.0, "auto"),
               ScaleCase(12000, 3, 704.0, 4032.0, "min"),
               ScaleCase(3000, 257, 704.0, 4032.0, "min"),
               ScaleCase(4, 3, 1200.0, 1600.0, "auto")]


def item_id(c):
    return "%s-%d-%s" % (c.entry, c.count, c.grid.replace(" ", "_"))


def scale_id(c):
    return "nf%d-nt%d-%g-%g-%s" % c


# --------------------------------------------------------------------------
# geometry and oracle patterns (host only)
# --------------------------------------------------------------------------
def axes():
    t = DT * np.arange(NT)
    f = F0 + DF * np.arange(NF)
    return t, f, TO.fft_axis(f, "us", NPAD), TO.fft_axis(t, "mHz", NPAD)


def curvatures(n=N_MAX, seed=11):
    """A shuffled geometric set; every count of a case is a prefix of it."""
    return np.random.default_rng(seed).permutation(np.geomspace(ETA_LO, ETA_HI, N_MAX))[:n]


def lower_check_needed(edges):
    """thth.cu lower_check_needed: can any (i, j) reach fd_inv < -nfd?"""
    _, _, _, fd = axes()
    th = TO.theta_centres(edges)
    dfd = np.diff(fd).mean()
    worst = math.floor(((th.min() - th.max()) - fd[0] + dfd / 2) / dfd) - 2.0
    return not worst >= -fd.shape[0]


def index_errors(etas, edges):
    """Per curvature: does the oracle's thth_map raise IndexError?  The mask and the
    fd index do not depend on eta; the tau index is the oracle's own expression."""
    _, _, tau, fd = axes()
    th, _, fd_inv, _ = TO.thth_indices(tau, fd, 1.0, edges)
    n = th.shape[0]
    th1 = np.ones((n, n)) * th
    th2 = th1.T
    sel = fd_inv < -fd.shape[0]
    d = (th1 ** 2 - th2 ** 2)[sel]
    dtau = np.diff(tau).mean()
    ti = ((np.asarray(etas)[:, None] * d[None, :]) - tau[0] + dtau / 2) // dtau
    return ((ti > 0) & (ti < tau.shape[0])).any(axis=1)


def thin_index_errors(e1, e2, edges1, edges2):
    """Per pair: does the oracle's two_curve_map raise IndexError?"""
    _, _, tau, fd = axes()
    c1 = (edges1[1:] + edges1[:-1]) / 2
    c2 = (edges2[1:] + edges2[:-1]) / 2
    th1 = np.ones((c2.shape[0], c1.shape[0])) * c1
    th2 = np.ones((c2.shape[0], c1.shape[0])) * c2[:, np.newaxis]
    dtau = np.diff(tau).mean()
    dfd = np.diff(fd).mean()
    fd_inv = ((th1 - th2) - fd[1] + dfd / 2) // dfd
    sel = fd_inv < -fd.shape[0]
    a, b = (th1 ** 2)[sel], (th2 ** 2)[sel]
    ti = ((np.asarray(e1)[:, None] * a[None, :] - np.asarray(e2)[:, None] * b[None, :]) -
          tau[1] + dtau / 2) // dtau
    return ((ti > 0) & (ti < tau.shape[0] - 1)).any(axis=1)


def thin_pairs(case):
    if case.grid == "wide grid":                 # 256 x 256 grid of (etas, etasArclet)
        g = np.geomspace(ETA_LO, ETA_HI, 256)
        return np.repeat(g, 256), np.tile(g, 256)
    rng = np.random.default_rng(13)
    e = np.geomspace(ETA_LO, ETA_HI, N_MAX)
    return rng.permutation(e), rng.permutation(e)


def samples(n, k=N_SAMPLE, seed=3):
    """The first and last four items, the four on each side of every 65535 boundary,
    then random items up to k."""
    s = set(range(4)) | set(range(n - 4, n))
    for b in range(LAUNCH, n, LAUNCH):
        s |= set(range(b - 4, min(b + 4, n)))
    rng = np.random.default_rng(seed)
    while len(s) < k:
        s.add(int(rng.integers(n)))
    return np.array(sorted(s))


def scale_input(c, desc, seed=17):
    """fp32-rounded input and its frequencies, ascending or descending."""
    rng = np.random.default_rng(seed)
    dyn = rng.exponential(1.0, (c.nf, c.nt)).astype(np.float32).astype(np.float64)
    f = np.linspace(c.f_lo, c.f_hi, c.nf)
    return (dyn[::-1].copy(), f[::-1].copy()) if desc else (dyn, f)


def scale_rows(c):
    """Output rows of Dynspec.scale_dyn (the reference's axis code)."""
    return DO.scale_dyn_lambda(np.zeros((c.nf, 1)), np.linspace(c.f_lo, c.f_hi, c.nf),
                               c.spacing)[0].shape[0]


# --------------------------------------------------------------------------
# tests without a GPU
# --------------------------------------------------------------------------
def test_item_case_table():
    """Each entry point keeps a case past 65,535 items; the sweep also keeps 65,535 and
    a count needing three scan launches; the batch caps see a second batch."""
    by = {}
    for c in ITEM_CASES:
        by.setdefault(c.entry, set()).add(c.count)
    assert set(by) == {"eta_sweep", "chisq_sweep", "thin_sweep", "asymmetry"}
    assert {LAUNCH, LAUNCH + 1} <= by["eta_sweep"] and math.ceil(max(by["eta_sweep"]) / LAUNCH) == 3
    for entry in ("chisq_sweep", "thin_sweep", "asymmetry"):
        assert max(by[entry]) > LAUNCH, entry
    assert 256 * 256 in by["thin_sweep"] and N_MAX in by["thin_sweep"]
    assert any(c.grid == "ordinary" and c.count > LAUNCH for c in ITEM_CASES)
    assert len({item_id(c) for c in ITEM_CASES}) == len(ITEM_CASES)
    # the per-item workspaces of chisq_sweep and asymmetry_batch (retrieval.cu) fit more
    # than 65535 items in the 3 GiB slab, so the 65535 cap is what splits the batch
    _, _, tau, fd = axes()
    ld, bins, slots = 32, tau.shape[0] * fd.shape[0], 64
    mat, qn = ld * ld, (ld + 1) * ld
    chisq = (mat + qn + ld + bins) * 8 + slots * 8 + bins * 4 + bins * 8
    asym = (mat + qn + ld) * 8
    assert (3 << 30) // chisq > LAUNCH and (3 << 30) // asym > LAUNCH


def test_geometry_and_index_error_mix():
    """WIDE needs the IndexError scan and ORDINARY does not; under WIDE every launch
    of <= 65535 curvatures (or pairs) holds curvatures that raise and ones that do
    not; no curvature crops below 3 centres."""
    assert lower_check_needed(WIDE) and not lower_check_needed(ORDINARY)
    _, _, tau, fd = axes()
    etas = curvatures()
    err = index_errors(etas, WIDE)
    assert not index_errors(etas, ORDINARY).any()
    for b in range(0, N_MAX, LAUNCH):
        blk = err[b:b + LAUNCH]
        assert blk.size == 1 or (blk.any() and not blk.all()), b
    for c in ITEM_CASES:
        if c.entry == "thin_sweep":
            e1, e2 = thin_pairs(c)
            assert e1.shape[0] == c.count
            terr = thin_index_errors(e1, e2, WIDE, WIDE)
            for b in range(0, c.count, LAUNCH):
                blk = terr[b:b + LAUNCH]
                assert blk.size == 1 or (blk.any() and not blk.all()), (c, b)
    for e in (ETA_LO, ETA_HI):
        for g in (WIDE, ORDINARY):
            assert TO.th_points(tau, fd, e, g).sum() >= 3


def test_index_error_patterns_match_oracle():
    """index_errors / thin_index_errors equal the oracle's own try/except, on random
    curvatures and on the ones next to the switch from raising to not raising."""
    _, _, tau, fd = axes()
    zero = np.zeros((tau.shape[0], fd.shape[0]), dtype=complex)
    etas = np.sort(curvatures())
    err = index_errors(etas, WIDE)
    k = int(np.flatnonzero(err[:-1] != err[1:])[0])
    pick = np.unique(np.concatenate([np.arange(k - 20, k + 20),
                                     np.random.default_rng(1).integers(0, N_MAX, 150)]))
    for eta, want in zip(etas[pick], err[pick]):
        try:
            TO.thth_map(zero, tau, fd, eta, WIDE)
            raised = False
        except IndexError:
            raised = True
        assert raised == want, eta
    e1, e2 = thin_pairs(ITEM_CASES[-2])
    terr = thin_index_errors(e1, e2, WIDE, WIDE)
    assert terr.any() and not terr.all()
    for j in np.random.default_rng(2).integers(0, N_MAX, 200):
        try:
            TO.two_curve_map(zero, tau, fd, e1[j], WIDE, e2[j], WIDE)
            raised = False
        except IndexError:
            raised = True
        assert raised == terr[j], j


def test_samples_cover_boundaries():
    for n in {c.count for c in ITEM_CASES}:
        s = set(samples(n))
        assert len(s) >= N_SAMPLE and {0, n - 1} <= s and max(s) == n - 1
        for b in range(LAUNCH, n, LAUNCH):
            assert set(range(b - 4, min(b + 4, n))) <= s, (n, b)


def test_scale_case_table():
    """Output rows of 65,535, 65,536 and 68,717 (with 'min' spacing on 704-4032 MHz),
    the 4-channel minimum, and nt = 257, one past the 128- and 256-thread blocks."""
    rows = {c: scale_rows(c) for c in SCALE_CASES}
    assert LAUNCH in rows.values() and LAUNCH + 1 in rows.values()
    wide = [r for c, r in rows.items() if c.spacing == "min" and c.nt == 3]
    assert wide and max(wide) > LAUNCH + 1 and max(wide) == 68717
    assert min(c.nf for c in SCALE_CASES) == 4
    assert any(c.nt % 256 == 1 and c.nt > 256 and c.nf >= 1000 for c in SCALE_CASES)


def test_wideband_fixture_pins_oracle(golden_dir):
    """oracle scale_dyn_lambda reproduces the unmodified reference's scale_dyn with
    'min' spacing on a 64-channel 704-4032 MHz band, ascending and descending
    (tests/golden/scale_dyn_wideband.npz, made by oracle/make_golden_lambda.py)."""
    g = np.load(os.path.join(golden_dir, "scale_dyn_wideband.npz"))
    for tag, sl in (("asc", slice(None)), ("desc", slice(None, None, -1))):
        lamdyn, lam, dlam = DO.scale_dyn_lambda(g["dyn"][sl], g[tag + "_freqs"], "min")
        ref = g[tag + "_lamdyn"]
        assert lamdyn.shape == ref.shape and ref.shape[0] > 5 * g["dyn"].shape[0]
        assert np.array_equal(lam, g[tag + "_lam"]) and dlam == float(g[tag + "_dlam"])
        assert np.abs(lamdyn - ref).max() <= 1e-12 * np.abs(ref).max()


# --------------------------------------------------------------------------
# GPU: shared input and references
# --------------------------------------------------------------------------
WORST = {}


def report(family, frac):
    WORST[family] = max(WORST.get(family, 0.0), float(frac))
    assert frac <= 1.0, (family, frac)


def synthetic_dynspec(seed=5):
    """A 12-image arc (eta 4e-3 s^3) with 10 % noise, mean removed."""
    rng = np.random.default_rng(seed)
    t, f, _, _ = axes()
    fdk = rng.uniform(-20.0, 20.0, 12)
    ak = (rng.normal(size=12) + 1j * rng.normal(size=12)) * np.exp(-(fdk / 15.0) ** 2)
    E = sum(a * np.exp(2j * np.pi * (x * 1e-3 * t[None, :] - 4e-3 * x ** 2 * (f[:, None] - F0)))
            for a, x in zip(ak, fdk))
    dyn = np.abs(E) ** 2
    dyn += rng.normal(0.0, 0.1 * dyn.mean(), dyn.shape)
    return dyn - dyn.mean()


@pytest.fixture(scope="module")
def sb():
    import scintools_b200
    from scintools_b200 import _device
    _device.device()
    return scintools_b200


@pytest.fixture(scope="module")
def data(sb):
    dyn = synthetic_dynspec()
    cs = sb.ththmod.conjugate_spectrum(dyn, NPAD, None)
    t, f, tau, fd = axes()
    yield dict(dyn=dyn, cs=cs, CS=cs.numpy(), t=t, f=f, tau=tau, fd=fd, cache={})
    if WORST:
        print("\nitem counts: worst error per family, as a fraction of its bar")
        for k in sorted(WORST):
            print("  %-28s %.3g" % (k, WORST[k]))
        sys.stdout.flush()


def split_calls(fn, n, *arrays):
    """fn over consecutive slices of at most SPLIT items, outputs concatenated."""
    outs = [fn(*[a[s:s + SPLIT] for a in arrays]) for s in range(0, n, SPLIT)]
    vals = np.concatenate([o[0] for o in outs])
    info = {k: np.concatenate([o[1][k] for o in outs]) for k in outs[0][1]}
    return vals, info


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def sweep_ref(th, data, grid, etas):
    key = ("sweep", grid)
    if key not in data["cache"]:
        edges = WIDE if grid == "wide" else ORDINARY
        data["cache"][key] = split_calls(
            lambda e: th.eta_sweep(data["cs"], data["tau"], data["fd"], e, edges,
                                   return_info=True), etas.shape[0], etas)
    return data["cache"][key]


# --------------------------------------------------------------------------
# a. eta_sweep (sb_eta_sweep: thth_prep's IndexError scan)
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in ITEM_CASES if c.entry == "eta_sweep"], ids=item_id)
def test_eta_sweep(sb, data, case):
    th = sb.ththmod
    edges = WIDE if case.grid == "wide" else ORDINARY
    etas = curvatures(case.count)
    got, info = th.eta_sweep(data["cs"], data["tau"], data["fd"], etas, edges, return_info=True)
    n = case.count
    ref, rinfo = sweep_ref(th, data, case.grid, curvatures(N_MAX if case.grid == "wide" else n))
    assert same_bits(got, ref[:n])
    for k in ("status", "nred", "iters"):
        assert same_bits(info[k], rinfo[k][:n]), k
    err = index_errors(etas, edges)
    assert np.array_equal((info["status"] & 1) != 0, err)
    assert np.array_equal(np.isnan(got), err) and (info["status"] & ~1 == 0).all()
    if case.grid == "ordinary":
        assert not err.any()
    for k in samples(n):
        if err[k]:
            continue
        key = ("eval", case.grid, k)        # the counts share their prefixes
        if key not in data["cache"]:
            data["cache"][key] = TO.Eval_calc(data["CS"], data["tau"], data["fd"], etas[k], edges)
        r = data["cache"][key]
        report("eta_sweep", abs(got[k] - r) / r / RTOL)
    assert (~err[samples(n)]).sum() >= 50


# --------------------------------------------------------------------------
# b. chisq_sweep (thth_prep, then batches of <= 65535)
# --------------------------------------------------------------------------
@pytest.mark.gpu
def test_chisq_sweep_65536(sb, data):
    from oracle import chisq_oracle as CO
    th = sb.ththmod
    n = LAUNCH + 1
    etas = curvatures(n)
    dyn, N = data["dyn"], 1.0

    def run(e):
        return th.chisq_sweep(dyn, data["cs"], data["tau"], data["fd"], e, WIDE, N,
                              return_info=True)

    got, info = run(etas)
    ref, rinfo = split_calls(run, n, etas)
    for k in ("w", "status", "nred", "iters"):
        assert same_bits(info[k], rinfo[k]), k
    err = index_errors(etas, WIDE)
    assert np.array_equal((info["status"] & 1) != 0, err) and (info["status"] & ~1 == 0).all()
    assert np.array_equal(np.isnan(got), err) and np.array_equal(np.isnan(ref), err)
    ok = ~err
    assert (np.abs(got[ok] - ref[ok]) <= 1e-6 * np.abs(ref[ok])).all()
    for k in samples(n):
        if err[k]:
            continue
        r = CO.chisq_calc(dyn, data["CS"], data["tau"], data["fd"], etas[k], WIDE, N)
        out = TO.modeler(data["CS"], data["tau"], data["fd"], etas[k], WIDE)
        wv = np.linalg.eigvalsh(out[0])
        model = out[3][:NF, :NT]
        rho = np.sqrt(np.sum(model ** 2) / np.sum((model - dyn) ** 2))
        bar = 2 * rho * (E_MODEL + E_VEC / ((wv[-1] - wv[-2]) / abs(wv[-1])))
        report("chisq_sweep", abs(got[k] - r) / r / bar)


# --------------------------------------------------------------------------
# c. thin_sweep (the IndexError scan over curvature pairs)
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in ITEM_CASES if c.entry == "thin_sweep"], ids=item_id)
def test_thin_sweep(sb, data, case):
    th = sb.ththmod
    e1, e2 = thin_pairs(case)
    n = case.count

    def run(a, b):
        return th.thin_sweep(data["cs"], data["tau"], data["fd"], a, WIDE, WIDE, 0.0,
                             etasArclet=b, return_info=True)

    got, info = run(e1, e2)
    ref, rinfo = split_calls(run, n, e1, e2)
    assert same_bits(got, ref)
    for k in ("status", "n1", "n2", "iters"):
        assert same_bits(info[k], rinfo[k]), k
    err = thin_index_errors(e1, e2, WIDE, WIDE)
    assert np.array_equal((info["status"] & 1) != 0, err) and (info["status"] & ~1 == 0).all()
    assert np.array_equal(np.isnan(got), err)
    for k in samples(n):
        if err[k]:
            continue
        r = TO.singularvalue_calc(data["CS"], data["tau"], data["fd"], e1[k], WIDE, e2[k],
                                  WIDE, 0.0)
        report("thin_sweep", abs(got[k] - r) / r / RTOL)


# --------------------------------------------------------------------------
# d. asymmetry_batch (thth_prep_table's scan, then batches of <= 65535)
# --------------------------------------------------------------------------
@pytest.mark.gpu
def test_asymmetry_batch_65536(sb, data):
    """65536 chunk geometries through sb_asymmetry_batch: three spectra, both grids and
    five curvatures in a non-periodic order.  Sampled chunks are bit-identical to
    single-chunk calls; the IndexError status of every chunk is the oracle's."""
    import torch
    from scintools_b200 import _device as D, _lib
    th = sb.ththmod
    n = LAUNCH + 1
    tau, fd = data["tau"], data["fd"]
    grids = (WIDE, ORDINARY)
    etas5 = np.array([5e-4, 1.2e-3, 2.5e-3, 4e-3, 6e-3])
    geoms = []
    for s in range(3):
        cs = th.conjugate_spectrum(synthetic_dynspec(seed=20 + s), NPAD, None)
        geoms.append([th._Geom(cs, tau, fd, g, True) for g in grids])
    rng = np.random.default_rng(29)
    si, gi, ei = rng.integers(0, 3, n), rng.integers(0, 2, n), rng.integers(0, 5, n)
    table = (_lib.ThthGeom * n)(*[geoms[a][b].g for a, b in zip(si, gi)])
    etas = etas5[ei]

    def call(tab, m, e):
        d_etas = D.upload(np.ascontiguousarray(e))
        o = [D.empty((m,), torch.float64) for _ in range(2)] + \
            [D.empty((m,), torch.int32) for _ in range(3)]
        _lib.check(_lib.lib.sb_asymmetry_batch(tab, m, d_etas.data_ptr(), 0.0, 0,
                                               *[x.data_ptr() for x in o], None,
                                               D.stream_ptr()))
        return [x.cpu().numpy() for x in o]

    asym, w, status, nred, iters = call(table, n, etas)
    err = np.zeros(n, bool)
    wide = gi == 0
    err[wide] = index_errors(etas[wide], WIDE)
    assert err.any() and not err.all()
    assert np.array_equal((status & 1) != 0, err)
    assert np.array_equal(np.isnan(asym[err]), np.ones(err.sum(), bool))
    assert np.isfinite(asym[~err & (status == 0)]).mean() > 0.9
    pick = set(range(LAUNCH - 4, n)) | set(range(4)) | \
        set(np.random.default_rng(4).integers(0, n, 40).tolist())
    for k in sorted(pick):
        one = call((_lib.ThthGeom * 1)(geoms[si[k]][gi[k]].g), 1, etas[k:k + 1])
        for a, b, name in zip((asym, w, status, nred, iters), one,
                              ("asym", "w", "status", "nred", "iters")):
            assert same_bits(a[k:k + 1], b), (k, name)


# --------------------------------------------------------------------------
# e. Dynspec.scale_dyn (spline_eval_kernel rows)
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("desc", [False, True], ids=["asc", "desc"])
@pytest.mark.parametrize("case", SCALE_CASES, ids=scale_id)
def test_scale_dyn(sb, case, desc):
    dyn, f = scale_input(case, desc)
    ds = sb.Dynspec(dyn=sb.BasicDyn(dyn, times=DT * np.arange(case.nt), freqs=f, dt=DT,
                                    df=float(f[1] - f[0])), verbose=False)
    ds.scale_dyn(scale="lambda", spacing=case.spacing)
    ref, lam, dlam = DO.scale_dyn_lambda(dyn, f, case.spacing)
    assert ds.lamdyn.shape == ref.shape == (scale_rows(case), case.nt)
    assert np.array_equal(ds.lam, lam) and ds.dlam == dlam
    scale = np.abs(dyn).max(axis=0)
    report("scale_dyn", (np.abs(ds.lamdyn - ref) / scale).max() / SCALE_TOL)


@pytest.mark.gpu
def test_scale_dyn_three_channels_refused(sb):
    """A cubic spline needs 4 knots: 3 channels raise, naming the minimum; the library
    keeps working."""
    from scintools_b200 import _lib
    c = ScaleCase(3, 3, 1200.0, 1600.0, "auto")
    dyn, f = scale_input(c, False)
    ds = sb.Dynspec(dyn=sb.BasicDyn(dyn, times=DT * np.arange(3), freqs=f, dt=DT,
                                    df=float(f[1] - f[0])), verbose=False)
    with pytest.raises(_lib.SbError, match="at least 4 channels"):
        ds.scale_dyn(scale="lambda")
    c = SCALE_CASES[-1]
    dyn, f = scale_input(c, False)
    ds = sb.Dynspec(dyn=sb.BasicDyn(dyn, times=DT * np.arange(3), freqs=f, dt=DT,
                                    df=float(f[1] - f[0])), verbose=False)
    ds.scale_dyn(scale="lambda")
    ref = DO.scale_dyn_lambda(dyn, f)[0]
    assert np.abs(ds.lamdyn - ref).max() <= SCALE_TOL * np.abs(dyn).max()
