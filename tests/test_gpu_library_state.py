"""The library's process-wide state: its streams and its workspace.

Every entry point shares state across calls: the nine grow-only workspace slots
(csrc/common.cuh), the twiddle tables cached per length (csrc/dynspec.cu), the theta-theta
column cache (csrc/thth.cu) and the ScalarBlock accumulators.  These tests check that a
result does not depend on that state.

A. Streams.  Each entry point takes a caller stream.  The library orders a call after the
   previous call whenever the stream changes (StreamFence, csrc/api.cu), because the
   workspace and the twiddle tables belong to the process, not to a stream.
   * test_twiddle_race: in a fresh process (where no table memory has held twiddles
     before), the first call of an FFT length is queued behind 0.1 s of other work on
     stream A, and a second call of the same length goes straight to stream B.  Without
     the ordering, B reads A's twiddle table before A's fill has run.  Only FFT entry
     points without index tables run here, so such a race gives wrong values, never wrong
     addresses.
   * test_overlapping_calls: two large calls back to back on two streams each give their
     default-stream result.  Without the ordering they share the workspace planes at the
     same time; whether that shows depends on how the kernels interleave, so this test is
     likely, not certain, to catch it.
   * test_side_stream: every case of the table below under torch.cuda.stream(s).
B. Workspace state.  CASES covers every public entry point at a small and a larger shape,
   each checked against its float64 oracle at the bar of that entry point's own test (the
   checks are those tests' functions).  Each case runs
   * cold: after sb_release();
   * after others: after every case ran at its larger shape, so every slot has been
     regrown and holds another driver's data;
   * small, large, small: the two small results agree.
   Entry points documented as deterministic (mosaic, scint_fit, svd_topk / correct_dyn,
   refill) must be bit-identical across states; the others, whose float atomics (the dyn
   statistics, cut_dyn's tile sums, rev_map, chisq) make the last bits order-dependent,
   are held to their oracle bar.  test_case_table_coverage (no GPU) fails if an entry
   point of include/scint_b200.h has no case.
"""
import contextlib
import importlib
import os
import re
import subprocess
import sys
from collections import namedtuple

import numpy as np
import pytest

from oracle import dynspec_oracle as DO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "scint_b200.h")
GOLDEN = os.path.join(ROOT, "tests", "golden")

# entry points that hold no library state a call could see
STATELESS = {"sb_abi_version", "sb_last_error", "sb_init", "sb_release", "sb_launch_count",
             "sb_profile_enable", "sb_profile_collect", "sb_convert_f64_f32",
             "sb_convert_f32_f64"}

SLEEP_CYCLES = 200_000_000      # torch.cuda._sleep: about 0.1 s at the H100's 1.98 GHz
AGREE = 1e-5                    # non-deterministic repeats: max-norm relative difference


def _m(name):
    """A sibling test module (imported on use: the table itself needs no device)."""
    return importlib.import_module(name)


def _sb():
    import scintools_b200
    from scintools_b200 import _device
    _device.device()
    return scintools_b200


def header_entry_points():
    with open(HEADER) as f:
        text = f.read()
    return sorted(set(re.findall(r"^[\w ]+\*?\s*\b(sb_\w+)\(", text, re.M)))


# --------------------------------------------------------------------------
# table B: one case per entry point family, each run(size) checks against its oracle and
# returns its outputs
# --------------------------------------------------------------------------
Case = namedtuple("Case", "name symbols deterministic run")


def _arrays(got):
    return list(got) if isinstance(got, tuple) else [got]


def _p(entry, **p):
    return (entry, p)


def _fftc(name, symbol, small, large):
    def wrap(spec):
        return lambda FL: FL._c(spec[0], **spec[1])
    s, l_ = wrap(small), wrap(large)

    def run(size):
        FL = _m("test_gpu_fft_lengths")
        c = (s if size == "small" else l_)(FL)
        inputs, device, check = FL.ENTRIES[c.entry]
        x = inputs(c)
        got = device(c, x)
        check(c, x, got)
        return _arrays(got)
    return Case(name, (symbol,), False, run)


def run_thth(size):
    """eta_sweep, Eval_calc, thth_map, thth_redmap, thin_sweep, rev_map, modeler and
    chisq_sweep through test_gpu_cs_layouts.py's checks, and two_curve_map (sb_thin_map)
    against the oracle's entries at the bar of thth_map's."""
    from oracle import thth_oracle as TO
    CL = _m("test_gpu_cs_layouts")
    sb = _sb()
    c = CL._c("half", 32, 128, 1, 65) if size == "small" else CL._c("chirp", 43, 101, 2, 33)

    def made(case):
        return CL.make_cs(sb, case)
    CL.test_sweep_and_maps(sb, made, c, None)
    CL.test_thin_modeler_rev_map_chisq(sb, made, c)
    cs, CS, _ = made(c)
    _, _, tau, fd = CL.axes(c.nf, c.nt, c.npad)
    edges, e2 = CL.grid(c.n), CL.grid(c.n // 2 + 1)
    got = sb.ththmod.two_curve_map(cs, tau, fd, CL.ETA_ARC, edges, CL.ETA_ARC, e2)[0]
    ref = TO.two_curve_map(CS, tau, fd, CL.ETA_ARC, edges, CL.ETA_ARC, e2)[0]
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-6 * np.abs(ref).max()
    eigs = sb.ththmod.eta_sweep(cs, tau, fd, CL.etas_of(c), edges)
    return [eigs, got]


def run_c2c(size):
    """The complex-visibility spectrum (sb_cs_c2c_f32) and the sweep on it."""
    CL = _m("test_gpu_cs_layouts")
    sb = _sb()
    c = CL._c("c2c", 127, 301, 0, 33) if size == "small" else CL._c("c2c", 43, 101, 2, 129, 8)
    CL.test_sweep_and_maps(sb, lambda case: CL.make_cs(sb, case), c, None)
    cs, _, _ = CL.make_cs(sb, c)
    _, _, tau, fd = CL.axes(c.nf, c.nt, c.npad)
    return [sb.ththmod.eta_sweep(cs, tau, fd, CL.etas_of(c), CL.grid(c.n))]


def run_vlbi(size):
    """VLBI_chunk_retrieval on the reference's fixtures: c, one station; a, three."""
    VL = _m("test_gpu_vlbi")
    from scintools_b200 import ththmod
    tag = "c" if size == "small" else "a"
    VL.test_vlbi_matches_reference(ththmod, GOLDEN, tag)
    f = VL._load(GOLDEN, tag)
    n_dish = int(f["n_dish"])
    p = VL._params(f, VL._inputs(f), n_dish)
    _, w, _, _, _ = ththmod._vlbi_run(p[0], p[1], p[2], p[3], p[4], p[7], n_dish, p[9])
    return [np.array([w])]


class _NoCapture:
    @staticmethod
    def disabled():
        return contextlib.nullcontext()


def run_asymmetry(size):
    """calc_asymmetry on the reference's fixture within its bound, and one chunk against the
    batch (a fixed shape: the fixture's)."""
    AS = _m("test_gpu_asymmetry")
    from scintools_b200 import ththmod
    f = np.load(os.path.join(GOLDEN, "asymmetry_sample.npz"))
    AS.test_case_a_within_bound(f, _NoCapture())
    if size == "large":
        AS.test_single_call_matches_batch(f)
    pars = AS.make_dynspec(f)._asymmetry_params()
    return [np.array([r[0] for r in ththmod.asymmetry_batch(pars)])]


def run_mosaic(size):
    MS = _m("test_gpu_mosaic")
    from scintools_b200 import ththmod as T
    name = "mosaic_sample" if size == "small" else "mosaic_synth"
    MS.test_mosaic_functions_against_oracle(GOLDEN, name, "")
    c = MS._case(GOLDEN, name, "")
    ch, x, p, D, N = c["chunks"], c["x"], c["p"], c["dspec"], c["N"]
    nF, nT = c["fullMos"].shape
    return [T.rotMos(ch, x), T.fullMos(ch, p), np.array([T.rotFit(x, ch)]), T.rotDer(x, ch),
            np.array([T.fullMosFit(p, ch, D, N)]), T.fullMosGrad(p, ch, D[:nF, :nT], N),
            T.fullMosHess(p, ch, D[:nF, :nT], N), T.rotInit(ch)]


def run_correct_dyn(size):
    """svd_model against prescribed factors (test_gpu_correct_dyn.py) and the svd=False
    passes of correct_dyn against the oracle."""
    CR = _m("test_gpu_correct_dyn")
    from scintools_b200 import ththmod
    nf, nt = (37, 1001) if size == "small" else (1024, 2048)
    A, M, s = CR.prescribed(nf, nt, 3, seed=nf + nt + 3)
    m, info = ththmod.svd_model(A, 3, return_info=True)
    assert info["converged"] and not info["tie"], info
    EM, _ = CR.model_bound(A, 3, info["residuals"], s)
    CR.check_model(m, M, EM)
    CR._check_svals(info, s, A)
    dyn = CR.structured_dyn(12, nf // 2 + 40, nt // 2 + 50)
    ds = CR._dynspec(dyn.copy())
    ds.correct_dyn(svd=False, nsmooth=7)
    ref = CR.types_ns(dyn)
    CR.CO.correct_dyn(ref, svd=False, nsmooth=7)
    x = np.where(np.nan_to_num(dyn) == 0, np.nan, np.nan_to_num(dyn))
    CR.check_bandpass_result(ds.dyn, ref.dyn, dict(frequency=True, time=True, nsmooth=7), x)
    return [m, info["s"], info["residuals"], ds.dyn, ds.bandpass]


def run_refill(size):
    """The biharmonic fill against spsolve and the masked median against medfilt."""
    RF = _m("test_gpu_refill")
    shape = (96, 128) if size == "small" else (192, 320)
    rng = np.random.default_rng(5)
    mask = rng.random(shape) < 0.05
    mask[shape[0] // 3:shape[0] // 3 + 12, 40:52] = True
    img = rng.exponential(1.0, shape)
    img[mask] = np.nan
    ref = RF.O.biharmonic(img, mask)
    got, info = RF._inpaint(img, mask)
    known = img[~mask]
    assert info["converged"] and info["residual"] <= 1e-10
    assert np.max(np.abs(got - ref)) / (known.max() - known.min()) <= RF.BAR
    dyn = rng.exponential(1.0, (shape[0] // 2, shape[1] // 2))
    dyn[rng.random(dyn.shape) < 0.1] = np.nan
    med = RF.O.refill(dyn, method="median", kernel_size=5)
    ds = RF._ds(dyn.copy())
    ds.refill(method="median", kernel_size=5)
    assert np.array_equal(ds.dyn, med)
    return [got, ds.dyn]


def run_scint_fit(size):
    """get_scint_params against the reference's fixtures, acf1d and acf2d_approx."""
    SP = _m("test_gpu_scint_params")
    fns = [fn for fn in SP.FIXTURES if "crafted" not in fn]
    fn = fns[0] if size == "small" else fns[-1]
    for f_, c in SP.CASES:
        if f_ == fn:
            SP.test_fixture_parity(fn, c)
    z = np.load(fn)
    out = []
    for method in ("acf1d", "acf2d_approx"):
        out += SP._fits(method, [SP._ds(z, "acf1d")])
    return out


def run_acf_model(size):
    """scint_sim.ACF against the float64 oracle at the bars of test_gpu_acf_model.py."""
    AM = _m("test_gpu_acf_model")
    kw = AM._random_kwargs(np.random.default_rng(1003))
    kw.update(nf=4, nt=5) if size == "small" else kw.update(nf=15, nt=23)
    a = AM._acf(**kw)
    _, ref, ref_ef = AM.AO.model(**kw)
    assert a.acf.shape == ref.shape
    assert np.max(np.abs(a.acf - ref)) <= 1e-12 * kw["amp"]
    assert np.max(np.abs(a.acf_efield - ref_ef)) <= 1e-14
    return [a.acf, a.acf_efield]


def run_sim(size):
    """Simulation with explicit noise against the oracle (test_gpu_sim.py's bars)."""
    from oracle import sim_oracle as SO
    from scintools_b200.scint_sim import Simulation
    SM = _m("test_gpu_sim")
    _sb()
    nx, ny, nf = (64, 128, 3) if size == "small" else (256, 512, 5)
    rng = np.random.default_rng(42)
    n1, n2 = rng.normal(size=(nx, ny)), rng.normal(size=(nx, ny))
    kw = dict(mb2=8, ar=1.3, psi=15, nx=nx, ny=ny, nf=nf, dlam=0.2, inner=0.002)
    ref = SO.SimOracle(noise_re=n1, noise_im=n2, **kw)
    got = Simulation(noise=(n1, n2), **kw)
    assert SM.maxrel(got.w, ref.w) < 1e-12
    assert SM.maxrel(got.xyp, ref.xyp) < 1e-10
    for k in ("spe", "xyi", "dyn"):
        assert SM.maxrel(getattr(got, k), getattr(ref, k)) < SM.RTOL, k
    return [got.w, got.xyp, got.dyn]


def run_slow_ft(size):
    from oracle import slow_ft_oracle as SFO
    SF = _m("test_gpu_slow_ft")
    nt, nf = (300, 20) if size == "small" else (3000, 70)
    rng = np.random.default_rng(nt + nf)
    x = rng.normal(size=(nt, nf))
    freqs = np.linspace(1300.0, 1500.0, nf)
    got = SF._slow_ft(x, freqs)
    SF._check(got, SFO.bluestein(x.astype(np.float32), freqs), "slow_ft %dx%d" % (nt, nf))
    return [got]


def run_scale_dyn(size):
    """scale_dyn(scale='lambda') against the reference's fixture (one shape: the fixture's)."""
    PA = _m("test_gpu_parity")
    PA.test_scale_dyn_lambda(_sb(), GOLDEN, None)
    return []


def run_norm_sspec(size):
    """norm_sspec rows and their average: the reference's fixture (small) and random
    geometries against numpy (large)."""
    AF = _m("test_gpu_arcfit")
    if size == "small":
        AF.test_norm_sspec_kernels_vs_reference(_sb(), GOLDEN)
    else:
        AF.test_norm_rows_random_geometry(_sb())
    return []


def run_cut_dyn(size):
    """cut_dyn tile by tile against calc_sspec / calc_acf (test_gpu_cut_dyn.py)."""
    CD = _m("test_gpu_cut_dyn")
    shape, tcuts, fcuts = ((101, 152), 2, 1) if size == "small" else ((200, 300), 4, 2)
    sb = _sb()
    ds = CD._ds(sb, np.random.default_rng(sum(shape)).exponential(1.0, shape))
    ds.cut_dyn(tcuts=tcuts, fcuts=fcuts)
    CD._check_tiles_vs_drivers(ds)
    return [ds.cutsspec, ds.cutacf]


CASES = [
    _fftc("sspec", "sb_sspec_f32",
          _p("sspec", nf=50, nt=120, window=True, halve=1, prewhite=0),
          _p("sspec", nf=300, nt=1000, window=True, halve=1, prewhite=0)),
    _fftc("acf", "sb_acf_f32",
          _p("acf", nf=50, nt=120, normalise=1), _p("acf", nf=300, nt=1000, normalise=1)),
    _fftc("acf_sspec", "sb_acf_sspec_f32",
          _p("acf_sspec", nf=50, nt=120, window=True, normalise=1),
          _p("acf_sspec", nf=300, nt=1000, window=True, normalise=1)),
    _fftc("cs", "sb_cs_f32",
          _p("cs", nf=32, nt=64, npad=1, pad=None, half=True, keep=0, mask=True),
          _p("cs", nf=128, nt=512, npad=1, pad=None, half=True, keep=0, mask=True)),
    _fftc("cs_chirp", "sb_cs_f32",
          _p("cs", nf=43, nt=101, npad=0, pad=0.375, half=False, keep=0, mask=False),
          _p("cs", nf=200, nt=301, npad=1, pad=0.375, half=False, keep=0, mask=False)),
    _fftc("ifft2", "sb_ifft2_c2c_f32",
          _p("ifft2", n0=64, n1=128, centred=1, crop0=0, crop1=0, real=False),
          _p("ifft2", n0=300, n1=500, centred=1, crop0=200, crop1=0, real=True)),
    _fftc("gerchberg_saxton", "sb_gerchberg_saxton_f32",
          _p("gs", n0=64, n1=128), _p("gs", n0=512, n1=1024)),
    _fftc("sim_screen", "sb_sim_screen",
          _p("screen", nx=64, ny=128), _p("screen", nx=512, ny=512)),
    _fftc("sim_intensity", "sb_sim_intensity",
          _p("intensity", nx=64, ny=64, nf=3), _p("intensity", nx=256, ny=256, nf=4)),
    Case("thth", ("sb_cs_f32", "sb_cs_bound_f32", "sb_eta_sweep", "sb_thth_map",
                  "sb_thin_sweep", "sb_thin_map", "sb_rev_map", "sb_herm_eigvec",
                  "sb_ifft2_c2c_f32", "sb_chisq_sweep"), False, run_thth),
    Case("cs_c2c", ("sb_cs_c2c_f32", "sb_eta_sweep", "sb_thth_map"), False, run_c2c),
    Case("vlbi", ("sb_cs_c2c_f32", "sb_vlbi_retrieval"), False, run_vlbi),
    Case("asymmetry", ("sb_cs_f32", "sb_cs_bound_f32", "sb_asymmetry_batch"), False,
         run_asymmetry),
    Case("mosaic", ("sb_mosaic_build", "sb_mosaic_rot", "sb_mosaic_overlap", "sb_mosaic_fit",
                    "sb_mosaic_hess"), True, run_mosaic),
    Case("correct_dyn", ("sb_svd_topk", "sb_svd_apply", "sb_bandpass_rows", "sb_bandpass_cols",
                         "sb_bandpass_divide"), True, run_correct_dyn),
    Case("refill", ("sb_inpaint_biharmonic_f64", "sb_medfilt_masked_f64"), True, run_refill),
    Case("scint_fit", ("sb_scint_fit_1d", "sb_scint_fit_2d", "sb_acf_f32"), True, run_scint_fit),
    Case("acf_model", ("sb_acf_model_f64",), False, run_acf_model),
    Case("simulation", ("sb_sim_weights", "sb_sim_screen", "sb_sim_intensity"), False, run_sim),
    Case("slow_ft", ("sb_slow_ft_f32",), False, run_slow_ft),
    Case("scale_dyn", ("sb_scale_dyn_lambda_f32", "sb_sspec_f32"), False, run_scale_dyn),
    Case("norm_sspec", ("sb_norm_sspec_f32", "sb_norm_sspec_avg_f32"), False, run_norm_sspec),
    Case("cut_dyn", ("sb_sspec_tiles_f32", "sb_acf_tiles_f32"), False, run_cut_dyn),
]
NAMES = [c.name for c in CASES]


def test_case_table_coverage():
    """Every entry point of the header that touches library state has a case, and every
    symbol a case names is one of them."""
    want = set(header_entry_points()) - STATELESS
    have = set().union(*(c.symbols for c in CASES))
    assert sorted(want - have) == []
    assert sorted(have - want) == []
    assert len(set(NAMES)) == len(NAMES)
    from_lib = {"sb_" + s for s in re.findall(r'"sb_(\w+)"', open(
        os.path.join(ROOT, "scintools_b200", "_lib.py")).read())}
    assert want <= from_lib


def same(case, a, b, what):
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape, (what, i)
        if case.deterministic:
            assert np.array_equal(x, y, equal_nan=True), "%s: output %d differs" % (what, i)
        else:
            xf, yf = x.astype(np.complex128), y.astype(np.complex128)
            fin = np.isfinite(yf)
            assert np.array_equal(np.isfinite(xf), fin), (what, i)
            d = np.abs(xf[fin] - yf[fin]).max(initial=0.0)
            assert d <= AGREE * np.abs(yf[fin]).max(initial=0.0), \
                "%s: output %d differs by %.3g of its maximum" % (
                    what, i, d / np.abs(yf[fin]).max())


COLD = {}


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_cold(name):
    from scintools_b200 import _lib
    _sb()
    _lib.check(_lib.lib.sb_release())
    COLD[name] = CASES[NAMES.index(name)].run("small")


@pytest.fixture(scope="module")
def grown():
    """Every case once at its larger shape: every slot regrown, holding foreign data."""
    _sb()
    for c in CASES:
        c.run("large")
    return True


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_after_others(grown, name):
    case = CASES[NAMES.index(name)]
    got = case.run("small")
    if name in COLD:
        same(case, got, COLD[name], name + ": cold vs after others")


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_small_large_small(name):
    case = CASES[NAMES.index(name)]
    a = case.run("small")
    case.run("large")
    same(case, case.run("small"), a, name + ": small, large, small")


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_side_stream(name):
    import torch
    case = CASES[NAMES.index(name)]
    ref = case.run("small")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = case.run("small")
    torch.cuda.synchronize()
    same(case, got, ref, name + ": side stream vs default stream")


# --------------------------------------------------------------------------
# A. streams, through the ABI with device inputs
# --------------------------------------------------------------------------
def _flip(x):
    """Other data of the same shapes: every 2-D array reversed on both axes."""
    return {k: (np.ascontiguousarray(v[::-1, ::-1]) if isinstance(v, np.ndarray) and v.ndim == 2
                else v) for k, v in x.items()}


def _prep_sspec(c, x):
    import torch
    FL = _m("test_gpu_fft_lengths")
    D, L = FL._dev()
    nf, nt = x["dyn"].shape
    NF, NT = DO.fft_lengths(nf, nt)
    dyn = D.upload(x["dyn"])
    wt, wf, swt, swf = FL._windows(D, x)
    out = D.empty((NF // 2, NT), torch.float32)

    def call(s):
        L.check(L.lib.sb_sspec_f32(dyn.data_ptr(), nf, nt, D.ptr(wt), D.ptr(wf), swt, swf, 0,
                                   1, 0, 0, 0, out.data_ptr(), s))
    return call, lambda: out.cpu().numpy(), (dyn, wt, wf)


def _prep_acf(c, x):
    import torch
    FL = _m("test_gpu_fft_lengths")
    D, L = FL._dev()
    nf, nt = x["dyn"].shape
    dyn = D.upload(x["dyn"])
    out = D.empty((2 * nf, 2 * nt), torch.float32)

    def call(s):
        L.check(L.lib.sb_acf_f32(dyn.data_ptr(), nf, nt, 1, c.p["normalise"], out.data_ptr(), s))
    return call, lambda: out.cpu().numpy(), (dyn,)


def _prep_cs(c, x):
    import torch
    FL = _m("test_gpu_fft_lengths")
    D, L = FL._dev()
    p = c.p
    nf, nt, npad = p["nf"], p["nt"], p["npad"]
    NF, NT = (npad + 1) * nf, (npad + 1) * nt
    pitch = NT // 2 + 4 if p["half"] else NT
    dspec = D.upload(x["dspec"])
    mask = D.upload(x["mask"]) if x["mask"] is not None else None
    out = D.zeros((NF, pitch, 2), torch.float32)
    pad = float(np.float32(np.nan if p["pad"] is None else p["pad"]))

    def call(s):
        L.check(L.lib.sb_cs_f32(dspec.data_ptr(), nf, nt, npad, pad, D.ptr(mask), int(p["half"]),
                                pitch, p["keep"], out.data_ptr(), s))
    return call, lambda: FL.to_complex(out.cpu().numpy()), (dspec, mask)


def _prep_ifft2(c, x):
    import torch
    FL = _m("test_gpu_fft_lengths")
    D, L = FL._dev()
    p = c.p
    c0, c1 = FL._crops(p)
    X = D.upload(x["X"])
    out = D.empty((c0, c1, 2), torch.float32)

    def call(s):
        L.check(L.lib.sb_ifft2_c2c_f32(X.data_ptr(), p["n0"], p["n1"], p["centred"], p["crop0"],
                                       p["crop1"], 3.0, 0, out.data_ptr(), s))
    return call, lambda: FL.to_complex(out.cpu().numpy()), (X,)


def _prep_screen(c, x):
    import torch
    FL = _m("test_gpu_fft_lengths")
    D, L = FL._dev()
    nx, ny = c.p["nx"], c.p["ny"]
    w, n1, n2 = D.upload(x["w"]), D.upload(x["n1"]), D.upload(x["n2"])
    out = D.empty((nx, ny), torch.float64)

    def call(s):
        L.check(L.lib.sb_sim_screen(nx, ny, w.data_ptr(), n1.data_ptr(), n2.data_ptr(), 0,
                                    out.data_ptr(), s))
    return call, lambda: out.cpu().numpy(), (w, n1, n2)


def _slow_ft_inputs(c):
    rng = np.random.default_rng(7)
    nt, nf = c.p["nt"], c.p["nf"]
    return {"x": rng.normal(size=(nt, nf)).astype(np.float32),
            "freqs": np.linspace(1300.0, 1500.0, nf)}


def _prep_slow_ft(c, x):
    import torch
    FL = _m("test_gpu_fft_lengths")
    D, L = FL._dev()
    nt, nf = x["x"].shape
    xs = D.upload(x["x"])
    fs = D.upload(x["freqs"] / x["freqs"][nf // 2])
    out = D.empty((nt, nf, 2), torch.float32)

    def call(s):
        L.check(L.lib.sb_slow_ft_f32(xs.data_ptr(), nt, nf, fs.data_ptr(), out.data_ptr(), s))
    return call, lambda: FL.to_complex(out.cpu().numpy()), (xs, fs)


def _check_slow_ft(c, x, got):
    from oracle import slow_ft_oracle as SFO
    _m("test_gpu_slow_ft")._check(got, SFO.bluestein(x["x"], x["freqs"]), "slow_ft race")


def _tiles_inputs(c):
    p = c.p
    rng = np.random.default_rng(11)
    return {"dyn": rng.exponential(1.0, (p["nfc"] * p["fnum"] + 3, p["ntc"] * p["tnum"] + 5))
            .astype(np.float32)}


def _prep_tiles(c, x):
    import torch
    FL = _m("test_gpu_fft_lengths")
    D, L = FL._dev()
    p = c.p
    nf, nt = x["dyn"].shape
    NF, NT = DO.fft_lengths(p["fnum"], p["tnum"])
    dyn = D.upload(x["dyn"])
    out = D.empty((p["nfc"], p["ntc"], NF // 2, NT), torch.float32)

    def call(s):
        L.check(L.lib.sb_sspec_tiles_f32(dyn.data_ptr(), nf, nt, p["fnum"], p["tnum"], p["nfc"],
                                         p["ntc"], 0, 0, 0.0, 0.0, out.data_ptr(), s))
    return call, lambda: out.cpu().numpy(), (dyn,)


def _check_tiles(c, x, got):
    FL = _m("test_gpu_fft_lengths")
    p = c.p
    for ii in range(p["nfc"]):
        for jj in range(p["ntc"]):
            tile = x["dyn"][ii * p["fnum"]:(ii + 1) * p["fnum"], jj * p["tnum"]:(jj + 1) * p["tnum"]]
            ref = FL.sspec_power(tile, None, None, False, True)
            lin = 10 ** (got[ii, jj].astype(np.float64) / 10)
            assert np.abs(lin - ref).max() <= 1e-5 * np.abs(ref).max(), (ii, jj)


def _fl(entry):
    FL = _m("test_gpu_fft_lengths")
    inputs, _, check = FL.ENTRIES[entry]
    return inputs, check


# name -> (case, inputs, prep, check); inputs / check None: test_gpu_fft_lengths.py's
RACE = {
    "sspec": (_p("sspec", nf=100, nt=300, window=False, halve=1, prewhite=0), None, _prep_sspec,
              None),
    "acf": (_p("acf", nf=100, nt=300, normalise=1), None, _prep_acf, None),
    "cs": (_p("cs", nf=64, nt=256, npad=1, pad=None, half=True, keep=0, mask=True), None,
           _prep_cs, None),
    "cs_chirp": (_p("cs", nf=43, nt=101, npad=2, pad=None, half=False, keep=0, mask=False), None,
                 _prep_cs, None),
    "ifft2": (_p("ifft2", n0=256, n1=512, centred=1, crop0=0, crop1=0, real=False), None,
              _prep_ifft2, None),
    "slow_ft": (_p("slow_ft", nt=1000, nf=16), _slow_ft_inputs, _prep_slow_ft, _check_slow_ft),
    "sim_screen": (_p("screen", nx=256, ny=256), None, _prep_screen, None),
    "sspec_tiles": (_p("tiles", nfc=2, ntc=3, fnum=40, tnum=60), _tiles_inputs, _prep_tiles,
                    _check_tiles),
}


def race(name):
    """Stream A: 0.1 s of sleep, then the first call of a length; stream B: the same length
    at once.  Both results against float64."""
    import torch
    FL = _m("test_gpu_fft_lengths")
    spec, inputs, prep, check = RACE[name]
    c = FL._c(spec[0], **spec[1])
    if inputs is None:
        inputs, check = _fl(c.entry)
    xa = inputs(c)
    xb = _flip(xa)
    call_a, fetch_a, keep_a = prep(c, xa)
    call_b, fetch_b, keep_b = prep(c, xb)
    torch.cuda.synchronize()
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(sa):
        torch.cuda._sleep(SLEEP_CYCLES)
        call_a(sa.cuda_stream)
    with torch.cuda.stream(sb):
        call_b(sb.cuda_stream)
    torch.cuda.synchronize()
    got_a, got_b = fetch_a(), fetch_b()
    errors = []
    for tag, x, got in (("stream A", xa, got_a), ("stream B", xb, got_b)):
        try:
            check(c, x, got)
        except AssertionError as e:
            errors.append("%s: %s" % (tag, e))
    del keep_a, keep_b
    return errors


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(RACE))
def test_twiddle_race(name):
    """In a fresh process, so the table's memory never held twiddles.  Its kernels are
    loaded when the context is made: a kernel loaded lazily at its first launch can make
    the host wait for the device, which would let stream A's sleep and fill finish before
    stream B's call is even made."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""),
               CUDA_MODULE_LOADING="EAGER")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--race", name], env=env,
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]


@pytest.mark.gpu
def test_overlapping_calls():
    """Two 4096 x 8192 secondary spectra of different data, and two chirp-z conjugate
    spectra, enqueued back to back on two streams: each equals its default-stream result.
    Without the library's cross-stream ordering the two calls share the workspace planes
    at once; this is likely to show it, not certain (it depends on how the kernels
    interleave)."""
    import torch
    FL = _m("test_gpu_fft_lengths")
    big = FL._c("sspec", nf=4096, nt=8192, window=False, halve=1, prewhite=0)
    chirp = FL._c("cs", nf=1000, nt=3001, npad=0, pad=None, half=False, keep=0, mask=False)
    for c, prep in ((big, _prep_sspec), (chirp, _prep_cs)):
        xa = FL.ENTRIES[c.entry][0](c)
        xb = _flip(xa)
        call_a, fetch_a, keep_a = prep(c, xa)
        call_b, fetch_b, keep_b = prep(c, xb)
        call_a(torch.cuda.current_stream().cuda_stream)
        ref_a = fetch_a()
        call_b(torch.cuda.current_stream().cuda_stream)
        ref_b = fetch_b()
        torch.cuda.synchronize()
        sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
        with torch.cuda.stream(sa):
            call_a(sa.cuda_stream)
        with torch.cuda.stream(sb):
            call_b(sb.cuda_stream)
        torch.cuda.synchronize()
        for got, ref in ((fetch_a(), ref_a), (fetch_b(), ref_b)):
            d = np.abs(got.astype(np.complex128) - ref)
            assert d.max() <= AGREE * np.abs(ref).max(), (c.entry, d.max() / np.abs(ref).max())
        del keep_a, keep_b


if __name__ == "__main__":
    # one twiddle-race case in this fresh process (test_twiddle_race)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    errs = race(sys.argv[sys.argv.index("--race") + 1])
    for e in errs:
        print(e)
    sys.exit(1 if errs else 0)
