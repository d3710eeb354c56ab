"""Arc asymmetry on the CPU: the numpy oracle's calc_asymmetry against the reference's
(tests/golden/asymmetry_sample.npz, made by oracle/make_golden_asymmetry.py), the port's
chunk planning of Dynspec.calc_asymmetry against the reference's chunk list, the device
code of sb::asymmetry_batch around the eigenpair (crop, gather, asymmetry) under the SIMT
emulator (tests/host_emu/asymmetry_emu.cpp), and the new C symbol."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import asymmetry_oracle as AO
from oracle import thth_oracle as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")


def _load(golden_dir):
    return np.load(os.path.join(golden_dir, "asymmetry_sample.npz"))


def _chunks(f):
    ncf, nct = f["asymmetry"].shape
    return AO.chunk_list(f["dyn"].astype(np.float64), f["freqs"], f["times"], int(f["cwf"]),
                         int(f["cwt"]), ncf, nct, float(f["ththeta"]), float(f["fref"]),
                         f["edges"], int(f["npad"]))


def test_oracle_asymmetry_matches_reference(golden_dir):
    """Every chunk of case a to 1e-10, and the NaN pattern of case a and the failures of b."""
    f = _load(golden_dir)
    ref = f["asymmetry"]
    assert ref.dtype == np.complex128 and ref.shape == (16, 4)
    got = np.zeros(ref.shape, complex)
    for cf, ct, d, e, t, fr, eta in _chunks(f):
        got[cf, ct] = AO.calc_asymmetry(d, e, t, fr, eta, int(f["npad"]))
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref)
    assert np.abs(got[fin] - ref[fin]).max() <= 1e-10
    times, freqs, cwf, cwt = f["times"], f["freqs"], int(f["cwf"]), int(f["cwt"])
    for tag in ("zero", "small", "wide"):
        d = np.zeros((cwf, cwt)) if tag == "zero" else f["b_dspec"]
        a = AO.calc_asymmetry(d, f["b_%s_edges" % tag], times[:cwt], freqs[cwf:2 * cwf],
                              float(f["b_%s_eta" % tag]), int(f["npad"]))
        assert np.isnan(a) and np.isnan(float(f["b_%s_asymm" % tag])), tag
        assert str(f["b_%s_printed" % tag]), tag


def test_dynspec_chunk_plan_matches_reference(golden_dir):
    """Dynspec._asymmetry_params on case a: the reference's slices (widths 32 / 48 / 64 / 80),
    curvatures, scaled edges and pad values (the chunk means after the NaNs are zeroed)."""
    import __graft_entry__ as g
    g.build()
    from scintools_b200.dynspec import BasicDyn, Dynspec
    f = _load(golden_dir)
    dyn = f["dyn"].astype(np.float64)
    ds = Dynspec(dyn=BasicDyn(dyn, times=f["times"], freqs=f["freqs"]), verbose=False)
    ds.cwf, ds.cwt, ds.npad = int(f["cwf"]), int(f["cwt"]), int(f["npad"])
    ds.ncf_fit, ds.nct_fit = f["asymmetry"].shape
    ds.fref, ds.edges, ds.ththeta = float(f["fref"]), f["edges"], float(f["ththeta"])
    pars = ds._asymmetry_params()
    assert len(pars) == 64
    nct = ds.nct_fit
    widths = set()
    for k, p in enumerate(pars):
        dspec2, edges, time2, freq2, eta, ct, cf, npad, verbose = p
        assert (cf, ct) == divmod(k, nct) and npad == 3 and verbose is False
        t0, t1 = f["tslice"][k]
        assert np.array_equal(time2, f["times"][t0:t1])
        assert dspec2.shape == (64, t1 - t0)
        widths.add(t1 - t0)
        assert eta == f["eta"][k]
        assert np.array_equal(edges, f["edges_cf"][cf])
        assert np.array_equal(freq2, f["freqs"][cf * 64:(cf + 1) * 64])
        assert np.isfinite(dspec2).all()
        assert dspec2.mean() == pytest.approx(f["pad"][k], rel=0, abs=1e-12)
    assert widths == {32, 48, 64, 80}
    # the NaNs of the field fall into three chunks of cf = 1; their zeros count in the mean
    has_nan = [np.isnan(dyn[64:128, t0:t1]).any() for t0, t1 in f["tslice"][4:8]]
    assert sum(has_nan) == 3


def _emu_lib():
    src = os.path.join(EMU, "asymmetry_emu.cpp")
    out = os.path.join(EMU, "_build", "asymmetry_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    csrc = os.path.join(ROOT, "scintools_b200", "csrc")
    newest = max([os.path.getmtime(os.path.join(csrc, f)) for f in os.listdir(csrc)] +
                 [os.path.getmtime(src), os.path.getmtime(os.path.join(EMU, "simt.h"))])
    if not os.path.exists(out) or os.path.getmtime(out) < newest:
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                        "-x", "c++", src, "-o", out], check=True)
    return ctypes.CDLL(out)


def test_asymmetry_gather_on_host(golden_dir):
    """Crop and gather of two chunks with their own spectra, axes, theta grids and
    curvatures from one geometry table (the second one cropped): sizes and zero pattern
    exact against the oracle's thth_redmap on the fp32-rounded spectra, entries to fp32
    rounding."""
    f = _load(golden_dir)
    cl = [c for c in _chunks(f) if c[1] == 1]           # width 48: 256 x 192, chirp-z sizes
    picks = [(cl[0], 1.0), (cl[9], 40.0)]
    npad = int(f["npad"])
    cs32, ax, ths, etas, reds = [], [], [], [], []
    for (cf, ct, d, e, t, fr, eta), scale in picks:
        CS, tau, fd = AO.spectrum(d, t, fr, npad)
        c32 = np.ascontiguousarray(CS.astype(np.complex64))
        cs32.append(c32)
        ax += [tau[0], np.diff(tau).mean(), abs(tau.max()), fd[0], np.diff(fd).mean(),
               abs(fd.max()) / 2]
        ths.append(TO.theta_centres(e))
        etas.append(eta * scale)
        red, _ = TO.thth_redmap(c32.astype(np.complex128), tau, fd, eta * scale, e)
        reds.append(red)
    n_th = len(ths[0])
    ld = (n_th + 31) // 32 * 32
    ntau, nfd = cs32[0].shape
    M = np.zeros((2, ld, ld), np.complex64)
    nred = np.zeros(2, np.int32)
    ax = np.array(ax)
    etas = np.array(etas)
    lib = _emu_lib()
    vp, c_i, c_ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    lib.emu_asym_gather.argtypes = [vp, c_i, c_ll, c_ll, vp, vp, c_i, vp, vp, vp]
    P = lambda a: a.ctypes.data_as(vp)   # noqa: E731
    lib.emu_asym_gather((vp * 2)(*[c.ctypes.data for c in cs32]), 2, ntau, nfd, P(ax),
                        (vp * 2)(*[t.ctypes.data for t in ths]), n_th, P(etas), P(nred), P(M))
    eps = np.finfo(np.float32).eps
    assert nred[0] == n_th and 3 <= nred[1] < n_th
    for k in range(2):
        n = reds[k].shape[0]
        assert nred[k] == n
        up = np.triu(np.ones((n, n), bool), 1)
        got = M[k, :n, :n].astype(np.complex128)
        ref = reds[k]
        assert np.array_equal(got[up] == 0, ref[up] == 0), k
        assert (got[~up] == 0).all()                      # untouched below / on the diagonal
        assert (np.abs(got[up] - ref[up]) <= 4 * eps * np.abs(ref[up])).all(), k
        assert np.array_equal(ref, np.conjugate(ref.T))   # the Hermitian fill mirrors the upper part


@pytest.mark.parametrize("m", [3, 4, 5, 6, 301])
def test_asymmetry_finish_on_host(m):
    """The asymmetry from a given V for both parities of m (m = 3: one element per side),
    to 1e-12 of the oracle; status bits give NaN; V is copied zero-padded, or zeros where
    no eigenvector was computed."""
    rng = np.random.default_rng(m)
    ld = (m + 31) // 32 * 32
    V = np.zeros((3, ld), np.complex64)
    for k in range(3):
        V[k, :m] = (rng.normal(size=m) + 1j * rng.normal(size=m)).astype(np.complex64)
    nred = np.full(3, m, np.int32)
    status = np.array([0, 8, 1], np.int32)
    asym = np.zeros(3)
    vout = np.full((3, ld), np.nan + 0j, np.complex64)
    lib = _emu_lib()
    vp, c_i = ctypes.c_void_p, ctypes.c_int
    lib.emu_asym_finish.argtypes = [vp, c_i, c_i, vp, vp, vp, vp]
    P = lambda a: a.ctypes.data_as(vp)   # noqa: E731
    lib.emu_asym_finish(P(V), 3, ld, P(nred), P(status), P(asym), P(vout))
    ref = AO.asymmetry_of(V[0, :m].astype(np.complex128))
    assert abs(asym[0] - ref) <= 1e-12
    assert np.isnan(asym[1]) and np.isnan(asym[2])
    assert np.array_equal(vout[:2], V[:2])
    assert (vout[2] == 0).all()


def test_asymmetry_zero_over_zero_is_nan():
    """A vector with weight only on its centre element: 0 / 0 -> NaN, as in numpy."""
    V = np.zeros((1, 32), np.complex64)
    V[0, 2] = 1.0
    asym = np.zeros(1)
    lib = _emu_lib()
    vp, c_i = ctypes.c_void_p, ctypes.c_int
    lib.emu_asym_finish.argtypes = [vp, c_i, c_i, vp, vp, vp, vp]
    P = lambda a: a.ctypes.data_as(vp)   # noqa: E731
    lib.emu_asym_finish(P(V), 1, 32, P(np.array([5], np.int32)), P(np.zeros(1, np.int32)),
                        P(asym), None)
    assert np.isnan(asym[0]) and np.isnan(AO.asymmetry_of(V[0, :5].astype(complex)))


def test_library_exports_asymmetry_symbol():
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _lib, ththmod
    from scintools_b200.dynspec import Dynspec
    assert "sb_asymmetry_batch" in _lib.EXPORTS and hasattr(_lib.lib, "sb_asymmetry_batch")
    assert _lib.lib.sb_abi_version() >= 5
    assert callable(ththmod.calc_asymmetry) and callable(ththmod.asymmetry_batch)
    assert callable(Dynspec.calc_asymmetry)
