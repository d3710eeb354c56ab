"""Flux-variation correction on the CPU: the float64 oracle (oracle/correct_dyn_oracle.py)
against the unmodified reference's Dynspec.correct_dyn (tests/golden/correct_dyn_*.npz,
made by oracle/make_golden_correct_dyn.py), the device code of csrc/svd.cu under the SIMT
emulator (tests/host_emu/correct_dyn_emu.cpp) against numpy float64, the argument errors
of the port raised before any device call, and the new C symbols."""
import ctypes
import os
import subprocess
import types

import numpy as np
import pytest

from oracle import correct_dyn_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")
U = 2.0 ** -24

SVD_CASES = ["s1", "s2", "s3", "p3", "full", "lam"]
BP_CASES = ["freq", "time", "both", "smooth", "lam"]


def load_case(golden_dir, fname, name):
    """(kwargs, inputs, expected) of one fixture case; svd_model comes back complex128."""
    f = np.load(os.path.join(golden_dir, fname))
    svd, nmodes, frequency, time, lamsteps, nsmooth = (int(v) for v in f[name + "_args"])
    kw = dict(svd=bool(svd), nmodes=nmodes, frequency=bool(frequency), time=bool(time),
              lamsteps=bool(lamsteps), nsmooth=None if nsmooth < 0 else nsmooth)
    names = str(f[name + "_inputs"]).split(",")
    inputs = dict(dyn=f["in_" + names[0]])
    if len(names) > 1:
        inputs["lamdyn"] = f["in_" + names[1]]
    want = {a: f[name + "_" + a] for a in ("dyn", "lamdyn", "svd_model", "bandpass")
            if name + "_" + a in f.files}
    if "svd_model" in want:
        want["svd_model"] = want["svd_model"].astype(np.complex128)
    dtypes = dict(kv.split("=") for kv in str(f[name + "_dtypes"]).split(","))
    return kw, inputs, want, dtypes


def check_result(got, want, kw, inputs, tol):
    """Compare the attributes after correct_dyn: the NaN pattern exactly; the model to tol
    of its largest element; array / |model| with that error propagated through the division
    (tol |out| + |a| tol max|M| / M^2); everything else to tol relative."""
    attr = "lamdyn" if kw["lamsteps"] else "dyn"
    for k, ref in want.items():
        g = np.asarray(got[k])
        assert g.shape == ref.shape, k
        assert np.array_equal(np.isnan(g), np.isnan(ref)), k
        fin = np.isfinite(ref)
        assert np.array_equal(np.isfinite(g), fin), k
        err = np.abs(g - ref)[fin]
        if k == "svd_model":
            bound = tol * np.abs(ref).max() + 1e-300
        elif k == attr and kw["svd"]:
            M = np.abs(want["svd_model"])
            a = np.nan_to_num(inputs[attr])
            with np.errstate(divide="ignore", invalid="ignore"):
                bound = (tol * np.abs(ref) + np.abs(a) * tol * M.max() / M ** 2)[fin]
        else:
            bound = tol * np.abs(ref)[fin] + 1e-300
        assert (err <= bound).all(), (k, float((err / np.maximum(bound, 1e-300)).max()))


@pytest.mark.parametrize("fname,name", [("correct_dyn_svd.npz", c) for c in SVD_CASES] +
                         [("correct_dyn_bandpass.npz", c) for c in BP_CASES])
def test_oracle_matches_reference(golden_dir, fname, name):
    """The oracle's correct_dyn on a plain object reproduces every attribute the reference
    left (NaN pattern bit-exact, values to 1e-12), including the caller's arrays it mutates."""
    kw, inputs, want, dtypes = load_case(golden_dir, fname, name)
    obj = types.SimpleNamespace(**{k: v.copy() for k, v in inputs.items()})
    dyn_obj = obj.dyn
    CO.correct_dyn(obj, **kw)
    got = {k: getattr(obj, k) for k in want}
    check_result(got, want, kw, inputs, 1e-12)
    if not (kw["svd"] and kw["lamsteps"]):      # the reference zeroes the caller's NaNs
        assert not np.isnan(dyn_obj).any()
    assert dtypes["dyn"] == "float64"
    if kw["svd"]:
        assert dtypes["svd_model"] == "complex128"


def test_fixture_layout(golden_dir):
    """The bandpass fixtures hold an all-zero channel and sub-integration, and the lamsteps
    case an all-zero lamdyn row; the svd fixtures zeros and NaNs; 'full' asks for more modes
    than min(nf, nt)."""
    _, inp, want, _ = load_case(golden_dir, "correct_dyn_bandpass.npz", "both")
    d = inp["dyn"]
    assert (d == 0).all(1).any() and (d == 0).all(0).any() and np.isnan(d).any()
    assert np.isnan(want["dyn"]).all(1).any() and np.isnan(want["dyn"]).all(0).any()
    _, inp, _, _ = load_case(golden_dir, "correct_dyn_bandpass.npz", "lam")
    assert (inp["lamdyn"] == 0).all(1).any()
    kw, inp, _, _ = load_case(golden_dir, "correct_dyn_svd.npz", "s1")
    assert (inp["dyn"] == 0).any() and np.isnan(inp["dyn"]).any()
    kw, inp, _, _ = load_case(golden_dir, "correct_dyn_svd.npz", "full")
    assert kw["nmodes"] >= min(inp["dyn"].shape)


# ---- device code under the SIMT emulator ----------------------------------------------

def _emu_lib():
    src = os.path.join(EMU, "correct_dyn_emu.cpp")
    out = os.path.join(EMU, "_build", "correct_dyn_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    csrc = os.path.join(ROOT, "scintools_b200", "csrc")
    newest = max([os.path.getmtime(os.path.join(csrc, f)) for f in os.listdir(csrc)] +
                 [os.path.getmtime(src), os.path.getmtime(os.path.join(EMU, "simt.h"))])
    if not os.path.exists(out) or os.path.getmtime(out) < newest:
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                        "-x", "c++", src, "-o", out], check=True)
    lib = ctypes.CDLL(out)
    vp, ci = ctypes.c_void_p, ctypes.c_int
    lib.emu_gram.argtypes = [vp, ci, ci, ci, vp, vp, vp]
    lib.emu_apply.argtypes = [vp, ci, ci, ci, vp, ci, vp, vp]
    lib.emu_orth.argtypes = [vp, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.emu_ql.argtypes = [ci, vp, vp, vp, ci]
    lib.emu_bandpass.argtypes = [vp, ci, ci, ci, vp, vp, ci, vp, vp, vp]
    for f in (lib.emu_gram, lib.emu_apply, lib.emu_orth, lib.emu_ql, lib.emu_bandpass):
        f.restype = ci
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _matrix(rng, nf, nt):
    A = (rng.exponential(1.0, (nf, nt)) * (1 + np.arange(nf))[:, None] ** 0.3).astype(np.float32)
    A.flat[rng.choice(A.size, 5, replace=False)] = 0.0
    A.flat[rng.choice(A.size, 3, replace=False)] = np.nan
    return A


@pytest.mark.parametrize("nf,nt,G", [(7, 37, 3), (20, 600, 4), (5, 1500, 2), (4, 3000, 3),
                                     (5, 6000, 2), (3, 9000, 2),
                                     (2, 12000, 1)])
def test_gram_pass_on_host(nf, nt, G):
    """svd_gram_kernel at every row width (1 .. 16 values per thread with the next row
    prefetched into shared memory, 32 without) over G blocks and
    svd_reduce_kernel: A^T (A x) against numpy float64, NaN read as 0; one block's share is
    checked on its own too."""
    lib = _emu_lib()
    rng = np.random.default_rng(nt)
    A = _matrix(rng, nf, nt)
    x = rng.normal(size=nt)
    part = np.zeros((G, nt))
    w = np.zeros(nt)
    assert lib.emu_gram(_p(A), nf, nt, G, _p(x), _p(part), _p(w)) == 0
    A64 = np.nan_to_num(A.astype(np.float64))
    ref = A64.T @ (A64 @ x)
    mag = np.abs(A64).T @ (np.abs(A64) @ np.abs(x))
    assert (np.abs(w - ref) <= 1e-13 * mag * np.sqrt(nt)).all()
    b = G - 1                                       # block b takes rows b, b + G, ...
    share = A64[b::G].T @ (A64[b::G] @ x)
    assert np.allclose(part[b], share, rtol=0, atol=1e-13 * mag.max() * np.sqrt(nt))


@pytest.mark.parametrize("nf,nt,k", [(9, 45, 1), (6, 700, 3), (4, 12000, 2)])
def test_apply_pass_on_host(nf, nt, k):
    """svd_apply_kernel: projections, model row and a / |model| against numpy float64 (the
    model and the quotient are rounded to float32 once)."""
    lib = _emu_lib()
    rng = np.random.default_rng(k + nt)
    A = _matrix(rng, nf, nt)
    Y = np.linalg.qr(rng.normal(size=(nt, k)))[0].T.copy()
    out = np.zeros((nf, nt), np.float32)
    model = np.zeros((nf, nt), np.float32)
    assert lib.emu_apply(_p(A), nf, nt, k, _p(Y), 2, _p(out), _p(model)) == 0
    A64 = np.nan_to_num(A.astype(np.float64))
    M = (A64 @ Y.T) @ Y
    mag = (np.abs(A64) @ np.abs(Y.T)) @ np.abs(Y)
    assert (np.abs(model - M) <= U * np.abs(M) + 1e-13 * mag).all()
    with np.errstate(divide="ignore", invalid="ignore"):
        q = A64 / np.abs(M)
        bound = 2 * U * np.abs(q) + np.abs(A64) * 1e-13 * mag / M ** 2
    assert np.array_equal(np.isnan(out), np.isnan(q))
    fin = np.isfinite(q)
    assert (np.abs(out - q)[fin] <= bound[fin]).all()


def _orth(lib, V, w, amax0):
    nq, nt = V.shape
    h1, h2, alpha, nrm, v = np.zeros(nq), np.zeros(nq), np.zeros(nq), np.zeros(1), np.zeros(nt)
    amax, restart = np.array([amax0]), np.zeros(1, np.int32)
    assert lib.emu_orth(_p(V), nq, nt, _p(w), _p(h1), _p(h2), _p(alpha), _p(nrm), _p(v),
                        _p(amax), _p(restart)) == 0
    return alpha, nrm[0], v, amax[0], int(restart[0])


def test_lanczos_vector_kernels_on_host():
    """svd_dots / svd_orth (twice) / svd_norm / svd_scale: the new Lanczos vector is w with
    its components along the previous ones removed, normalised; alpha is the Rayleigh
    quotient and amax its running maximum.  A w inside span(V) is a breakdown: beta is
    recorded as 0 and svd_restart_kernel supplies a unit vector orthogonal to V instead."""
    lib = _emu_lib()
    rng = np.random.default_rng(5)
    nt, nq = 300, 4
    V = np.linalg.qr(rng.normal(size=(nt, nq)))[0].T.copy()
    w0 = rng.normal(size=nt) + 3 * V[nq - 1]
    alpha, nrm, v, amax, restart = _orth(lib, V, w0.copy(), 1.0)
    r = w0 - V.T @ (V @ w0)
    assert restart == 0 and np.allclose(nrm, np.linalg.norm(r), rtol=1e-13)
    assert np.allclose(v, r / np.linalg.norm(r), rtol=0, atol=1e-13)
    assert abs(alpha[nq - 1] - V[nq - 1] @ w0) <= 1e-13 * np.abs(w0).sum()
    assert amax == max(1.0, alpha[nq - 1])
    assert np.abs(V @ v).max() < 1e-14
    w1 = 5.0 * V[nq - 1] + 2.0 * V[0]                 # B v_m inside the Krylov space
    alpha, nrm, v, amax, restart = _orth(lib, V, w1.copy(), 0.0)
    assert restart == 1 and nrm == 0.0 and abs(alpha[nq - 1] - 5.0) < 1e-13
    assert abs(np.linalg.norm(v) - 1.0) < 1e-14 and np.abs(V @ v).max() < 1e-14
    alpha, nrm, v2, amax, restart = _orth(lib, V, w1.copy(), 0.0)
    assert np.array_equal(v, v2)                      # the restart vector is deterministic
    Vfull = np.linalg.qr(rng.normal(size=(6, 6)))[0].T.copy()
    alpha, nrm, v, amax, restart = _orth(lib, Vfull, 2.0 * Vfull[5].copy(), 0.0)
    assert restart == 1 and not v.any()               # nothing is left to restart from


@pytest.mark.parametrize("n", [1, 2, 7, 60])
def test_tridiagonal_ql(n):
    """The host QL of T_m: eigenvalues and eigenvectors against numpy, and the last-row-only
    mode the stopping rule uses; a split (zero off-diagonal) and a repeated value included."""
    lib = _emu_lib()
    rng = np.random.default_rng(n)
    d = rng.normal(size=n)
    e = np.abs(rng.normal(size=n))
    if n >= 7:
        e[3] = 0.0
        d[5] = d[6] = 1.0
        e[5] = 0.0
    T = np.diag(d) + np.diag(e[:n - 1], 1) + np.diag(e[:n - 1], -1)
    w_ref, Z_ref = np.linalg.eigh(T)
    dd, ee, Z = d.copy(), e.copy(), np.eye(n)
    assert lib.emu_ql(n, _p(dd), _p(ee), _p(Z), n) == 0
    o = np.argsort(dd)
    assert np.allclose(dd[o], w_ref, rtol=0, atol=1e-13 * max(1, np.abs(w_ref).max()))
    assert np.allclose(T @ Z, Z * dd, atol=1e-12)
    assert np.allclose(Z.T @ Z, np.eye(n), atol=1e-12)
    d2, e2, z = d.copy(), e.copy(), np.zeros(n)
    z[-1] = 1.0
    assert lib.emu_ql(n, _p(d2), _p(e2), _p(z), 1) == 0
    assert np.array_equal(d2, dd) and np.allclose(z, Z[-1], atol=1e-13)


@pytest.mark.parametrize("zero_as_nan,rows,cols", [(1, True, True), (0, True, True),
                                                   (1, False, True), (1, True, False)])
def test_bandpass_kernels_on_host(zero_as_nan, rows, cols):
    """bandpass_row / col (+ reduce over row chunks) / divide against the oracle's float64
    arithmetic on a dyn with an all-zero channel and sub-integration and NaN pixels."""
    lib = _emu_lib()
    rng = np.random.default_rng(11 + zero_as_nan)
    nf, nt = 13, 300
    A = _matrix(rng, nf, nt)
    A[4] = 0.0
    A[:, 250] = 0.0
    x = np.nan_to_num(A.astype(np.float64))
    if zero_as_nan:
        x[x == 0] = np.nan
    rowdiv = 1.0 + rng.random(nf) if rows else None
    coldiv = 1.0 + rng.random(nt) if cols else None
    rm, cm = np.zeros(nf), np.zeros(nt)
    out = np.zeros((nf, nt), np.float32)
    assert lib.emu_bandpass(_p(A), nf, nt, zero_as_nan, _p(rowdiv), _p(coldiv), 4, _p(rm),
                            _p(cm), _p(out)) == 0
    ref_r = CO._nanmean_or_nan(x, 1)
    q = x / rowdiv[:, None] if rows else x
    ref_c = CO._nanmean_or_nan(q, 0)
    ref_o = q / coldiv[None, :] if cols else q
    for got, ref, tol in ((rm, ref_r, 1e-14), (cm, ref_c, 1e-14), (out, ref_o, U)):
        assert np.array_equal(np.isnan(got), np.isnan(ref))
        fin = np.isfinite(ref)
        assert (np.abs(got - ref)[fin] <= tol * np.abs(ref)[fin]).all()
    assert np.isnan(rm[4]) == bool(zero_as_nan) and np.isnan(cm[250]) == bool(zero_as_nan)


# ---- host layer -----------------------------------------------------------------------

def test_argument_errors_before_device(monkeypatch):
    """nmodes < 1 or above the cap, non-integer nmodes, shapes outside the envelope, complex
    or non-2-D input, and a missing velocity array raise before any device call."""
    from scintools_b200 import _device, ththmod
    from scintools_b200.dynspec import BasicDyn, Dynspec

    def no_device(*a, **k):
        raise AssertionError("device touched")

    monkeypatch.setattr(_device, "device", no_device)
    ok = np.ones((4, 6))
    for arr, n, exc in [(ok, 0, ValueError), (ok, -2, ValueError), (ok, 33, ValueError),
                        (ok, 1.5, TypeError), (np.ones((32769, 1)), 1, ValueError),
                        (np.ones((2, 16385)), 1, ValueError), (np.ones(5), 1, ValueError),
                        (np.ones((0, 3)), 1, ValueError), (ok + 0j, 1, TypeError)]:
        with pytest.raises(exc):
            ththmod.svd_model(arr, n)
    t = np.arange(6) * 10.0
    f = 1400 + np.arange(4) * 0.5
    ds = Dynspec(dyn=BasicDyn(ok.copy(), times=t, freqs=f, dt=10.0, df=0.5), verbose=False)
    for kw, exc in [(dict(nmodes=0), ValueError), (dict(nmodes=40), ValueError),
                    (dict(velocity=True), ValueError),
                    (dict(velocity=True, lamsteps=True), ValueError)]:
        with pytest.raises(exc):
            ds.correct_dyn(**kw)
    ds.dyn = np.ones((3, 16385))
    for svd in (True, False):
        with pytest.raises(ValueError):
            ds.correct_dyn(svd=svd)
    assert not hasattr(ds, "svd_model")          # nothing named svd_model on the class


def test_library_exports_correct_dyn_symbols():
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _lib, ththmod
    from scintools_b200.dynspec import Dynspec
    for n in ("sb_svd_topk", "sb_svd_apply", "sb_bandpass_rows", "sb_bandpass_cols",
              "sb_bandpass_divide"):
        assert n in _lib.EXPORTS
    assert _lib.lib.sb_abi_version() >= 7
    assert callable(ththmod.svd_model) and callable(Dynspec.correct_dyn)
    assert "svd_model" not in dir(Dynspec)
