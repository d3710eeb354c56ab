"""Flux-variation correction on the GPU (Dynspec.correct_dyn, ththmod.svd_model; sb_svd_*,
sb_bandpass_*) against the reference's fixtures, prescribed spectra whose truth needs no SVD,
and the float64 oracle (oracle/correct_dyn_oracle.py) at sizes the fixtures do not reach.

Bounds.  u = 2^-24.  A is the float64 input with NaN read as 0; the device works on its
float32 narrowing A~ = A + E, |E_ij| <= u |A_ij|, so ||E||_2 <= ||E||_F <= eps := u ||A||_F.
 - Singular values: Weyl gives |s~_j - s_j| <= eps.  The solver returns theta_j with
   |theta_j - s~_j^2| <= rho_j (Kahan's bound for the reported true residual rho_j, which
   the solver accepts only at <= 1e-11 theta_1), so |sqrt(theta_j) - s~_j| <=
   min(rho_j / s~_j, sqrt(rho_j)).  Test: eps + min(2 rho_j / s_j, sqrt(rho_j)), doubled.
 - Model: the device model is A~ P~ with P~ = Y Y^T, the truth A P with P the projector on
   the top-k right singular vectors (the row space when k >= rank).  ||A~ P~ - A P||_2 <=
   ||E||_2 + s_1 ||P~ - P||_2 and ||P~ - P||_2 = sin(Theta) <= sin_narrow + sin_solver:
   Wedin for A vs A~, sin_narrow <= sqrt(2) eps / (s_k - s_{k+1} - eps); Davis-Kahan for
   the Ritz subspace of A~^T A~, sin_solver <= ||rho||_2 / ((s_k - eps)^2 -
   (s_{k+1} + eps)^2).  Every element is at most the 2-norm, and the stored model adds one
   float32 rounding: |m_dev - m| <= E_M := 2 (eps + s_1 sin(Theta)) + 2 u |m|.
 - a / |m|: a~ carries u, the quotient is rounded to float32 once (u), and the model error
   enters to first order as |a| E_M / m^2: bound 2 u |out| + 2 |a| E_M / m^2, checked
   where |m| >= 4 E_M (first order holds there; the NaN pattern is checked everywhere).
 - Bandpass (svd=False, all data >= 0): a mean of non-negative values each carrying u has
   relative error <= u (the float64 sums add far less).  A smoothed vector S b has relative
   error <= kappa u with kappa = (|S| b) / |S b| (1 without smoothing), computed here from
   savgol_filter's own matrix.  The row quotient then carries u (1 + kappa_b), the column
   mean of it u (1 + max kappa_b), the final quotient adds kappa_t times that and one
   float32 rounding: |out_dev - out| <= 2 u (2 + kappa_b,i + kappa_t,j (1 + max kappa_b))
   |out|.  Bandpass vectors: 2 u relative.
"""
import os
import warnings

import numpy as np
import pytest

from oracle import correct_dyn_oracle as CO

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SVD_CASES = ["s1", "s2", "s3", "p3", "full", "lam"]
BP_CASES = ["freq", "time", "both", "smooth", "lam"]


def load_case(golden_dir, fname, name):
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
    dtypes = dict(kv.split("=") for kv in str(f[name + "_dtypes"]).split(","))
    return kw, inputs, want, dtypes


def _dynspec(dyn, lamdyn=None):
    from scintools_b200.dynspec import BasicDyn, Dynspec
    nf, nt = dyn.shape
    t = np.arange(nt) * 8.0
    f = 1400.0 + np.arange(nf) * 0.25
    ds = Dynspec(dyn=BasicDyn(dyn, times=t, freqs=f, dt=8.0, df=0.25), verbose=False)
    if lamdyn is not None:
        ds.lamdyn = lamdyn
    return ds


def model_bound(a, k, rho, svals=None):
    """(E_M without the 2 u |m| term, s) for the float64 input a (NaN -> 0) and k modes."""
    a = np.nan_to_num(np.asarray(a, dtype=np.float64))
    s = np.linalg.svd(a, compute_uv=False) if svals is None else np.asarray(svals)
    eps = U * np.sqrt(np.sum(a * a))
    s1 = s[0] if s.size else 0.0
    sk = s[k - 1] if k <= s.size else 0.0
    sk1 = s[k] if k < s.size else 0.0
    if k >= np.sum(s > eps):                       # the model is the row space projection
        sk = s[np.sum(s > eps) - 1] if np.sum(s > eps) else 0.0
        sk1 = 0.0
    gap_s = sk - sk1 - eps
    gap_l = (sk - eps) ** 2 - (sk1 + eps) ** 2
    if s1 == 0.0:
        return 0.0, s
    assert gap_s > 0 and gap_l > 0, "test matrix has no gap at k"
    sin = np.sqrt(2) * eps / gap_s + np.linalg.norm(rho) / gap_l
    return 2 * (eps + s1 * sin), s


def check_model(model, M, EM):
    m = np.asarray(model).real
    err = np.abs(m - M)
    bound = EM + 2 * U * np.abs(M) + 1e-300
    assert (err <= bound).all(), float((err / bound).max())


def check_quotient(out, a, M, EM):
    """out = a / |M| within 2 u |out| + 2 |a| E_M / M^2 where |M| >= 4 E_M; NaN pattern
    everywhere."""
    a = np.nan_to_num(np.asarray(a, dtype=np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        ref = a / np.abs(M)
    assert np.array_equal(np.isnan(out), np.isnan(ref))
    use = np.isfinite(ref) & (np.abs(M) >= 4 * EM)
    with np.errstate(divide="ignore", invalid="ignore"):
        bound = 2 * U * np.abs(ref) + 2 * np.abs(a) * EM / M ** 2
    err = np.abs(out - ref)
    assert (err[use] <= bound[use] + 1e-300).all(), float((err[use] / bound[use]).max())
    assert use.mean() > 0.98


def _kappa(b, nsmooth):
    from scipy.signal import savgol_filter
    if nsmooth is None:
        return np.ones_like(b)
    S = savgol_filter(np.eye(b.size), nsmooth, 1, axis=0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return (np.abs(S) @ np.abs(b)) / np.abs(S @ b)


def check_bandpass_result(ds_attr_out, ref_out, kw, x_for_means):
    """Elementwise bound of the module docstring for svd=False."""
    assert np.array_equal(np.isnan(ds_attr_out), np.isnan(ref_out))
    fin = np.isfinite(ref_out)
    n = kw["nsmooth"]
    x = x_for_means
    kb = np.ones(x.shape[0])
    if kw["frequency"]:
        b = CO._zeros_to_mean(CO._nanmean_or_nan(x, 1))
        kb = np.nan_to_num(_kappa(np.nan_to_num(b), n), nan=1.0)
        from scipy.signal import savgol_filter
        x = x / (savgol_filter(b, n, 1) if n else b)[:, None]
    kt = np.ones(x.shape[1])
    if kw["time"]:
        t = CO._zeros_to_mean(CO._nanmean_or_nan(x, 0))
        kt = np.nan_to_num(_kappa(np.nan_to_num(t), n), nan=1.0)
    rel = 2 * U * (2 + kb[:, None] + kt[None, :] * (1 + kb.max()))
    err = np.abs(ds_attr_out - ref_out)
    assert (err[fin] <= (rel * np.abs(ref_out))[fin]).all()


# ---- fixtures --------------------------------------------------------------------------

@pytest.mark.parametrize("fname,name", [("correct_dyn_svd.npz", c) for c in SVD_CASES] +
                         [("correct_dyn_bandpass.npz", c) for c in BP_CASES])
def test_fixture_parity(golden_dir, fname, name):
    """Device Dynspec.correct_dyn on every reference fixture: the NaN pattern exactly, values
    within the bounds above, the reference's dtypes and attributes."""
    kw, inputs, want, dtypes = load_case(golden_dir, fname, name)
    lam = inputs["lamdyn"].copy() if "lamdyn" in inputs else None
    ds = _dynspec(inputs["dyn"].copy(), lam)
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        ds.correct_dyn(**kw)
    attr = "lamdyn" if kw["lamsteps"] else "dyn"
    for k, ref in want.items():
        got = getattr(ds, k)
        assert str(got.dtype) == dtypes[k], k
        assert got.shape == ref.shape, k
    for k in ("svd_model", "bandpass"):
        assert hasattr(ds, k) == (k in want)
    if attr != "dyn":                         # the other array: only NaN -> 0, exactly
        assert np.array_equal(ds.dyn, want["dyn"], equal_nan=True)
    sel = inputs[attr]
    if kw["svd"]:
        k = kw["nmodes"]
        a = np.nan_to_num(sel)
        rho = np.zeros(k)                     # the fixture call has no info: use the cap
        s = np.linalg.svd(a, compute_uv=False)
        rho[:] = 1e-11 * s[0] ** 2
        EM, _ = model_bound(a, k, rho, s)
        M = want["svd_model"]
        check_model(ds.svd_model, M, EM)
        assert not np.any(ds.svd_model.imag)
        check_quotient(getattr(ds, attr), a, M, EM)
    else:
        x = np.nan_to_num(sel)
        if attr == "dyn" and (kw["frequency"] or kw["time"]):
            x = np.where(x == 0, np.nan, x)
        check_bandpass_result(getattr(ds, attr), want[attr], kw, x)
        if "bandpass" in want:
            b = want["bandpass"]
            assert np.array_equal(np.isnan(ds.bandpass), np.isnan(b))
            fin = np.isfinite(b)
            assert (np.abs(ds.bandpass - b)[fin] <= 2 * U * np.abs(b)[fin]).all()


@pytest.mark.parametrize("name", ["s1", "s2", "s3", "p3", "full"])
def test_svd_model_on_fixtures(golden_dir, name):
    """ththmod.svd_model returns the reference's complex128 model within the bound, with
    info: converged, steps, singular values against numpy's."""
    from scintools_b200 import ththmod
    kw, inputs, want, _ = load_case(golden_dir, "correct_dyn_svd.npz", name)
    a = np.nan_to_num(inputs["dyn"])
    m, info = ththmod.svd_model(a, kw["nmodes"], return_info=True)
    assert m.dtype == np.complex128 and info["converged"] and not info["tie"]
    k = kw["nmodes"]
    EM, s = model_bound(a, k, info["residuals"])
    check_model(m, want["svd_model"], EM)
    _check_svals(info, s, a)


def _check_svals(info, s, a):
    eps = U * np.sqrt(np.sum(np.asarray(a, dtype=np.float64) ** 2))
    k = info["s"].size
    st = np.zeros(k)
    st[:min(k, s.size)] = s[:k]
    rho = info["residuals"]
    assert (rho <= 1e-11 * max(st[0], 1e-300) ** 2 + 1e-300).all()
    with np.errstate(divide="ignore"):
        sol = np.minimum(np.where(st > 0, 2 * rho / st, np.inf), np.sqrt(rho))
    assert (np.abs(info["s"] - st) <= 2 * (eps + sol) + 1e-300).all()


# ---- prescribed spectra ------------------------------------------------------------------

def prescribed(nf, nt, k, seed=0, s=None):
    """A = sum_i s_i u_i v_i^T with orthonormal factors: s_i = 1 - i / (2k) for i < k, then
    a tail 0.25 * 0.8^(i-k); the truth of the rank-k model needs no SVD."""
    rng = np.random.default_rng(seed)
    if s is None:
        r = min(nf, nt, k + 8)
        s = np.concatenate([1.0 - 0.5 * np.arange(min(k, r)) / k,
                            0.25 * 0.8 ** np.arange(max(r - k, 0))])
    r = s.size
    Uf = np.linalg.qr(rng.normal(size=(nf, r)))[0]
    Vf = np.linalg.qr(rng.normal(size=(nt, r)))[0]
    A = (Uf * s) @ Vf.T
    kk = min(k, r)
    M = (Uf[:, :kk] * s[:kk]) @ Vf[:, :kk].T
    return A, M, s


@pytest.mark.parametrize("nf,nt,k", [(1, 50, 1), (50, 1, 1), (2, 3, 1), (2, 3, 2), (37, 1001, 3),
                                     (1001, 37, 3), (37, 1001, 16), (1024, 2048, 1),
                                     (1024, 2048, 3), (1024, 2048, 16), (1024, 2048, 32),
                                     (4096, 8192, 1), (4096, 8192, 3), (4096, 8192, 32)])
def test_prescribed_spectrum(nf, nt, k):
    """Singular values and the model against the prescribed factors; converged, no tie."""
    from scintools_b200 import ththmod
    A, M, s = prescribed(nf, nt, k, seed=nf + nt + k)
    m, info = ththmod.svd_model(A, k, return_info=True)
    assert info["converged"] and not info["tie"], info
    EM, _ = model_bound(A, k, info["residuals"], s)
    check_model(m, M, EM)
    _check_svals(info, s, A)


def test_rank_deficient_zero_and_constant():
    """Rank < k ends on an exact breakdown with the model = A; the zero matrix gives M = 0
    and an all-NaN correct_dyn (0 / 0, as the reference); a constant matrix gives M = c and
    ones."""
    from scintools_b200 import ththmod
    A, _, s = prescribed(300, 500, 2, seed=3, s=np.array([2.0, 0.5]))
    m, info = ththmod.svd_model(A, 3, return_info=True)
    assert info["converged"] and info["breakdown"] and info["steps"] < 20
    EM, _ = model_bound(A, 3, info["residuals"], s)
    check_model(m, A, EM)
    for shape in [(1, 1), (1, 40), (40, 1), (64, 200)]:
        Z = np.zeros(shape)
        m, info = ththmod.svd_model(Z, 1, return_info=True)
        assert info["converged"] and info["breakdown"] and not m.any() and info["s"][0] == 0
        ds = _dynspec(Z.copy())
        ds.correct_dyn()
        assert np.isnan(ds.dyn).all() and not ds.svd_model.any()
        C = np.full(shape, 2.5)
        m, info = ththmod.svd_model(C, 2, return_info=True)
        assert info["converged"] and info["breakdown"]
        assert np.abs(m.real - 2.5).max() <= 2 * (U * 2.5 * np.sqrt(C.size)) + 4 * U * 2.5
        ds = _dynspec(C.copy())
        ds.correct_dyn()
        assert np.abs(ds.dyn - 1.0).max() <= 8 * U * np.sqrt(C.size) + 4 * U


def test_envelope_corners_and_limits():
    """The four corners of the size envelope run (the largest, 32768 x 16384, on a
    prescribed rank-3 matrix, checked on the device in row blocks); one past either side
    raises ValueError, and the C ABI answers SB_ERR_UNSUPPORTED there."""
    import torch
    from scintools_b200 import _device as D, _lib, ththmod
    for shape in [(1, 1), (1, 16384), (32768, 1)]:
        A = 1.0 + np.random.default_rng(1).random(shape)
        m, info = ththmod.svd_model(A, 1, return_info=True)
        assert info["converged"]
        assert np.abs(m.real - A).max() <= 4 * U * A.max() * np.sqrt(A.size) + 4 * U * A.max()
    nf, nt, k = 32768, 16384, 3
    rng = np.random.default_rng(7)
    s = np.array([3.0, 2.0, 1.0, 0.3])
    Uf = np.linalg.qr(rng.normal(size=(nf, 4)))[0]
    Vf = np.linalg.qr(rng.normal(size=(nt, 4)))[0]
    A = np.empty((nf, nt), np.float32)
    for r0 in range(0, nf, 4096):
        A[r0:r0 + 4096] = (Uf[r0:r0 + 4096] * s) @ Vf.T
    out, model, info = ththmod._svd_run(A, k)
    assert info["converged"] and not info["tie"]
    eps = U * np.sqrt(np.sum(s ** 2))
    sin = np.sqrt(2) * eps / (s[2] - s[3] - eps) + np.linalg.norm(info["residuals"]) / \
        ((s[2] - eps) ** 2 - (s[3] + eps) ** 2)
    EM = 2 * (eps + s[0] * sin)
    Ud = torch.from_numpy(Uf[:, :k] * s[:k]).to(D.device())
    Vd = torch.from_numpy(Vf[:, :k]).to(D.device())
    worst = 0.0
    for r0 in range(0, nf, 4096):
        Mb = Ud[r0:r0 + 4096] @ Vd.T
        err = (model[r0:r0 + 4096].double() - Mb).abs()
        worst = max(worst, float((err / (EM + 2 * U * Mb.abs())).max()))
    assert worst <= 1.0, worst
    assert np.allclose(info["s"], s[:k], rtol=0, atol=4 * eps)
    del out, model
    for shape in [(32769, 1), (1, 16385)]:
        with pytest.raises(ValueError):
            ththmod.svd_model(np.ones(shape, np.float32))
        d = D.empty((8,), torch.float32)
        V = D.empty((8,), torch.float64)
        sv, rs, g, st = np.zeros(1), np.zeros(1), np.zeros(1), np.zeros(4, np.int32)
        rc = _lib.lib.sb_svd_topk(d.data_ptr(), shape[0], shape[1], 1, V.data_ptr(),
                                  sv.ctypes.data, rs.ctypes.data, g.ctypes.data, st.ctypes.data,
                                  D.stream_ptr())
        assert rc == -4
        rc = _lib.lib.sb_bandpass_rows(d.data_ptr(), shape[0], shape[1], 0, V.data_ptr(),
                                       D.stream_ptr())
        assert rc == -4


# ---- realistic data ----------------------------------------------------------------------

def structured_dyn(seed, nf, nt, dead=True):
    rng = np.random.default_rng(seed)
    f = np.linspace(0, 1, nf)
    t = np.linspace(0, 1, nt)
    band = 1.0 + 0.6 * np.sin(2 * np.pi * 1.3 * f) ** 2 + 0.3 * f
    gain = 0.7 + 0.3 * np.cos(2 * np.pi * 0.8 * t) + 0.1 * t
    dyn = band[:, None] * gain[None, :] * rng.exponential(1.0, (nf, nt))
    idx = rng.choice(nf * nt, 400, replace=False)
    dyn.flat[idx[:300]] = 0.0
    dyn.flat[idx[300:]] = np.nan
    if dead:                   # an all-zero channel and sub-integration
        dyn[nf // 3] = 0.0
        dyn[:, nt // 5] = 0.0
    return dyn


def test_realistic_dyn_against_oracle_svd():
    """The notebook's sequence ds.correct_dyn(); ds.calc_sspec() at 1024 x 2048 on a seeded
    dyn with band and gain structure: dyn and svd_model against the oracle's numpy SVD.
    (No all-zero channel here: its model row is 0 and the channel becomes 0/0 = NaN, as in
    the reference, which the notebook avoids by running refill first.)"""
    dyn = structured_dyn(11, 1024, 2048, dead=False)
    ds = _dynspec(dyn.copy())
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)
        ds.correct_dyn()
    a = np.nan_to_num(dyn)
    ref = types_ns(dyn)
    CO.correct_dyn(ref)
    from scintools_b200 import ththmod
    _, info = ththmod.svd_model(a, 1, return_info=True)
    EM, s = model_bound(a, 1, info["residuals"])
    check_model(ds.svd_model, ref.svd_model, EM)
    check_quotient(ds.dyn, a, ref.svd_model, EM)
    _check_svals(info, s, a)
    ds.calc_sspec()
    assert np.isfinite(ds.sspec).any()


def types_ns(dyn, lamdyn=None):
    import types
    o = types.SimpleNamespace(dyn=dyn.copy())
    if lamdyn is not None:
        o.lamdyn = lamdyn.copy()
    return o


@pytest.mark.parametrize("kw", [dict(), dict(nsmooth=7), dict(time=False),
                                dict(frequency=False)])
def test_realistic_bandpass_against_oracle(kw):
    """svd=False at 1024 x 2048 (all-zero channel and sub-integration included) against the
    oracle."""
    dyn = structured_dyn(12, 1024, 2048)
    ds = _dynspec(dyn.copy())
    ds.correct_dyn(svd=False, **kw)
    ref = types_ns(dyn)
    CO.correct_dyn(ref, svd=False, **kw)
    full = dict(frequency=True, time=True, nsmooth=None)
    full.update(kw)
    x = np.where(np.nan_to_num(dyn) == 0, np.nan, np.nan_to_num(dyn))
    check_bandpass_result(ds.dyn, ref.dyn, full, x)
    if full["frequency"]:
        fin = np.isfinite(ref.bandpass)
        assert np.array_equal(np.isfinite(ds.bandpass), fin)
        assert (np.abs(ds.bandpass - ref.bandpass)[fin] <= 2 * U * ref.bandpass[fin]).all()


# ---- behaviour ---------------------------------------------------------------------------

def test_deterministic():
    """Two calls give bit-identical models, quotients, singular values and residuals."""
    from scintools_b200 import ththmod
    A, _, _ = prescribed(2048, 4096, 3, seed=21)
    m1, i1 = ththmod.svd_model(A, 3, return_info=True)
    m2, i2 = ththmod.svd_model(A, 3, return_info=True)
    assert np.array_equal(m1, m2) and np.array_equal(i1["s"], i2["s"])
    assert np.array_equal(i1["residuals"], i2["residuals"]) and i1["steps"] == i2["steps"]
    dyn = structured_dyn(4, 512, 1024)
    out = []
    for _ in range(2):
        ds = _dynspec(dyn.copy())
        ds.correct_dyn(nmodes=2)
        out.append((ds.dyn, ds.svd_model))
        ds = _dynspec(dyn.copy())
        ds.correct_dyn(svd=False, nsmooth=5)
        out.append((ds.dyn, ds.bandpass))
    for a, b in zip(out[:2], out[2:]):
        assert np.array_equal(a[0], b[0], equal_nan=True)
        assert np.array_equal(a[1], b[1], equal_nan=True)


def test_tie_at_the_boundary_is_reported():
    """s_k = s_{k+1}: the truncation is not defined; info reports the tie (not converged)
    and both entry points warn.  Lanczos finds the second copy after its first Krylov space
    breaks down, through the restart."""
    from scintools_b200 import ththmod
    A, _, _ = prescribed(200, 300, 2, seed=5, s=np.array([3.0, 2.0, 2.0, 1.0]))
    with pytest.warns(RuntimeWarning, match="equal"):
        m, info = ththmod.svd_model(A, 2, return_info=True)
    assert info["tie"] and not info["converged"]
    assert np.allclose(info["s"], [3.0, 2.0], atol=1e-5)
    ds = _dynspec(A.copy())
    with pytest.warns(RuntimeWarning, match="equal"):
        ds.correct_dyn(nmodes=2)
    assert hasattr(ds, "svd_model")
    m, info = ththmod.svd_model(A, 3, return_info=True)     # a gap at 3: fine
    assert info["converged"] and not info["tie"]


def test_dtypes_side_effects_and_scale_dyn():
    """dtype=float32 gives float32 / complex64 with the same values; the warning print on a
    second call; a missing lamdyn is made by scale_dyn first; NaN pixels of the caller's
    array are zeroed in place."""
    from scintools_b200 import BasicDyn, Dynspec
    dyn = structured_dyn(6, 64, 128)
    ds64, ds32 = _dynspec(dyn.copy()), _dynspec(dyn.copy())
    ds64.correct_dyn()
    ds32.correct_dyn(dtype=np.float32)
    assert ds32.dyn.dtype == np.float32 and ds32.svd_model.dtype == np.complex64
    assert np.array_equal(ds32.dyn.astype(np.float64), ds64.dyn, equal_nan=True)
    ds32.correct_dyn(svd=False, dtype=np.float32)
    assert ds32.bandpass.dtype == np.float32
    import io
    import contextlib
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        ds64.correct_dyn()
    assert "Warning: An svd_model exists" in buf.getvalue()
    caller = dyn.copy()
    ds = _dynspec(caller)
    ds.correct_dyn(svd=False)
    assert not np.isnan(caller).any()
    t = np.arange(128) * 8.0
    f = 1400.0 + np.arange(64) * 0.25
    a = Dynspec(dyn=BasicDyn(np.nan_to_num(dyn), times=t, freqs=f, dt=8.0, df=0.25),
                verbose=False)
    b = Dynspec(dyn=BasicDyn(np.nan_to_num(dyn), times=t, freqs=f, dt=8.0, df=0.25),
                verbose=False)
    a.correct_dyn(lamsteps=True)
    b.scale_dyn()
    b.correct_dyn(lamsteps=True)
    assert np.array_equal(a.lamdyn, b.lamdyn, equal_nan=True)
    assert np.array_equal(a.svd_model, b.svd_model)
