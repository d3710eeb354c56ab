"""Wavefield mosaic fit on the GPU (sb_mosaic_*, ththmod.rotInit ... fullMosHess) against the
float64 oracle (oracle/mosaic_oracle.py) on the reference's fixtures.

Bound.  Every device result is a float64 sum of per-pixel terms computed in float32.  To
first order a float32 value made of k rounded operations has relative error <= k u,
u = 2^-24, against the magnitude the oracle reports as sum|terms| (which replaces |W| by
Wabs = sum |A y| and |wt| by Wabs^2 + |dspec|).  Per term, in the tile kernel:
  y = m (chunk e^{i phi}): cos / sin rounded 0.5, the complex product 3, the two ramps
      0.5 + 0.5 and their product 1, m * z 1                                  ->  6.5 u
  W = sum A y: A rounded 0.5, A * y 1, three additions 3, on top of y           -> 11 u
  rotFit |W|^2: 2 x 11 + square and add 2 = 24 u; rotDer Im(conj(W) y):
      11 + 6.5 + two products and a difference 3 = 20.5 u                       -> c = 24
  overlap y_u conj(y_v) (no phase, e = 1 exactly): 2 x 3 + 3                     -> c = 9
  wt = |W|^2 - dspec: 24 + 1 = 25 u against Wabs^2 + |dspec|; N^2 1, division 1;
  chi-square wt^2 / N^2: 2 x 25 + 1 + 2 = 53 u; gradient 4 wt t / N^2 with
      t = y conj(W) (6.5 + 11 + 3 = 20.5): 25 + 20.5 + 2 + 2 = 49.5 u;
  Hessian 8 t_u t_v + 4 wt g (g = y_u conj(y_v): 6.5 + 6.5 + 3 = 16):
      max(2 x 20.5 + 2, 25 + 16 + 1) + sum 1 + N^2 and division 2 = 46 u         -> c = 56
The amplitudes multiplying the Hessian's pair sums are applied in float64.  The float64
accumulation (at most 2^28 terms) adds less than 2^-25 u.  rotInit propagates the overlap
bound (c = 9) through its recurrence to first order (mosaic_oracle.rot_init).
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_MOS, C_ROT, C_OVL, C_FIT = 12, 24, 9, 56


def _case(golden_dir, name, pre):
    f = np.load(os.path.join(golden_dir, name + ".npz"))
    return {k[len(pre):]: f[k] for k in f.files if k.startswith(pre) and
            (pre or not k.startswith("b2_"))}


def _within(got, ref, mag, c):
    got, ref, mag = np.asarray(got), np.asarray(ref), np.asarray(mag)
    assert got.shape == ref.shape
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref)
    err = np.abs(got - ref)[fin]
    bar = c * U * mag[fin] + 1e-30
    assert (err <= bar).all(), float((err / bar).max())
    return float((err / bar).max()) if err.size else 0.0


@pytest.mark.parametrize("name,pre", [("mosaic_sample", ""), ("mosaic_synth", ""),
                                      ("mosaic_synth", "b2_")])
def test_mosaic_functions_against_oracle(golden_dir, name, pre):
    from oracle import mosaic_oracle as MO
    from scintools_b200 import ththmod as T
    c = _case(golden_dir, name, pre)
    ch, x, p, D, N = c["chunks"], c["x"], c["p"], c["dspec"], c["N"]
    if "rotMos" not in c:       # case a stores one copy: p = (x, ones) there
        P = ch.shape[0] * ch.shape[1]
        assert np.array_equal(p, np.concatenate([x, np.ones(P)]))
        c["rotMos"] = c["fullMos"]
    nF, nT = c["fullMos"].shape
    W, Wa = MO.rot_mos(ch, x)
    _within(T.rotMos(ch, x), W, Wa, C_MOS)
    W, Wa = MO.full_mos(ch, p)
    _within(T.fullMos(ch, p), W, Wa, C_MOS)
    v, a = MO.rot_fit(ch, x)
    _within(T.rotFit(x, ch), v, a, C_ROT)
    v, a = MO.rot_der(ch, x)
    got = T.rotDer(x, ch)
    assert got.shape == x.shape
    _within(got, v, a, C_ROT)
    v, a = MO.full_fit(ch, p, D, N)
    _within(T.fullMosFit(p, ch, D, N), v, a, C_FIT)
    v, a = MO.full_grad(ch, p, D[:nF, :nT], N)
    _within(T.fullMosGrad(p, ch, D[:nF, :nT], N), v, a, C_FIT)
    v, a = MO.full_hess(ch, p, D[:nF, :nT], N)
    H = T.fullMosHess(p, ch, D[:nF, :nT], N)
    _within(H, v, a, C_FIT)
    assert np.array_equal(np.isnan(H), np.isnan(H.T))
    xi, err = MO.rot_init(ch, C_OVL * U)
    got = T.rotInit(ch)
    nz = np.abs(ch).reshape(-1, ch.shape[2] * ch.shape[3]).max(1)[1:] > 0
    d = np.abs(np.angle(np.exp(1j * (got - xi))))
    assert (d[nz] <= err[nz] + 1e-12).all()
    assert (got[~nz] == 0).all()


def test_rotmos_of_rotinit_is_mosaic(golden_dir):
    from scintools_b200 import ththmod as T
    c = _case(golden_dir, "mosaic_synth", "")
    ch = c["chunks"]
    W = T.rotMos(ch, T.rotInit(ch))
    ref = T.mosaic(ch.astype(complex))
    assert np.abs(W - ref).max() <= 1e-5 * np.abs(ref).max()


def test_model_sparse_deterministic_and_cached(golden_dir):
    from scintools_b200 import _lib
    from scintools_b200 import ththmod as T
    c = _case(golden_dir, "mosaic_sample", "")
    ch, p, D, N = c["chunks"], c["p"], c["dspec"], c["N"]
    m = T.MosaicModel(ch, D, N)
    H = m.hess(p)
    Hs = m.hess(p, sparse=True)
    assert np.array_equal(Hs.toarray(), H)
    m2 = T.MosaicModel(ch, D, N)
    q = p + 0.01
    assert m2.fit(q) == m.fit(q) and np.array_equal(m2.grad(q), m.grad(q))
    assert np.array_equal(m2.hess(q), m.hess(q))
    n0 = _lib.lib.sb_launch_count()
    m.fit(p - 0.01)
    n1 = _lib.lib.sb_launch_count()
    m.grad(p - 0.01)
    assert _lib.lib.sb_launch_count() == n1          # grad shares the fit pass
    m.hess(p - 0.01)
    n2 = _lib.lib.sb_launch_count()
    m.hess(p + 0.02)
    n3 = _lib.lib.sb_launch_count()
    assert n3 - n2 == (n2 - n1) + 1                  # only the new p builds the mosaic again
    assert n1 - n0 >= 2


def test_known_answer_newton_fit(golden_dir):
    """Chunks E a_k e^{i psi_k} of one wavefield with |E|^2 = dspec: the fit from rotInit
    and A = 1 reaches A_k e^{i phi_k} = e^{i psi_0} / (a_k e^{i psi_k}) up to one sign."""
    from scipy.optimize import minimize
    from scintools_b200 import ththmod as T
    rng = np.random.default_rng(5)
    ncf, nct, cwf, cwt = 3, 3, 16, 16
    nF, nT = (ncf + 1) * cwf // 2, (nct + 1) * cwt // 2
    E = rng.normal(size=(nF, nT)) + 1j * rng.normal(size=(nF, nT)) + 2
    P = ncf * nct
    a = rng.uniform(0.7, 1.4, P)
    psi = rng.uniform(-np.pi, np.pi, P)
    ch = np.zeros((ncf, nct, cwf, cwt), complex)
    for k in range(P):
        cf, ct = divmod(k, nct)
        ch[cf, ct] = E[cf * cwf // 2:cf * cwf // 2 + cwf, ct * cwt // 2:ct * cwt // 2 + cwt] * \
            a[k] * np.exp(1j * psi[k])
    ch = ch.astype(np.complex64)
    D = np.abs(E) ** 2
    N = np.ones_like(D)
    m = T.MosaicModel(ch, D, N)
    x0 = m.rot_init()
    want = np.exp(1j * psi[0]) / (a * np.exp(1j * psi))
    assert np.abs(np.angle(np.exp(1j * (x0 - np.angle(want[1:] / want[0]))))).max() < 1e-4
    p0 = np.concatenate([x0, np.ones(P)])
    res = minimize(m.fit, p0, jac=m.grad, hess=m.hess, method="trust-exact")
    # converged, or stopped at the float32 floor of the fit (status 2: the model no longer
    # predicts the float32 decrease) after the gradient fell by more than 10^3
    g0 = np.abs(m.grad(p0)).max()
    assert res.success or (res.status == 2 and np.abs(res.jac).max() < 1e-3 * g0), res.message
    A = res.x[P - 1:] * np.exp(1j * np.concatenate([[0], res.x[:P - 1]]))
    s = np.sign(np.real(A[0] / want[0]))
    assert np.abs(A * s - want).max() < 1e-3 * np.abs(want).max()
    assert res.fun < 1e-6 * np.sum(D ** 2)


@pytest.mark.parametrize("ncf,nct,cwf,cwt", [(256, 257, 2, 2), (65536, 1, 2, 4)])
def test_counts_past_65535(ncf, nct, cwf, cwt):
    from oracle import mosaic_oracle as MO
    from scintools_b200 import ththmod as T
    rng = np.random.default_rng(ncf)
    ch = (rng.normal(size=(ncf, nct, cwf, cwt)) +
          1j * rng.normal(size=(ncf, nct, cwf, cwt))).astype(np.complex64)
    P = ncf * nct
    p = np.concatenate([rng.uniform(-3, 3, P - 1), rng.uniform(0.5, 2, P)])
    m = MO.Layers(ch)
    D = (rng.uniform(0, 4, m.shape)).astype(np.float32)
    N = np.ones(m.shape, np.float32)
    mod = T.MosaicModel(ch, D, N)
    W, Wa = MO.full_mos(ch, p)
    _within(mod.full_mos(p), W, Wa, C_MOS)
    v, a = MO.full_grad(ch, p, D, N)
    _within(mod.grad(p), v, a, C_FIT)
    Hs = mod.hess(p, sparse=True).tocoo()
    ref, mag = MO.full_hess(ch, p, D, N, sparse=True)
    ref, mag = ref.tocsr(), mag.tocsr()
    r, c = Hs.row, Hs.col
    assert len(r) == ref.nnz                        # the same entries, each once
    want = np.asarray(ref[r, c]).ravel()
    bar = C_FIT * U * np.asarray(mag[r, c]).ravel() + 1e-30
    assert (np.abs(Hs.data - want) <= bar).all(), float((np.abs(Hs.data - want) / bar).max())


def test_known_answer_sparse_trust_constr():
    """The same known answer at 32 x 32 chunks of 8 x 8 (2047 parameters) with the sparse
    Hessian handed to trust-constr."""
    from scipy.optimize import minimize
    from scintools_b200 import ththmod as T
    rng = np.random.default_rng(6)
    ncf, nct, cwf, cwt = 32, 32, 8, 8
    nF, nT = (ncf + 1) * cwf // 2, (nct + 1) * cwt // 2
    E = rng.normal(size=(nF, nT)) + 1j * rng.normal(size=(nF, nT)) + 2
    P = ncf * nct
    a = rng.uniform(0.7, 1.4, P)
    psi = rng.uniform(-np.pi, np.pi, P)
    ch = np.zeros((ncf, nct, cwf, cwt), complex)
    for k in range(P):
        cf, ct = divmod(k, nct)
        ch[cf, ct] = E[cf * cwf // 2:cf * cwf // 2 + cwf, ct * cwt // 2:ct * cwt // 2 + cwt] * \
            a[k] * np.exp(1j * psi[k])
    ch = ch.astype(np.complex64)
    D = np.abs(E) ** 2
    N = np.ones_like(D)
    m = T.MosaicModel(ch, D, N)
    p0 = np.concatenate([m.rot_init(), np.ones(P)])
    # the float32 pixels leave a gradient floor near 1e-4 (|wt| ~ 1e-6 |dspec| per pixel);
    # the start's gradient is ~1e4 and a gradient of 1e-3 means amplitude errors ~1e-7
    res = minimize(m.fit, p0, jac=m.grad, hess=lambda q: m.hess(q, sparse=True),
                   method="trust-constr", options=dict(gtol=1e-3, xtol=1e-12, maxiter=200))
    assert res.success, res.message
    want = np.exp(1j * psi[0]) / (a * np.exp(1j * psi))
    A = res.x[P - 1:] * np.exp(1j * np.concatenate([[0], res.x[:P - 1]]))
    s = np.sign(np.real(A[0] / want[0]))
    assert np.abs(A * s - want).max() < 1e-3 * np.abs(want).max()
    assert res.fun < 1e-6 * np.sum(D ** 2)
