"""GPU tests of Dynspec.refill and dynspec.inpaint_biharmonic (csrc/inpaint.cu).

Biharmonic: against the oracle's spsolve (oracle/refill_oracle.py) on several mask shapes,
with the bar max |got - ref| <= 1e-7 (max - min of the known pixels).  The solver stops at
||b - A x|| <= 1e-10 ||b||; the error that leaves grows with the condition number of the
system (about L^4 for a hole of width L), so the bar is an empirical one: every case prints
its error and iteration count.  Median and mean: bit for bit against the reference's
fixtures and scipy.signal.medfilt.
"""
import glob
import os

import numpy as np
import pytest

from oracle import refill_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "refill_*.npz")))
BAR = 1e-7


def _ds(dyn):
    from scintools_b200.dynspec import BasicDyn, Dynspec
    nf, nt = dyn.shape
    return Dynspec(dyn=BasicDyn(dyn, times=np.arange(max(nt, 3)) * 10.0,
                                freqs=1400.0 + 0.1 * np.arange(max(nf, 3))), verbose=False)


def _inpaint(img, mask):
    from scintools_b200.dynspec import inpaint_biharmonic
    return inpaint_biharmonic(img, mask, return_info=True)


def _kw(z):
    ks = z["kernel_size"]
    return dict(method=str(z["method"]), zeros=bool(z["zeros"]),
                kernel_size=int(ks) if ks.shape == () else tuple(int(k) for k in ks),
                linear=bool(z["linear"]))


@pytest.mark.parametrize("fn", FIXTURES, ids=[os.path.basename(f)[7:-4] for f in FIXTURES])
def test_fixture_parity(fn):
    """refill in place: median / mean bit for bit against the reference, biharmonic within
    the bar of the oracle's fixture."""
    z = np.load(fn)
    dyn = z["dyn_in"].copy()
    ds = _ds(dyn)
    ds.refill(**_kw(z))
    assert ds.dyn is dyn                        # filled in place
    ref = z["dyn_out"]
    if str(z["source"]) == "reference":
        assert np.array_equal(dyn, ref)
    else:
        d = z["dyn_in"]
        known = d[~(np.isnan(d) | (d == 0))]
        err = np.max(np.abs(dyn - ref)) / (known.max() - known.min())
        print("%s: max err %.2e of the known range" % (os.path.basename(fn), err))
        assert err <= BAR


def _masks():
    rng = np.random.default_rng(7)
    nf, nt = 96, 128
    out = {}
    out["random5"] = rng.random((nf, nt)) < 0.05
    out["random20"] = rng.random((nf, nt)) < 0.20
    m = np.zeros((nf, nt), bool)
    m[[3, 40, 41, 90], :] = True
    m[:, [0, 17, 64, 65, 127]] = True
    out["channels_subints"] = m
    m = np.zeros((nf, nt), bool)
    m[30:62, 50:82] = True
    out["block32"] = m
    m = np.zeros((nf, nt), bool)
    m[0, 40:50] = m[nf - 1, 60:75] = m[30:40, 0] = m[50:58, nt - 1] = True     # edges
    m[:3, :4] = m[:2, nt - 3:] = m[nf - 4:, :2] = m[nf - 3:, nt - 5:] = True    # corners
    m[1, 20:23] = m[nf - 2, 100] = m[70, 1] = m[20, nt - 2] = True               # 1 px in
    out["edges_corners"] = m
    m = np.zeros((nf, nt), bool)
    m[45, 77] = True
    out["single"] = m
    return out


MASKS = _masks()


@pytest.mark.parametrize("name", sorted(MASKS))
def test_against_spsolve(name):
    rng = np.random.default_rng(len(name))
    mask = MASKS[name]
    img = rng.exponential(1.0, mask.shape)
    img[mask] = np.nan
    ref = O.biharmonic(img, mask)
    got, info = _inpaint(img, mask)
    known = img[~mask]
    err = np.max(np.abs(got - ref)) / (known.max() - known.min())
    print("%s: %d unknowns, %d iterations (%d restarts), residual %.2e, max err %.2e"
          % (name, mask.sum(), info["iterations"], info["restarts"], info["residual"], err))
    assert info["converged"] and info["residual"] <= 1e-10
    assert np.array_equal(got[~mask], img[~mask])
    assert err <= BAR


@pytest.mark.parametrize("shape", [(300, 1), (1, 300)])
def test_one_pixel_wide(shape):
    rng = np.random.default_rng(3)
    img = rng.normal(size=shape)
    mask = np.zeros(shape, bool)
    flat = mask.ravel()
    flat[[0, 1, 50, 51, 52, 120, 298, 299]] = True
    flat[200:230] = True
    img[mask] = np.nan
    ref = O.biharmonic(img, mask)
    got, info = _inpaint(img, mask)
    known = img[~mask]
    err = np.max(np.abs(got - ref)) / (known.max() - known.min())
    print("%s: %d iterations, residual %.2e, max err %.2e"
          % (shape, info["iterations"], info["residual"], err))
    assert info["converged"] and err <= BAR


def test_cubic_known_answer():
    f, mask = O.cubic_case()
    got, info = _inpaint(np.where(mask, np.nan, f), mask)
    known = f[~mask]
    err = np.max(np.abs(got - f)) / (known.max() - known.min())
    print("cubic: %d iterations, max err %.2e of the known range" % (info["iterations"], err))
    assert info["converged"] and err <= BAR


@pytest.mark.parametrize("ks", [3, 5, 7, (3, 5), 31])
def test_median_is_medfilt(ks):
    """The masked median equals scipy.signal.medfilt at every filled pixel, bit for bit,
    including windows past the image edge (31 on a 40 x 50 image)."""
    rng = np.random.default_rng(11)
    dyn = rng.exponential(1.0, (40, 50))
    dyn[rng.random(dyn.shape) < 0.1] = np.nan
    dyn[5, :] = 0.0
    ref = O.refill(dyn, method="median", kernel_size=ks)
    ds = _ds(dyn.copy())
    ds.refill(method="median", kernel_size=ks)
    assert np.array_equal(ds.dyn, ref)


def test_in_place_effects():
    """zeros become NaN and are then filled; zeros=False leaves them; the object is kept."""
    rng = np.random.default_rng(12)
    dyn = rng.exponential(1.0, (20, 30))
    dyn[4, 5] = 0.0
    dyn[7, 8] = np.nan
    for zeros in (True, False):
        for method in ("biharmonic", "median", "mean"):
            d = dyn.copy()
            ds = _ds(d)
            ds.refill(method=method, zeros=zeros)
            assert ds.dyn is d and not np.any(np.isnan(d))
            assert (d[4, 5] == 0.0) == (not zeros)
            if method != "biharmonic":
                assert np.array_equal(d, O.refill(dyn, method=method, zeros=zeros))


def test_large_residual_and_clip():
    """4096 x 8192 with about 1.7 M unknowns: the float64 residual of the discrete system,
    formed on the host with a sparse mat-vec, meets the stopping rule; the values lie in
    the known range; a second solve is bit-identical, with the same steps and restarts."""
    rng = np.random.default_rng(13)
    nf, nt = 4096, 8192
    i = np.arange(nf)[:, None]
    j = np.arange(nt)[None, :]
    img = np.sin(i / 150.0) * np.cos(j / 230.0) + 1e-3 * rng.normal(size=(nf, nt))
    mask = rng.random((nf, nt)) < 0.05
    mask[[100, 101, 2000, 4095], :] = True
    mask[:, [0, 3000, 3001, 6000]] = True
    mask[1000:1064, 5000:5256] = True
    img[mask] = np.nan
    got, info = _inpaint(img, mask)
    again, info2 = _inpaint(img, mask)          # 528 blocks per launch: repeats bit for bit
    assert np.array_equal(got.view(np.uint64), again.view(np.uint64)) and info == info2
    known = img[~mask]
    x = got[mask]
    print("large: %d unknowns, %d iterations (%d restarts), residual %.2e"
          % (mask.sum(), info["iterations"], info["restarts"], info["residual"]))
    assert 1.6e6 < mask.sum() < 1.9e6
    assert info["converged"]
    assert np.all(x >= known.min()) and np.all(x <= known.max())
    clipped = (x == known.min()) | (x == known.max())
    A, b, pix = O.system(img, mask)
    r = b - A @ x
    if clipped.any():        # rows that touch a clipped unknown do not see the solver's x
        touch = np.asarray((abs(A) @ clipped.astype(float)) > 0).ravel()
        r = r[~touch]
    rel = np.linalg.norm(r) / np.linalg.norm(b)
    print("large: host residual %.2e, %d clipped" % (rel, clipped.sum()))
    assert rel <= 1e-10 * (1 + 1e-6)


def test_half_step_stop_in_every_block():
    """Isolated pixels, none within two of another: the Jacobi-scaled matrix is the
    identity, so the run stops in kernel C of the first step (the half step).  With about
    470 k unknowns every one of the 528 blocks of that launch must still apply its share of
    the last x update, whatever order the blocks run in."""
    rng = np.random.default_rng(17)
    nf, nt = 2048, 2048
    img = rng.exponential(1.0, (nf, nt))
    mask = np.zeros((nf, nt), bool)
    mask[::3, ::3] = True
    img[mask] = np.nan
    ref = O.biharmonic(img, mask)
    for _ in range(2):
        got, info = _inpaint(img, mask)
        known = img[~mask]
        err = np.max(np.abs(got - ref)) / (known.max() - known.min())
        print("isolated: %d unknowns, %d iterations (%d restarts), max err %.2e"
              % (mask.sum(), info["iterations"], info["restarts"], err))
        assert info["converged"] and info["iterations"] == 1 and info["restarts"] == 0
        assert err <= BAR


def test_large_block_tolerance():
    """A 64 x 256 hole, larger than any above: refill's tol reaches the solver, and
    tol=1e-13 brings the fill within the bar of spsolve (the default 1e-10 does not, see
    DESIGN.md section 5a; its error is printed)."""
    from scintools_b200.dynspec import inpaint_biharmonic
    rng = np.random.default_rng(18)
    nf, nt = 128, 384
    i = np.arange(nf)[:, None]
    j = np.arange(nt)[None, :]
    dyn = np.sin(i / 40.0) * np.cos(j / 60.0) + 1e-3 * rng.normal(size=(nf, nt)) + 2.0
    mask = rng.random((nf, nt)) < 0.05
    mask[32:96, 64:320] = True
    dyn[mask] = np.nan
    ref = O.biharmonic(dyn, mask)
    known = dyn[~mask]
    for tol in (1e-10, 1e-13):
        got, info = inpaint_biharmonic(dyn, mask, return_info=True, tol=tol)
        err = np.max(np.abs(got - ref)) / (known.max() - known.min())
        print("64 x 256 block, tol %.0e: %d iterations (%d restarts), residual %.2e, max err "
              "%.2e" % (tol, info["iterations"], info["restarts"], info["residual"], err))
        assert info["converged"] and info["residual"] <= tol
    assert err <= BAR
    d = dyn.copy()
    ds = _ds(d)
    ds.refill(tol=1e-13)
    assert np.array_equal(d, got)


def test_deterministic():
    mask = MASKS["random20"] | MASKS["block32"]
    img = np.random.default_rng(14).exponential(1.0, mask.shape)
    img[mask] = np.nan
    a, ia = _inpaint(img, mask)
    b, ib = _inpaint(img, mask)
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64)) and ia == ib


def test_limits_both_sides():
    from scintools_b200.dynspec import inpaint_biharmonic
    rng = np.random.default_rng(15)
    base = rng.normal(size=(10, 12))
    base[3, 4] = np.nan
    d = base.copy()
    d[0, 0] = np.inf
    with pytest.raises(ValueError):
        _ds(d).refill()
    _ds(base.copy()).refill()                              # the same without the inf
    with pytest.raises(ValueError):
        _ds(np.full((5, 6), np.nan)).refill()
    d = np.full((5, 6), np.nan)
    d[2, 3] = 1.5                                          # one known pixel is enough
    ds = _ds(d)
    ds.refill()
    assert np.all(ds.dyn == 1.5)
    for shape in [(32769, 1), (1, 16385)]:
        with pytest.raises(ValueError):
            inpaint_biharmonic(np.zeros(shape), np.zeros(shape, bool))
    for shape in [(32768, 1), (1, 16384)]:
        img = np.arange(np.prod(shape), dtype=np.float64).reshape(shape)
        mask = np.zeros(shape, bool)
        mask.ravel()[[5, 700, 9000]] = True
        got, info = inpaint_biharmonic(img, mask, return_info=True)
        assert info["converged"]
        assert np.max(np.abs(got - img)) <= 1e-6 * img.max()          # linear: exact
    for method in ("linear", "cubic", "nearest"):
        with pytest.raises(NotImplementedError):
            _ds(base.copy()).refill(method=method)


def test_cap_warns_and_stores():
    from scintools_b200.dynspec import inpaint_biharmonic
    mask = MASKS["block32"]
    img = np.random.default_rng(16).exponential(1.0, mask.shape)
    with pytest.warns(RuntimeWarning):
        got, info = inpaint_biharmonic(img, mask, return_info=True, maxit=5)
    assert not info["converged"] and info["iterations"] == 5
    assert np.all(np.isfinite(got))
