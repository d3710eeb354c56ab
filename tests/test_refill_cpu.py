"""CPU tests of Dynspec.refill: the float64 oracle (oracle/refill_oracle.py) against the
reference's fixtures (tests/golden/refill_*.npz, made by oracle/make_golden_refill.py), the
biharmonic stencils at every edge and corner, the known answer of a cubic field, and the
argument errors of the port raised before any device call."""
import glob
import os

import numpy as np
import pytest
from scipy.ndimage import laplace

from oracle import refill_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "refill_*.npz")))


def _kw(z):
    ks = z["kernel_size"]
    return dict(method=str(z["method"]), zeros=bool(z["zeros"]),
                kernel_size=int(ks) if ks.shape == () else tuple(int(k) for k in ks),
                linear=bool(z["linear"]))


@pytest.mark.parametrize("fn", FIXTURES, ids=[os.path.basename(f)[7:-4] for f in FIXTURES])
def test_oracle_matches_fixtures(fn):
    """Median and mean fills bit for bit against the reference; the biharmonic fixtures are
    the oracle's own output (kept to pin it)."""
    z = np.load(fn)
    got = O.refill(z["dyn_in"], **_kw(z))
    assert not np.any(np.isnan(got))
    assert np.array_equal(got, z["dyn_out"])


def test_fixtures_cover_the_cases():
    names = {os.path.basename(f)[7:-4] for f in FIXTURES}
    assert names == {"median_k3", "median_k5", "median_k3x7", "median_k5_nozeros", "mean",
                     "mean_nozeros", "linear_off", "biharmonic", "biharmonic_nozeros"}
    assert sum(os.path.getsize(f) for f in FIXTURES) < 400_000
    for f in FIXTURES:
        z = np.load(f)
        assert str(z["source"]) == ("oracle" if "biharmonic" in f else "reference")
        d = z["dyn_in"]
        assert np.isnan(d).any() and (d == 0).any()
        # the fills changed only the NaN pixels (and the zeros with zeros=True)
        gap = np.isnan(d) | ((d == 0) if bool(z["zeros"]) else False)
        assert np.array_equal(z["dyn_out"][~gap], d[~gap])


def _direct_stencil(nf, nt, i, j):
    """laplace(laplace(e_p)) on the clipped 5x5 box, placed in a 5x5 array centred on p."""
    li, lj = max(i - 2, 0), max(j - 2, 0)
    hi, hj = min(i + 3, nf), min(j + 3, nt)
    e = np.zeros((hi - li, hj - lj))
    e[i - li, j - lj] = 1.0
    S = laplace(laplace(e))
    out = np.zeros((5, 5))
    out[li - i + 2:hi - i + 2, lj - j + 2:hj - j + 2] = S
    return out


@pytest.mark.parametrize("shape", [(1, 1), (1, 7), (7, 1), (2, 3), (3, 9), (4, 4), (6, 11),
                                   (9, 5), (12, 13)])
def test_border_stencils(shape):
    """The port's class tables and the oracle's per-box stencils are laplace(laplace(e_p)) on
    the clipped box at every pixel: every edge, every corner, images narrower than 5."""
    from scintools_b200.dynspec import _stencil_tables
    nf, nt = shape
    rcls, ccls, tables = _stencil_tables(nf, nt)
    assert tables.shape[0] <= 5 and tables.shape[1] <= 5
    for i in range(nf):
        for j in range(nt):
            ref = _direct_stencil(nf, nt, i, j)
            assert np.array_equal(tables[rcls[i], ccls[j]], ref), (i, j)
            (lo_i, er, oi), (lo_j, ec, oj) = O.box(nf, i), O.box(nt, j)
            S = O.stencil((er, ec), (oi, oj))
            assert np.array_equal(ref[2 - oi:2 - oi + er, 2 - oj:2 - oj + ec], S)
    if nf >= 5 and nt >= 5:
        inner = tables[rcls[nf // 2], ccls[nt // 2]]
        want = np.zeros((5, 5))
        want[2, 2] = 20
        want[1, 2] = want[3, 2] = want[2, 1] = want[2, 3] = -8
        want[1, 1] = want[1, 3] = want[3, 1] = want[3, 3] = 2
        want[0, 2] = want[4, 2] = want[2, 0] = want[2, 4] = 1
        assert np.array_equal(inner, want)


def test_oracle_system_rows_are_the_stencils():
    rng = np.random.default_rng(4)
    nf, nt = 9, 7
    img = rng.normal(size=(nf, nt))
    mask = rng.random((nf, nt)) < 0.4
    A, b, pix = O.system(img, mask)
    A = A.toarray()
    for k, p in enumerate(pix):
        i, j = divmod(int(p), nt)
        S = _direct_stencil(nf, nt, i, j)
        row, rhs = np.zeros(pix.size), 0.0
        for di in range(-2, 3):
            for dj in range(-2, 3):
                ii, jj = i + di, j + dj
                if 0 <= ii < nf and 0 <= jj < nt and S[di + 2, dj + 2] != 0:
                    q = ii * nt + jj
                    if mask[ii, jj]:
                        row[np.searchsorted(pix, q)] = S[di + 2, dj + 2]
                    else:
                        rhs -= S[di + 2, dj + 2] * img[ii, jj]
        assert np.array_equal(A[k], row)
        assert abs(b[k] - rhs) <= 1e-13 * max(1.0, abs(rhs))


def test_cubic_known_answer():
    f, mask = O.cubic_case()
    assert f[mask].min() > f[~mask].min() and f[mask].max() < f[~mask].max()
    g = O.biharmonic(np.where(mask, np.nan, f), mask)
    assert np.max(np.abs(g - f)) <= 1e-9 * np.max(np.abs(f))


# ---- Python layer -------------------------------------------------------------------------
def _ds(dyn):
    from scintools_b200.dynspec import BasicDyn, Dynspec
    nf, nt = dyn.shape
    return Dynspec(dyn=BasicDyn(dyn, times=np.arange(max(nt, 3)) * 10.0,
                                freqs=1400.0 + 0.1 * np.arange(max(nf, 3))), verbose=False)


def test_argument_errors_before_device(monkeypatch):
    """Every ValueError / NotImplementedError of refill and inpaint_biharmonic is raised
    before any device call, and self.dyn is left as it was."""
    from scintools_b200 import _device, dynspec

    def no_device(*a, **k):
        raise AssertionError("device touched")

    monkeypatch.setattr(_device, "device", no_device)
    rng = np.random.default_rng(0)
    base = rng.normal(size=(8, 9))
    base[2, 3] = np.nan
    base[4, 4] = 0.0
    cases = []
    d = base.copy()
    d[1, 1] = np.inf
    cases += [(d, dict(method="biharmonic")), (d, dict(method="median", kernel_size=3))]
    d = base.copy()
    d[1, 1] = -np.inf
    cases.append((d, dict(method="biharmonic")))
    cases.append((np.full((4, 5), np.nan), dict(method="biharmonic")))
    d = np.zeros((4, 5))
    d[0, 0] = np.nan
    cases.append((d, dict(method="median", kernel_size=3)))      # zeros -> all masked
    cases.append((np.zeros((32769, 1)), dict(method="biharmonic", zeros=False)))
    cases.append((np.zeros((1, 16385)), dict(method="median", zeros=False, kernel_size=3)))
    for ks in (4, (3, 4), 33, 0, (3, 5, 7), 2.5):
        cases.append((base.copy(), dict(method="median", kernel_size=ks)))
    for dyn, kw in cases:
        ds = _ds(dyn)
        before = ds.dyn.copy()
        with pytest.raises(ValueError):
            ds.refill(**kw)
        assert ds.dyn is dyn
        assert np.array_equal(ds.dyn, before, equal_nan=True), kw
    for method in ("linear", "cubic", "nearest"):
        ds = _ds(base.copy())
        with pytest.raises(NotImplementedError):
            ds.refill(method=method)
        assert np.array_equal(ds.dyn, base, equal_nan=True)
    img = rng.normal(size=(6, 6))
    mask = np.zeros((6, 6), bool)
    mask[2, 2] = True
    bad = img.copy()
    bad[0, 0] = np.nan                                           # NaN outside the mask
    for im, m in [(bad, mask), (img, np.ones((6, 6))), (img, mask[:5]), (img[0], mask[0]),
                  (np.where(mask, np.inf, img), mask)]:
        with pytest.raises(ValueError):
            dynspec.inpaint_biharmonic(im, m)


def test_host_paths_without_device(monkeypatch):
    """'mean', unknown names, linear=False and masks with nothing to fill never reach the
    device; they match the oracle bit for bit."""
    from scintools_b200 import _device

    def no_device(*a, **k):
        raise AssertionError("device touched")

    monkeypatch.setattr(_device, "device", no_device)
    z = np.load(os.path.join(ROOT, "tests", "golden", "refill_mean.npz"))
    for kw in (dict(method="mean"), dict(method="mean", zeros=False),
               dict(method="linear", linear=False), dict(method="other")):
        ds = _ds(z["dyn_in"].copy())
        ds.refill(**kw)
        assert np.array_equal(ds.dyn, O.refill(z["dyn_in"], **kw))
    full = np.random.default_rng(1).normal(size=(6, 7)) + 5.0
    for method in ("biharmonic", "median"):
        ds = _ds(full.copy())
        ds.refill(method=method)
        assert np.array_equal(ds.dyn, full)


def test_library_exports_refill_symbols():
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _lib
    for name in ("sb_inpaint_biharmonic_f64", "sb_medfilt_masked_f64"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib, name)
