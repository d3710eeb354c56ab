"""scint_sim.Brightness without a GPU: the float64 oracle (oracle/brightness_oracle.py)
against the unmodified reference's fixtures (oracle/make_golden_brightness.py), the cell
rule against griddata, the triangulation each fixture was made on, and the argument and
size errors, which are raised before any device work."""
import glob
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import brightness_oracle as BO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "brightness_*.npz")))
IDS = [os.path.basename(fn)[11:-4] for fn in FIXTURES]
EXACT = ("x", "fd", "td", "thetax", "thetay", "jacobian")


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


def _kw(z):
    return json.loads(str(z["kwargs"]))


@pytest.fixture(scope="module")
def models():
    out = {}
    for fn in FIXTURES:
        out[fn] = BO.model(**_kw(np.load(fn)))
    return out


def check_against_fixture(z, m):
    """m (a dict of Brightness attributes) against the reference's fixture z, at the bars of
    the device tests: the axes, thetax, thetay and the Jacobian bit-equal; acf_efield within
    4 ulp of its maximum (1); B within 1e-12 max B; SS with the same NaNs and within
    1e-12 max B max jacobian (x2 after the flip); LSS within 1e-9 dB where SS > 0; acf within
    1e-12 (or NaN everywhere, as numpy's FFT spreads a NaN)."""
    eps = np.finfo(np.float64).eps
    if "x" not in z:                                   # the default-size case: samples
        for k in ("x", "fd", "td"):
            assert _sha(m[k]) == str(z[k + "_sha256"]), k
        got = {k: np.ravel(m[k])[z[k + "_idx"]] for k in ("acf_efield", "B", "thetax", "thetay",
                                                          "jacobian", "SS", "LSS", "acf")}
        ref = {k: z[k + "_val"] for k in got}
        mb, mj = np.max(m["B"]), np.max(m["jacobian"])
    else:
        got, ref = m, {k: z[k] for k in getattr(z, "files", z)}
        mb, mj = ref["B"].max(), ref["jacobian"].max()
        for k in ("x", "fd", "td"):
            assert np.array_equal(got[k], ref[k]), k
    for k in ("thetax", "thetay", "jacobian"):
        assert np.array_equal(got[k], ref[k]), k
    assert np.max(np.abs(got["acf_efield"] - ref["acf_efield"])) <= 4 * eps
    assert np.max(np.abs(got["B"] - ref["B"])) <= 1e-12 * mb
    fin = np.isfinite(ref["SS"])
    assert np.array_equal(np.isfinite(got["SS"]), fin)
    assert np.max(np.abs(got["SS"] - ref["SS"])[fin], initial=0) <= 2e-12 * mb * mj
    pos = fin & (ref["SS"] > 0)
    assert np.max(np.abs(got["LSS"] - ref["LSS"])[pos], initial=0) <= 1e-9
    if np.isfinite(ref["acf"]).all():
        assert np.max(np.abs(got["acf"] - ref["acf"])) <= 1e-12
    else:
        assert np.isnan(ref["acf"]).all() and np.isnan(got["acf"]).all()


@pytest.mark.parametrize("fn", FIXTURES, ids=IDS)
def test_oracle_reproduces_fixture(fn, models):
    check_against_fixture(np.load(fn), models[fn])


@pytest.mark.parametrize("fn", FIXTURES, ids=IDS)
def test_triangulation_is_the_fixtures(fn, models):
    """The installed qhull splits every cell as it did for the fixture; the port's bitmap
    equals the oracle's."""
    from scintools_b200.scint_sim import lattice_diagonals
    z = np.load(fn)
    x = models[fn]["x"]
    main = BO.diagonals(x)
    assert BO.diag_sha256(main) == str(z["diag_sha256"]), "qhull triangulates differently"
    assert np.array_equal(lattice_diagonals(x), np.packbits(np.ravel(main)))


def _queries(x, rng, m):
    lo, hi, d = x[0], x[-1], x[1] - x[0]
    q = [rng.uniform(lo - 3 * d, hi + 3 * d, (2, m)),                   # some outside
         np.stack([rng.choice(x, m), rng.uniform(lo, hi, m)]),         # on lattice lines
         np.stack([rng.uniform(lo, hi, m), rng.choice(x, m)]),
         np.stack([rng.choice(x, m), rng.choice(x, m)]),               # on lattice points
         np.stack([rng.choice([lo, hi], m), rng.uniform(lo, hi, m)])]  # on the hull
    return np.concatenate(q, axis=1)


@pytest.mark.parametrize("fn", FIXTURES, ids=IDS)
def test_cell_rule_equals_griddata(fn, models):
    from scipy.interpolate import griddata
    m = models[fn]
    x, B = m["x"], m["B"]
    rng = np.random.default_rng(len(x))
    q = _queries(x, rng, 2000 if len(x) > 100 else 4000)
    X, Y = np.meshgrid(x, x)
    ref = griddata((np.ravel(X), np.ravel(Y)), np.ravel(B), (q[0], q[1]), method="linear")
    got = BO.cell_interp(x, BO.diagonals(x), B, q[0], q[1])
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    fin = ~np.isnan(ref)
    assert fin.sum() > 0.5 * len(ref)
    assert np.max(np.abs(got[fin] - ref[fin])) <= 1e-15 * B.max()


# ---- argument and size errors, raised before any device work --------------------------------
class _Touched(Exception):
    pass


@pytest.fixture
def no_device(monkeypatch):
    from scintools_b200 import scint_sim as S

    def touched(*a, **k):
        raise _Touched()
    for name in ("upload", "empty", "zeros", "device"):
        monkeypatch.setattr(S.D, name, touched)
    return S


SMALL = dict(nx=1, dx=0.1, nf=0.1, df=0.02, nt=1, dt=0.1)


def test_plot_raises_first(no_device):
    S = no_device
    with pytest.raises(NotImplementedError):
        S.Brightness(plot=True)
    b = S.Brightness.__new__(S.Brightness)
    for meth in ("plot_acf_efield", "plot_brightness", "plot_sspec", "plot_cuts", "plot_acf"):
        with pytest.raises(NotImplementedError):
            getattr(b, meth)()


@pytest.mark.parametrize("kw", [dict(ar=0), dict(ar=1, alpha=np.inf), dict(ar=np.nan)])
def test_non_finite_form(no_device, kw):
    with pytest.raises(ValueError):
        no_device.Brightness(**dict(SMALL, **kw))


def test_lattice_size_limit(no_device):
    S = no_device
    assert len(np.arange(-51.2, 51.2, 0.1)) == 1024
    assert len(np.arange(-51.25, 51.25, 0.1)) == 1025
    with pytest.raises(_Touched):                      # at the limit: reaches the device
        S.Brightness(**dict(SMALL, nx=51.2))
    with pytest.raises(ValueError):
        S.Brightness(**dict(SMALL, nx=51.25))


@pytest.mark.parametrize("axis", ["td", "fd"])
def test_query_size_limit(no_device, monkeypatch, axis):
    S = no_device
    monkeypatch.setattr(S, "lattice_diagonals", lambda x: np.zeros(1, np.uint8))
    at = dict(nt=204.8, dt=0.1) if axis == "td" else dict(nf=204.8, df=0.1)
    over = dict(nt=204.85, dt=0.1) if axis == "td" else dict(nf=204.85, df=0.1)
    key = "nt" if axis == "td" else "nf"
    assert len(np.arange(-at[key], at[key], 0.1)) == 4096
    assert len(np.arange(-over[key], over[key], 0.1)) == 4097
    with pytest.raises(_Touched):
        S.brightness_batch([{}], **dict(SMALL, **at))
    with pytest.raises(ValueError):
        S.brightness_batch([{}], **dict(SMALL, **over))
    with pytest.raises(ValueError):                   # one bad set stops the whole batch
        S.brightness_batch([{}, dict(ar=0)], **SMALL)


def _with_lattice(S, X, Y):
    b = S.Brightness.__new__(S.Brightness)
    b.__dict__.update(dict(ar=1.0, psi=0, alpha=1.67, thetagx=0, thetagy=0, thetarx=0,
                           thetary=0), **SMALL)
    b.X, b.Y, b.B = X, Y, np.ones_like(X)
    return b


def test_lattice_must_be_a_meshgrid(no_device):
    S = no_device
    x = np.arange(-1, 1, 0.1)
    X, Y = np.meshgrid(x, x)
    for bad in [(X, X), (Y, X), np.meshgrid(x[::-1], x[::-1]), (X[:, :-1], Y[:, :-1]),
                np.meshgrid(np.sort(np.r_[x, 0.05]), x)[:1] * 2]:
        with pytest.raises(ValueError):
            _with_lattice(S, *bad).calc_SS()
    with pytest.raises(_Touched):
        _with_lattice(S, X, Y).calc_SS()


def test_triangulation_must_be_half_cells(monkeypatch):
    import scipy.spatial
    from scintools_b200 import scint_sim as S

    class Skewed:
        def __init__(self, pts):
            n = int(round(np.sqrt(len(pts))))
            tri = []
            for i in range(n - 1):
                for j in range(n - 1):
                    p = i * n + j
                    tri += [[p, p + 1, p + n + 1], [p, p + n, p + n + 1]]
            tri[0] = [0, 2, n]                         # spans two cells
            self.simplices = np.array(tri)
    monkeypatch.setattr(scipy.spatial, "Delaunay", Skewed)
    monkeypatch.setattr(S, "_TRIANGULATIONS", {})
    with pytest.raises(ValueError):
        S.lattice_diagonals(np.arange(5.0) + 0.125)


def test_batch_keywords(no_device):
    S = no_device
    assert S.brightness_batch([], **SMALL) == []
    with pytest.raises(TypeError):
        S.brightness_batch([dict(nx=3)], **SMALL)
    with pytest.raises(TypeError):
        S.brightness_batch([{}], ar=2, **SMALL)
