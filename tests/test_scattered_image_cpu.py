"""Dynspec.calc_scattered_image without a GPU: the oracle (oracle/scattered_image_oracle.py)
against the unmodified reference's fixtures (oracle/make_golden_scattered_image.py), the
host's spline knots and band factors against scipy's RectBivariateSpline, every reference
exception and every size limit raised before any device work by both entry points, and the
new header's symbol."""
import json
import os
import re

import numpy as np
import pytest
from scipy.interpolate import RectBivariateSpline

from oracle import scattered_image_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "scatim_arc_48x80.npz")
Z = np.load(FIXTURE)
CASES = sorted(k[:-len("_kwargs")] for k in Z.files if k.endswith("_kwargs"))
# the curvature comes from the reference's fit_arc, which raised: only the port's own
# fit_arc (on the device) can run these
FIT_RAISES = [c for c in CASES if c.startswith("fit_freq")]


def call_args(z, name):
    """(keyword arguments, preset attributes) of a fixture call, arrays filled in."""
    kw = json.loads(str(z[name + "_kwargs"]))
    preset = json.loads(str(z[name + "_preset"]))
    src = kw.get("input_sspec")
    if src is not None:
        spec, fd, td = z["sspec"].copy(), z["fdop"], z["tdel"]
        if src == "alt":
            spec, fd, td = z["alt_sspec"].copy(), z["alt_fdop"], z["alt_tdel"]
        elif src == "minf":
            spec.flat[z["minf_idx"]] = -np.inf
        elif src == "nan":
            spec.flat[z["nan_idx"]] = np.nan
        kw.update(input_sspec=spec, input_fdop=fd.copy(), input_tdel=td.copy())
    return kw, preset


def fitted(z, name, preset):
    """preset plus the curvature the reference's fit_arc found, for calls that ran it."""
    kw = json.loads(str(z[name + "_kwargs"]))
    out = dict(preset)
    if "input_eta" not in kw and kw.get("fit_arc", True) and not preset and \
            str(z[name + "_raises"]) == "":
        key = "betaeta" if kw.get("lamsteps") else "eta"
        out[key] = float(z[name + "_" + key])
    return out


def port_dynspec(z, preset):
    from scintools_b200.dynspec import BasicDyn, Dynspec
    dyn = z["dyn"]
    nf, nt = dyn.shape
    freqs = float(z["f0"]) + float(z["df"]) * np.arange(nf)
    times = float(z["dt"]) * np.arange(nt)
    ds = Dynspec(dyn=BasicDyn(dyn.copy(), name="golden", header=["golden"], times=times,
                              freqs=freqs, nchan=nf, nsub=nt, bw=float(z["df"]) * nf,
                              df=float(z["df"]), freq=float(np.mean(freqs)),
                              tobs=float(z["dt"]) * nt, dt=float(z["dt"]), mjd=60000),
                 verbose=False, process=False)
    ds.sspec, ds.lamsspec = z["sspec"].copy(), z["lamsspec"].copy()
    ds.fdop, ds.tdel, ds.beta = z["fdop"].copy(), z["tdel"].copy(), z["beta"].copy()
    for k, v in preset.items():
        setattr(ds, k, np.float64(ds.freq) if v == "float64" else v)
    return ds


def oracle_call(z, name):
    """The fixture call through the oracle: (image, axis)."""
    kw, preset = call_args(z, name)
    preset = fitted(z, name, preset)
    freq = float(np.mean(float(z["f0"]) + float(z["df"]) * np.arange(z["dyn"].shape[0])))
    if "input_sspec" in kw:
        spec, fd, td = kw["input_sspec"], kw["input_fdop"], kw["input_tdel"]
    else:
        spec = z["lamsspec"] if kw.get("lamsteps") else z["sspec"]
        fd, td = z["fdop"], z["tdel"]
    if "input_eta" in kw:
        eta = kw["input_eta"]
    elif not kw.get("fit_arc", True):
        eta = td[len(td) - 1] / fd[len(fd) - 1] ** 2
    elif kw.get("lamsteps"):
        ref_freq = kw.get("ref_freq", 1400)
        eta = preset["betaeta"] / (freq / ref_freq) ** 2 * (299792458.0 * 1e6 /
                                                           ((ref_freq * 1e6) ** 2))
    elif "eta" in preset:
        eta = preset["eta"]
    else:
        raise AttributeError("'Dynspec' object has no attribute 'eta'")
    opts = {k: kw[k] for k in ("sampling", "plot_log", "use_angle", "use_spatial", "s", "veff",
                               "d") if k in kw}
    with np.errstate(all="ignore"):
        return SO.scattered_image(spec, fd, td, eta, freq=freq, **opts)


def check_image(z, name, im, ax, bar=1e-10):
    assert np.array_equal(ax, z[name + "_ax"])
    assert im.dtype == np.float64
    if name + "_image" in z.files:
        ref = z[name + "_image"]
        assert im.shape == ref.shape
        nan = np.isnan(ref)
        assert np.array_equal(np.isnan(im), nan)
        scale = np.max(np.abs(ref[~nan]), initial=0.0)
        assert np.max(np.abs(im - ref)[~nan], initial=0.0) <= bar * scale
        return
    assert im.shape == tuple(z[name + "_shape"])
    got = im.flat[z[name + "_idx"]]
    assert np.max(np.abs(got - z[name + "_val"])) <= bar * float(z[name + "_absmax"])


@pytest.mark.parametrize("name", [c for c in CASES if c not in FIT_RAISES])
def test_oracle_reproduces_fixture(name):
    raises = str(Z[name + "_raises"])
    if raises:
        with pytest.raises(Exception) as e:
            oracle_call(Z, name)
        assert type(e.value).__name__ == raises
        return
    im, ax = oracle_call(Z, name)
    check_image(Z, name, im, ax, bar=0.0)


def test_fixture_covers_the_issue_cases():
    raised = {str(Z[c + "_raises"]) for c in CASES}
    assert {"StopIteration", "AttributeError", "ValueError", "IndexError", "TypeError"} <= raised
    for c in ("s0_nolog", "s1", "eta", "s157", "eta_nolog", "flim0", "wrap", "minf", "alt",
              "fit_lam", "nan_nolog"):
        assert str(Z[c + "_raises"]) == "", c
    assert np.isnan(Z["nan_nolog_image"]).all()


def _axes(rng, m):
    return np.cumsum(rng.uniform(0.05, 1.0, m)) - rng.uniform(0, 3)


def test_knots_equal_scipy():
    from scintools_b200.dynspec import spline_tables
    rng = np.random.default_rng(0)
    axes = [_axes(rng, m) for m in (4, 5, 6, 9, 64, 257)]
    axes += [Z["tdel"], Z["fdop"], Z["alt_fdop"], Z["fdop"][:9]]
    for x in axes:
        sp = RectBivariateSpline(x, Z["fdop"][:8], np.zeros((len(x), 8)))
        assert np.array_equal(spline_tables(x)[0], sp.get_knots()[0])


def solve(Zd, fac):
    """L U X = Zd down axis 0 with the band factors, in numpy."""
    l2, l1, dinv, u1, u2 = fac
    m = Zd.shape[0]
    Y = Zd.copy()
    for i in range(m):
        if i >= 1:
            Y[i] -= l1[i] * Y[i - 1]
        if i >= 2:
            Y[i] -= l2[i] * Y[i - 2]
    for i in range(m - 1, -1, -1):
        if i + 1 < m:
            Y[i] -= u1[i] * Y[i + 1]
        if i + 2 < m:
            Y[i] -= u2[i] * Y[i + 2]
        Y[i] *= dinv[i]
    return Y


@pytest.mark.parametrize("case", ["random_4x4", "random_5x7", "random_64x150", "random_200x97",
                                  "fixture", "fixture_crop"])
def test_band_factors_give_scipys_coefficients(case):
    from scintools_b200.dynspec import spline_tables
    rng = np.random.default_rng(len(case))
    if case.startswith("random"):
        mx, my = map(int, case.split("_")[1].split("x"))
        x, y = _axes(rng, mx), _axes(rng, my)
        data = rng.uniform(0, 5, (mx, my)) ** 3
    else:
        x, y = Z["tdel"], Z["fdop"]
        data = 10 ** (Z["sspec"] / 10)
        if case == "fixture_crop":
            x, y, data = x[3:40], y[100:180], data[3:40, 100:180]
    C = solve(solve(data, spline_tables(x)[1]).T, spline_tables(y)[1]).T
    ref = RectBivariateSpline(x, y, data).get_coeffs().reshape(len(x), len(y))
    assert np.max(np.abs(C - ref)) <= 1e-13 * np.max(np.abs(data))


class _Touched(Exception):
    pass


@pytest.fixture
def no_device(monkeypatch):
    from scintools_b200 import _device

    def touched(*a, **k):
        raise _Touched()
    for name in ("upload", "upload_f32", "empty", "zeros", "device"):
        monkeypatch.setattr(_device, name, touched)
    return _device


@pytest.mark.parametrize("name", [c for c in CASES if str(Z[c + "_raises"]) and
                                  c not in FIT_RAISES])
def test_reference_exceptions_before_device(no_device, name):
    from scintools_b200.dynspec import scattered_image_batch
    kw, preset = call_args(Z, name)
    ds = port_dynspec(Z, preset)
    exc = str(Z[name + "_raises"])
    with pytest.raises(Exception) as e:
        ds.calc_scattered_image(**kw)
    assert type(e.value).__name__ == exc
    assert not hasattr(ds, "scattered_image")
    if "input_eta" in kw and not (kw.get("use_angle") or kw.get("use_spatial")):
        spec = kw.get("input_sspec", Z["sspec"])
        fd, td = kw.get("input_fdop", Z["fdop"]), kw.get("input_tdel", Z["tdel"])
        with pytest.raises(Exception) as e:
            scattered_image_batch(np.stack([spec, spec]), fd, td, kw["input_eta"],
                                  sampling=kw.get("sampling", 64),
                                  plot_log=kw.get("plot_log", True))
        assert type(e.value).__name__ == exc


def test_plotting_raises_first(no_device):
    ds = port_dynspec(Z, {})
    for kw in (dict(plot=True), dict(plot_fit=True)):
        with pytest.raises(NotImplementedError):
            ds.calc_scattered_image(input_eta=0.35, **kw)


def test_sampling_limit(no_device):
    from scintools_b200.dynspec import scattered_image_batch
    ds = port_dynspec(Z, {})
    with pytest.raises(_Touched):
        ds.calc_scattered_image(input_eta=0.35, sampling=4096)
    with pytest.raises(ValueError):
        ds.calc_scattered_image(input_eta=0.35, sampling=4097)
    with pytest.raises(ValueError):
        scattered_image_batch(Z["sspec"][None], Z["fdop"], Z["tdel"], 0.35, sampling=4097)


def limit_case(axis, n):
    """A spectrum whose crop has n delays (axis "delay") or n Doppler columns."""
    if axis == "doppler":
        # flim == 0 keeps every column; tlim = 5 rows on the delay axis fdop[:5]
        fdop = np.arange(n, dtype=np.float64) - n // 2
        tdel = np.arange(8, dtype=np.float64)
        eta = 4.5 / fdop[0] ** 2
        return np.zeros((8, n)), fdop, tdel, eta
    # flim == 1, int(0.02 * 8) = 0: columns [1:7], every row
    fdop = np.arange(-4.0, 4.0)
    tdel = np.arange(n, dtype=np.float64)
    eta = (n - 1) / 12.0
    return np.zeros((n, 8)), fdop, tdel, eta


@pytest.mark.parametrize("axis,limit", [("doppler", 32768), ("delay", 65536)])
def test_crop_size_limits(no_device, axis, limit):
    from scintools_b200.dynspec import _scatim_crop, scattered_image_batch
    ds = port_dynspec(Z, {})
    for n, exc in ((limit, _Touched), (limit + 1, ValueError)):
        spec, fd, td, eta = limit_case(axis, n)
        rows, cols, _, _ = _scatim_crop(spec.shape, fd, td, eta)
        size = (rows[1] - rows[0]) if axis == "delay" else (cols[1] - cols[0])
        assert size == n
        with pytest.raises(exc):
            ds.calc_scattered_image(input_sspec=spec, input_fdop=fd, input_tdel=td,
                                    input_eta=eta, sampling=2)
        with pytest.raises(exc):
            scattered_image_batch(spec[None], fd, td, eta, sampling=2)


def test_overflowing_db_value(no_device):
    ds = port_dynspec(Z, {})
    spec = Z["sspec"].copy()
    spec[2, 128] = 3090.0
    with pytest.raises(ValueError):
        ds.calc_scattered_image(input_sspec=spec, input_fdop=Z["fdop"], input_tdel=Z["tdel"],
                                input_eta=0.35)
    spec[2, 128] = 3080.0
    with pytest.raises(_Touched):
        ds.calc_scattered_image(input_sspec=spec, input_fdop=Z["fdop"], input_tdel=Z["tdel"],
                                input_eta=0.35)


def test_symbol_in_its_own_header():
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _lib
    text = open(os.path.join(ROOT, "include", "scint_b200_scatim.h")).read()
    names = re.findall(r"^int (sb_\w+)\(", text, re.M)
    assert names == ["sb_scattered_image_f64"]
    assert hasattr(_lib.lib, names[0])
    assert names[0] not in _lib.EXPORTS
    main = open(os.path.join(ROOT, "include", "scint_b200.h")).read()
    assert names[0] not in main
    assert _lib.lib.sb_abi_version() == 8
