"""scint_sim.ACF without a device: the float64 oracle (the direct double sum) against the
reference's fixtures, the port's host axes bit for bit against the oracle's and the
fixtures', and the argument errors raised before any device call.
Fixtures: oracle/make_golden_acf_model.py."""
import glob
import json
import os

import numpy as np
import pytest

from oracle import acf_model_oracle as AO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "acf_model_*.npz")))
IDS = [os.path.basename(fn)[10:-4] for fn in FIXTURES]
# the smallest ACF (3 x 3) with manual sampling that puts one grid exactly at the
# 16384-point limit, or one point past it
MAIN_AT = dict(nt=3, nf=3, auto_sampling=False, spatial_factor=1, resolution_factor=16383,
               core_factor=1)
MAIN_OVER = dict(MAIN_AT, resolution_factor=16384)
CORE_AT = dict(MAIN_AT, resolution_factor=1, core_factor=16383)
CORE_OVER = dict(CORE_AT, core_factor=16384)
AXES = ("fn", "tn", "sn", "snp", "ddnun", "dsp", "sp_fac", "res_fac", "core_fac", "nf", "nt")


def _kwargs(z):
    return json.loads(str(z["kwargs"]))


def _host(kwargs):
    """An ACF object with the constructor's attributes set and calc_acf not run."""
    from scintools_b200.scint_sim import ACF
    a = ACF.__new__(ACF)
    calls = []
    a.calc_acf = lambda: calls.append(1)
    ACF.__init__(a, **kwargs)
    assert calls == [1]
    return a


def test_fixture_set():
    assert len(FIXTURES) == 12


@pytest.mark.parametrize("fn", FIXTURES, ids=IDS)
def test_oracle_matches_reference(fn):
    z = np.load(fn)
    if "ar8" in fn:
        pytest.skip("the direct sum at ar=8 takes minutes on a CPU; the GPU test covers it")
    ax, acf, ef = AO.model(**_kwargs(z))
    assert acf.shape == z["acf"].shape
    amp = _kwargs(z).get("amp", 1)
    assert np.max(np.abs(acf - z["acf"])) <= 1e-12 * amp
    for k in AXES:
        assert np.array_equal(np.asarray(ax[k]), z[k]), k
    if "acf_efield" in z.files:
        assert np.max(np.abs(ef - z["acf_efield"])) <= 1e-14
    for w in json.loads(str(z["sspec"])):
        ref = z["sspec_%s" % w[0]]
        got = AO.sspec(z["acf"], w[0], w[1])
        assert np.max(np.abs(10 ** (got / 10) - 10 ** (ref / 10))) <= 1e-12 * np.max(
            10 ** (ref / 10))


@pytest.mark.parametrize("fn", FIXTURES, ids=IDS)
def test_host_axes_bit_exact(fn):
    z = np.load(fn)
    kw = _kwargs(z)
    a = _host(kw)
    h = a._axes()
    o = AO.axes(**kw)
    for k in ("snp", "snp2", "dnun", "snx", "sny", "ddnun", "fn"):
        assert np.array_equal(h[k], o[k]), k
    assert np.array_equal(h["t2"], o["tn"])
    assert h["sigxn"] == o["sigxn"] and h["sigyn"] == o["sigyn"]
    assert h["step1"] == o["h1"] and h["step2"] == o["h2"]
    for k in ("dsp", "sp_fac", "res_fac", "core_fac", "nf", "nt"):
        assert getattr(a, k) == z[k], k
    assert np.array_equal(h["fn"], z["fn"]) and np.array_equal(h["t2"], z["tn"])
    assert np.array_equal(h["snp"], z["snp"]) and h["ddnun"] == z["ddnun"]


def test_wn_rows():
    """taumax=4 puts an exact zero in the lags, taumax=3.7 does not: wn is dropped there."""
    h4 = _host(dict(phasegrad=0.3, wn=0.1, taumax=4, nt=51))._axes()
    h37 = _host(dict(phasegrad=0.3, wn=0.1, taumax=3.7, nt=51))._axes()
    assert np.count_nonzero(h4["snx"] == 0) == 1
    assert np.count_nonzero(h37["snx"] == 0) == 0
    assert abs(h37["snx"][25]) < 1e-15


@pytest.mark.parametrize("kw,exc", [
    (dict(nf=1), IndexError),
    (dict(nf=0), IndexError),
    (dict(nt=1), ZeroDivisionError),
    (dict(amp=0), ZeroDivisionError),
    (dict(amp=0, phasegrad=0.2), ZeroDivisionError),
    (dict(taumax=0), ZeroDivisionError),
    (dict(ar=0), ValueError),
    (dict(ar=-1), ValueError),
    (dict(psi=np.nan), ValueError),
    (dict(phasegrad=np.inf), ValueError),
    (dict(wn=np.nan), ValueError),
    (dict(dnumax=0), ValueError),
    (dict(nf=8192), ValueError),
    (dict(nt=8192), ValueError),
    (dict(ar=16.7), ValueError),               # core grid 16451 points per side
    (MAIN_OVER, ValueError),
    (CORE_OVER, ValueError),
    (dict(plot=True), NotImplementedError),
])
def test_argument_errors_before_device(kw, exc, monkeypatch):
    from scintools_b200 import _device
    from scintools_b200.scint_sim import ACF
    monkeypatch.setattr(_device, "device", lambda: pytest.fail("device touched"))
    with pytest.raises(exc):
        ACF(**kw)


@pytest.mark.parametrize("kw,n1,n2", [
    (MAIN_AT, 16384, 16384), (MAIN_OVER, 16385, 16385),
    (CORE_AT, 2, 16384), (CORE_OVER, 2, 16385),
    (dict(ar=16.6), 4069, 16269), (dict(ar=16.7), 4114, 16451),
])
def test_grid_sizes_at_the_limit(kw, n1, n2):
    """The grid sizes the limit tests rely on, from the host axes alone."""
    from scintools_b200.scint_sim import _arange_len
    a = _host(kw)
    h1, h2 = a.dsp / a.res_fac, a.dsp / (a.res_fac * a.core_fac)
    half = a.sp_fac * a.taumax
    assert _arange_len(-half, half + h1, h1) == n1
    assert _arange_len(-half, half + h2, h2) == n2
    if max(n1, n2) <= 16384:
        h = a._axes()
        assert (len(h["snp"]), len(h["snp2"])) == (n1, n2)


def test_plot_methods_raise(monkeypatch):
    from scintools_b200 import _device
    monkeypatch.setattr(_device, "device", lambda: pytest.fail("device touched"))
    a = _host({})
    for m in (a.plot_acf, a.plot_acf_efield, a.plot_sspec):
        with pytest.raises(NotImplementedError):
            m()
    with pytest.raises(NotImplementedError):
        type(a).calc_acf(a, plot=True)
