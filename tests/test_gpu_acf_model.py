"""scint_sim.ACF on the device (csrc/acf_model.cu) against the unmodified reference's
fixtures (oracle/make_golden_acf_model.py), the float64 direct-sum oracle
(oracle/acf_model_oracle.py) and its own symmetries.

Tolerances:
  acf          1e-12 amp absolute (the float64 bilinear form reorders the reference's sum;
               the ACF peaks at amp (1 + wn/amp)^2)
  acf_efield   1e-14 absolute, the table peaks at 1
  sspec        linear amplitude |F| = 10^(sspec/10), max |got - ref| <= 1e-5 max |ref|: the
               bound tests/test_gpu_fft_lengths.py establishes for every fp32 output of the
               chirp-z transform (MAX_FP32)
"""
import glob
import json
import os

import numpy as np
import pytest

from oracle import acf_model_oracle as AO

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "acf_model_*.npz")))
IDS = [os.path.basename(fn)[10:-4] for fn in FIXTURES]
AXES = ("fn", "tn", "sn", "snp", "ddnun", "dsp", "sp_fac", "res_fac", "core_fac", "nf", "nt")
MAX_FP32 = 1e-5
# the smallest ACF with one grid at the 16384-point limit or one point past it
MAIN_AT = dict(nt=3, nf=3, auto_sampling=False, spatial_factor=1, resolution_factor=16383,
               core_factor=1)
MAIN_OVER = dict(MAIN_AT, resolution_factor=16384)
CORE_AT = dict(MAIN_AT, resolution_factor=1, core_factor=16383)
CORE_OVER = dict(CORE_AT, core_factor=16384)
# nt = nf = 8191 on a five-point grid
N_AT = dict(nt=8191, nf=8191, phasegrad=0.1, theta=30, psi=40, auto_sampling=False,
            spatial_factor=0.001, resolution_factor=1, core_factor=1)


def _acf(**kw):
    from scintools_b200.scint_sim import ACF
    return ACF(**kw)


def _lin(s):
    return 10 ** (np.asarray(s, np.float64) / 10)


def _sspec_err(got, ref):
    return np.max(np.abs(_lin(got) - _lin(ref))) / np.max(_lin(ref))


@pytest.mark.parametrize("fn", FIXTURES, ids=IDS)
def test_fixture(fn):
    z = np.load(fn)
    kw = json.loads(str(z["kwargs"]))
    a = _acf(**kw)
    amp = kw.get("amp", 1)
    assert a.acf.shape == z["acf"].shape and a.acf.dtype == np.float64
    err = np.max(np.abs(a.acf - z["acf"]))
    print("%s: max |acf - reference| = %.2e" % (os.path.basename(fn), err))
    assert err <= 1e-12 * amp
    for k in AXES:
        assert np.array_equal(np.asarray(getattr(a, k)), z[k]), k
    ef = z["acf_efield"] if "acf_efield" in z.files else AO.efield(
        z["snp"], kw.get("ar", 1), kw.get("alpha", 5 / 3))
    assert a.acf_efield.shape == ef.shape
    assert np.max(np.abs(a.acf_efield - ef)) <= 1e-14
    for window, frac in json.loads(str(z["sspec"])):
        a.calc_sspec(window=window, window_frac=frac)
        e = _sspec_err(a.sspec, z["sspec_%s" % window])
        print("  sspec %s: %.2e of max" % (window, e))
        assert e <= MAX_FP32


def _random_kwargs(rng):
    kw = dict(psi=float(rng.uniform(0, 90)), ar=float(rng.uniform(0.5, 2.5)),
              alpha=float(rng.uniform(1.0, 2.0)), taumax=float(rng.uniform(2, 5)),
              dnumax=float(rng.uniform(1, 5)), nf=int(rng.integers(3, 16)),
              nt=int(rng.integers(3, 24)), amp=float(rng.uniform(0.3, 2)),
              wn=float(rng.uniform(0, 0.3)), auto_sampling=False,
              spatial_factor=float(rng.uniform(0.8, 2)),
              resolution_factor=float(rng.uniform(0.5, 1.5)),
              core_factor=float(rng.uniform(1, 3)))
    if rng.uniform() < 0.6:
        kw.update(phasegrad=float(rng.uniform(0.05, 0.6)), theta=float(rng.uniform(-90, 90)))
    return kw


@pytest.mark.parametrize("seed", range(20))
def test_random_against_oracle(seed):
    kw = _random_kwargs(np.random.default_rng(1000 + seed))
    a = _acf(**kw)
    _, ref, ref_ef = AO.model(**kw)
    assert a.acf.shape == ref.shape
    assert np.max(np.abs(a.acf - ref)) <= 1e-12 * kw["amp"]
    assert np.max(np.abs(a.acf_efield - ref_ef)) <= 1e-14


@pytest.mark.parametrize("kw", [
    dict(wn=0.2, amp=0.8),
    dict(phasegrad=0.3, wn=0.1, taumax=4, amp=1.5),
    dict(psi=60, ar=2, alpha=1.4, wn=0.05),
    dict(phasegrad=0.5, theta=45, nt=50, nf=20, wn=0.1, amp=0.8),
], ids=["quadrant", "half_plane", "anisotropic", "pg05"])
def test_properties(kw):
    a = _acf(**kw)
    nf, nt = a.acf.shape
    amp, wn = kw.get("amp", 1), kw.get("wn", 0)
    # zero lag: amp (1 + wn/amp)^2 (the lags include an exact zero here)
    assert a.acf[nf // 2, nt // 2] == pytest.approx(amp * (1 + wn / amp) ** 2, rel=1e-15)
    if kw.get("phasegrad", 0) == 0:
        assert np.array_equal(a.acf, a.acf[::-1, :])
        assert np.array_equal(a.acf, a.acf[:, ::-1])
    else:
        # frequency lags != 0 are placed by the point reflection; the zero-lag row holds
        # every time lag as computed, symmetric to the rounding of linspace's lags
        off = np.arange(nf) != nf // 2
        assert np.array_equal(a.acf[off], a.acf[::-1, ::-1][off])
        assert np.max(np.abs(a.acf[nf // 2] - a.acf[nf // 2, ::-1])) <= 1e-15 * amp
    # column 0 (frequency lag 0) in closed form
    ax = AO.axes(**kw)
    g0 = AO.column0(ax)
    col = a.acf[nf // 2, :]
    want = amp * g0 ** 2
    if ax["quadrant"]:
        want = np.concatenate((want[:0:-1], want))
    assert np.max(np.abs(col - want)) <= 1e-15 * amp


def test_wn_dropped_without_exact_zero_lag():
    a4 = _acf(phasegrad=0.3, wn=0.1, taumax=4, nt=51)
    a37 = _acf(phasegrad=0.3, wn=0.1, taumax=3.7, nt=51)
    assert a4.acf[25, 25] == pytest.approx(1.1 ** 2, rel=1e-15)
    assert a37.acf[25, 25] == pytest.approx(1.0, abs=1e-12)


def test_repeat_bit_identical():
    kw = dict(psi=30, phasegrad=0.2, ar=2, nt=51, nf=51)
    a, b = _acf(**kw), _acf(**kw)
    assert np.array_equal(a.acf, b.acf) and np.array_equal(a.acf_efield, b.acf_efield)
    b.calc_acf()
    assert np.array_equal(a.acf, b.acf)


def test_calc_acf_rereads_attributes():
    a = _acf(nt=21, nf=11)
    a.phasegrad, a.theta, a.wn = 0.25, 30, 0.1
    a.calc_acf()
    b = _acf(nt=21, nf=11, phasegrad=0.25, theta=30, wn=0.1)
    assert np.array_equal(a.acf, b.acf)


def test_smallest_acf_and_sspec():
    a = _acf(nt=3, nf=3, phasegrad=0.2)
    _, ref, _ = AO.model(nt=3, nf=3, phasegrad=0.2)
    assert a.acf.shape == (3, 3)
    assert np.max(np.abs(a.acf - ref)) <= 1e-12
    for w in ("hanning", "blackman", "hamming"):
        a.calc_sspec(window=w, window_frac=1)
        assert a.sspec.shape == (3, 3)
        assert _sspec_err(a.sspec, AO.sspec(a.acf, w, 1)) <= MAX_FP32


@pytest.mark.parametrize("kw", [MAIN_AT, CORE_AT], ids=["main", "core"])
def test_grid_limit_accepted(kw):
    a = _acf(**kw)
    ax = AO.axes(**kw)
    assert a.acf.shape == (3, 3) and np.all(np.isfinite(a.acf))
    assert a.acf_efield.shape == (len(a.snp),) * 2
    assert max(len(ax["snp"]), len(ax["snp2"])) == 16384
    assert np.array_equal(a.acf, a.acf[::-1, :]) and np.array_equal(a.acf, a.acf[:, ::-1])
    # the zero lag and the closed-form column
    assert a.acf[1, 1] == 1.0
    assert np.max(np.abs(a.acf[1, :] - AO.column0(ax)[[1, 0, 1]] ** 2)) <= 1e-15


@pytest.mark.parametrize("kw", [MAIN_OVER, CORE_OVER, dict(N_AT, nt=8192),
                                dict(N_AT, nf=8192)], ids=["main", "core", "nt", "nf"])
def test_limit_rejected(kw):
    with pytest.raises(ValueError):
        _acf(**kw)


def test_largest_acf():
    a = _acf(**N_AT)
    assert a.acf.shape == (8191, 8191) and np.all(np.isfinite(a.acf))
    off = np.arange(8191) != 4095
    assert np.array_equal(a.acf[off], a.acf[::-1, ::-1][off])
    ax = AO.axes(**N_AT)
    assert np.max(np.abs(a.acf[4095, :] - AO.column0(ax) ** 2)) <= 1e-15
    # a few lags of the last frequency column against the direct sum
    sub = dict(ax, snx=ax["snx"][::1000], sny=ax["sny"][::1000],
               dnun=ax["dnun"][[0, 1, 4095]])
    g = AO.gamma(sub)
    # gamma's columns are dnun[0], dnun[1] (core grid), dnun[4095] (main grid)
    got = a.acf[4095 + 4095, ::1000]
    assert np.max(np.abs(got - np.abs(g[:, 2]) ** 2)) <= 1e-12


def test_library_rejects_sizes_without_launch():
    import torch
    from scintools_b200 import _device as D
    from scintools_b200 import _lib
    buf = D.zeros((16, ), torch.float64)
    p = buf.data_ptr()
    for n1, n2, nd, ns in [(16385, 4, 2, 2), (4, 16385, 2, 2), (4, 4, 4097, 2),
                           (4, 4, 2, 8192), (4, 4, 1, 2), (0, 4, 2, 2)]:
        m = _lib.AcfModel(p, p, p, p, p, n1, n2, nd, ns, 0, 0.0, 0.0, 1.0, 5 / 6, 0.1, 0.1,
                          0.0, 1.0)
        before = _lib.lib.sb_launch_count()
        with pytest.raises(_lib.SbError):
            _lib.check(_lib.lib.sb_acf_model_f64(m, p, p, D.stream_ptr()))
        assert _lib.lib.sb_launch_count() == before
