"""GPU tests of Dynspec.get_scint_params / get_acf_tilt / dynspec.get_scint_params_batch
(csrc/scintfit.cu) against the reference's fixtures (oracle/make_golden_scint_params.py)
and the tight float64 oracle (oracle/scint_params_oracle.py).

The fixture's float64 ACF is set as ds.acf, so the fits are compared without the float32
FFT error.  Well-conditioned fits (every error estimated, tau and dnu constrained): the
parameters within 1e-4 of the reference's (lmfit's own 1e-7 tolerances leave about that)
and 1e-7 of the tight oracle's minimum, the errors within 1e-2 of the reference's and 1e-6
of lmfit's formula at the device's point.  Degenerate fits (a parameter running away):
chi-square no worse than the reference's.  Every fit: the relative gradient of chi-square
at the device's point (max |J_i . r| / (|J_i| |r|)) at most 1e-8, except a fit whose
parameter runs away without bound (the crafted 'fallback' ACF, flat in time): there the
device follows the runaway to max_nfev and reports success=False and no errors, where
lmfit stops on its 1e-7 tolerances.

lmfit's tolerances leave more than 1e-4 in a weakly determined parameter of a large 2-D
fit (phasegrad of the third J0437-4715 observation: 2.3e-4, or 0.02 of its error, with the
device's chi-square lower), so a parameter passes within 1e-4 relative or 0.05 of the
reference's error when the device's chi-square is no higher than the reference's."""
import glob
import os

import numpy as np
import pytest

from oracle import scint_params_oracle as SO

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "scint_params_*.npz")))
CASES = [(fn, c) for fn in FIXTURES for c in SO.fixture_cases(np.load(fn))]
IDS = ["%s:%s" % (os.path.basename(fn)[13:-4], c) for fn, c in CASES]


def _ds(z, case):
    from scintools_b200.dynspec import Dynspec
    return SO.fixture_dynspec(z, case, Dynspec)


def _well_conditioned(z, q):
    if q + "value_tau" in z.files and z[q + "value_tau"] > 10 * z["meta"][2]:
        return False        # tau running past ten observation lengths: degenerate
    for n in SO.SLOTS:
        k = q + "stderr_" + n
        if k in z.files and bool(z[q + "vary_" + n]):
            if not np.isfinite(z[k]):
                return False
            if n in ("tau", "dnu") and z[k] > abs(z[q + "value_" + n]):
                return False
    return True


def _device_args(ds, kw, res):
    """The data of the device's last fit, for the oracle: rebuilt by the port's host steps."""
    from scintools_b200 import dynspec as P
    full_frame, nscale = kw.get("full_frame", False), kw.get("nscale", 5)
    acf = ds.acf
    pl = P._scint_nofit(_copy(ds), full_frame, nscale, kw.get("bartlett", True),
                        kw.get("weighted", True))
    if kw.get("method", "acf1d") == "acf1d":
        return 1, (pl["xdata_t"], pl["xdata_f"], pl["ydata_t"], pl["ydata_f"],
                   pl["weights_t"], pl["weights_f"])
    rows, cols, tt, ft = P._scint_crop_2d(ds, pl["tau"], pl["dnu"], nscale, full_frame, False)
    w = SO.weights_2d_rule(acf, rows, cols, tt, ft, ds.nsub, ds.nchan, ds.tobs, ds.bw,
                           kw.get("weighted", True))
    y = acf[rows[0]:rows[-1] + 1, cols[0]:cols[-1] + 1]
    return 2, (tt[cols], ft[rows], y, w, ds.tobs, ds.bw)


def _copy(ds):
    from scintools_b200.dynspec import Dynspec
    c = Dynspec.__new__(Dynspec)
    c.__dict__.update({k: v for k, v in ds.__dict__.items()})
    return c


def _check_fit(res, kind, args, names, ref_q=None, z=None):
    p = {n: res.params[n].value for n in SO.SLOTS if n in res.params}
    var = [n for n in names if res.params[n].vary]
    err, chi, rel = SO.stderr_at(kind, args, p, var)
    print("chisqr %.12g (oracle at the device point %.12g), rel gradient %.2e, nfev %d"
          % (res.chisqr, chi, rel, res.nfev))
    if not res.success:     # a runaway: the cap, and no errors
        assert z is not None and not _well_conditioned(z, ref_q)
        assert all(res.params[n].stderr is None for n in var)
        return
    assert rel <= 1e-8
    assert res.chisqr == pytest.approx(chi, rel=1e-9)
    for n in var:
        if res.params[n].stderr is not None and np.isfinite(err[n]):
            assert res.params[n].stderr == pytest.approx(err[n], rel=1e-6), n
    if z is None:
        return
    if _well_conditioned(z, ref_q):
        tight, _, trel = SO.fit_tight(kind, args, p, var)
        assert trel <= 1e-9
        assert res.chisqr <= float(z[ref_q + "chisqr"]) * (1 + 1e-12)
        for n in var:
            ref = float(z[ref_q + "value_" + n])
            se = float(z[ref_q + "stderr_" + n])
            assert abs(p[n] - ref) <= max(1e-4 * abs(ref), 0.05 * se, 1e-9), n
            assert p[n] == pytest.approx(tight[n], rel=1e-7, abs=1e-12), n
            se = float(z[ref_q + "stderr_" + n])
            assert res.params[n].stderr == pytest.approx(se, rel=1e-2), n
    elif _same_start(z, ref_q, res):
        assert res.chisqr <= float(z[ref_q + "chisqr"]) * (1 + 1e-6)


def _same_start(z, q, res):
    """The device's fit started where the reference's did (a 2-D fit starts from the 1-D
    result only when that one has errors)."""
    return all(float(z[q + "p0_" + n]) == pytest.approx(res.init_values[n], rel=1e-4)
               for n in ("tau", "dnu", "amp") if n in res.init_values)


@pytest.mark.parametrize("fn,case", CASES, ids=IDS)
def test_fixture_parity(fn, case):
    z = np.load(fn)
    ds = _ds(z, case)
    kw = SO.fixture_kwargs(z, case)
    call = str(z[case + "/call"])
    err = str(z[case + "/error"])
    if err:
        with pytest.raises({"IndexError": IndexError, "ValueError": ValueError}[err]):
            ds.get_scint_params(**kw)
        return
    if case.startswith("acf2d_from_tilt"):
        ds.acf_tilt = float(z[case + "/fit1/p0_phasegrad"])
        ds.acf_tilt_err = 1.0
    res = None
    if call in ("scint", "scint+tilt"):
        res = ds.get_scint_params(**kw)
    if call in ("tilt", "scint+tilt"):
        ds.get_acf_tilt()
    # attributes the host derives without the fit: exactly the reference's
    for n in ("dnu_est", "dnu_esterr", "tscat_est", "modulation_index", "wnerr"):
        assert getattr(ds, n) == z[case + "/attr_" + n][()], n
    if kw.get("method") == "nofit":
        for k in z.files:
            if k.startswith(case + "/attr_"):
                assert getattr(ds, k.split("attr_")[1]) == z[k][()]
        return
    if call == "tilt" or call == "scint+tilt":
        # the rows and parabolas are the reference's; fse_tilt also carries the fit's tau, dnu
        for n, tol in (("acf_tilt", 1e-12), ("acf_tilt_err", 1e-9), ("fse_tilt", 1e-4)):
            assert getattr(ds, n) == pytest.approx(float(z[case + "/attr_" + n]), rel=tol), n
    if res is None:
        return
    qs = list(SO.fit_keys(z, case))
    kind, args = _device_args(ds, kw, res)
    names = [n for n in SO.SLOTS if n in res.params]
    _check_fit(res, kind, args, names, qs[-1], z)
    # the 1-D fit a 2-D fit starts from is a fit too
    assert ds.scint_param_method == kw.get("method", "acf1d")
    assert ds.report and "chi-square" in ds.report
    # tauerr and dnuerr carry the fit errors, held to 1e-2 of the reference's
    for n, tol in (("tau", 2e-3), ("dnu", 2e-3), ("amp", 2e-3), ("nscint", 2e-3),
                   ("fse_tau", 2e-3), ("fse_dnu", 2e-3), ("tscat", 2e-3), ("talpha", 2e-3),
                   ("tauerr", 1e-2), ("dnuerr", 1e-2)):
        ref = z[case + "/attr_" + n][()]
        if _well_conditioned(z, qs[-1]) and np.isfinite(ref):
            assert getattr(ds, n) == pytest.approx(float(ref), rel=tol), n
    if kw.get("method") == "acf2d_approx":
        assert ds.acf_model.shape == args[2].shape
        assert ds.wn == (0 if "sim:mb2=" in ds.name else 1 - ds.amp)


def _fits(method, dss, **kw):
    from scintools_b200.dynspec import get_scint_params_batch
    res = get_scint_params_batch(dss, method=method, **kw)
    return [np.array([r.params[n].value for n in SO.SLOTS if n in r.params] +
                     [r.chisqr, r.nfev] +
                     [r.params[n].stderr or np.nan for n in ("tau", "dnu", "amp")])
            for r in res]


@pytest.mark.parametrize("method", ["acf1d", "acf2d_approx"])
def test_batch_bit_identical(method):
    """A fit's result is the same bits alone, in batches of 1, 7 and 64, shuffled, and on
    a repeat."""
    base = []
    for fn in FIXTURES:
        z = np.load(fn)
        if "crafted" in fn:
            continue
        base.append(_ds(z, "acf1d"))
    alone = [_fits(method, [d])[0] for d in base]
    rng = np.random.default_rng(1)
    for size in (1, 7, 64):
        pick = rng.integers(0, len(base), size)
        dss = [_copy(base[i]) for i in pick]
        got = _fits(method, dss)
        for i, g in zip(pick, got):
            assert np.array_equal(g, alone[i], equal_nan=True)
    again = _fits(method, [_copy(d) for d in base[::-1]])[::-1]
    for a, b in zip(again, alone):
        assert np.array_equal(a, b, equal_nan=True)


def test_more_than_65535_fits():
    """70,000 1-D fits in one call of sb_scint_fit_1d against single calls."""
    import torch
    from scintools_b200 import _device as D, _lib
    z = np.load(os.path.join(ROOT, "tests", "golden", "scint_params_synthetic.npz"))
    acf = SO.fixture_acf(z, "acf1d")
    d_acf = D.upload(np.ascontiguousarray(acf))
    nf2, nt2 = acf.shape
    n = 70000
    rng = np.random.default_rng(4)
    n0 = rng.integers(6, 60, n)
    n1 = rng.integers(6, 40, n)
    wts = rng.uniform(0.5, 2.0, (n, 100))
    d_w = D.upload(wts)
    descs = []
    for i in range(n):
        d = _lib.ScintFit()
        d.acf, d.aux, d.pitch = d_acf.data_ptr(), d_w.data_ptr() + 800 * i, nt2
        d.s0, d.s1 = 8.0, 0.25
        d.p0 = (_lib.c_dbl * 5)(100.0 * rng.uniform(0.5, 2), 1.0 * rng.uniform(0.5, 2), 0.9,
                                5 / 3, 0.0)
        d.r0, d.c0, d.n0 = nf2 // 2, nt2 // 2, int(n0[i])
        d.r1, d.c1, d.n1 = nf2 // 2, nt2 // 2, int(n1[i])
        d.vary, d.bounded, d.weighted, d.max_nfev = 0b111, 0b111, 1, 50000
        descs.append(d)
    arr = (_lib.ScintFit * n)(*descs)
    out = D.empty((n, 11), torch.float64)
    info = D.empty((n, 2), torch.int32)
    _lib.check(_lib.lib.sb_scint_fit_1d(arr, n, out.data_ptr(), info.data_ptr(), D.stream_ptr()))
    out, info = D.download(out), D.download(info)
    # random crops and weights: some fits run away to the cap; each must still match alone
    print("statuses:", {int(s): int(c) for s, c in zip(*np.unique(info[:, 1], return_counts=True))})
    for i in list(rng.integers(0, n, 40)) + [0, 65535, 65536, n - 1]:
        o1 = D.empty((1, 11), torch.float64)
        i1 = D.empty((1, 2), torch.int32)
        one = (_lib.ScintFit * 1)(descs[i])
        _lib.check(_lib.lib.sb_scint_fit_1d(one, 1, o1.data_ptr(), i1.data_ptr(), D.stream_ptr()))
        assert np.array_equal(D.download(o1)[0], out[i], equal_nan=True)
        assert np.array_equal(D.download(i1)[0], info[i])


@pytest.mark.parametrize("fn", [f for f in FIXTURES if "j0437" in f])
@pytest.mark.parametrize("method", ["acf1d", "acf2d_approx"])
def test_end_to_end_device_acf(fn, method):
    """From dyn with the device's ACF: the reference's crop boxes, parameters within 1e-3."""
    from scintools_b200 import dynspec as P
    z = np.load(fn)
    ds = _ds(z, "acf1d")
    del ds.acf
    res = ds.get_scint_params(method=method)
    assert ds.acf.shape == (2 * ds.dyn.shape[0], 2 * ds.dyn.shape[1])
    case = "acf1d" if method == "acf1d" else "acf2d"
    q = list(SO.fit_keys(z, case))
    pl = P._scint_nofit(_copy(ds), False, 5, True, True)
    assert pl["nt_c"] == len(z[q[0] + "arg0"]) and pl["nf_c"] == len(z[q[0] + "arg1"])
    if method == "acf2d_approx":
        rows, cols, _, _ = P._scint_crop_2d(ds, pl["tau"], pl["dnu"], 5, False, False)
        assert [rows[0], len(rows), cols[0], len(cols)] == [int(v) for v in z[q[1] + "box"]]
    if _well_conditioned(z, q[-1]):
        for n in res.params:
            if res.params[n].vary:
                assert res.params[n].value == pytest.approx(float(z[q[-1] + "value_" + n]),
                                                            rel=1e-3, abs=1e-6), n


def test_known_recovery():
    """The crafted sheared ACF is the 2-D model with tau 60 s, dnu 3 MHz, phasegrad 8/60
    min/MHz plus noise: the 2-D fit recovers tau and dnu within three reported errors."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "scint_params_crafted.npz"))
    ds = _ds(z, "sheared_acf2d_approx")
    res = ds.get_scint_params(method="acf2d_approx")
    for n, truth in (("tau", 60.0), ("dnu", 3.0)):
        p = res.params[n]
        print(n, p.value, p.stderr)
        assert abs(p.value - truth) <= 3 * p.stderr


def test_full_frame_2d_large():
    """acf2d_approx, full_frame=True, on a 1024 x 2048 spectrum (ACF 2048 x 4096): a
    stationary point with lmfit's errors there, and the tight oracle's minimum from it."""
    from scintools_b200.dynspec import Dynspec
    nf, nt, dt, df = 1024, 2048, 8.0, 0.05
    tl = (np.arange(2 * nt) - nt) * dt
    fl = (np.arange(2 * nf) - nf) * df
    T, F = np.meshgrid(tl, fl)
    acf = np.exp(-(np.abs((T - 20 * F) / 300.0) ** 2.5 +
                   np.abs(F / (2.0 / np.log(2))) ** 1.5) ** (2 / 3))
    acf *= (1 - np.abs(T) / (nt * dt)) * (1 - np.abs(F) / (nf * df))
    acf += np.random.default_rng(2).normal(0, 0.002, acf.shape)
    acf[nf, nt] += 0.05
    acf /= acf.max()
    ds = Dynspec.__new__(Dynspec)
    ds.dyn = np.random.default_rng(3).exponential(1.0, (nf, nt))
    ds.name = "large"
    ds.dt, ds.df, ds.tobs, ds.bw, ds.nsub, ds.nchan, ds.freq = dt, df, nt * dt, nf * df, nt, \
        nf, 1400.0
    ds.acf = acf
    kw = dict(method="acf2d_approx", full_frame=True)
    res = ds.get_scint_params(**kw)
    kind, args = _device_args(ds, kw, res)
    assert args[2].shape == (2 * nf - 1, 2 * nt - 1)
    _check_fit(res, kind, args, list(SO.SLOTS))
    p = {n: res.params[n].value for n in SO.SLOTS}
    tight, _, trel = SO.fit_tight(kind, args, p, ["tau", "dnu", "amp", "phasegrad"])
    for n in ("tau", "dnu", "amp", "phasegrad"):
        assert p[n] == pytest.approx(tight[n], rel=1e-7, abs=1e-12), n


@pytest.mark.parametrize("shape,ok", [((2, 5), True), ((1, 5), False), ((2, 4), False)])
def test_size_limits(shape, ok):
    from scintools_b200.dynspec import BasicDyn, Dynspec
    rng = np.random.default_rng(0)
    dyn = rng.exponential(1.0, shape)
    ds = Dynspec(dyn=BasicDyn(dyn, times=np.arange(max(shape[1], 3)) * 10.0,
                              freqs=1400 + 0.5 * np.arange(max(shape[0], 3)), df=0.5),
                 verbose=False)
    ds.dyn = dyn
    if ok:
        try:                    # the guesses of so short a cut may meet the reference's
            ds.get_scint_params(method="nofit")         # squeeze()[0] IndexError
        except IndexError:
            pass
        assert ds.acf.shape == (4, 10)
    else:
        with pytest.raises(ValueError):
            ds.get_scint_params(method="acf1d")


def test_nan_in_dyn_raises():
    z = np.load(os.path.join(ROOT, "tests", "golden", "scint_params_synthetic.npz"))
    ds = _ds(z, "acf1d")
    del ds.acf
    ds.dyn[5, 7] = np.nan
    with pytest.raises(ValueError):
        ds.get_scint_params(method="acf1d")
