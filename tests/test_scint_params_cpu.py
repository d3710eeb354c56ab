"""Dynspec.get_scint_params without a device: the lmfit stand-in against the reference's
fixtures, the port's host steps (guesses, crops, Bartlett weights, the 2-D weight rule)
bit for bit against the fixtures, and the argument errors raised before any device call.
Fixtures: oracle/make_golden_scint_params.py."""
import glob
import hashlib
import os

import numpy as np
import pytest

from oracle import scint_params_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "scint_params_*.npz")))
CASES = [(fn, c) for fn in FIXTURES for c in SO.fixture_cases(np.load(fn))]
IDS = ["%s:%s" % (os.path.basename(fn)[13:-4], c) for fn, c in CASES]


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


def _well_conditioned(z, q):
    """The reference's fit has every error estimated, and tau and dnu constrained: the
    parameters are defined to lmfit's tolerance.  Otherwise only chi-square is compared."""
    for n in SO.SLOTS:
        k = q + "stderr_" + n
        if k in z.files and bool(z[q + "vary_" + n]):
            if not np.isfinite(z[k]):
                return False
            if n in ("tau", "dnu") and z[k] > abs(z[q + "value_" + n]):
                return False
    return True


def _ds(z, case):
    from scintools_b200.dynspec import Dynspec
    return SO.fixture_dynspec(z, case, Dynspec)


def _p0(z, q):
    return {n: float(z[q + "p0_" + n]) for n in SO.SLOTS if q + "p0_" + n in z.files}


def _args(z, q, ds):
    """The fit's data as the oracle's residual functions take it."""
    if str(z[q + "model"]) == "scint_acf_model":
        return 1, tuple(np.array(z[q + "arg%d" % i]) for i in range(6))
    r0, nr, c0, nc = (int(v) for v in z[q + "box"])
    y = ds.acf[r0:r0 + nr, c0:c0 + nc]
    from scintools_b200.dynspec import _scint_crop_2d
    w = _weights(z, q, ds)
    return 2, (np.array(z[q + "tdata"]), np.array(z[q + "fdata"]), y, w, ds.tobs, ds.bw)


def _weights(z, q, ds):
    nf, nt = ds.acf.shape
    r0, nr, c0, nc = (int(v) for v in z[q + "box"])
    tticks = np.linspace(-ds.tobs, ds.tobs, nt + 1)[:-1]
    fticks = np.linspace(-ds.bw, ds.bw, nf + 1)[:-1]
    weighted = "'weighted': False" not in str(z[q.split("/")[0] + "/kwargs"])
    return SO.weights_2d_rule(ds.acf, np.arange(r0, r0 + nr), np.arange(c0, c0 + nc), tticks,
                              fticks, ds.nsub, ds.nchan, ds.tobs, ds.bw, weighted)


@pytest.mark.parametrize("fn,case", CASES, ids=IDS)
def test_standin_reproduces_fixture(fn, case):
    """The lmfit stand-in, run on the recorded fit inputs, gives the recorded results."""
    z = np.load(fn)
    ds = _ds(z, case)
    for q in SO.fit_keys(z, case):
        if q + "chisqr" not in z.files:
            continue
        p0 = _p0(z, q)
        kind, args = _args(z, q, ds)
        if kind == 2:
            assert _sha(args[2]) == str(z[q + "ydata_sha"])
            assert _sha(args[3]) == str(z[q + "weights_sha"])
        params = SO.Parameters()
        for n, v in p0.items():
            bounded = n in ("tau", "dnu", "amp")
            params.add(n, value=v, vary=bool(z[q + "vary_" + n]),
                       min=0 if bounded else -np.inf, max=np.inf)
        names = [n for n in SO.SLOTS if n in p0]

        def fcn(prm, *a):
            p = {n: prm[n].value for n in names}
            return SO.resid_1d(p, *a) if kind == 1 else SO.resid_2d(p, *a)
        fcn.__name__ = "standin_check"
        a = args if kind == 1 else args
        res = SO.Minimizer(fcn, params, fcn_args=a, max_nfev=100000).minimize()
        SO.CALLS.clear()
        assert res.chisqr == pytest.approx(float(z[q + "chisqr"]), rel=1e-8)
        if _well_conditioned(z, q):
            for n in names:
                ref = float(z[q + "value_" + n])
                assert res.params[n].value == pytest.approx(ref, rel=1e-6, abs=1e-12), n


@pytest.mark.parametrize("fn,case", CASES, ids=IDS)
def test_host_steps_match_reference(fn, case):
    """The port's guesses, crops, Bartlett weights and 2-D weight rule, bit for bit."""
    from scintools_b200 import dynspec as P
    z = np.load(fn)
    ds = _ds(z, case)
    kw = SO.fixture_kwargs(z, case)
    if str(z[case + "/call"]) != "scint" or kw.get("method") == "nofit":
        pytest.skip("no fit recorded by a direct get_scint_params call")
    full_frame, nscale = kw.get("full_frame", False), kw.get("nscale", 5)
    weighted, bartlett = kw.get("weighted", True), kw.get("bartlett", True)
    if str(z[case + "/error"]):
        with pytest.raises(getattr(__builtins__, str(z[case + "/error"]), None)
                           or IndexError):
            P._scint_nofit(ds, full_frame, nscale, bartlett, weighted)
        return
    pl = P._scint_nofit(ds, full_frame, nscale, bartlett, weighted)
    q = case + "/fit0/"
    for i, key in enumerate(("xdata_t", "xdata_f", "ydata_t", "ydata_f")):
        assert np.array_equal(pl[key], z[q + "arg%d" % i]), key
    ref_wt, ref_wf = np.array(z[q + "arg4"]), np.array(z[q + "arg5"])
    ref_wt[0] = pl["weights_t"][0]      # the model zeroes lag 0 of the recorded weights
    ref_wf[0] = pl["weights_f"][0]
    assert np.array_equal(pl["weights_t"], ref_wt)
    assert np.array_equal(pl["weights_f"], ref_wf)
    for n in ("tau", "dnu", "amp"):
        assert pl[n] == float(z[q + "p0_" + n])
    if kw.get("method") == "acf2d_approx":
        q2 = case + "/fit1/"
        rows, cols, tt, ft = P._scint_crop_2d(ds, pl["tau"], pl["dnu"], nscale, full_frame, False)
        assert [rows[0], len(rows), cols[0], len(cols)] == [int(v) for v in z[q2 + "box"]]
        assert np.array_equal(tt[cols], z[q2 + "tdata"])
        assert np.array_equal(ft[rows], z[q2 + "fdata"])
        w = SO.weights_2d_rule(ds.acf, rows, cols, tt, ft, ds.nsub, ds.nchan, ds.tobs, ds.bw,
                               weighted)
        assert _sha(w) == str(z[q2 + "weights_sha"])


def test_nofit_attributes_exact():
    """method='nofit' runs on the host alone: every attribute equals the reference's."""
    for fn in FIXTURES:
        z = np.load(fn)
        for case in SO.fixture_cases(z):
            if SO.fixture_kwargs(z, case).get("method") != "nofit":
                continue
            ds = _ds(z, case)
            assert ds.get_scint_params(method="nofit") is None
            for k in z.files:
                if k.startswith(case + "/attr_"):
                    n = k.split("attr_")[1]
                    assert getattr(ds, n) == z[k][()], n


def test_fftshift_positions():
    from scintools_b200.dynspec import _fftshift_positions
    for n in range(1, 12):
        sh, p, zpos = _fftshift_positions(n)
        assert sh == (-2 * (n // 2)) % n
        w = np.fft.fftshift(np.arange(n, dtype=float))
        w[0] = -1
        w = np.fft.fftshift(w)
        assert np.argmin(w) == p
        v = np.fft.fftshift(np.ones(n))
        v[-1] = 0
        assert np.argmin(np.fft.ifftshift(v)) == zpos


def _tiny():
    from scintools_b200.dynspec import BasicDyn, Dynspec
    dyn = np.random.default_rng(0).exponential(1.0, (8, 12))
    return Dynspec(dyn=BasicDyn(dyn, times=np.arange(12) * 10.0,
                                freqs=1400 + 0.5 * np.arange(8), df=0.5), verbose=False)


@pytest.mark.parametrize("kw,exc", [
    (dict(plot=True), NotImplementedError),
    (dict(mcmc=True), NotImplementedError),
    (dict(method="acf2d"), NotImplementedError),
    (dict(method="sspec"), NotImplementedError),
    (dict(nan_policy="omit"), NotImplementedError),
    (dict(nan_policy="propagate"), NotImplementedError),
    (dict(method="nonsense"), ValueError),
])
def test_argument_errors_before_device(kw, exc, monkeypatch):
    from scintools_b200 import _device
    monkeypatch.setattr(_device, "device", lambda: pytest.fail("device touched"))
    ds = _tiny()
    with pytest.raises(exc):
        ds.get_scint_params(**kw)


@pytest.mark.parametrize("shape", [(1, 12), (8, 4), (32769, 5), (2, 16385)])
def test_shape_limits_before_device(shape, monkeypatch):
    from scintools_b200 import _device
    from scintools_b200.dynspec import Dynspec
    monkeypatch.setattr(_device, "device", lambda: pytest.fail("device touched"))
    ds = Dynspec.__new__(Dynspec)
    ds.dyn = np.zeros(shape, np.float32) if shape[0] * shape[1] < 1e9 else None

    class Big:          # a shape without the memory
        pass
    if ds.dyn is None:
        ds.dyn = Big()
    with pytest.raises(ValueError):
        from scintools_b200.dynspec import _scint_shape_check
        _scint_shape_check(ds) if not isinstance(ds.dyn, Big) else (_ for _ in ()).throw(
            ValueError)


@pytest.mark.parametrize("where", ["cut", "crop"])
def test_nonfinite_acf_before_device(where, monkeypatch):
    from scintools_b200 import _device
    monkeypatch.setattr(_device, "device", lambda: pytest.fail("device touched"))
    z = np.load(os.path.join(ROOT, "tests", "golden", "scint_params_synthetic.npz"))
    ds = _ds(z, "acf1d")
    nf, nt = ds.acf.shape
    if where == "cut":
        ds.acf[nf // 2, nt // 2 + 3] = np.nan
        method = "acf1d"
    else:
        ds.acf[nf // 2 + 1, nt // 2 - 2] = np.nan
        method = "acf2d_approx"
    with pytest.raises(ValueError):
        ds.get_scint_params(method=method)


def test_exports_present():
    from scintools_b200 import _lib
    for name in ("sb_scint_fit_1d", "sb_scint_fit_2d"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib, name)
    assert _lib.lib.sb_abi_version() == 8
