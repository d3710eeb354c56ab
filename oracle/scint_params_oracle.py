"""Host restatements behind Dynspec.get_scint_params (TEST INFRASTRUCTURE, see
oracle/__init__.py).

(a) ``lmfit`` -- a stand-in for the parts of lmfit the reference's get_scint_params uses:
    Parameters / Parameter, Minimizer(...).minimize() with the 'leastsq' method, and
    fit_report.  It is a restatement, written because lmfit is not installed where the
    fixtures are made: scipy.optimize.leastsq with xtol = ftol = gtol = 1e-7 and maxfev =
    max_nfev, lmfit's bound transforms (min only: x -> min - 1 + sqrt(x^2 + 1)), the residual
    raveled, ValueError on a NaN residual (nan_policy='raise'), the covariance scaled by the
    transforms' gradients and by redchi, stderr None where leastsq returns no covariance.
    ``install()`` puts it in sys.modules['lmfit']; every Minimizer it builds is recorded in
    ``CALLS`` (model name, fcn_args, starting parameters, result).

(b) A tight float64 restatement of the two models with analytic Jacobians (``resid_1d``,
    ``resid_2d``), minimised to a relative gradient of 1e-12 (``fit_tight``), and lmfit's
    standard errors at any given point (``stderr_at``).  The device results are checked
    against these.
"""
import sys
import types
from collections import OrderedDict
from copy import deepcopy

import numpy as np

SLOTS = ("tau", "dnu", "amp", "alpha", "phasegrad")
LN2 = np.log(2)

# ---------------------------------------------------------------------------
# (a) the lmfit stand-in
# ---------------------------------------------------------------------------
CALLS = []


class Parameter:
    def __init__(self, name, value=None, vary=True, min=-np.inf, max=np.inf):
        self.name, self.vary, self.min, self.max = name, vary, min, max
        self.value = value
        self.stderr = None

    @property
    def value(self):
        return self._val

    @value.setter
    def value(self, v):
        if v is not None and self.min is not None:
            v = max(self.min, min(self.max, v)) if np.isfinite(v) else v
        self._val = v

    # lmfit's transforms (Parameter.setup_bounds / from_internal / scale_gradient)
    def to_internal(self):
        if np.isfinite(self.min) and not np.isfinite(self.max):
            return np.sqrt((self.value - self.min + 1.0) ** 2 - 1)
        if not np.isfinite(self.min) and not np.isfinite(self.max):
            return self.value
        raise NotImplementedError("bounds other than min-only or none")

    def from_internal(self, x):
        if np.isfinite(self.min):
            return self.min - 1.0 + np.sqrt(x * x + 1)
        return x

    def scale_gradient(self, x):
        if np.isfinite(self.min):
            return x / np.sqrt(x * x + 1)
        return 1.0


class Parameters(OrderedDict):
    def add(self, name, value=None, vary=True, min=-np.inf, max=np.inf):
        self[name] = Parameter(name, value, vary, min, max)

    def valuesdict(self):
        return OrderedDict((k, p.value) for k, p in self.items())


class AbortFitException(Exception):
    pass


class MinimizerResult:
    pass


class Minimizer:
    def __init__(self, userfcn, params, fcn_args=(), nan_policy='raise', max_nfev=None,
                 **kws):
        self.userfcn, self.params, self.fcn_args = userfcn, params, fcn_args
        self.nan_policy, self.max_nfev = nan_policy, max_nfev
        self.record = {"model": userfcn.__name__, "params0": deepcopy(params),
                       "fcn_args": fcn_args}
        CALLS.append(self.record)

    def minimize(self, method='leastsq'):
        from scipy.optimize import leastsq
        params = deepcopy(self.params)
        names = [k for k, p in params.items() if p.vary]
        x0 = np.array([params[k].to_internal() for k in names], dtype=np.float64)
        nfev = [0]
        last = [x0]
        maxfev = self.max_nfev if self.max_nfev is not None else 2000 * (len(names) + 1)

        def resid(x):
            nfev[0] += 1
            last[0] = x
            if nfev[0] > maxfev:
                raise AbortFitException()
            for k, xi in zip(names, x):
                params[k]._val = params[k].from_internal(xi)
            out = np.asarray(self.userfcn(params, *self.fcn_args), dtype=np.float64).ravel()
            if self.nan_policy == 'raise' and np.isnan(out).any():
                raise ValueError("NaN values detected in your input data or the output of "
                                 "your objective/model function - fitting algorithms cannot "
                                 "handle this!")
            return out

        res = MinimizerResult()
        res.aborted = False
        try:
            best, cov_x, info, msg, ier = leastsq(resid, x0, full_output=1, xtol=1e-7,
                                                  ftol=1e-7, gtol=1e-7, maxfev=maxfev)
            res.success = ier in (1, 2, 3, 4)
        except AbortFitException:
            best, cov_x, ier = last[0], None, -1
            res.success, res.aborted = False, True
        for k, xi in zip(names, best):
            params[k]._val = params[k].from_internal(xi)
        r = np.asarray(self.userfcn(params, *self.fcn_args), dtype=np.float64).ravel()
        res.residual = r
        res.nfev = nfev[0]
        res.ndata = r.size
        res.nvarys = len(names)
        res.nfree = res.ndata - res.nvarys
        res.chisqr = float((r ** 2).sum())
        res.redchi = res.chisqr / max(1, res.nfree)
        res.ier = ier
        res.var_names = names
        res.covar = None
        if cov_x is not None and not res.aborted:
            g = np.array([params[k].scale_gradient(xi) for k, xi in zip(names, best)])
            res.covar = cov_x * np.outer(g, g) * res.redchi
            for i, k in enumerate(names):
                params[k].stderr = float(np.sqrt(res.covar[i, i]))
        res.params = params
        self.record["result"] = res
        return res


def fit_report(result):
    lines = ["[[Fit Statistics]]", "    # function evals = %d" % result.nfev,
             "    chi-square = %r" % result.chisqr, "[[Variables]]"]
    for k, p in result.params.items():
        lines.append("    %s: %r +/- %r" % (k, p.value, p.stderr))
    return "\n".join(lines)


def install():
    """Put the stand-in in sys.modules['lmfit'] (before oracle.ref_loader.load())."""
    mod = types.ModuleType("lmfit")
    mod.Parameters, mod.Parameter, mod.Minimizer = Parameters, Parameter, Minimizer
    mod.fit_report, mod.MinimizerResult = fit_report, MinimizerResult
    mod.__b200_standin__ = True
    sys.modules["lmfit"] = mod
    return mod


# ---------------------------------------------------------------------------
# (b) tight restatement
# ---------------------------------------------------------------------------
def resid_1d(p, xt, xf, yt, yf, wt, wf, jac=False):
    """scint_acf_model (time cut then frequency cut) at p = {tau, dnu, amp, alpha}; with
    jac=True also d(residual)/d(tau, dnu, amp, alpha) [n][4]."""
    wt = np.array(wt, dtype=np.float64)
    wf = np.array(wf, dtype=np.float64)
    wt[0] = wf[0] = 0.0
    tau, dnu, amp, alpha = p["tau"], p["dnu"], p["amp"], p["alpha"]
    tri_t = 1 - xt / max(xt)
    tri_f = 1 - xf / max(xf)
    q = xt / tau
    u = q ** alpha
    et = np.exp(-u)
    mt = amp * et * tri_t
    ef = np.exp(-(xf / (dnu / LN2)))
    mf = amp * ef * tri_f
    r = np.concatenate(((yt - mt) * wt, (yf - mf) * wf))
    if not jac:
        return r
    J = np.zeros((r.size, 4))
    nt = xt.size
    J[:nt, 0] = -wt * mt * alpha * u / tau
    J[nt:, 1] = -wf * mf * xf * LN2 / dnu ** 2
    J[:nt, 2] = -wt * et * tri_t
    J[nt:, 2] = -wf * ef * tri_f
    with np.errstate(divide='ignore', invalid='ignore'):
        J[:nt, 3] = np.where(xt > 0, wt * mt * u * np.log(np.where(xt > 0, q, 1.0)), 0.0)
    return r, J


def model_weights_2d(weights):
    """The weights scint_acf_model_2d_approx applies: fftshift, [-1, -1] = 0, ifftshift."""
    w = np.fft.fftshift(np.array(weights, dtype=np.float64))
    w[-1, -1] = 0
    return np.fft.ifftshift(w)


def resid_2d(p, tdata, fdata, ydata, weights, tobs, bw, jac=False):
    """scint_acf_model_2d_approx at p = {tau, dnu, amp, alpha, phasegrad}, raveled; with
    jac=True also d(residual)/d(tau, dnu, amp, alpha, phasegrad) [n][5].  weights are the
    ones the reference passes in fcn_args."""
    w = model_weights_2d(weights)
    tau, dnu, amp, alpha, pg = p["tau"], p["dnu"], p["amp"], p["alpha"], p["phasegrad"]
    t = np.asarray(tdata)[None, :]
    f = np.asarray(fdata)[:, None]
    a = (t - pg * 60 * f) / tau
    pw = 3 * alpha / 2
    A = np.abs(a) ** pw
    B = np.abs(f / (dnu / LN2)) ** 1.5
    S = A + B
    Q = S ** (2 / 3)
    tri = (1 - np.abs(t) / tobs) * (1 - np.abs(f) / bw)
    e = np.exp(-Q)
    m = amp * e * tri
    r = ((ydata - m) * w).ravel()
    if not jac:
        return r
    with np.errstate(divide='ignore', invalid='ignore'):
        h = np.where(S > 0, w * m * (2 / 3) * Q / S, 0.0)
        dAda = np.where(a != 0, pw * A / np.where(a != 0, a, 1.0), 0.0)
        la = np.where(a != 0, np.log(np.abs(np.where(a != 0, a, 1.0))), 0.0)
    J = np.stack([h * (-pw * A / tau), h * (-1.5 * B / dnu), -w * e * tri,
                  np.where(a != 0, h * 1.5 * A * la, 0.0),
                  h * dAda * (-60.0 * f / tau)], axis=-1)
    return r, J.reshape(-1, 5)


def _fun(kind, args):
    if kind == 1:
        return lambda p, jac=False: resid_1d(p, *args, jac=jac)
    return lambda p, jac=False: resid_2d(p, *args, jac=jac)


def stderr_at(kind, args, p, names):
    """lmfit's standard errors of the varying parameters `names` at p:
    sqrt(diag(inv(J^T J)) redchi) in the external parameters (the bound transform's
    gradients cancel).  Returns (dict name -> stderr, chisqr, relative gradient)."""
    fun = _fun(kind, args)
    r, J = fun(p, jac=True)
    cols = [SLOTS.index(n) for n in names]
    J = J[:, cols]
    chi = float(r @ r)
    redchi = chi / max(1, r.size - len(names))
    C = np.linalg.inv(J.T @ J)
    g = J.T @ r
    rel = np.max(np.abs(g) / np.sqrt(np.maximum(np.sum(J * J, axis=0) * chi, 1e-300)))
    return {n: float(np.sqrt(C[i, i] * redchi)) for i, n in enumerate(names)}, chi, rel


def fit_tight(kind, args, p0, names, bounded=("tau", "dnu", "amp")):
    """Minimise chi-square from p0 (dict) over `names`, in lmfit's internal variables for
    the bounded ones, to a relative gradient of 1e-12 (scipy's MINPACK lm with the
    analytic Jacobian, then Gauss-Newton polishing).  Returns (p, chisqr, rel gradient)."""
    from scipy.optimize import least_squares
    fun = _fun(kind, args)
    cols = [SLOTS.index(n) for n in names]
    bmask = np.array([n in bounded for n in names])

    def ext(x):
        return np.where(bmask, -1.0 + np.sqrt(x * x + 1), x)

    def unpack(x):
        p = dict(p0)
        p.update(zip(names, ext(x)))
        return p

    def r(x):
        return fun(unpack(x))

    def jac(x):
        _, J = fun(unpack(x), jac=True)
        return J[:, cols] * np.where(bmask, x / np.sqrt(x * x + 1), 1.0)[None, :]

    v0 = np.array([p0[n] for n in names], dtype=np.float64)
    with np.errstate(invalid='ignore'):
        x = np.where(bmask, np.sqrt((v0 + 1.0) ** 2 - 1), v0)
    sol = least_squares(r, x, jac=jac, method='lm', xtol=1e-15, ftol=1e-15, gtol=1e-15,
                        max_nfev=100000)
    x = sol.x
    # Gauss-Newton polishing to a relative gradient of 1e-12 (or until a step stops helping)
    for _ in range(30):
        p = unpack(x)
        if stderr_at(kind, args, p, names)[2] <= 1e-12:
            break
        rv, J = r(x), jac(x)
        step = np.linalg.lstsq(J, -rv, rcond=None)[0]
        if not np.sum(r(x + step) ** 2) <= np.sum(rv ** 2):
            break
        x = x + step
    p = unpack(x)
    _, chi, rel = stderr_at(kind, args, p, names)
    return p, chi, rel


# ---------------------------------------------------------------------------
# fixtures (tests/golden/scint_params_*.npz, oracle/make_golden_scint_params.py)
# ---------------------------------------------------------------------------
META = ("dt", "df", "tobs", "bw", "nsub", "nchan", "freq")


def fixture_cases(z):
    """Case names of a fixture file, in file order."""
    seen = []
    for k in z.files:
        if "/" in k and k.split("/")[0] not in seen:
            seen.append(k.split("/")[0])
    return seen


def fixture_acf(z, case):
    """The reference's float64 ACF of a case: the crafted one, or the ACF of dyn recomputed
    by oracle.dynspec_oracle.calc_acf and checked against the stored sha256."""
    import hashlib
    from oracle import dynspec_oracle as DO
    for k in z.files:
        if k.startswith("acf_") and k != "acf_sha" and case.startswith(k[4:] + "_"):
            return np.array(z[k])
    acf = DO.calc_acf(z["dyn"])
    assert hashlib.sha256(acf.tobytes()).hexdigest() == str(z["acf_sha"])
    return acf


def fixture_dynspec(z, case, cls):
    """An object of class cls (the port's Dynspec) with the fixture's attributes and ACF."""
    ds = cls.__new__(cls)
    ds.dyn = np.array(z["dyn"], dtype=np.float64)
    name = str(z["name"])
    if case.startswith("simname"):
        name = "sim:mb2=2.0,ar=1"
    ds.name = name
    for k, v in zip(META, z["meta"]):
        setattr(ds, k, int(v) if k in ("nsub", "nchan") else float(v))
    ds.acf = fixture_acf(z, case)
    return ds


def fixture_kwargs(z, case):
    import ast
    return ast.literal_eval(str(z[case + "/kwargs"]))


def fit_keys(z, case):
    k = 0
    while "%s/fit%d/model" % (case, k) in z.files:
        yield "%s/fit%d/" % (case, k)
        k += 1


def weights_2d_rule(acf, rows, cols, tticks, fticks, nsub, nchan, tobs, bw, weighted):
    """The 2-D fcn_args weights (before the model's own shift), made the way the device
    makes them: the formula at the position the two fftshifts move each weight from, then
    1e10 at the position the first shift's [0][0] lands on.  Materialised for the tests."""
    from scintools_b200.dynspec import _fftshift_positions
    y = acf[rows[0]:rows[-1] + 1, cols[0]:cols[-1] + 1]
    at = ((tobs - abs(tticks)) / max(tticks))[cols]
    af = ((bw - abs(fticks)) / max(fticks))[rows]
    with np.errstate(divide='ignore', invalid='ignore'):
        N = (float(nsub * nchan) * at[None, :]) * af[:, None]
        e = 1 / np.sqrt(N)
        e[~np.isfinite(e)] = np.inf
        w = 1 / e if weighted else np.ones_like(y)
        w[y - 1 / w < 0] = 0
    shf, pf, _ = _fftshift_positions(len(rows))
    sht, pt, _ = _fftshift_positions(len(cols))
    w = w[(np.arange(len(rows)) + shf) % len(rows)][:, (np.arange(len(cols)) + sht) % len(cols)]
    w[pf, pt] = 1e10
    return w
