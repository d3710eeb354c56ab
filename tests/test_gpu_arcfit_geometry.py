"""The arc-fit resampling kernels (csrc/normsspec.cu) at every geometry edge against
float64 numpy, and Dynspec.norm_sspec / fit_arc against the unmodified reference on
more spectra (tests/golden/arcfit_*.npz, made by oracle/make_golden_arcfit.py).

norm_sspec_rows_kernel resamples each delay row with np.interp onto the normalised
Doppler axis and sums the power of the unmasked samples; norm_sspec_avg_kernel
scrunches the rows with weights.  CASES puts each size on one axis with small
ones on the others and builds the inputs that reach each branch of the kernel:
selections of 0, 1, 2 and all columns, imax on a Doppler sample and one ulp
either side, the delay-zero row (s = 0: one NaN knot), queries on knots and on
both ends of a selection, unmasked queries outside [x0, xl], NaN queries, NaN
columns as cutmid writes them, and +-inf samples that reach every NaN fallback
of np.interp.  test_case_table_coverage (no GPU) restates those branches as
predicates on the inputs and fails if an edit to the table drops one.

The reference is float64 numpy on the same float32 samples the device receives.
Bounds:
  mask   bit for bit.  It is a comparison of fp64 values that both sides compute
         with the same correctly rounded operations.
  norm   np.float32(np.interp(...)) bit for bit.  interp_one makes numpy's interval
         search and its NaN fallbacks with the same correctly rounded __ddiv_rn /
         __dsub_rn / __dmul_rn / __dadd_rn steps, in the same order, so any
         difference is a bug, not rounding.
  power  the mean of the n terms t = 10^(r/10) of the unmasked finite samples (np.ma's
         safe division in normSspec / 10 masks +-inf).  CUDA's pow is within 2 ulp and
         the host's within 1; the two sums run in different orders, each within
         (n - 1) 2^-53 sum|t|; the division adds one ulp each:
             |got - ref| <= (n + 4) 2^-52 sum|t| / n
  avg    sum w v / sum w over the rows with a sample, from the same float32 samples
         (the kernel's own output): both sums in any order, the products and the
         division, on either side:
             |got - ref| <= (n + 2) 2^-52 (sum|w v| + |ref| sum|w|) / |sum w|
         Against the reference's fixtures the float32 rounding of the samples the
         average reads adds 2^-24 sum|w v| / |sum w|.
  Non-finite references (+-inf, NaN) must be matched exactly.
"""
import json
import os
import zlib
from collections import namedtuple

import numpy as np
import pytest

from test_arcfit_cpu import _bare_dynspec, numpy_norm_rows

U52 = 2.0 ** -52
U24 = 2.0 ** -24

# worst error seen per family in this process: error / bound
MEASURED = {}


def _record(family, ratio):
    MEASURED[family] = max(MEASURED.get(family, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    if MEASURED:
        capture = request.config.pluginmanager.getplugin("capturemanager")
        with capture.global_and_fixture_disabled():
            print("\narc-fit geometry: worst error / bound per family (bits: samples that differ)")
            for k in sorted(MEASURED):
                print("  %-28s %.3g" % (k, MEASURED[k]))


# --------------------------------------------------------------------------
# the case table
# --------------------------------------------------------------------------
Case = namedtuple("Case", "nr nc nq eta maxnormfac fdop_kind sample_kind tdel_kind query_kind")

DT = 7.3        # s: calc_sspec's Doppler step 1e3 / (nc dt) is no power of two
STEP = 0.25     # exact Doppler step of the "pow2" axis


def case_id(c):
    return "nr%d-nc%d-nq%d-eta%r-m%r-%s-%s-%s-%s" % c


def _rng(c, salt=""):
    return np.random.default_rng(zlib.crc32((case_id(c) + salt).encode()))


def make_fdop(c):
    n = c.nc
    if c.fdop_kind == "sspec":      # calc_sspec: fd * 1e3 / (ncfft * dt)
        fd = np.arange(-(n // 2), n - n // 2, dtype=np.float64)
        return fd * 1e3 / (n * DT)
    k = np.arange(n, dtype=np.float64)
    if c.fdop_kind == "pow2":
        return (k - n // 2) * STEP
    if c.fdop_kind == "halfbin":    # no zero Doppler: the smallest selection has 2 samples
        return (k - n / 2 + 0.5) * STEP
    if c.fdop_kind == "long_right":  # the positive end is the longer: |fdop[hi]| > |fdop[lo]|
        return (k - n // 2 + 3) * STEP
    if c.fdop_kind == "positive":
        return (k + 1.5) * STEP
    if c.fdop_kind == "jitter":     # the uniform-step guess lands one interval either side
        return (k - n // 2 + _rng(c, "jitter").uniform(-0.3, 0.3, n)) * STEP
    if c.fdop_kind == "wide_first":  # first step 1.5 x: guesses fall short (right loop)
        return np.concatenate(([-(n // 2) * STEP - 0.5 * STEP], (k[1:] - n // 2) * STEP))
    if c.fdop_kind == "narrow_first":  # first step 0.5 x: guesses overshoot (left loop)
        return np.concatenate(([-(n // 2) * STEP + 0.5 * STEP], (k[1:] - n // 2) * STEP))
    raise ValueError(c.fdop_kind)


def make_tdel(c):
    i = np.arange(c.nr, dtype=np.float64)
    if c.tdel_kind == "lin":
        return (i + 1) * 0.37
    if c.tdel_kind == "zero":       # startbin = 0: the delay-zero row
        return i * 0.37
    if c.tdel_kind == "exact":      # sqrt(tdel / eta) = 2^(i mod 4 - 1), exactly
        return c.eta * 4.0 ** (i % 4 - 1)
    raise ValueError(c.tdel_kind)


def _selection(fdop, s, mnf):
    sel = np.flatnonzero(np.abs(fdop) <= mnf * s)
    return (sel[0], sel[-1]) if sel.size else (None, None)


def make_queries(c, fdop, tdel):
    m, nq = c.maxnormfac, c.nq
    if c.query_kind == "lin":       # norm_sspec's own axis
        return np.linspace(-m, m, nq)
    if c.query_kind == "wide":      # beyond +-maxnormfac on both sides
        return np.linspace(-1.4 * m, 1.4 * m, nq)
    if c.query_kind == "nan":
        x = np.linspace(-1.2 * m, 1.2 * m, nq)
        x[::7] = np.nan
        return x
    if c.query_kind == "knots":     # fdop[k] / s exactly: both ends first, then the interior
        ends, inner = [], []
        for ii in sorted({0, 1 % c.nr, c.nr // 2, c.nr - 1}):
            s = np.sqrt(tdel[ii] / c.eta)
            lo, hi = _selection(fdop, s, m)
            if lo is None:
                continue
            with np.errstate(invalid="ignore"):     # s = 0: one NaN knot
                xp = fdop[lo:hi + 1] / s
            ends += [xp[0], xp[-1]]
            inner += list(xp[1:-1][_rng(c, "k%d" % ii).permutation(max(len(xp) - 2, 0))[:64]])
        x = np.array(ends + inner + list(np.linspace(-1.2 * m, 1.2 * m, nq)))
        return x[:nq]
    raise ValueError(c.query_kind)


def make_samples(c):
    rng = _rng(c, "samples")
    x = rng.normal(0.0, 10.0, (c.nr, c.nc))
    mid = c.nc // 2
    if c.sample_kind == "cutmid":   # dynspec.py:2049: int(nc/2 - cutmid//2):int(nc/2 + cutmid//2)
        x[:, max(mid - 2, 0):mid + 2] = np.nan
    elif c.sample_kind == "special":
        # near the middle, inside every non-trivial selection, and at random columns
        pats = ([np.nan], [-np.inf], [np.inf], [-np.inf, np.inf], [np.inf, -np.inf],
                [np.inf, np.inf], [-np.inf, -np.inf])
        for ii in range(c.nr):
            p = pats[ii % len(pats)]
            at = mid + 1 + (ii // len(pats)) % 3
            if at + len(p) <= c.nc:
                x[ii, at:at + len(p)] = p
            for q in pats:
                at = int(rng.integers(0, max(c.nc - 1, 1)))
                x[ii, at:at + len(q)] = q[:c.nc - at]
    elif c.sample_kind == "db_zero":  # 10 log10 of exact-zero power bins
        x[rng.random(x.shape) < 0.03] = -np.inf
    elif c.sample_kind != "normal":
        raise ValueError(c.sample_kind)
    return x.astype(np.float32)


def make_weights(c):
    return _rng(c, "weights").uniform(-0.5, 2.0, c.nr)


_INPUTS = {}


def inputs(c):
    if c not in _INPUTS:
        fdop, tdel = make_fdop(c), make_tdel(c)
        _INPUTS.clear()
        _INPUTS[c] = dict(sspec=make_samples(c), fdop=fdop, tdel=tdel,
                          fdopnew=make_queries(c, fdop, tdel), weights=make_weights(c))
    return _INPUTS[c]


def _C(nr, nc, nq, fdop_kind, sample_kind="normal", tdel_kind="lin", query_kind="lin",
       eta=0.3, m=1.0):
    return Case(nr, nc, nq, eta, m, fdop_kind, sample_kind, tdel_kind, query_kind)


M15 = 1.5
CASES = [
    # smallest accepted call; two-column rows
    _C(1, 2, 1, "halfbin", m=40.0),
    _C(2, 2, 2, "halfbin", "special", query_kind="wide", m=40.0),
    # three columns: the zero-Doppler sample alone, then all three
    _C(2, 3, 2, "sspec", "special", "zero", "knots", eta=0.3, m=5.0),
    _C(3, 3, 255, "sspec", "normal", "lin", "nan", eta=0.3, m=100.0),
    # sizes around one 256-thread pass, in columns and in queries
    _C(4, 255, 255, "jitter", "special", "lin", "knots", m=30.0),
    _C(4, 256, 256, "long_right", "normal", "lin", "wide", m=200.0),
    _C(5, 257, 257, "sspec", "cutmid", "zero", "lin", eta=1e-4, m=1.0),
    _C(6, 257, 256, "positive", "special", "lin", "wide", m=100.0),
    _C(3, 256, 257, "narrow_first", "special", "lin", "knots", m=60.0),
    _C(3, 255, 256, "wide_first", "normal", "lin", "knots", m=60.0),
    _C(3, 1024, 20000, "sspec", "db_zero", "lin", "lin", eta=2e-3, m=2.0),
    _C(3, 16385, 300, "sspec", "special", "lin", "knots", eta=3e-3, m=2.0),
    _C(2, 16385, 1, "jitter", "cutmid", "zero", "lin", m=2000.0),
    _C(4097, 256, 257, "sspec", "cutmid", "lin", "lin", eta=1e-3, m=2.0),
    _C(4097, 3, 2, "sspec", "db_zero", "zero", "nan", eta=1.0, m=3.0),
    # imax on a Doppler sample (s exact, fdop on a 0.25 grid) and one ulp either side
    _C(8, 64, 129, "pow2", "special", "exact", "knots", eta=0.5, m=M15),
    _C(8, 64, 129, "pow2", "normal", "exact", "nan", eta=0.5, m=float(np.nextafter(M15, 2.0))),
    _C(8, 64, 129, "pow2", "special", "exact", "knots", eta=0.5,
       m=float(np.nextafter(M15, 1.0))),
    # no selected sample (hi < lo) next to two-sample rows
    _C(6, 40, 64, "halfbin", "special", "lin", "nan", eta=1.0, m=0.3),
    # NaN queries on one-sample rows, the delay-zero row among them
    _C(5, 41, 70, "sspec", "normal", "zero", "nan", eta=5.0, m=0.35),
    _C(6, 40, 33, "pow2", "special", "zero", "knots", eta=1.0, m=0.4),
]

# (what, rows call (nr, nc, nq) or avg call (nr, nq), words of nothing: SbError before any launch)
LIMITS = [("rows nr < 1", "rows", (0, 4, 4)), ("rows nc < 2", "rows", (1, 1, 4)),
          ("rows nq < 1", "rows", (1, 4, 0)), ("avg nr < 1", "avg", (0, 4)),
          ("avg nq < 1", "avg", (1, 0))]


# --------------------------------------------------------------------------
# reference and the branches it takes
# --------------------------------------------------------------------------
def reference_rows(x):
    """np.interp per row on the float32 samples, with the reference's selection and
    mask expressions (dynspec.py:2093-2127).  A row without a selected sample is all
    masked with NaN power (np.interp would raise; the kernel masks it)."""
    sspec = x["sspec"].astype(np.float64)
    fdop, tdel, fdopnew = x["fdop"], x["tdel"], x["fdopnew"]
    eta, mnf = x["eta"], x["maxnormfac"]
    nr, nq = sspec.shape[0], fdopnew.size
    norm = np.full((nr, nq), np.nan)
    mask = np.ones((nr, nq), bool)
    power = np.full(nr, np.nan)
    terms = [np.zeros(0)] * nr
    for ii in range(nr):
        s = np.sqrt(tdel[ii] / eta)
        sel = abs(fdop) <= mnf * s
        if not sel.any():
            continue
        with np.errstate(invalid="ignore"):
            ifdop = fdop[sel] / s
            r = np.interp(fdopnew, ifdop, sspec[ii, sel])
            m = (np.abs(fdopnew) > np.max(np.abs(ifdop))) | np.isnan(r)
        norm[ii], mask[ii] = r, m
        # np.ma's safe division in normSspec / 10 masks +-inf samples out of the power
        terms[ii] = np.power(10, r[~m & np.isfinite(r)] / 10)
        if terms[ii].size:
            power[ii] = np.mean(terms[ii])
    return norm, mask, power, terms


def reference_avg(norm32, w):
    v = norm32.astype(np.float64)
    ok = ~np.isnan(v)
    with np.errstate(invalid="ignore", divide="ignore"):
        wv = np.where(ok, w[:, None] * np.where(ok, v, 0.0), 0.0)
        den = (w[:, None] * ok).sum(axis=0)
        num = wv.sum(axis=0)
        avg = np.where(den != 0, num / np.where(den != 0, den, 1.0), np.nan)
        bound = (ok.sum(axis=0) + 2) * U52 * (np.abs(wv).sum(axis=0) + np.abs(avg) *
                                              (np.abs(w)[:, None] * ok).sum(axis=0)) / np.abs(den)
    return avg, bound


def row_geometry(x):
    """Per row: s, imax, (lo, hi) of the selection (None when empty)."""
    out = []
    for ii in range(x["sspec"].shape[0]):
        s = np.sqrt(x["tdel"][ii] / x["eta"])
        out.append((s, x["maxnormfac"] * s, _selection(x["fdop"], s, x["maxnormfac"])))
    return out


def branches(x):
    """The branches of interp_one / the mask that the inputs reach (the coverage test)."""
    got = set()
    fdop, fdopnew = x["fdop"], x["fdopnew"]
    nc = fdop.size
    af = np.abs(fdop)
    step = fdop[1] - fdop[0]
    if x["fdop_kind"] == "sspec" and np.log2(abs(step)) % 1 != 0:
        got.add("sspec axis, step not a power of two")
    for ii, (s, imax, (lo, hi)) in enumerate(row_geometry(x)):
        row = x["sspec"][ii].astype(np.float64)
        n = 0 if lo is None else hi - lo + 1
        got.add("selection %s" % ({0: "0", 1: "1", 2: "2", nc: "all"}.get(n, "other")))
        if x["tdel"][ii] == 0:
            got.add("delay-zero row")
        for k in np.flatnonzero(af <= 2 * abs(imax) + abs(step)):
            if imax == af[k]:
                got.add("imax on a sample")
            elif imax == np.nextafter(af[k], np.inf):
                got.add("imax one ulp above a sample")
            elif imax == np.nextafter(af[k], -np.inf):
                got.add("imax one ulp below a sample")
        if n == 0:
            continue
        if lo < 256 <= hi:
            got.add("selection across the 256-thread pass")
        if fdopnew.size > 256:
            got.add("queries past one 256-thread pass")
        nanq = np.isnan(fdopnew)
        if nanq.any():
            got.add("NaN query, %s" % ("one sample" if n == 1 else "longer row"))
        if n == 1:
            continue
        with np.errstate(invalid="ignore"):     # s = 0: one NaN knot
            xp = fdop[lo:hi + 1] / s
        yp = row[lo:hi + 1]
        x0, xl = xp[0], xp[-1]
        amax = max(abs(x0), abs(xl))
        q = fdopnew[~nanq]
        if np.isin(q, xp[1:-1]).any():
            got.add("query on an interior knot")
        if (q == x0).any() and (q == xl).any():
            got.add("queries on both ends of the selection")
        if ((q > xl) & (np.abs(q) <= amax)).any() or ((q < x0) & (np.abs(q) <= amax)).any():
            got.add("unmasked query outside [x0, xl]")
        if abs(xp[-1]) > abs(xp[0]) and ((np.abs(q) > abs(xp[0])) & (np.abs(q) <= amax)).any():
            got.add("mask decided by the high end")
        if np.isnan(yp).any() and (~np.isnan(yp)).any():
            got.add("NaN samples next to valid ones")
        inside = q[(q >= x0) & (q <= xl)]
        j = np.clip(np.searchsorted(xp, inside, side="right") - 1, 0, len(xp) - 1)
        guess = np.clip(np.floor((inside * s - fdop[lo]) / step), 0, len(xp) - 1).astype(int)
        if (guess > j).any():
            got.add("left settle loop")
        if (guess < j).any():
            got.add("right settle loop")
        interp = (j < len(xp) - 1) & (xp[j] != inside)
        jj, xi = j[interp], inside[interp]
        if jj.size:
            yj, yk = yp[jj], yp[jj + 1]
            with np.errstate(invalid="ignore"):
                slope = (yk - yj) / (xp[jj + 1] - xp[jj])
                r1 = slope * (xi - xp[jj]) + yj
                r2 = slope * (xi - xp[jj + 1]) + yk
            f1 = np.isnan(r1)
            if (f1 & ~np.isnan(r2)).any():
                got.add("fallback: second expression")
            if (f1 & np.isnan(r2) & (yj == yk)).any():
                got.add("fallback: equal infinities")
            if (f1 & np.isnan(r2) & np.isinf(yj) & np.isinf(yk) & (yj != yk)).any():
                got.add("fallback: -inf next to +inf")
            if (f1 & (np.isnan(yj) ^ np.isnan(yk))).any():
                got.add("fallback: isolated NaN sample")
    return got


REQUIRED = {
    "selection 0", "selection 1", "selection 2", "selection all",
    "imax on a sample", "imax one ulp above a sample", "imax one ulp below a sample",
    "delay-zero row", "selection across the 256-thread pass",
    "queries past one 256-thread pass", "NaN query, one sample", "NaN query, longer row",
    "query on an interior knot", "queries on both ends of the selection",
    "unmasked query outside [x0, xl]", "mask decided by the high end",
    "NaN samples next to valid ones", "left settle loop", "right settle loop",
    "fallback: second expression", "fallback: equal infinities",
    "fallback: -inf next to +inf", "fallback: isolated NaN sample",
    "sspec axis, step not a power of two",
}


def full_inputs(c):
    x = dict(inputs(c))
    x.update(eta=c.eta, maxnormfac=c.maxnormfac, fdop_kind=c.fdop_kind)
    return x


# --------------------------------------------------------------------------
# device calls
# --------------------------------------------------------------------------
def _dev():
    from scintools_b200 import _device as D, _lib
    D.device()
    return D, _lib


def device_rows(x):
    import torch
    D, L = _dev()
    nr, nc = x["sspec"].shape
    nq = x["fdopnew"].size
    s, fd, td, fn = (D.upload(np.ascontiguousarray(x[k])) for k in ("sspec", "fdop", "tdel",
                                                                    "fdopnew"))
    out = D.empty((nr, nq), torch.float32)
    pw = D.empty((nr,), torch.float64)
    L.check(L.lib.sb_norm_sspec_f32(s.data_ptr(), nr, nc, fd.data_ptr(), td.data_ptr(),
                                    float(x["eta"]), float(x["maxnormfac"]), fn.data_ptr(), nq,
                                    out.data_ptr(), pw.data_ptr(), D.stream_ptr()))
    return out, pw.cpu().numpy()


def device_avg(d_norm, w):
    import torch
    D, L = _dev()
    nr, nq = d_norm.shape
    dw = D.upload(np.ascontiguousarray(w, dtype=np.float64))
    avg = D.empty((nq,), torch.float64)
    L.check(L.lib.sb_norm_sspec_avg_f32(d_norm.data_ptr(), nr, nq, dw.data_ptr(), avg.data_ptr(),
                                        D.stream_ptr()))
    return avg.cpu().numpy()


def check_bounded(family, got, ref, bound):
    fin = np.isfinite(ref)
    assert np.array_equal(got[~fin], ref[~fin], equal_nan=True), \
        "%s: non-finite values differ at %s" % (family, np.flatnonzero(
            ~(np.isclose(got[~fin], ref[~fin], equal_nan=True)))[:8])
    if fin.any():
        err = np.abs(got[fin] - ref[fin])
        ratio = err / np.where(bound[fin] > 0, bound[fin], np.inf)
        ratio[err == 0] = 0.0
        _record(family, ratio.max())
        assert ratio.max() <= 1.0, "%s: %.3g of the bound at %d" % (
            family, ratio.max(), np.flatnonzero(fin)[ratio.argmax()])


def run_case(c):
    x = full_inputs(c)
    norm, mask, power, terms = reference_rows(x)
    d_norm, p = device_rows(x)
    got = d_norm.cpu().numpy()
    assert np.array_equal(np.isnan(got), mask), "mask differs at %s" % (
        np.argwhere(np.isnan(got) != mask)[:8].tolist())
    want = np.where(mask, np.nan, norm).astype(np.float32)
    same = (got.view(np.uint32) == want.view(np.uint32)) | mask
    _record("norm (bits)", (~same).sum())
    assert same.all(), "norm differs at %s: %s vs %s" % (
        np.argwhere(~same)[:4].tolist(), got[~same][:4], want[~same][:4])
    n = np.array([t.size for t in terms])
    bound = (n + 4) * U52 * np.array([t.sum() for t in terms]) / np.maximum(n, 1)
    check_bounded("power", p, power, bound)
    avg, abound = reference_avg(got, x["weights"])
    check_bounded("avg", device_avg(d_norm, x["weights"]), avg, abound)


# --------------------------------------------------------------------------
# the table and the limits (no GPU)
# --------------------------------------------------------------------------
def test_case_table_coverage():
    """Every size of the issue's list and every branch of interp_one and the mask is
    reached by some case, and the table's ids are unique."""
    assert {2, 3, 255, 256, 257, 1024, 16385} <= {c.nc for c in CASES}
    assert {1, 2, 255, 256, 257, 20000} <= {c.nq for c in CASES}
    assert {1, 2, 4097} <= {c.nr for c in CASES}
    got = set()
    for c in CASES:
        got |= branches(full_inputs(c))
    assert sorted(REQUIRED - got) == []
    assert len({case_id(c) for c in CASES}) == len(CASES)
    ok = {(1, 2, 1)}
    assert ok <= {(c.nr, c.nc, c.nq) for c in CASES}


def test_reference_rows_is_numpy_norm_rows():
    """Where every row has a selection, reference_rows is test_arcfit_cpu's
    numpy_norm_rows: samples and mask to the bit, power up to the order of its sum."""
    n = 0
    for c in CASES:
        if c.nr < 2 or c.nr * c.nq > 4e5:
            continue
        x = full_inputs(c)
        if any(lo is None for _, _, (lo, _) in row_geometry(x)):
            continue
        norm, mask, power, _ = reference_rows(x)
        w = x["weights"]
        with np.errstate(all="ignore"):
            n0, p0, _ = numpy_norm_rows(x["sspec"].astype(np.float64), x["fdop"], x["tdel"],
                                        c.eta, c.maxnormfac, x["fdopnew"], lambda p: w)
        n0 = n0.reshape(norm.shape)
        assert np.array_equal(np.isnan(n0), mask), case_id(c)
        assert np.array_equal(n0[~mask], norm[~mask]), case_id(c)
        assert np.allclose(p0, power, rtol=1e-13, atol=0, equal_nan=True), case_id(c)
        n += 1
    assert n >= 8


# --------------------------------------------------------------------------
# GPU
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_norm_sspec_geometry(case):
    run_case(case)


@pytest.mark.gpu
def test_limits_rejected_before_launch():
    """nr < 1, nc < 2, nq < 1 raise SbError before any launch; the smallest accepted
    call (one row, two columns, one query; one row and one query for the average)
    runs and matches the reference."""
    import torch
    D, L = _dev()
    buf = D.zeros((64,), torch.float64)
    p = buf.data_ptr()
    n0 = L.lib.sb_launch_count()
    for what, kind, dims in LIMITS:
        with pytest.raises(L.SbError):
            if kind == "rows":
                nr, nc, nq = dims
                L.check(L.lib.sb_norm_sspec_f32(p, nr, nc, p, p, 1.0, 1.0, p, nq, p, p,
                                                D.stream_ptr()))
            else:
                nr, nq = dims
                L.check(L.lib.sb_norm_sspec_avg_f32(p, nr, nq, p, p, D.stream_ptr()))
    assert L.lib.sb_launch_count() == n0
    run_case(CASES[0])
    assert L.lib.sb_launch_count() == n0 + 2


# --------------------------------------------------------------------------
# the reference's norm_sspec / fit_arc on the arcfit_*.npz fixtures
# --------------------------------------------------------------------------
FIXTURES = ["arcfit_61x103.npz", "arcfit_zeros_48x90.npz"]


def fixture_calls():
    out = []
    for fn in FIXTURES:
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", fn)
        with np.load(path) as g:
            out += [(fn, k[:-len("_kind")]) for k in sorted(g.files) if k.endswith("_kind")]
    return out


CALLS = fixture_calls()


def fixture_dynspec(g, name):
    """The port's Dynspec on the fixture's float32-valued spectra, with the centre
    frequency held as the reference held it."""
    ds = _bare_dynspec(g)
    ds.sspec = g["sspec"].astype(np.float64)
    ds.lamsspec = g["lamsspec"].astype(np.float64)
    ds.tdel, ds.beta, ds.fdop = g["tdel"].copy(), g["beta"].copy(), g["fdop"].copy()
    ds.freq = np.float64(g["freq"]) if name.endswith("_f64") else float(g["freq"])
    return ds


def run_fixture_call(g, name):
    """-> (Dynspec, exception type name or "")"""
    ds = fixture_dynspec(g, name)
    kind, kw = str(g[name + "_kind"]), json.loads(str(g[name + "_kwargs"]))
    try:
        with np.errstate(all="ignore"):
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                getattr(ds, kind)(**kw)
    except Exception as e:          # noqa: BLE001 -- the type is what is compared
        return ds, type(e).__name__
    return ds, ""


def _eta_keys(g, name):
    kw = json.loads(str(g[name + "_kwargs"]))
    pre = "betaeta" if kw.get("lamsteps") else "eta"
    return [(pre + suf, "_eta" + suf) for suf in (("_left", "_right") if kw.get("asymm")
                                                  else ("",))], pre


def test_fixture_inventory(golden_dir):
    """The fixtures hold what they are for: both lamsteps, startbin 0, cutmid 0 and wide,
    weighted=False, powerspec_cut (also keeping a single row, which the reference rejects),
    numsteps, asymm, -inf bins, and reference raises."""
    kws, raises = [], set()
    for fn, name in CALLS:
        with np.load(os.path.join(golden_dir, fn)) as g:
            kw = json.loads(str(g[name + "_kwargs"]))
            kws.append((str(g[name + "_kind"]), kw))
            raises.add(str(g[name + "_raises"]))
            if kw.get("powerspec_cut") and str(g[name + "_raises"]):
                raises.add("powerspec_cut " + str(g[name + "_raises"]))
            if fn.startswith("arcfit_zeros"):
                assert np.isneginf(g["sspec"]).any() and np.isneginf(g["lamsspec"]).any()
            assert g["sspec"].dtype == g["lamsspec"].dtype == np.float32
    for kind in ("norm_sspec", "fit_arc"):
        ks = [k for t, k in kws if t == kind]
        assert {k["lamsteps"] for k in ks} == {True, False}
        assert any(k.get("startbin", 1 if kind == "norm_sspec" else 3) == 0 for k in ks)
        assert any(k.get("cutmid", 0 if kind == "norm_sspec" else 3) == 0 for k in ks)
        assert any(k.get("cutmid", 0) >= 15 for k in ks)
        assert any("numsteps" in k for k in ks)
    assert any(k.get("weighted") is False for t, k in kws if t == "norm_sspec")
    assert any(k.get("powerspec_cut") for t, k in kws)
    assert any(k.get("asymm") for t, k in kws)
    assert {"", "ValueError", "TypeError", "powerspec_cut ValueError"} <= raises


@pytest.mark.parametrize("fn,name", CALLS, ids=["%s-%s" % (f[:-4], n) for f, n in CALLS])
def test_fixture_host_glue(fn, name, golden_dir, monkeypatch):
    """The host glue with the numpy restatement of the resampling (no GPU) reproduces
    each fixture call: the same exception, or the same numbers."""
    from scintools_b200 import arcfit
    from oracle import dynspec_oracle as DO
    monkeypatch.setattr(arcfit, "_norm_rows", numpy_norm_rows)
    with np.load(os.path.join(golden_dir, fn)) as g:
        ds, raised = run_fixture_call(g, name)
        assert raised == str(g[name + "_raises"])
        if raised:
            return
        kw = json.loads(str(g[name + "_kwargs"]))
        if str(g[name + "_kind"]) == "norm_sspec":
            got = np.ma.filled(ds.normsspec, np.nan)
            assert np.array_equal(np.ma.getmaskarray(ds.normsspec), g[name + "_mask"])
            assert np.array_equal(got.astype(np.float32), g[name + "_normsspec"], equal_nan=True)
            assert np.allclose(np.ma.filled(ds.normsspecavg, np.nan), g[name + "_normsspecavg"],
                               rtol=1e-12, atol=0, equal_nan=True)
            assert np.allclose(np.ma.filled(ds.powerspectrum, np.nan),
                               g[name + "_powerspectrum"], rtol=1e-12, equal_nan=True)
            if not kw["lamsteps"] and not kw.get("powerspec_cut"):
                with np.errstate(all="ignore"):
                    norm, avg, fdopnew, td, power = DO.norm_sspec(
                        g["sspec"], g["fdop"], g["tdel"], kw["eta"], float(g["freq"]),
                        startbin=kw["startbin"], cutmid=kw["cutmid"],
                        maxnormfac=kw.get("maxnormfac", 5), numsteps=kw.get("numsteps"),
                        weighted=kw.get("weighted", True))
                assert np.array_equal(np.ma.getmaskarray(norm), g[name + "_mask"])
                assert np.allclose(np.ma.filled(avg, np.nan), g[name + "_normsspecavg"],
                                   rtol=1e-12, equal_nan=True)
                assert np.array_equal(fdopnew, g[name + "_fdop"])
            return
        keys, pre = _eta_keys(g, name)
        for attr, key in keys:
            for q in ("", "err", "err2"):
                a = attr.replace(pre, pre + q) if q else attr
                assert np.allclose(getattr(ds, a), float(g[name + key.replace("_eta", "_eta" + q)]),
                                   rtol=1e-9, equal_nan=True), a
        assert np.allclose(ds.noise, float(g[name + "_noise"]), rtol=1e-12, equal_nan=True)
        assert ds.eta_array.size == int(g[name + "_eta_array_n"])
        assert np.allclose(ds.eta_array[[0, -1]], g[name + "_eta_array_ends"], rtol=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("fn,name", CALLS, ids=["%s-%s" % (f[:-4], n) for f, n in CALLS])
def test_fixture_device(fn, name, golden_dir, monkeypatch):
    """The device reproduces each fixture call: the same exception; masks bit for bit,
    samples as np.float32 of the reference's, power and scrunched profile within the
    module's bounds; fit_arc's curvature as test_fit_arc_end_to_end holds it."""
    from scintools_b200 import arcfit
    _dev()
    rec = {}

    def recording(sspec, fdop, tdel, eta, mnf, fdopnew, weights_fn, want_2d=True):
        def wf(p):
            w = weights_fn(p)           # weights, or (weights, rows the average reads)
            w, rows = w if isinstance(w, tuple) else (w, np.ones(len(p), bool))
            rec["w"], rec["rows"] = np.asarray(w, dtype=np.float64), np.asarray(rows, bool)
            return (rec["w"], rec["rows"])
        out = arcfit.norm_rows_device(sspec, fdop, tdel, eta, mnf, fdopnew, wf, want_2d)
        rec["norm"] = out[0]
        return out

    monkeypatch.setattr(arcfit, "_norm_rows", recording)
    with np.load(os.path.join(golden_dir, fn)) as g:
        ds, raised = run_fixture_call(g, name)
        assert raised == str(g[name + "_raises"])
        if raised:
            return
        if str(g[name + "_kind"]) == "norm_sspec":
            mask = g[name + "_mask"]
            assert np.array_equal(np.ma.getmaskarray(ds.normsspec), mask)
            got = np.ma.filled(ds.normsspec, np.nan).astype(np.float32)
            want = g[name + "_normsspec"]
            same = (got.view(np.uint32) == want.view(np.uint32)) | mask
            _record("fixture norm (bits)", (~same).sum())
            assert same.all(), np.argwhere(~same)[:4].tolist()
            # power: the fixture holds the reference's means of 10^(r/10) over the unmasked
            # samples; its terms are recomputed from the same float64 samples
            ref_p = g[name + "_powerspectrum"]
            nrm = rec["norm"]
            fin = np.isfinite(nrm)
            t = np.where(fin, 10.0 ** (np.where(fin, nrm, 0.0) / 10), 0.0)
            n = fin.sum(axis=1)
            # the samples the device summed are float64; nrm is their float32 rounding,
            # which moves each term by up to ln(10)/10 |r| 2^-24 of itself
            tb = t * (1 + np.log(10) / 10 * np.abs(np.where(fin, nrm, 0.0)) * U24)
            bound = (n + 4) * U52 * tb.sum(axis=1) / np.maximum(n, 1)
            check_bounded("fixture power", np.ma.filled(ds.powerspectrum, np.nan), ref_p, bound)
            # scrunched profile over the rows it reads: the reference averages float64
            # samples, the device their float32 rounding
            w, nrm = rec["w"][rec["rows"]], nrm[rec["rows"]]
            ok = ~np.isnan(nrm)
            avg, abound = reference_avg(nrm.astype(np.float32), w)
            v = np.where(ok, np.abs(nrm), 0.0)
            with np.errstate(invalid="ignore", divide="ignore"):
                den = np.abs((w[:, None] * ok).sum(axis=0))
                abound = abound + U24 * (np.abs(w)[:, None] * v).sum(axis=0) / den
            ref_a = g[name + "_normsspecavg"]
            check_bounded("fixture avg", np.ma.filled(ds.normsspecavg, np.nan), ref_a,
                          np.where(np.isfinite(abound), abound, 0.0))
            return
        keys, pre = _eta_keys(g, name)
        for attr, key in keys:
            e0, got = float(g[name + key]), float(getattr(ds, attr))
            if np.isnan(e0):
                assert np.isnan(got), attr
                continue
            err2 = float(g[name + key.replace("_eta", "_etaerr2")])
            assert got == pytest.approx(e0, rel=2e-3), attr
            assert abs(got - e0) < 0.05 * err2, attr
            e1 = float(g[name + key.replace("_eta", "_etaerr")])
            assert float(getattr(ds, attr.replace(pre, pre + "err"))) == pytest.approx(
                e1, rel=0.05), attr
