"""Generate the fixtures of the psrflux loader and the cleaning steps: the UNMODIFIED
reference's Dynspec (via oracle/ref_loader.py) after load_file, trim_edges, zap, crop_dyn
and __add__.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python oracle/make_golden_clean.py

Writes tests/golden/clean_golden.npz.  ``file/<name>`` holds the text of each psrflux file
the cases load (the tests write it to a temporary directory):
  clean_j0437.dynspec      the first 12 sub-integrations of one J0437-4715 observation, all
                           512 channels (descending frequencies, a short first
                           sub-integration, two zero bands at the edges)
  clean_ascending.dynspec  ascending frequencies, constant sub-integration time
  clean_short.dynspec      three short leading sub-integrations, two MJD0 lines
  clean_nomjd.dynspec      no MJD0 line
  clean_badcount.dynspec   one sample missing
and per case ``<case>/<attr>`` (dyn, times, freqs, nchan, nsub, bw, df, freq, dt, tobs, mjd,
name, header), ``<case>/input`` for the crafted arrays, ``<case>/error`` (the exception type
name) and ``<case>/stdout`` where the call prints.
"""
import contextlib
import io
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
FILES = ("clean_j0437.dynspec", "clean_ascending.dynspec", "clean_short.dynspec",
         "clean_nomjd.dynspec", "clean_badcount.dynspec")
DIR = tempfile.mkdtemp()

from oracle import ref_loader  # noqa: E402

J0437 = os.path.join(ref_loader.REFERENCE_ROOT, "scintools", "examples", "data", "J0437-4715",
                     "p111220_074112.rf.pcm.dynspec")
ATTRS = ("dyn", "times", "freqs", "nchan", "nsub", "bw", "df", "freq", "dt", "tobs", "mjd",
         "name", "header")


def excerpt(nsub=12):
    out = []
    with open(J0437) as f:
        for line in f:
            if not line.startswith("#") and int(line.split()[0]) >= nsub:
                break
            out.append(line)
    with open(os.path.join(DIR, "clean_j0437.dynspec"), "w") as f:
        f.writelines(out)


def write_psrflux(name, tmin, freqs, dyn, mjd_lines, drop_last=False):
    lines = ["# Dynamic spectrum computed by psrflux\n"]
    lines += ["# MJD0: %s\n" % m for m in mjd_lines[:1]]
    lines += ["# Flux units: ReferenceFluxDensity\n"]
    lines += ["# MJD0: %s\n" % m for m in mjd_lines[1:]]
    lines += ["# isub ichan time(min) freq(MHz) flux flux_err\n"]
    for i, t in enumerate(tmin):
        for j, fr in enumerate(freqs):
            lines.append("%4d %4d %10.4f %12.6f %+e %+e\n" % (i, j, t, fr, dyn[j, i], 0.0))
    if drop_last:
        lines = lines[:-1]
    with open(os.path.join(DIR, name), "w") as f:
        f.writelines(lines)


def crafted_files():
    rng = np.random.default_rng(11)
    nf, nt = 24, 16
    freqs = 1300.0 + 0.5 * np.arange(nf)
    dyn = np.round(rng.exponential(1.0, (nf, nt)), 4)
    dyn[:2] = 0.0
    write_psrflux("clean_ascending.dynspec", 0.5 * np.arange(nt), freqs, dyn, ["55500.125"])
    steps = [0.0833, 0.0833, 0.0833] + [0.5, 0.5017, 0.4983, 0.5033, 0.4967] * 3
    tmin = np.round(np.concatenate([[0.0], np.cumsum(steps)]), 4)[:nt]
    write_psrflux("clean_short.dynspec", tmin, freqs[::-1], dyn, ["55000.25", "56000.5"])
    write_psrflux("clean_nomjd.dynspec", 0.5 * np.arange(nt), freqs, dyn, [])
    write_psrflux("clean_badcount.dynspec", 0.5 * np.arange(nt), freqs, dyn, ["55500.125"],
                  drop_last=True)


def record(out, case, ds, err=None, stdout=None, inp=None):
    if err is not None:
        out[case + "/error"] = np.array(type(err).__name__)
    else:
        out[case + "/error"] = np.array("")
        for a in ATTRS:
            if hasattr(ds, a):
                out[case + "/" + a] = np.asarray(getattr(ds, a))
    if stdout is not None:
        out[case + "/stdout"] = np.array(stdout)
    if inp is not None:
        out[case + "/input"] = np.asarray(inp)


def run(fn):
    buf = io.StringIO()
    err = None
    res = None
    with contextlib.redirect_stdout(buf):
        try:
            res = fn()
        except Exception as e:   # the reference's exception is the expected result
            err = e
    return res, err, buf.getvalue()


def crafted_arrays():
    """name -> (dyn, bandwagon_frac) for trim_edges"""
    rng = np.random.default_rng(3)
    out = {}
    a = rng.exponential(1.0, (20, 30))
    a[:3] = 0.0
    a[-2:] = np.nan
    a[5, 4] = np.nan
    a[10, :] = 0.0                  # an interior zero row stays
    a[:, 0] = 0.0
    a[:, -1] = np.nan
    out["nan"] = (a, 0.5)
    a = rng.exponential(1.0, (16, 20))
    a[0, :10] = 0.0                 # exactly frac * nc zeros: stays
    a[-1, :11] = 0.0                # one more: goes, and the next row is checked
    a[-2, :10] = np.nan
    out["exact"] = (a, 0.5)
    a = rng.exponential(1.0, (12, 14))
    a[0, 3] = 0.0
    a[1, 5] = np.nan
    a[-1, 0] = 0.0
    a[4, 0] = 0.0
    out["frac0"] = (a, 0.0)
    a = rng.exponential(1.0, (12, 14))
    a[0, :13] = 0.0
    a[1, :] = 0.0
    a[2, :] = 0.0
    a[:, -1] = 0.0
    out["frac1"] = (a, 1.0)
    # columns: 30 rows, 10 trimmed; zeros over the 20 kept rows of column 0 are 12, more
    # than half of 20 but not of the original 30, so it stays (the reference's quirk);
    # column 1 has 16 > 15 and goes
    a = rng.exponential(1.0, (30, 12))
    a[:6] = 0.0
    a[-4:] = 0.0
    a[6:18, -1] = 0.0
    a[6:22, 0] = 0.0
    out["colquirk"] = (a, 0.5)
    a = rng.exponential(1.0, (10, 8))
    a[:, :] = 0.0
    a[4, 3] = np.nan
    out["allrows"] = (a, 0.5)
    a = rng.exponential(1.0, (10, 8))
    a[:, ::2] = 0.0
    a[::2, 1::2] = 0.0
    out["allcols"] = (a, 0.3)
    a = rng.exponential(1.0, (9, 11))
    out["untouched"] = (a, 0.5)
    return out


def zap_arrays():
    rng = np.random.default_rng(9)
    out = {}
    out["odd"] = rng.exponential(1.0, (9, 13))
    out["even"] = rng.exponential(1.0, (10, 13))
    a = rng.normal(0.0, 1.0, (12, 20))
    a[0, :3] = np.inf
    a[5, 5] = -np.inf
    a[3, 3] = 60.0
    a[rng.random(a.shape) < 0.1] = np.nan
    out["inf"] = a
    out["allnan"] = np.full((4, 6), np.nan)
    a = np.ones((7, 9))
    a[::3, ::2] = 4.0
    out["mdev0"] = a
    return out


def basic(R, dyn, name="crafted"):
    nf, nt = dyn.shape
    freqs = 1400.0 + 0.25 * np.arange(nf)
    times = 8.0 * np.arange(nt)
    b = R.dynspec.BasicDyn(dyn, name=name, header=["crafted"], times=times, freqs=freqs,
                           nchan=nf, nsub=nt, bw=0.25 * nf, df=0.25, freq=float(freqs.mean()),
                           tobs=8.0 * nt, dt=8.0, mjd=58000.5)
    return R.dynspec.Dynspec(dyn=b, verbose=False, process=False)


def main():
    R = ref_loader.load()
    Dyn = R.dynspec.Dynspec
    excerpt()
    crafted_files()
    g = lambda n: os.path.join(DIR, n)  # noqa: E731
    out = {}
    # loading
    loads = {
        "load_j0437": dict(filename=g("clean_j0437.dynspec")),
        "load_j0437_keep": dict(filename=g("clean_j0437.dynspec"), remove_short_subs=False),
        "load_ascending": dict(filename=g("clean_ascending.dynspec")),
        "load_short": dict(filename=g("clean_short.dynspec")),
        "load_short_thresh": dict(filename=g("clean_short.dynspec"), subint_thresh=50.0),
        "load_short_mjd": dict(filename=g("clean_short.dynspec"), mjd=57000.75),
        "load_nomjd": dict(filename=g("clean_nomjd.dynspec")),
        "load_nomjd_mjd": dict(filename=g("clean_nomjd.dynspec"), mjd=57000.75),
        "load_badcount": dict(filename=g("clean_badcount.dynspec")),
    }
    for case, kw in loads.items():
        ds, err, _ = run(lambda: Dyn(verbose=False, process=False, **kw))
        record(out, case, ds, err)
    # the printed summary of a verbose load (the timing line differs between runs)
    _, _, text = run(lambda: Dyn(filename=g("clean_ascending.dynspec"), verbose=True))
    out["load_verbose/stdout"] = np.array(text)
    # trim_edges
    ds, err, _ = run(lambda: Dyn(filename=g("clean_j0437.dynspec"), verbose=False))
    j = ds
    _, err, _ = run(lambda: j.trim_edges())
    record(out, "trim_j0437", j, err)
    for name, (a, frac) in crafted_arrays().items():
        ds = basic(R, a.copy())
        _, err, _ = run(lambda: ds.trim_edges(bandwagon_frac=frac))
        record(out, "trim_" + name, ds, err, inp=a)
        out["trim_" + name + "/frac"] = np.array(frac)
    # zap: the trimmed J0437 excerpt, and crafted arrays
    for sigma in (7, 3.0, 1.5):
        ds, _, _ = run(lambda: Dyn(filename=g("clean_j0437.dynspec"), verbose=False))
        ds.trim_edges()
        _, err, _ = run(lambda: ds.zap(sigma=sigma))
        record(out, "zap_j0437_s%g" % sigma, ds, err)
        out["zap_j0437_s%g/sigma" % sigma] = np.array(float(sigma))
    for name, a in zap_arrays().items():
        for sigma in (7, 2.0, 0.5):
            ds = basic(R, a.copy())
            _, err, _ = run(lambda: ds.zap(sigma=sigma))
            case = "zap_%s_s%g" % (name, sigma)
            record(out, case, ds, err, inp=a)
            out[case + "/sigma"] = np.array(float(sigma))
    # crop_dyn
    crops = {"crop_band": dict(fmin=1530.0, fmax=1560.0),
             "crop_time": dict(tmin=1.0, tmax=4.0),
             "crop_tobs": dict(tmin=0.5, tmax=100.0),
             "crop_both": dict(fmin=1500.0, fmax=1600.0, tmin=2.0, tmax=5.5)}
    for case, kw in crops.items():
        ds, _, _ = run(lambda: Dyn(filename=g("clean_j0437.dynspec"), verbose=False))
        _, err, _ = run(lambda: ds.crop_dyn(**kw))
        record(out, case, ds, err)
    # __add__: the excerpt after itself with a 95.3 s gap, with no gap, and a different band
    a, _, _ = run(lambda: Dyn(filename=g("clean_j0437.dynspec"), verbose=False))
    for case, extra in (("add_gap", 95.3), ("add_nogap", 0.0)):
        m = a.mjd + (a.tobs + extra) / 86400
        b, _, _ = run(lambda: Dyn(filename=g("clean_j0437.dynspec"), verbose=False, mjd=m))
        res, err, text = run(lambda: a + b)
        record(out, case, res, err, stdout=text)
        out[case + "/mjd_b"] = np.array(m)
    c, _, _ = run(lambda: Dyn(filename=g("clean_ascending.dynspec"), verbose=False))
    d, _, _ = run(lambda: Dyn(filename=g("clean_ascending.dynspec"), verbose=False,
                               mjd=c.mjd + 0.01))
    res, err, text = run(lambda: c + d)
    record(out, "add_band", res, err, stdout=text)
    out["add_band/mjd_b"] = np.array(c.mjd + 0.01)
    for name in FILES:
        with open(g(name)) as f:
            out["file/" + name] = np.array(f.read())
    np.savez_compressed(os.path.join(GOLD, "clean_golden.npz"), **out)
    print("wrote %d keys" % len(out))


if __name__ == "__main__":
    main()
