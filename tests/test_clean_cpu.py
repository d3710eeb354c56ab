"""CPU: the psrflux loader, remove_short_subs, info, crop_dyn and __add__ against the
unmodified reference's attributes (tests/golden/clean_golden.npz, made by
oracle/make_golden_clean.py), with exact equality; trim_edges's host walk, crop and
bookkeeping with its zero counts restated in numpy; and every error raised without touching
the device."""
import os

import numpy as np
import pytest

from scintools_b200 import _device
from scintools_b200 import dynspec as DS
from scintools_b200.dynspec import BasicDyn, Dynspec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Z = np.load(os.path.join(ROOT, "tests", "golden", "clean_golden.npz"))
ATTRS = ("dyn", "times", "freqs", "nchan", "nsub", "bw", "df", "freq", "dt", "tobs", "mjd",
         "name", "header")


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """The fixture's psrflux files, written out: name -> path"""
    d = tmp_path_factory.mktemp("psrflux")
    for k in Z.files:
        if k.startswith("file/"):
            (d / k[5:]).write_text(str(Z[k]))
    return lambda name: str(d / name)


def cases(prefix):
    return sorted({k.split("/")[0] for k in Z.files if k.startswith(prefix)})


def same_attrs(ds, case):
    for a in ATTRS:
        key = case + "/" + a
        if key not in Z.files:
            continue
        ref = Z[key]
        got = np.asarray(getattr(ds, a))
        if ref.dtype.kind in "US":
            assert got.tolist() == ref.tolist(), (case, a)
        else:
            assert got.shape == ref.shape, (case, a, got.shape, ref.shape)
            assert np.array_equal(got, ref, equal_nan=True), (case, a)


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(_device, "device", lambda: pytest.fail("device touched"))


def numpy_counts(dyn):
    """_zero_counts restated in numpy"""
    z = (dyn == 0) | np.isnan(dyn)
    return z.sum(axis=1), lambda r0, r1: z[r0:r1].sum(axis=0)


def crafted(case):
    a = Z[case + "/input"].copy()
    nf, nt = a.shape
    freqs = 1400.0 + 0.25 * np.arange(nf)
    b = BasicDyn(a, name="crafted", header=["crafted"], times=8.0 * np.arange(nt), freqs=freqs,
                 nchan=nf, nsub=nt, bw=0.25 * nf, df=0.25, freq=float(freqs.mean()),
                 tobs=8.0 * nt, dt=8.0, mjd=58000.5)
    return Dynspec(dyn=b, verbose=False)


LOADS = {
    "load_j0437": dict(filename="clean_j0437.dynspec"),
    "load_j0437_keep": dict(filename="clean_j0437.dynspec", remove_short_subs=False),
    "load_ascending": dict(filename="clean_ascending.dynspec"),
    "load_short": dict(filename="clean_short.dynspec"),
    "load_short_thresh": dict(filename="clean_short.dynspec", subint_thresh=50.0),
    "load_short_mjd": dict(filename="clean_short.dynspec", mjd=57000.75),
    "load_nomjd": dict(filename="clean_nomjd.dynspec"),
    "load_nomjd_mjd": dict(filename="clean_nomjd.dynspec", mjd=57000.75),
    "load_badcount": dict(filename="clean_badcount.dynspec"),
}


@pytest.mark.parametrize("case", sorted(LOADS))
def test_load_file(case, files, no_device):
    kw = dict(LOADS[case])
    kw["filename"] = files(kw["filename"])
    err = str(Z[case + "/error"])
    if err:
        with pytest.raises({"AttributeError": AttributeError, "ValueError": ValueError}[err]):
            Dynspec(verbose=False, **kw)
        return
    ds = Dynspec(verbose=False, **kw)
    same_attrs(ds, case)
    assert ds.filename == kw["filename"] and ds.lamsteps is False


def test_load_j0437_shape(files):
    """The excerpt's descending band is flipped and its short first sub-integration goes."""
    ds = Dynspec(filename=files("clean_j0437.dynspec"), verbose=False)
    assert ds.dyn.shape == (512, 11) and np.all(np.diff(ds.freqs) > 0)
    assert np.count_nonzero(~ds.dyn.any(axis=1)) >= 114


def test_verbose_load_prints_the_reference_summary(capsys, files, no_device):
    Dynspec(filename=files("clean_ascending.dynspec"))
    got = capsys.readouterr().out.splitlines()
    ref = str(Z["load_verbose/stdout"]).splitlines()
    strip = lambda lines: [s for s in lines if not s.startswith("...LOADED in")]  # noqa: E731
    assert strip(got)[1:] == strip(ref)[1:]      # the first names the file's full path
    assert len(got) == len(ref)


@pytest.mark.parametrize("case", cases("trim_"))
def test_trim_edges_host(case, files, monkeypatch):
    monkeypatch.setattr(DS, "_zero_counts", numpy_counts)
    monkeypatch.setattr(_device, "device", lambda: pytest.fail("device touched"))
    if case == "trim_j0437":
        ds = Dynspec(filename=files("clean_j0437.dynspec"), verbose=False)
        frac = 0.5
    else:
        ds = crafted(case)
        frac = float(Z[case + "/frac"])
    err = str(Z[case + "/error"])
    if err:
        before = ds.dyn.copy()
        with pytest.raises(IndexError):
            ds.trim_edges(bandwagon_frac=frac)
        assert np.array_equal(ds.dyn, before, equal_nan=True)   # nothing changed
        return
    ds.trim_edges(bandwagon_frac=frac)
    same_attrs(ds, case)


@pytest.mark.parametrize("shape", [(0, 5), (4, 0)])
def test_trim_edges_empty_before_device(shape, no_device):
    ds = Dynspec(dyn=BasicDyn(np.zeros(shape), times=[0.0, 8.0], freqs=[1.0, 2.0, 3.0]),
                 verbose=False)
    with pytest.raises(IndexError):
        ds.trim_edges()


@pytest.mark.parametrize("case", cases("crop_"))
def test_crop_dyn(case, files, no_device):
    kw = {"crop_band": dict(fmin=1530.0, fmax=1560.0),
          "crop_time": dict(tmin=1.0, tmax=4.0),
          "crop_tobs": dict(tmin=0.5, tmax=100.0),
          "crop_both": dict(fmin=1500.0, fmax=1600.0, tmin=2.0, tmax=5.5)}[case]
    ds = Dynspec(filename=files("clean_j0437.dynspec"), verbose=False)
    ds.crop_dyn(**kw)
    same_attrs(ds, case)


@pytest.mark.parametrize("case", cases("add_"))
def test_add(case, capsys, files, no_device):
    fn = "clean_ascending.dynspec" if case == "add_band" else "clean_j0437.dynspec"
    a = Dynspec(filename=files(fn), verbose=False)
    b = Dynspec(filename=files(fn), verbose=False, mjd=float(Z[case + "/mjd_b"]))
    capsys.readouterr()
    res = a + b
    assert capsys.readouterr().out == str(Z[case + "/stdout"])
    same_attrs(res, case)
    a += b
    same_attrs(a, case)

