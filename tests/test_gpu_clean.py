"""GPU tests of trim_edges and zap (csrc/clean.cu): every fixture of the unmodified
reference (tests/golden/clean_golden.npz) reproduced exactly, NaN included; a seeded
4096 x 8192 spectrum with zero bands, NaN and outliers against a numpy restatement, bit for
bit; a caller stream; and the tutorial's single-file chain from the J0437-4715 excerpt."""
import numpy as np
import pytest
from test_clean_cpu import Z, cases, crafted, files, same_attrs  # noqa: F401  (files: fixture)

pytestmark = pytest.mark.gpu


def j0437(files):
    from scintools_b200.dynspec import Dynspec
    return Dynspec(filename=files("clean_j0437.dynspec"), verbose=False)


def np_trim(dyn, frac):
    """The reference's trim_edges walk restated on whole counts: (r0, r1, c0, c1)."""
    z = (dyn == 0) | np.isnan(dyn)
    nr, nc = dyn.shape
    rz = z.sum(axis=1)
    keep = ~((rz > frac * nc) | (rz == nc))
    r = np.flatnonzero(keep)
    r0, r1 = r[0], r[-1] + 1
    cz = z[r0:r1].sum(axis=0)
    keep = ~((cz > frac * nr) | (cz == r1 - r0))
    c = np.flatnonzero(keep)
    return r0, r1, c[0], c[-1] + 1


def np_zap(x, sigma):
    x = x.copy()
    with np.errstate(all="ignore"):
        med = np.median(x[~np.isnan(x)])
        d = np.abs(x - med)
        mdev = np.median(d[~np.isnan(d)])
        x[d / mdev > sigma] = np.nan
    return x, med, mdev


@pytest.mark.parametrize("case", cases("trim_"))
def test_trim_edges_fixtures(case, files):
    if case == "trim_j0437":
        ds, frac = j0437(files), 0.5
    else:
        ds, frac = crafted(case), float(Z[case + "/frac"])
    if str(Z[case + "/error"]):
        before = ds.dyn.copy()
        with pytest.raises(IndexError):
            ds.trim_edges(bandwagon_frac=frac)
        assert np.array_equal(ds.dyn, before, equal_nan=True)
        return
    ds.trim_edges(bandwagon_frac=frac)
    same_attrs(ds, case)


@pytest.mark.parametrize("case", cases("zap_"))
def test_zap_fixtures(case, files):
    sigma = float(Z[case + "/sigma"])
    if case.startswith("zap_j0437"):
        ds = j0437(files)
        ds.trim_edges()
    else:
        ds = crafted(case)
    ds.zap(sigma=sigma)
    same_attrs(ds, case)


def _big():
    rng = np.random.default_rng(2024)
    nf, nt = 4096, 8192
    dyn = rng.exponential(1.0, (nf, nt))
    dyn[:300] = 0.0                          # zero bands at both band edges
    dyn[-170:] = 0.0
    dyn[:, :5] = np.nan
    dyn[1000:1003] = 0.0                     # interior zero rows stay
    dyn[rng.random((nf, nt)) < 0.01] = np.nan
    dyn[rng.random((nf, nt)) < 0.2] = 0.0
    hot = rng.random((nf, nt)) < 1e-3
    dyn[hot] *= 100.0
    return dyn


def test_fullsize_trim_and_zap_match_numpy():
    from scintools_b200.dynspec import BasicDyn, Dynspec
    dyn = _big()
    nf, nt = dyn.shape
    r0, r1, c0, c1 = np_trim(dyn, 0.5)
    ref = dyn[r0:r1, c0:c1].copy()
    ref[np.isnan(ref)] = 0
    ds = Dynspec(dyn=BasicDyn(dyn.copy(), times=10.0 * np.arange(nt),
                              freqs=1000.0 + 0.1 * np.arange(nf)), verbose=False)
    ds.trim_edges()
    assert (r0, r1, c0, c1) == (300, nf - 170, 5, nt)
    assert np.array_equal(ds.dyn, ref)
    assert np.array_equal(ds.freqs, 1000.0 + 0.1 * np.arange(nf)[r0:r1])
    # zap of the raw spectrum (NaN kept) and of the trimmed one
    for x in (dyn, ds.dyn):
        for sigma in (7, 3.0):
            want, med, mdev = np_zap(x, sigma)
            d2 = Dynspec(dyn=BasicDyn(x.copy(), times=10.0 * np.arange(x.shape[1]),
                                      freqs=1000.0 + 0.1 * np.arange(x.shape[0])),
                         verbose=False)
            d2.zap(sigma=sigma)
            assert np.array_equal(d2.dyn, want, equal_nan=True)
            assert _stats(x, sigma) == (med, mdev)


def _stats(x, sigma, stream=None):
    import torch
    from scintools_b200 import _device as D
    from scintools_b200 import _lib
    d = D.upload(np.ascontiguousarray(x, dtype=np.float64))
    st = D.empty((2,), torch.float64)
    ptr = D.stream_ptr() if stream is None else stream.cuda_stream
    _lib.check(_lib.lib.sb_zap_f64(d.data_ptr(), d.numel(), float(sigma), st.data_ptr(), ptr))
    if stream is not None:
        stream.synchronize()
    s = D.download(st)
    return float(s[0]), float(s[1])


def test_zap_stats_edge_cases():
    for x in (np.array([3.0]), np.array([1.0, 4.0]), np.full(7, np.nan), np.array([np.inf] * 5 +
              [1.0, 2.0]), np.array([-np.inf, np.inf]), np.ones(1001)):
        _, med, mdev = np_zap(x, 7.0)
        got = _stats(x, 7.0)
        assert (got[0] == med or (np.isnan(got[0]) and np.isnan(med))) and \
            (got[1] == mdev or (np.isnan(got[1]) and np.isnan(mdev))), (x, got, med, mdev)


def test_caller_stream():
    import torch
    from scintools_b200 import _device as D
    from scintools_b200 import _lib
    D.device()
    rng = np.random.default_rng(8)
    x = rng.exponential(1.0, (512, 1024))
    x[:20] = 0.0
    x[rng.random(x.shape) < 0.05] = np.nan
    want, med, mdev = np_zap(x, 4.0)
    s = torch.cuda.Stream()
    assert _stats(x, 4.0, s) == (med, mdev)
    with torch.cuda.stream(s):
        d = D.upload(x)
        rows = D.empty((512,), torch.int32)
        cols = D.empty((1024,), torch.int32)
        _lib.check(_lib.lib.sb_dyn_zero_counts_f64(d.data_ptr(), 512, 1024, 0, 512,
                                                   rows.data_ptr(), cols.data_ptr(),
                                                   s.cuda_stream))
        st = D.empty((2,), torch.float64)
        _lib.check(_lib.lib.sb_zap_f64(d.data_ptr(), d.numel(), 4.0, st.data_ptr(),
                                       s.cuda_stream))
    s.synchronize()
    z = (x == 0) | np.isnan(x)
    assert np.array_equal(D.download(rows), z.sum(axis=1))
    assert np.array_equal(D.download(cols), z.sum(axis=0))
    assert np.array_equal(D.download(d), want, equal_nan=True)


def test_tutorial_chain_from_j0437(files):
    """arc_modelling's single-file steps: load, trim_edges, refill, correct_dyn,
    calc_sspec, scale_dyn, fit_arc."""
    ds = j0437(files)
    ds.trim_edges()
    ds.refill()
    ds.correct_dyn()
    ds.calc_sspec()
    ds.scale_dyn()
    ds.calc_sspec(lamsteps=True)
    ds.fit_arc(lamsteps=True, etamin=2, etamax=400, delmax=1, numsteps=1e3, nsmooth=7,
               startbin=2)
    assert ds.dyn.shape == (398, 11) and np.all(np.isfinite(ds.dyn))
    assert np.isfinite(ds.betaeta)
    print("J0437 excerpt: betaeta %.6g +/- %.3g" % (ds.betaeta, ds.betaetaerr))
