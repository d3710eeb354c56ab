"""Arc asymmetry (Dynspec.calc_asymmetry, ththmod.calc_asymmetry / asymmetry_batch,
sb_asymmetry_batch) against the reference (tests/golden/asymmetry_sample.npz, made by
oracle/make_golden_asymmetry.py from the unmodified reference).

Error bound.  The device finds the top eigenvector of a perturbed matrix A + E with a
Lanczos residual r: V_gpu = V + dV after one global phase, and (Davis-Kahan, sin theta <=
(||E|| + ||r||) / gap, |dV| <= sqrt(2) sin theta)

    |dV| <= sqrt(2) (c 2^-24 ||A||_F + tol |w|) / (w1 - w2)

with w1 > w2 the two largest eigenvalues of the reference's thth_red and ||A||_F its
Frobenius norm.  c counts the fp32 perturbations of A relative to ||A||_F: 1 for rounding
every gathered entry, 1 for the fp32 Jacobian, 17 for the fp32 conjugate spectrum (the
transform tests hold fp32 complex outputs to 1e-6 ~ 17 * 2^-24 normwise) and 17 for the
fp32 mat-vec of the Lanczos steps (rounding errors of n = 301 terms accumulate like
sqrt(n) 2^-24 per row): c = 36.  tol = 2e-6 is the residual the solver accepts at its
iteration cap (anything worse is flagged SB_ETA_NOT_CONVERGED and gives NaN).  With
L, R the weights of the two halves and S = L + R, |dL| + |dR| <= 2 |dV| to first order,
so

    |a_gpu - a_ref| <= 2 (1 + |a_ref|) / S * |dV|,

and every element of |V|^2 moves by at most (2 |V_i| + |dV|) |dV|."""
import contextlib
import io
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C_GATHER, TOL_ACCEPT = 36.0, 2e-6


@pytest.fixture(scope="module")
def f(golden_dir):
    return np.load(os.path.join(golden_dir, "asymmetry_sample.npz"))


def make_dynspec(f):
    from scintools_b200.dynspec import BasicDyn, Dynspec
    ds = Dynspec(dyn=BasicDyn(f["dyn"].astype(np.float64), times=f["times"], freqs=f["freqs"]),
                 verbose=False)
    ds.cwf, ds.cwt, ds.npad = int(f["cwf"]), int(f["cwt"]), int(f["npad"])
    ds.ncf_fit, ds.nct_fit = f["asymmetry"].shape
    ds.fref, ds.edges, ds.ththeta = float(f["fref"]), f["edges"], float(f["ththeta"])
    return ds


def _dV(f):
    return np.sqrt(2) * (C_GATHER * 2.0 ** -24 * f["fro"] + TOL_ACCEPT * np.abs(f["w1"])) / \
        (f["w1"] - f["w2"])


def test_case_a_within_bound(f, capsys):
    """Dynspec.calc_asymmetry on 16 x 4 chunks of widths 32 / 48 / 64 / 80 (radix and
    chirp-z sizes): complex [ncf][nct], the reference's NaN pattern, every finite chunk and
    every element of |V|^2 within the first-order bound."""
    from scintools_b200 import ththmod
    ds = make_dynspec(f)
    ds.calc_asymmetry()
    ref = f["asymmetry"]
    assert ds.asymmetry.dtype == np.complex128 and ds.asymmetry.shape == ref.shape
    assert np.array_equal(np.isnan(ds.asymmetry), np.isnan(ref))
    assert (ds.asymmetry.imag == 0).all()
    a_ref, a_gpu = ref.real.ravel(), ds.asymmetry.real.ravel()
    dV = _dV(f)
    bound = 2 * (1 + np.abs(a_ref)) / f["S"] * dV
    fin = np.isfinite(a_ref)
    frac = np.abs(a_gpu - a_ref)[fin] / bound[fin]
    assert frac.max() <= 1.0, (frac.max(), np.argmax(frac))
    res, info = ththmod.asymmetry_batch(ds._asymmetry_params(), return_info=True)
    assert np.array_equal(np.array([r[0] for r in res]), a_gpu)        # same calls, same bits
    assert (info["nred"] == f["nred"]).all() and (info["status"] == 0).all()
    vfrac = 0.0
    for k in range(len(res)):
        n = int(f["nred"][k])
        v2 = np.abs(info["V"][k]) ** 2
        r2 = f["V2"][k, :n].astype(np.float64)
        # the stored |V|^2 is float32: add its rounding
        vb = (2 * np.sqrt(r2) + dV[k]) * dV[k] + 2.0 ** -24 * r2
        vfrac = max(vfrac, (np.abs(v2 - r2) / vb).max())
    assert vfrac <= 1.0
    with capsys.disabled():
        print("\nasymmetry case a: worst error %.3g of its bound (asymmetry), %.3g (|V|^2)"
              % (frac.max(), vfrac))


def test_single_call_matches_batch(f):
    """ththmod.calc_asymmetry on one chunk is bit-identical to that chunk's entry of the
    batched call, one chunk of each width."""
    from scintools_b200 import ththmod
    pars = make_dynspec(f)._asymmetry_params()
    batch = ththmod.asymmetry_batch(pars)
    for k in (0, 5, 10, 15, 33):
        one = ththmod.calc_asymmetry(pars[k])
        assert one[1:] == (pars[k][6], pars[k][5])
        assert one[0] == batch[k][0], k


def test_small_slab_is_bit_identical(f, tmp_path):
    """SB_SWEEP_SLAB_MB=1 (one chunk per batch) gives the default run's bits."""
    code = ("import sys, numpy as np; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from test_gpu_asymmetry import make_dynspec\n"
            "f = np.load(%r)\n"
            "ds = make_dynspec(f); ds.calc_asymmetry()\n"
            "np.save(%r, ds.asymmetry)\n") % (ROOT, os.path.join(ROOT, "tests"),
                                              os.path.join(ROOT, "tests", "golden",
                                                           "asymmetry_sample.npz"),
                                              str(tmp_path / "small.npy"))
    env = dict(os.environ, SB_SWEEP_SLAB_MB="1")
    subprocess.run([sys.executable, "-c", code], check=True, env=env, cwd=ROOT)
    ds = make_dynspec(f)
    ds.calc_asymmetry()
    small = np.load(tmp_path / "small.npy")
    assert np.array_equal(small.view(np.uint64), ds.asymmetry.view(np.uint64))


@pytest.mark.parametrize("tag", ["zero", "small", "wide"])
def test_failures_give_nan_with_message(f, tag):
    """An all-zero chunk, a crop of fewer than 3 centres and a grid past the fd axis: NaN,
    the reason printed, no exception (as the reference's try/except)."""
    from scintools_b200 import ththmod
    cwf, cwt = int(f["cwf"]), int(f["cwt"])
    d = np.zeros((cwf, cwt)) if tag == "zero" else f["b_dspec"]
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        a, idx_f, idx_t = ththmod.calc_asymmetry(
            (d, f["b_%s_edges" % tag], f["times"][:cwt], f["freqs"][cwf:2 * cwf],
             float(f["b_%s_eta" % tag]), 0, 1, int(f["npad"]), False))
    assert np.isnan(a) and np.isnan(float(f["b_%s_asymm" % tag]))
    assert (idx_f, idx_t) == (1, 0)
    assert buf.getvalue().strip()


def test_oversized_raises_before_launch_and_library_stays_usable(f):
    """More than 4096 theta centres, or a padded chunk past the chirp-z limit: SbError naming
    the limit, raised before any launch; a normal chunk still works afterwards."""
    from scintools_b200 import _lib, ththmod
    pars = make_dynspec(f)._asymmetry_params()
    d, edges, t, fr, eta = pars[0][:5]
    n0 = _lib.lib.sb_launch_count()
    with pytest.raises(_lib.SbError, match="4096"):
        ththmod.asymmetry_batch([pars[0], (d, np.linspace(-0.3, 0.3, 4098), t, fr, eta, 0, 0, 3,
                                           False)])
    dt = t[1] - t[0]
    wide = np.zeros((64, 2100))
    with pytest.raises(_lib.SbError, match="8192"):
        ththmod.calc_asymmetry((wide, edges, dt * np.arange(2100), fr, eta, 0, 0, 3, False))
    assert _lib.lib.sb_launch_count() == n0
    ref = ththmod.asymmetry_batch(pars[:1])[0][0]
    assert abs(ref - f["asymmetry"][0, 0].real) < 1e-3


def test_mismatched_geometries_are_rejected(f):
    """sb_asymmetry_batch refuses chunks that do not share the spectrum size."""
    from scintools_b200 import _device as D, _lib, ththmod
    import torch
    pars = make_dynspec(f)._asymmetry_params()
    geoms, keep = [], []
    for p in (pars[0], pars[1]):                     # widths 32 and 48
        d, edges, t, fr = p[:4]
        fd = ththmod.fft_axis(t, "mHz", 3)
        tau = ththmod.fft_axis(fr, "us", 3)
        cs = ththmod.conjugate_spectrum(d, 3, None)
        g = ththmod._Geom(cs, tau, fd, edges, True)
        keep.append((cs, g))
        geoms.append(g.g)
    arr = (_lib.ThthGeom * 2)(*geoms)
    etas = D.upload(np.array([pars[0][4], pars[1][4]]))
    o = [D.empty((2,), torch.float64) for _ in range(2)] + [D.empty((2,), torch.int32)
                                                             for _ in range(3)]
    rc = _lib.lib.sb_asymmetry_batch(arr, 2, etas.data_ptr(), 0.0, 0, *[x.data_ptr() for x in o],
                                     None, D.stream_ptr())
    assert rc == -2 and b"differs" in _lib.lib.sb_last_error()


def test_dynspec_contract(f):
    ds = make_dynspec(f)
    with pytest.raises(ValueError):
        ds.calc_asymmetry(pool=object())
    assert not hasattr(ds, "asymmetry")
