"""Dynspec.calc_scattered_image and scattered_image_batch on the device (csrc/scatim.cu):
every fixture of the unmodified reference (oracle/make_golden_scattered_image.py) within
1e-10 of the image's largest magnitude with the same exceptions, scipy's RectBivariateSpline
on a full-size spectrum and at each crop-size limit, a bicubic polynomial reproduced, batches
bit-identical to single calls in any order and grouping, and the library-state cases of
tests/test_gpu_library_state.py for sb_scattered_image_f64."""
import importlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CPU = importlib.import_module("test_scattered_image_cpu")
LS = importlib.import_module("test_gpu_library_state")
grown = LS.grown
Z = CPU.Z
BAR = 1e-10


def rel_err(got, ref):
    return np.max(np.abs(got - ref)) / np.max(np.abs(ref))


@pytest.mark.parametrize("name", [c for c in CPU.CASES if c not in CPU.FIT_RAISES])
def test_fixture(name):
    """Calls that ran the reference's fit_arc get the curvature it found preset."""
    kw, preset = CPU.call_args(Z, name)
    ds = CPU.port_dynspec(Z, CPU.fitted(Z, name, preset))
    raises = str(Z[name + "_raises"])
    if raises:
        with pytest.raises(Exception) as e:
            ds.calc_scattered_image(**kw)
        assert type(e.value).__name__ == raises
        assert not hasattr(ds, "scattered_image")
        return
    ds.calc_scattered_image(**kw)
    CPU.check_image(Z, name, ds.scattered_image, ds.scattered_image_ax, BAR)


@pytest.mark.parametrize("name", CPU.FIT_RAISES + ["fit_lam"])
def test_fit_arc_path(name):
    """Neither eta nor betaeta set: the port's own fit_arc runs first.  Its exception is the
    reference's; where it returns, the image is the oracle's at the curvature it found."""
    kw, preset = CPU.call_args(Z, name)
    ds = CPU.port_dynspec(Z, preset)
    raises = str(Z[name + "_raises"])
    if raises:
        with pytest.raises(Exception) as e:
            ds.calc_scattered_image(**kw)
        assert type(e.value).__name__ == raises
        assert not hasattr(ds, "scattered_image")
        return
    ds.calc_scattered_image(**kw)
    assert abs(ds.betaeta / float(Z[name + "_betaeta"]) - 1) < 1e-3
    Zp = dict(Z)
    Zp[name + "_betaeta"] = ds.betaeta
    im, ax = CPU.oracle_call(Zp, name)
    assert np.array_equal(ds.scattered_image_ax, ax)
    assert rel_err(ds.scattered_image, im) <= BAR


def test_full_size_against_scipy():
    """The 4096 x 16384 secondary spectrum of a seeded 4096 x 8192 dynamic spectrum."""
    from oracle import scattered_image_oracle as SO
    from scintools_b200.dynspec import BasicDyn, Dynspec
    rng = np.random.default_rng(4096)
    nf, nt, dt, df = 4096, 8192, 2.0, 0.05
    dyn = rng.gamma(2.0, 1.0, (nf, nt)).astype(np.float32)
    ds = Dynspec(dyn=BasicDyn(dyn, times=dt * np.arange(nt), freqs=1400 + df * np.arange(nf),
                              dt=dt, df=df), verbose=False)
    ds.calc_sspec()
    assert ds.sspec.shape == (4096, 16384)
    eta = float(np.max(ds.tdel)) / (0.4 * np.max(ds.fdop)) ** 2
    ds.calc_scattered_image(input_eta=eta, sampling=64, plot_log=False)
    ref, ax = SO.scattered_image(ds.sspec, ds.fdop, ds.tdel, eta, 64, plot_log=False)
    assert np.array_equal(ds.scattered_image_ax, ax)
    err = rel_err(ds.scattered_image, ref)
    print("full size: worst error %.3g of max |image|" % err)
    assert err <= BAR


@pytest.mark.parametrize("axis,n", [("doppler", 32768), ("delay", 65536)])
def test_crop_limits_against_scipy(axis, n):
    from oracle import scattered_image_oracle as SO
    from scintools_b200.dynspec import Dynspec
    spec, fd, td, eta = CPU.limit_case(axis, n)
    spec = 10 * np.log10(np.random.default_rng(n).uniform(0.5, 2.0, spec.shape))
    ds = Dynspec.__new__(Dynspec)
    ds.calc_scattered_image(input_sspec=spec, input_fdop=fd, input_tdel=td, input_eta=eta,
                            sampling=20)
    ref, ax = SO.scattered_image(spec, fd, td, eta, 20)
    assert np.array_equal(ds.scattered_image_ax, ax)
    assert rel_err(ds.scattered_image, ref) <= BAR


def test_bicubic_polynomial_is_reproduced():
    """The interpolant is exact for cubics: every image point inside the data range is the
    polynomial times fdop_y; past the last delay, the value at the last delay."""
    from scintools_b200.dynspec import Dynspec
    td = np.linspace(0.0, 3.0, 97)
    fd = np.linspace(-2.0, 2.0, 130)
    p = lambda t, f: (1.5 + 0.3 * t - 0.2 * t ** 2 + 0.05 * t ** 3) * \
        (2.0 - 0.4 * f + 0.1 * f ** 2 + 0.07 * f ** 3)              # noqa: E731
    T, F = np.meshgrid(td, fd, indexing="ij")
    spec = 10 * np.log10(p(T, F))
    eta = 1.0
    ds = Dynspec.__new__(Dynspec)
    ds.calc_scattered_image(input_sspec=spec, input_fdop=fd, input_tdel=td, input_eta=eta,
                            sampling=40, plot_log=False)
    ax, im = ds.scattered_image_ax, ds.scattered_image
    fy = np.linspace(0, ax[-1], 41)
    X, Y = np.meshgrid(ax, fy)
    q = (X ** 2 + Y ** 2) * eta
    want = p(np.minimum(q, td[-1]), X) * Y
    got = im[40:]
    inside = q <= td[-1]
    assert inside.any() and (~inside).any()
    scale = np.max(np.abs(want))
    assert np.max(np.abs(got - want)[inside]) <= 1e-12 * scale
    assert np.max(np.abs(got - want)[~inside]) <= 1e-12 * scale


@pytest.fixture(scope="module")
def tiles():
    """cut_dyn of a 512 x 1024 dynamic spectrum into 8 x 8 tiles, and the tiles' axes."""
    from scintools_b200.dynspec import BasicDyn, Dynspec
    rng = np.random.default_rng(64)
    dyn = rng.gamma(2.0, 1.0, (512, 1024))
    ds = Dynspec(dyn=BasicDyn(dyn, times=8.0 * np.arange(1024),
                              freqs=1300 + 0.25 * np.arange(512), dt=8.0, df=0.25),
                 verbose=False)
    ds.cut_dyn(tcuts=7, fcuts=7)
    fdop, tdel, _ = ds.calc_sspec(input_dyn=ds.cutdyn[0, 0])
    eta = float(np.max(tdel)) / (0.5 * np.max(fdop)) ** 2
    return ds.cutsspec, fdop, tdel, eta


def single(spec, fdop, tdel, eta, sampling=32, plot_log=True):
    from scintools_b200.dynspec import Dynspec
    ds = Dynspec.__new__(Dynspec)
    ds.calc_scattered_image(input_sspec=spec, input_eta=eta, input_fdop=fdop, input_tdel=tdel,
                            sampling=sampling, plot_log=plot_log)
    return ds.scattered_image, ds.scattered_image_ax


def test_repeat_is_bit_identical(tiles):
    S, fd, td, eta = tiles
    a = single(S[2, 3], fd, td, eta)
    b = single(S[2, 3], fd, td, eta)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("n", [1, 7, 64])
def test_batch_equals_single_calls(tiles, n):
    from scintools_b200.dynspec import scattered_image_batch
    S, fd, td, eta = tiles
    flat = S.reshape((-1,) + S.shape[2:])[:n]
    etas = eta * (1 + 0.05 * np.arange(n) / max(n, 1))        # several crops
    ref = [single(flat[k], fd, td, etas[k]) for k in range(n)]
    im, ax = scattered_image_batch(flat, fd, td, etas, sampling=32)
    for k in range(n):
        assert np.array_equal(im[k], ref[k][0]), k
        assert np.array_equal(ax[k], ref[k][1]), k
    shared = [single(flat[k], fd, td, eta, plot_log=False)[0] for k in range(n)]
    im2, _ = scattered_image_batch(flat, fd, td, eta, sampling=32, plot_log=False)
    for k in range(n):
        assert np.array_equal(im2[k], shared[k]), k


def test_batch_order_groups_and_shape(tiles, monkeypatch):
    from scintools_b200 import dynspec as DS
    S, fd, td, eta = tiles
    im, ax = DS.scattered_image_batch(S, fd, td, eta, sampling=16)
    assert im.shape == (8, 8, 33, 33) and ax.shape == (8, 8, 33)
    flat = S.reshape((-1,) + S.shape[2:])
    order = np.random.default_rng(5).permutation(64)
    im_p, _ = DS.scattered_image_batch(flat[order], fd, td, eta, sampling=16)
    assert np.array_equal(im_p, im.reshape(64, 33, 33)[order])
    # groups of three items: the same bits as one group
    mx, my = S.shape[2], S.shape[3]
    monkeypatch.setattr(DS, "_SCATIM_GROUP_BYTES", 3 * 8 * (mx * my + 33 * 33))
    im_g, _ = DS.scattered_image_batch(S, fd, td, eta, sampling=16)
    assert np.array_equal(im_g, im)


# ---- library state: the cases of tests/test_gpu_library_state.py for sb_scattered_image_f64
def run_scatim(size):
    from oracle import scattered_image_oracle as SO
    S, fd, td = CPU.Z["sspec"], CPU.Z["fdop"], CPU.Z["tdel"]
    sampling = 16 if size == "small" else 100
    out = []
    for eta in (0.35, 0.2):
        im, ax = single(S, fd, td, eta, sampling)
        ref, _ = SO.scattered_image(S, fd, td, eta, sampling)
        assert rel_err(im, ref) <= BAR
        out.append(im)
    return out


CASE = LS.Case("scattered_image", ("sb_scattered_image_f64",), True, run_scatim)


def test_cold():
    from scintools_b200 import _lib
    LS._sb()
    _lib.check(_lib.lib.sb_release())
    LS.same(CASE, CASE.run("small"), run_scatim("small"), "cold vs repeat")


def test_after_others(grown):
    a = CASE.run("small")
    from scintools_b200 import _lib
    _lib.check(_lib.lib.sb_release())
    LS.same(CASE, a, CASE.run("small"), "after others vs cold")


def test_small_large_small():
    a = CASE.run("small")
    CASE.run("large")
    LS.same(CASE, CASE.run("small"), a, "small, large, small")


def test_side_stream():
    import torch
    ref = CASE.run("small")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = CASE.run("small")
    torch.cuda.synchronize()
    LS.same(CASE, got, ref, "side stream vs default stream")
