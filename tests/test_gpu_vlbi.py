"""Multi-station theta-theta retrieval (ththmod.VLBI_chunk_retrieval, sb_vlbi_retrieval,
sb_cs_c2c_f32) against the reference's wavefields (tests/golden/vlbi_sample_*.npz, made
by oracle/make_golden_vlbi.py from the unmodified reference) and the numpy oracle.

Error bounds, as in test_gpu_chisq.py: the eigenvalue to 2e-6 |w| + eps32 ||A||_F;
the eigenvector, after one global phase, to (E_VEC + eps32 ||A||_F / w) / relgap with
relgap = (w1 - w2) / w1 of the composite; every station's wavefield, after the SAME
phase, to E_MODEL plus that eigenvector bound, relative to its norm.  Sharing one
phase checks the phases between the stations, which VLBI users rely on."""
import os

import numpy as np
import pytest

from oracle import thth_oracle as TO
from oracle import vlbi_oracle as VO

pytestmark = pytest.mark.gpu

E_MODEL, E_VEC = 5e-5, 4e-6
EPS32 = np.finfo(np.float32).eps


@pytest.fixture(scope="module")
def th():
    from scintools_b200 import ththmod
    return ththmod


def _load(golden_dir, tag):
    return np.load(os.path.join(golden_dir, "vlbi_sample_%s.npz" % tag))


def _inputs(f, n_dish=None):
    n_dish = int(f["n_dish"]) if n_dish is None else n_dish
    autos = set(VO.auto_indices(n_dish))
    return [f["dspec"][k].real if k in autos else f["dspec"][k] for k in range(len(f["dspec"]))]


def _params(f, dlist, n_dish):
    return (dlist, f["edges"], f["time"], f["freq"], float(f["eta"]), 0, 0, int(f["npad"]),
            n_dish, float(f["tau_mask"]) if "tau_mask" in f.files else 0.0, False)


def _bounds(w, w1, w2, fro):
    relgap = (w1 - w2) / w1
    return 2e-6 * abs(w) + EPS32 * fro, (E_VEC + EPS32 * fro / w1) / relgap


def _check(models, w, V, ref_models, w_ref, V_ref, w1, w2, fro, label):
    bw, bv = _bounds(w_ref, w1, w2, fro)
    assert abs(w - w_ref) <= bw, (label, w, w_ref, bw)
    ph = np.vdot(V_ref, V)
    ph /= abs(ph)
    ev = np.linalg.norm(V - ph * V_ref)
    assert ev <= bv, (label, ev, bv)
    worst = ev / bv
    for d, ref in enumerate(ref_models):
        # model_E is linear in conj(V): the same phase, conjugated, for every station
        err = np.linalg.norm(models[d] - np.conj(ph) * ref) / np.linalg.norm(ref)
        b = E_MODEL + bv
        assert err <= b, (label, d, err, b)
        worst = max(worst, err / b)
    print("%s: worst error %.3g of its bound" % (label, worst))


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_vlbi_matches_reference(th, golden_dir, tag):
    """a: 3 stations, 256 x 512 (radix); b: 2 stations, 256 x 568 (chirp-z) with a tau
    mask; c: one station."""
    f = _load(golden_dir, tag)
    n_dish = int(f["n_dish"])
    p = _params(f, _inputs(f), n_dish)
    model, w, V, info, err = th._vlbi_run(p[0], p[1], p[2], p[3], p[4], p[7], n_dish, p[9])
    assert err is None and info["status"] == 0 and info["nred"] == int(f["nred"])
    _check(model, w, V, f["model_E"], float(f["w"]), f["V"], float(f["w1"]), float(f["w2"]),
           float(f["fro"]), "case " + tag)
    out, idx_f, idx_t = th.VLBI_chunk_retrieval(p)
    assert (idx_f, idx_t) == (0, 0) and len(out) == n_dish
    assert all(o.shape == f["model_E"][0].shape and o.dtype == complex for o in out)


def test_vlbi_one_station_matches_single_chunk(th, golden_dir):
    """n_dish = 1 is single_chunk_retrieval of the station's dynamic spectrum."""
    f = _load(golden_dir, "c")
    d = f["dspec"][0].real
    (one,), _, _ = th.VLBI_chunk_retrieval(_params(f, [d], 1))
    single, _, _ = th.single_chunk_retrieval((d, f["edges"], f["time"], f["freq"],
                                              float(f["eta"]), 0, 0, int(f["npad"]), 0.0, False))
    ph = np.vdot(single, one)
    ph /= abs(ph)
    _, bv = _bounds(float(f["w"]), float(f["w1"]), float(f["w2"]), float(f["fro"]))
    err = np.linalg.norm(one - ph * single) / np.linalg.norm(single)
    assert err <= E_MODEL + bv, (err, E_MODEL + bv)


def test_vlbi_zero_visibility_is_block_diagonal(th, golden_dir):
    """V12 = 0: the station with the larger top eigenvalue gets its single-station
    wavefield, the other one (its spectrum halved, so the gap is clear) nothing."""
    f = _load(golden_dir, "a")
    i1, i2 = f["dspec"][0].real, 0.5 * f["dspec"][3].real
    z = np.zeros_like(f["dspec"][1])
    (e1, e2), _, _ = th.VLBI_chunk_retrieval(_params(f, [i1, z, i2], 2))
    w1 = th._vlbi_run([i1], f["edges"], f["time"], f["freq"], float(f["eta"]), 3, 1, 0.0)[1]
    w2 = th._vlbi_run([i2], f["edges"], f["time"], f["freq"], float(f["eta"]), 3, 1, 0.0)[1]
    assert w1 > 1.2 * w2
    single, _, _ = th.single_chunk_retrieval((i1, f["edges"], f["time"], f["freq"],
                                              float(f["eta"]), 0, 0, 3, 0.0, False))
    ph = np.vdot(single, e1)
    ph /= abs(ph)
    # the bound of the two-station composite itself: its norm and its two top eigenvalues
    # (the second may be station 1's own second eigenvalue rather than station 2's top)
    _, x = VO.VLBI_chunk_retrieval([i1, z, i2], f["edges"], f["time"], f["freq"],
                                   float(f["eta"]), 3, 2, return_all=True)
    ev = np.linalg.eigvalsh(x["composite"])
    _, bv = _bounds(ev[-1], ev[-1], ev[-2], np.linalg.norm(x["composite"]))
    assert np.linalg.norm(e1 - ph * single) <= (E_MODEL + bv) * np.linalg.norm(single)
    assert np.linalg.norm(e2) <= (E_MODEL + bv) * np.linalg.norm(e1)


def test_vlbi_failures(th, golden_dir):
    """d: all-zero input raises the reference's ArpackError, a grid past the fd axis its
    IndexError; argument errors raise ValueError."""
    f = _load(golden_dir, "d")

    def real_autos(lst):                       # [I1, V12, I2]
        return [x if k == 1 else x.real for k, x in enumerate(lst)]

    with pytest.raises(Exception) as ex:
        th.VLBI_chunk_retrieval(_params(f, real_autos(f["zero_dspec"]), 2))
    assert type(ex.value).__name__ == str(f["zero_error"])
    p = list(_params(f, real_autos(f["wide_dspec"]), 2))
    p[1], p[4] = f["wide_edges"], float(f["wide_eta"])
    with pytest.raises(Exception) as ex:
        th.VLBI_chunk_retrieval(tuple(p))
    assert type(ex.value).__name__ == str(f["wide_error"])
    # a crop of one theta centre: the reference fails on edges_red, for any n_dish
    p = list(_params(f, real_autos(f["wide_dspec"]), 2))
    p[4] = float(f["one_eta"])
    for lst, nd in ((p[0], 2), (p[0][:1], 1)):
        p[0], p[8] = lst, nd
        with pytest.raises(Exception) as ex:
            th.VLBI_chunk_retrieval(tuple(p))
        assert type(ex.value).__name__ == str(f["one_error"]), nd
    a = _load(golden_dir, "a")
    good = _inputs(a)
    with pytest.raises(ValueError, match="entries"):
        th.VLBI_chunk_retrieval(_params(a, good[:5], 3))
    bad = list(good)
    bad[2] = bad[2][:, :-1]
    with pytest.raises(ValueError, match="shape"):
        th.VLBI_chunk_retrieval(_params(a, bad, 3))
    bad = list(good)
    bad[1] = bad[1].copy()
    bad[1][3, 4] = np.nan
    with pytest.raises(ValueError, match="finite"):
        th.VLBI_chunk_retrieval(_params(a, bad, 3))


def test_vlbi_composite_size_limit(th):
    """n_dish * nred = 8192 runs (an all-zero composite: one mat-vec, w = 0); 8193 is
    refused with an error naming the limit, and the library keeps working."""
    from scintools_b200 import _lib
    nf, nt = 16, 16
    time = np.arange(nt) * 10.0
    freq = 1400.0 + 0.05 * np.arange(nf)
    z = [np.zeros((nf, nt))]
    for n_dish, nedge in ((1, 8193), (2, 4097)):
        # every centre inside the crop; the shift keeps the smallest |centre| unique
        edges = np.linspace(-1.0, 1.0, nedge) + 1e-6
        _, w, _, info, _ = th._vlbi_run(z * (n_dish * (n_dish + 1) // 2), edges, time, freq,
                                        1e-3, 0, n_dish, 0.0)
        assert n_dish * info["nred"] == 8192 and info["status"] == 2 and w == 0.0
    with pytest.raises(_lib.SbError, match="8192"):
        th._vlbi_run(z, np.linspace(-1.0, 1.0, 8194) + 1e-6, time, freq, 1e-3, 0, 1, 0.0)
    f_edges = np.linspace(-1.0, 1.0, 64) + 1e-6
    _, w, _, info, _ = th._vlbi_run(z, f_edges, time, freq, 1e-3, 0, 1, 0.0)
    assert info["nred"] == 63 and info["status"] == 2


@pytest.mark.parametrize("shape", [(65536, 8), (8, 16384), (32768, 3), (3, 8192)])
def test_cs_c2c_largest_sizes(th, shape):
    """sb_cs_c2c_f32 at the largest size of each path and axis against np.fft.fft2; the
    next size up is refused with the limits in the message."""
    from scintools_b200 import _lib
    rng = np.random.default_rng(sum(shape))
    x = rng.normal(size=shape) + 1j * rng.normal(size=shape)
    got = th.conjugate_spectrum(x, 0, 0.0).numpy()
    ref = np.fft.fftshift(np.fft.fft2(x.astype(np.complex64).astype(np.complex128)))
    assert np.linalg.norm(got - ref) <= 2e-6 * np.linalg.norm(ref)
    big = (shape[0] * 2, shape[1]) if shape[0] > shape[1] else (shape[0], shape[1] * 2)
    if shape[1] == 3 or shape[0] == 3:
        big = (shape[0] + 1, shape[1]) if shape[0] > shape[1] else (shape[0], shape[1] + 1)
    with pytest.raises(_lib.SbError, match="outside"):
        th.conjugate_spectrum(np.zeros(big, complex), 0, 0.0)


@pytest.mark.parametrize("shape", [(8, 12), (8, 16), (4, 16), (3, 16), (16, 3)])
def test_cs_c2c_mask_mean_and_small_sizes(th, shape):
    """Tau row mask and device-side mean padding on both paths (8 x 16 with npad 1 is a
    power-of-two 16 x 32: radix; 8 x 12 -> 16 x 24: chirp-z); the lower size limits from
    both sides: 4 x 16 (a power of two below the radix minimum of 8) and 3 on either axis
    run on the chirp-z path, 2 on either axis is refused."""
    from scintools_b200 import _lib
    rng = np.random.default_rng(shape[0] * 100 + shape[1])
    x = rng.normal(size=shape) + 1j * rng.normal(size=shape)
    npad = 1 if shape[0] == 8 else 0
    tau = TO.fft_axis(1400 + 0.05 * np.arange(shape[0]), "us", npad)
    mask = 3.0 if npad else 0.0
    got = th.conjugate_spectrum(x, npad, None, tau, mask).numpy()
    xs = x.astype(np.complex64).astype(np.complex128)
    pad = np.pad(xs, ((0, npad * shape[0]), (0, npad * shape[1])), constant_values=xs.mean())
    ref = np.fft.fftshift(np.fft.fft2(pad))
    ref[np.abs(tau) < mask] = 0
    if npad:
        assert (np.abs(tau) < mask).sum() > 1 and (got[np.abs(tau) < mask] == 0).all()
    assert np.linalg.norm(got - ref) <= 2e-6 * np.linalg.norm(ref)
    low = (2, shape[1]) if shape[0] <= shape[1] else (shape[0], 2)
    with pytest.raises(_lib.SbError, match="outside"):
        th.conjugate_spectrum(np.zeros(low, complex), 0, 0.0)


def synthetic_stations(n_dish, nf, nt, seed):
    """Point images on the arc tau = eta fd^2 seen by every station with a per-image,
    per-station phase, plus noise.  Returns (list, time, freq, eta, edges)."""
    rng = np.random.default_rng(seed)
    dt, df, eta = 100.0, 0.05, 2.0
    t = np.arange(nt) * dt
    f = 1400.0 + np.arange(nf) * df
    fdk = rng.uniform(-1.5, 1.5, 24)
    ak = (rng.normal(size=24) + 1j * rng.normal(size=24)) * np.exp(-(fdk / 1.0) ** 2)
    E = []
    for d in range(n_dish):
        ph = np.exp(2j * np.pi * rng.uniform(size=24) * 0.2 * d)
        E.append(sum(a * p * np.exp(2j * np.pi * (fd_ * 1e-3 * t[None, :] -
                                                  eta * fd_ ** 2 * (f[:, None] - f[0])))
                     for a, p, fd_ in zip(ak, ph, fdk)))
    sig = np.mean(np.abs(E[0]) ** 2)
    out = []
    for d1 in range(n_dish):
        for d2 in range(d1, n_dish):
            if d1 == d2:
                x = np.abs(E[d1]) ** 2 + rng.normal(0, 0.05 * sig, (nf, nt))
                out.append(x - x.mean())
            else:
                out.append(E[d1] * np.conj(E[d2]) +
                           0.05 * sig * (rng.normal(size=(nf, nt)) + 1j * rng.normal(size=(nf, nt))))
    return out, t, f, eta, np.linspace(-2.0, 2.0, 200)


def test_vlbi_large_matches_oracle(th):
    """3 stations on a 256 x 512 conjugate spectrum (128 x 256 chunk, npad = 1)."""
    dl, t, f, eta, edges = synthetic_stations(3, 128, 256, 11)
    models, x = VO.VLBI_chunk_retrieval(dl, edges, t, f, eta, 1, 3, 0.0, return_all=True)
    ev = np.linalg.eigvalsh(x["composite"])
    assert (ev[-1] - ev[-2]) / ev[-1] > 1e-2
    got, w, V, info, err = th._vlbi_run(dl, edges, t, f, eta, 1, 3, 0.0)
    assert err is None and info["status"] == 0
    _check(got, w, V, models, x["w"], x["V"], ev[-1], ev[-2], np.linalg.norm(x["composite"]),
           "large")
