"""Generate tests/golden/chisq_sample_64x150.npz by running the UNMODIFIED
reference's ththmod.chisq_calc (via oracle/ref_loader.py) on the tutorial chunk.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only,
after oracle/make_golden.py has written thth_sample_64x150.npz:

    python -m oracle.make_golden_chisq

The fixture is committed; the GPU box never needs the reference.
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import ref_loader  # noqa: E402


def _chisq_case(thth, u, dspec, CS, tau, fd, etas, edges, N, mask):
    """Reference chisq_calc per curvature plus what the GPU test's error bound
    needs: the two largest eigenvalues of thth_red and the masked norms of the
    model and of the residual (from the reference's modeler)."""
    rows = []
    for e in etas:
        c = thth.chisq_calc(dspec, CS, tau, fd, e * u.s ** 3, edges * u.mHz, N, mask)
        out = thth.modeler(CS, tau, fd, e * u.s ** 3, edges * u.mHz)
        wv = np.linalg.eigvalsh(np.asarray(out[0]))
        model = np.asarray(out[3])[:dspec.shape[0], :dspec.shape[1]]
        rows.append((c, wv[-1], wv[-2], np.sqrt(np.sum(model[mask] ** 2)),
                     np.sqrt(np.sum((model - dspec)[mask] ** 2)), out[0].shape[0]))
    r = np.array(rows)
    return dict(chisq=r[:, 0], w1=r[:, 1], w2=r[:, 2], model_norm=r[:, 3], resid_norm=r[:, 4],
                nred=r[:, 5].astype(np.int32))


def golden_chisq(pkg):
    """ththmod.chisq_calc: the chi-square search of THTHSample.ipynb (cells 36-44)
    on the tutorial chunk of thth_sample_64x150.npz.
      a: cell 40 -- CS of dspec2 - mean padded with 0 (256 x 600, chirp-z path),
         dspec2 itself as the data, N from the whole noisy dynamic spectrum;
      b: cell 44 on the 64 x 128 piece -- CS padded with the mean (256 x 512, radix
         path), a seeded mask with ~10 % False and a NaN in dspec outside the mask;
      c: an all-zero CS with a non-zero dspec (the reference raises: ARPACK)."""
    u = sys.modules["astropy.units"]
    thth = pkg.ththmod
    g = np.load(os.path.join(GOLD, "thth_sample_64x150.npz"))
    arch = np.load(os.path.join(ref_loader.REFERENCE_ROOT, "scintools", "examples", "data",
                                "ththsims", "Sample_Data.npz"))
    rng = np.random.default_rng(7)                        # the noise of golden_thth
    dspec = np.abs(arch["Espec"]) ** 2 + rng.normal(0, 20, arch["Espec"].shape)
    temp = np.fft.fftshift(np.abs(np.fft.fft2(dspec) / np.sqrt(dspec.shape[0] * dspec.shape[1])) ** 2)
    N = np.sqrt(temp[: temp.shape[0] // 6, : temp.shape[1] // 6].mean())
    npad = int(g["npad"])
    edges = np.linspace(-0.4, 0.4, 512)
    etas = np.linspace(12.5, 100.0, 100)
    dspec2 = g["dspec2"]
    out = dict(N=N, npad=npad, edges=edges, etas=etas)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        # (a)
        pad = np.pad(dspec2 - dspec2.mean(), ((0, npad * dspec2.shape[0]), (0, npad * dspec2.shape[1])),
                     mode="constant", constant_values=0)
        CS = np.fft.fftshift(np.fft.fft2(pad))
        tau, fd = g["tau"] * u.us, g["fd"] * u.mHz
        mask = np.ones(dspec2.shape, dtype=bool)
        for k, v in _chisq_case(thth, u, dspec2, CS, tau, fd, etas, edges, N, mask).items():
            out["a_" + k] = v
        # (b)
        db = np.copy(dspec2[:, :128])
        time_b = g["time"][:128]
        pad = np.pad(db, ((0, npad * db.shape[0]), (0, npad * db.shape[1])), mode="constant",
                     constant_values=db.mean())
        CS_b = np.fft.fftshift(np.fft.fft2(pad))
        fd_b = thth.fft_axis(time_b * u.s, u.mHz, npad)
        tau_b = thth.fft_axis(g["freq"] * u.MHz, u.us, npad)
        mrng = np.random.default_rng(13)
        mask_b = mrng.random(db.shape) > 0.1
        i, j = np.argwhere(~mask_b)[0]
        db_nan = np.copy(db)
        db_nan[i, j] = np.nan
        for k, v in _chisq_case(thth, u, db_nan, CS_b, tau_b, fd_b, etas, edges, N, mask_b).items():
            out["b_" + k] = v
        out.update(b_dspec=db_nan, b_mask=mask_b, b_time=time_b, b_tau=np.asarray(tau_b.value),
                   b_fd=np.asarray(fd_b.value), b_nan_index=np.array([i, j]))
        # (c)
        zeros = np.zeros_like(CS_b)
        err = []
        for e in etas[::20]:
            try:
                thth.chisq_calc(db, zeros, tau_b, fd_b, e * u.s ** 3, edges * u.mHz, N)
                err.append("")
            except Exception as ex:  # noqa: BLE001
                err.append(type(ex).__name__)
        out.update(c_etas=etas[::20], c_error=np.array(err))
    np.savez_compressed(os.path.join(GOLD, "chisq_sample_64x150.npz"), **out)
    print("chisq: a argmin eta %.2f, b argmin eta %.2f, c errors %s"
          % (etas[np.argmin(out["a_chisq"])], etas[np.argmin(out["b_chisq"])], set(err)))


if __name__ == "__main__":
    golden_chisq(ref_loader.load())
