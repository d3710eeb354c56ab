"""Generate tests/golden/thth_notebook_1317.npz by running the UNMODIFIED
reference's ththmod (via oracle/ref_loader.py) on one chunk of the tutorial field
at the settings of THTHSample.ipynb cell 18.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only:

    python -m oracle.make_golden_grids

The fixture is committed; the GPU box never needs the reference.

Cell 18 calls prep_thetatheta(cwf=128, edges_lim=.3, eta_min=30,
eta_max=109.11037416158051): 1318 edges (1317 theta centres, ld 1344) and chunks of
128 x 150.  With npad = 3 the conjugate spectrum is 512 x 600 (chirp-z path).  The
chunk is cf = 0, ct = 0 of the field of thth_sample_64x150.npz (|Espec|^2 plus
seeded noise), and single_search pads it with its mean.  The fixture records:
  etas, eigs  Eval_calc on every 16th curvature of the chunk's grid;
  w, V2       modeler's top eigenvalue and |V|^2 at one curvature, with the two
              top eigenvalues of its thth_red (eigvalsh) and its Frobenius norm
              for the GPU test's first-order bound.
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

CWF, CWT, NPAD, FW = 128, 150, 3, 0.1
EDGES_LIM, ETA_MIN, ETA_MAX = 0.3, 30.0, 109.11037416158051


def golden_grids(pkg):
    u = sys.modules["astropy.units"]
    thth = pkg.ththmod
    arch = np.load(os.path.join(ref_loader.REFERENCE_ROOT, "scintools", "examples", "data",
                                "ththsims", "Sample_Data.npz"))
    rng = np.random.default_rng(7)                        # the noise of golden_thth
    dspec = np.abs(arch["Espec"]) ** 2 + rng.normal(0, 20, arch["Espec"].shape)
    freqs, times = arch["f_MHz"], arch["t_s"]
    # prep_thetatheta (reference dynspec.py:1348-1537) with the cell-18 keywords
    fref = freqs.mean()
    fd0 = thth.fft_axis(times[:CWT] * u.s, u.mHz)
    tau0 = thth.fft_axis(freqs[:CWF] * u.MHz, u.us)
    fd_cut = (fd0.max().value / 2) * (fref / freqs.max())
    edges_lim = min(EDGES_LIM, fd_cut)
    edges = np.asarray(thth.min_edges(edges_lim * u.mHz, fd0, tau0,
                                      ETA_MAX * (fref / freqs.min()) * u.s ** 3, 2).value) \
        * (freqs.min() / fref)
    neta = int(1 + (np.log10(ETA_MAX) - np.log10(ETA_MIN)) / np.log10(1 + FW / 10))
    chunk = np.copy(dspec[:CWF, :CWT])
    f_c, t_c = freqs[:CWF], times[:CWT]
    etas_all = np.logspace(np.log10(ETA_MIN), np.log10(ETA_MAX), neta) * (fref / f_c.mean()) ** 2
    etas = etas_all[::16]
    # single_search's spectrum (ththmod.py:777-787): padded with the chunk mean
    fd = thth.fft_axis(t_c * u.s, u.mHz, NPAD)
    tau = thth.fft_axis(f_c * u.MHz, u.us, NPAD)
    pad = np.pad(chunk, ((0, NPAD * CWF), (0, NPAD * CWT)), mode="constant",
                 constant_values=chunk.mean())
    CS = np.fft.fftshift(np.fft.fft2(pad))
    eta_m = etas[len(etas) // 2]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        eigs = np.array([thth.Eval_calc(CS, tau, fd, e * u.s ** 3, edges * u.mHz) for e in etas])
        out = thth.modeler(CS, tau, fd, eta_m * u.s ** 3, edges * u.mHz)
    red = np.asarray(out[0])
    wv = np.linalg.eigvalsh(red)
    V = np.asarray(out[6]).ravel()
    np.savez_compressed(
        os.path.join(GOLD, "thth_notebook_1317.npz"),
        chunk=chunk, freq=f_c, time=t_c, npad=NPAD, edges=edges, etas_all=etas_all, etas=etas,
        eigs=eigs, fd=np.asarray(fd.value), tau=np.asarray(tau.value), eta_model=eta_m,
        w=float(np.asarray(out[5]).ravel()[0]), V2=np.abs(V) ** 2, nred=red.shape[0],
        w1=wv[-1], w2=wv[-2], fro=np.linalg.norm(red))
    print("grids: %d edges, %d curvatures (every 16th of %d), nred at the model curvature %d, "
          "peak eta %.2f" % (edges.shape[0], etas.shape[0], neta, red.shape[0],
                             etas[np.argmax(eigs)]))


if __name__ == "__main__":
    golden_grids(ref_loader.load())
