"""Generate tests/golden/vlbi_sample_*.npz by running the UNMODIFIED reference's
ththmod.VLBI_chunk_retrieval (via oracle/ref_loader.py) on stations cut from the
tutorial field.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Run in the build container only,
after oracle/make_golden.py has written thth_sample_64x150.npz:

    python -m oracle.make_golden_vlbi

The reference's eigsh is wrapped (not changed) so that the composite matrix it
received and the (w, V) it returned are recorded next to its wavefields: the
global phase of the stored V is the one the stored wavefields carry.
The fixtures are committed; the GPU box never needs the reference.
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

OFFSETS = (0, 8, 16)          # time offsets of the stations in the tutorial field


def stations(espec, nt, n_dish, seed):
    """[I1, V12, .., V1N, I2, .., IN] from E_d = espec[:, s_d:s_d + nt]: I_d = |E_d|^2 +
    noise minus its mean, V_ij = E_i conj(E_j) + complex noise."""
    rng = np.random.default_rng(seed)
    E = [espec[:, s:s + nt] for s in OFFSETS[:n_dish]]
    sig = np.mean(np.abs(E[0]) ** 2)
    out = []
    for d1 in range(n_dish):
        for d2 in range(d1, n_dish):
            if d1 == d2:
                x = np.abs(E[d1]) ** 2 + rng.normal(0, 0.05 * sig, E[d1].shape)
                out.append(x - x.mean())
            else:
                x = E[d1] * np.conjugate(E[d2])
                x = x + 0.05 * sig * (rng.normal(size=x.shape) + 1j * rng.normal(size=x.shape))
                out.append(x)
    return out


def run_case(thth, u, dlist, time, freq, eta, edges, npad, n_dish, tau_mask):
    """Reference call with eigsh recorded; returns the fixture entries."""
    seen = []
    orig = thth.eigsh

    def spy(a, *args, **kw):
        seen.append(np.array(a))
        w, V = orig(a, *args, **kw)
        seen.append((w, V))
        return w, V

    thth.eigsh = spy
    try:
        model_E, _, _ = thth.VLBI_chunk_retrieval(
            (dlist, edges * u.mHz, time * u.s, freq * u.MHz, eta * u.s ** 3, 0, 0, npad,
             n_dish, tau_mask * u.us, False))
    finally:
        thth.eigsh = orig
    comp, (w, V) = seen
    ev = np.linalg.eigvalsh(comp)
    gap = (ev[-1] - ev[-2]) / abs(ev[-1])
    assert gap >= 1e-2, "relative eigengap %g too small for the error bounds" % gap
    return dict(model_E=np.array(model_E), w=float(w[0]), V=V[:, 0], w1=ev[-1], w2=ev[-2],
                fro=np.linalg.norm(comp), nred=comp.shape[0] // n_dish)


def expect_raise(thth, u, dlist, time, freq, eta, edges, npad, n_dish):
    try:
        thth.VLBI_chunk_retrieval((dlist, edges * u.mHz, time * u.s, freq * u.MHz,
                                   eta * u.s ** 3, 0, 0, npad, n_dish, 0 * u.us, False))
    except Exception as ex:  # noqa: BLE001
        return type(ex).__name__
    return ""


def golden_vlbi(pkg):
    u = sys.modules["astropy.units"]
    thth = pkg.ththmod
    g = np.load(os.path.join(GOLD, "thth_sample_64x150.npz"))
    arch = np.load(os.path.join(ref_loader.REFERENCE_ROOT, "scintools", "examples", "data",
                                "ththsims", "Sample_Data.npz"))
    nf = g["dspec2"].shape[0]
    espec = arch["Espec"][:nf]                         # the channels of thth_sample_64x150
    freq, time_all = g["freq"], g["time"]
    eta = float(g["ss_eta_fit"])
    edges = np.linspace(-0.4, 0.4, 256)
    cases = {"a": (3, 128, 3, 0.0, 1), "b": (2, 142, 3, 0.4, 2), "c": (1, 128, 3, 0.0, 3)}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for tag, (n_dish, nt, npad, tau_mask, seed) in cases.items():
            dlist = stations(espec, nt, n_dish, seed)
            time = time_all[:nt]
            out = run_case(thth, u, dlist, time, freq, eta, edges, npad, n_dish, tau_mask)
            out.update(dspec=np.array(dlist, dtype=complex), time=time, freq=freq, eta=eta,
                       edges=edges, npad=npad, n_dish=n_dish, tau_mask=tau_mask)
            np.savez_compressed(os.path.join(GOLD, "vlbi_sample_%s.npz" % tag), **out)
            print("vlbi %s: %d stations, nred %d, w %.6g, gap %.3g" %
                  (tag, n_dish, out["nred"], out["w"], (out["w1"] - out["w2"]) / out["w1"]))
        # (d) all-zero inputs; a theta grid that reaches past the fd axis (IndexError)
        nt = 128
        zeros = [np.zeros((nf, nt)), np.zeros((nf, nt), complex), np.zeros((nf, nt))]
        err_zero = expect_raise(thth, u, zeros, time_all[:nt], freq, eta, edges, 3, 2)
        wide = np.linspace(-40.0, 40.0, 64)
        dlist = stations(espec, nt, 2, 4)
        err_wide = expect_raise(thth, u, dlist, time_all[:nt], freq, 0.01, wide, 3, 2)
        # a curvature so large that the crop keeps only the centre theta = 0
        err_one = expect_raise(thth, u, dlist, time_all[:nt], freq, 1e9, edges, 3, 2)
        np.savez_compressed(os.path.join(GOLD, "vlbi_sample_d.npz"),
                            zero_dspec=np.array(zeros, dtype=complex), zero_error=err_zero,
                            wide_dspec=np.array(dlist, dtype=complex), wide_edges=wide,
                            wide_eta=0.01, wide_error=err_wide, one_eta=1e9,
                            one_error=err_one, time=time_all[:nt], freq=freq,
                            eta=eta, edges=edges, npad=3, n_dish=2)
        print("vlbi d: zero -> %r, wide grid -> %r, one centre -> %r"
              % (err_zero, err_wide, err_one))


if __name__ == "__main__":
    golden_vlbi(ref_loader.load())
