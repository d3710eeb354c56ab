"""Unit-free CPU restatement of ththmod.VLBI_chunk_retrieval (ththmod.py:1223-1387).

TEST INFRASTRUCTURE (see oracle/__init__.py).  float64 numpy built from the
theta-theta gather, rev_map and scipy eigsh of oracle/thth_oracle.py.  Units as
there: tau [us], fd / edges [mHz], eta [s^3], time [s], freq [MHz].
"""
import numpy as np
from scipy.sparse.linalg import eigsh

from oracle import thth_oracle as TO


def auto_indices(n_dish):
    """Positions of the station spectra I_d in [I1, V12, .., V1N, I2, V23, .., IN]."""
    return [n_dish * (n_dish + 1) // 2 - (n_dish - d) * (n_dish - d + 1) // 2
            for d in range(n_dish)]


def pair_index(n_dish, d1, d2):
    """Position of the spectrum of stations (d1, d1 + d2) in the same list."""
    return n_dish * (n_dish + 1) // 2 - (n_dish - d1) * (n_dish - d1 + 1) // 2 + d2


def spectra(dspec2_list, time, freq, npad, n_dish, tau_mask=0.0):
    """Conjugate spectra of every entry: station spectra padded with their mean,
    visibilities with zero; rows with |tau| < tau_mask zeroed.  Returns (list, tau, fd)."""
    fd = TO.fft_axis(time, "mHz", npad)
    tau = TO.fft_axis(freq, "us", npad)
    autos = set(auto_indices(n_dish))
    out = []
    for k, d in enumerate(dspec2_list):
        d = np.asarray(d)
        pad_value = d.mean() if k in autos else 0
        p = np.pad(d, ((0, npad * d.shape[0]), (0, npad * d.shape[1])), mode="constant",
                   constant_values=pad_value)
        cs = np.fft.fftshift(np.fft.fft2(p))
        cs[np.abs(tau) < tau_mask] = 0
        out.append(cs)
    return out, tau, fd


def composite(cs_list, tau, fd, eta, edges, n_dish):
    """Block matrix of the cropped theta-theta maps: block (d1, d1 + d2) holds the
    conjugate transpose of the pair's map, block (d1 + d2, d1) the map itself.
    Returns (matrix, edges_red)."""
    autos = set(auto_indices(n_dish))
    reds = []
    edges_red = None
    for k, cs in enumerate(cs_list):
        red, edges_red = TO.thth_redmap(cs, tau, fd, eta, edges, hermetian=k in autos)
        reds.append(red)
    n = reds[0].shape[0]
    comp = np.zeros((n_dish * n, n_dish * n), dtype=complex)
    for d1 in range(n_dish):
        for d2 in range(n_dish - d1):
            t = reds[pair_index(n_dish, d1, d2)]
            comp[d1 * n:(d1 + 1) * n, (d1 + d2) * n:(d1 + d2 + 1) * n] = np.conjugate(t.T)
            comp[(d1 + d2) * n:(d1 + d2 + 1) * n, d1 * n:(d1 + 1) * n] = t
    return comp, edges_red


def station_models(w, V, n_dish, tau, fd, eta, edges_red, shape):
    """Wavefield of each station from its slice of the eigenvector: rev_map of the
    matrix whose only non-zero row, n//2, is conj(V_d) sqrt(w), then the cropped,
    scaled inverse transform."""
    n = V.shape[0] // n_dish
    out = []
    for d in range(n_dish):
        m = np.zeros((n, n), dtype=complex)
        m[n // 2, :] = np.conjugate(V[d * n:(d + 1) * n]) * np.sqrt(w)
        recov = TO.rev_map(m, tau, fd, eta, edges_red, hermetian=False)
        e = np.fft.ifft2(np.fft.ifftshift(recov))[:shape[0], :shape[1]]
        out.append(e * (shape[0] * shape[1] / 4))
    return out


def VLBI_chunk_retrieval(dspec2_list, edges, time, freq, eta, npad, n_dish, tau_mask=0.0,
                         return_all=False):
    """Wavefields of all stations for one chunk.  With ``return_all`` also returns a
    dict with w, V and the composite matrix.  The eigenvector's global phase is
    arbitrary (ARPACK start vector)."""
    cs_list, tau, fd = spectra(dspec2_list, time, freq, npad, n_dish, tau_mask)
    comp, edges_red = composite(cs_list, tau, fd, eta, edges, n_dish)
    w, V = eigsh(comp, 1, which="LA")
    w, V = w[0], V[:, 0]
    models = station_models(w, V, n_dish, tau, fd, eta, edges_red, np.shape(dspec2_list[0]))
    if return_all:
        return models, dict(w=w, V=V, composite=comp, edges_red=edges_red, tau=tau, fd=fd)
    return models
