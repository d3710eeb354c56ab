"""Unit-free CPU restatement of ththmod.calc_asymmetry (ththmod.py:2385-2463) and of the
chunk loop of Dynspec.calc_asymmetry (dynspec.py:1892-1918).

TEST INFRASTRUCTURE (see oracle/__init__.py).  float64 numpy on top of the ``modeler``
of oracle/thth_oracle.py.  Units as there: tau [us], fd / edges [mHz], eta [s^3],
time [s], freq [MHz].
"""
import numpy as np

from oracle import thth_oracle as TO


def split(V):
    """(left, right) halves of the eigenvector: V[:(m-1)//2] and V[1+(m-1)//2:], the centre
    element dropped (for even m the split is uneven)."""
    m = V.shape[0]
    return V[:(m - 1) // 2], V[1 + (m - 1) // 2:]


def asymmetry_of(V):
    """(sum|left|^2 - sum|right|^2) / (sum|left|^2 + sum|right|^2); 0 / 0 is NaN."""
    left, right = split(V)
    a, b = np.sum(np.abs(left) ** 2), np.sum(np.abs(right) ** 2)
    with np.errstate(invalid="ignore"):
        return (a - b) / (a + b)


def spectrum(dspec2, time, freq, npad):
    """(CS, tau, fd) of calc_asymmetry: the chunk padded with its own mean (not 0), fft2,
    fftshift; no tau rows masked."""
    dspec2 = np.asarray(dspec2)
    fd = TO.fft_axis(time, "mHz", npad)
    tau = TO.fft_axis(freq, "us", npad)
    pad = np.pad(dspec2, ((0, npad * dspec2.shape[0]), (0, npad * dspec2.shape[1])),
                 mode="constant", constant_values=dspec2.mean())
    return np.fft.fftshift(np.fft.fft2(pad)), tau, fd


def calc_asymmetry(dspec2, edges, time, freq, eta, npad, return_all=False):
    """Asymmetry of one chunk, NaN where the reference's try/except gives NaN.  With
    ``return_all`` also a dict with thth_red, w and V (None on failure)."""
    CS, tau, fd = spectrum(dspec2, time, freq, npad)
    try:
        thth_red, _, _, _, edges_red, w, V = TO.modeler(CS, tau, fd, eta, edges)
        asymm = asymmetry_of(V)
        extra = dict(thth_red=thth_red, w=w, V=V, edges_red=edges_red)
    except Exception:  # noqa: BLE001  (the reference: print(e); asymm = nan)
        asymm = np.nan
        extra = dict(thth_red=None, w=None, V=None, edges_red=None)
    if return_all:
        return asymm, extra
    return asymm


def chunk_list(dyn, freqs, times, cwf, cwt, ncf, nct, ththeta, fref, edges, npad):
    """The (cf, ct, dspec2, edges, time, freq, eta) list of Dynspec.calc_asymmetry, with its
    time slice ct*cwt//2 : (ct+1)*cwt (widths cwt + ct*cwt/2) and the NaNs of a chunk
    zeroed after its nanmean is subtracted."""
    out = []
    for cf in range(ncf):
        fs = slice(cf * cwf, (cf + 1) * cwf)
        freq2 = np.copy(freqs[fs])
        freq = freq2.mean()
        eta = ththeta * (fref / freq) ** 2
        for ct in range(nct):
            ts = slice(ct * cwt // 2, (ct + 1) * cwt)
            dspec2 = np.copy(dyn[fs, ts])
            dspec2 -= np.nanmean(dspec2)
            dspec2 = np.nan_to_num(dspec2)
            out.append((cf, ct, dspec2, edges * (freq / fref), np.copy(times[ts]), freq2, eta))
    return out


def dynspec_asymmetry(dyn, freqs, times, cwf, cwt, ncf, nct, ththeta, fref, edges, npad):
    """Dynspec.calc_asymmetry: complex [ncf][nct] array of the chunks' asymmetries."""
    res = np.zeros((ncf, nct), dtype=complex)
    for cf, ct, d, e, t, f, eta in chunk_list(dyn, freqs, times, cwf, cwt, ncf, nct, ththeta,
                                              fref, edges, npad):
        res[cf, ct] = calc_asymmetry(d, e, t, f, eta, npad)
    return res
