"""Float64 restatement of Dynspec.correct_dyn and svd_model (reference dynspec.py:3325-3410,
scint_utils.py:705-729, ththmod.py:18-35).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Written from the semantics, not from the
reference's code: the model comes from numpy's thin SVD (full_matrices=False), so no
nt x nt factor is formed, and it is kept real (the reference's is complex with a zero
imaginary part).  ``correct_dyn`` works on any object with the Dynspec attributes it reads
(dyn, and lamdyn / vdyn / vlamdyn when selected) and has the same side effects, so the GPU
tests can use it at sizes the fixtures do not reach.
"""
import numpy as np
from scipy.signal import savgol_filter


def svd_model(arr, nmodes=1):
    """(model, s): the rank-nmodes model of a real 2-D array and all singular values."""
    a = np.asarray(arr, dtype=np.float64)
    u, s, vt = np.linalg.svd(a, full_matrices=False)
    k = min(nmodes, s.size)
    return (u[:, :k] * s[:k]) @ vt[:k], s


def _nanmean_or_nan(x, axis):
    """numpy nanmean without its empty-slice warning (an all-NaN slice gives NaN)."""
    cnt = np.sum(~np.isnan(x), axis=axis)
    tot = np.nansum(x, axis=axis)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(cnt > 0, tot / np.maximum(cnt, 1), np.nan)


def _zeros_to_mean(v):
    v = np.array(v, dtype=np.float64)
    v[v == 0] = np.mean(v)
    return v


def correct_dyn(obj, svd=True, nmodes=1, frequency=True, time=True, lamsteps=False,
                nsmooth=None, velocity=False):
    """Apply correct_dyn to ``obj`` in place (float64).  Sets obj.svd_model (real) or
    obj.bandpass, replaces the selected array and zeroes NaN pixels of the arrays the
    reference mutates.  lamdyn must already exist when lamsteps is set."""
    if lamsteps:
        attr = "vlamdyn" if velocity else "lamdyn"
    else:
        attr = "vdyn" if velocity else "dyn"
    if not hasattr(obj, attr):
        raise ValueError("Need to run scale_dyn with a model")
    arr = getattr(obj, attr)
    arr[np.isnan(arr)] = 0
    if svd:
        model, _ = svd_model(arr, nmodes)
        obj.svd_model = model
        with np.errstate(invalid="ignore", divide="ignore"):
            setattr(obj, attr, arr / np.abs(model))
        return
    # The reference turns zeros of obj.dyn into NaN before each pass and back into zeros
    # at the end.  They are zeros of the selected array only if it is obj.dyn itself.
    missing = (arr == 0) if (arr is obj.dyn and (frequency or time)) else np.zeros(arr.shape, bool)
    x = np.where(missing, np.nan, arr)
    with np.errstate(invalid="ignore", divide="ignore"):
        if frequency:
            obj.bandpass = _zeros_to_mean(_nanmean_or_nan(x, 1))
            bp = savgol_filter(obj.bandpass, nsmooth, 1) if nsmooth is not None else obj.bandpass
            x = x / bp[:, None]
        if time:
            ts = _zeros_to_mean(_nanmean_or_nan(x, 0))
            if nsmooth is not None:
                ts = savgol_filter(ts, nsmooth, 1)
            x = x / ts[None, :]
    main = obj.dyn
    main[np.isnan(main)] = 0
    setattr(obj, attr, x)
