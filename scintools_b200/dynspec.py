"""CUDA-native mirror of the FFT / theta-theta part of scintools.dynspec.

Keeps the ``Dynspec`` method names, signatures and attribute side effects of
the reference for the arc-measurement hot path:

  calc_sspec         dynspec.py:3584-3748  -> sb_sspec_f32
  calc_acf           dynspec.py:3750-3814  -> sb_acf_f32 (+ sspec route)
  prep_thetatheta    dynspec.py:1348-1537  (host bookkeeping, unit free)
  thetatheta_single  dynspec.py:1539-1655  -> sb_cs_f32 + sb_eta_sweep
  fit_thetatheta     dynspec.py:1657-1763  -> per chunk ththmod.single_search

Real data starts here too: ``Dynspec(filename=...)`` reads a psrflux file (load_file,
remove_short_subs, info, auto_processing; dynspec.py:144-257, :422-440, :4130-4143, host
only, with np.loadtxt), ``trim_edges`` (:259-328) takes its zero counts from
sb_dyn_zero_counts_f64 and crops once on the host, ``zap`` (:3856-3870 -> sb_zap_f64) finds
both medians by a radix select on the device, and ``crop_dyn`` (:3816-3854) and ``__add__``
(:81-142) are the reference's indexing on the host.  Not here: write_file, sort_dyn,
plotting, and the lmfit models other than get_scint_params's.
Units: times in s, freqs in MHz, eta in s^3, edges in mHz, tau in us.

Also here: get_scint_params / get_acf_tilt (dynspec.py:2283-3156 -> sb_scint_fit_1d /
sb_scint_fit_2d, batched over spectra by get_scint_params_batch), refill (dynspec.py:3273-3323 -> sb_inpaint_biharmonic_f64 or
sb_medfilt_masked_f64), correct_dyn (dynspec.py:3325-3410 -> sb_svd_topk + sb_svd_apply, or the
sb_bandpass_* passes), scale_dyn('lambda') (dynspec.py:3926-3957 -> sb_scale_dyn_lambda_f32),
thetatheta_chunks / calc_wavefield / gerchberg_saxton (:1765-1896), cut_dyn (:3158-3271 ->
sb_sspec_tiles_f32 + sb_acf_tiles_f32, every tile in one batched pass), and, through
``arcfit.ArcFitMixin``, norm_sspec / fit_arc (:1920-2183, :970-1346), and
calc_scattered_image (:3412-3582 -> sb_scattered_image_f64, batched over spectra by
scattered_image_batch).

Provenance: ``prep_thetatheta`` is the reference's dynspec.py:1348-1537 with the
astropy units stripped, line for line (host scalar bookkeeping that SURVEY.md a11
keeps in Python; identical attributes are the contract).  The chunk loops of
``fit_thetatheta`` / ``thetatheta_chunks`` follow :1680-1712 / :1790-1828 the same
way, and so do load_file, remove_short_subs, info, auto_processing, crop_dyn,
__add__ and trim_edges's bookkeeping.  Restated reference glue, not new design.
"""
import os
import time
from copy import deepcopy as cp

import numpy as np

from . import _device as D
from . import _lib
from . import ththmod as thth
from . import units as U
from .arcfit import ArcFitMixin

_WINDOWS = {"hanning": np.hanning, "hamming": np.hamming,
            "blackman": np.blackman, "bartlett": np.bartlett}


def get_window(nt, nf, window="hanning", frac=0.1):
    """Edge taper (scint_utils.py:810-832): returns (chan_window[nt],
    subint_window[nf]) -- the first one runs along the TIME axis."""
    try:
        fn = _WINDOWS[window.lower()]
    except KeyError:
        raise ValueError("Window unknown.. Please add it!")
    cw = fn(int(np.floor(frac * nt)))
    sw = fn(int(np.floor(frac * nf)))
    chan_window = np.insert(cw, int(np.ceil(len(cw) / 2)),
                            np.ones([nt - len(cw)]))
    subint_window = np.insert(sw, int(np.ceil(len(sw) / 2)),
                              np.ones([nf - len(sw)]))
    return chan_window, subint_window


def is_valid(array):
    """scint_utils.py:87-91."""
    return np.isfinite(array) * (~np.isnan(array))


# ----------------------------------------------------------------------
# gap filling (csrc/inpaint.cu)
# ----------------------------------------------------------------------
_FILL_MAX_NF, _FILL_MAX_NT = 32768, 16384
_MEDFILT_MAX_SIDE = 31


def _fill_check(image, mask):
    """ValueError, before any device work, for what the gap fills do not take."""
    if image.ndim != 2 or mask.shape != image.shape:
        raise ValueError("need a 2-D image and a mask of its shape")
    nf, nt = image.shape
    if not (1 <= nf <= _FILL_MAX_NF and 1 <= nt <= _FILL_MAX_NT):
        raise ValueError("shape %s is outside 1..%d x 1..%d" % (image.shape, _FILL_MAX_NF,
                                                                  _FILL_MAX_NT))
    if np.any(np.isinf(image)):
        raise ValueError("the image has an infinite pixel")
    if np.all(mask):
        raise ValueError("every pixel is masked: nothing to fill from")


def _axis_classes(n):
    """Class of every index along an axis of length n: the (extent, centre offset) of the
    5-point window [i-2, i+2] clipped to [0, n).  Returns (cls uint8 [n], [(extent, offset)])."""
    i = np.arange(n)
    lo = np.maximum(i - 2, 0)
    key = np.minimum(i + 3, n) - lo, i - lo
    kinds = sorted(set(zip(*(k.tolist() for k in key))))
    index = {k: c for c, k in enumerate(kinds)}
    return np.array([index[k] for k in zip(*(k.tolist() for k in key))], np.uint8), kinds


def _stencil_tables(nf, nt):
    """Stencils of the biharmonic system, S = laplace(laplace(e_p)) on the clipped 5x5 box
    (scipy.ndimage, mode 'reflect'), one per pair of row and column classes, centred on the
    pixel: tables float64 [nrc][ncc][5][5], zero outside the box."""
    from scipy.ndimage import laplace
    rcls, rk = _axis_classes(nf)
    ccls, ck = _axis_classes(nt)
    tables = np.zeros((len(rk), len(ck), 5, 5))
    for a, (er, orow) in enumerate(rk):
        for c, (ec, ocol) in enumerate(ck):
            box = np.zeros((er, ec))
            box[orow, ocol] = 1.0
            tables[a, c, 2 - orow:2 - orow + er, 2 - ocol:2 - ocol + ec] = laplace(laplace(box))
    return rcls, ccls, tables


def _biharmonic_values(image, mask, tol, maxit):
    """Inpainted values at the masked pixels, in row-major order, and the solver info."""
    import torch
    nf, nt = image.shape
    pix = np.flatnonzero(mask).astype(np.int32)
    known = image[~mask]
    rcls, ccls, tables = _stencil_tables(nf, nt)
    d_img = D.upload(np.ascontiguousarray(image, dtype=np.float64))
    d_pix, d_tab = D.upload(pix), D.upload(tables)
    d_rc, d_cc = D.upload(rcls), D.upload(ccls)
    out = D.empty((pix.size,), torch.float64)
    info = np.zeros(3, np.int32)
    resid = np.zeros(1)
    _lib.check(_lib.lib.sb_inpaint_biharmonic_f64(
        d_img.data_ptr(), nf, nt, d_pix.data_ptr(), pix.size, d_tab.data_ptr(),
        d_rc.data_ptr(), tables.shape[0], d_cc.data_ptr(), tables.shape[1],
        float(known.min()), float(known.max()), float(tol), int(maxit), out.data_ptr(),
        info.ctypes.data, resid.ctypes.data, D.stream_ptr()))
    info = {"iterations": int(info[0]), "residual": float(resid[0]),
            "converged": bool(info[1]), "restarts": int(info[2])}
    if not info["converged"]:
        import warnings
        warnings.warn("biharmonic inpainting stopped after %d iterations at relative residual "
                      "%.3g (tol %.3g)" % (info["iterations"], info["residual"], tol),
                      RuntimeWarning, stacklevel=3)
    return D.download(out), info


def inpaint_biharmonic(image, mask, return_info=False, tol=1e-10, maxit=50000):
    """Biharmonic inpainting of the pixels where mask is non-zero: skimage >= 0.19's
    ``restoration.inpaint_biharmonic(image, mask, split_into_regions=False)`` for a 2-D
    image, solved on the device.

    One unknown per masked pixel; its equation is the stencil laplace(laplace(e_p))
    (scipy.ndimage, mode 'reflect') on the 5x5 box around it clipped to the image, with the
    known pixels moved to the right-hand side.  The system is solved matrix-free by
    BiCGSTAB with Jacobi scaling in float64 until ||b - A x|| <= tol ||b||, or for at most
    ``maxit`` steps; the result is clipped to [min, max] of the known pixels.  Returns a
    float64 copy of the image with the masked pixels filled, and with return_info=True also
    a dict: iterations, residual (the final ||b - A x|| / ||b||), converged, restarts.  A
    solve that stops at the cap warns (RuntimeWarning) and still returns its result.

    ValueError, before any device work: an image that is not 2-D, a mask of another shape,
    a shape outside 1..32768 x 1..16384, an infinite pixel (the deviation from skimage:
    there the result depends on SuperLU's elimination order), a NaN pixel that is not
    masked, or a mask that covers every pixel.  No masked pixel: the copy, 0 iterations."""
    image = np.array(image, dtype=np.float64)
    mask = np.asarray(mask).astype(bool)
    _fill_check(image, mask)
    if np.any(np.isnan(image[~mask])):
        raise ValueError("the image has a NaN pixel outside the mask")
    info = {"iterations": 0, "residual": 0.0, "converged": True, "restarts": 0}
    if np.any(mask):
        vals, info = _biharmonic_values(image, mask, tol, maxit)
        image[mask] = vals
    return (image, info) if return_info else image


def _median_values(image, mask, kernel_size, nan_value):
    """scipy.signal.medfilt(image with NaN read as nan_value, kernel_size) at the masked
    pixels, in row-major order."""
    import torch
    nf, nt = image.shape
    pix = np.flatnonzero(mask).astype(np.int32)
    kh, kw = kernel_size
    d_img = D.upload(np.ascontiguousarray(image, dtype=np.float64))
    d_pix = D.upload(pix)
    out = D.empty((pix.size,), torch.float64)
    _lib.check(_lib.lib.sb_medfilt_masked_f64(d_img.data_ptr(), nf, nt, d_pix.data_ptr(),
                                              pix.size, kh, kw, float(nan_value),
                                              out.data_ptr(), D.stream_ptr()))
    return D.download(out)


def _medfilt_size(kernel_size):
    """medfilt's kernel_size for a 2-D array: a scalar or one size per axis, each odd."""
    ks = np.asarray(kernel_size)
    if ks.shape == ():
        ks = np.repeat(ks, 2)
    if ks.shape != (2,) or not np.issubdtype(ks.dtype, np.integer):
        raise ValueError("kernel_size must be an integer or two integers")
    for k in ks:
        if k % 2 != 1:
            raise ValueError("Each element of kernel_size should be odd.")
        if not 1 <= k <= _MEDFILT_MAX_SIDE:
            raise ValueError("kernel sizes above %d are not supported" % _MEDFILT_MAX_SIDE)
    return int(ks[0]), int(ks[1])


# ----------------------------------------------------------------------
# scintillation scales (csrc/scintfit.cu)
# ----------------------------------------------------------------------
_ACF_MIN_NF, _ACF_MAX_NF, _ACF_MIN_NT, _ACF_MAX_NT = 2, 32768, 5, 16384
_SLOTS = ("tau", "dnu", "amp", "alpha", "phasegrad")
_FIT_STATUS = {1: "converged", 2: "converged (no decrease left at float64 precision)",
               -1: "stopped at max_nfev", -2: "non-finite residual"}


class FitParam:
    """One fitted parameter: value, and stderr (None where not estimated)."""

    def __init__(self, name, value, stderr=None, vary=True):
        self.name, self.value, self.stderr, self.vary = name, value, stderr, vary

    def __repr__(self):
        return "<FitParam %s = %r +/- %r>" % (self.name, self.value, self.stderr)


class ScintFitResult:
    """What get_scint_params returns: the fields callers of the reference read from
    lmfit's MinimizerResult.  params[name].value / .stderr, chisqr, redchi = chisqr /
    (ndata - nvarys), ndata (every residual, zero-weight ones included, as lmfit counts),
    nvarys, nfev (model evaluations; each also gives the analytic Jacobian), success (False
    when the fit stopped at max_nfev), message, init_values (the starting values of the
    varying parameters)."""

    def __init__(self, params, chisqr, ndata, nvarys, nfev, status, method, init_values):
        self.params = params
        self.init_values = init_values
        self.chisqr = chisqr
        self.ndata = ndata
        self.nvarys = nvarys
        self.redchi = chisqr / max(1, ndata - nvarys)
        self.nfev = nfev
        self.status = status
        self.success = status > 0
        self.message = _FIT_STATUS.get(status, "status %d" % status)
        self.method = method

    def report(self):
        """Plain-text summary (not lmfit's fit_report layout)."""
        lines = ["[[Fit: %s, Levenberg-Marquardt on the device]]" % self.method,
                 "    %s after %d evaluations" % (self.message, self.nfev),
                 "    data points = %d, variables = %d" % (self.ndata, self.nvarys),
                 "    chi-square = %.10g, reduced chi-square = %.10g" % (self.chisqr, self.redchi),
                 "[[Variables]]"]
        for p in self.params.values():
            if not p.vary:
                lines.append("    %-10s %.10g (fixed)" % (p.name + ":", p.value))
            elif p.stderr is None:
                lines.append("    %-10s %.10g +/- (not estimated)" % (p.name + ":", p.value))
            else:
                lines.append("    %-10s %.10g +/- %.4g" % (p.name + ":", p.value, p.stderr))
        return "\n".join(lines)


def _scint_args_check(method, plot, mcmc, nan_policy):
    if plot:
        raise NotImplementedError("plotting is outside the GPU path")
    if mcmc:
        raise NotImplementedError("mcmc sampling is outside the GPU path")
    if method == 'acf2d':
        raise NotImplementedError("method='acf2d' (the fit of the scint_sim.ACF model) is "
                                  "not ported")
    if method == 'sspec':
        raise NotImplementedError("method='sspec' does not work in the reference either")
    if method not in ('nofit', 'acf1d', 'acf2d_approx'):
        raise ValueError("method must be 'nofit', 'acf1d' or 'acf2d_approx'")
    if nan_policy != 'raise':
        raise NotImplementedError("only nan_policy='raise' is supported")


def _scint_shape_check(ds):
    nf, nt = np.shape(ds.dyn)
    if not (_ACF_MIN_NF <= nf <= _ACF_MAX_NF and _ACF_MIN_NT <= nt <= _ACF_MAX_NT):
        raise ValueError("dynspec %d x %d is outside the supported sizes (nf %d..%d, nt %d..%d)"
                         % (nf, nt, _ACF_MIN_NF, _ACF_MAX_NF, _ACF_MIN_NT, _ACF_MAX_NT))
    if hasattr(ds, 'acf') and np.shape(ds.acf) != (2 * nf, 2 * nt):
        raise ValueError("self.acf has shape %s, not 2 x %s" % (np.shape(ds.acf), (nf, nt)))


def _acf_stacks(dynspecs):
    """One float64 device stack [n][2 nf][2 nt] per (nf, nt) group: the ACF a Dynspec holds
    is uploaded into its slice; a missing one is made by the ACF driver into a float32
    slice, widened on the device and stored as self.acf, as calc_acf would.  Returns
    {id(ds): (stack, slice index)}."""
    import torch
    groups = {}
    for ds in dynspecs:
        groups.setdefault(np.shape(ds.dyn), []).append(ds)
    where = {}
    for (nf, nt), members in groups.items():
        stack = D.empty((len(members), 2 * nf, 2 * nt), torch.float64)
        tmp = None
        for k, ds in enumerate(members):
            if hasattr(ds, 'acf'):
                stack[k].copy_(torch.from_numpy(np.ascontiguousarray(ds.acf, dtype=np.float64)))
            else:
                if tmp is None:
                    tmp = D.empty((2 * nf, 2 * nt), torch.float32)
                d = D.upload_f32(np.asarray(ds.dyn))
                _lib.check(_lib.lib.sb_acf_f32(d.data_ptr(), nf, nt, 1, 1, tmp.data_ptr(),
                                               D.stream_ptr()))
                _lib.check(_lib.lib.sb_convert_f32_f64(tmp.data_ptr(), stack[k].data_ptr(),
                                                       tmp.numel(), D.stream_ptr()))
                ds.acf = D.download(stack[k])
            where[id(ds)] = (stack, k)
    return where


def _contiguous_prefix(inds, n):
    """(count) of a crop index vector that must be 0, 1, ..., count - 1."""
    inds = np.atleast_1d(inds)
    if inds.size == 0 or not np.array_equal(inds, np.arange(inds.size)) or inds.size > n:
        raise ValueError("the ACF cut crop is not a prefix of the lags (negative dt or df?)")
    return inds.size


def _scint_nofit(ds, full_frame, nscale, bartlett, weighted):
    """The reference's host steps up to the first fit (dynspec.py:2575-2687), on ds.acf:
    initial guesses, crops, the nofit attributes and the 1-D weights.  Returns the 1-D plan."""
    acf = ds.acf
    nf, nt = np.shape(acf)
    ydata_f = acf[int(nf/2):, int(nt/2)]
    xdata_f = ds.df * np.linspace(0, len(ydata_f)-1, len(ydata_f))
    ydata_t = acf[int(nf/2), int(nt/2):]
    xdata_t = ds.dt * np.linspace(0, len(ydata_t)-1, len(ydata_t))

    wn = min([ydata_f[0]-ydata_f[1], ydata_t[0]-ydata_t[1]])
    amp = max([ydata_f[0] - wn, ydata_t[0] - wn])
    if np.argwhere(ydata_t < amp/np.e).squeeze().size == 0:
        tau = ds.dt if ydata_t[1] < 0 else ds.tobs
    else:
        tau = xdata_t[np.argwhere(ydata_t < amp/np.e).squeeze()[0]]
    if np.argwhere(ydata_f < amp/2).squeeze().size == 0:
        dnu = ds.df if ydata_f[1] < 0 else ds.bw
    else:
        dnu = xdata_f[np.argwhere(ydata_f < amp/2).squeeze()[0]]

    if not full_frame:
        t_inds = np.argwhere(xdata_t <= nscale*tau).squeeze()
        f_inds = np.argwhere(xdata_f <= nscale*dnu).squeeze()
        if nscale*tau <= 5*ds.dt:
            t_inds = np.argwhere(xdata_t <= 5*ds.dt).squeeze()
        if nscale*dnu <= 5*ds.df:
            f_inds = np.argwhere(xdata_f <= 5*ds.df).squeeze()
        nt_c = _contiguous_prefix(t_inds, len(xdata_t))
        nf_c = _contiguous_prefix(f_inds, len(xdata_f))
        xdata_t = xdata_t[t_inds]
        ydata_t = ydata_t[t_inds]
        xdata_f = xdata_f[f_inds]
        ydata_f = ydata_f[f_inds]
    else:
        nt_c, nf_c = len(xdata_t), len(xdata_f)

    ds.tau = tau
    ds.dnu = dnu
    ds.amp = amp
    ds.wn = wn

    tau_half = xdata_t[np.argmin(abs(ydata_t - amp/2))]
    if tau_half < ds.dt:
        tau_half = ds.dt
    elif tau_half > ds.tobs:
        tau_half = ds.tobs
    nscint = (1 + 0.2*ds.bw/(ds.dnu)) * (1 + 0.2*ds.tobs/(tau_half))
    ds.dnuerr = dnu / np.sqrt(nscint)
    ds.tauerr = tau / np.sqrt(nscint)
    ds.amperr = amp / np.sqrt(nscint)
    ds.wnerr = wn / np.sqrt(nscint)
    ds.tscat = 1/(2*np.pi*ds.dnu)
    ds.nscint = nscint
    ds.scint_param_method = 'nofit'

    valid = ds.dyn[is_valid(ds.dyn) * (ds.dyn != 0)]
    mean = np.mean(valid)
    flux_var_est = mean**2
    flux_var = np.var(valid)
    ds.dnu_est = ds.df * (flux_var/flux_var_est - 1)
    if ds.dnu_est < 0:
        ds.dnu_est = 0
    ds.dnu_esterr = ds.dnu_est / np.sqrt(nscint)
    if ds.dnu_est > 0:
        ds.tscat_est = 1/(2*np.pi*ds.dnu_est)
    else:
        ds.tscat_est = 0
    ds.modulation_index = np.sqrt(flux_var)/mean

    t_errors = np.ones(np.shape(xdata_t))/np.sqrt((nt/2))
    t_errors[0] = 1e-3
    f_errors = np.ones(np.shape(xdata_f))/np.sqrt((nf/2))
    f_errors[0] = 1e-3
    if bartlett:
        var_t = np.ones(np.shape(ydata_t)) / (nt / 2)
        var_t[0] = 1e-10
        var_t[2:] *= 1 + 2 * np.cumsum(ydata_t[1:-1] ** 2)
        t_errors = np.sqrt(var_t)
        var_f = np.ones(np.shape(ydata_f)) / (nf / 2)
        var_f[0] = 1e-10
        var_f[2:] *= 1 + 2 * np.cumsum(ydata_f[1:-1] ** 2)
        f_errors = np.sqrt(var_f)
    weights_t = 1/t_errors if weighted else np.ones(np.shape(ydata_t))
    weights_f = 1/f_errors if weighted else np.ones(np.shape(ydata_f))
    return dict(tau=tau, dnu=dnu, amp=amp, nt_c=nt_c, nf_c=nf_c, xdata_t=xdata_t,
                xdata_f=xdata_f, ydata_t=ydata_t, ydata_f=ydata_f, weights_t=weights_t,
                weights_f=weights_f)


def _fftshift_positions(n):
    """Along one axis of length n, where the reference's weight shifts put things
    (dynspec.py:2785-2789 and scint_models.py:156-158): the roll sh of the weights
    (fftshift twice maps the weight of index (k + sh) mod n to index k), the index that
    gets 1e10, and the index the model zeroes."""
    ar = np.arange(n)
    perm = np.fft.fftshift(np.fft.fftshift(ar))
    sh = int(perm[0])
    assert np.array_equal(perm, (ar + sh) % n)
    m = np.zeros(n)
    m[0] = 1
    p = int(np.argmax(np.fft.fftshift(m)))
    m = np.zeros(n)
    m[-1] = 1
    z = int(np.argmax(np.fft.ifftshift(m)))
    return sh, p, z


def _scint_crop_2d(ds, tau, dnu, nscale, full_frame, verbose):
    """The 2-D crop of dynspec.py:2716-2783, as index vectors into ds.acf: returns (rows,
    cols, tticks, fticks), rows / cols contiguous."""
    nf, nt = np.shape(ds.acf)
    tticks = np.linspace(-ds.tobs, ds.tobs, nt + 1)[:-1]
    fticks = np.linspace(-ds.bw, ds.bw, nf + 1)[:-1]
    wn_loc = np.unravel_index(np.argmax(ds.acf, axis=None), ds.acf.shape)
    fleft = wn_loc[0]
    fright = nf - wn_loc[0] - 1
    fmin = wn_loc[0] - min(fleft, fright)
    fmax = wn_loc[0] + min(fleft, fright) + 1
    tleft = wn_loc[1]
    tright = nt - wn_loc[1] - 1
    tmin = wn_loc[1] - min(tleft, tright)
    tmax = wn_loc[1] + min(tleft, tright) + 1
    rows = np.arange(nf)[fmin:fmax]
    cols = np.arange(nt)[tmin:tmax]
    if nscale is not None and not full_frame:
        ntau = nscale
        ndnu = nscale
        if ntau > (ds.tobs / tau):
            if verbose:
                print('WARNING: nscale exceeds range in time lag')
            tmin = 0
            tmax = nt
        else:
            tframe = int(round(ntau * (tau / ds.dt)))
            tmin = int(np.floor(len(cols) / 2)) - tframe
            tmax = int(np.floor(len(cols) / 2)) + tframe + 1
        if ndnu > (ds.bw / dnu):
            if verbose:
                print('WARNING: nscale exceeds range in frequency lag')
            # the reference sets the time bounds here (dynspec.py:2766-2767)
            tmin = 0
            tmax = nf
        else:
            fframe = int(round(ndnu * (dnu / ds.df)))
            fmin = int(np.floor(len(rows) / 2)) - fframe
            fmax = int(np.floor(len(rows) / 2)) + fframe + 1
        rows = rows[fmin:fmax]
        cols = cols[tmin:tmax]
    if rows.size == 0 or cols.size == 0:
        raise ValueError("the 2-D ACF crop is empty")
    return rows, cols, tticks, fticks


def _acf2d_model(p, tdata, fdata, tobs, bw):
    """scint_acf_model_2d_approx's model (scint_models.py:123-161) at the parameters p
    (dict), as [nf][nt], before the weights."""
    amp, dnu, tau, alpha = p['amp'], p['dnu'], p['tau'], p['alpha']
    mu = p['phasegrad']*60
    t = np.reshape(tdata, (len(tdata), 1))
    f = np.reshape(fdata, (1, len(fdata)))
    model = amp * np.exp(-(abs((t - mu*f)/tau)**(3 * alpha / 2) +
                         abs(f / (dnu / np.log(2)))**(3 / 2))**(2 / 3))
    model = np.multiply(model, 1-np.divide(abs(t), tobs))
    model = np.multiply(model, 1-np.divide(abs(f), bw))
    return np.transpose(model)


def _run_fits(kind, descs):
    """One batched fit (sb_scint_fit_1d / _2d, synchronous) of the ScintFit descriptors;
    returns (out [n][11], info [n][2]) on the host."""
    import torch
    n = len(descs)
    arr = (_lib.ScintFit * n)(*descs)
    out = D.empty((n, 11), torch.float64)
    info = D.empty((n, 2), torch.int32)
    fn = _lib.lib.sb_scint_fit_1d if kind == 1 else _lib.lib.sb_scint_fit_2d
    _lib.check(fn(arr, n, out.data_ptr(), info.data_ptr(), D.stream_ptr()))
    return D.download(out), D.download(info)


def _result(out, info, desc, names, fixed, ndata, method):
    vary = desc.vary
    params = {}
    for s, name in enumerate(_SLOTS):
        if name not in names:
            continue
        v = bool((vary >> s) & 1)
        err = float(out[5 + s]) if v and np.isfinite(out[5 + s]) else None
        params[name] = FitParam(name, float(out[s]), err, v)
    for name, value in fixed.items():
        params[name] = FitParam(name, value, None, False)
    init = {n: float(desc.p0[s]) for s, n in enumerate(_SLOTS) if (vary >> s) & 1}
    return ScintFitResult(params, float(out[10]), int(ndata), bin(vary).count("1"),
                          int(info[0]), int(info[1]), method, init)


def _check_status(res, what):
    if res.status == -2:
        raise ValueError("%s: the fit met a non-finite residual (NaN values detected in the "
                         "output of the model function)" % what)


def get_scint_params_batch(dynspecs, method='acf1d', **kwargs):
    """Dynspec.get_scint_params on each Dynspec of the list, with the fits of all of them
    batched on the device: sets on each exactly what get_scint_params(**kwargs) would set on
    it alone and returns the list of results (None for method='nofit').  The objects are
    grouped by the shape of their dynamic spectrum; each group's ACFs form one device stack,
    and each group's fits run as one batch.  Keyword arguments as get_scint_params."""
    import torch
    a = dict(plot=False, alpha=5/3, mcmc=False, full_frame=False, nscale=5, verbose=False,
             nan_policy='raise', weighted=True, tau_vary_2d=True, tau_input=None,
             bartlett=True, get_fit_report=True)
    ignored = ('nwalkers', 'steps', 'burn', 'nitr', 'lnsigma', 'progress', 'display',
               'filename', 'dpi', 'workers')
    for k in kwargs:
        if k not in a and k not in ignored:
            raise TypeError("get_scint_params() got an unexpected keyword argument '%s'" % k)
    a.update({k: v for k, v in kwargs.items() if k in a})
    _scint_args_check(method, a['plot'], a['mcmc'], a['nan_policy'])
    dynspecs = list(dynspecs)
    for ds in dynspecs:
        _scint_shape_check(ds)
    alpha, verbose, weighted = a['alpha'], a['verbose'], a['weighted']
    if method == 'nofit':
        for ds in dynspecs:
            if not hasattr(ds, 'acf'):
                ds.calc_acf()
            _scint_nofit(ds, a['full_frame'], a['nscale'], a['bartlett'], weighted)
        return [None] * len(dynspecs)
    # the host steps, and every check they make, come before the device work on an ACF the
    # object already holds; a missing ACF is made first
    where = _acf_stacks([ds for ds in dynspecs if not hasattr(ds, 'acf')])
    plans = [_scint_nofit(ds, a['full_frame'], a['nscale'], a['bartlett'], weighted)
             for ds in dynspecs]
    for pl in plans:
        for nm, y in (("time", pl['ydata_t']), ("frequency", pl['ydata_f'])):
            if not np.all(np.isfinite(y)):
                raise ValueError("the ACF %s cut has non-finite values (NaN values detected in "
                                 "the input data)" % nm)
    crops = []
    if method == 'acf2d_approx':
        for ds, pl in zip(dynspecs, plans):
            rows, cols, tticks, fticks = _scint_crop_2d(ds, pl['tau'], pl['dnu'], a['nscale'],
                                                        a['full_frame'], verbose)
            box = ds.acf[rows[0]:rows[-1] + 1, cols[0]:cols[-1] + 1]
            if not np.all(np.isfinite(box)):
                raise ValueError("the 2-D ACF crop has non-finite values (NaN values detected "
                                 "in the input data)")
            crops.append((rows, cols, tticks, fticks))
    where.update(_acf_stacks([ds for ds in dynspecs if id(ds) not in where]))

    # ---- 1-D fit (dynspec.py:2651-2708) ----
    vary1 = 0b111 | (0b1000 if alpha is None else 0)
    descs, keep = [], []
    for ds, pl in zip(dynspecs, plans):
        if verbose:
            print('Initial guesses:', '\ntau:', pl['tau'], '\ndnu:', pl['dnu'],
                  '\namp:', pl['amp'])
            if method == 'acf2d_approx':
                print("\nInitialising model with 1D fit")
            else:
                print("\nPerforming least-squares fit to 1D ACF model")
        stack, k = where[id(ds)]
        nf2, nt2 = stack.shape[1:]
        w = D.upload(np.concatenate((pl['weights_t'], pl['weights_f'])).astype(np.float64))
        keep.append(w)
        d = _lib.ScintFit()
        d.acf = stack[k].data_ptr()
        d.aux = w.data_ptr()
        d.pitch = nt2
        d.s0, d.s1 = float(ds.dt), float(ds.df)
        p0 = [max(pl['tau'], 0.0), max(pl['dnu'], 0.0), max(pl['amp'], 0.0),
              5/3 if alpha is None else alpha, 0.0]
        d.p0 = (_lib.c_dbl * 5)(*[float(v) for v in p0])
        d.r0, d.c0, d.n0 = nf2 // 2, nt2 // 2, pl['nt_c']
        d.r1, d.c1, d.n1 = nf2 // 2, nt2 // 2, pl['nf_c']
        d.vary, d.bounded, d.weighted = vary1, 0b111, 1
        d.max_nfev = 10000 * (4 + 1)
        descs.append(d)
    out, info = _run_fits(1, descs)
    names1 = ("tau", "dnu", "amp", "alpha")
    results = []
    for i, (ds, pl) in enumerate(zip(dynspecs, plans)):
        fixed = {'nt': np.shape(ds.acf)[1], 'nf': np.shape(ds.acf)[0]}
        r = _result(out[i], info[i], descs[i], names1, fixed, pl['nt_c'] + pl['nf_c'], 'acf1d')
        _check_status(r, "1-D fit")
        results.append(r)

    # ---- 2-D fit (dynspec.py:2710-2841) ----
    if method == 'acf2d_approx':
        descs, keep, cuts = [], [], []
        vary2 = 0b10110 | (0b1000 if alpha is None else 0) | (1 if a['tau_vary_2d'] else 0)
        for i, (ds, pl) in enumerate(zip(dynspecs, plans)):
            r1 = results[i]
            p0 = {'tau': pl['tau'], 'dnu': pl['dnu'], 'amp': pl['amp']}
            if r1.params['dnu'].stderr is not None:
                p0 = {n: r1.params[n].value for n in ('tau', 'dnu', 'amp')}
            if a['tau_input'] is not None:
                p0['tau'] = a['tau_input']
            p0['alpha'] = 5/3 if alpha is None else alpha
            p0['phasegrad'] = 0.0
            if hasattr(ds, 'acf_tilt') and ds.acf_tilt_err is not None:
                p0['phasegrad'] = ds.acf_tilt
            rows, cols, tticks, fticks = crops[i]
            at = (ds.tobs - abs(tticks)) / max(tticks)
            af = (ds.bw - abs(fticks)) / max(fticks)
            tdata, fdata = tticks[cols], fticks[rows]
            aux = D.upload(np.concatenate((tdata, fdata, at[cols], af[rows])).astype(np.float64))
            keep.append(aux)
            shf, pf, zf = _fftshift_positions(len(rows))
            sht, pt, zt = _fftshift_positions(len(cols))
            stack, k = where[id(ds)]
            d = _lib.ScintFit()
            d.acf = stack[k].data_ptr()
            d.aux = aux.data_ptr()
            d.pitch = stack.shape[2]
            d.s0, d.s1, d.c = float(ds.tobs), float(ds.bw), float(ds.nsub * ds.nchan)
            vals = [p0[n] for n in _SLOTS]
            for s in range(3):
                if (vary2 >> s) & 1:
                    vals[s] = max(vals[s], 0.0)
            d.p0 = (_lib.c_dbl * 5)(*[float(v) for v in vals])
            d.r0, d.c0, d.n0, d.n1 = int(rows[0]), int(cols[0]), len(rows), len(cols)
            d.shf, d.sht, d.pf, d.pt, d.zf, d.zt = shf, sht, pf, pt, zf, zt
            d.vary, d.bounded, d.weighted = vary2, 0b111, 1 if weighted else 0
            d.max_nfev = 10000 * ((4 if alpha is not None else 5) + 1)
            descs.append(d)
            cuts.append((tdata, fdata))
            if verbose:
                print("\nPerforming least-squares fit to approximate 2D ACF model")
        out, info = _run_fits(2, descs)
        for i, ds in enumerate(dynspecs):
            fixed = {'nt': np.shape(ds.acf)[1], 'nf': np.shape(ds.acf)[0], 'tobs': ds.tobs,
                     'bw': ds.bw, 'freq': ds.freq}
            nd = descs[i].n0 * descs[i].n1
            r = _result(out[i], info[i], descs[i], _SLOTS, fixed, nd, 'acf2d_approx')
            _check_status(r, "2-D fit")
            results[i] = r
        for ds, r, (tdata, fdata) in zip(dynspecs, results, cuts):
            ds._scint_crop = (tdata, fdata)
    for ds, r in zip(dynspecs, results):
        _scint_finish(ds, r, method, alpha, verbose, a['get_fit_report'])
    torch.cuda.current_stream().synchronize()
    return results


def _scint_finish(ds, results, method, alpha, verbose, get_fit_report):
    """The reference's attributes after the fit (dynspec.py:2946-3049)."""
    if results.params['tau'].stderr is None or \
       results.params['dnu'].stderr is None:
        print("\n Warning: Could not estimate uncertainties")
    elif (results.params['tau'].stderr > results.params['tau'].value or
          results.params['dnu'].stderr > results.params['dnu'].value):
        print("\n Warning: Parameters unconstrained")
    ds.scint_param_method = method
    if get_fit_report:
        ds.report = results.report()
        if verbose:
            print("===== Fit Report Below =====")
            print(ds.report)
            print(" ")
    ds.tau = results.params['tau'].value
    ds.dnu = results.params['dnu'].value
    ds.tscat = 1/(2*np.pi*ds.dnu)
    if ds.dnu < ds.df:
        print("Warning: Scint bandwidth < channel bandwidth.")
    nscint = (1 + 0.2*ds.bw/(ds.dnu)) * (1 + 0.2*ds.tobs/(ds.tau*np.log(2)))
    ds.nscint = nscint
    ds.fse_tau = ds.tau/(2*np.sqrt(nscint))
    fit_tau = results.params['tau'].stderr
    ds.fse_dnu = ds.dnu/(2*np.sqrt(nscint))
    fit_dnu = results.params['dnu'].stderr
    if verbose:
        print("\nFinite scintle errors (tau, dnu):\n", ds.fse_tau, ds.fse_dnu)
        print("\nFit errors (tau, dnu):\n", fit_tau, fit_dnu)
    if fit_dnu is None:
        fit_dnu = np.inf
    if fit_tau is None:
        fit_tau = np.inf
    ds.tauerr = np.sqrt(fit_tau**2 + ds.fse_tau**2)
    ds.dnuerr = np.sqrt(fit_dnu**2 + ds.fse_dnu**2)
    ds.amp = results.params['amp'].value
    ds.amperr = results.params['amp'].stderr
    ds.wn = 1 - ds.amp
    if 'sim:mb2=' in ds.name:
        ds.wn = 0
    if alpha is None:
        ds.talpha = results.params['alpha'].value
        ds.talphaerr = results.params['alpha'].stderr
    else:
        ds.talpha = alpha
        ds.talphaerr = 0
    if method == 'acf2d_approx':
        tdata, fdata = ds.__dict__.pop('_scint_crop')
        p = {n: results.params[n].value for n in _SLOTS}
        model = _acf2d_model(p, tdata, fdata, ds.tobs, ds.bw)
        weights = np.ones(np.shape(model))
        weights = np.fft.fftshift(weights)
        weights[-1, -1] = 0
        weights = np.fft.ifftshift(weights)
        ds.acf_model = -((np.zeros(np.shape(model)) - model) * weights)
        ds.phasegrad = results.params['phasegrad'].value
        fit_ph = results.params['phasegrad'].stderr
        if fit_ph is None:
            fit_ph = np.inf
        fse_ph = ds.phasegrad * np.sqrt((ds.fse_dnu/ds.dnu)**2 + (ds.fse_tau/ds.tau)**2)
        ds.phasegraderr = fit_ph
        ds.fse_phasegrad = fse_ph
    if verbose:
        print("\n\t ACF FIT PARAMETERS\n")
        print("tau:\t\t\t{val} +/- {err} s".format(val=ds.tau, err=ds.tauerr))
        print("dnu:\t\t\t{val} +/- {err} MHz".format(val=ds.dnu, err=ds.dnuerr))
        if alpha is None:
            print("alpha:\t\t\t{val} +/- {err}".format(val=ds.talpha, err=ds.talphaerr))
        if method == 'acf2d_approx':
            err = np.sqrt(ds.phasegraderr**2 + fse_ph**2)
            print("phase grad:\t\t{val} +/- {err}".format(val=ds.phasegrad, err=err))


def _cut_dyn_device(dyn, fnum, tnum, nfc, ntc, dtype):
    """Secondary spectra [nfc][ntc][nrfft/2][ncfft] and ACFs [nfc][ntc][2 fnum][2 tnum] of
    the fnum x tnum tiles of dyn [nfc fnum][ntc tnum] (Dynspec.cut_dyn), as dtype."""
    import torch
    nrfft = int(2 ** (np.ceil(np.log2(fnum)) + 1))
    ncfft = int(2 ** (np.ceil(np.log2(tnum)) + 1))
    chan_window, subint_window = get_window(tnum, fnum, window='hanning', frac=0.1)
    d = D.upload_f32(dyn)
    wt = D.upload(chan_window.astype(np.float32))
    wf = D.upload(subint_window.astype(np.float32))
    sec = D.empty((nfc, ntc, nrfft // 2, ncfft), torch.float32)
    acf = D.empty((nfc, ntc, 2 * fnum, 2 * tnum), torch.float32)
    _lib.check(_lib.lib.sb_sspec_tiles_f32(
        d.data_ptr(), nfc * fnum, ntc * tnum, fnum, tnum, nfc, ntc, wt.data_ptr(),
        wf.data_ptr(), float(chan_window.sum()), float(subint_window.sum()), sec.data_ptr(),
        D.stream_ptr()))
    _lib.check(_lib.lib.sb_acf_tiles_f32(
        d.data_ptr(), nfc * fnum, ntc * tnum, fnum, tnum, nfc, ntc, acf.data_ptr(),
        D.stream_ptr()))
    return D.download(sec, dtype), D.download(acf, dtype)


# ----------------------------------------------------------------------
# scattered image (csrc/scatim.cu)
# ----------------------------------------------------------------------
# sizes the device takes (include/scint_b200_scatim.h)
_SCATIM_MIN_M = 4
_SCATIM_MAX_MX, _SCATIM_MAX_MY = 65536, 32768     # crop box: delays, Doppler columns
_SCATIM_MAX_SAMPLING = 4096
_SCATIM_MAX_ITEMS = 65535
_SCATIM_GROUP_BYTES = 4 << 30   # device memory of one batched pass, coefficients and images
_SCATIM_TABLES = {}             # sha256 of an axis -> (knots, band factors)


def spline_knots(x):
    """The knots RectBivariateSpline(..., s=0) puts on the axis x: [x0]*4 + x[2:-2] +
    [x_last]*4."""
    x = np.asarray(x, dtype=np.float64)
    return np.concatenate([np.repeat(x[:1], 4), x[2:-2], np.repeat(x[-1:], 4)])


def spline_basis(t, x):
    """FITPACK's fpbisp per point: clamp x to [t_3, t_m], take the interval l (the largest in
    [3, m-1] with t_l <= x) and the four nonzero cubic B-splines there (fpbspl's recurrence).
    Returns (l, h [len(x)][4]); B-spline l - 3 + i has the value h[:, i]."""
    t = np.asarray(t, dtype=np.float64)
    m = len(t) - 4
    x = np.clip(np.asarray(x, dtype=np.float64), t[3], t[m])
    l = np.clip(np.searchsorted(t, x, side="right") - 1, 3, m - 1)
    h = np.zeros((len(x), 4))
    h[:, 0] = 1.0
    for j in range(1, 4):
        hh = h[:, :j].copy()
        h[:, 0] = 0.0
        for i in range(1, j + 1):
            tr, tl = t[l + i], t[l + i - j]
            same = tr == tl
            with np.errstate(all="ignore"):
                f = hh[:, i - 1] / (tr - tl)
                h[:, i - 1] = np.where(same, h[:, i - 1], h[:, i - 1] + f * (tr - x))
                h[:, i] = np.where(same, 0.0, f * (x - tl))
    return l, h


def spline_tables(x):
    """Knots and band factors of the interpolating cubic spline on the strictly increasing
    axis x (m >= 4 points), cached by content.  The collocation matrix A[i][j] = B_j(x_i)
    has two sub- and two superdiagonals and is totally positive, so A = L U without
    pivoting is stable (de Boor).  Factors [5][m]: L[i][i-2], L[i][i-1], 1 / U[i][i],
    U[i][i+1], U[i][i+2] (include/scint_b200_scatim.h)."""
    import hashlib
    x = np.ascontiguousarray(x, dtype=np.float64)
    key = hashlib.sha256(x.tobytes()).hexdigest()
    if key not in _SCATIM_TABLES:
        m = len(x)
        t = spline_knots(x)
        l, h = spline_basis(t, x)
        band = np.zeros((5, m))                       # A[i][i + d] at band[d + 2][i]
        for i4 in range(4):
            d = l - 3 + i4 - np.arange(m)
            nz = h[:, i4] != 0
            if np.any(np.abs(d[nz]) > 2):
                raise ValueError("collocation matrix is not banded")
            band[d[nz] + 2, np.arange(m)[nz]] = h[nz, i4]
        lo2, lo1, dg, up1, up2 = (list(map(float, r)) for r in band)
        for k in range(m):
            p = dg[k]
            if k + 1 < m:
                f = lo1[k + 1] / p
                lo1[k + 1] = f
                dg[k + 1] -= f * up1[k]
                up1[k + 1] -= f * up2[k]
            if k + 2 < m:
                f = lo2[k + 2] / p
                lo2[k + 2] = f
                lo1[k + 2] -= f * up1[k]
                dg[k + 2] -= f * up2[k]
        fac = np.array([lo2, lo1, 1.0 / np.array(dg), up1, up2])
        _SCATIM_TABLES[key] = (t, fac)
    return _SCATIM_TABLES[key]


def _scatim_crop(shape, fdop, tdel, eta):
    """calc_scattered_image's crop (dynspec.py:3514-3525) by the reference's own expressions:
    StopIteration where its next() raises.  Returns the row and column ranges of a spectrum
    of the given shape and the cropped (delay, Doppler) axes."""
    fdop = np.asarray(fdop)
    tdel = np.asarray(tdel)
    nf = len(fdop)
    below = eta * fdop**2 < np.max(tdel)
    if not np.any(below):
        raise StopIteration
    flim = int(np.argmax(below))
    rows = cols = slice(None)
    if flim == 0:
        above = tdel > eta * fdop[0] ** 2
        if not np.any(above):
            raise StopIteration
        rows = slice(None, int(np.argmax(above)))
        tdel = fdop[rows]
    else:
        cols = slice(flim - int(0.02*nf), nf - flim + int(0.02*nf))
        fdop = fdop[cols]
    r0, r1, _ = rows.indices(shape[0])
    c0, c1, _ = cols.indices(shape[1])
    return (r0, max(r1, r0)), (c0, max(c1, c0)), tdel, fdop


def _scatim_grid(fdop, sampling):
    """The image axes (dynspec.py:3553-3555) and scipy's checks: fdop_x, fdop_y."""
    nx, ny = 2*sampling+1, sampling+1
    fdop_x = np.linspace(-max(fdop), max(fdop), nx)
    fdop_y = np.linspace(0, max(fdop), ny)
    return fdop_x, fdop_y


def _scatim_spline_check(x, y, shape):
    """RectBivariateSpline(x, y, z)'s argument checks in its order (ValueError), then the
    sizes the device takes."""
    x, y = np.ravel(x), np.ravel(y)
    if not np.all(np.diff(x) > 0.0):
        raise ValueError('x must be strictly increasing')
    if not np.all(np.diff(y) > 0.0):
        raise ValueError('y must be strictly increasing')
    if not x.size == shape[0]:
        raise ValueError('x dimension of z must have same number of elements as x')
    if not y.size == shape[1]:
        raise ValueError('y dimension of z must have same number of elements as y')
    if x.size < _SCATIM_MIN_M or y.size < _SCATIM_MIN_M:
        raise ValueError("Error on entry, no approximation returned: a cubic spline needs at "
                         "least 4 points per axis (%d x %d)" % (x.size, y.size))
    if x.size > _SCATIM_MAX_MX or y.size > _SCATIM_MAX_MY:
        raise ValueError("scattered image: crop of %d delays x %d Doppler columns is outside "
                         "the supported sizes (up to %d x %d)"
                         % (x.size, y.size, _SCATIM_MAX_MX, _SCATIM_MAX_MY))


def _scatim_values_check(crop, plot_log, nx):
    """The spectrum values the device takes: every dB value must give a finite linear power
    (at most about 3082 dB).  A NaN makes every coefficient and so every pixel NaN, so with
    plot_log the reference's plot_scattered_image raises ValueError (no finite non-zero
    pixel after the shift); otherwise, with a one-pixel image (sampling=0), it raises
    IndexError in centres_to_edges.  Raised here before any device work."""
    top = np.max(crop)
    if np.isnan(top):
        if plot_log:
            raise ValueError("zero-size array to reduction operation maximum which has no "
                             "identity (the scattered image is NaN: the spectrum has NaN)")
        return
    with np.errstate(over="ignore"):
        if np.isinf(10**(top / 10)):
            raise ValueError("scattered image: a dB value of %r overflows the linear spectrum"
                             % top)
    if plot_log and nx < 2:
        raise IndexError("index 1 is out of bounds for axis 0 with size 1 (plotting a "
                         "one-pixel scattered image)")


def _scatim_plan(shape, fdop, tdel, eta, sampling):
    """Every host step of one item before the device: crop, grid, checks and tables."""
    rows, cols, x, y = _scatim_crop(shape, fdop, tdel, eta)
    fdop_x, fdop_y = _scatim_grid(y, sampling)
    _scatim_spline_check(x, y, (rows[1] - rows[0], cols[1] - cols[0]))
    if not 0 <= sampling <= _SCATIM_MAX_SAMPLING:
        raise ValueError("scattered image: sampling %r is outside 0..%d"
                         % (sampling, _SCATIM_MAX_SAMPLING))
    return dict(rows=rows, cols=cols, x=x, y=y, fdop_x=fdop_x, fdop_y=fdop_y)


def _scatim_device(spec, pitch, offsets, etas, plan, shift):
    """Images [len(offsets)][nx][nx] of the items of one crop (device tensor spec, row pitch
    elements, each item's crop at offsets[k]), in groups of at most _SCATIM_GROUP_BYTES."""
    import torch
    tx, fx = spline_tables(plan["x"])
    ty, fy = spline_tables(plan["y"])
    mx, my = len(plan["x"]), len(plan["y"])
    nx, ny = len(plan["fdop_x"]), len(plan["fdop_y"])
    up = lambda a: D.upload(np.ascontiguousarray(a, dtype=np.float64))   # noqa: E731
    keep = [up(v) for v in (tx, fx, ty, fy, plan["fdop_x"], plan["fdop_y"])]
    n = len(offsets)
    out = D.empty((n, nx, nx), torch.float64)
    per = 8 * (mx * my + nx * nx)
    step = int(max(1, min(_SCATIM_MAX_ITEMS, _SCATIM_GROUP_BYTES // per)))
    d_off = D.upload(np.asarray(offsets, dtype=np.int64))
    d_eta = up(etas)
    for k0 in range(0, n, step):
        k1 = min(n, k0 + step)
        s = _lib.ScatIm()
        s.nitem, s.mx, s.my, s.nx, s.ny, s.shift = k1 - k0, mx, my, nx, ny, 1 if shift else 0
        s.pitch, s.sspec = pitch, spec.data_ptr()
        s.offset, s.eta = d_off[k0:].data_ptr(), d_eta[k0:].data_ptr()
        s.tx, s.fx, s.ty, s.fy, s.ax, s.ay = (t.data_ptr() for t in keep)
        s.image = out[k0:].data_ptr()
        _lib.check(_lib.lib.sb_scattered_image_f64(s, D.stream_ptr()))
    return out


def scattered_image_batch(sspecs, fdop, tdel, eta, sampling=64, plot_log=True):
    """The scattered image of every secondary spectrum of a stack, in batched device passes.

    sspecs [..., ntdel, nfdop] (dB, e.g. Dynspec.cutsspec), fdop [nfdop], tdel [ntdel];
    eta a scalar or one curvature per spectrum.  Returns (images [..., nx, nx], axes) with
    nx = 2*sampling + 1.  Image k is bit-identical to
    Dynspec.calc_scattered_image(input_sspec=sspecs[k], input_eta=eta[k], input_fdop=fdop,
    input_tdel=tdel, sampling=sampling, plot_log=plot_log)'s scattered_image, and the same
    errors are raised, before any device work.  axes [..., nx] holds each spectrum's
    scattered_image_ax (they differ only where the curvatures give different crops).
    Spectra whose curvatures give the same crop share a device pass.  Limits as calc_scattered_image's: crops of 4..65536 delays by
    4..32768 Doppler columns, sampling 0..4096 (ValueError)."""
    S = np.asarray(sspecs, dtype=np.float64)
    if S.ndim < 2:
        raise ValueError("sspecs must be [..., ntdel, nfdop]")
    lead = S.shape[:-2]
    S = np.ascontiguousarray(S.reshape((-1,) + S.shape[-2:]))
    K, nr, nc = S.shape
    etas = np.broadcast_to(np.asarray(eta, dtype=np.float64).ravel()
                           if np.ndim(eta) else np.float64(eta), (K,))
    plans, groups = [], {}
    for k in range(K):
        p = _scatim_plan((nr, nc), fdop, tdel, etas[k], sampling)
        _scatim_values_check(S[k, p["rows"][0]:p["rows"][1], p["cols"][0]:p["cols"][1]],
                             plot_log, len(p["fdop_x"]))
        plans.append(p)
        groups.setdefault((p["rows"], p["cols"]), []).append(k)
    nx = 2 * sampling + 1
    images = np.empty((K, nx, nx))
    axes = np.array([p["fdop_x"] for p in plans]).reshape((K, nx))
    if K:
        spec = D.upload(S)
        for (rows, cols), ks in groups.items():
            offs = [k * nr * nc + rows[0] * nc + cols[0] for k in ks]
            out = _scatim_device(spec, nc, offs, etas[ks], plans[ks[0]], plot_log)
            images[ks] = D.download(out)
    return images.reshape(lead + (nx, nx)), axes.reshape(lead + (nx,))


# ----------------------------------------------------------------------
# band edges (csrc/clean.cu)
# ----------------------------------------------------------------------
def _zero_counts(dyn):
    """Each row's count of entries of dyn that are 0 or NaN, and a function of the kept rows
    (r0, r1) that returns each column's count over them (sb_dyn_zero_counts_f64).  The array
    is read once for the first, and the smaller of the trimmed bands and the kept rows once
    more for the second."""
    import torch
    nr, nc = np.shape(dyn)
    d = D.upload(np.ascontiguousarray(dyn, dtype=np.float64))
    rows = D.empty((nr,), torch.int32)
    cols = D.empty((3, nc), torch.int32)

    def count(a, b, rc, cc):
        _lib.check(_lib.lib.sb_dyn_zero_counts_f64(d.data_ptr(), nr, nc, a, b, D.ptr(rc),
                                                   D.ptr(cc), D.stream_ptr()))

    def kept(r0, r1):
        if nr - (r1 - r0) <= r1 - r0:
            count(0, r0, None, cols[1])
            count(r1, nr, None, cols[2])
            c = D.download(cols).astype(np.int64)
            return c[0] - c[1] - c[2]
        count(r0, r1, None, cols[1])
        return D.download(cols[1]).astype(np.int64)

    count(0, nr, rows, cols[0])
    return D.download(rows).astype(np.int64), kept


class BasicDyn:
    """Container with the attributes Dynspec.load_dyn_obj reads
    (dynspec.py:4146-4230)."""

    def __init__(self, dyn, name="BasicDyn", header=["BasicDyn"], times=[],
                 freqs=[], nchan=None, nsub=None, bw=None, df=None,
                 freq=None, tobs=None, dt=None, mjd=60000):
        times = np.asarray(times)
        freqs = np.asarray(freqs)
        if times.size == 0 or freqs.size == 0:
            raise ValueError("must input array of times and frequencies")
        self.name = name
        self.header = header
        self.times = times
        self.freqs = freqs
        self.nchan = nchan if nchan is not None else len(freqs)
        self.nsub = nsub if nsub is not None else len(times)
        self.bw = bw if bw is not None else abs(max(freqs)) - abs(min(freqs))
        self.df = df if df is not None else freqs[1] - freqs[2]
        self.freq = freq if freq is not None else np.mean(np.unique(freqs))
        self.tobs = tobs
        self.dt = dt if dt is not None else times[1] - times[0]
        self.mjd = mjd
        self.dyn = dyn


class Dynspec(ArcFitMixin):

    def __init__(self, filename=None, dyn=None, verbose=True, process=False,
                 lamsteps=False, remove_short_subs=True, subint_thresh=2.33,
                 mjd=None):
        if filename:
            self.load_file(filename, verbose=verbose, process=process,
                           lamsteps=lamsteps, subint_thresh=subint_thresh,
                           remove_short_subs=remove_short_subs, mjd=mjd)
        elif dyn is not None:
            self.load_dyn_obj(dyn, verbose=verbose, process=process,
                              lamsteps=lamsteps)
        else:
            print("Error: No dynamic spectrum file or object")

    def load_dyn_obj(self, dyn, verbose=True, process=True, lamsteps=False):
        """dynspec.py:378-420."""
        self.name = dyn.name
        self.header = dyn.header
        self.times = dyn.times
        self.freqs = dyn.freqs
        self.nchan = dyn.nchan
        self.nsub = dyn.nsub
        self.bw = dyn.bw
        self.df = dyn.df
        self.freq = dyn.freq
        self.dt = dyn.dt
        self.tobs = dyn.tobs if getattr(dyn, "tobs", None) is not None else \
            np.ptp(self.times) + self.dt
        self.mjd = dyn.mjd if getattr(dyn, "mjd", None) is not None else 60000.0
        self.dyn = dyn.dyn
        self.lamsteps = lamsteps
        for extra in ("eta", "betaeta"):      # Simulation objects carry these
            if hasattr(dyn, extra):
                setattr(self, extra, getattr(dyn, extra))
        if process:
            self.calc_acf()
            self.calc_sspec(lamsteps=lamsteps)
        if verbose:
            print("LOADED DYNSPEC OBJECT {0}".format(self.name))

    # ------------------------------------------------------------------
    # psrflux files and joining (host only: parsing, indexing, bookkeeping)
    # ------------------------------------------------------------------
    def __add__(self, other):
        """Concatenation in time with the gap between the observations zero-filled
        (reference dynspec.py:81-142).  ``a += b`` goes through here too."""
        print("Now adding {} ...".format(other.name))
        if self.freq != other.freq \
                or self.bw != other.bw or self.df != other.df:
            print("WARNING: Code does not yet account for different \
                  frequency properties")
        bw = self.bw
        df = self.df
        freqs = self.freqs
        freq = self.freq
        nchan = self.nchan
        dt = self.dt
        timegap = round((other.mjd - self.mjd)*86400
                        - self.tobs, 1)  # time between two dynspecs
        extratimes = np.arange(0, timegap, dt)
        if timegap < dt:
            extratimes = [0]
            nextra = 0
        else:
            nextra = len(extratimes)
        dyngap = np.zeros([np.shape(self.dyn)[0], nextra])
        name = self.name.split('.')[0] + "+" + other.name.split('.')[0] \
            + ".dynspec"
        header = self.header + other.header
        nsub = self.nsub + nextra + other.nsub
        tobs = self.tobs + timegap + other.tobs
        times = np.linspace(0, tobs, nsub)
        mjd = np.min([self.mjd, other.mjd])  # mjd for earliest dynspec
        newdyn = np.concatenate((self.dyn, dyngap, other.dyn), axis=1)
        newdyn = BasicDyn(newdyn, name=name, header=header, times=times,
                          freqs=freqs, nchan=nchan, nsub=nsub, bw=bw,
                          df=df, freq=freq, tobs=tobs, dt=dt, mjd=mjd)
        return Dynspec(dyn=newdyn, verbose=False, process=False)

    def load_file(self, filename, verbose=True, process=False, lamsteps=False,
                  remove_short_subs=True, subint_thresh=2.33, mjd=None):
        """Load a psrflux dynamic spectrum (reference dynspec.py:144-230): the first
        ``MJD0:`` header line gives self.mjd unless ``mjd`` is given (neither:
        AttributeError), rows are flipped into ascending frequency when the file lists
        them descending, and short leading sub-integrations are removed when the
        sub-integration times vary.  A file of other than nsub x nchan samples raises
        numpy's reshape ValueError."""
        if verbose:
            start = time.time()
            print("LOADING {0}...".format(filename))
        head = []
        with open(filename, "r") as file:
            for line in file:
                if line.startswith("#"):
                    headline = str.strip(line[1:])
                    head.append(headline)
                    if str.split(headline) != []:
                        if str.split(headline)[0] == 'MJD0:':
                            if not hasattr(self, 'mjd'):  # first occurrence
                                self.mjd = float(str.split(headline)[1])
        self.name = os.path.basename(filename)
        self.filename = filename
        self.header = head
        rawdata = np.loadtxt(filename).transpose()
        self.times = np.unique(rawdata[2]*60)  # leading edge of integration (s)
        if mjd is not None:
            self.mjd = mjd
        else:
            self.mjd = self.mjd + self.times[0] / 86400
        self.times = self.times - self.times[0]
        self.freqs = rawdata[3]
        fluxes = rawdata[4]
        self.nchan = int(np.max(rawdata[1])) + 1
        self.bw = self.freqs[-1] - self.freqs[0]
        self.df = round(self.bw/self.nchan, 5)
        self.bw = round(self.bw + self.df, 2)
        self.nsub = int(np.max(rawdata[0])) + 1
        self.dt = np.mean(np.diff(self.times))
        self.tobs = np.max(self.times) + self.dt
        self.freqs = np.unique(self.freqs)
        self.freq = round(np.mean(self.freqs), 2)
        fluxes = fluxes.reshape([self.nsub, self.nchan]).transpose()
        if self.df < 0:  # ascending frequency, like self.freqs
            self.df = -self.df
            self.bw = -self.bw
            fluxes = np.flip(fluxes, 0)
        self.dyn = fluxes
        if remove_short_subs and np.std(np.diff(self.times)) != 0:
            self.remove_short_subs(threshold=subint_thresh)
        self.lamsteps = lamsteps
        if process:
            self.auto_processing(lamsteps=lamsteps)
        if verbose:
            end = time.time()
            print("...LOADED in {0} seconds\n".format(round(end - start, 2)))
            self.info()

    def remove_short_subs(self, threshold=2.33):
        """Drop leading sub-integrations shorter than the mean of the others by more than
        threshold standard deviations (reference dynspec.py:232-257)."""
        dt0 = np.abs(np.diff(self.times))[0]
        dt = np.mean(np.abs(np.diff(self.times))[1:])
        sdt = np.std(np.abs(np.diff(self.times))[1:])
        while dt0 - dt <= -threshold*sdt and sdt >= 0:
            self.dyn = np.delete(self.dyn, (0), axis=1)
            self.times = np.delete(self.times, (0))
            dt0 = np.abs(np.diff(self.times))[0]
            dt = np.mean(np.abs(np.diff(self.times))[1:])
            sdt = np.std(np.abs(np.diff(self.times))[1:])
        self.mjd += np.min(self.times)/86400
        self.times -= np.min(self.times)
        self.nsub = len(self.times)
        self.dt = round(np.mean(np.diff(self.times)), 3)
        self.tobs = round(max(self.times) + self.dt, 3)

    def auto_processing(self, lamsteps=False, remove_short_sub=True):
        """trim_edges, refill, calc_acf, scale_dyn (lamsteps), calc_sspec (reference
        dynspec.py:422-440)."""
        self.trim_edges(remove_short_sub=remove_short_sub)
        self.refill()
        self.calc_acf()
        if lamsteps:
            self.scale_dyn()
        self.calc_sspec(lamsteps=lamsteps)

    def info(self):
        """Print the observation's properties (reference dynspec.py:4130-4143)."""
        print("\t OBSERVATION PROPERTIES\n")
        print("filename:\t\t\t{0}".format(self.name))
        print("MJD:\t\t\t\t{0}".format(self.mjd))
        print("Centre frequency (MHz):\t\t{0}".format(self.freq))
        print("Bandwidth (MHz):\t\t{0}".format(self.bw))
        print("Channel bandwidth (MHz):\t{0}".format(self.df))
        print("Integration time (s):\t\t{0}".format(self.tobs))
        print("Subintegration time (s):\t{0}".format(self.dt))
        return

    def crop_dyn(self, fmin=0, fmax=np.inf, tmin=0, tmax=np.inf):
        """Keep frequencies in [fmin, fmax] MHz and times in [tmin, tmax] minutes
        (reference dynspec.py:3816-3854)."""
        crop_array = np.array((self.freqs >= fmin)*(self.freqs <= fmax))
        self.dyn = self.dyn[crop_array, :]
        self.freqs = self.freqs[crop_array]
        self.nchan = len(self.freqs)
        self.bw = round(max(self.freqs) - min(self.freqs) + self.df, 2)
        self.freq = round(np.mean(self.freqs), 2)
        tmin = tmin*60  # to seconds
        tmax = tmax*60
        if tmax < self.tobs:
            self.tobs = tmax - tmin
        else:
            self.tobs = self.tobs - tmin
        crop_array = np.array((self.times >= tmin)*(self.times <= tmax))
        self.dyn = self.dyn[:, crop_array]
        self.nsub = len(self.dyn[0, :])
        self.times = self.times[crop_array]
        self.mjd += np.min(self.times)/86400
        self.times -= np.min(self.times)

    # ------------------------------------------------------------------
    # band edges and zapping (csrc/clean.cu)
    # ------------------------------------------------------------------
    def trim_edges(self, bandwagon_frac=0.5, remove_short_sub=True):
        """Remove the band edges (reference dynspec.py:259-328): bottom rows first, then
        top rows, then left and right columns, each while its count of zero or NaN entries
        is greater than bandwagon_frac * n or it is all zero.  n is the column count for
        rows and the row count before trimming for columns (the reference's), while a
        column's zeros are counted over the rows kept.  NaN entries of self.dyn become 0;
        the bookkeeping attributes follow the reference's expressions.

        The zero counts come from the device in one read of the array; the host picks the
        kept box and takes one crop.  Deviation: when every row or every column would go,
        the reference's IndexError is raised before anything is changed (the reference has
        set NaN to 0 by then).  remove_short_sub is accepted and unused, as there."""
        dyn = self.dyn
        nr, nc = np.shape(dyn)
        if nr == 0 or nc == 0:
            raise IndexError("index 0 is out of bounds for axis 0 with size 0")
        rz, cz = _zero_counts(dyn)
        gone = (rz > bandwagon_frac*nc) | (rz == nc)
        if np.all(gone):
            raise IndexError("index 0 is out of bounds for axis 0 with size 0")
        r0, r1 = int(np.argmin(gone)), nr - int(np.argmin(gone[::-1]))
        cz = cz(r0, r1)
        gone = (cz > bandwagon_frac*nr) | (cz == r1 - r0)
        if np.all(gone):
            raise IndexError("index 0 is out of bounds for axis 1 with size 0")
        c0, c1 = int(np.argmin(gone)), nc - int(np.argmin(gone[::-1]))
        dyn[np.isnan(dyn)] = 0
        if (r0, r1, c0, c1) != (0, nr, 0, nc):
            self.dyn = dyn[r0:r1, c0:c1].copy()
        if (r0, r1) != (0, nr):
            self.freqs = np.delete(self.freqs, np.r_[0:r0, r1:nr])
        if (c0, c1) != (0, nc):
            self.times = np.delete(self.times, np.r_[0:c0, c1:nc])
        self.mjd += np.min(self.times)/86400
        self.times -= np.min(self.times)  # start at 0
        self.nchan = len(self.freqs)
        self.bw = round(max(self.freqs) - min(self.freqs) + self.df, 3)
        self.freq = round(np.mean(self.freqs), 3)
        self.nsub = len(self.times)
        self.dt = round(np.mean(np.diff(self.times)), 3)
        self.tobs = round(max(self.times) + self.dt, 3)
        self.df = self.bw / self.nchan

    def zap(self, sigma=7):
        """Basic RFI zapping (reference dynspec.py:3856-3870): NaN where
        |dyn - med| / mdev > sigma, med the median of the pixels that are not NaN and mdev
        the median of the deviations that are not NaN, both exactly numpy's.  Runs on the
        device; a float64 C-contiguous self.dyn is changed in place, any other is replaced
        by its float64 result."""
        import torch
        d = D.upload(np.ascontiguousarray(self.dyn, dtype=np.float64))
        stats = D.empty((2,), torch.float64)
        _lib.check(_lib.lib.sb_zap_f64(d.data_ptr(), d.numel(), float(sigma),
                                       stats.data_ptr(), D.stream_ptr()))
        dyn = self.dyn
        if isinstance(dyn, np.ndarray) and dyn.dtype == np.float64 and \
                dyn.flags.c_contiguous and dyn.flags.writeable:
            torch.from_numpy(dyn).copy_(d)
        else:
            self.dyn = D.download(d)

    # ------------------------------------------------------------------
    # gap filling (csrc/inpaint.cu)
    # ------------------------------------------------------------------
    def refill(self, method='biharmonic', zeros=True, kernel_size=5, linear=True, tol=1e-10,
               maxit=50000):
        """Replace the NaN pixels of self.dyn, and its zeros if ``zeros`` (reference
        dynspec.py:3273-3323), in place, in the reference's order:

        1. zeros: self.dyn[self.dyn == 0] = NaN;
        2. 'biharmonic': inpaint_biharmonic of the NaN pixels (skimage's system, solved
           on the device, see ``inpaint_biharmonic``), written into those pixels;
           'median': scipy.signal.medfilt(kernel_size) of a copy whose NaN pixels hold the
           mean of the valid ones (zero padding at the edges), computed on the device at
           the NaN pixels only and written there; 'linear' / 'cubic' / 'nearest' with
           linear=True: NotImplementedError (the reference's griddata triangulates the
           valid pixels, and on a pixel lattice qhull's choice among co-circular points
           cannot be matched); with linear=False, or any other name (e.g. 'mean'), nothing;
        3. the NaN pixels left get np.mean of the valid ones.

        The means are the reference's numpy expressions on the host.  For 'biharmonic' and
        'median', ValueError before anything is changed when self.dyn has an infinite pixel
        (a deliberate deviation: the reference's biharmonic result there depends on
        SuperLU's elimination order), every pixel would be masked, or the shape is outside
        1..32768 x 1..16384; 'median' also rejects an even size (as medfilt does) and sizes
        above 31.  A biharmonic solve that does not converge warns (RuntimeWarning) and
        its result is still stored.

        tol and maxit (not in the reference) are the biharmonic solver's stopping rule,
        ||b - A x|| <= tol ||b||, and its step cap.  The error the rule leaves grows with
        the size of the largest hole (about L^4 for a hole L pixels wide): at the default
        1e-10, holes up to 32 x 32 come within 1e-7 of the known range of the direct
        solution, but a 64 x 256 block only within about 1e-4; tol=1e-13 brings that to
        about 5e-8 for twice the steps."""
        if method in ('linear', 'cubic', 'nearest') and linear:
            raise NotImplementedError(
                "griddata interpolation is not on the GPU path: its triangulation of a pixel "
                "lattice is not reproducible; use method='biharmonic' or 'median'")
        if method in ('biharmonic', 'median'):
            dyn = np.asarray(self.dyn)
            masked = np.isnan(dyn)
            if zeros:
                masked |= dyn == 0
            _fill_check(dyn, masked)
            if method == 'median':
                size = _medfilt_size(kernel_size)
        if zeros:
            self.dyn[self.dyn == 0] = np.nan
        if method == 'biharmonic':
            nan = np.isnan(self.dyn)
            if np.any(nan):
                self.dyn[nan] = _biharmonic_values(self.dyn, nan, tol, maxit)[0]
        elif method == 'median':
            if kernel_size == 5:
                print("Warning: kernel size is set to default.")
            nan = np.isnan(self.dyn)
            if np.any(nan):
                meanval = np.mean(self.dyn[is_valid(self.dyn)])
                self.dyn[nan] = _median_values(self.dyn, nan, size, meanval)
        meanval = np.mean(self.dyn[is_valid(self.dyn)])
        self.dyn[np.isnan(self.dyn)] = meanval

    # ------------------------------------------------------------------
    # flux-variation correction (csrc/svd.cu)
    # ------------------------------------------------------------------
    def correct_dyn(self, svd=True, nmodes=1, frequency=True, time=True,
                    lamsteps=False, nsmooth=None, velocity=False, dtype=np.float64):
        """Correct for flux variations in time and frequency (reference
        dynspec.py:3325-3410), with the reference's side effects:

        - the array is self.dyn, self.lamdyn (lamsteps; made by scale_dyn if
          missing), self.vdyn or self.vlamdyn (velocity; ValueError if missing);
          its NaN pixels are set to 0 in place and the result replaces it;
        - svd=True: self.svd_model is the rank-nmodes model M (complex, zero
          imaginary part) and the array becomes array / |M| (inf / NaN where M is 0);
          frequency, time and nsmooth are ignored;
        - svd=False: self.bandpass = nanmean over time (zeros replaced by its
          mean), divided out (savgol_filter(., nsmooth, 1) first if nsmooth), then
          the same over frequency on the quotient.  Zeros of self.dyn count as
          NaN in both passes, so when the array is self.dyn every zero or NaN
          pixel comes out NaN; NaN pixels of self.dyn are set to 0.

        dtype=np.float64 returns float64 / complex128 like the reference;
        np.float32 skips the widening.  nmodes must be in 1..32 and the array
        at most 32768 x 16384 (ValueError before any device work).  A solver
        that does not converge, or a tie between singular values nmodes and
        nmodes+1, raises a RuntimeWarning; the result is still stored."""
        import torch
        from scipy.signal import savgol_filter
        if svd:
            thth._svd_check_modes(nmodes)
        if hasattr(self, 'svd_model'):
            print('Warning: An svd_model exists. Check before applying twice')
        if lamsteps:
            if velocity:
                if not hasattr(self, 'vlamdyn'):
                    raise ValueError('Need to run scale_dyn with a model')
                attr = 'vlamdyn'
            else:
                if not hasattr(self, 'lamdyn'):
                    self.scale_dyn(lamsteps=lamsteps)
                attr = 'lamdyn'
        elif velocity:
            if not hasattr(self, 'vdyn'):
                raise ValueError('Need to run scale_dyn with a model')
            attr = 'vdyn'
        else:
            attr = 'dyn'
        dyn = getattr(self, attr)
        thth._svd_check(dyn, nmodes if svd else 1)
        dyn[np.isnan(dyn)] = 0
        cdt = np.complex64 if np.dtype(dtype) == np.float32 else np.complex128
        if svd:
            out, model, _ = thth._svd_run(dyn, int(nmodes))
            self.svd_model = D.download(model).astype(cdt)
        else:
            nf, nt = dyn.shape
            # the reference sets zeros of self.dyn to NaN before each pass: they are
            # the selected array's zeros only when that array is self.dyn
            zero_nan = 1 if (dyn is self.dyn and (frequency or time)) else 0
            d = D.upload_f32(dyn)
            rowdiv = coldiv = None
            if frequency:
                m = D.empty((nf,), torch.float64)
                _lib.check(_lib.lib.sb_bandpass_rows(d.data_ptr(), nf, nt, zero_nan,
                                                     m.data_ptr(), D.stream_ptr()))
                bandpass = m.cpu().numpy()
                bandpass[bandpass == 0] = np.mean(bandpass)
                self.bandpass = bandpass.astype(dtype)
                if nsmooth is not None:
                    bandpass = savgol_filter(bandpass, nsmooth, 1)
                rowdiv = D.upload(np.ascontiguousarray(bandpass, dtype=np.float64))
            if time:
                m = D.empty((nt,), torch.float64)
                _lib.check(_lib.lib.sb_bandpass_cols(d.data_ptr(), nf, nt, zero_nan,
                                                     D.ptr(rowdiv), m.data_ptr(),
                                                     D.stream_ptr()))
                timestructure = m.cpu().numpy()
                timestructure[timestructure == 0] = np.mean(timestructure)
                if nsmooth is not None:
                    timestructure = savgol_filter(timestructure, nsmooth, 1)
                coldiv = D.upload(np.ascontiguousarray(timestructure, dtype=np.float64))
            out = D.empty((nf, nt), torch.float32)
            _lib.check(_lib.lib.sb_bandpass_divide(d.data_ptr(), nf, nt, zero_nan,
                                                   D.ptr(rowdiv), D.ptr(coldiv),
                                                   out.data_ptr(), D.stream_ptr()))
            self.dyn[np.isnan(self.dyn)] = 0
        setattr(self, attr, D.download(out, np.dtype(dtype)))

    # ------------------------------------------------------------------
    # secondary spectrum
    # ------------------------------------------------------------------
    def _pick_dyn(self, lamsteps, velocity, trap):
        """The array calc_sspec transforms (reference dynspec.py:3642-3663): the
        wavelength-rescaled copy is made on demand (scale_dyn -> self.lamdyn);
        velocity / trapezoid resampling is outside the GPU hot path and must have
        been set by the caller."""
        if lamsteps and not velocity and not hasattr(self, "lamdyn"):
            self.scale_dyn()
        for flag, attr in ((lamsteps and velocity, "vlamdyn"),
                           (lamsteps, "lamdyn"), (velocity, "vdyn"),
                           (trap, "trapdyn")):
            if flag:
                if not hasattr(self, attr):
                    raise NotImplementedError(
                        "velocity / trapezoid resampling is outside the GPU hot "
                        "path; set self.%s first" % attr)
                return cp(getattr(self, attr))
        return self.dyn

    def calc_sspec(self, prewhite=False, halve=True, plot=False,
                   lamsteps=False, input_dyn=None, input_x=None, input_y=None,
                   trap=False, window='hanning', window_frac=0.1,
                   return_sspec=False, velocity=False, dtype=np.float64):
        """Secondary spectrum (reference dynspec.py:3584-3748).

        Same arguments and side effects (sets self.sspec / fdop / tdel [/ beta],
        or returns (fdop, yaxis, sec)).  The array comes back as float64 like
        the reference's; pass dtype=np.float32 to skip the widening."""
        import torch
        if plot:
            raise NotImplementedError("plotting is outside the GPU hot path")
        dyn = self._pick_dyn(lamsteps, velocity, trap) if input_dyn is None \
            else input_dyn
        dyn = np.asarray(dyn)
        nf, nt = dyn.shape
        if prewhite and not halve:
            raise RuntimeError('Cannot apply prewhite to full frame')
        nrfft = int(2 ** (np.ceil(np.log2(nf)) + 1))
        ncfft = int(2 ** (np.ceil(np.log2(nt)) + 1))
        d = D.upload_f32(dyn)
        wt = wf = None
        swt = swf = 0.0
        if window is not None:
            chan_window, subint_window = get_window(nt, nf, window=window,
                                                    frac=window_frac)
            swt, swf = float(chan_window.sum()), float(subint_window.sum())
            wt = D.upload(chan_window.astype(np.float32))
            wf = D.upload(subint_window.astype(np.float32))
        if halve:
            td = np.array(list(range(0, int(nrfft / 2))))
        else:
            td = np.array(list(range(0, int(nrfft))))
        fd = np.array(list(range(int(-ncfft / 2), int(ncfft / 2))))
        fdop = np.reshape(np.multiply(fd, 1e3 / (ncfft * self.dt)), [len(fd)])
        tdel = np.reshape(np.divide(td, (nrfft * self.df)), [len(td)])
        pd1 = pd2 = None
        if prewhite:   # post-darken vectors, dynspec.py:3706-3711
            pd1 = D.upload(np.power(np.sin(np.multiply(np.pi / ncfft, fd)), 2)
                           .astype(np.float32))
            pd2 = D.upload(np.power(np.sin(np.multiply(np.pi / nrfft, td)), 2)
                           .astype(np.float32))
        sec = D.empty((len(td), ncfft), torch.float32)
        _lib.check(_lib.lib.sb_sspec_f32(
            d.data_ptr(), nf, nt, D.ptr(wt), D.ptr(wf), swt, swf,
            1 if prewhite else 0, 1 if halve else 0, 1, D.ptr(pd1), D.ptr(pd2),
            sec.data_ptr(), D.stream_ptr()))
        sec = D.download(sec, dtype)
        np.seterr(divide='ignore')      # reference side effect (:3720)
        beta = None
        if lamsteps:
            beta = np.divide(td, (nrfft * self.dlam))
        if input_dyn is None and not return_sspec:
            if lamsteps:
                if velocity:
                    self.vlamsspec = sec
                else:
                    self.lamsspec = sec
            elif velocity:
                self.vsspec = sec
            elif trap:
                self.trapsspec = sec
            else:
                self.sspec = sec
            self.fdop = fdop
            self.tdel = tdel
            if lamsteps:
                self.beta = beta
        else:
            return fdop, (beta if lamsteps else tdel), sec

    # ------------------------------------------------------------------
    # autocovariance
    # ------------------------------------------------------------------
    # ------------------------------------------------------------------
    # wavelength rescaling (csrc/scale_dyn.cu)
    # ------------------------------------------------------------------
    @staticmethod
    def _spline_tables(x, xq):
        """Column-independent tables of the not-a-knot cubic spline through the
        ascending knots ``x`` evaluated at ``xq`` (= scipy interp1d(kind='cubic'),
        checked on the CPU to 1e-16): Thomas factors of the second-derivative
        system and the four weights of (y_i, y_i+1, M_i, M_i+1) per query."""
        x = np.asarray(x, dtype=np.float64)
        xq = np.asarray(xq, dtype=np.float64)
        n = x.shape[0]
        h = np.diff(x)
        a = np.zeros(n)
        b = np.zeros(n)
        c = np.zeros(n)
        a[1:n - 1] = h[:-1]
        b[1:n - 1] = 2 * (h[:-1] + h[1:])
        c[1:n - 1] = h[1:]
        p0 = h[0] / h[1]
        pn = h[n - 2] / h[n - 3]
        b[1] += h[0] * (1 + p0)
        c[1] -= h[0] * p0
        a[1] = 0.0
        b[n - 2] += h[n - 2] * (1 + pn)
        a[n - 2] -= h[n - 2] * pn
        c[n - 2] = 0.0
        cpr = np.zeros(n)
        inv = np.zeros(n)
        for i in range(1, n - 1):
            inv[i] = 1.0 / (b[i] - a[i] * cpr[i - 1])
            cpr[i] = c[i] * inv[i]
        g = np.zeros(n)
        g[:n - 1] = 6.0 / h
        idx = np.clip(np.searchsorted(x, xq, side="right") - 1, 0, n - 2)
        hi = h[idx]
        dl = x[idx + 1] - xq
        dr = xq - x[idx]
        W = np.stack([dl / hi, dr / hi, (dl ** 3 / hi - hi * dl) / 6,
                      (dr ** 3 / hi - hi * dr) / 6], axis=1)
        return dict(a=a, cp=cpr, inv=inv, g=g, p0=p0, pn=pn, idx=idx, W=W)

    def scale_dyn(self, scale='lambda', spacing='auto', **kwargs):
        """Resample the dynamic spectrum to equal wavelength steps (reference
        dynspec.py:3872-3957, scale='lambda' only) -> self.lamdyn, self.lam,
        self.nlam, self.dlam."""
        import torch
        from scipy.constants import c as c_light
        if not (('lambda' in scale) or ('wavelength' in scale)):
            raise NotImplementedError("only scale='lambda' is on the GPU path")
        freqs = np.array(self.freqs, dtype=np.float64)
        nf, nt = self.dyn.shape
        lams = np.divide(c_light, freqs * 10 ** 6)
        adl = np.abs(np.diff(lams))
        if spacing == 'auto':
            dlam = (np.max(lams) - np.min(lams)) / len(freqs)
        else:
            dlam = {'max': np.max, 'median': np.median, 'mean': np.mean,
                    'min': np.min}[spacing](adl)
        lam_eq = np.arange(np.min(lams) + 1e-10, np.max(lams) - 1e-10, dlam)
        feq = np.round(np.divide(c_light, lam_eq) / 10 ** 6, 6)
        if max(feq) > max(freqs):
            feq[np.argmax(feq)] = max(freqs)
        if min(feq) < min(freqs):
            feq[np.argmin(feq)] = min(freqs)
        d = np.diff(freqs)
        if np.all(d > 0):
            flip, x = 0, freqs
        elif np.all(d < 0):
            flip, x = 1, freqs[::-1]
        else:
            raise ValueError("scale_dyn needs a monotonic frequency axis")
        T = self._spline_tables(x, feq)
        f32 = lambda v: D.upload(np.ascontiguousarray(v, dtype=np.float32))
        dd = D.upload_f32(np.asarray(self.dyn))
        nlam = feq.shape[0]
        out = D.empty((nlam, nt), torch.float32)
        a, cpr, inv, g = f32(T["a"]), f32(T["cp"]), f32(T["inv"]), f32(T["g"])
        idx = D.upload(np.ascontiguousarray(T["idx"], dtype=np.int32))
        W = f32(T["W"])
        _lib.check(_lib.lib.sb_scale_dyn_lambda_f32(
            dd.data_ptr(), nf, nt, flip, a.data_ptr(), cpr.data_ptr(), inv.data_ptr(),
            g.data_ptr(), float(T["p0"]), float(T["pn"]), idx.data_ptr(), W.data_ptr(), nlam,
            out.data_ptr(), D.stream_ptr()))
        self.dlam = dlam
        self.lamdyn = out.cpu().numpy().astype(np.float64)
        self.lam = np.flipud(lam_eq)
        self.nlam = len(self.lam)

    def calc_acf(self, method='direct', input_dyn=None, normalise=True,
                 window_frac=0.1, dtype=np.float64):
        """Autocovariance function (reference dynspec.py:3750-3814)."""
        import torch
        if method == 'direct':
            src = np.asarray(self.dyn if input_dyn is None else input_dyn)
            nf, nt = src.shape
            d = D.upload_f32(src)
            out = D.empty((2 * nf, 2 * nt), torch.float32)
            _lib.check(_lib.lib.sb_acf_f32(
                d.data_ptr(), nf, nt, 1 if input_dyn is None else 0,
                1 if normalise else 0, out.data_ptr(), D.stream_ptr()))
            arr = D.download(out, dtype)
        elif method == 'sspec':     # FFT of the secondary spectrum, :3798-3807
            src = np.asarray(self.dyn)
            nf, nt = src.shape
            nrfft = int(2 ** (np.ceil(np.log2(nf)) + 1))
            ncfft = int(2 ** (np.ceil(np.log2(nt)) + 1))
            cw, sw = get_window(nt, nf, window='hanning', frac=window_frac)
            d = D.upload_f32(src)
            wt = D.upload(cw.astype(np.float32))
            wf = D.upload(sw.astype(np.float32))
            out = D.empty((nrfft, ncfft), torch.float32)
            _lib.check(_lib.lib.sb_acf_sspec_f32(
                d.data_ptr(), nf, nt, wt.data_ptr(), wf.data_ptr(),
                float(cw.sum()), float(sw.sum()), 1 if normalise else 0,
                out.data_ptr(), D.stream_ptr()))
            arr = D.download(out, dtype)
        else:
            print('Method not understood. Choose "direct" or "sspec"')
            return
        if input_dyn is None:
            self.acf = arr
        else:
            return arr

    def cut_dyn(self, tcuts=0, fcuts=0, plot=False, filename=None, dpi=200, lamsteps=False,
                maxfdop=np.inf, figsize=(8, 13), display=True, dtype=np.float64):
        """Cut the dynamic spectrum into (fcuts+1) x (tcuts+1) tiles (reference
        dynspec.py:3158-3271) and transform every tile in one batched pass
        (sb_sspec_tiles_f32, sb_acf_tiles_f32).

        fnum = floor(len(freqs) / (fcuts+1)) channels by tnum = floor(len(times) / (tcuts+1))
        subintegrations per tile; trailing rows and columns that do not fill a tile are
        dropped.  Tile (ii, jj) is self.dyn[ii*fnum:(ii+1)*fnum, jj*tnum:(jj+1)*tnum].  Sets
        - self.cutdyn [fcuts+1][tcuts+1][fnum][tnum] (float64, the tiles themselves);
        - self.cutsspec [fcuts+1][tcuts+1][nrfft/2][ncfft]: each tile's
          calc_sspec(input_dyn=tile, lamsteps=lamsteps) (Hanning window, halved, dB);
        - self.cutacf [fcuts+1][tcuts+1][2 fnum][2 tnum]: each tile's calc_acf(input_dyn=tile)
          (no mean subtracted, normalised by its zero lag).  The reference computes these
          ACFs and discards them; they are kept because a per-tile scintillation fit needs them.
        A NaN makes its own tile NaN and no other.  lamsteps changes no array; as in the
        reference, it needs self.dlam (AttributeError otherwise).  dtype=np.float32 skips
        the widening of cutsspec and cutacf.

        Errors, raised before any device work: NotImplementedError for plot=True;
        ValueError for a tile outside the sizes the single-spectrum drivers accept
        (fnum 2..32768, tnum 5..16384; the reference accepts smaller tiles)."""
        if plot:
            raise NotImplementedError("plotting is outside the GPU hot path")
        if lamsteps:
            self.dlam       # the reference's calc_sspec reads it here
        nchan, nsub = len(self.freqs), len(self.times)
        nfc, ntc = int(fcuts) + 1, int(tcuts) + 1
        fnum, tnum = nchan // nfc, nsub // ntc
        if not (_ACF_MIN_NF <= fnum <= _ACF_MAX_NF and _ACF_MIN_NT <= tnum <= _ACF_MAX_NT):
            raise ValueError("cut_dyn: tiles of %d x %d are outside the supported sizes "
                             "(fnum %d..%d, tnum %d..%d)" % (fnum, tnum, _ACF_MIN_NF, _ACF_MAX_NF,
                                                              _ACF_MIN_NT, _ACF_MAX_NT))
        dyn = np.asarray(self.dyn)[:nfc * fnum, :ntc * tnum]
        if dyn.shape != (nfc * fnum, ntc * tnum):
            raise ValueError("cut_dyn: self.dyn %s is smaller than freqs x times" %
                             (np.shape(self.dyn),))
        self.cutdyn = dyn.reshape(nfc, fnum, ntc, tnum).transpose(0, 2, 1, 3).astype(np.float64)
        self.cutsspec, self.cutacf = _cut_dyn_device(dyn, fnum, tnum, nfc, ntc, dtype)
        np.seterr(divide='ignore')      # calc_sspec's side effect (:3720)

    # ------------------------------------------------------------------
    # scattered image (csrc/scatim.cu)
    # ------------------------------------------------------------------
    def calc_scattered_image(self, input_sspec=None, input_eta=None, input_fdop=None,
                             input_tdel=None, sampling=64, lamsteps=False, trap=False,
                             ref_freq=1400, clean=True, s=None, veff=None, d=None,
                             fit_arc=True, plot_fit=False, plot=False, plot_log=True,
                             use_angle=False, use_spatial=False):
        """The scattered image: the secondary spectrum mapped onto the sky along the arc
        (reference dynspec.py:3412-3582).  Sets self.scattered_image [nx][nx] (float64,
        nx = 2*sampling + 1) and self.scattered_image_ax (fdop_x), as the reference does.

        The host runs the reference's own expressions for the spectrum and axes
        (self.lamsspec / trapsspec / sspec, made by calc_sspec if missing; the delay axis is
        self.tdel in every mode), the curvature (fit_arc(lamsteps, log_parabola=True) when
        neither eta nor betaeta is set; betaeta converted at ref_freq with lamsteps; the
        last delay over the last Doppler squared with fit_arc=False), the crop (the
        reference's: with flim == 0 the delay axis becomes fdop[:tlim], and a negative
        column start wraps as numpy's slice does) and the image grid.  The device computes
        10**(sspec/10) of the crop, the interpolating bicubic spline of
        RectBivariateSpline(tdel, fdop, .) by two banded solves, and its values at
        ((fdop_x**2 + fdop_y**2) * eta, fdop_x) as FITPACK evaluates them (clamped to the
        data range), times fdop_y, mirrored (csrc/scatim.cu).  It agrees with scipy's
        fit to rounding: the banded LU and FITPACK's Givens QR differ in the last bits.

        plot_log=True (the default) does not draw but applies what the reference's
        plot_scattered_image does to the stored image in place: image -= min(image);
        image += 1e-10.  Its errors come first: TypeError for use_angle / use_spatial with
        s, veff (or d) left as None, ValueError when the image has no finite pixel, which
        happens exactly when the crop holds a NaN, and IndexError for sampling=0 (a one-pixel
        axis has no pixel edges).

        Deviations: ``clean`` is accepted and skipped: the reference's griddata result is
        assigned to a variable it never reads, so no output changes.  plot=True and
        plot_fit=True raise NotImplementedError.  The spectrum is read as float64.  Raised as
        ValueError before any device work: crops outside 4..65536 delays by 4..32768
        Doppler columns (scipy also needs at least 4 points per axis), sampling outside
        0..4096, and a dB value whose linear power overflows float64 (above about
        3082 dB).  Every reference exception (StopIteration from the crop, AttributeError
        from the curvature, scipy's ValueErrors, the plot checks above) is raised before any
        device work.  scattered_image_batch does the same for a stack of spectra."""
        if plot or plot_fit:
            raise NotImplementedError("plotting is outside the GPU hot path")
        if input_sspec is None:
            if lamsteps:
                if not hasattr(self, 'lamsspec'):
                    self.calc_sspec(lamsteps=lamsteps)
                sspec = self.lamsspec
            elif trap:
                if not hasattr(self, 'trapsspec'):
                    self.calc_sspec(trap=trap)
                sspec = self.trapsspec
            else:
                if not hasattr(self, 'sspec'):
                    self.calc_sspec(lamsteps=lamsteps)
                sspec = self.sspec
            fdop = cp(self.fdop)
            tdel = cp(self.tdel)
        else:
            sspec, fdop, tdel = input_sspec, input_fdop, input_tdel
        nf, nt = len(fdop), len(tdel)
        sspec = np.asarray(sspec, dtype=np.float64)
        if input_eta is None and fit_arc:
            if not hasattr(self, 'betaeta') and not hasattr(self, 'eta'):
                self.fit_arc(lamsteps=lamsteps, log_parabola=True, plot=plot_fit)
            if lamsteps:
                c = 299792458.0  # m/s
                beta_to_eta = c * 1e6 / ((ref_freq * 1e6)**2)
                eta = self.betaeta / (self.freq / ref_freq)**2
                eta = eta*beta_to_eta
            else:
                eta = self.eta
        elif input_eta is None:
            eta = tdel[nt-1] / fdop[nf-1]**2
        else:
            eta = input_eta
        plan = _scatim_plan(sspec.shape, fdop, tdel, eta, sampling)
        if plot_log:
            # plot_scattered_image's axis conversions (dynspec.py:916-927), for their errors
            c = 299792458.0  # m/s
            if use_angle or use_spatial:
                thetarad = (plan["fdop_x"] / (1e9 * self.freq)) * (c * s / (veff * 1000))
                if not use_angle:
                    ((thetarad * 180 / np.pi) * 3600) * (1 - s) * d * 1000
        (r0, r1), (c0, c1) = plan["rows"], plan["cols"]
        rows = sspec[r0:r1]
        _scatim_values_check(rows[:, c0:c1], plot_log, len(plan["fdop_x"]))
        spec = D.upload(rows)
        out = _scatim_device(spec, sspec.shape[1], [c0], [float(eta)], plan, plot_log)
        self.scattered_image = D.download(out)[0]
        self.scattered_image_ax = plan["fdop_x"]

    # ------------------------------------------------------------------
    # scintillation scales (csrc/scintfit.cu)
    # ------------------------------------------------------------------
    def get_scint_params(self, method="acf1d", plot=False, alpha=5/3, mcmc=False,
                         full_frame=False, nscale=5, nwalkers=50, steps=10000, burn=0.25,
                         nitr=1, lnsigma=True, verbose=False, progress=True, display=True,
                         filename=None, dpi=200, nan_policy='raise', weighted=True, workers=1,
                         tau_vary_2d=True, tau_input=None, bartlett=True, get_fit_report=True):
        """Scintillation timescale tau (s) and decorrelation bandwidth dnu (MHz) from
        self.acf (reference dynspec.py:2470-3156), computed with calc_acf() if missing.

        method 'nofit' (estimates from the 1/e and 1/2 levels, returns None), 'acf1d' (the
        two central ACF cuts) or 'acf2d_approx' (the approximate 2-D model with a phase
        gradient, started from the 1-D fit).  alpha=None frees the exponent.  The
        reference's attributes are set (tau, dnu, amp, wn, their errors, tscat, nscint,
        fse_tau, fse_dnu, talpha, talphaerr, scint_param_method; the nofit estimates
        dnu_est, dnu_esterr, tscat_est, modulation_index, wnerr; for acf2d_approx
        acf_model, phasegrad, phasegraderr, fse_phasegrad) and its warnings printed.

        The least-squares fits run on the device (Levenberg-Marquardt with analytic float64
        Jacobians, lmfit's bound transform for tau, dnu and amp, and lmfit's standard
        errors); the result's fields are those of lmfit's MinimizerResult that callers
        read (see ScintFitResult).  Deviations: self.report is a plain-text summary, not
        lmfit's fit_report layout; the fit stops at a stationary point, tighter than
        lmfit's 1e-7 tolerances.  NotImplementedError, before any device work, for plot,
        mcmc, method 'acf2d' / 'sspec' and nan_policy other than 'raise'; ValueError for a
        non-finite ACF cut or crop, a non-finite residual during a fit, or a dynamic
        spectrum outside nf 2..32768, nt 5..16384.  nwalkers, steps, burn, nitr, lnsigma,
        progress, display, filename, dpi and workers only concern mcmc and plotting."""
        return get_scint_params_batch(
            [self], method=method, plot=plot, alpha=alpha, mcmc=mcmc, full_frame=full_frame,
            nscale=nscale, verbose=verbose, nan_policy=nan_policy, weighted=weighted,
            tau_vary_2d=tau_vary_2d, tau_input=tau_input, bartlett=bartlett,
            get_fit_report=get_fit_report)[0]

    def get_acf_tilt(self, plot=False, tmax=None, fmax=None, display=True, filename=None,
                     nscale=0.8, nscaleplot=2, nmin=5, dpi=200, method='acf1d', tmaxplot=None,
                     fmaxplot=None):
        """Tilt of the ACF in min/MHz, proportional to the phase gradient along Veff
        (reference dynspec.py:2283-2468): a 7-point parabola through the peak of every
        frequency-lag row within fmax, and a weighted straight line through the peaks.
        Sets acf_tilt, acf_tilt_err and fse_tilt; runs calc_acf and get_scint_params(method)
        first when self.acf / self.dnu are missing.  Host arithmetic on self.acf."""
        from .arcfit import fit_parabola
        if plot:
            raise NotImplementedError("plotting is outside the GPU path")
        if not hasattr(self, 'acf'):
            self.calc_acf()
        if not hasattr(self, 'dnu'):
            self.get_scint_params(method=method)
        if tmax is None:
            tmax = nscale*self.tau/60
        if fmax is None:
            fmax = nscale*self.dnu
        acf = cp(self.acf)
        nr, nc = np.shape(acf)
        t_delays = np.linspace(-self.tobs/60, self.tobs/60, nc+1)[:-1]
        f_shifts = np.linspace(-self.bw, self.bw, nr+1)[:-1]
        inds = np.argwhere(abs(f_shifts) <= fmax)
        if len(inds) < nmin:
            inds = np.argwhere(abs(f_shifts) <= nmin*self.df)
        peak_array = []
        peakerr_array = []
        y_array = []
        for ii in inds:
            x_max = np.argmax(acf[ii, :]).squeeze()
            ydata = np.array(acf[ii, x_max - 3:x_max + 4]).squeeze()
            xdata = t_delays[x_max - 3:x_max + 4]
            yfit, peak, peakerr = fit_parabola(xdata, ydata)
            peak_array.append(peak)
            peakerr_array.append(peakerr)
            y_array.append(f_shifts[ii])
        peak_array = np.array(peak_array).squeeze()
        y_array = np.array(y_array).squeeze()
        peakerr_array = np.array(peakerr_array).squeeze()
        params, pcov = np.polyfit(peak_array, y_array, 1, cov=True, w=1/peakerr_array)
        xfit = (y_array - params[1])/params[0]
        errors = []
        for i in range(len(params)):
            errors.append(np.absolute(pcov[i][i])**0.5)
        errors = np.array(errors).squeeze()
        res = np.array(peak_array - xfit).squeeze()
        reduced_chi_sq = np.sum(res**2/peakerr_array**2)/(len(xfit) - 2)
        errors *= np.sqrt(reduced_chi_sq)
        self.acf_tilt = 1/(float(params[0].squeeze()))
        acf_tilt_err = float(errors[0].squeeze()) * 1/float(params[0].squeeze())**2
        N = (1 + 0.2*self.bw/(self.dnu)) * (1 + 0.2*self.tobs/(self.tau*np.log(2)))
        fse_tau = self.tau/(2*np.sqrt(N))
        fse_dnu = self.dnu/(2*np.sqrt(N))
        self.fse_tilt = self.acf_tilt * np.sqrt((fse_dnu/self.dnu)**2 + (fse_tau/self.tau)**2)
        self.acf_tilt_err = acf_tilt_err

    # ------------------------------------------------------------------
    # theta-theta
    # ------------------------------------------------------------------
    def prep_thetatheta(self, fw=.1, npad=3, verbose=False,
                        fitting_proc='standard', **kwargs):
        """Set up the theta-theta search (reference dynspec.py:1348-1537).

        Recognises cwf, cwt, fref, eta_min, eta_max, nedge, edges_lim, tau_lim,
        tau_mask and, for fitting_proc='thin', arclet_lim and center_cut."""
        fitting_procs = ['standard', 'thin', 'incoherent']
        assert fitting_proc in fitting_procs, \
            f'fitting_proc must be one of {fitting_procs}'
        self.thetatheta_proc = fitting_proc
        self.npad = npad
        self.fw = fw
        if 'cwf' in kwargs:
            self.cwf = 2 * (kwargs['cwf'] // 2)
            self.ncf_fit = self.dyn.shape[0] // self.cwf
            self.ncf_ret = (self.dyn.shape[0] // (self.cwf // 2)) - 1
        else:
            self.cwf = self.dyn.shape[0]
            self.ncf_fit = self.ncf_ret = 1
        if 'cwt' in kwargs:
            self.cwt = 2 * (kwargs['cwt'] // 2)
            self.nct_fit = self.dyn.shape[1] // self.cwt
            self.nct_ret = (self.dyn.shape[1] // (self.cwt // 2)) - 1
        else:
            self.cwt = self.dyn.shape[1]
            self.nct_fit = self.nct_ret = 1
        tau_lim = float(U.value(kwargs['tau_lim'], "us")) \
            if 'tau_lim' in kwargs else None
        self.fref = float(U.value(kwargs['fref'], "MHz")) \
            if 'fref' in kwargs else float(np.mean(self.freqs))

        fd = U.value(thth.fft_axis(self.times[:self.cwt], "mHz"), "mHz")
        tau = U.value(thth.fft_axis(self.freqs[:self.cwf], "us"), "us")
        eta_min = 4 * (tau[1] - tau[0]) / fd.max() ** 2
        eta_max = tau.max() / (fd[1] - fd[0]) ** 2
        eta_min *= (np.max(self.freqs) / self.fref) ** 2
        eta_max *= (np.min(self.freqs) / self.fref) ** 2
        if 'eta_min' in kwargs:
            eta_min = max((float(U.value(kwargs['eta_min'], "s3")), eta_min))
        if 'eta_max' in kwargs:
            eta_max = min((float(U.value(kwargs['eta_max'], "s3")), eta_max))
        if not ('eta_min' in kwargs and 'eta_max' in kwargs):
            c = 299792458.0
            if not hasattr(self, "betaeta"):
                # Hough prior (reference dynspec.py:1458-1466): eta [s^3] -> betaeta
                # [1/(m mHz^2)] = eta * fref^2 [MHz^2 = 1e12 s^-2] / c / (1e6 s^2/mHz^-2)
                to_beta = self.fref ** 2 * 1e12 / c / 1e6
                self.fit_arc(lamsteps=True, numsteps=1e4, etamin=eta_min * to_beta,
                             etamax=eta_max * to_beta, delmax=tau_lim, plot=False)
            eta_hough = c * self.betaeta / self.fref ** 2 * 1e-12 * 1e6
            err_hough = c * 2 * max((self.betaetaerr, self.betaetaerr2)) \
                / self.fref ** 2 * 1e-12 * 1e6
            if 'eta_min' not in kwargs:
                eta_min = max((eta_min, eta_hough - err_hough))
            if 'eta_max' not in kwargs:
                eta_max = min((eta_max, eta_hough + err_hough))
        self.eta_min, self.eta_max = float(eta_min), float(eta_max)
        l0 = np.log10(self.eta_min)
        l1 = np.log10(self.eta_max)
        self.neta = int(1 + (l1 - l0) / np.log10(1 + self.fw / 10))

        if self.thetatheta_proc == 'thin':
            fd_cut = fd.max() * (self.fref / np.max(self.freqs))
        else:
            fd_cut = (fd.max() / 2) * (self.fref / np.max(self.freqs))
        if 'edges_lim' in kwargs:
            edges_lim = min((float(U.value(kwargs['edges_lim'], "mHz")), fd_cut))
        else:
            edges_lim = fd_cut
        if tau_lim is not None:
            edges_lim = min((edges_lim, np.sqrt(tau_lim / self.eta_max)))
        if 'nedge' in kwargs:
            assert np.mod(kwargs['nedge'], 2) == 0, 'nedge must be even!'
            self.edges = np.linspace(-edges_lim, edges_lim, kwargs['nedge'])
        else:
            self.edges = U.value(thth.min_edges(
                edges_lim, fd, tau,
                self.eta_max * (self.fref / np.min(self.freqs)), 2), "mHz") \
                * (np.min(self.freqs) / self.fref)
        if self.thetatheta_proc == 'thin':
            self.arclet_lim = float(U.value(kwargs['arclet_lim'], "mHz")) \
                if 'arclet_lim' in kwargs else float(edges_lim)
            self.center_cut = float(U.value(kwargs['center_cut'], "mHz")) \
                if 'center_cut' in kwargs else 0.0
        self.thth_tau_mask = float(U.value(kwargs['tau_mask'], "us")) \
            if 'tau_mask' in kwargs else 0.0
        if verbose:
            print("\n\t THETA-THETA PROPERTIES\n")
            print(f'Channels per chunk: {self.cwf}')
            print(f'Time bins per chunk: {self.cwt}')
            print(f'Number of fitting chunks: {self.ncf_fit}x{self.nct_fit}')
            print(f'Reference Frequency: {self.fref}')
            print(f'Eta range: {self.eta_min} to {self.eta_max} '
                  f'with {self.neta} points')
            print(f'Edges has {self.edges.shape[0]} point out to '
                  f'{self.edges[-1]}')
            print(f'Zero paddings: {self.npad}')

    def _chunk_etas(self, fmean):
        return np.logspace(np.log10(self.eta_min), np.log10(self.eta_max),
                           self.neta) * (self.fref / fmean) ** 2

    def thetatheta_single(self, cf=0, ct=0, fname=None, verbose=False,
                          plot=False, arrays=True):
        """Theta-theta on one chunk (reference dynspec.py:1539-1655).
        Returns (etas, eigs, popt) as the reference does with arrays=True."""
        if not hasattr(self, 'cwf'):
            self.prep_thetatheta(verbose=verbose)
        if plot:
            raise NotImplementedError("plotting is outside the GPU hot path")
        cf = min(cf, self.ncf_fit - 1)
        ct = min(ct, self.nct_fit - 1)
        fs = slice(cf * self.cwf, (cf + 1) * self.cwf)
        ts = slice(ct * self.cwt, (ct + 1) * self.cwt)
        time2 = np.asarray(self.times[ts], dtype=np.float64)
        freq2 = np.asarray(self.freqs[fs], dtype=np.float64)
        tau = U.value(thth.fft_axis(freq2, "us", self.npad), "us")
        fd = U.value(thth.fft_axis(time2, "mHz", self.npad), "mHz")
        dspec2 = np.copy(self.dyn[fs, ts]).astype(np.float64)
        dspec2 -= np.nanmean(dspec2)
        etas = self._chunk_etas(freq2.mean())
        edges = self.edges * (freq2.mean() / self.fref)
        if self.thetatheta_proc == 'thin':
            # dynspec.py:1593-1600: one singularvalue_calc per curvature
            cs = thth.conjugate_spectrum(np.nan_to_num(dspec2), self.npad, 0.0,
                                         tau, self.thth_tau_mask)
            eigs = thth.thin_sweep(cs, tau, fd, etas, edges,
                                   edges[np.abs(edges) < self.arclet_lim],
                                   self.center_cut)
        else:
            cs = thth.conjugate_spectrum(
                np.nan_to_num(dspec2), self.npad, 0.0, tau, self.thth_tau_mask,
                ncols_keep=thth.needed_fd_columns(fd, edges))
            eigs = thth.eta_sweep(cs, tau, fd, etas, edges,
                                  self.thetatheta_proc == 'standard')
        if not np.all(np.isfinite(eigs)) and verbose:
            print("some curvatures failed (NaN)")
        eta_fit, eta_sig, popt = thth.peak_fit(etas, eigs, self.fw)
        self.last_eta_fit, self.last_eta_sig = eta_fit, eta_sig
        if arrays:
            good = np.isfinite(eigs)
            return etas[good], eigs[good], popt

    def fit_thetatheta(self, verbose=False, plot=False, pool=None,
                       time_avg=False):
        """Loop theta-theta over all fitting chunks and fit eta ~ nu^-2
        (reference dynspec.py:1657-1763).  ``pool`` must be None: a CUDA
        context does not survive fork; the chunks run back to back on the GPU
        (each one already fills it)."""
        if pool is not None:
            raise ValueError("fit_thetatheta on the GPU path takes pool=None "
                             "(CUDA is not fork-safe); chunks are batched on "
                             "the device instead")
        if plot:
            raise NotImplementedError("plotting is outside the GPU hot path")
        if not hasattr(self, 'cwf'):
            self.prep_thetatheta(verbose=verbose)
        self.eta_evo = np.zeros((self.ncf_fit, self.nct_fit))
        self.eta_evo_err = np.zeros((self.ncf_fit, self.nct_fit))
        self.f0s = np.zeros(self.ncf_fit)
        self.t0s = np.zeros(self.nct_fit)
        coher = (self.thetatheta_proc != 'incoherent')
        pars, where = [], []
        for cf in range(self.ncf_fit):
            fs = slice(cf * self.cwf, (cf + 1) * self.cwf)
            freq2 = np.copy(self.freqs[fs]).astype(np.float64)
            self.f0s[cf] = freq2.mean()
            etas = self._chunk_etas(freq2.mean())
            for ct in range(self.nct_fit):
                ts = slice(ct * self.cwt, (ct + 1) * self.cwt)
                time2 = np.copy(self.times[ts]).astype(np.float64)
                dspec2 = np.copy(self.dyn[fs, ts]).astype(np.float64)
                dspec2 -= np.nanmean(dspec2)
                dspec2 = np.nan_to_num(dspec2)
                scale = freq2.mean() / self.fref
                params = [dspec2, freq2, time2, etas, self.edges * scale, None,
                          False, self.fw, self.npad, coher]
                if self.thetatheta_proc == 'thin':
                    params += [verbose,
                               self.edges[np.abs(self.edges) < self.arclet_lim]
                               * scale, self.center_cut]
                else:
                    params += [self.thth_tau_mask, verbose]
                pars.append(params)
                where.append((cf, ct))
                self.t0s[ct] = time2.mean()
        # the reference's pool.map over the chunks (dynspec.py:1715-1719): here the
        # chunks run back to back on the GPU
        if self.thetatheta_proc == 'thin':
            results = [thth.single_search_thin(p) for p in pars]
        else:
            results = thth.search_batch(pars)
        for (cf, ct), res in zip(where, results):
            self.eta_evo[cf, ct] = U.value(res[0], "s3")
            self.eta_evo_err[cf, ct] = U.value(res[1], "s3")
        f0 = self.f0s[:, np.newaxis]
        if time_avg:
            eta_avg = np.nanmean(self.eta_evo, 1)
            eta_count = np.nansum(self.eta_evo, 1) / eta_avg
            avg_err = np.nanstd(self.eta_evo, 1) / np.sqrt(eta_count - 1)
            tofit = np.isfinite(eta_avg) * np.isfinite(avg_err)
            A = (np.sum(eta_avg[tofit] / (self.f0s * avg_err)[tofit] ** 2) /
                 np.sum(1 / (self.f0s ** 2 * avg_err)[tofit] ** 2))
            A_err = np.sqrt(1 / np.sum(2 / ((self.f0s ** 2) * avg_err)[tofit] ** 2))
        else:
            tofit = np.isfinite(self.eta_evo) * np.isfinite(self.eta_evo_err)
            A = (np.sum(self.eta_evo[tofit] / (f0 * self.eta_evo_err)[tofit] ** 2) /
                 np.sum(1 / ((f0 ** 2) * self.eta_evo_err)[tofit] ** 2))
            A_err = np.sqrt(1 / np.sum(2 / ((f0 ** 2) * self.eta_evo_err)[tofit] ** 2))
        self.ththeta = A / self.fref ** 2
        self.ththetaerr = A_err / self.fref ** 2

    def _asymmetry_params(self, verbose=False):
        """The reference's calc_asymmetry chunk list (dynspec.py:1895-1913), including its
        time slice ct*cwt//2 : (ct+1)*cwt, whose width grows with ct (cwt + ct*cwt/2)."""
        pars = []
        for cf in range(self.ncf_fit):
            fs = slice(cf * self.cwf, (cf + 1) * self.cwf)
            freq2 = np.copy(self.freqs[fs]).astype(np.float64)
            freq = freq2.mean()
            eta = self.ththeta * (self.fref / freq) ** 2
            for ct in range(self.nct_fit):
                ts = slice(ct * self.cwt // 2, (ct + 1) * self.cwt)
                time2 = np.copy(self.times[ts]).astype(np.float64)
                dspec2 = np.copy(self.dyn[fs, ts]).astype(np.float64)
                dspec2 -= np.nanmean(dspec2)
                dspec2 = np.nan_to_num(dspec2)
                pars.append((dspec2, self.edges * (freq / self.fref), time2, freq2, eta, ct, cf,
                             self.npad, verbose))
        return pars

    def calc_asymmetry(self, verbose=False, pool=None):
        """Arc asymmetry of every fitting chunk (reference dynspec.py:1892-1918) ->
        self.asymmetry, complex [ncf_fit][nct_fit] like the reference's array (the values
        are real; NaN where a chunk fails).  Runs fit_thetatheta first if ththeta is not
        set.  All chunks run through ththmod.asymmetry_batch; ``pool`` must be None (see
        fit_thetatheta)."""
        if pool is not None:
            raise ValueError("calc_asymmetry on the GPU path takes pool=None "
                             "(CUDA is not fork-safe); chunks are batched on "
                             "the device instead")
        if not hasattr(self, "ththeta"):
            self.fit_thetatheta(verbose=verbose)
        self.asymmetry = np.zeros((self.ncf_fit, self.nct_fit), dtype=complex)
        for a, cf, ct in thth.asymmetry_batch(self._asymmetry_params(verbose)):
            self.asymmetry[cf, ct] = a

    def thetatheta_chunks(self, verbose=False, pool=None, memmap=False, group=None):
        """Phase retrieval on every half-overlapping retrieval chunk
        (reference dynspec.py:1765-1828) -> self.chunks [ncf_ret][nct_ret][cwf][cwt].
        ``pool`` must be None (see fit_thetatheta); memmap is not supported.
        Under torch.distributed (one process per GPU) the chunks are
        block-partitioned over the ranks of ``group`` and all-gathered, the
        counterpart of the reference's ``pool.map`` over chunks (:1815-1828)."""
        if pool is not None:
            raise ValueError("thetatheta_chunks on the GPU path takes pool=None "
                             "(CUDA is not fork-safe)")
        if memmap:
            raise NotImplementedError("memmap chunk storage is outside the GPU path")
        if not hasattr(self, "ththeta"):
            self.fit_thetatheta(verbose=verbose)
        from . import sharding
        pars = []
        for cf in range(self.ncf_ret):
            fs = slice(cf * (self.cwf // 2), cf * (self.cwf // 2) + self.cwf)
            freq2 = np.copy(self.freqs[fs]).astype(np.float64)
            freq = freq2.mean()
            eta = self.ththeta * (self.fref / freq) ** 2
            for ct in range(self.nct_ret):
                ts = slice(ct * (self.cwt // 2), ct * (self.cwt // 2) + self.cwt)
                time2 = np.copy(self.times[ts]).astype(np.float64)
                dspec2 = np.copy(self.dyn[fs, ts]).astype(np.float64)
                dspec2 -= np.nanmean(dspec2)
                dspec2 = np.nan_to_num(dspec2)
                pars.append((dspec2, self.edges * (freq / self.fref), time2, freq2, eta, ct, cf,
                             self.npad, self.thth_tau_mask, verbose))

        def one(p):
            e = thth.single_chunk_retrieval(p)[0]
            return np.concatenate((e.real.ravel(), e.imag.ravel()))

        L = self.cwf * self.cwt
        flat = sharding.sharded_map(one, pars, 2 * L, group)
        self.chunks = (flat[:, :L] + 1j * flat[:, L:]).reshape(
            self.ncf_ret, self.nct_ret, self.cwf, self.cwt)

    def calc_wavefield(self, verbose=False, pool=None, gs=False, memmap=False,
                       niter=1):
        """Mosaic the retrieved chunks into self.wavefield (reference
        dynspec.py:1830-1856); gs=True refines it with ``niter``
        Gerchberg-Saxton iterations."""
        if not hasattr(self, "chunks"):
            self.thetatheta_chunks(verbose=verbose, pool=pool, memmap=memmap)
        self.wavefield = thth.mosaic(self.chunks)
        if gs:
            self.gerchberg_saxton(verbose=verbose, pool=pool, niter=niter)

    def gerchberg_saxton(self, niter=1, verbose=False, pool=None):
        """Gerchberg-Saxton refinement of self.wavefield: measured amplitude
        where the dynamic spectrum is finite and positive, causality
        (tau < 0 zeroed) in between (reference dynspec.py:1858-1896).  The
        wavefield must have power-of-two sizes."""
        import torch
        from . import _device as D, _lib
        self.calc_wavefield(verbose=verbose, pool=pool)
        n0, n1 = self.wavefield.shape
        d = np.asarray(self.dyn[:n0, :n1], dtype=np.float64)
        pos = np.isfinite(d) * (d > 0)
        tau = U.value(thth.fft_axis(np.asarray(self.freqs[:n0], dtype=np.float64), "us"), "us")
        W = self.wavefield * np.sqrt(d[pos].mean() / np.abs(self.wavefield[pos] ** 2).mean())
        W[pos] = np.sqrt(d[pos]) * np.exp(1j * np.angle(W[pos]))
        if niter > 0:
            amp = np.full((n0, n1), np.nan, dtype=np.float32)
            amp[pos] = np.sqrt(d[pos])
            rowmask = np.fft.ifftshift(tau < 0).astype(np.uint8)     # unshifted row order
            wd, ad, md = D.upload_f32(W), D.upload(amp), D.upload(rowmask)
            _lib.check(_lib.lib.sb_gerchberg_saxton_f32(wd.data_ptr(), ad.data_ptr(),
                                                        md.data_ptr(), n0, n1, int(niter),
                                                        D.stream_ptr()))
            a = wd.cpu().numpy()
            W = a[..., 0].astype(np.float64) + 1j * a[..., 1].astype(np.float64)
        self.wavefield = W
