"""CUDA-native mirror of scintools.ththmod's curvature-search API.

Same function names, argument order and failure behaviour as the reference
(scintools/ththmod.py); the arithmetic runs in libscint_b200 on the GPU:

  fft_axis       ththmod.py:473-493   (host numpy: bit-identical axes)
  thth_map       ththmod.py:56-116    -> sb_thth_map
  thth_redmap    ththmod.py:119-173   -> sb_thth_map + crop
  Eval_calc      ththmod.py:371-401   -> sb_eta_sweep (one eta)
  eta_sweep      the eta loop of single_search, ththmod.py:789-811 (batched)
  chisq_calc     ththmod.py:330-368   -> sb_chisq_sweep (one eta)
  chisq_sweep    the chisq_calc loop of THTHSample.ipynb's chi-square search
                 (batched; host: per-curvature rev_map centres, / N)
  single_search  ththmod.py:715-895   -> sb_cs_f32 + sb_eta_sweep + host fit
  VLBI_chunk_retrieval ththmod.py:1223-1387 -> sb_cs_f32 / sb_cs_c2c_f32 +
                 sb_vlbi_retrieval (host: rev_map centres, input checks)
  calc_asymmetry ththmod.py:2385-2463 -> sb_cs_f32 + sb_asymmetry_batch (one chunk)
  asymmetry_batch the chunk loop of Dynspec.calc_asymmetry (batched per padded shape)
  rotInit, rotMos, rotFit, rotDer, fullMos, fullMosFit, fullMosGrad, fullMosHess
                 ththmod.py:1708-2310 -> sb_mosaic_* (MosaicModel keeps the chunks
                 resident; rotInit's scalar recurrence runs on the host)
  svd_model      ththmod.py:18-35 / scint_utils.py:705-729 -> sb_svd_topk +
                 sb_svd_apply (the top nmodes triplets only; Dynspec.correct_dyn
                 uses the same driver)
  min_edges      ththmod.py:1671-1705 (host)
  chi_par        ththmod.py:38-53     (host)

``CS`` may be a numpy array (uploaded on every call, like the reference's
per-call semantics) or a ``DeviceCS`` that keeps the spectrum resident.
There is no CPU fallback.

Provenance: ``peak_fit`` (ththmod.py:813-859), ``mask_func`` / ``mosaic``
(:1478-1554) and ``min_edges`` (:1671-1705) are the reference's host code with
the units stripped, line for line -- sequential numpy / scipy glue that stays
on the host in both implementations and must give identical numbers.  Restated
reference code, not new design.
"""
import ctypes
import warnings

import numpy as np
from scipy.optimize import curve_fit

from . import _device as D
from . import _lib
from . import units as U

DEFAULT_TOL = 2e-5


def chi_par(x, A, x0, C):
    """Parabola for fitting to the eigenvalue curve (ththmod.py:38-53)."""
    return A * (x - x0) ** 2 + C


def unit_checks(var, name, desired):
    """Reference: ththmod.py:1639-1668.  Returns the float64 value in the
    desired unit ('us', 'mHz', 's3', 's', 'MHz')."""
    return U.value(var, desired)


def fft_axis(x, unit, pad=0):
    """Fourier-conjugate coordinates (ththmod.py:473-493).

    ``unit`` may be the strings 'mHz' / 'us' or the astropy units; ``x`` is in
    s (for mHz) or MHz (for us) when it carries no unit."""
    uname = unit if isinstance(unit, str) else str(unit)
    if uname not in ("mHz", "us"):
        raise ValueError("fft_axis: unit must be mHz or us, got %r" % (unit,))
    xv = U.value(x, "s" if uname == "mHz" else "MHz")
    f = np.fft.fftfreq((pad + 1) * xv.shape[0], xv[1] - xv[0])
    if uname == "mHz":
        f = f * 1.0e3
    return U.wrap(np.fft.fftshift(f), uname, like=x)


class DeviceCS:
    """A conjugate spectrum resident in HBM.

    full: float32 tensor [ntau][nfd][2] (fftshifted, like the reference's CS).
    half (``nfd`` given): [ntau][pitch][2] holding only the fd >= 0 columns
    (unshifted k = 0..nfd/2) of the CS of a REAL dynamic spectrum; the other
    half is its Hermitian mirror and is never materialised."""

    def __init__(self, tensor, nfd=None, ncols_valid=None, bound=None):
        assert tensor.dim() == 3 and tensor.shape[2] == 2
        self.t = tensor
        # device float: upper bound of max |CS| (sb_cs_bound_f32) or None -> the sweep scans
        self.bound = bound
        self.half = nfd is not None
        self.pitch = int(tensor.shape[1])
        self.shape = (int(tensor.shape[0]), int(nfd) if self.half else self.pitch)
        # half-plane only: number of fd >= 0 columns that were computed
        self.ncols_valid = ncols_valid if ncols_valid is not None else \
            (self.shape[1] // 2 + 1 if self.half else self.shape[1])

    @classmethod
    def from_numpy(cls, CS):
        CS = np.asarray(CS)
        if not np.iscomplexobj(CS):
            CS = CS.astype(np.complex128)   # abs(CS) of the incoherent mode
        return cls(D.upload_f32(CS))

    def numpy(self):
        """The full fftshifted complex128 array (expands a half-plane CS)."""
        a = self.t.cpu().numpy()
        if not self.half:
            return (a[..., 0] + 1j * a[..., 1]).astype(np.complex128)
        ntau, nfd = self.shape
        h = nfd // 2
        if self.ncols_valid < h + 1:
            raise ValueError("this DeviceCS holds only the first %d fd columns "
                             "(built with fd_max); it cannot be expanded"
                             % self.ncols_valid)
        a = a[:, :h + 1]                         # drop the pitch padding
        pos = (a[..., 0] + 1j * a[..., 1]).astype(np.complex128)   # unshifted columns 0..h
        full = np.empty((ntau, nfd), dtype=np.complex128)
        full[:, h:] = pos[:, :h]                 # shifted columns h..nfd-1
        full[:, 0] = pos[:, h]                   # Nyquist column
        rows = (ntau - np.arange(ntau)) % ntau   # mirrored (shifted) row index
        full[:, 1:h] = np.conj(pos[rows][:, h - 1:0:-1])
        return full


def _as_device_cs(CS):
    return CS if isinstance(CS, DeviceCS) else DeviceCS.from_numpy(CS)


def theta_centres(edges):
    """Recentred bin centres, ththmod.py:83-84 (same numpy expressions)."""
    edges = np.asarray(edges, dtype=np.float64)
    th = (edges[1:] + edges[:-1]) / 2
    th = th - th[np.abs(th) == np.abs(th).min()]
    return np.ascontiguousarray(th)


class _Geom:
    """Host-side evaluation of the scalars of thth_map / thth_redmap with the
    reference's own expressions, packed into struct sb_thth_geom."""

    def __init__(self, cs, tau, fd, edges, coherent=True):
        tau = U.value(tau, "us")
        fd = U.value(fd, "mHz")
        edges = U.value(edges, "mHz")
        if cs is not None and cs.shape != (tau.shape[0], fd.shape[0]):
            raise ValueError("CS shape %r does not match (len(tau), len(fd)) "
                             "= (%d, %d)" % (cs.shape, tau.shape[0], fd.shape[0]))
        self.cs = cs
        self.th = theta_centres(edges)
        self.th_dev = D.upload(self.th)
        g = _lib.ThthGeom()
        g.cs = cs.t.data_ptr() if cs is not None else None
        g.ntau, g.nfd = tau.shape[0], fd.shape[0]
        g.tau0 = float(tau[0])
        g.dtau = float(np.diff(tau).mean())
        g.tau_absmax = float(np.abs(tau.max()))
        g.fd0 = float(fd[0])
        g.dfd = float(np.diff(fd).mean())
        g.fd_half = float(np.abs(fd.max()) / 2)
        g.th_cents = self.th_dev.data_ptr()
        g.th_cents_host = self.th.ctypes.data
        g.n_th = self.th.shape[0]
        g.coherent = 1 if coherent else 0
        g.cs_half = 1 if (cs is not None and cs.half) else 0
        g.cs_pitch = cs.pitch if cs is not None else fd.shape[0]
        g.cs_valid_cols = int(cs.ncols_valid) if (cs is not None and cs.half) else 0
        g.cs_bound = cs.bound.data_ptr() if (cs is not None and cs.bound is not None) else None
        self.g = g
        if cs is not None and cs.half and cs.ncols_valid < fd.shape[0] // 2 + 1:
            need = needed_fd_columns(fd, edges)
            if need is None or need > cs.ncols_valid:
                raise ValueError("this DeviceCS was built for a narrower theta "
                                 "grid (%d fd columns); rebuild it" % cs.ncols_valid)

    @property
    def ref(self):
        return ctypes.byref(self.g)


_pinned_pool = {}


def _pinned_take(neta):
    """Four pinned host buffers (eigs f64, status / nred / iters i32) of length neta."""
    import torch
    free = _pinned_pool.setdefault(neta, [])
    if free:
        return free.pop()
    return [torch.empty((neta,), dtype=dt, pin_memory=True)
            for dt in (torch.float64, torch.int32, torch.int32, torch.int32)]


def _pinned_give(bufs):
    free = _pinned_pool.setdefault(int(bufs[0].shape[0]), [])
    if len(free) < 4:
        free.append(bufs)


class _SweepJob:
    """An eta sweep in flight on the current stream: device outputs, pinned host
    mirrors (asynchronous device->host copies) and the event that marks them
    complete.  ``finish()`` waits for the event only -- the stream keeps running
    whatever was enqueued after the sweep."""

    def __init__(self, cs, geom, d_etas, neta, tol, max_iter, pinned):
        import torch
        self.keep = (cs, geom, d_etas)           # referenced until the kernels ran
        self.eigs = D.empty((neta,), torch.float64)
        self.status = D.empty((neta,), torch.int32)
        self.nred = D.empty((neta,), torch.int32)
        self.iters = D.empty((neta,), torch.int32)
        _lib.check(_lib.lib.sb_eta_sweep(geom.ref, d_etas.data_ptr(), neta, tol,
                                         max_iter, self.eigs.data_ptr(),
                                         self.status.data_ptr(), self.nred.data_ptr(),
                                         self.iters.data_ptr(), D.stream_ptr()))
        self.host = None
        if pinned:
            # pinned read-back buffers come from a small pool: a fresh cudaHostAlloc per
            # job would synchronise the device and serialise the pipeline
            self.host = _pinned_take(neta)
            for h, t in zip(self.host, (self.eigs, self.status, self.nred, self.iters)):
                h.copy_(t, non_blocking=True)
            self.event = torch.cuda.Event()
            self.event.record()

    def finish(self, return_info=False):
        if self.host is not None:
            self.event.synchronize()
            out, st, nred, iters = [h.numpy().copy() for h in self.host]
            _pinned_give(self.host)
            self.host = None
        else:
            out = self.eigs.cpu().numpy()
            st = self.status.cpu().numpy()
            nred = self.nred.cpu().numpy()
            iters = self.iters.cpu().numpy()
        self.keep = None
        # iteration cap hit without convergence: ARPACK raises ArpackNoConvergence in
        # the reference and the eta loop stores NaN (ththmod.py:795-799)
        out[(st & 8) != 0] = np.nan
        if return_info:
            return out, dict(status=st, nred=nred, iters=iters)
        return out


def _sweep_launch(CS, tau, fd, etas, edges, coher=True, tol=DEFAULT_TOL, max_iter=0,
                  pinned=False):
    cs = _as_device_cs(CS)
    geom = _Geom(cs, tau, fd, edges, coher)
    ev = np.ascontiguousarray(np.atleast_1d(U.value(etas, "s3")))
    return _SweepJob(cs, geom, D.upload(ev), ev.shape[0], tol, max_iter, pinned)


def eta_sweep(CS, tau, fd, etas, edges, coher=True, tol=DEFAULT_TOL,
              max_iter=0, return_info=False):
    """Largest-eigenvalue curve over ``etas`` (float64 array, NaN where the
    reference's try/except would have stored NaN, ththmod.py:789-799).

    One launch sequence for the whole sweep: crop masks, gather + Hermitian
    fill, Lanczos; one eta per thread block."""
    return _sweep_launch(CS, tau, fd, etas, edges, coher, tol, max_iter).finish(return_info)


def Eval_calc(CS, tau, fd, eta, edges):
    """Dominant eigenvalue of the theta-theta matrix (ththmod.py:371-401).

    Raises like the reference where scipy/numpy would have raised (callers such
    as single_search turn that into NaN)."""
    eigs, info = eta_sweep(CS, tau, fd, np.array([float(U.value(eta, "s3"))]),
                           edges, True, return_info=True)
    st = int(info["status"][0])
    if st & 1:
        raise IndexError("theta-theta point maps outside the conjugate "
                         "spectrum (fd_inv < -nfd)")
    if st & 2:
        raise ValueError("starting vector is zero (row n//2 of the "
                         "theta-theta matrix is empty)")
    if st & 4:
        raise TypeError("theta-theta matrix too small for eigsh (n < 3)")
    return float(eigs[0])


def thth_map(CS, tau, fd, eta, edges, hermetian=True, return_indices=False):
    """Map from the conjugate spectrum to theta-theta space (ththmod.py:56-116).

    Returns the complex128 N x N matrix; with ``return_indices`` also the
    bit-exact tau_inv, fd_inv (int32) and pnts (bool) arrays of
    ththmod.py:94-100."""
    import torch
    cs = _as_device_cs(CS)
    geom = _Geom(cs, tau, fd, edges, True)
    n = geom.g.n_th
    out = D.empty((n, n, 2), torch.float32)
    err = D.zeros((1,), torch.int32)
    ti = fi = pn = None
    if return_indices:
        ti = D.empty((n, n), torch.int32)
        fi = D.empty((n, n), torch.int32)
        pn = D.empty((n, n), torch.uint8)
    _lib.check(_lib.lib.sb_thth_map(geom.ref, float(U.value(eta, "s3")),
                                    1 if hermetian else 0, out.data_ptr(),
                                    D.ptr(ti), D.ptr(fi), D.ptr(pn), 0,
                                    err.data_ptr(), D.stream_ptr()))
    if int(err.cpu()[0]) & 1:
        raise IndexError("index out of bounds (fd_inv < -nfd), ththmod.py:104")
    a = out.cpu().numpy()
    thth = a[..., 0].astype(np.float64) + 1j * a[..., 1].astype(np.float64)
    if return_indices:
        return thth, ti.cpu().numpy(), fi.cpu().numpy(), pn.cpu().numpy().astype(bool)
    return thth


def th_points(tau, fd, eta, edges):
    """Crop mask of thth_redmap (ththmod.py:153-156), evaluated on the GPU."""
    import torch
    geom = _Geom(None, tau, fd, edges, True)
    mask = D.empty((geom.g.n_th,), torch.uint8)
    _lib.check(_lib.lib.sb_thth_map(geom.ref, float(U.value(eta, "s3")), 1, 0,
                                    0, 0, 0, mask.data_ptr(), 0,
                                    D.stream_ptr()))
    return mask.cpu().numpy().astype(bool)


def thth_redmap(CS, tau, fd, eta, edges, hermetian=True):
    """Largest fully-covered square of the theta-theta map (ththmod.py:119-173).
    Returns (thth_red, edges_red)."""
    import torch
    cs = _as_device_cs(CS)
    geom = _Geom(cs, tau, fd, edges, True)
    n = geom.g.n_th
    out = D.empty((n, n, 2), torch.float32)
    err = D.zeros((1,), torch.int32)
    mask = D.empty((n,), torch.uint8)
    _lib.check(_lib.lib.sb_thth_map(geom.ref, float(U.value(eta, "s3")),
                                    1 if hermetian else 0, out.data_ptr(), 0,
                                    0, 0, mask.data_ptr(), err.data_ptr(),
                                    D.stream_ptr()))
    if int(err.cpu()[0]) & 1:
        raise IndexError("index out of bounds (fd_inv < -nfd), ththmod.py:104")
    sel = mask.cpu().numpy().astype(bool)
    a = out.cpu().numpy()
    thth = a[..., 0].astype(np.float64) + 1j * a[..., 1].astype(np.float64)
    red = thth[sel, :][:, sel]
    er = geom.th[sel]
    er = (er[:-1] + er[1:]) / 2
    step = np.diff(er).mean()
    edges_red = np.concatenate((np.array([er[0] - step]), er,
                                np.array([er[-1] + step])))
    return red, U.wrap(edges_red, "mHz", like=edges)


def needed_fd_columns(fd, edges):
    """How many fd >= 0 columns of the conjugate spectrum a theta-theta map on
    ``edges`` can touch: above the diagonal fd = theta_j - theta_i lies in
    (0, max(theta) - min(theta)].  Returns None when the grid reaches past the
    fd axis (gathers wrap to negative fd -> every column may be needed)."""
    fd = U.value(fd, "mHz")
    th = theta_centres(U.value(edges, "mHz"))
    dfd = float(np.diff(fd).mean())
    span = float(th.max() - th.min())
    n = fd.shape[0]
    if n % 2 or not np.isfinite(span) or dfd <= 0 or fd[n // 2] != 0.0:
        return None
    cmax = int(np.floor(span / dfd + 0.5)) + 2          # +2 bins of slack
    if cmax >= n // 2:
        return None
    return cmax + 1


def conjugate_spectrum(dspec2, npad, pad_value=None, tau=None, tau_mask=0.0,
                       half=True, ncols_keep=None):
    """CS stage of single_search (ththmod.py:777-787): pad, fft2, fftshift,
    zero |tau| < tau_mask.  Returns a DeviceCS.  ``pad_value=None`` pads with
    dspec2.mean() like single_search; 0.0 reproduces
    Dynspec.thetatheta_single (dynspec.py:1575-1579).  ``half=True`` keeps only
    the fd >= 0 half on the device (the spectrum of a real array is Hermitian;
    ``.numpy()`` still returns the full array).  ``ncols_keep`` (half-plane
    only; see needed_fd_columns) restricts the transform to the fd columns a
    given theta grid can reach.  A complex ``dspec2`` (a VLBI visibility) goes
    through sb_cs_c2c_f32 and always gives the full plane (``half`` and
    ``ncols_keep`` are ignored; ``pad_value=None`` pads with its complex mean)."""
    import torch
    if not isinstance(dspec2, torch.Tensor) and np.iscomplexobj(dspec2):
        return _conjugate_spectrum_c2c(np.asarray(dspec2), npad, pad_value, tau, tau_mask)
    if isinstance(dspec2, torch.Tensor):     # already staged on the device (search_batch)
        dd = dspec2
        if dd.dtype != torch.float32 or not dd.is_cuda or dd.dim() != 2 or not dd.is_contiguous():
            raise ValueError("device dynamic spectra must be contiguous float32 [nf][nt]")
    else:
        dd = D.upload_f32(np.asarray(dspec2))
    nf, nt = int(dd.shape[0]), int(dd.shape[1])
    if pad_value is None:
        pad_value = float("nan")     # = dspec2.mean(), evaluated on the device
    NF, NT = (npad + 1) * nf, (npad + 1) * nt
    if (NF & (NF - 1)) or (NT & (NT - 1)) or NT < 16 or NF < 4:
        half = False        # chirp-z path for arbitrary lengths: full plane
    pitch = NT // 2 + 16 if half else NT
    cs = D.empty((NF, pitch, 2), torch.float32)
    mask = _tau_rowmask(tau, tau_mask)
    keep = int(ncols_keep) if (half and ncols_keep) else 0
    _lib.check(_lib.lib.sb_cs_f32(dd.data_ptr(), nf, nt, npad, float(pad_value),
                                  D.ptr(mask), 1 if half else 0, pitch, keep,
                                  cs.data_ptr(), D.stream_ptr()))
    bound = D.empty((1,), torch.float32)
    _lib.check(_lib.lib.sb_cs_bound_f32(dd.data_ptr(), nf, nt, npad, float(pad_value),
                                        bound.data_ptr(), D.stream_ptr()))
    return DeviceCS(cs, nfd=NT if half else None,
                    ncols_valid=keep if keep else None, bound=bound)


def _tau_rowmask(tau, tau_mask):
    if tau is None or tau_mask is None:
        return None
    m = np.abs(U.value(tau, "us")) < float(U.value(tau_mask, "us"))
    return D.upload(m.astype(np.uint8)) if m.any() else None


def _conjugate_spectrum_c2c(dspec2, npad, pad_value, tau, tau_mask):
    """conjugate_spectrum of a complex chunk (a VLBI visibility) via sb_cs_c2c_f32:
    always the full plane, no magnitude bound."""
    import torch
    if dspec2.ndim != 2:
        raise ValueError("dynamic spectrum must be 2-D, got shape %r" % (dspec2.shape,))
    nf, nt = dspec2.shape
    dd = D.upload_f32(dspec2.astype(np.complex128))
    pad = complex(np.nan, 0.0) if pad_value is None else complex(pad_value)
    NF, NT = (npad + 1) * nf, (npad + 1) * nt
    cs = D.empty((NF, NT, 2), torch.float32)
    mask = _tau_rowmask(tau, tau_mask)
    _lib.check(_lib.lib.sb_cs_c2c_f32(dd.data_ptr(), nf, nt, npad, pad.real, pad.imag,
                                      D.ptr(mask), cs.data_ptr(), D.stream_ptr()))
    return DeviceCS(cs)


def peak_fit(etas, eigs, fw):
    """Parabola fit of the eigenvalue peak (ththmod.py:813-859); stays on the
    host (scipy curve_fit) as in the reference.  NaNs on failure."""
    try:
        etas = np.asarray(etas, dtype=np.float64)
        eigs = np.asarray(eigs, dtype=np.float64)
        good = np.isfinite(eigs)
        etas, eigs = etas[good], eigs[good]
        pk = etas[eigs == eigs.max()]
        win = np.abs(etas - pk) < fw * pk
        ef, gf = etas[win], eigs[win]
        C = gf.max()
        x0 = ef[gf == C][0]
        if x0 == ef[0]:
            A = (gf[-1] - C) / ((ef[-1] - x0) ** 2)
        else:
            A = (gf[0] - C) / ((ef[0] - x0) ** 2)
        popt, _ = curve_fit(chi_par, ef, gf, p0=np.array([A, x0, C]))
        eta_fit = popt[1]
        eta_sig = np.sqrt((gf - chi_par(ef, *popt)).std() / np.abs(popt[0]))
        return eta_fit, eta_sig, popt
    except Exception:  # noqa: BLE001  (reference: bare except -> NaN)
        return np.nan, np.nan, None


def single_search(params):
    """Curvature search for one chunk (ththmod.py:715-895).

    ``params`` is the reference's 12-element list
    [dspec2, freq, time, etas, edges, name, plot, fw, npad, coher, tauMask,
    verbose]; returns (eta_fit, eta_sig, freq.mean(), time.mean(), eigs).
    Plotting is not part of the hot path: ``plot=True`` raises."""
    return _search_finish(_search_launch(params, None))


def _search_launch(params, staged, pinned=False):
    """Enqueue the device work of one single_search (CS + sweep) on the current
    stream; nothing here waits for the GPU."""
    (dspec2, freq, time, etas, edges, name, plot, fw, npad, coher, tauMask,
     verbose) = params
    if plot:
        raise NotImplementedError("plotting is outside the GPU hot path; "
                                  "use scintools.ththmod.plot_func on the "
                                  "returned eigenvalues")
    if staged is not None:
        dspec2 = staged
    time_v = U.value(time, "s")
    freq_v = U.value(freq, "MHz")
    etas_v = U.value(etas, "s3")
    try:
        theta_centres(U.value(edges, "mHz"))
    except ValueError:
        # every thth_map raises (the recentring ties on an even grid); the reference's eta
        # loop stores NaN for each curvature
        return _NanSweep(np.atleast_1d(etas_v).shape[0]), params, time_v, freq_v, etas_v
    fd = U.value(fft_axis(time_v, "mHz", npad), "mHz")
    tau = U.value(fft_axis(freq_v, "us", npad), "us")
    cs = conjugate_spectrum(dspec2, npad, None, tau, tauMask,
                            ncols_keep=needed_fd_columns(fd, edges))
    job = _sweep_launch(cs, tau, fd, etas_v, edges, bool(coher), pinned=pinned)
    return job, params, time_v, freq_v, etas_v


class _NanSweep:
    """The eigenvalues of a sweep that fails at every curvature."""

    def __init__(self, neta):
        self.neta = neta

    def finish(self):
        return np.full(self.neta, np.nan)


def _search_finish(launched):
    """Wait for the eigenvalues of a launched search and fit the peak on the host."""
    job, params, time_v, freq_v, etas_v = launched
    (_, freq, time, etas, _, _, _, fw, _, _, _, verbose) = params
    eigs = job.finish()
    eta_fit, eta_sig, _ = peak_fit(etas_v, eigs, fw)
    if verbose:
        print("Chunk completed (eta = %s +- %s at %s)" %
              (eta_fit, eta_sig, freq_v.mean()), flush=True)
    return (U.wrap(eta_fit, "s3", like=etas), U.wrap(eta_sig, "s3", like=etas),
            U.wrap(freq_v.mean(), "MHz", like=freq),
            U.wrap(time_v.mean(), "s", like=time), eigs)


_copy_stream = {}


def search_batch(params_list):
    """single_search over a sequence of chunks -- the loop of
    Dynspec.fit_thetatheta (dynspec.py:1680-1712) / ``pool.map(single_search,
    pars)`` (:1715-1719) -- as a two-deep software pipeline:

      * the host->device copy of chunk i+1 runs on a persistent copy stream
        while chunk i is swept (asynchronous when the dynamic spectra sit in
        pinned host memory; float64 input is narrowed on the device);
      * the device work of chunk i+1 (CS + sweep + asynchronous read-back of
        the eigenvalues into pinned memory) is enqueued BEFORE the host waits
        for chunk i and fits its parabola, so the GPU never idles behind the
        host-side scipy fit.

    Returns the list of single_search results, in order."""
    import torch
    params_list = list(params_list)
    if not params_list:
        return []
    dev = D.device()
    main = torch.cuda.current_stream()
    side = _copy_stream.get(dev)
    if side is None:
        side = _copy_stream[dev] = torch.cuda.Stream()

    def stage(p):
        a = np.asarray(p[0])
        if a.dtype not in (np.float32, np.float64):
            a = a.astype(np.float64)
        with torch.cuda.stream(side):
            t = torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)
            if t.dtype != torch.float32:
                t32 = torch.empty(t.shape, dtype=torch.float32, device=t.device)
                _lib.check(_lib.lib.sb_convert_f64_f32(t.data_ptr(), t32.data_ptr(), t.numel(),
                                                       side.cuda_stream))
                t = t32
            ev = torch.cuda.Event()
            ev.record(side)
        t.record_stream(main)
        return t, ev

    out = []
    staged = stage(params_list[0])
    prev = None
    for i, p in enumerate(params_list):
        t, ev = staged
        main.wait_event(ev)
        launched = _search_launch(p, t, pinned=True)
        staged = stage(params_list[i + 1]) if i + 1 < len(params_list) else None
        if prev is not None:
            out.append(_search_finish(prev))
        prev = launched
    out.append(_search_finish(prev))
    return out


# ---------------------------------------------------------------------------
# "thin" (arclet) theta-theta: two-curvature map + largest singular value
# ---------------------------------------------------------------------------
class _ThinGeom(_Geom):
    """sb_thth_geom with the conventions of two_curve_map (ththmod.py:1585-
    1617): plain bin centres, offsets tau[1] / fd[1], tau.max()."""

    def __init__(self, cs, tau, fd, edges1, edges2):
        tauv = U.value(tau, "us")
        fdv = U.value(fd, "mHz")
        e1 = np.asarray(U.value(edges1, "mHz"), dtype=np.float64)
        e2 = np.asarray(U.value(edges2, "mHz"), dtype=np.float64)
        if cs.shape != (tauv.shape[0], fdv.shape[0]):
            raise ValueError("CS shape does not match (len(tau), len(fd))")
        self.cs = cs
        self.th = np.ascontiguousarray((e1[1:] + e1[:-1]) / 2)
        self.th2 = np.ascontiguousarray((e2[1:] + e2[:-1]) / 2)
        self.th_dev = D.upload(self.th)
        self.th2_dev = D.upload(self.th2)
        g = _lib.ThthGeom()
        g.cs = cs.t.data_ptr()
        g.ntau, g.nfd = tauv.shape[0], fdv.shape[0]
        g.tau0 = float(tauv[1])
        g.dtau = float(np.diff(tauv).mean())
        g.tau_absmax = float(tauv.max())
        g.fd0 = float(fdv[1])
        g.dfd = float(np.diff(fdv).mean())
        g.fd_half = 0.0
        g.th_cents = self.th_dev.data_ptr()
        g.th_cents_host = self.th.ctypes.data
        g.n_th = self.th.shape[0]
        g.coherent = 1
        g.cs_half = 1 if cs.half else 0
        g.cs_pitch = cs.pitch
        self.g = g
        if cs.half and cs.ncols_valid < fdv.shape[0] // 2 + 1:
            raise ValueError("thin theta-theta needs a DeviceCS with all fd columns")


def thin_sweep(CS, tau, fd, etas, edges, edgesArclet, centerCut, etasArclet=None,
               power=False, tol=DEFAULT_TOL, max_iter=0, return_info=False):
    """Largest singular value of the two-curvature theta-theta map for every
    curvature (the eta loop of single_search_thin, ththmod.py:589-627; one
    singularvalue_calc per eta, :496-512).  NaN where numpy would raise."""
    import torch
    cs = _as_device_cs(CS)
    geom = _ThinGeom(cs, tau, fd, edges, edgesArclet)
    e1 = np.ascontiguousarray(np.atleast_1d(U.value(etas, "s3")))
    e2 = e1 if etasArclet is None else \
        np.ascontiguousarray(np.atleast_1d(U.value(etasArclet, "s3")))
    neta = e1.shape[0]
    d1, d2 = D.upload(e1), D.upload(e2)
    sv = D.empty((neta,), torch.float64)
    aux = [D.empty((neta,), torch.int32) for _ in range(4)]
    _lib.check(_lib.lib.sb_thin_sweep(
        geom.ref, geom.th2_dev.data_ptr(), geom.th2.shape[0],
        float(U.value(centerCut, "mHz")), 1 if power else 0, d1.data_ptr(),
        d2.data_ptr(), neta, tol, max_iter, sv.data_ptr(), aux[0].data_ptr(),
        aux[1].data_ptr(), aux[2].data_ptr(), aux[3].data_ptr(), D.stream_ptr()))
    out = sv.cpu().numpy()
    if return_info:
        return out, dict(status=aux[0].cpu().numpy(), n1=aux[1].cpu().numpy(),
                         n2=aux[2].cpu().numpy(), iters=aux[3].cpu().numpy())
    return out


def two_curve_map(CS, tau, fd, eta1, edges1, eta2, edges2):
    """Two-curvature theta-theta map (ththmod.py:1557-1636).
    Returns (thth_red, edges_red1, edges_red2)."""
    import torch
    cs = _as_device_cs(CS)
    geom = _ThinGeom(cs, tau, fd, edges1, edges2)
    e1v, e2v = float(U.value(eta1, "s3")), float(U.value(eta2, "s3"))
    n1, n2 = geom.th.shape[0], geom.th2.shape[0]
    out = D.empty((n2, n1, 2), torch.float32)
    err = D.zeros((1,), torch.int32)
    _lib.check(_lib.lib.sb_thin_map(geom.ref, geom.th2_dev.data_ptr(), n2, 0, e1v, e2v,
                                    out.data_ptr(), err.data_ptr(), D.stream_ptr()))
    if int(err.cpu()[0]) & 1:
        raise IndexError("index out of bounds (fd_inv < -nfd), ththmod.py:1614")
    a = out.cpu().numpy()
    thth = a[..., 0].astype(np.float64) + 1j * a[..., 1].astype(np.float64)
    tauv = U.value(tau, "us")
    ed1 = np.asarray(U.value(edges1, "mHz"), dtype=np.float64)
    ed2 = np.asarray(U.value(edges2, "mHz"), dtype=np.float64)
    p1 = np.abs(geom.th) < np.sqrt(tauv.max() / e1v)
    p2 = np.abs(geom.th2) < np.sqrt(tauv.max() / e2v)
    er1 = np.zeros(p1.sum() + 1)
    er1[:-1] = ed1[:-1][p1]
    er1[-1] = ed1[1:][p1].max()
    er2 = np.zeros(p2.sum() + 1)
    er2[:-1] = ed2[:-1][p2]
    er2[-1] = ed2[1:][p2].max()
    return (thth[p2, :][:, p1], U.wrap(er1, "mHz", like=edges1),
            U.wrap(er2, "mHz", like=edges2))


def singularvalue_calc(CS, tau, fd, eta, edges, etaArclet, edgesArclet, centerCut):
    """ththmod.py:496-512."""
    sv, info = thin_sweep(CS, tau, fd, np.array([float(U.value(eta, "s3"))]), edges,
                          edgesArclet, centerCut,
                          etasArclet=np.array([float(U.value(etaArclet, "s3"))]),
                          return_info=True)
    if int(info["status"][0]) & 1:
        raise IndexError("theta-theta point maps outside the conjugate spectrum")
    if not np.isfinite(sv[0]):
        raise np.linalg.LinAlgError("SVD did not converge")
    return float(sv[0])


def single_search_thin(params):
    """Thin-arclet curvature search for one chunk (ththmod.py:515-712).
    ``params`` is the reference's 13-element list
    [dspec2, freq, time, etas, edges, name, plot, fw, npad, coher, verbose,
    edgesArclet, centerCut]."""
    (dspec2, freq, time, etas, edges, name, plot, fw, npad, coher, verbose,
     edgesArclet, centerCut) = params
    if plot:
        raise NotImplementedError("plotting is outside the GPU hot path")
    time_v = U.value(time, "s")
    freq_v = U.value(freq, "MHz")
    etas_v = U.value(etas, "s3")
    fd = U.value(fft_axis(time_v, "mHz", npad), "mHz")
    tau = U.value(fft_axis(freq_v, "us", npad), "us")
    cs = conjugate_spectrum(dspec2, npad, None)
    eigs = thin_sweep(cs, tau, fd, etas_v, edges, edgesArclet, centerCut,
                      power=not coher)
    eta_fit, eta_sig, _ = peak_fit(etas_v, eigs, fw)
    if verbose:
        print("Chunk completed (eta = %s +- %s at %s)" %
              (eta_fit, eta_sig, freq_v.mean()), flush=True)
    return (U.wrap(eta_fit, "s3", like=etas), U.wrap(eta_sig, "s3", like=etas),
            U.wrap(freq_v.mean(), "MHz", like=freq),
            U.wrap(time_v.mean(), "s", like=time), eigs)


# ---------------------------------------------------------------------------
# phase retrieval: inverse map, rank-1 model, wavefield of one chunk
# ---------------------------------------------------------------------------
def _c64(t):
    a = t.cpu().numpy()
    return a[..., 0].astype(np.float64) + 1j * a[..., 1].astype(np.float64)


def _hist_edges(tau, fd):
    """The np.histogram2d bin edges of rev_map (ththmod.py:211-216), (fd, tau).  Raises
    numpy's ValueError when either descends, as the reference's rev_map does for a
    descending tau or fd axis (a BasicDyn with descending frequencies, say)."""
    tau, fd = U.value(tau, "us"), U.value(fd, "mHz")
    fe = (np.linspace(0, fd.shape[0], fd.shape[0] + 1) - .5) * (fd[1] - fd[0]) + fd[0]
    te = (np.linspace(0, tau.shape[0], tau.shape[0] + 1) - .5) * (tau[1] - tau[0]) + tau[0]
    for k, e in enumerate((fe, te)):
        if np.any(e[:-1] > e[1:]):
            raise ValueError("`bins[%d]` must be monotonically increasing, when an array" % k)
    return fe, te


def _index_error(th, tau, fd, eta):
    """Does thth_map raise IndexError (fd_inv < -nfd on a point of the pnts mask,
    ththmod.py:94-104) at curvature eta?  The reference's expressions on the host, a
    block of rows at a time; for the error paths of non-ascending axes, where the
    device sweeps that report it cannot run."""
    tau, fd = np.asarray(tau, dtype=np.float64), np.asarray(fd, dtype=np.float64)
    dtau, dfd = np.diff(tau).mean(), np.diff(fd).mean()
    for r0 in range(0, th.shape[0], 256):
        th2 = th[r0:r0 + 256, np.newaxis]
        fd_inv = (((th[np.newaxis, :] - th2) - fd[0] + dfd / 2) // dfd).astype(int)
        tau_inv = (((eta * (th[np.newaxis, :] ** 2 - th2 ** 2)) - tau[0] + dtau / 2)
                   // dtau).astype(int)
        pnts = (tau_inv > 0) * (tau_inv < tau.shape[0]) * (fd_inv < fd.shape[0])
        if np.any(pnts & (fd_inv < -fd.shape[0])):
            return True
    return False


def _check_rev_axes(tau, fd, edges, eta):
    """Before any device work of an entry point whose reference ends in rev_map
    (chisq_calc, VLBI_chunk_retrieval): on a descending axis raise what the reference
    raises first -- IndexError from thth_map, the crop's exception from thth_redmap,
    else rev_map's ValueError.  (A zero theta-theta matrix, whose eigsh error would come
    before rev_map's, also gives the ValueError.)"""
    tau, fd = U.value(tau, "us"), U.value(fd, "mHz")
    try:
        _hist_edges(tau, fd)
    except ValueError:
        th = theta_centres(U.value(edges, "mHz"))
        if _index_error(th, tau, fd, eta):
            raise IndexError("theta-theta point maps outside the conjugate "
                             "spectrum (fd_inv < -nfd)") from None
        _, errs = _rev_centres(th, tau, fd, np.array([eta]), min_crop=0)
        if errs[0] is not None:
            raise errs[0] from None
        raise


def _rev_map_device(thth_dev, n, tau, fd, eta, edges, hermetian):
    """sb_rev_map on a device theta-theta matrix; returns the device recov
    [ntau][nfd][2] (= the reference's ``recov.T`` before any host copy)."""
    import torch
    tau = U.value(tau, "us")
    fd = U.value(fd, "mHz")
    _hist_edges(tau, fd)
    th = theta_centres(U.value(edges, "mHz"))
    if th.shape[0] != n:
        raise ValueError("thth is %d x %d but edges give %d centres" % (n, n, th.shape[0]))
    recov = D.empty((tau.shape[0], fd.shape[0], 2), torch.float32)
    th_dev = D.upload(th)
    _lib.check(_lib.lib.sb_rev_map(
        thth_dev.data_ptr(), n, th_dev.data_ptr(), float(U.value(eta, "s3")),
        float(tau[0]), float(tau[1] - tau[0]), tau.shape[0],
        float(fd[0]), float(fd[1] - fd[0]), fd.shape[0], 1 if hermetian else 0,
        recov.data_ptr(), D.stream_ptr()))
    return recov


def rev_map(thth, tau, fd, eta, edges, hermetian=True):
    """Inverse map from theta-theta to the conjugate spectrum
    (ththmod.py:176-258).  Returns the complex [len(tau)][len(fd)] array."""
    thth = np.asarray(thth)
    n = thth.shape[0]
    if thth.ndim != 2 or thth.shape[1] != n:
        raise ValueError("thth must be square")
    _hist_edges(tau, fd)
    recov =_c64(_rev_map_device(D.upload_f32(thth.astype(np.complex128)), n, tau, fd, eta,
                                 edges, hermetian))
    if not hermetian:
        # the (0, 0) bin holds the zero-Jacobian diagonal points: NaN real part,
        # imaginary part sum(imag / 0) -> nan_to_num (ththmod.py:219-258)
        with np.errstate(divide="ignore", invalid="ignore"):
            h = np.sum(np.diagonal(thth).imag / 0.0)
        if np.isinf(h):
            fe, te = _hist_edges(tau, fd)
            bx = np.searchsorted(fe, 0.0, side="right") - 1
            by = np.searchsorted(te, 0.0, side="right") - 1
            if 0 <= bx < fe.shape[0] - 1 and 0 <= by < te.shape[0] - 1:
                recov[by, bx] = np.nan_to_num(complex(0.0, h))
    return recov


def _top_eigenpair(thth_red):
    """eigsh(thth_red, 1, which='LA') on the device (sb_herm_eigvec)."""
    import torch
    n = thth_red.shape[0]
    a = D.upload_f32(np.asarray(thth_red).astype(np.complex128))
    w = D.empty((1,), torch.float64)
    V = D.empty((n, 2), torch.float32)
    info = D.zeros((2,), torch.int32)
    _lib.check(_lib.lib.sb_herm_eigvec(a.data_ptr(), n, n, 0.0, 0, w.data_ptr(), V.data_ptr(),
                                       info.data_ptr(), D.stream_ptr()))
    wv = float(w.cpu()[0])
    if not np.isfinite(wv):
        raise np.linalg.LinAlgError("theta-theta matrix has a zero start vector / no eigenpair")
    if int(info.cpu()[1]) & 8:
        # iteration cap without convergence: ARPACK raises ArpackNoConvergence here
        raise np.linalg.LinAlgError("top eigenpair did not converge")
    return wv, _c64(V), V


def modeler(CS, tau, fd, eta, edges, hermetian=True):
    """Model theta-theta, conjugate spectrum and dynamic spectrum from the top
    eigenpair (ththmod.py:261-327).  Returns (thth_red, thth2_red, recov, model,
    edges_red, w, V).  Any padded CS size (powers of two take the radix path, other
    sizes the chirp-z inverse); V has an arbitrary global phase, like ARPACK's."""
    import torch
    if not hermetian:
        raise NotImplementedError(
            "modeler(hermetian=False) raises IndexError in the reference "
            "(ththmod.py:316-320) and is not part of the GPU path")
    tauv, fdv = U.value(tau, "us"), U.value(fd, "mHz")
    thth_red, edges_red = thth_redmap(CS, tau, fd, eta, edges, hermetian=True)
    w, V, _ = _top_eigenpair(thth_red)
    thth2_red = np.outer(V, np.conjugate(V)) * np.abs(w)
    n = thth_red.shape[0]
    recov_dev = _rev_map_device(D.upload_f32(thth2_red), n, tauv, fdv, eta, edges_red, True)
    model = D.empty((tauv.shape[0], fdv.shape[0]), torch.float32)
    _lib.check(_lib.lib.sb_ifft2_c2c_f32(recov_dev.data_ptr(), tauv.shape[0], fdv.shape[0], 1,
                                         0, 0, 1.0, 1, model.data_ptr(), D.stream_ptr()))
    return (thth_red, thth2_red, _c64(recov_dev), model.cpu().numpy().astype(np.float64),
            edges_red, w, V)


def single_chunk_retrieval(params):
    """Phase retrieval on one chunk (ththmod.py:1390-1476).  ``params`` is the
    reference's tuple (dspec2, edges, time, freq, eta, idx_t, idx_f, npad,
    tauMask, verbose); returns (model_E, idx_f, idx_t).  A chunk that cannot
    be recovered gives zeros, as in the reference."""
    import torch
    dspec2, edges, time, freq, eta, idx_t, idx_f, npad, tauMask, verbose = params
    dspec2 = np.asarray(dspec2, dtype=np.float64)
    time_v, freq_v = U.value(time, "s"), U.value(freq, "MHz")
    if verbose:
        print("Starting Chunk %s-%s" % (idx_f, idx_t), flush=True)
    fd = U.value(fft_axis(time_v, "mHz", npad), "mHz")
    tau = U.value(fft_axis(freq_v, "us", npad), "us")
    nf, nt = dspec2.shape
    try:
        cs = conjugate_spectrum(dspec2, npad, None, tau, float(U.value(tauMask, "us")))
        thth_red, edges_red = thth_redmap(cs, tau, fd, eta, edges, hermetian=True)
        w, V, _ = _top_eigenpair(thth_red)
        n = thth_red.shape[0]
        ththE = np.zeros((n, n), dtype=np.complex128)
        with np.errstate(invalid="ignore"):
            ththE[n // 2, :] = np.conjugate(V) * np.sqrt(w)
        recov_dev = _rev_map_device(D.upload_f32(ththE), n, tau, fd, eta, edges_red, False)
        out = D.empty((nf, nt, 2), torch.float32)
        _lib.check(_lib.lib.sb_ifft2_c2c_f32(recov_dev.data_ptr(), tau.shape[0], fd.shape[0], 1,
                                             nf, nt, nf * nt / 4.0, 0, out.data_ptr(),
                                             D.stream_ptr()))
        model_E = _c64(out)
        if verbose:
            print("Chunk %s-%s success" % (idx_f, idx_t), flush=True)
    except _lib.SbError:
        # a library error (unsupported size, CUDA failure) is not a data failure:
        # never turn it into a silent all-zero chunk
        raise
    except Exception as e:          # data failures, as in ththmod.py:1470-1475
        print(e, flush=True)
        model_E = np.zeros(dspec2.shape, dtype=complex)
    return (model_E, idx_f, idx_t)


def _rev_centres(th, tau, fd, etas, min_crop=3):
    """rev_map bin centres of modeler for every curvature: theta_centres of the
    edges_red of thth_redmap (ththmod.py:153-170, :204-205), with the
    reference's expressions.  Returns float64 [neta][len(th)] (row k holds the
    cropped count of them) and, per curvature, the exception numpy raises on the
    way (None if none).  Crops of fewer than ``min_crop`` centres are skipped (the
    chi-square path leaves them to the device, which reports SB_ETA_TOO_SMALL);
    with ``min_crop=0`` they give the reference's own exception: IndexError from
    edges_red for 0 or 1 centres, ValueError from the centres of 2."""
    out = np.zeros((etas.shape[0], th.shape[0]))
    errs = [None] * etas.shape[0]
    for k, eta in enumerate(etas):
        sel = ((th ** 2) * eta < np.abs(tau.max())) * (np.abs(th) < np.abs(fd.max()) / 2)
        m = int(sel.sum())
        if m < min_crop:
            continue
        try:
            er = th[sel]
            er = (er[:-1] + er[1:]) / 2
            with warnings.catch_warnings():      # a crop of 2: the mean of no steps is NaN
                warnings.simplefilter("ignore", RuntimeWarning)
                step = np.diff(er).mean()
            edges_red = np.concatenate((np.array([er[0] - step]), er, np.array([er[-1] + step])))
            out[k, :m] = theta_centres(edges_red)
        except Exception as e:  # noqa: BLE001  (raised again by chisq_calc)
            errs[k] = e
    return out, errs


def _chisq_run(dspec, CS, tau, fd, etas, edges, mask, tol, max_iter):
    """sb_chisq_sweep: unnormalised sums, eigenvalues, status, sizes, iterations
    and the host-side errors of _rev_centres."""
    import torch
    d = np.asarray(dspec)
    if d.ndim != 2:
        raise ValueError("dspec must be 2-D, got shape %r" % (d.shape,))
    _hist_edges(tau, fd)
    if mask is not None:
        mask = np.asarray(mask, dtype=bool)
        if mask.shape != d.shape:
            # what numpy raises for (model - dspec)[mask] (ththmod.py:367)
            raise IndexError("mask shape %r does not match dspec shape %r"
                             % (mask.shape, d.shape))
    cs = _as_device_cs(CS)
    geom = _Geom(cs, tau, fd, edges, True)
    tauv, fdv = U.value(tau, "us"), U.value(fd, "mHz")
    ev = np.ascontiguousarray(np.atleast_1d(U.value(etas, "s3")), dtype=np.float64)
    neta = ev.shape[0]
    th_red, errs = _rev_centres(geom.th, tauv, fdv, ev)
    d_etas, d_th = D.upload(ev), D.upload(th_red)
    d_dspec = D.upload_f32(d)
    d_mask = D.upload(np.ascontiguousarray(mask, dtype=np.uint8)) if mask is not None else None
    ssq = D.empty((neta,), torch.float64)
    w = D.empty((neta,), torch.float64)
    aux = [D.empty((neta,), torch.int32) for _ in range(3)]
    _lib.check(_lib.lib.sb_chisq_sweep(
        geom.ref, d_etas.data_ptr(), neta, d_th.data_ptr(), float(tauv[1] - tauv[0]),
        float(fdv[1] - fdv[0]), d_dspec.data_ptr(), d.shape[0], d.shape[1], D.ptr(d_mask),
        float(tol), int(max_iter), ssq.data_ptr(), w.data_ptr(), aux[0].data_ptr(),
        aux[1].data_ptr(), aux[2].data_ptr(), D.stream_ptr()))
    info = dict(w=w.cpu().numpy(), status=aux[0].cpu().numpy(), nred=aux[1].cpu().numpy(),
                iters=aux[2].cpu().numpy())
    return ssq.cpu().numpy(), info, errs


def chisq_sweep(dspec, CS, tau, fd, etas, edges, N, mask=None, return_info=False,
                tol=0.0, max_iter=0):
    """chisq_calc (ththmod.py:330-368) for every curvature in ``etas``: the loop
    of the chi-square search in the reference's THTHSample notebook, batched on
    the device (one launch sequence, one number per curvature back).

    Returns float64 ``sum over mask of (model - dspec)**2 / N`` per curvature
    (an array ``N`` broadcasts as in numpy: shape (len(etas),) + N.shape), NaN
    where chisq_calc would raise.  ``return_info`` adds a dict with the top
    eigenvalues ``w``, the SB_ETA_* ``status`` bits, the cropped sizes ``nred``
    and the Lanczos ``iters``.  ``CS`` may be a numpy array or a DeviceCS.  A descending
    tau or fd axis raises ValueError (every chisq_calc on it would raise) before any
    device work."""
    ssq, info, errs = _chisq_run(dspec, CS, tau, fd, etas, edges, mask, tol, max_iter)
    ssq[(info["status"] & 8) != 0] = np.nan        # ArpackNoConvergence in the reference
    ssq[[e is not None for e in errs]] = np.nan
    Nv = np.asarray(N, dtype=np.float64)
    chisq = ssq.reshape(ssq.shape + (1,) * Nv.ndim) / Nv
    if return_info:
        return chisq, info
    return chisq


def chisq_calc(dspec, CS, tau, fd, eta, edges, N, mask=None):
    """Chi-square of the rank-1 theta-theta model of the dynamic spectrum
    (ththmod.py:330-368): np.sum((model - dspec)[mask] ** 2) / N with model =
    modeler(...)[3][:dspec.shape[0], :dspec.shape[1]].  ``mask`` defaults to
    np.isfinite(dspec).  Raises where the reference raises."""
    _check_rev_axes(tau, fd, edges, float(U.value(eta, "s3")))
    ssq, info, errs = _chisq_run(dspec, CS, tau, fd, np.array([float(U.value(eta, "s3"))]),
                                 edges, mask, 0.0, 0)
    st = int(info["status"][0])
    if st & 1:
        raise IndexError("theta-theta point maps outside the conjugate "
                         "spectrum (fd_inv < -nfd)")
    if st & 4:
        raise TypeError("theta-theta matrix too small for eigsh (n < 3)")
    if st & 2:
        # ARPACK error -9 in the reference: every start vector is mapped to zero
        raise RuntimeError("starting vector is zero: the theta-theta matrix is zero")
    if st & 8:
        raise np.linalg.LinAlgError("top eigenpair did not converge")
    if errs[0] is not None:
        raise errs[0]
    return ssq[0] / np.asarray(N, dtype=np.float64)


def _vlbi_auto_indices(n_dish):
    """Positions of the station spectra in [I1, V12, .., V1N, I2, V23, .., IN]
    (ththmod.py:1289-1291)."""
    return {n_dish * (n_dish + 1) // 2 - (n_dish - d) * (n_dish - d + 1) // 2
            for d in range(n_dish)}


def _vlbi_run(dspec2_list, edges, time, freq, eta, npad, n_dish, tauMask, tol=0.0, max_iter=0):
    """Conjugate spectra (sb_cs_f32 / sb_cs_c2c_f32, full plane) and sb_vlbi_retrieval for
    one chunk.  Returns (model_E complex128 [n_dish][nf][nt], w, V complex128
    [n_dish nred], info dict with iters / status / nred, host-side error or None)."""
    import torch
    n_dish = int(n_dish)
    if n_dish < 1:
        raise ValueError("n_dish must be at least 1, got %d" % n_dish)
    dl = [np.asarray(d) for d in dspec2_list]
    if len(dl) != n_dish * (n_dish + 1) // 2:
        raise ValueError("dspec2_list has %d entries; %d stations need n_dish (n_dish + 1) / 2 = %d"
                         % (len(dl), n_dish, n_dish * (n_dish + 1) // 2))
    shape = dl[0].shape
    if len(shape) != 2:
        raise ValueError("dynamic spectra must be 2-D, got shape %r" % (shape,))
    for k, d in enumerate(dl):
        if d.shape != shape:
            raise ValueError("dspec2_list[%d] has shape %r, dspec2_list[0] %r" % (k, d.shape, shape))
        if not np.all(np.isfinite(d)):
            raise ValueError("dspec2_list[%d] is not finite" % k)
    npad = int(npad)
    time_v, freq_v = U.value(time, "s"), U.value(freq, "MHz")
    eta_v = float(U.value(eta, "s3"))
    fd = U.value(fft_axis(time_v, "mHz", npad), "mHz")
    tau = U.value(fft_axis(freq_v, "us", npad), "us")
    tm = float(U.value(tauMask, "us"))
    _check_rev_axes(tau, fd, edges, eta_v)
    autos = _vlbi_auto_indices(n_dish)
    cs_list = [conjugate_spectrum(d, npad, None if k in autos else 0.0, tau, tm, half=False)
               for k, d in enumerate(dl)]
    geom = _Geom(cs_list[0], tau, fd, edges, True)
    # min_crop=0: a crop of fewer than 3 centres raises what the reference raises there
    th_red, errs = _rev_centres(geom.th, tau, fd, np.array([eta_v]), min_crop=0)
    n_th = geom.th.shape[0]
    nf, nt = shape
    ptrs = (ctypes.c_void_p * len(cs_list))(*[c.t.data_ptr() for c in cs_list])
    d_th = D.upload(np.ascontiguousarray(th_red[0]))
    model = D.empty((n_dish, nf, nt, 2), torch.float32)
    w = D.empty((1,), torch.float64)
    V = D.zeros((n_dish * n_th, 2), torch.float32)
    info = D.zeros((3,), torch.int32)
    _lib.check(_lib.lib.sb_vlbi_retrieval(
        geom.ref, ptrs, n_dish, eta_v, d_th.data_ptr(), float(tau[1] - tau[0]),
        float(fd[1] - fd[0]), nf, nt, float(tol), int(max_iter), model.data_ptr(),
        w.data_ptr(), V.data_ptr(), info.data_ptr(), D.stream_ptr()))
    iv = info.cpu().numpy()
    inf = dict(iters=int(iv[0]), status=int(iv[1]), nred=int(iv[2]))
    return _c64(model), float(w.cpu()[0]), _c64(V)[:n_dish * inf["nred"]], inf, errs[0]


def VLBI_chunk_retrieval(params):
    """Phase retrieval on one chunk from several stations' dynamic spectra and their
    visibilities (ththmod.py:1223-1387; Baker et al. 2023).  ``params`` is the
    reference's tuple (dspec2_list, edges, time, freq, eta, idx_t, idx_f, npad,
    n_dish, tauMask, verbose) with dspec2_list ordered [I1, V12, .., V1N, I2, V23,
    .., IN]; returns (model_E, idx_f, idx_t), model_E a list of n_dish complex
    wavefields.  Raises where the reference raises: IndexError when the theta grid
    reaches past the fd axis, scipy's ArpackError when every spectrum is zero,
    IndexError (0 or 1) or ValueError (2) when the crop keeps fewer than 3 theta
    centres, rev_map's ValueError on a descending tau or fd axis.  ValueError for a list
    length other than n_dish (n_dish + 1) / 2, mismatched shapes or non-finite input."""
    (dspec2_list, edges, time, freq, eta, idx_t, idx_f, npad, n_dish, tauMask,
     verbose) = params
    if verbose:
        print("Starting Chunk %s-%s" % (idx_f, idx_t), flush=True)
    model, _, _, info, err = _vlbi_run(dspec2_list, edges, time, freq, eta, npad, n_dish,
                                       tauMask)
    st = info["status"]
    if st & 1:
        raise IndexError("theta-theta point maps outside the conjugate "
                         "spectrum (fd_inv < -nfd)")
    if err is not None:          # fewer than 3 centres in the crop (SB_ETA_TOO_SMALL included)
        raise err
    if st & 2:
        from scipy.sparse.linalg import ArpackError
        # what eigsh raises in the reference: every start vector maps to zero
        raise ArpackError(-9, {-9: "Starting vector is zero (the composite matrix is zero)."})
    if st & 8:
        raise np.linalg.LinAlgError("top eigenpair did not converge")
    if verbose:
        print("Chunk %s-%s success" % (idx_f, idx_t), flush=True)
    return ([model[d] for d in range(model.shape[0])], idx_f, idx_t)


# messages printed for the chunks whose asymmetry the reference's try/except turns into NaN
_ASYM_FAILURES = (
    (1, "theta-theta point maps outside the conjugate spectrum (fd_inv < -nfd)"),
    (4, "theta-theta matrix too small for eigsh (n < 3)"),
    (2, "starting vector is zero: the theta-theta matrix is zero"),
    (8, "top eigenpair did not converge"),
)


def _asym_check_sizes(NF, NT, n_th):
    """The limits of sb_asymmetry_batch for spectra of NF x NT and n_th theta centres."""
    if n_th > 4096:
        raise _lib.SbError("calc_asymmetry: theta-theta grid of %d centres exceeds the "
                           "supported 4096" % n_th)
    pow2 = not (NF & (NF - 1)) and not (NT & (NT - 1))
    if pow2 and NF >= 4 and NT >= 16:
        ok = NF <= 65536 and NT <= 32768
    else:
        ok = 3 <= NF <= 32768 and 3 <= NT <= 8192
    if not ok:
        raise _lib.SbError("calc_asymmetry: padded chunk %d x %d outside 4..65536 x 16..32768 "
                           "(powers of two) / 3..32768 x 3..8192 (other sizes)" % (NF, NT))


def asymmetry_batch(params_list, return_info=False, tol=0.0, max_iter=0):
    """calc_asymmetry (ththmod.py:2385-2463) over a sequence of chunks: the loop of
    Dynspec.calc_asymmetry (dynspec.py:1892-1918).  Each entry is the reference's tuple
    (dspec2, edges, time, freq, eta, idx_t, idx_f, npad, verbose).

    Chunks are grouped by padded shape and theta grid size; per group the spectra are made
    (sb_cs_f32, padded with each chunk's mean) and one sb_asymmetry_batch call crops,
    gathers, solves and reduces every chunk.  Every group's sizes are checked before any
    device work.  Returns [(asymm, idx_f, idx_t), ...] in input order; a chunk the
    reference cannot recover prints the reason and gives NaN.  Library errors
    (_lib.SbError) are raised.  ``return_info`` adds a dict of per-chunk arrays ``w``,
    ``status``, ``nred``, ``iters`` and the list ``V`` of eigenvectors (length nred,
    arbitrary global phase)."""
    import torch
    params_list = list(params_list)
    prep, groups, failed = [], {}, {}
    for k, p in enumerate(params_list):
        dspec2, edges, time, freq, eta, idx_t, idx_f, npad, verbose = p
        d = np.asarray(dspec2, dtype=np.float64)
        if d.ndim != 2:
            raise ValueError("dynamic spectrum must be 2-D, got shape %r" % (d.shape,))
        npad = int(npad)
        ev = U.value(edges, "mHz")
        NF, NT = (npad + 1) * d.shape[0], (npad + 1) * d.shape[1]
        prep.append((d, ev, U.value(time, "s"), U.value(freq, "MHz"),
                     float(U.value(eta, "s3")), npad))
        try:
            theta_centres(ev)
        except ValueError as e:     # thth_map raises in the reference's try: NaN
            failed[k] = str(e)
            continue
        groups.setdefault((NF, NT, len(ev) - 1), []).append(k)
    for NF, NT, n_th in groups:
        _asym_check_sizes(NF, NT, n_th)
    n = len(params_list)
    asym = np.full(n, np.nan)
    info = dict(w=np.full(n, np.nan), status=np.zeros(n, np.int32), nred=np.zeros(n, np.int32),
                iters=np.zeros(n, np.int32), V=[None] * n)
    for p in params_list:
        if p[8]:
            print("Starting Chunk %s-%s" % (p[6], p[5]), flush=True)
    for (NF, NT, n_th), ks in groups.items():
        keep = []
        for k in ks:
            d, ev, time_v, freq_v, _, npad = prep[k]
            fd = U.value(fft_axis(time_v, "mHz", npad), "mHz")
            tau = U.value(fft_axis(freq_v, "us", npad), "us")
            cs = conjugate_spectrum(d, npad, None)
            keep.append(_Geom(cs, tau, fd, ev, True))
        nb = len(ks)
        geoms = (_lib.ThthGeom * nb)(*[g.g for g in keep])
        d_etas = D.upload(np.array([prep[k][4] for k in ks]))
        ld = (n_th + 31) // 32 * 32
        out = D.empty((nb,), torch.float64)
        w = D.empty((nb,), torch.float64)
        aux = [D.empty((nb,), torch.int32) for _ in range(3)]
        V = D.empty((nb, ld, 2), torch.float32) if return_info else None
        _lib.check(_lib.lib.sb_asymmetry_batch(
            geoms, nb, d_etas.data_ptr(), float(tol), int(max_iter), out.data_ptr(),
            w.data_ptr(), aux[0].data_ptr(), aux[1].data_ptr(), aux[2].data_ptr(), D.ptr(V),
            D.stream_ptr()))
        asym[ks] = out.cpu().numpy()
        for key, t in zip(("w", "status", "nred", "iters"), [w] + aux):
            info[key][ks] = t.cpu().numpy()
        if return_info:
            Vh = _c64(V)
            for j, k in enumerate(ks):
                info["V"][k] = Vh[j, :info["nred"][k]]
        del keep
    res = []
    for k, p in enumerate(params_list):
        idx_t, idx_f, verbose = p[5], p[6], p[8]
        st = int(info["status"][k])
        msg = [m for bit, m in _ASYM_FAILURES if st & bit]
        if k in failed:
            msg = [failed[k]]
        elif not msg:
            # the reference's modeler ends in rev_map, which raises on a descending axis
            _, _, time_v, freq_v, _, npad = prep[k]
            try:
                _hist_edges(fft_axis(freq_v, "us", npad), fft_axis(time_v, "mHz", npad))
            except ValueError as e:
                msg = [str(e)]
                asym[k] = np.nan
        if msg:
            print(msg[0], flush=True)
        elif verbose:       # 0 / 0 (no weight off the centre element) is NaN without an error
            print("Chunk %s-%s success" % (idx_f, idx_t), flush=True)
        res.append((float(asym[k]), idx_f, idx_t))
    if return_info:
        return res, info
    return res


def calc_asymmetry(params):
    """Arc asymmetry of one chunk from its theta-theta eigenvector (ththmod.py:2385-2463).
    ``params`` is the reference's tuple (dspec2, edges, time, freq, eta, idx_t, idx_f,
    npad, verbose); returns (asymm, idx_f, idx_t).  The chunk is padded with its mean;
    the eigenvector V of the cropped matrix (m centres) gives
    (|V[:(m-1)//2]|^2 - |V[(m+1)//2:]|^2) / (|V[:(m-1)//2]|^2 + |V[(m+1)//2:]|^2).
    A chunk the reference cannot recover prints the reason and gives NaN; library errors
    (_lib.SbError: unsupported size, CUDA) are raised.  Same kernels as asymmetry_batch."""
    return asymmetry_batch([params])[0]


def mask_func(w):
    """sin^2 ramp used to weight overlapping chunks (ththmod.py:1478-1489)."""
    x = np.linspace(0, w - 1, w)
    return np.sin((np.pi / 2) * x / w) ** 2


def mosaic(chunks):
    """Stitch the half-overlapping wavefield chunks [ncf][nct][cwf][cwt] into one
    wavefield, rotating each new chunk to the phase of what is already there
    (ththmod.py:1492-1554).  Sequential by construction: host numpy."""
    ncf, nct, cwf, cwt = chunks.shape
    hf, ht = cwf // 2, cwt // 2
    E = np.zeros(((ncf - 1) * hf + cwf, (nct - 1) * ht + cwt), dtype=complex)
    up_f, up_t = mask_func(hf), mask_func(ht)
    for cf in range(ncf):
        for ct in range(nct):
            new = chunks[cf, ct, :, :]
            fs = slice(cf * cwf // 2, cf * cwf // 2 + cwf)
            ts = slice(ct * cwt // 2, ct * cwt // 2 + cwt)
            mask = np.ones(new.shape)
            if cf > 0:
                mask[:hf, :] *= up_f[:, np.newaxis]
            if cf < ncf - 1:
                mask[hf:, :] *= 1 - up_f[:, np.newaxis]
            if ct > 0:
                mask[:, :ht] *= up_t
            if ct < nct - 1:
                mask[:, ht:] *= 1 - up_t
            rot = np.angle((E[fs, ts] * np.conjugate(new) * mask).mean())
            E[fs, ts] += new * mask * np.exp(1j * rot)
    return E


def min_edges(fd_lim, fd, tau, eta, factor=2):
    """Minimum edges array that oversamples the CS (ththmod.py:1671-1705)."""
    fd_lim_v = float(U.value(fd_lim, "mHz"))
    fdv, tauv = U.value(fd, "mHz"), U.value(tau, "us")
    eta_v = float(U.value(eta, "s3"))
    dtau_lim = (tauv[1] - tauv[0]) / factor
    dtau_lim /= 2 * eta_v * fd_lim_v
    dfd_lim = (fdv[1] - fdv[0]) / factor
    npoints = (2 * fd_lim_v) // (min(dfd_lim, dtau_lim))
    npoints += np.mod(npoints, 2)
    return U.wrap(np.linspace(-fd_lim_v, fd_lim_v, int(npoints)), "mHz",
                  like=fd_lim)



class MosaicModel:
    """The chunks [ncf][nct][cwf][cwt] uploaded once (complex64) for the mosaic fit of
    ththmod.py:1708-2310, on the device (sb_mosaic_*).

    ``rot_init()``, ``rot_mos(x)``, ``rot_fit(x)``, ``rot_der(x)`` take the phase of every
    chunk after the first; ``full_mos(p)``, ``fit(p)``, ``grad(p)``, ``hess(p, sparse=False)``
    take p = (those phases, then one amplitude per chunk).  Entries past them are ignored
    (their gradient and Hessian rows are zero); a shorter vector raises IndexError.  The
    last wavefield and the last fit / gradient are cached per parameter vector, so ``fit``,
    ``grad`` and ``hess`` at one p (as scipy.optimize.minimize calls them) build the
    mosaic once.  ``dspec`` and ``N`` (noise standard deviation) are cropped to the mosaic
    shape and must be at least that large.  fit and grad skip NaN terms (nansum);
    rot_fit, rot_der and hess let NaN propagate.  Pixels are float32 arithmetic with
    float64 sums; ``hess(sparse=True)`` gives a scipy.sparse.csr_matrix."""

    def __init__(self, chunks, dspec=None, N=None):
        ch = np.asarray(chunks)
        if ch.ndim != 4:
            raise ValueError("chunks must be 4-D [ncf][nct][cwf][cwt], got shape %r" % (ch.shape,))
        ncf, nct, cwf, cwt = (int(n) for n in ch.shape)
        _check_widths(ch.shape)
        hf, ht = (cwf // 2 if ncf > 1 else cwf), (cwt // 2 if nct > 1 else cwt)
        if min(ncf, nct, cwf, cwt) < 1 or hf > 2048 or ht > 2048 or ncf * nct >= 2 ** 28:
            raise _lib.SbError("mosaic: %d x %d chunks of %d x %d outside the supported "
                               "geometry (half-chunk extent <= 2048, fewer than 2^28 chunks)"
                               % (ncf, nct, cwf, cwt))
        self.dims = (ncf, nct, cwf, cwt)
        self.P = ncf * nct
        self.shape = ((ncf - 1) * (cwf // 2) + cwf, (nct - 1) * (cwt // 2) + cwt)
        if dspec is not None or N is not None:
            dspec, N = self._crop(dspec, "dspec"), self._crop(N, "N")
        self._ch = D.upload(ch.astype(np.complex64, copy=False))
        self._D = None if dspec is None else D.upload(dspec)
        self._N = None if N is None else D.upload(N)
        import torch
        self._W = D.empty(self.shape + (2,), torch.float32)
        self._wkey = None
        self._fkey = self._rkey = None

    def _crop(self, a, name):
        if a is None:
            raise ValueError("MosaicModel: dspec and N are needed together")
        a = np.asarray(a)
        nF, nT = self.shape
        if a.ndim != 2 or a.shape[0] < nF or a.shape[1] < nT:
            raise ValueError("%s of shape %r is smaller than the mosaic %r" % (name, a.shape, self.shape))
        return np.ascontiguousarray(a[:nF, :nT], dtype=np.float32)

    def _params(self, p, with_amp):
        p = np.asarray(p, dtype=np.float64)
        need = 2 * self.P - 1 if with_amp else self.P - 1
        if p.ndim != 1 or p.shape[0] < need:
            raise IndexError("parameter vector of length %d; %d chunks need %d"
                             % (p.shape[0] if p.ndim else 0, self.P, need))
        phi = np.concatenate([[0.0], p[:self.P - 1]])
        amp = p[self.P - 1:2 * self.P - 1].copy() if with_amp else None
        return p, phi, amp

    def _build(self, phi, amp):
        key = (phi.tobytes(), None if amp is None else amp.tobytes())
        if key != self._wkey:
            self._dphi = D.upload(phi)
            self._damp = None if amp is None else D.upload(amp)
            ncf, nct, cwf, cwt = self.dims
            _lib.check(_lib.lib.sb_mosaic_build(self._ch.data_ptr(), ncf, nct, cwf, cwt,
                                                self._dphi.data_ptr(), D.ptr(self._damp),
                                                self._W.data_ptr(), D.stream_ptr()))
            self._wkey = key
            self._fkey = self._rkey = None

    def _wave(self):
        a = self._W.cpu().numpy()
        return (a[..., 0] + 1j * a[..., 1]).astype(np.complex128)

    def rot_init(self):
        """Phase of every chunk after the first that stacks it coherently onto the chunks
        before it (ththmod.py:1791-1856).  The device sums each chunk's overlap with its
        (at most four) earlier neighbours; the recurrence rot_k = angle(sum_j e^{i rot_j}
        C_kj) runs on the host in float64.  A chunk whose sum is exactly zero (an all-zero
        chunk) gets 0, where the reference returns the angle of a signed zero (0 or +-pi);
        such a chunk adds nothing to the mosaic either way."""
        import cmath
        import torch
        ncf, nct, cwf, cwt = self.dims
        C = D.empty((self.P, 4, 2), torch.float64)
        _lib.check(_lib.lib.sb_mosaic_overlap(self._ch.data_ptr(), ncf, nct, cwf, cwt,
                                              C.data_ptr(), D.stream_ptr()))
        c = C.cpu().numpy()
        c = (c[..., 0] + 1j * c[..., 1]).tolist()
        rot = [0.0] * self.P
        for k in range(1, self.P):
            cf, ct = divmod(k, nct)
            s = 0j
            for e, (jf, jt) in enumerate(((cf - 1, ct - 1), (cf - 1, ct), (cf - 1, ct + 1),
                                          (cf, ct - 1))):
                if jf >= 0 and 0 <= jt < nct:
                    s += cmath.exp(1j * rot[jf * nct + jt]) * c[k][e]
            rot[k] = cmath.phase(s) if s != 0 else 0.0
        return np.array(rot[1:])

    def rot_mos(self, x):
        """ththmod.rotMos (:1708-1770): complex128 mosaic with phases x."""
        _, phi, _ = self._params(x, False)
        self._build(phi, None)
        return self._wave()

    def _rot(self, x):
        import torch
        x, phi, _ = self._params(x, False)
        self._build(phi, None)
        if self._rkey is None:
            ncf, nct, cwf, cwt = self.dims
            out = D.empty((self.P + 1,), torch.float64)
            _lib.check(_lib.lib.sb_mosaic_rot(self._ch.data_ptr(), ncf, nct, cwf, cwt,
                                              self._dphi.data_ptr(), self._W.data_ptr(),
                                              out.data_ptr(), out.data_ptr() + 8,
                                              D.stream_ptr()))
            self._rkey = out.cpu().numpy()
        return x, self._rkey

    def rot_fit(self, x):
        """ththmod.rotFit (:1773-1788): -sum |rotMos(x)|^2 (NaN propagates)."""
        return float(-self._rot(x)[1][0])

    def rot_der(self, x):
        """ththmod.rotDer (:1859-1919): d rotFit / d x, shaped like x."""
        x, r = self._rot(x)
        out = np.zeros(x.shape)
        out[:self.P - 1] = r[2:]
        return out

    def full_mos(self, p):
        """ththmod.fullMos (:1922-1987): complex128 mosaic with phases and amplitudes p."""
        _, phi, amp = self._params(p, True)
        self._build(phi, amp)
        return self._wave()

    def _need_data(self):
        if self._D is None:
            raise ValueError("MosaicModel: fit / grad / hess need dspec and N")

    def _fit(self, p):
        import torch
        p, phi, amp = self._params(p, True)
        self._need_data()
        self._build(phi, amp)
        if self._fkey is None:
            ncf, nct, cwf, cwt = self.dims
            out = D.empty((2 * self.P + 1,), torch.float64)
            _lib.check(_lib.lib.sb_mosaic_fit(self._ch.data_ptr(), ncf, nct, cwf, cwt,
                                              self._dphi.data_ptr(), self._damp.data_ptr(),
                                              self._W.data_ptr(), self._D.data_ptr(),
                                              self._N.data_ptr(), out.data_ptr(),
                                              out.data_ptr() + 8, D.stream_ptr()))
            self._fkey = out.cpu().numpy()
        return p, self._fkey

    def fit(self, p):
        """ththmod.fullMosFit (:1990-2016): nansum(((|W|^2 - dspec) / N)^2)."""
        return float(self._fit(p)[1][0])

    def grad(self, p):
        """ththmod.fullMosGrad (:2019-2102): gradient of fit, length len(p)."""
        p, r = self._fit(p)
        g = r[1:].reshape(self.P, 2)
        out = np.zeros(p.shape[0])
        out[self.P - 1:2 * self.P - 1] = g[:, 0]
        out[:self.P - 1] = g[1:, 1]
        return out

    def hess(self, p, sparse=False):
        """ththmod.fullMosHess (:2105-2310): Hessian of fit, (len(p), len(p)); from the
        sums over each pair of neighbouring chunks.  NaN propagates."""
        import torch
        p, phi, amp = self._params(p, True)
        self._need_data()
        self._build(phi, amp)
        ncf, nct, cwf, cwt = self.dims
        n = 40 * self.P
        rows, cols = D.empty((n,), torch.int64), D.empty((n,), torch.int64)
        vals = D.empty((n,), torch.float64)
        _lib.check(_lib.lib.sb_mosaic_hess(self._ch.data_ptr(), ncf, nct, cwf, cwt,
                                           self._dphi.data_ptr(), self._damp.data_ptr(),
                                           self._W.data_ptr(), self._D.data_ptr(),
                                           self._N.data_ptr(), rows.data_ptr(), cols.data_ptr(),
                                           vals.data_ptr(), D.stream_ptr()))
        r, c, v = rows.cpu().numpy(), cols.cpu().numpy(), vals.cpu().numpy()
        keep = r >= 0
        r, c, v = r[keep], c[keep], v[keep]
        m = p.shape[0]
        if sparse:
            from scipy.sparse import csr_matrix
            return csr_matrix((v, (r, c)), shape=(m, m))
        H = np.zeros((m, m))
        H[r, c] = v
        return H


def _check_widths(shape):
    """The reference's ramps broadcast only onto even halves: an axis with more than one
    chunk needs an even width (ValueError otherwise, as in the reference)."""
    ncf, nct, cwf, cwt = shape
    if (ncf > 1 and cwf % 2) or (nct > 1 and cwt % 2):
        raise ValueError("chunk width %d x %d: an axis with more than one chunk needs an "
                         "even width" % (cwf, cwt))


def _grad_data(chunks, dspec, N):
    """fullMosGrad / fullMosHess index dspec with the mosaic's shape exactly and N by
    slices of it: dspec must be the mosaic's shape, N at least that."""
    ch = np.asarray(chunks)
    if ch.ndim == 4:
        _check_widths(ch.shape)
        ncf, nct, cwf, cwt = ch.shape
        shape = ((ncf - 1) * (cwf // 2) + cwf, (nct - 1) * (cwt // 2) + cwt)
        if np.shape(dspec) != shape:
            raise ValueError("dspec of shape %r does not match the mosaic %r"
                             % (np.shape(dspec), shape))
        if np.ndim(N) != 2 or np.shape(N)[0] < shape[0] or np.shape(N)[1] < shape[1]:
            raise ValueError("N of shape %r is smaller than the mosaic %r" % (np.shape(N), shape))


def _check_p(chunks, p, with_amp):
    ch = np.asarray(chunks)
    P = ch.shape[0] * ch.shape[1] if ch.ndim == 4 else 0
    need = 2 * P - 1 if with_amp else P - 1
    if np.ndim(p) != 1 or np.shape(p)[0] < need:
        raise IndexError("parameter vector of length %d; %d chunks need %d"
                         % (np.size(p), P, need))


def rotInit(chunks):
    """ththmod.rotInit (ththmod.py:1791-1856) on the device; see MosaicModel.rot_init."""
    return MosaicModel(chunks).rot_init()


def rotMos(chunks, x):
    """ththmod.rotMos (ththmod.py:1708-1770) on the device."""
    _check_p(chunks, x, False)
    return MosaicModel(chunks).rot_mos(x)


def rotFit(x, chunks):
    """ththmod.rotFit (ththmod.py:1773-1788) on the device."""
    _check_p(chunks, x, False)
    return MosaicModel(chunks).rot_fit(x)


def rotDer(x, chunks):
    """ththmod.rotDer (ththmod.py:1859-1919) on the device."""
    _check_p(chunks, x, False)
    return MosaicModel(chunks).rot_der(x)


def fullMos(chunks, p):
    """ththmod.fullMos (ththmod.py:1922-1987) on the device."""
    _check_p(chunks, p, True)
    return MosaicModel(chunks).full_mos(p)


def fullMosFit(p, chunks, dspec, N):
    """ththmod.fullMosFit (ththmod.py:1990-2016) on the device; dspec and N are cropped
    to the mosaic."""
    _check_p(chunks, p, True)
    return MosaicModel(chunks, dspec, N).fit(p)


def fullMosGrad(p, chunks, dspec, N):
    """ththmod.fullMosGrad (ththmod.py:2019-2102) on the device; dspec must have the
    mosaic's shape and N at least that."""
    _check_p(chunks, p, True)
    _grad_data(chunks, dspec, N)
    return MosaicModel(chunks, dspec, N).grad(p)


def fullMosHess(p, chunks, dspec, N):
    """ththmod.fullMosHess (ththmod.py:2105-2310) on the device, dense (len(p), len(p));
    dspec must have the mosaic's shape and N at least that."""
    _check_p(chunks, p, True)
    _grad_data(chunks, dspec, N)
    return MosaicModel(chunks, dspec, N).hess(p)


# ---- rank-k SVD model (Dynspec.correct_dyn) ------------------------------------------

SVD_MAX_MODES = 32
SVD_MAX_NF, SVD_MAX_NT = 32768, 16384


def _svd_check(arr, nmodes):
    """Argument checks of svd_model / Dynspec.correct_dyn, raised before any device call:
    a real 2-D array of at most SVD_MAX_NF x SVD_MAX_NT and 1 <= nmodes <= SVD_MAX_MODES."""
    a = np.asarray(arr)
    if np.iscomplexobj(a):
        raise TypeError("svd_model takes a real array, not %s" % a.dtype)
    if a.ndim != 2:
        raise ValueError("svd_model takes a 2-D array, got shape %s" % (a.shape,))
    _svd_check_modes(nmodes)
    nf, nt = a.shape
    if not (1 <= nf <= SVD_MAX_NF and 1 <= nt <= SVD_MAX_NT):
        raise ValueError("svd_model: shape %d x %d is outside 1..%d x 1..%d"
                         % (nf, nt, SVD_MAX_NF, SVD_MAX_NT))
    return a


def _svd_check_modes(nmodes):
    if not isinstance(nmodes, (int, np.integer)) or isinstance(nmodes, bool):
        raise TypeError("nmodes must be an integer, got %r" % (nmodes,))
    if not 1 <= nmodes <= SVD_MAX_MODES:
        raise ValueError("nmodes must be in 1..%d, got %d" % (SVD_MAX_MODES, nmodes))


def _svd_run(arr, nmodes, want_out=True, want_model=True):
    """Device driver of svd_model and Dynspec.correct_dyn(svd=True) for a checked array:
    the top-nmodes right singular vectors (sb_svd_topk), then one pass that writes
    arr / |model| and the model (sb_svd_apply).  NaN pixels are read as 0.  Returns
    (out, model, info): float32 device tensors (or None) and the solver's info dict.
    Warns (RuntimeWarning) when the solver did not converge or the truncation boundary
    is a tie."""
    import torch
    nf, nt = arr.shape
    d = D.upload_f32(arr)
    V = D.empty((nmodes, nt), torch.float64)
    s = np.zeros(nmodes)
    res = np.zeros(nmodes)
    gap = np.zeros(1)
    st = np.zeros(4, np.int32)
    _lib.check(_lib.lib.sb_svd_topk(d.data_ptr(), nf, nt, nmodes, V.data_ptr(),
                                    s.ctypes.data, res.ctypes.data, gap.ctypes.data,
                                    st.ctypes.data, D.stream_ptr()))
    out = D.empty((nf, nt), torch.float32) if want_out else None
    model = D.empty((nf, nt), torch.float32) if want_model else None
    _lib.check(_lib.lib.sb_svd_apply(d.data_ptr(), nf, nt, nmodes, V.data_ptr(), D.ptr(out),
                                     D.ptr(model), D.stream_ptr()))
    info = dict(s=s, residuals=res, steps=int(st[0]), converged=bool(st[1]), tie=bool(st[2]),
                breakdown=bool(st[3]), gap=float(gap[0]))
    if info["tie"]:
        warnings.warn("svd_model: singular values %d and %d are equal to float32 precision; "
                      "the rank-%d model is not defined by the data" % (nmodes, nmodes + 1, nmodes),
                      RuntimeWarning, stacklevel=3)
    elif not info["converged"]:
        warnings.warn("svd_model: the rank-%d model did not converge (%d Lanczos steps)"
                      % (nmodes, info["steps"]), RuntimeWarning, stacklevel=3)
    return out, model, info


def svd_model(arr, nmodes=1, return_info=False):
    """ththmod.svd_model (ththmod.py:18-35): the rank-nmodes model of a real 2-D array,
    complex128 with zero imaginary part like the reference's.  Only the top nmodes
    singular triplets are computed (csrc/svd.cu); NaN pixels are read as 0.
    nmodes >= min(arr.shape) gives the whole matrix, as in the reference.

    ``return_info`` adds a dict: ``s`` (the nmodes singular values, descending),
    ``residuals`` (||A^T A v_j - s_j^2 v_j||_2 from a final pass), ``steps`` (Lanczos
    steps), ``converged``, ``tie`` (s_nmodes = s_nmodes+1 to float32 precision),
    ``breakdown`` (the Krylov space became invariant: the model is exact) and ``gap``
    (the lower bound on the eigenvalue gap of A^T A at the truncation the stopping rule
    used).  Non-convergence and ties also raise a RuntimeWarning."""
    a = _svd_check(arr, nmodes)
    _, model, info = _svd_run(a, int(nmodes), want_out=False)
    m = D.download(model).astype(np.complex128)
    return (m, info) if return_info else m
