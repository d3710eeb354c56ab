"""Dynspec.calc_scattered_image (reference dynspec.py:3412-3582) restated for a given
spectrum, axes and curvature, with scipy's RectBivariateSpline as the spline.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Needs numpy and scipy only, so the GPU tests
may use it.  ``scattered_image`` runs the reference's steps from the linear spectrum to the
stored image: the crop, the image grid, the fit and ``.ev``, the mirror, and with
``plot_log`` plot_scattered_image's in-place shift and its ValueError.  ``clean`` is left out:
the reference discards its result.
"""
import numpy as np
from scipy.interpolate import RectBivariateSpline


def is_valid(array):
    return np.isfinite(array) * ~np.isnan(array)


def crop(linsspec, fdop, tdel, eta):
    """The reference's crop (:3514-3525): (linsspec, delay axis, Doppler axis)."""
    nf = len(fdop)
    flim = next(i for i, delay in enumerate(eta * fdop**2) if delay < np.max(tdel))
    if flim == 0:
        tlim = next(i for i, delay in enumerate(tdel) if delay > eta * fdop[0] ** 2)
        linsspec = linsspec[:tlim, :]
        tdel = fdop[:tlim]
    else:
        linsspec = linsspec[:, flim-int(0.02*nf):nf-flim+int(0.02*nf)]
        fdop = fdop[flim-int(0.02*nf):nf-flim+int(0.02*nf)]
    return linsspec, tdel, fdop


def scattered_image(sspec, fdop, tdel, eta, sampling=64, plot_log=True, use_angle=False,
                    use_spatial=False, s=None, veff=None, d=None, freq=1400.0):
    """(scattered_image, scattered_image_ax) as the reference stores them; with plot_log,
    plot_scattered_image's axis conversions, shift and errors up to its centres_to_edges."""
    fdop = np.asarray(fdop)
    tdel = np.asarray(tdel)
    with np.errstate(over="ignore"):
        linsspec = 10**(np.asarray(sspec, dtype=np.float64) / 10)
    linsspec, tdel, fdop = crop(linsspec, fdop, tdel, eta)
    nx, ny = 2*sampling+1, sampling+1
    fdop_x = np.linspace(-max(fdop), max(fdop), nx)
    fdop_y = np.linspace(0, max(fdop), ny)
    fdop_x_est, fdop_y_est = np.meshgrid(fdop_x, fdop_y)
    tdel_est = (fdop_x_est**2 + fdop_y_est**2) * eta
    interp = RectBivariateSpline(tdel, fdop, linsspec)
    image = interp.ev(tdel_est, fdop_x_est) * fdop_y_est
    scat_im = np.zeros((nx, nx))
    scat_im[ny-1:nx, :] = image
    scat_im[0:ny-1, :] = image[ny-1:0:-1, :]
    if plot_log:
        c = 299792458.0  # m/s
        xyaxes = fdop_x
        if use_angle or use_spatial:
            thetarad = (xyaxes / (1e9 * freq)) * (c * s / (veff * 1000))
            xyaxes = (thetarad * 180 / np.pi) * 3600
            if not use_angle:
                xyaxes = xyaxes * (1 - s) * d * 1000
        scat_im -= np.min(scat_im)
        scat_im += 1e-10
        with np.errstate(all="ignore"):
            lg = 10 * np.log10(scat_im)
        if not np.any(is_valid(lg) * np.array(np.abs(lg) > 0)):
            raise ValueError("zero-size array to reduction operation maximum which has no "
                             "identity")
        np.abs(xyaxes[1] - xyaxes[0])       # centres_to_edges: IndexError on one pixel
    return scat_im, fdop_x
