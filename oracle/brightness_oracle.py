"""Float64 oracle for scint_sim.Brightness (reference scint_sim.py:768-958).

TEST INFRASTRUCTURE (see oracle/__init__.py).  numpy and scipy only, so the GPU tests may
use it.

* ``efield`` and ``acf`` are the reference's numpy expressions (numpy's FFT).
* ``calc_ss`` restates calc_SS without its loop: thetax, thetay and the Jacobian by the same
  IEEE operations in the same order (the squares of ``thetax + thetagx`` by the scalar
  power the reference's loop uses, which is C pow and not always x*x), so they are
  bit-equal to the reference's.  Its two ``griddata`` calls become ``cell_interp``.
* ``cell_interp`` is the cell rule: griddata(method='linear') on the lattice
  meshgrid(x, x) interpolates barycentrically on qhull's triangulation, which splits each
  lattice cell along one diagonal (``diagonals``).  Find the query's cell from x, the
  diagonal from the cell's bit, and weight the three corners of the half it lies in.
  Queries more than 100 DBL_EPSILON outside the lattice's bounding box are NaN, as qhull's
  find_simplex makes them.
"""
import hashlib
import math

import numpy as np

HULL_EPS = 100 * np.finfo(np.float64).eps


def diagonals(x):
    """(n-1, n-1) bool: True where the Delaunay triangulation griddata builds on
    meshgrid(x, x) splits cell (i, j) along (x[j], x[i])-(x[j+1], x[i+1]).  Raises if a
    simplex is not half a lattice cell."""
    from scipy.spatial import Delaunay
    n = len(x)
    X, Y = np.meshgrid(x, x)
    s = Delaunay(np.column_stack((np.ravel(X), np.ravel(Y)))).simplices
    i, j = s // n, s % n
    i0, j0 = i.min(axis=1), j.min(axis=1)
    assert (i.max(axis=1) - i0 == 1).all() and (j.max(axis=1) - j0 == 1).all()
    assert len(s) == 2 * (n - 1) ** 2
    # a half cell on the main diagonal holds both (j0, i0) and (j0 + 1, i0 + 1)
    has00 = ((i == i0[:, None]) & (j == j0[:, None])).any(axis=1)
    has11 = ((i == i0[:, None] + 1) & (j == j0[:, None] + 1)).any(axis=1)
    main = np.zeros((n - 1, n - 1), dtype=np.int64)
    np.add.at(main, (i0, j0), (has00 & has11).astype(np.int64))
    assert np.isin(main, (0, 2)).all()
    return main == 2


def diag_sha256(main):
    return hashlib.sha256(np.packbits(np.ravel(main)).tobytes()).hexdigest()


def cell_interp(x, main, B, qx, qy):
    """The linear interpolant of B on meshgrid(x, x) at (qx, qy), by the cell rule."""
    x = np.asarray(x, dtype=np.float64)
    qx, qy = np.broadcast_arrays(np.asarray(qx, np.float64), np.asarray(qy, np.float64))
    n = len(x)
    inside = ((qx >= x[0] - HULL_EPS) & (qx <= x[-1] + HULL_EPS) &
              (qy >= x[0] - HULL_EPS) & (qy <= x[-1] + HULL_EPS))
    j = np.clip(np.searchsorted(x, np.where(inside, qx, x[0]), side="right") - 1, 0, n - 2)
    i = np.clip(np.searchsorted(x, np.where(inside, qy, x[0]), side="right") - 1, 0, n - 2)
    u = (qx - x[j]) / (x[j + 1] - x[j])
    v = (qy - x[i]) / (x[i + 1] - x[i])
    f00, f10, f01, f11 = B[i, j], B[i, j + 1], B[i + 1, j], B[i + 1, j + 1]
    m = main[i, j]
    lo = u >= v
    val_main = np.where(lo, (1 - u) * f00 + (u - v) * f10 + v * f11,
                        (1 - v) * f00 + (v - u) * f01 + u * f11)
    low = u + v <= 1
    val_anti = np.where(low, (1 - u - v) * f00 + u * f10 + v * f01,
                        (u + v - 1) * f11 + (1 - v) * f10 + (1 - u) * f01)
    return np.where(inside, np.where(m, val_main, val_anti), np.nan)


def efield(ar=1.0, psi=0, alpha=1.67, dx=0.1, nx=30):
    """x, X, Y, acf_efield and B, as calc_brightness computes them."""
    x = np.arange(-nx, nx, dx)
    X, Y = np.meshgrid(x, x)
    R = (ar**2 - 1) / (ar**2 + 1)
    cosa = np.cos(2 * (90 - psi) * np.pi/180)
    sina = np.sin(2 * (90 - psi) * np.pi/180)
    a = (1 - R * cosa) / np.sqrt(1 - R**2)
    b = (1 + R * cosa) / np.sqrt(1 - R**2)
    c = -2 * R * sina / np.sqrt(1 - R**2)
    Rho = np.exp(-0.5*(a * X**2 + b * Y**2 + c * X * Y) ** (alpha/2))
    B = np.abs(np.fft.ifftshift(np.fft.fft2(np.fft.fftshift(Rho))))
    return x, X, Y, Rho, B


def calc_ss(B, x, thetagx=0, thetagy=0, thetarx=0, thetary=0, df=0.02, dt=0.08, nf=10, nt=80,
            main=None):
    """fd, td, thetax, thetay, jacobian, SS and LSS of calc_SS, vectorised."""
    fd = np.arange(-nf, nf, df)
    td = np.arange(-nt, nt, dt)
    colx = fd - thetagx + thetarx
    colq = np.array([math.pow(float(v + thetagx), 2) for v in colx])
    s = td[:, None] - colq[None, :] + thetarx**2 + thetary**2
    pos = s > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.sqrt(np.where(pos, s, 1.0))
        thetay = np.where(pos, 0.0 + (r - thetagy), 0.0)
        amp = np.where(pos, np.where(r < 0.5*df, 2/df, 1/r), 10**(-6))
    thetax = np.broadcast_to(colx, s.shape).copy()
    if main is None:
        main = diagonals(x)
    g1 = cell_interp(x, main, B, thetax, thetay)
    g2 = cell_interp(x, main, B, thetax, -thetay)
    SS = g1 * amp + g2 * amp
    rev = np.flip(np.flip(SS[1:, 1:], axis=0), axis=1).copy()
    SS[1:, 1:] = SS[1:, 1:] + rev
    with np.errstate(divide="ignore", invalid="ignore"):
        LSS = 10*np.log10(SS)
    return fd, td, thetax, thetay, amp, SS, LSS


def acf(SS):
    a = np.real(np.fft.fftshift(np.fft.fft2(np.fft.fftshift(SS))))
    return a / np.max(a)


def model(ar=1.0, psi=0, alpha=1.67, thetagx=0, thetagy=0, thetarx=0, thetary=0, df=0.02,
          dt=0.08, dx=0.1, nf=10, nt=80, nx=30, main=None):
    """Every attribute of Brightness(**kwargs) as a dict."""
    x, X, Y, Rho, B = efield(ar, psi, alpha, dx, nx)
    fd, td, thetax, thetay, jac, SS, LSS = calc_ss(B, x, thetagx, thetagy, thetarx, thetary,
                                                   df, dt, nf, nt, main)
    return dict(x=x, X=X, Y=Y, acf_efield=Rho, B=B, fd=fd, td=td, thetax=thetax,
                thetay=thetay, jacobian=jac, SS=SS, LSS=LSS, acf=acf(SS))
