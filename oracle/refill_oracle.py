"""Float64 restatement of Dynspec.refill (reference dynspec.py:3273-3323) with its biharmonic
inpainting defined as skimage >= 0.19's inpaint_biharmonic(split_into_regions=False).

TEST INFRASTRUCTURE (see oracle/__init__.py).  scikit-image is not available here, so the
biharmonic system is written from its definition:
  - one unknown per masked pixel, in row-major order;
  - row p is S_p = scipy.ndimage.laplace(laplace(e_p)) on the 5x5 box [p-2, p+2] clipped to
    the image (mode 'reflect'), e_p the unit impulse at p in that box;
  - masked neighbours go into the matrix, known ones to the right-hand side;
  - the scipy.sparse system is solved by spsolve and the solution clipped to [min, max] of
    the known pixels.
The stencils are built per pixel from its own clipped box (cached by the box's extents and
offsets), not from the product's class tables.
"""
import numpy as np
from scipy import sparse
from scipy.ndimage import laplace
from scipy.signal import medfilt
from scipy.sparse.linalg import spsolve


def box(n, i):
    """(lo, extent, offset) of the window [i-2, i+2] clipped to [0, n)."""
    lo = max(i - 2, 0)
    return lo, min(i + 3, n) - lo, i - lo


def stencil(shape, center):
    """laplace(laplace(e)) on an array of `shape` with the unit impulse at `center`."""
    e = np.zeros(shape)
    e[center] = 1.0
    return laplace(laplace(e))


def system(image, mask):
    """(A csr, b, pix): the biharmonic system of the masked pixels, pix their flat indices."""
    image = np.asarray(image, dtype=np.float64)
    mask = np.asarray(mask, dtype=bool)
    nf, nt = image.shape
    pix = np.flatnonzero(mask)
    unk = -np.ones(nf * nt, np.int64)
    unk[pix] = np.arange(pix.size)
    pi, pj = np.divmod(pix, nt)
    li, lj = np.maximum(pi - 2, 0), np.maximum(pj - 2, 0)
    keys = np.stack([np.minimum(pi + 3, nf) - li, pi - li, np.minimum(pj + 3, nt) - lj, pj - lj])
    kinds, which = np.unique(keys, axis=1, return_inverse=True)
    which = which.ravel()
    rows, cols, vals = [], [], []
    b = np.zeros(pix.size)
    flat = image.ravel()
    for g in range(kinds.shape[1]):
        er, orow, ec, ocol = (int(v) for v in kinds[:, g])
        ks = np.flatnonzero(which == g)
        S = stencil((er, ec), (orow, ocol))
        for a, c in zip(*np.nonzero(S)):
            q = (pi[ks] - orow + a) * nt + (pj[ks] - ocol + c)
            u = unk[q]
            m = u >= 0
            rows.append(ks[m])
            cols.append(u[m])
            vals.append(np.full(m.sum(), S[a, c]))
            np.subtract.at(b, ks[~m], S[a, c] * flat[q[~m]])
    A = sparse.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                          shape=(pix.size, pix.size))
    return A, b, pix


def biharmonic(image, mask):
    """The image with its masked pixels inpainted (float64 copy)."""
    out = np.array(image, dtype=np.float64)
    mask = np.asarray(mask, dtype=bool)
    if not mask.any():
        return out
    A, b, pix = system(out, mask)
    x = np.atleast_1d(spsolve(A.tocsc(), b))
    known = out[~mask]
    out.ravel()[pix] = np.clip(x, known.min(), known.max())
    return out


def is_valid(array):
    return np.isfinite(array) * (~np.isnan(array))


def refill(dyn, method='biharmonic', zeros=True, kernel_size=5, linear=True):
    """The array Dynspec.refill leaves in self.dyn (a float64 copy of dyn is worked on)."""
    dyn = np.array(dyn, dtype=np.float64)
    if zeros:
        dyn[dyn == 0] = np.nan
    nan = np.isnan(dyn)
    if method == 'biharmonic':
        dyn[nan] = biharmonic(dyn, nan)[nan]
    elif method == 'median':
        array = dyn.copy()
        array[nan] = np.mean(array[is_valid(array)])
        dyn[nan] = medfilt(array, kernel_size=kernel_size)[nan]
    elif method in ('linear', 'cubic', 'nearest') and linear:
        raise NotImplementedError("griddata interpolation")
    dyn[np.isnan(dyn)] = np.mean(dyn[is_valid(dyn)])
    return dyn


def cubic_case(nf=30, nt=40):
    """A field with zero bilaplacian (a monotone cubic in the row index plus x y^2 terms)
    and holes at least 2 pixels from every edge, inside the known range."""
    i, j = np.mgrid[0:nf, 0:nt].astype(np.float64)
    f = 0.002 * i ** 3 + 0.5 * i + 0.003 * j * (i - 3) ** 2 - 0.01 * i * (j - 5) ** 2
    mask = np.zeros((nf, nt), bool)
    mask[5:12, 6:20] = True
    mask[nf - 8:nf - 3, nt - 10:nt - 4] = True
    mask[15, 2] = mask[2, 20] = mask[nf - 3, 9] = True
    return f, mask
