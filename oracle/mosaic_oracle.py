"""Float64 restatement of the wavefield mosaic fit (ththmod.rotInit ... fullMosHess) in the
pairwise / half-tile form the device code uses.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Written from the math, not from the
reference's loops:

  chunk k = cf*nct + ct, y_k = mask_k chunk_k placed at rows cf*(cwf//2), cols ct*(cwt//2);
  W = sum_k A_k e^{i phi_k} y_k;  wt = |W|^2 - dspec;  t_k = e^{i phi_k} y_k conj(W).

Chunks with cf, ct of the same parities never overlap, so the mosaic is four "layers" (one
per parity pair), each a plain placement of its chunks, with a map from pixel to chunk.
Per-chunk sums are bincounts over one layer; per-pair sums are bincounts over the pixels
two layers (or one layer with itself) share.  Every function returns its value and
sum|terms| of the same shape (the magnitudes the float32 device error bounds scale with:
|W| is replaced by Wabs = sum_k |A_k y_k| and |wt| by Wabs^2 + |dspec|, which bound the
float32-computed values).

The reference's rotDer, fullMosGrad and fullMosHess scale a copy of each chunk in place
(y *= mask, and in fullMosHess y *= e^{i phi}), which keeps complex64 chunks complex64;
``Layers.y`` reproduces those roundings so that the comparison with the reference is exact
to float64 rounding.
"""
import numpy as np


def ramp(h):
    x = np.linspace(0, h - 1, h)
    return np.sin((np.pi / 2) * x / h) ** 2


class Layers:
    def __init__(self, chunks):
        chunks = np.asarray(chunks)
        ncf, nct, cwf, cwt = chunks.shape
        if (ncf > 1 and cwf % 2) or (nct > 1 and cwt % 2):
            raise ValueError("odd chunk width on an axis with more than one chunk")
        hf, ht = cwf // 2, cwt // 2
        self.ncf, self.nct, self.cwf, self.cwt, self.P = ncf, nct, cwf, cwt, ncf * nct
        self.shape = ((ncf - 1) * hf + cwf, (nct - 1) * ht + cwt)
        self.Y = np.zeros((4,) + self.shape, complex)
        self.Y32 = np.zeros((4,) + self.shape, complex)
        self.c64 = chunks.dtype == np.complex64
        self.I = np.full((4,) + self.shape, -1, np.int64)
        uf, ut = ramp(hf), ramp(ht)
        for cf in range(ncf):
            mf = np.ones(cwf)
            if cf > 0:
                mf[:hf] *= uf
            if cf < ncf - 1:
                mf[hf:] *= 1 - uf
            for ct in range(nct):
                mt = np.ones(cwt)
                if ct > 0:
                    mt[:ht] *= ut
                if ct < nct - 1:
                    mt[ht:] *= 1 - ut
                L = 2 * (cf % 2) + ct % 2
                fs = slice(cf * hf, cf * hf + cwf)
                ts = slice(ct * ht, ct * ht + cwt)
                self.Y[L, fs, ts] = chunks[cf, ct] * mf[:, None] * mt[None, :]
                self.Y32[L, fs, ts] = self.Y[L, fs, ts].astype(chunks.dtype)
                self.I[L, fs, ts] = cf * nct + ct

    def y(self, phi, round_phase=False):
        """e^{i phi_k} y_k per layer, with the reference's in-place roundings"""
        y = self.Y32 * self.coef(np.exp(1j * phi))
        return y.astype(np.complex64).astype(complex) if (round_phase and self.c64) else y

    def coef(self, v):
        """per-layer pixel map of a per-chunk value (0 off the chunks)"""
        return np.append(np.asarray(v), 0)[self.I]

    def chunk_sum(self, vals):
        """sum of per-layer pixel values over each chunk's pixels -> [P]"""
        ok = self.I >= 0
        return np.bincount(self.I[ok], weights=vals[ok], minlength=self.P)

    def pairs(self):
        """(layer a, layer b, pixel mask, earlier chunk, later chunk) for every pair of
        distinct layers"""
        for a in range(4):
            for b in range(a + 1, 4):
                ok = (self.I[a] >= 0) & (self.I[b] >= 0)
                ia, ib = self.I[a][ok], self.I[b][ok]
                yield a, b, ok, np.minimum(ia, ib), np.maximum(ia, ib), ia <= ib


def params(lay, p, with_amp):
    P = lay.P
    p = np.asarray(p, np.float64)
    need = 2 * P - 1 if with_amp else P - 1
    if p.shape[0] < need:
        raise IndexError("parameter vector of length %d, need %d" % (p.shape[0], need))
    phi = np.concatenate([[0.0], p[:P - 1]])
    amp = p[P - 1:2 * P - 1] if with_amp else np.ones(P)
    return phi, amp


def mos(lay, phi, amp):
    c = amp * np.exp(1j * phi)
    W = (lay.Y * lay.coef(c)).sum(0)
    Wabs = (np.abs(lay.Y) * lay.coef(np.abs(amp))).sum(0)
    return W, Wabs


def rot_mos(chunks, x):
    lay = Layers(chunks)
    return mos(lay, *params(lay, x, False))


def full_mos(chunks, p):
    lay = Layers(chunks)
    return mos(lay, *params(lay, p, True))


def rot_fit(chunks, x):
    W, Wabs = rot_mos(chunks, x)
    return -np.sum(np.abs(W) ** 2), np.sum(Wabs ** 2)


def rot_der(chunks, x):
    lay = Layers(chunks)
    phi, amp = params(lay, x, False)
    W, Wabs = mos(lay, phi, amp)
    y = lay.y(phi)
    d = 2 * lay.chunk_sum(np.imag(np.conj(W) * y))
    a = 2 * lay.chunk_sum(Wabs * np.abs(y))
    out, oabs = np.zeros(np.shape(x)), np.zeros(np.shape(x))
    out[:lay.P - 1], oabs[:lay.P - 1] = d[1:], a[1:]
    return out, oabs


def overlaps(chunks):
    """C [P][4] complex: C[k][e] = sum y_j conj(y_k) with the earlier neighbour j of type e
    ((cf-1, ct-1), (cf-1, ct), (cf-1, ct+1), (cf, ct-1)), and sum|terms|."""
    lay = Layers(chunks)
    P, nct = lay.P, lay.nct
    C = np.zeros((P, 4), complex)
    A = np.zeros((P, 4))
    for a, b, ok, j, k, _ in lay.pairs():
        ya, yb = lay.Y[a][ok], lay.Y[b][ok]
        aj = lay.I[a][ok] == j
        yj, yk = np.where(aj, ya, yb), np.where(aj, yb, ya)
        prod = yj * np.conj(yk)
        df = k // nct - j // nct
        dt = k % nct - j % nct
        e = np.select([(df == 1) & (dt == 1), (df == 1) & (dt == 0), (df == 1) & (dt == -1)],
                      [0, 1, 2], 3)
        key = k * 4 + e
        C.ravel()[:] += np.bincount(key, weights=prod.real, minlength=4 * P) + \
            1j * np.bincount(key, weights=prod.imag, minlength=4 * P)
        A.ravel()[:] += np.bincount(key, weights=np.abs(prod), minlength=4 * P)
    return C, A


def rot_init(chunks, eps=0.0):
    """x [P-1] and the first-order bound on |x - x_computed| when every overlap sum C[k][e]
    carries an absolute error eps * sum|terms| (propagated through the recurrence;
    an all-zero chunk, whose angle the reference leaves to the signs of zeros, gets 0)."""
    C, A = overlaps(chunks)
    P, nct = C.shape[0], np.shape(chunks)[1]
    rot = np.zeros(P)
    err = np.zeros(P)
    for k in range(1, P):
        cf, ct = divmod(k, nct)
        s, b = 0j, 0.0
        for e, (jf, jt) in enumerate(((cf - 1, ct - 1), (cf - 1, ct), (cf - 1, ct + 1),
                                      (cf, ct - 1))):
            if jf < 0 or jt < 0 or jt >= nct:
                continue
            j = jf * nct + jt
            s += np.exp(1j * rot[j]) * C[k, e]
            b += abs(C[k, e]) * err[j] + eps * A[k, e]
        if s != 0:
            rot[k] = np.angle(s)
            err[k] = b / abs(s)
        else:
            err[k] = np.inf if b > 0 else 0.0
    return rot[1:], err[1:]


def _fit_terms(lay, p, dspec, N, round_phase=False):
    phi, amp = params(lay, p, True)
    W, Wabs = mos(lay, phi, amp)
    n2 = N[:W.shape[0], :W.shape[1]] ** 2
    D = dspec[:W.shape[0], :W.shape[1]]
    wt = np.abs(W) ** 2 - D
    wabs = Wabs ** 2 + np.abs(D)
    y = lay.y(phi, round_phase)
    return phi, amp, W, Wabs, n2, wt, wabs, y


def full_fit(chunks, p, dspec, N):
    lay = Layers(chunks)
    _, _, W, _, _, wt, wabs, _ = _fit_terms(lay, p, dspec, N)
    # the reference divides by N in float64 before squaring; gradient and Hessian square a
    # float32 N in float32 (Nse ** 2), as _fit_terms does
    n2 = np.asarray(N[:W.shape[0], :W.shape[1]], np.float64) ** 2
    t = wt ** 2 / n2
    return np.nansum(t), np.nansum(np.where(np.isnan(t), np.nan, wabs ** 2 / n2))


def full_grad(chunks, p, dspec, N):
    lay = Layers(chunks)
    P = lay.P
    phi, amp, W, Wabs, n2, wt, wabs, y = _fit_terms(lay, p, dspec, N)
    g = 4 * wt * y * np.conj(W) / n2
    bad = np.isnan(g.real) | np.isnan(g.imag)
    g = np.where(bad, 0, g)
    ga = np.where(bad, 0, 4 * wabs * np.abs(y) * Wabs / n2)
    gA, gP = lay.chunk_sum(g.real), lay.chunk_sum(g.imag)
    aA = lay.chunk_sum(ga)
    out, oabs = np.zeros(len(p)), np.zeros(len(p))
    out[P - 1:2 * P - 1], oabs[P - 1:2 * P - 1] = gA, aA
    out[:P - 1] = -amp[1:] * gP[1:]
    oabs[:P - 1] = np.abs(amp[1:]) * aA[1:]
    return out, oabs


def full_hess(chunks, p, dspec, N, sparse=False):
    """Hessian and sum|terms| per entry, dense (len(p), len(p)) arrays or, with
    ``sparse``, scipy.sparse.csr_matrix pairs (every entry is set once)."""
    lay = Layers(chunks)
    P = lay.P
    n = len(p)
    phi, amp, W, Wabs, n2, wt, wabs, y = _fit_terms(lay, p, dspec, N, True)
    t = y * np.conj(W)
    ya = np.abs(y)
    R, C, V, M = [], [], [], []

    def put(r, c, v, m, sym=True):
        R.append(r)
        C.append(c)
        V.append(v)
        M.append(m)
        if sym:
            put(c, r, v, m, False)

    iA = lambda k: k + P - 1           # noqa: E731
    # diagonal: one layer with itself
    s1, s2a, s2b, s3a, s3b, ab = (np.zeros(P) for _ in range(6))
    for L in range(4):
        ok = lay.I[L] >= 0
        k = lay.I[L][ok]
        tt, yy, w, q = t[L][ok], ya[L][ok], wt[ok], n2[ok]
        y2 = yy ** 2
        if lay.c64:
            y2 = (y[L][ok] * np.conj(y[L][ok])).astype(np.complex64).real.astype(float)
        mag = (8 * (yy * Wabs[ok]) ** 2 + 4 * wabs[ok] * yy ** 2 + 4 * wabs[ok] * yy * Wabs[ok]) / q
        for arr, v in ((s1, (8 * tt.real ** 2 + 4 * w * y2) / q),
                       (s2a, -8 * tt.imag * tt.real / q), (s2b, -4 * w * tt.imag / q),
                       (s3a, (8 * tt.imag ** 2 + 4 * w * y2) / q), (s3b, -4 * w * tt.real / q),
                       (ab, mag)):
            arr += np.bincount(k, weights=v, minlength=P)
    ks = np.arange(P)
    put(iA(ks), iA(ks), s1, ab, False)
    k1 = ks[1:]
    m = np.abs(amp[k1]) * ab[k1]
    put(iA(k1), k1 - 1, amp[k1] * s2a[k1] + s2b[k1], m)
    put(k1 - 1, k1 - 1, amp[k1] ** 2 * s3a[k1] + amp[k1] * s3b[k1], np.abs(amp[k1]) * m, False)
    # pairs: two layers
    for a, b, ok, j, k, aj in lay.pairs():
        tu = np.where(aj, t[a][ok], t[b][ok])
        tv = np.where(aj, t[b][ok], t[a][ok])
        yu = np.where(aj, y[a][ok], y[b][ok])
        yv = np.where(aj, y[b][ok], y[a][ok])
        w, q = wt[ok], n2[ok]
        gy = yu * np.conj(yv)
        if lay.c64:     # a product of two complex64 arrays in the reference
            gy = gy.astype(np.complex64).astype(complex)
        yy = np.abs(gy)
        mag = (8 * yy * Wabs[ok] ** 2 + 4 * wabs[ok] * yy) / q
        kk, inv = np.unique(j * P + k, return_inverse=True)
        q0, q1, q2, q3, qm = [np.bincount(inv, weights=v, minlength=len(kk))
                              for v in ((8 * tu.real * tv.real + 4 * w * gy.real) / q,
                                        (-8 * tv.imag * tu.real + 4 * w * gy.imag) / q,
                                        (-8 * tu.imag * tv.real - 4 * w * gy.imag) / q,
                                        (8 * tu.imag * tv.imag + 4 * w * gy.real) / q, mag)]
        uu, vv = kk // P, kk % P
        Au, Av = amp[uu], amp[vv]
        put(iA(uu), iA(vv), q0, qm)
        put(iA(uu), vv - 1, Av * q1, np.abs(Av) * qm)
        sel = uu > 0
        put(iA(vv)[sel], uu[sel] - 1, (Au * q2)[sel], (np.abs(Au) * qm)[sel])
        put(uu[sel] - 1, vv[sel] - 1, (Au * Av * q3)[sel], (np.abs(Au * Av) * qm)[sel])
    R, C, V, M = (np.concatenate(x) for x in (R, C, V, M))
    if sparse:
        from scipy.sparse import csr_matrix
        return (csr_matrix((V, (R, C)), shape=(n, n)), csr_matrix((M, (R, C)), shape=(n, n)))
    H, Ha = np.zeros((n, n)), np.zeros((n, n))
    H[R, C] = V
    Ha[R, C] = M
    return H, Ha
