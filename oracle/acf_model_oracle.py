"""Float64 oracle for scint_sim.ACF (the analytic intensity ACF of Rickett et al. 2014,
App. A; reference scint_sim.py:417-765).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Numpy only, so the GPU tests may use it.

``model(**kwargs)`` evaluates the direct double sum of every lag over the full spatial grid,

    gamma(s, nu) = -i h^2 / (2 pi nu) sum_{x,y} G(x, y) exp(i ((x - sx)^2 + (y - sy)^2) / (2 nu))

one complex exponential per grid point per lag, as the reference does; it does not use the
separation into two chirp vectors that the device uses.  The full ACF is placed by index
arithmetic (|lag| for the mirrored quadrant, the point reflection for the half plane), not
by the reference's flips.  Cost: n^2 exponentials per lag, seconds for the grids of a few
hundred points the tests use.
"""
import numpy as np


def axes(psi=0, phasegrad=0, theta=0, ar=1, alpha=5/3, taumax=4, dnumax=4, nf=51, nt=51,
         amp=1, wn=0, spatial_factor=2, resolution_factor=1, core_factor=2,
         auto_sampling=True):
    """The sampling of the reference's constructor and calc_acf: grids, lags and scalars."""
    nf = nf + 1 if nf % 2 == 0 else nf
    nt = nt + 1 if nt % 2 == 0 else nt
    if auto_sampling:
        sp_fac, res_fac, core_fac = 6 * ar / taumax, 1 + ar / 3, 4
    else:
        sp_fac, res_fac, core_fac = spatial_factor, resolution_factor, core_factor
    dsp = 4 * taumax / (nt - 1)
    ang = (90 - psi) * np.pi / 180          # velocity angle to the e-field major axis
    gang = (90 - psi - theta) * np.pi / 180
    h1, h2 = dsp / res_fac, dsp / (res_fac * core_fac)
    half = sp_fac * taumax
    dnun = np.linspace(0, dnumax, int(np.ceil(nf / 2)))
    if phasegrad == 0:
        tn = np.linspace(0, taumax, int(np.ceil(nt / 2)))
        t_axis = np.concatenate((-tn[:0:-1], tn))
    else:
        tn = np.linspace(-taumax, taumax, nt)
        t_axis = tn
    return dict(nf=nf, nt=nt, sp_fac=sp_fac, res_fac=res_fac, core_fac=core_fac, dsp=dsp,
                snp=np.arange(-half, half + h1, h1), snp2=np.arange(-half, half + h2, h2),
                h1=h1, h2=h2, dnun=dnun, ddnun=np.abs(dnun[1] - dnun[0]),
                fn=np.concatenate((-dnun[:0:-1], dnun)), tn=t_axis, sn=t_axis,
                lag_t=tn, snx=np.cos(ang) * tn, sny=np.sin(ang) * tn,
                sigxn=phasegrad * np.cos(gang), sigyn=phasegrad * np.sin(gang),
                quadrant=phasegrad == 0, alph2=alpha / 2, ar=ar, amp=amp, wn=wn)


def efield(snp, ar, alpha):
    """G[i][j] = exp(-0.5 ((snp[j] / sqrt(ar))^2 + (snp[i] sqrt(ar))^2)^(alpha / 2))."""
    x = snp[None, :] / np.sqrt(ar)
    y = snp[:, None] * np.sqrt(ar)
    return np.exp(-0.5 * (x ** 2 + y ** 2) ** (alpha / 2))


def column0(a):
    """gamma at dnun = 0, the e-field ACF at each lag, with wn/amp at the zero lag(s)."""
    g = np.exp(-0.5 * ((a["snx"] / np.sqrt(a["ar"])) ** 2 +
                       (a["sny"] * np.sqrt(a["ar"])) ** 2) ** a["alph2"])
    zero = np.zeros(len(g), bool)
    if a["quadrant"]:
        zero[0] = True
    else:
        zero[a["snx"] == 0] = True
    return g + np.where(zero, a["wn"] / a["amp"], 0.0)


def gamma(a):
    """The complex e-field ACF of every (time lag, frequency lag), [nsn][ndnun]."""
    nsn, nd = len(a["snx"]), len(a["dnun"])
    out = np.zeros((nsn, nd), np.complex128)
    out[:, 0] = column0(a)
    for k in range(1, nd):
        snp, h = (a["snp2"], a["h2"]) if k == 1 else (a["snp"], a["h1"])
        G = efield(snp, a["ar"], 2 * a["alph2"])
        nu = a["dnun"][k]
        for s in range(nsn):
            sx = a["snx"][s] - 2 * a["sigxn"] * nu
            sy = a["sny"][s] - 2 * a["sigyn"] * nu
            arg = ((snp[None, :] - sx) ** 2 + (snp[:, None] - sy) ** 2) / (2 * nu)
            out[s, k] = -1j * h * h * np.sum(G * np.exp(1j * arg)) / (2 * np.pi * nu)
    return out


def place(I, quadrant):
    """The full [nf][nt] ACF from the intensity I[lag][dnun-column]."""
    nsn, nd = I.shape
    f = np.arange(2 * nd - 1) - (nd - 1)                 # signed frequency-lag index
    if quadrant:
        t = np.arange(2 * nsn - 1) - (nsn - 1)
        return I[np.abs(t)[None, :], np.abs(f)[:, None]]
    t = np.arange(nsn)
    pos = f[:, None] >= 0
    return np.where(pos, I[t[None, :], np.abs(f)[:, None]],
                    I[(nsn - 1 - t)[None, :], np.abs(f)[:, None]])


def model(**kwargs):
    """(axes, acf [nf][nt], acf_efield) in float64."""
    a = axes(**kwargs)
    g = gamma(a)
    acf = a["amp"] * place(np.abs(g) ** 2, a["quadrant"])
    return a, acf, efield(a["snp"], a["ar"], 2 * a["alph2"])


def sspec(acf, window="hanning", frac=1):
    """10 log10 |fftshift(fft2(fftshift(windowed acf)))| in float64 (scint_sim.py:728-742)."""
    nf, nt = acf.shape
    fns = {"hanning": np.hanning, "hamming": np.hamming, "blackman": np.blackman,
           "bartlett": np.bartlett}
    fn = fns[window.lower()]

    def taper(n):
        w = fn(int(np.floor(frac * n)))
        return np.insert(w, int(np.ceil(len(w) / 2)), np.ones(n - len(w)))

    arr = acf * taper(nt)[None, :] * taper(nf)[:, None]
    return 10 * np.log10(np.abs(np.fft.fftshift(np.fft.fft2(np.fft.fftshift(arr)))))
