"""CUDA-native mirror of scintools.scint_sim.Simulation
(reference scintools/scint_sim.py:23-311), scint_sim.ACF (:417-765) and
scint_sim.Brightness (:768-958).

Same constructor signature and the same attributes afterwards (w, xyp, xyi,
spe, spi, dyn, freqs, times, df, dt, eta, betaeta, ...), so the result drops
into ``Dynspec(dyn=Simulation(...))`` exactly like the reference's.  The phase
screen and the per-frequency Fresnel propagation run in libscint_b200
(sb_sim_weights / sb_sim_screen / sb_sim_intensity).

Noise: ``seed`` parity with the reference needs the legacy MT19937 stream,
which is sequential; by default the two ``randn(nx, ny)`` fields are therefore
drawn on the host exactly as the reference does (scint_sim.py:173,201-202) and
uploaded.  ``device_rng=True`` draws statistically equivalent Gaussian noise
on the GPU instead (counter-based Philox; no host pass, not the same stream).
Explicit fields can be passed as ``noise=(re, im)``.

Provenance: the scalar bookkeeping -- ``set_constants`` (scint_sim.py:137-167),
``get_dynspec`` / ``get_pulse`` (:238-274) and the unit / axis tail of ``__init__``
(:81-133) -- follows the reference LINE BY LINE (same expressions, comments
dropped), because the drop-in contract is "identical attributes" and SURVEY.md
a12 / a15 keep this glue in Python.  It is restated reference code, not new design;
what is new here is everything that touches the device.  ``ACF`` follows the same rule:
its axes and scalars are the reference's numpy expressions, and the double sum of every
lag runs in libscint_b200 (sb_acf_model_f64).  So does ``Brightness``, whose device half is
sb_brightness_f64 (include/scint_b200_brightness.h).
"""
import numpy as np
import scipy.constants as sc
from scipy.special import gamma

from . import _device as D
from . import _lib


class Simulation():

    def __init__(self, mb2=2, rf=1, ds=0.01, alpha=5 / 3, ar=1, psi=0,
                 inner=0.001, ns=256, nf=256, dlam=0.25, lamsteps=False,
                 seed=None, nx=None, ny=None, dx=None, dy=None, plot=False,
                 verbose=False, freq=1400, dt=30, mjd=60000, nsub=None,
                 efield=False, noise=None, device_rng=False, keep_device=False, lazy=False):
        if plot:
            raise NotImplementedError("plotting is outside the GPU hot path")
        self.mb2 = mb2
        self.rf = rf
        self.ds = ds
        self.dx = dx if dx is not None else ds
        self.dy = dy if dy is not None else ds
        self.alpha = alpha
        self.ar = ar
        self.psi = psi
        self.inner = inner
        self.nx = nx if nx is not None else ns
        self.ny = ny if ny is not None else ns
        self.nf = nf
        self.dlam = dlam
        self.lamsteps = lamsteps
        self.seed = seed
        self._noise = noise
        self._device_rng = device_rng
        self._keep_device = keep_device
        # lazy=True (batch production, BASELINE config 4): the big arrays w / xyp (fp64
        # nx x ny) and xyi stay on the device and are downloaded on first attribute
        # access; spe / spi / dyn and the scalars are always on the host
        self._lazy = bool(lazy)

        self.set_constants()
        if verbose:
            print('Computing screen phase')
        self.get_screen()
        if verbose:
            print('Getting intensity...')
        self.get_intensity(verbose=verbose)
        if nf > 1:
            if verbose:
                print('Computing dynamic spectrum')
            self.get_dynspec()
        self.get_pulse()

        # physical units, scint_sim.py:81-133
        self.name = 'sim:mb2={0},ar={1},psi={2},dlam={3}'.format(
            self.mb2, self.ar, self.psi, self.dlam)
        if lamsteps:
            self.name += ',lamsteps'
        self.header = [self.name, 'MJD0: {}'.format(mjd)]
        dyn = np.real(self.spe) if efield else self.spi
        self.dt = dt
        self.freq = freq
        self.nsub = int(np.shape(dyn)[0]) if nsub is None else nsub
        self.nchan = int(np.shape(dyn)[1])
        if not lamsteps:
            self.df = self.freq * self.dlam / (self.nchan - 1)
            self.freqs = self.freq + np.arange(-self.nchan / 2,
                                               self.nchan / 2, 1) * self.df
        else:
            self.lam = sc.c / (self.freq * 10 ** 6)
            self.dl = self.lam * self.dlam / (self.nchan - 1)
            self.lams = self.lam + np.arange(-self.nchan / 2,
                                             self.nchan / 2, 1) * self.dl
            self.freqs = sc.c / self.lams / 10 ** 6
            self.freq = (np.max(self.freqs) - np.min(self.freqs)) / 2
        self.bw = max(self.freqs) - min(self.freqs)
        self.times = self.dt * np.arange(0, self.nsub)
        self.df = self.bw / self.nchan
        self.tobs = float(self.times[-1] - self.times[0])
        self.mjd = mjd
        if nsub is not None:
            dyn = dyn[0:nsub, :]
        self.dyn = np.transpose(dyn)

        V = self.ds / self.dt
        lambda0 = self.freq
        k = 2 * np.pi / lambda0
        L = self.rf ** 2 * k
        self.eta = L / (2 * V ** 2) / 10 ** 6 / np.cos(psi * np.pi / 180) ** 2
        c = 299792458.0
        beta_to_eta = c * 1e6 / ((self.freq * 10 ** 6) ** 2)
        self.betaeta = self.eta / beta_to_eta
        if not keep_device and not self._lazy:
            self._d_xyp = None

    def __getattr__(self, name):
        # only reached when the attribute is not set yet: lazy download of the big arrays
        src = {"w": "_d_w", "xyp": "_d_xyp", "xyi": "_d_xyi"}.get(name)
        if src is not None and self.__dict__.get("_lazy") and self.__dict__.get(src) is not None:
            val = self.__dict__[src].cpu().numpy().astype(np.float64)
            self.__dict__[name] = val
            if not (name == "xyp" and self.__dict__.get("_keep_device")):
                self.__dict__[src] = None
            return val
        raise AttributeError(name)

    def set_constants(self):
        """scint_sim.py:137-167 (host scalars)."""
        ns = 1
        lenx = self.nx * self.dx
        leny = self.ny * self.dy
        self.ffconx = (2.0 / (ns * lenx * lenx)) * (np.pi * self.rf) ** 2
        self.ffcony = (2.0 / (ns * leny * leny)) * (np.pi * self.rf) ** 2
        dqx = 2 * np.pi / lenx
        dqy = 2 * np.pi / leny
        a2 = self.alpha * 0.5
        aa = 1.0 + a2
        ab = 1.0 - a2
        cdrf = 2.0 ** (self.alpha) * np.cos(self.alpha * np.pi * 0.25) \
            * gamma(aa) / self.mb2
        self.s0 = self.rf * cdrf ** (1.0 / self.alpha)
        cmb2 = self.alpha * self.mb2 / (4 * np.pi * gamma(ab) *
                                        np.cos(self.alpha * np.pi * 0.25) * ns)
        self.consp = cmb2 * dqx * dqy / (self.rf ** self.alpha)
        self.scnorm = 1.0 / (self.nx * self.ny)
        self.sref = self.rf ** 2 / self.s0

    def get_screen(self):
        """Phase screen (scint_sim.py:169-207) on the device, float64."""
        import torch
        nx, ny = self.nx, self.ny
        p = _lib.SimParams(nx, ny, self.dx, self.dy, self.alpha, self.ar,
                           self.psi, self.inner, self.consp)
        d_w = D.empty((nx, ny), torch.float64)
        _lib.check(_lib.lib.sb_sim_weights(p, d_w.data_ptr(), D.stream_ptr()))
        n1 = n2 = None
        seed = 0
        if self._noise is not None:
            n1 = D.upload(np.asarray(self._noise[0], dtype=np.float64))
            n2 = D.upload(np.asarray(self._noise[1], dtype=np.float64))
        elif self._device_rng:
            seed = int(self.seed) if self.seed is not None and self.seed >= 0 \
                else int(np.random.SeedSequence().entropy % (1 << 63))
        else:
            np.random.seed(self.seed)          # legacy stream, as the reference
            n1 = D.upload(np.random.randn(nx, ny))
            n2 = D.upload(np.random.randn(nx, ny))
        d_xyp = D.empty((nx, ny), torch.float64)
        _lib.check(_lib.lib.sb_sim_screen(nx, ny, d_w.data_ptr(), D.ptr(n1),
                                          D.ptr(n2), seed, d_xyp.data_ptr(),
                                          D.stream_ptr()))
        self._d_xyp = d_xyp
        if self._lazy:
            self._d_w = d_w
        else:
            self.w = d_w.cpu().numpy()
            self.xyp = d_xyp.cpu().numpy()

    def _scales(self):
        out = np.empty(self.nf, dtype=np.float64)
        for ifreq in range(self.nf):
            if self.lamsteps:
                out[ifreq] = 1.0 + self.dlam * (ifreq - 1 - (self.nf / 2)) / self.nf
            else:
                out[ifreq] = 1 / (1.0 + self.dlam * (-0.5 + ifreq / self.nf))
        return out

    def get_intensity(self, verbose=True):
        """Fresnel propagation per frequency (scint_sim.py:209-236, 294-311)."""
        import torch
        nx, ny, nf = self.nx, self.ny, self.nf
        if getattr(self, "_d_xyp", None) is None:
            self._d_xyp = D.upload(np.asarray(self.xyp, dtype=np.float64))
        scales = np.ascontiguousarray(self._scales())
        d_spe = D.empty((nf, nx, 2), torch.float32)
        d_xyi = D.empty((nx, ny), torch.float32)
        _lib.check(_lib.lib.sb_sim_intensity(
            nx, ny, nf, self._d_xyp.data_ptr(), scales.ctypes.data, self.ffconx,
            self.ffcony, d_spe.data_ptr(), d_xyi.data_ptr(), D.stream_ptr()))
        a = d_spe.cpu().numpy()
        spe_t = (a[..., 0] + 1j * a[..., 1]).astype(np.csingle)   # [nf][nx]
        self.spe = np.ascontiguousarray(spe_t.T)                  # [nx][nf]
        if self._lazy:
            self._d_xyi = d_xyi
        else:
            self.xyi = d_xyi.cpu().numpy().astype(np.float64)

    def get_dynspec(self):
        """scint_sim.py:238-252."""
        if self.nf == 1:
            print('no spectrum because nf=1')
        self.spi = np.real(np.multiply(self.spe, np.conj(self.spe)))
        self.x = np.linspace(0, self.dx * (self.nx), (self.nx))
        ifreq = np.linspace(0, self.nf - 1, self.nf)
        lam_norm = 1.0 + self.dlam * (ifreq - 1 - (self.nf / 2)) / self.nf
        self.lams = lam_norm / np.mean(lam_norm)
        frfreq = 1.0 + self.dlam * (-0.5 + ifreq / self.nf)
        self.freqs = frfreq / np.mean(frfreq)

    def get_pulse(self):
        """scint_sim.py:254-274 (small 1-D FFT, host numpy as the reference)."""
        p = np.fft.fft(np.multiply(self.spe, np.blackman(self.nf)), 2 * self.nf)
        p = np.real(p * np.conj(p))
        self.pulsewin = np.transpose(np.roll(p, self.nf))
        if self._lazy and "xyp" not in self.__dict__:
            col = self._d_xyp[:, int(self.ny / 2)].cpu().numpy()   # one column, not 8 n^2 bytes
        else:
            col = self.xyp[:, int(self.ny / 2)]
        self.dm = col * self.dlam / np.pi


# sizes the device contraction takes (csrc/acf_model.cu)
_ACF_MAX_GRID = 16384
_ACF_MAX_N = 8191


def _arange_len(start, stop, step):
    """len(np.arange(start, stop, step)), from numpy's own formula, without allocating; a
    zero step raises ZeroDivisionError as np.arange does."""
    return max(int(np.ceil((float(stop) - float(start)) / float(step))), 0)


class ACF():
    """The theoretical intensity ACF of Rickett et al. (2014, App. A) for an anisotropic
    medium with a phase gradient (scint_sim.py:417-765).

    Same constructor signature and the same attributes afterwards: alpha ar psi phasegrad
    theta amp wn taumax dnumax nf nt sp_fac res_fac core_fac dsp ddnun fn tn sn snp acf
    acf_efield.  The axes are built on the host with the reference's expressions; the
    e-field ACF and the double sum of every (time lag, frequency lag) run on the device in
    float64 as a bilinear form (csrc/acf_model.cu).  No device memory is held afterwards.

    The reference's errors are kept, raised before any device work: even nf / nt become
    odd; nf = 1 raises IndexError, nt = 1 and amp = 0 ZeroDivisionError.  Deviations:
    non-finite parameters, ar <= 0 and dnumax = 0 raise ValueError (the reference returns
    NaN), as do spatial grids of more than 16384 points per side and nf or nt above 8191.
    ``plot=True`` and the ``plot_*`` methods raise NotImplementedError.
    """

    def __init__(self, psi=0, phasegrad=0, theta=0, ar=1, alpha=5/3,
                 taumax=4, dnumax=4, nf=51, nt=51, amp=1, wn=0,
                 spatial_factor=2, resolution_factor=1, core_factor=2,
                 auto_sampling=True, plot=False, display=True):
        if plot:
            raise NotImplementedError("plotting is outside the GPU hot path")
        self.alpha = alpha
        self.ar = ar
        self.psi = psi
        self.phasegrad = phasegrad
        self.theta = theta
        self.amp = amp
        self.wn = wn
        self.taumax = taumax
        spmax = taumax
        self.dnumax = dnumax
        if nf % 2 == 0:
            nf += 1
        if nt % 2 == 0:
            nt += 1
        self.nf = nf
        self.nt = nt
        if auto_sampling:
            self.sp_fac = 6 * ar/spmax
            self.res_fac = 1 + ar/3
            self.core_fac = 4
        else:
            self.sp_fac = spatial_factor
            self.res_fac = resolution_factor
            self.core_fac = core_factor
        self.dsp = 4*spmax/(nt-1)
        self.calc_acf()

    def _axes(self):
        """The host half of calc_acf (scint_sim.py:538-587, 630-637): every axis and scalar
        in the reference's expressions and order, so its exceptions come first.  Then the
        checks this port adds.  Returns a dict; nothing touches the device."""
        alph2 = self.alpha/2
        spmax = self.taumax
        dnumax = self.dnumax
        dsp = self.dsp
        phasegrad = self.phasegrad
        theta = self.theta
        amp = self.amp
        wn = self.wn
        xi = 90 - self.psi
        with np.errstate(all="ignore"):
            Vx = np.cos(xi*np.pi/180)
            Vy = np.sin(xi*np.pi/180)
            sigxn = phasegrad * np.cos((xi - theta)*np.pi/180)
            sigyn = phasegrad * np.sin((xi - theta)*np.pi/180)
            ar = self.ar
            sqrtar = np.sqrt(ar)
        dnun = np.linspace(0, dnumax, int(np.ceil(self.nf/2)))
        ddnun = np.abs(dnun[1] - dnun[0])
        sp_fac = self.sp_fac
        res_fac = self.res_fac
        core_fac = self.res_fac * self.core_fac
        start, stop1, stop2 = -sp_fac*spmax, sp_fac*spmax + dsp/res_fac, \
            sp_fac*spmax + dsp/core_fac
        n1 = _arange_len(start, stop1, dsp/res_fac)
        n2 = _arange_len(start, stop2, dsp/core_fac)
        quadrant = phasegrad == 0
        if quadrant:
            tn = np.linspace(0, (spmax), int(np.ceil(self.nt/2)))
            snx = Vx*tn
            sny = Vy*tn
        else:
            tn = np.linspace(-(spmax), (spmax), self.nt)
            snx = np.cos(xi*np.pi/180)*tn
            sny = np.sin(xi*np.pi/180)*tn
        wn_amp = wn/amp
        scalars = [self.alpha, self.ar, self.psi, phasegrad, theta, amp, wn, spmax, dnumax,
                   dsp, sp_fac, res_fac, core_fac, wn_amp]
        if not all(np.isfinite(np.asarray(v, dtype=np.float64)).all() for v in scalars):
            raise ValueError("ACF parameters must be finite")
        if not ar > 0:
            raise ValueError("ar must be positive (the reference returns NaN)")
        if dnumax == 0:
            raise ValueError("dnumax must be non-zero (the reference divides by it)")
        if not (1 <= n1 <= _ACF_MAX_GRID and 1 <= n2 <= _ACF_MAX_GRID):
            raise ValueError("spatial grids of %d and %d points are outside 1..%d"
                             % (n1, n2, _ACF_MAX_GRID))
        if not (3 <= self.nf <= _ACF_MAX_N and 3 <= self.nt <= _ACF_MAX_N):
            raise ValueError("nf = %s and nt = %s must be within 3..%d"
                             % (self.nf, self.nt, _ACF_MAX_N))
        snp = np.arange(-sp_fac*spmax, sp_fac*spmax + dsp/res_fac, dsp/res_fac)
        snp2 = np.arange(-sp_fac*spmax, sp_fac*spmax + dsp/core_fac, dsp/core_fac)
        assert len(snp) == n1 and len(snp2) == n2
        if quadrant:
            t2 = np.concatenate((np.flip(-tn[1:]), tn)).squeeze()
        else:
            t2 = tn
        f2 = np.concatenate((np.flip(-dnun[1:]), dnun)).squeeze()
        return dict(alph2=alph2, sigxn=float(sigxn), sigyn=float(sigyn),
                    sqrtar=float(sqrtar), dnun=dnun, ddnun=ddnun, snp=snp, snp2=snp2,
                    step1=dsp/res_fac, step2=dsp/core_fac, quadrant=bool(quadrant),
                    snx=np.asarray(snx, dtype=np.float64),
                    sny=np.asarray(sny, dtype=np.float64), wn_amp=float(wn_amp),
                    amp=float(amp), fn=f2, t2=t2)

    def calc_acf(self, plot=False):
        """Computes the 2-D ACF of intensity vs time and frequency lag (scint_sim.py:494-678),
        re-reading the attributes as the reference does."""
        if plot:
            raise NotImplementedError("plotting is outside the GPU hot path")
        import torch
        ax = self._axes()
        snp, snp2, dnun = ax["snp"], ax["snp2"], ax["dnun"]
        nsn, ndnun = len(ax["snx"]), len(dnun)
        nt_out = 2 * nsn - 1 if ax["quadrant"] else nsn
        d = [D.upload(np.ascontiguousarray(v, dtype=np.float64))
             for v in (snp, snp2, dnun, ax["snx"], ax["sny"])]
        m = _lib.AcfModel(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(),
                          d[4].data_ptr(), len(snp), len(snp2), ndnun, nsn,
                          int(ax["quadrant"]), ax["sigxn"], ax["sigyn"], ax["sqrtar"],
                          float(ax["alph2"]), float(ax["step1"]), float(ax["step2"]),
                          ax["wn_amp"], ax["amp"])
        d_acf = D.empty((2 * ndnun - 1, nt_out), torch.float64)
        d_ef = D.empty((len(snp), len(snp)), torch.float64)
        _lib.check(_lib.lib.sb_acf_model_f64(m, d_acf.data_ptr(), d_ef.data_ptr(),
                                              D.stream_ptr()))
        self.ddnun = ax["ddnun"]
        self.fn = ax["fn"]
        self.tn = ax["t2"]
        self.sn = ax["t2"]
        self.snp = snp
        self.acf = d_acf.cpu().numpy()
        self.acf_efield = d_ef.cpu().numpy()

    def calc_sspec(self, window='hanning', window_frac=1):
        """The secondary spectrum of the ACF, 10 log10 |fftshift(fft2(fftshift(windowed)))|
        (scint_sim.py:728-742), through the chirp-z 2-D transform (float32).  For a real
        input |fft2| = n0 n1 |ifft2|."""
        import torch
        from .dynspec import get_window
        nf, nt = np.shape(self.acf)
        chan_window, subint_window = get_window(nt, nf, window=window, frac=window_frac)
        arr = np.multiply(chan_window, self.acf)
        arr = np.transpose(np.multiply(subint_window, np.transpose(arr)))
        arr = np.fft.fftshift(arr)
        d_in = D.upload_f32(arr.astype(np.complex128))
        d_out = D.empty((nf, nt, 2), torch.float32)
        _lib.check(_lib.lib.sb_ifft2_c2c_f32(d_in.data_ptr(), nf, nt, 0, 0, 0,
                                              float(nf) * float(nt), 0, d_out.data_ptr(),
                                              D.stream_ptr()))
        a = d_out.cpu().numpy().astype(np.float64)
        amp = np.fft.fftshift(np.hypot(a[..., 0], a[..., 1]))
        with np.errstate(divide="ignore"):
            self.sspec = 10*np.log10(amp)

    def plot_acf(self, display=True, contour=True, filled=False):
        raise NotImplementedError("plotting is outside the GPU hot path")

    def plot_acf_efield(self, display=True):
        raise NotImplementedError("plotting is outside the GPU hot path")

    def plot_sspec(self, display=True, vmin=None, vmax=None):
        raise NotImplementedError("plotting is outside the GPU hot path")


# sizes the device takes (include/scint_b200_brightness.h)
_BRIGHT_MAX_N = 1024          # lattice points per side
_BRIGHT_MAX_Q = 4096          # len(td), len(fd)
_BRIGHT_NPAR = 7
_BRIGHT_EFIELD, _BRIGHT_SSPEC, _BRIGHT_ACF = 1, 2, 4
_BRIGHT_GROUP_BYTES = 4 << 30  # device memory of one batched pass, outputs and workspace
_BRIGHT_SET_KEYS = ("ar", "psi", "alpha", "thetagx", "thetagy", "thetarx", "thetary")
_BRIGHT_GRID_KEYS = ("nx", "dx", "nf", "df", "nt", "dt")
_TRIANGULATIONS = {}           # sha256 of the lattice axis -> packed diagonal bits


def lattice_diagonals(x):
    """The diagonal qhull splits each cell of the lattice meshgrid(x, x) along, as
    griddata((X.ravel(), Y.ravel()), ...) triangulates it: (n-1)^2 bits, cell k = i (n-1) + j,
    set where the cell's two triangles share the corners (x[j], x[i]) and (x[j+1], x[i+1]),
    packed by np.packbits.  Built once per lattice (scipy.spatial.Delaunay, seconds on 600^2)
    and cached.  Raises ValueError if any simplex is not half of a lattice cell."""
    import hashlib
    x = np.ascontiguousarray(x, dtype=np.float64)
    key = hashlib.sha256(x.tobytes()).hexdigest()
    if key not in _TRIANGULATIONS:
        from scipy.spatial import Delaunay
        n = len(x)
        X, Y = np.meshgrid(x, x)
        simp = Delaunay(np.column_stack((np.ravel(X), np.ravel(Y)))).simplices
        i, j = simp // n, simp % n
        i0, j0 = i.min(axis=1), j.min(axis=1)
        corner = (i - i0[:, None]) * 2 + (j - j0[:, None])      # 0 (j,i) 1 (j+1,i) 2 3
        half = ((i.max(axis=1) - i0 == 1) & (j.max(axis=1) - j0 == 1) &
                (np.sort(corner, axis=1) != np.sort(corner, axis=1)[:, [1, 2, 0]]).all(axis=1))
        if len(simp) != 2 * (n - 1) ** 2 or not half.all():
            raise ValueError("the triangulation of the lattice has simplices that are not half "
                             "of a lattice cell; the cell rule does not apply")
        missing = 6 - corner.sum(axis=1)
        main = (missing == 1) | (missing == 2)
        cell = i0 * (n - 1) + j0
        count = np.bincount(cell, minlength=(n - 1) ** 2)
        nmain = np.bincount(cell, weights=main, minlength=(n - 1) ** 2)
        nmiss = np.bincount(cell, weights=missing, minlength=(n - 1) ** 2)
        # two triangles per cell on one diagonal: missing corners {1, 2} or {0, 3}
        if not ((count == 2).all() and np.isin(nmain, (0, 2)).all() and (nmiss == 3).all()):
            raise ValueError("the triangulation of the lattice does not split every cell in two "
                             "along one diagonal; the cell rule does not apply")
        _TRIANGULATIONS[key] = np.packbits(nmain > 0)
    return _TRIANGULATIONS[key]


def _efield_host(o):
    """calc_brightness's host half (scint_sim.py:843-852): the reference's expressions."""
    x = np.arange(-o.nx, o.nx, o.dx)
    X, Y = np.meshgrid(x, x)
    with np.errstate(all="ignore"):
        R = (o.ar**2 - 1) / (o.ar**2 + 1)
        cosa = np.cos(2 * (90 - o.psi) * np.pi/180)
        sina = np.sin(2 * (90 - o.psi) * np.pi/180)
        a = (1 - R * cosa) / np.sqrt(1 - R**2)
        b = (1 + R * cosa) / np.sqrt(1 - R**2)
        c = -2 * R * sina / np.sqrt(1 - R**2)
    if not np.isfinite([a, b, c]).all():
        raise ValueError("the quadratic form of ar = %r, psi = %r is not finite (a=%r, b=%r, "
                         "c=%r)" % (o.ar, o.psi, a, b, c))
    alph2 = o.alpha/2
    if not np.isfinite(alph2):
        raise ValueError("alpha must be finite")
    if not 2 <= len(x) <= _BRIGHT_MAX_N:
        raise ValueError("the lattice has %d points per side, outside 2..%d"
                         % (len(x), _BRIGHT_MAX_N))
    return x, X, Y, [float(a), float(b), float(c), float(alph2)]


def _lattice_axis(o):
    """The vector X, Y are the meshgrid of (calc_SS re-reads them); ValueError if they are
    not the meshgrid of one strictly increasing vector."""
    X, Y = np.asarray(o.X, dtype=np.float64), np.asarray(o.Y, dtype=np.float64)
    B = np.asarray(o.B)
    if X.ndim != 2 or X.shape[0] != X.shape[1] or Y.shape != X.shape or B.shape != X.shape:
        raise ValueError("X, Y and B must be square arrays of one shape")
    x = X[0]
    if not (np.array_equal(X, np.broadcast_to(x, X.shape)) and
            np.array_equal(Y, np.broadcast_to(x[:, None], X.shape)) and
            np.all(np.diff(x) > 0)):
        raise ValueError("X, Y must be meshgrid(x, x) of one strictly increasing x")
    if not 2 <= len(x) <= _BRIGHT_MAX_N:
        raise ValueError("the lattice has %d points per side, outside 2..%d"
                         % (len(x), _BRIGHT_MAX_N))
    return np.ascontiguousarray(x)


def _sspec_host(o):
    """calc_SS's host half (scint_sim.py:901-925): the axes, each Doppler column's thetax,
    (thetax + thetagx)**2 by the reference's scalar power (C pow, which is not always x*x),
    and the scalars, each by the reference's expression."""
    import math
    fd = np.arange(-o.nf, o.nf, o.df)
    td = np.arange(-o.nt, o.nt, o.dt)
    if not (1 <= len(td) <= _BRIGHT_MAX_Q and 1 <= len(fd) <= _BRIGHT_MAX_Q):
        raise ValueError("len(td) = %d and len(fd) = %d must be within 1..%d"
                         % (len(td), len(fd), _BRIGHT_MAX_Q))
    colx = fd - o.thetagx + o.thetarx
    colq = np.array([math.pow(float(v + o.thetagx), 2) for v in colx])
    rx2, ry2 = o.thetarx**2, o.thetary**2
    scal = dict(half_df=float(0.5*o.df), jac_cap=float(2/o.df), jac_out=float(10**(-6)))
    return fd, td, colx, colq, [float(o.thetagy), float(rx2), float(ry2)], scal


def _run(objs, stages):
    """One device pass of the given stages for a list of Brightness objects that share their
    lattice and query grid.  Stages not run here take their inputs from the objects' B and
    SS.  The host halves run (and raise) before any device work."""
    import torch
    ns = len(objs)
    par = np.zeros((ns, _BRIGHT_NPAR))
    hosts = [None] * ns
    x = None
    if stages & _BRIGHT_EFIELD:
        for k, o in enumerate(objs):
            x, X, Y, p = _efield_host(o)
            hosts[k] = (x, X, Y)
            par[k, :4] = p
    q = None
    if stages & _BRIGHT_SSPEC:
        if x is None:
            x = _lattice_axis(objs[0])
        q = [_sspec_host(o) for o in objs]
        for k, h in enumerate(q):
            par[k, 4:] = h[4]
    n = len(x) if x is not None else 2
    ntd = nfd = 1
    if stages & _BRIGHT_SSPEC:
        fd, td = q[0][0], q[0][1]
        ntd, nfd = len(td), len(fd)
    elif stages & _BRIGHT_ACF:
        ntd, nfd = np.shape(objs[0].SS)
    z = lambda shape: D.empty(shape, torch.float64)   # noqa: E731
    keep = []

    def up(a):
        t = D.upload(np.ascontiguousarray(a, dtype=np.float64))
        keep.append(t)
        return t.data_ptr()
    m = _lib.Brightness()
    m.nset, m.n, m.ntd, m.nfd, m.stages = ns, n, ntd, nfd, stages
    out = {}
    if stages & (_BRIGHT_EFIELD | _BRIGHT_SSPEC):
        m.x, m.par = up(x), up(par)
    if stages & _BRIGHT_EFIELD:
        out["acf_efield"], out["B"] = z((ns, n, n)), z((ns, n, n))
        m.rho, m.B = out["acf_efield"].data_ptr(), out["B"].data_ptr()
    elif stages & _BRIGHT_SSPEC:
        m.B = up(np.stack([np.asarray(o.B, dtype=np.float64) for o in objs]))
    if stages & _BRIGHT_SSPEC:
        bits = lattice_diagonals(x)
        d_bits = D.upload(bits)
        keep.append(d_bits)
        m.diag, m.td = d_bits.data_ptr(), up(td)
        m.colx, m.colq = up(np.stack([h[2] for h in q])), up(np.stack([h[3] for h in q]))
        m.half_df, m.jac_cap, m.jac_out = (q[0][5][k] for k in ("half_df", "jac_cap", "jac_out"))
        for k in ("thetax", "thetay", "jacobian", "SS", "LSS"):
            out[k] = z((ns, ntd, nfd))
        m.thetax, m.thetay, m.jac = (out[k].data_ptr() for k in ("thetax", "thetay", "jacobian"))
        m.ss, m.lss = out["SS"].data_ptr(), out["LSS"].data_ptr()
    elif stages & _BRIGHT_ACF:
        m.ss = up(np.stack([np.asarray(o.SS, dtype=np.float64) for o in objs]))
    if stages & _BRIGHT_ACF:
        out["acf"] = z((ns, ntd, nfd))
        m.acf = out["acf"].data_ptr()
    _lib.check(_lib.lib.sb_brightness_f64(m, D.stream_ptr()))
    host = {k: v.cpu().numpy() for k, v in out.items()}
    for k, o in enumerate(objs):
        if stages & _BRIGHT_EFIELD:
            o.x, (o.X, o.Y) = hosts[k][0], hosts[k][1:]
        if stages & _BRIGHT_SSPEC:
            o.fd, o.td = q[k][0], q[k][1]
        for name, arr in host.items():
            setattr(o, name, arr[k])


class Brightness():
    """The delay-Doppler model of an anisotropic scattered image interfering with an
    unscattered wave (Yao et al. 2020, modified by Coles; scint_sim.py:768-958).

    Same constructor signature, defaults and attributes afterwards: ar alpha psi thetagx
    thetagy thetarx thetary df dt dx nf nt nx ncuts x X Y acf_efield B fd td thetax thetay
    jacobian SS LSS acf.  calc_brightness, calc_SS and calc_acf re-read the attributes the
    reference reads and can be called on their own; calc_acf=True with calc_sspec=False
    raises AttributeError on SS, as the reference does.  The axes and scalars are the
    reference's numpy expressions; the e-field ACF, both 2-D DFTs (float64 matrix products on
    the tensor cores), the secondary spectrum and its interpolation run on the device
    (csrc/brightness.cu).  The interpolation is griddata's linear interpolant, evaluated
    through the lattice's triangulation (lattice_diagonals), so it agrees with griddata to
    rounding and is NaN where griddata is.

    Deviations, raised as ValueError before any device work: a non-finite quadratic form
    (ar = 0, for example), lattices of more than 1024 points per side, len(td) or len(fd)
    above 4096, X / Y that are not meshgrid(x, x) of one increasing x, and a triangulation
    with a simplex that is not half a lattice cell.  ``plot=True`` and the ``plot_*``
    methods raise NotImplementedError.  brightness_batch evaluates many parameter sets in
    one pass, each bit-identical to its own Brightness(...).
    """

    def __init__(self, ar=1.0, psi=0, alpha=1.67, thetagx=0, thetagy=0,
                 thetarx=0, thetary=0, df=0.02, dt=0.08, dx=0.1,
                 nf=10, nt=80, nx=30, ncuts=5, plot=False, contour=True,
                 figsize=(10, 8), calc_sspec=True, calc_acf=True):
        if plot:
            raise NotImplementedError("plotting is outside the GPU hot path")
        self.ar = ar
        self.alpha = alpha
        self.thetagx = thetagx
        self.thetagy = thetagy
        self.thetarx = thetarx
        self.thetary = thetary
        self.psi = psi
        self.df = df
        self.dt = dt
        self.dx = dx
        self.nf = nf
        self.nt = nt
        self.nx = nx
        self.ncuts = ncuts
        if calc_acf and not calc_sspec:
            self.calc_brightness()
            self.calc_acf()     # AttributeError on self.SS, as the reference
        _run([self], _BRIGHT_EFIELD | (_BRIGHT_SSPEC if calc_sspec else 0) |
             (_BRIGHT_ACF if calc_acf else 0))

    def calc_brightness(self):
        """acf_efield and B = |ifftshift(fft2(fftshift(acf_efield)))| (scint_sim.py:838-869)."""
        _run([self], _BRIGHT_EFIELD)

    def calc_SS(self):
        """thetax, thetay, jacobian, SS and LSS from B on the lattice X, Y
        (scint_sim.py:871-951)."""
        _run([self], _BRIGHT_SSPEC)

    def calc_acf(self):
        """acf = real(fftshift(fft2(fftshift(SS)))) / its maximum (scint_sim.py:953-958)."""
        _run([self], _BRIGHT_ACF)

    def plot_acf_efield(self, figsize=(6, 6)):
        raise NotImplementedError("plotting is outside the GPU hot path")

    def plot_brightness(self, figsize=(6, 6)):
        raise NotImplementedError("plotting is outside the GPU hot path")

    def plot_sspec(self, figsize=(6, 6)):
        raise NotImplementedError("plotting is outside the GPU hot path")

    def plot_cuts(self, figsize=(6, 6)):
        raise NotImplementedError("plotting is outside the GPU hot path")

    def plot_acf(self, figsize=(6, 6), contour=False):
        raise NotImplementedError("plotting is outside the GPU hot path")


def brightness_batch(params, **shared):
    """One Brightness per dict of ``params``, computed in batched device passes.

    Each dict holds any of ``ar psi alpha thetagx thetagy thetarx thetary``; ``shared`` holds
    the grid keywords ``nx dx nf df nt dt``; every other argument takes Brightness's default.
    The sets share one lattice, one triangulation and one set of DFT twiddle matrices and run
    in groups of at most 4 GiB of device memory.  Each returned object is bit-identical to
    Brightness(**dict, **shared).  Every set's host half runs (and raises) before any device
    work."""
    bad = set(shared) - set(_BRIGHT_GRID_KEYS)
    if bad:
        raise TypeError("brightness_batch: %s are not grid keywords (%s)"
                        % (sorted(bad), " ".join(_BRIGHT_GRID_KEYS)))
    objs = []
    for p in params:
        bad = set(p) - set(_BRIGHT_SET_KEYS)
        if bad:
            raise TypeError("brightness_batch: %s are not per-set keywords (%s)"
                            % (sorted(bad), " ".join(_BRIGHT_SET_KEYS)))
        o = Brightness.__new__(Brightness)
        kw = dict(ar=1.0, psi=0, alpha=1.67, thetagx=0, thetagy=0, thetarx=0, thetary=0,
                  df=0.02, dt=0.08, dx=0.1, nf=10, nt=80, nx=30, ncuts=5)
        kw.update(shared)
        kw.update(p)
        o.__dict__.update(kw)
        objs.append(o)
    if not objs:
        return []
    for o in objs:              # every error before the first launch
        _efield_host(o)
        _sspec_host(o)
    x = _efield_host(objs[0])[0]
    fd, td = _sspec_host(objs[0])[:2]
    lattice_diagonals(x)
    ntd, nfd = len(td), len(fd)
    n2, nq = len(x) ** 2, ntd * nfd
    twiddles = 16 * max(n2, ntd * ntd + nfd * nfd)
    per_set = 8 * (2 * n2 + 7 * nq) + 16 * max(n2, nq)
    group = int(max(1, min(65535, (_BRIGHT_GROUP_BYTES - twiddles) // per_set)))
    for g in range(0, len(objs), group):
        _run(objs[g:g + group], _BRIGHT_EFIELD | _BRIGHT_SSPEC | _BRIGHT_ACF)
    return objs
