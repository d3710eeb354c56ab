"""CUDA-native mirror of scintools.scint_sim.Simulation
(reference scintools/scint_sim.py:23-311).

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
what is new here is everything that touches the device.
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
