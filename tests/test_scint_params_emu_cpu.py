"""The device code of the scintillation-scale fits (csrc/scintfit.cu) on the CPU under the
SIMT emulator (tests/host_emu/scintfit_emu.cpp): the unchanged kernels, launched as the
driver launches them, on small 1-D and 2-D problems with several chunks per fit.  The
parameters are within 1e-9 of the tight float64 oracle (oracle/scint_params_oracle.py),
every fit ends at a stationary point, and each fit's bits are the same alone and in a
batch of three."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import scint_params_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(EMU, "scintfit_emu.cpp")
    out = os.path.join(EMU, "_build", "scintfit_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-x",
                    "c++", src, "-o", out], check=True)
    return ctypes.CDLL(out)


def _surface(nf, nt, dt, df, tau, dnu, shear, seed):
    """A small ACF: the 2-D model (tau, dnu, shear s/MHz) with noise and a centre spike."""
    tl = (np.arange(2 * nt) - nt) * dt
    fl = (np.arange(2 * nf) - nf) * df
    T, F = np.meshgrid(tl, fl)
    m = np.exp(-(np.abs((T - shear * F) / tau) ** 2.5 +
                 np.abs(F / (dnu / np.log(2))) ** 1.5) ** (2 / 3))
    m *= (1 - np.abs(T) / (nt * dt)) * (1 - np.abs(F) / (nf * df))
    m += np.random.default_rng(seed).normal(0, 0.01, m.shape)
    m[nf, nt] += 0.05
    return np.ascontiguousarray(m / m.max())


class Problem:
    """One fit: the port's host steps on a Dynspec holding `acf`, as get_scint_params does."""

    def __init__(self, kind, nf, nt, seed, weighted=True):
        from scintools_b200 import _lib
        from scintools_b200 import dynspec as P
        dt, df = 10.0, 0.5
        ds = P.Dynspec.__new__(P.Dynspec)
        ds.dyn = np.ones((nf, nt))
        ds.name = "emu"
        ds.dt, ds.df, ds.tobs, ds.bw, ds.nsub, ds.nchan = dt, df, nt * dt, nf * df, nt, nf
        ds.acf = _surface(nf, nt, dt, df, 60.0 + 10 * seed, 3.0 + seed, 5.0 * seed, seed)
        pl = P._scint_nofit(ds, False, 5, True, weighted)
        d = _lib.ScintFit()
        d.pitch = 2 * nt
        self.keep = [ds.acf]
        if kind == 1:
            self.aux = np.concatenate((pl["weights_t"], pl["weights_f"]))
            d.s0, d.s1 = dt, df
            d.r0, d.c0, d.n0 = nf, nt, pl["nt_c"]
            d.r1, d.c1, d.n1 = nf, nt, pl["nf_c"]
            d.vary, d.max_nfev = 0b111, 50000
            self.p0 = dict(tau=pl["tau"], dnu=pl["dnu"], amp=pl["amp"], alpha=5 / 3,
                           phasegrad=0.0)
            self.args = (pl["xdata_t"], pl["xdata_f"], pl["ydata_t"], pl["ydata_f"],
                         pl["weights_t"], pl["weights_f"])
            self.names = ["tau", "dnu", "amp"]
        else:
            rows, cols, tt, ft = P._scint_crop_2d(ds, pl["tau"], pl["dnu"], 5, True, False)
            at = (ds.tobs - abs(tt)) / max(tt)
            af = (ds.bw - abs(ft)) / max(ft)
            self.aux = np.concatenate((tt[cols], ft[rows], at[cols], af[rows]))
            shf, pf, zf = P._fftshift_positions(len(rows))
            sht, pt, zt = P._fftshift_positions(len(cols))
            d.s0, d.s1, d.c = ds.tobs, ds.bw, float(nf * nt)
            d.r0, d.c0, d.n0, d.n1 = int(rows[0]), int(cols[0]), len(rows), len(cols)
            d.shf, d.sht, d.pf, d.pt, d.zf, d.zt = shf, sht, pf, pt, zf, zt
            d.vary, d.max_nfev, d.weighted = 0b11111, 60000, int(weighted)
            self.p0 = dict(tau=pl["tau"], dnu=pl["dnu"], amp=pl["amp"], alpha=5 / 3,
                           phasegrad=0.0)
            w = SO.weights_2d_rule(ds.acf, rows, cols, tt, ft, nf, nt, ds.tobs, ds.bw, weighted)
            y = ds.acf[rows[0]:rows[-1] + 1, cols[0]:cols[-1] + 1]
            self.args = (tt[cols], ft[rows], y, w, ds.tobs, ds.bw)
            self.names = list(SO.SLOTS)
        self.aux = np.ascontiguousarray(self.aux, dtype=np.float64)
        d.acf, d.aux = ds.acf.ctypes.data, self.aux.ctypes.data
        d.p0 = (_lib.c_dbl * 5)(*[float(self.p0[n]) for n in SO.SLOTS])
        d.bounded = 0b111
        self.desc, self.kind = d, kind


def _run(emu, probs):
    from scintools_b200 import _lib
    arr = (_lib.ScintFit * len(probs))(*[p.desc for p in probs])
    out = np.zeros((len(probs), 11))
    info = np.zeros((len(probs), 2), np.int32)
    assert emu.emu_scint_fit(probs[0].kind, arr, len(probs), out.ctypes.data_as(ctypes.c_void_p),
                             info.ctypes.data_as(ctypes.c_void_p)) == 0
    return out, info


@pytest.mark.parametrize("kind,nf,nt", [(1, 20, 40), (2, 16, 40), (2, 21, 33)])
def test_kernels_match_tight_oracle(emu, kind, nf, nt):
    probs = [Problem(kind, nf, nt, s) for s in range(3)]
    out, info = _run(emu, probs)
    for i, pr in enumerate(probs):
        p = dict(pr.p0)
        p.update({n: out[i, s] for s, n in enumerate(SO.SLOTS) if n in pr.names})
        var = pr.names if kind == 1 else ["tau", "dnu", "amp", "alpha", "phasegrad"]
        tight, chi, trel = SO.fit_tight(kind, pr.args, p, var)
        err, chi_dev, rel = SO.stderr_at(kind, pr.args, p, var)
        print("kind %d fit %d: status %d, %d evaluations, %d points, rel gradient %.1e"
              % (kind, i, info[i, 1], info[i, 0], pr.args[2].size, rel))
        assert info[i, 1] > 0
        assert rel <= 1e-8
        assert out[i, 10] == pytest.approx(chi_dev, rel=1e-12)
        for s, n in enumerate(SO.SLOTS):
            if n in var:
                assert out[i, s] == pytest.approx(tight[n], rel=1e-9, abs=1e-12), n
                assert out[i, 5 + s] == pytest.approx(err[n], rel=1e-6), n
        if kind == 2:
            assert pr.args[2].size > 1024        # several chunks per fit


@pytest.mark.parametrize("kind", [1, 2])
def test_alone_and_batched_bit_identical(emu, kind):
    probs = [Problem(kind, 16, 36, s) for s in range(3)]
    both = _run(emu, probs)
    for i, pr in enumerate(probs):
        alone = _run(emu, [pr])
        assert np.array_equal(alone[0][0], both[0][i], equal_nan=True)
        assert np.array_equal(alone[1][0], both[1][i])
    rev = _run(emu, probs[::-1])
    assert np.array_equal(rev[0][::-1], both[0], equal_nan=True)
