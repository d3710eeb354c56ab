"""Time of the scintillation-scale fits (Dynspec.get_scint_params, sb_scint_fit_1d / _2d),
with the card read in the same run.

    python profiles/probe_scint_params.py

1. acf1d on a batch of 4096 seeded spectra of 128 x 256 through
   dynspec.get_scint_params_batch, end to end (device ACFs, host steps, one batched fit;
   one warm-up batch of 64 first), against the lmfit stand-in (oracle/scint_params_oracle.py,
   scipy's MINPACK with forward differences) on 64 of the same fits, per spectrum.
2. acf2d_approx with full_frame=True on a 2048 x 4096 ACF (a 1024 x 2048 spectrum): the
   whole call timed with CUDA events after a warm-up, divided by the device's evaluations
   (one evaluation and one solve launch per LM iteration); the fp64 operations and bytes
   of one evaluation from the shape; and one host evaluation of the oracle's residual and
   Jacobian for comparison."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def spectra(n, nf, nt, seed):
    """n spectra: Gaussian-correlated intensity (tau ~ 40 s, dnu ~ 1 MHz, dt 8 s, df 0.25)."""
    rng = np.random.default_rng(seed)
    kt = np.fft.fftfreq(2 * nt, 8.0)[None, :]
    kf = np.fft.fftfreq(2 * nf, 0.25)[:, None]
    out = []
    for _ in range(n):
        tau, dnu = rng.uniform(25, 60), rng.uniform(0.6, 1.5)
        amp = np.exp(-(np.pi * tau * kt) ** 2 - (np.pi * dnu * kf) ** 2)
        z = np.fft.ifft2(amp * (rng.normal(size=amp.shape) + 1j * rng.normal(size=amp.shape)))
        out.append(np.abs(z[:nf, :nt]) ** 2)
    return out


def dynspecs(dyns):
    from scintools_b200.dynspec import Dynspec
    out = []
    for d in dyns:
        ds = Dynspec.__new__(Dynspec)
        ds.dyn, ds.name = d, "probe"
        ds.dt, ds.df, ds.nsub, ds.nchan, ds.freq = 8.0, 0.25, d.shape[1], d.shape[0], 1400.0
        ds.tobs, ds.bw = 8.0 * d.shape[1], 0.25 * d.shape[0]
        out.append(ds)
    return out


def main():
    import torch
    from oracle import scint_params_oracle as SO
    from scintools_b200 import dynspec as P
    print("card:", card())
    # ---- 1: batched acf1d ----
    dyns = spectra(4096, 128, 256, 5)
    P.get_scint_params_batch(dynspecs(dyns[:64]), method="acf1d")
    torch.cuda.synchronize()
    dss = dynspecs(dyns)
    t0 = time.perf_counter()
    res = P.get_scint_params_batch(dss, method="acf1d")
    torch.cuda.synchronize()
    t_batch = time.perf_counter() - t0
    nfev = np.array([r.nfev for r in res])
    print("acf1d batch of 4096 (128 x 256): %.3f s end to end, %.1f us per spectrum; "
          "device evaluations per fit: median %d, max %d; all succeeded: %s"
          % (t_batch, 1e6 * t_batch / 4096, np.median(nfev), nfev.max(),
             all(r.success for r in res)))
    t_host = 0.0
    for ds in dss[:64]:
        pl = P._scint_nofit(ds, False, 5, True, True)
        args = (pl["xdata_t"], pl["xdata_f"], pl["ydata_t"], pl["ydata_f"], pl["weights_t"],
                pl["weights_f"])
        prm = SO.Parameters()
        for n in ("tau", "dnu", "amp"):
            prm.add(n, value=pl[n], min=0, max=np.inf)
        prm.add("alpha", value=5 / 3, vary=False)

        def fcn(p, *a):
            return SO.resid_1d(p.valuesdict(), *a)
        t0 = time.perf_counter()
        SO.Minimizer(fcn, prm, fcn_args=args, max_nfev=50000).minimize()
        t_host += time.perf_counter() - t0
    print("lmfit stand-in (host, one process): %.1f us per spectrum over 64 (fit only, "
          "ACF and host steps excluded)" % (1e6 * t_host / 64))
    SO.CALLS.clear()

    # ---- 2: acf2d_approx, full frame, 2048 x 4096 ----
    nf, nt, dt, df = 1024, 2048, 8.0, 0.05
    tl = (np.arange(2 * nt) - nt) * dt
    fl = (np.arange(2 * nf) - nf) * df
    T, F = np.meshgrid(tl, fl)
    acf = np.exp(-(np.abs((T - 20 * F) / 300.0) ** 2.5 +
                   np.abs(F / (2.0 / np.log(2))) ** 1.5) ** (2 / 3))
    acf *= (1 - np.abs(T) / (nt * dt)) * (1 - np.abs(F) / (nf * df))
    acf += np.random.default_rng(2).normal(0, 0.002, acf.shape)
    acf[nf, nt] += 0.05
    acf /= acf.max()
    ds = dynspecs([np.random.default_rng(3).exponential(1.0, (nf, nt))])[0]
    ds.dt, ds.df, ds.tobs, ds.bw = dt, df, nt * dt, nf * df
    ds.acf = acf
    ds.get_scint_params(method="acf2d_approx", full_frame=True)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    res = ds.get_scint_params(method="acf2d_approx", full_frame=True)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1)
    npts = (2 * nf - 1) * (2 * nt - 1)
    nv = 4
    # per point: the model (pow x3, exp, log, ~40 flops) and the partial sums of the
    # upper triangle of J^T J, J^T r and r^T r (2 (nv (nv+1)/2 + nv + 1) flops); bytes: the
    # ACF read at the point and at the weight's shifted position, 16 bytes
    flops = npts * (40 + 2 * (nv * (nv + 1) // 2 + nv + 1))
    print("acf2d_approx full frame 2048 x 4096 (%d points): %.1f ms for the call (host steps "
          "and the 1-D fit included), %d evaluations of the 2-D fit" % (npts, ms, res.nfev))
    rows, cols, tt, ft = P._scint_crop_2d(ds, 300.0, 2.0, 5, True, False)
    w = SO.weights_2d_rule(acf, rows, cols, tt, ft, ds.nsub, ds.nchan, ds.tobs, ds.bw, True)
    args = (tt[cols], ft[rows], acf[rows[0]:rows[-1] + 1, cols[0]:cols[-1] + 1], w, ds.tobs,
            ds.bw)
    p = {n: res.params[n].value for n in SO.SLOTS}
    t0 = time.perf_counter()
    SO.resid_2d(p, *args, jac=True)
    t_eval = time.perf_counter() - t0
    print("per evaluation: %.2f ms of the whole call / %d; %.3g fp64 flop and %.3g bytes "
          "from the shape; host oracle residual + Jacobian: %.0f ms"
          % (ms / res.nfev, res.nfev, flops, npts * 16.0, 1e3 * t_eval))


if __name__ == "__main__":
    main()
