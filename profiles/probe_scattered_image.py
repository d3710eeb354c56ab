"""Time of the scattered image (Dynspec.calc_scattered_image, scattered_image_batch,
sb_scattered_image_f64), with the card read in the same run.

    python profiles/probe_scattered_image.py [out.json]

Sizes: the secondary spectrum of a seeded 1024 x 2048 and 4096 x 8192 dynamic spectrum
(1024 x 4096 and 4096 x 16384), each with a curvature whose crop keeps the central 2/5 of
the Doppler columns, and the 64 tiles of cut_dyn(7, 7) of the 4096 x 8192 one (512 x 2048
each) in one batch.  sampling=64 (the default) throughout.

  stages   device time per kernel from torch.profiler over 5 calls (after a warm-up), per
           call: si_linear (10**(x/10) of the crop), si_delay, si_doppler, si_eval,
           si_shift; and GB/s against the bytes each pass must move: linear 16, delay 32,
           doppler 32 bytes per crop element (one read and one write per sweep)
  call     the public call end to end (upload, device, download), host clock, median of 5
  scipy    RectBivariateSpline(tdel, fdop, linsspec) and .ev at the image points on this
           host, once (the 64-tile case: one tile, times 64)"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KERNELS = ("si_linear", "si_delay", "si_doppler", "si_eval", "si_shift")
BYTES = {"si_linear": 16, "si_delay": 32, "si_doppler": 32}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def dynspec(nf, nt, seed):
    from scintools_b200.dynspec import BasicDyn, Dynspec
    rng = np.random.default_rng(seed)
    dyn = rng.gamma(2.0, 1.0, (nf, nt)).astype(np.float32)
    return Dynspec(dyn=BasicDyn(dyn, times=8.0 * np.arange(nt),
                                freqs=1300 + 0.05 * np.arange(nf), dt=8.0, df=0.05),
                   verbose=False)


def stage_times(fn, ncall=5):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(ncall):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                out[k] += ev.device_time_total / 1e3 / ncall      # ms per call
    return out


def host_time(fn, n=5):
    import torch
    fn()
    ts = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def scipy_time(spec, fdop, tdel, eta, sampling=64):
    from scipy.interpolate import RectBivariateSpline
    from oracle.scattered_image_oracle import crop
    lin, x, y = crop(10 ** (spec / 10), fdop, tdel, eta)
    t0 = time.perf_counter()
    sp = RectBivariateSpline(x, y, lin)
    t1 = time.perf_counter()
    fx = np.linspace(-max(y), max(y), 2 * sampling + 1)
    fy = np.linspace(0, max(y), sampling + 1)
    X, Y = np.meshgrid(fx, fy)
    sp.ev((X ** 2 + Y ** 2) * eta, X)
    t2 = time.perf_counter()
    return {"fit_s": t1 - t0, "ev_s": t2 - t1, "crop": list(lin.shape)}


def main(out_path):
    from scintools_b200 import dynspec as DS
    res = {"card": card(), "cases": {}}
    for nf, nt in ((1024, 2048), (4096, 8192)):
        ds = dynspec(nf, nt, nf)
        ds.calc_sspec()
        S, fd, td = ds.sspec, ds.fdop, ds.tdel
        eta = float(np.max(td)) / (0.2 * np.max(fd)) ** 2
        plan = DS._scatim_plan(S.shape, fd, td, eta, 64)
        mxy = (plan["rows"][1] - plan["rows"][0]) * (plan["cols"][1] - plan["cols"][0])
        call = lambda: ds.calc_scattered_image(input_sspec=S, input_fdop=fd,  # noqa: E731
                                               input_tdel=td, input_eta=eta)
        st = stage_times(call)
        case = {"sspec": list(S.shape), "crop_elems": mxy, "stages_ms": st,
                "GBps": {k: BYTES[k] * mxy / (st[k] * 1e-3) / 1e9 for k in BYTES if st[k]},
                "device_ms": sum(st.values()), "call_s": host_time(call),
                "scipy": scipy_time(S, fd, td, eta)}
        res["cases"]["%dx%d" % (nf, nt)] = case
        print(json.dumps({"%dx%d" % (nf, nt): case}), flush=True)
        if nf == 4096:
            ds.cut_dyn(tcuts=7, fcuts=7)
            T = ds.cutsspec
            tfd, ttd, _ = ds.calc_sspec(input_dyn=ds.cutdyn[0, 0])
            teta = float(np.max(ttd)) / (0.2 * np.max(tfd)) ** 2
            p = DS._scatim_plan(T.shape[2:], tfd, ttd, teta, 64)
            tm = (p["rows"][1] - p["rows"][0]) * (p["cols"][1] - p["cols"][0]) * 64
            batch = lambda: DS.scattered_image_batch(T, tfd, ttd, teta)  # noqa: E731
            st = stage_times(batch)
            sc = scipy_time(T[0, 0], tfd, ttd, teta)
            case = {"tiles": list(T.shape), "crop_elems": tm, "stages_ms": st,
                    "GBps": {k: BYTES[k] * tm / (st[k] * 1e-3) / 1e9 for k in BYTES if st[k]},
                    "device_ms": sum(st.values()), "call_s": host_time(batch),
                    "scipy": dict(sc, fit_s_x64=64 * sc["fit_s"], ev_s_x64=64 * sc["ev_s"])}
            res["cases"]["cut_dyn_64"] = case
            print(json.dumps({"cut_dyn_64": case}), flush=True)
    res["card_after"] = card()
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "probe_scattered_image.json")
