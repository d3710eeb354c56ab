"""Device time of the flux-variation correction (Dynspec.correct_dyn): the top-k solver
(sb_svd_topk), its A^T A passes, the final pass (sb_svd_apply), the bandpass passes
(svd=False) and the end-to-end call from a host array, with the card read in the same run.

    python profiles/probe_correct_dyn.py

Sizes 4096 x 8192 and 8192 x 16384, a seeded dyn with band and gain structure (scintles
times a bandpass and a gain curve), nmodes 1 and 3.  One warm-up call per shape, then the
minimum over 5 timed calls.  Bytes per Lanczos step: the matrix once, plus the float64
column partials written and read back (G x nt x 8 twice; G = one CTA per SM at these row
widths, the register / shared-memory limit of svd_gram_kernel).  The re-orthogonalisation
reads the Lanczos vectors (L2-resident at these sizes) and is not counted.  Peak: the H100
SXM data sheet's 3.35 TB/s."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_GBS = 3350.0


def card():
    """Name, power limit and SM clocks of GPU 0, read in the same run (read-only query)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def structured_dyn(nf, nt, seed=0):
    rng = np.random.default_rng(seed)
    f = np.linspace(0, 1, nf, dtype=np.float32)
    t = np.linspace(0, 1, nt, dtype=np.float32)
    band = 1.0 + 0.6 * np.sin(2 * np.pi * 1.3 * f) ** 2 + 0.3 * f
    gain = 0.7 + 0.3 * np.cos(2 * np.pi * 0.8 * t) + 0.1 * t
    dyn = rng.standard_exponential((nf, nt), dtype=np.float32)
    dyn *= band[:, None]
    dyn *= gain[None, :]
    return dyn


def main():
    import torch
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _device as D, _lib
    from scintools_b200.dynspec import BasicDyn, Dynspec
    lib = _lib.lib
    print("card: %s" % card(), flush=True)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    st = D.stream_ptr

    def events():
        return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    for nf, nt in ((4096, 8192), (8192, 16384)):
        torch.cuda.empty_cache()
        host = structured_dyn(nf, nt)
        d = D.upload(host)
        step_bytes = nf * nt * 4 + 2 * sms * nt * 8
        for k in (1, 3):
            V = D.empty((k, nt), torch.float64)
            out = D.empty((nf, nt), torch.float32)
            model = D.empty((nf, nt), torch.float32)
            s, res, gap, info = np.zeros(k), np.zeros(k), np.zeros(1), np.zeros(4, np.int32)
            best = None
            for it in range(6):
                torch.cuda.synchronize()
                lib.sb_profile_enable(1)
                a, b = events()
                a.record()
                _lib.check(lib.sb_svd_topk(d.data_ptr(), nf, nt, k, V.data_ptr(), s.ctypes.data,
                                           res.ctypes.data, gap.ctypes.data, info.ctypes.data,
                                           st()))
                b.record()
                c, e = events()
                c.record()
                _lib.check(lib.sb_svd_apply(d.data_ptr(), nf, nt, k, V.data_ptr(),
                                            out.data_ptr(), model.data_ptr(), st()))
                e.record()
                torch.cuda.synchronize()
                ms = np.zeros(16)
                cnt = np.zeros(16, np.int32)
                lib.sb_profile_collect(ms.ctypes.data, cnt.ctypes.data, 16)
                lib.sb_profile_enable(0)
                row = (a.elapsed_time(b), c.elapsed_time(e), ms[12] / max(cnt[12], 1),
                       int(cnt[12]))
                if it and (best is None or row[0] < best[0]):
                    best = row
            solve, apply_ms, per_pass, npass = best
            steps = int(info[0])
            print("%d x %d nmodes %d: solver %.3f ms, %d Lanczos steps + %d residual passes, "
                  "A^T A pass %.1f us = %.0f GB/s (%.0f %% of 3.35 TB/s, %.1f MB moved), final "
                  "pass %.3f ms = %.0f GB/s (A read, out and model written), converged %d, "
                  "s = %s" % (nf, nt, k, solve, steps, npass - steps, per_pass * 1e3,
                              step_bytes / per_pass / 1e6, 100 * step_bytes / per_pass / 1e6 /
                              PEAK_GBS, step_bytes / 1e6, apply_ms,
                              3 * nf * nt * 4 / apply_ms / 1e6, info[1],
                              np.array2string(s, precision=6)), flush=True)
            # end to end from a host float64 array, PCIe copies included
            best = None
            for it in range(4):
                ds = Dynspec(dyn=BasicDyn(host.astype(np.float64), times=np.arange(nt) * 8.0,
                                          freqs=1400 + 0.01 * np.arange(nf), dt=8.0, df=0.01),
                             verbose=False)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ds.correct_dyn(nmodes=k)
                torch.cuda.synchronize()
                dt = (time.perf_counter() - t0) * 1e3
                if it and (best is None or dt < best):
                    best = dt
            print("%d x %d nmodes %d: Dynspec.correct_dyn end to end (float64 in and out, "
                  "PCIe copies, NaN pass on the host) %.1f ms" % (nf, nt, k, best), flush=True)
            del V, out, model
        # svd=False: the three passes on the device
        mr, mc = D.empty((nf,), torch.float64), D.empty((nt,), torch.float64)
        rowdiv = D.upload(1.0 + np.random.default_rng(1).random(nf))
        coldiv = D.upload(1.0 + np.random.default_rng(2).random(nt))
        out = D.empty((nf, nt), torch.float32)
        best = None
        for it in range(6):
            torch.cuda.synchronize()
            ev = [events() for _ in range(3)]
            ev[0][0].record()
            _lib.check(lib.sb_bandpass_rows(d.data_ptr(), nf, nt, 1, mr.data_ptr(), st()))
            ev[0][1].record()
            ev[1][0].record()
            _lib.check(lib.sb_bandpass_cols(d.data_ptr(), nf, nt, 1, rowdiv.data_ptr(),
                                            mc.data_ptr(), st()))
            ev[1][1].record()
            ev[2][0].record()
            _lib.check(lib.sb_bandpass_divide(d.data_ptr(), nf, nt, 1, rowdiv.data_ptr(),
                                              coldiv.data_ptr(), out.data_ptr(), st()))
            ev[2][1].record()
            torch.cuda.synchronize()
            row = [x.elapsed_time(y) for x, y in ev]
            if it and (best is None or sum(row) < sum(best)):
                best = row
        mb = nf * nt * 4 / 1e6
        print("%d x %d svd=False: rows %.3f ms (%.0f GB/s), cols %.3f ms (%.0f GB/s), divide "
              "%.3f ms (%.0f GB/s)" % (nf, nt, best[0], mb / best[0], best[1], mb / best[1],
                                       best[2], 2 * mb / best[2]), flush=True)
        best = None
        for it in range(4):
            ds = Dynspec(dyn=BasicDyn(host.astype(np.float64), times=np.arange(nt) * 8.0,
                                      freqs=1400 + 0.01 * np.arange(nf), dt=8.0, df=0.01),
                         verbose=False)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ds.correct_dyn(svd=False, nsmooth=7)
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) * 1e3
            if it and (best is None or dt < best):
                best = dt
        print("%d x %d svd=False nsmooth=7: Dynspec.correct_dyn end to end %.1f ms"
              % (nf, nt, best), flush=True)
        del d, out, host


if __name__ == "__main__":
    main()
