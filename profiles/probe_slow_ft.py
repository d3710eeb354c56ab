"""Device time per pass of the frequency-scaled Doppler transform (scint_utils.slow_FT,
sb_slow_ft_f32), with the card read in the same run.

    python profiles/probe_slow_ft.py

Shapes (ntime x nfreq) 1024 x 1024, 4096 x 4096, 32768 x 8192, and 4096 x 3000 for the
chirp-z delay rows.  Input: seeded normal noise, freqs 400-800 MHz.  One warm-up call per
shape, then 7 timed calls; minimum and median of each profiling slot (14 slow_ft_doppler,
15 slow_ft_delay) and of CUDA events around the whole call.

Bytes each pass must move, from the shapes (P = M x nfreq x 8, the work plane, M the
convolution length; X = ntime x nfreq x 8, the output):
  Doppler: kernel transform (pass A writes P, pass B reads and writes P) 3 P; forward
           (input ntime x nfreq x 4 read, P written; P read twice, P written) 4 P + in;
           inverse (P read, P written; P read, X written) 3 P + X.
  Delay:   power-of-two rows read and write X in place; chirp-z rows also write and read
           the ntime x MT x 8 row buffer.
Peak: the H100 SXM data sheet's 3.35 TB/s."""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_GBS = 3350.0
SHAPES = [(1024, 1024), (4096, 4096), (32768, 8192), (4096, 3000)]


def card():
    """Name, power limit and SM clocks of GPU 0, read in the same run (read-only query)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def pow2_at_least(v):
    p = 8
    while p < v:
        p *= 2
    return p


def pass_bytes(nt, nf):
    M = pow2_at_least(2 * nt - 1)
    P, X = M * nf * 8, nt * nf * 8
    doppler = 10 * P + nt * nf * 4 + X
    if nf >= 8 and nf & (nf - 1) == 0:
        delay = 2 * X
    else:
        delay = 2 * X + 2 * nt * pow2_at_least(2 * nf - 1) * 8
    return doppler, delay


def main():
    import torch
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _device as D, _lib
    lib = _lib.lib
    print("card: %s" % card(), flush=True)
    st = D.stream_ptr
    for nt, nf in SHAPES:
        rng = np.random.default_rng(0)
        x = D.upload(rng.standard_normal((nt, nf), dtype=np.float32))
        freqs = np.linspace(400.0, 800.0, nf)
        s = D.upload(freqs / freqs[nf // 2])
        out = D.empty((nt, nf, 2), torch.float32)
        rows = []
        for it in range(8):
            lib.sb_profile_enable(1)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            _lib.check(lib.sb_slow_ft_f32(x.data_ptr(), nt, nf, s.data_ptr(), out.data_ptr(), st()))
            b.record()
            torch.cuda.synchronize()
            ms = np.zeros(16)
            cnt = np.zeros(16, np.int32)
            _lib.check(lib.sb_profile_collect(ms.ctypes.data, cnt.ctypes.data, 16))
            lib.sb_profile_enable(0)
            if it:
                rows.append((a.elapsed_time(b), ms[14], ms[15]))
        r = np.array(rows)
        mn, md = r.min(axis=0), np.median(r, axis=0)
        bd, bl = pass_bytes(nt, nf)
        print("%d x %d: call min %.3f / median %.3f ms; doppler min %.3f / median %.3f ms, "
              "%.2f GB, %.0f GB/s (%.0f %% of 3.35 TB/s); delay min %.3f / median %.3f ms, "
              "%.2f GB, %.0f GB/s (%.0f %%)"
              % (nt, nf, mn[0], md[0], mn[1], md[1], bd / 1e9, bd / mn[1] / 1e6,
                 100 * bd / mn[1] / 1e6 / PEAK_GBS, mn[2], md[2], bl / 1e9, bl / mn[2] / 1e6,
                 100 * bl / mn[2] / 1e6 / PEAK_GBS), flush=True)
        del x, s, out
    _lib.check(lib.sb_release())


if __name__ == "__main__":
    main()
