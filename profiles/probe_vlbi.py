"""Multi-station retrieval (ththmod.VLBI_chunk_retrieval): device time of one chunk
(CUDA events around the conjugate spectra and sb_vlbi_retrieval, after warm-up), the
call end to end, and one CPU core running the numpy oracle (oracle/vlbi_oracle.py),
on two workloads:
  a     3 stations, 64 x 128 chunk, CS 256 x 512 (tests/golden/vlbi_sample_a.npz);
  large 3 stations, 128 x 256 synthetic chunk, npad = 1, CS 256 x 512 with 199 theta
        centres (the large case of tests/test_gpu_vlbi.py).
Prints the card's name and power limit and one JSON line."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from threadpoolctl import threadpool_limits  # noqa: E402

from oracle import vlbi_oracle as VO  # noqa: E402
from scintools_b200 import _device as D, ththmod as thth  # noqa: E402
from test_gpu_vlbi import synthetic_stations  # noqa: E402


def case_a():
    f = np.load(os.path.join(ROOT, "tests", "golden", "vlbi_sample_a.npz"))
    autos = set(VO.auto_indices(3))
    dl = [f["dspec"][k].real if k in autos else f["dspec"][k] for k in range(6)]
    return dl, f["edges"], f["time"], f["freq"], float(f["eta"]), int(f["npad"])


def case_large():
    dl, t, f, eta, edges = synthetic_stations(3, 128, 256, 11)
    return dl, edges, t, f, eta, 1


def measure(name, dl, edges, t, f, eta, npad, reps=5):
    run = lambda: thth._vlbi_run(dl, edges, t, f, eta, npad, 3, 0.0)   # noqa: E731
    run()
    run()
    torch.cuda.synchronize()
    # device time: from before the first conjugate spectrum to after the retrieval call
    ev = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        cs_orig, cc_orig = thth._lib.lib.sb_cs_f32, thth._lib.lib.sb_cs_c2c_f32
        v_orig = thth._lib.lib.sb_vlbi_retrieval
        first = [True]

        def start(o):
            def call(*args):
                if first[0]:
                    a.record()
                    first[0] = False
                return o(*args)
            return call

        def stop(*args):
            rc = v_orig(*args)
            b.record()
            return rc
        thth._lib.lib.sb_cs_f32 = start(cs_orig)
        thth._lib.lib.sb_cs_c2c_f32 = start(cc_orig)
        thth._lib.lib.sb_vlbi_retrieval = stop
        try:
            run()
        finally:
            thth._lib.lib.sb_cs_f32, thth._lib.lib.sb_cs_c2c_f32 = cs_orig, cc_orig
            thth._lib.lib.sb_vlbi_retrieval = v_orig
        ev.append((a, b))
    torch.cuda.synchronize()
    dev_ms = sorted(a.elapsed_time(b) for a, b in ev)
    t0 = time.perf_counter()
    for _ in range(reps):
        thth.VLBI_chunk_retrieval((dl, edges, t, f, eta, 0, 0, npad, 3, 0.0, False))
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / reps
    with threadpool_limits(limits=1):
        t0 = time.perf_counter()
        VO.VLBI_chunk_retrieval(dl, edges, t, f, eta, npad, 3)
        cpu = (time.perf_counter() - t0) * 1e3
    return {"case": name, "chunk": list(np.shape(dl[0])), "npad": npad,
            "n_th": int(len(edges) - 1), "device_ms_min": dev_ms[0],
            "device_ms_median": dev_ms[len(dev_ms) // 2], "call_wall_ms": wall,
            "oracle_1core_ms": cpu}


def main():
    D.device()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("gpu:", q, flush=True)
    out = {"gpu": q, "results": [measure("a", *case_a()), measure("large", *case_large())]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
