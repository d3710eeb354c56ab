"""calc_sspec / calc_acf at BASELINE config 2 (4096x8192), a few calls each: run under
`ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum` for a
per-kernel launch list."""
import sys
import numpy as np
sys.path.insert(0, ".")
from scintools_b200 import BasicDyn, Dynspec
rng = np.random.default_rng(2)
dyn = rng.exponential(1.0, (4096, 8192)).astype(np.float32)
ds = Dynspec(dyn=BasicDyn(dyn, times=10.0 * np.arange(8192), freqs=1400 + 0.03125 * np.arange(4096),
                          dt=10.0, df=0.03125), verbose=False)
for _ in range(2):
    ds.calc_sspec(dtype=np.float32)
for _ in range(2):
    ds.calc_acf(dtype=np.float32)
