"""SASS opcode histogram per kernel of the built library (no GPU needed):
  python profiles/sass_histogram.py [TMA_LIST] > histogram.txt
With TMA_LIST, also writes to that file every kernel that contains TMA instructions
(UTMALDG = cp.async.bulk.tensor, UBLKCP = cp.async.bulk), LDGSTS (cp.async), mbarrier
operations (SYNCS) or tensor-core instructions (LDSM = ldmatrix, HMMA = mma.sync), with the
counts."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "scintools_b200", "lib", "libscint_b200.so")


def main():
    txt = subprocess.run(["cuobjdump", "-sass", LIB], check=True, capture_output=True, text=True).stdout
    kernels = collections.OrderedDict()
    cur = None
    for line in txt.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = collections.Counter()
            continue
        m = re.search(r"/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_]+)", line)
        if m and cur:
            kernels[cur][m.group(1)] += 1
    def demangle(n):
        try:
            return subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()[:150]
        except Exception:
            return n
    special = ("UTMALDG", "UTMASTG", "UBLKCP", "LDGSTS", "LDSM", "HMMA", "SYNCS")
    tma_lines = []
    print("# %d kernels in %s" % (len(kernels), os.path.relpath(LIB, ROOT)))
    for name, c in kernels.items():
        tot = sum(c.values())
        d = demangle(name)
        print("\n%s\n  total %d: %s" % (d, tot, ", ".join("%s %d" % kv for kv in c.most_common(14))))
        hit = {k: c[k] for k in special if c.get(k)}
        if hit:
            tma_lines.append("%s\n    %s" % (d, ", ".join("%s %d" % kv for kv in hit.items())))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            fh.write("# kernels of libscint_b200.so with TMA / cp.async / mbarrier / tensor-core instructions\n"
                     "# (cuobjdump -sass; UTMALDG = cp.async.bulk.tensor, UBLKCP = cp.async.bulk, LDSM = ldmatrix, HMMA = mma.sync,\n"
                     "#  LDGSTS = cp.async, SYNCS = mbarrier)\n\n")
            fh.write("\n".join(tma_lines) + "\n")


if __name__ == "__main__":
    main()
