"""The FFT engine at every supported transform length against float64 numpy
DFTs, and every size limit of the entry points from both sides.

Every product output goes through one set of FFT templates chosen by length
(fft_core.cuh, fft_kernels.cuh, fft_generic.cuh, chirp.cuh):
  rows     one CTA per row in shared memory, N = 8 .. 16384 (SB_ROW_DISPATCH),
           r2c / c2r / c2c, fp32 and fp64;
  columns  R = 4 .. 65536 split by split_len into two tile passes R1 x R2 with
           tile lengths 2 .. 256 (SB_TILE_DISPATCH); the first pass of
           cols_forward and of the ACF fetches its tile by TMA when the live
           rows are whole R2 groups, by plain loads otherwise;
  chirp-z  every other size; its kernel table is made by a row transform for
           M <= 16384 and by a column pass above.
CASES puts each length on one axis next to a small one on the other, so every
case stays small.  test_case_table_coverage (no GPU) restates the dispatch and
fails if an edit to the shapes drops a template.

References are float64 numpy on the same float32-rounded inputs the device
receives.  Bounds, from the arithmetic:
  fp32 complex outputs   ||got - ref||_2 / ||ref||_2 <= 1e-6
  fp32 power outputs     <= 2e-6 (squaring doubles the relative field error)
  every fp32 output      max|got - ref| / max|ref| <= 1e-5
  unit impulses          |got - ref| <= 4e-6 max(1, |ref|) in every bin (~64 ulp)
  fp64 screen            normwise and max-norm <= 1e-12
  fp64 prewhite sspec    every bin within 1e-6 of its own value (the low delay
                         bins are where an fp32 transform loses ~1e-4)
  fp64 Gerchberg-Saxton  10 iterations within 1e-6 (fp32 iterations pass 1e-5
                         within three); fp32 iterations: one, every element held
                         to the fp32 transform bound divided by |w| (gs_check)
"""
import os
import subprocess
import sys
import zlib
from collections import namedtuple
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import dynspec_oracle as DO
from oracle import sim_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ROW_LENGTHS = [1 << p for p in range(3, 15)]     # SB_ROW_DISPATCH: 8 .. 16384
TILE_LENGTHS = [1 << p for p in range(1, 9)]     # SB_TILE_DISPATCH: 2 .. 256
COL_LENGTHS = [1 << p for p in range(2, 17)]     # four-step columns: 4 .. 65536

NORM_FP32 = 1e-6
NORM_FP32_POWER = 2e-6
MAX_FP32 = 1e-5
BIN_IMPULSE = 4e-6
NORM_FP64_SCREEN = 1e-12
BIN_PREWHITE = 1e-6
GS_FP64 = 1e-6

# worst error seen per (family, metric) in this process: (error, bound)
MEASURED = {}


# --------------------------------------------------------------------------
# the dispatch, restated
# --------------------------------------------------------------------------
def next_pow2(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def is_pow2(v):
    return v > 0 and v & (v - 1) == 0


def split_len(R):
    """split_len() of fft_kernels.cuh."""
    p = 0
    while (1 << p) < R:
        p += 1
    r1 = 1 << ((p + 1) // 2)
    return r1, R // r1


def col_load(live, R):
    """First column pass of cols_forward / acf: TMA when the live rows are whole R2 groups."""
    _, r2 = split_len(R)
    return "tma" if live % r2 == 0 and live >= r2 else "plain"


def cs_pow2(nf, nt, npad):
    """conj_spectrum(): the radix path, else chirp-z."""
    NF, NT = (npad + 1) * nf, (npad + 1) * nt
    return is_pow2(NF) and is_pow2(NT) and NT // 2 >= 8 and NF >= 4


def templates(case):
    """The FFT templates one case launches, read off the host drivers."""
    e, p = case.entry, case.p
    out = set()

    def cols(tag, prec, R, load):
        r1, r2 = split_len(R)
        out.update({("col", tag, prec, R, load), ("tile", prec, r1), ("tile", prec, r2)})

    def chirp(tag, n0, n1):       # conj_spectrum_bluestein / ifft2_c2c_any
        mt, mf = next_pow2(2 * n1 - 1), next_pow2(2 * n0 - 1)
        out.add(("row", tag, "c2c", "f32", mt))
        cols(tag, "f32", mf, "plain")
        for m in (mt, mf):        # bluestein_tables
            if m <= 16384:
                out.add(("chirp_table", tag, "row"))
            else:
                cols(tag + "_table", "f32", m, "plain")
                out.add(("chirp_table", tag, "col"))

    if e in ("sspec", "acf_sspec"):
        nf, nt = p["nf"], p["nt"]
        NF, NT = 2 * next_pow2(nf), 2 * next_pow2(nt)
        if p.get("prewhite"):
            out.add(("row", "sspec_prewhite", "r2c", "f64", NT // 2))
            cols("sspec_prewhite", "f64", NF, "plain")
        else:
            out.add(("row", "sspec", "r2c", "f32", NT // 2))
            cols("sspec", "f32", NF, col_load(nf, NF))
        if e == "acf_sspec":
            out.add(("row", "acf_sspec", "r2c", "f32", NT // 2))
            cols("acf_sspec", "f32", NF, col_load(NF, NF))
    elif e == "acf":
        PF, PT = next_pow2(2 * p["nf"]), next_pow2(2 * p["nt"])
        out.add(("row", "acf", "r2c", "f32", PT // 2))
        out.add(("row", "acf", "c2r", "f32", PT // 2))
        cols("acf", "f32", PF, col_load(p["nf"], PF))
    elif e == "cs":
        nf, nt, npad = p["nf"], p["nt"], p["npad"]
        if cs_pow2(nf, nt, npad):
            NF, NT = (npad + 1) * nf, (npad + 1) * nt
            out.add(("row", "cs", "r2c", "f32", NT // 2))
            cols("cs", "f32", NF, col_load(nf, NF))
        else:
            chirp("cs_chirp", (npad + 1) * nf, (npad + 1) * nt)
    elif e in ("ifft2", "gs"):
        n0, n1 = p["n0"], p["n1"]
        if is_pow2(n0) and is_pow2(n1):
            prec = "f64" if e == "gs" and n1 <= 8192 else "f32"
            out.add(("row", e, "c2c", prec, n1))
            cols(e, prec, n0, "plain")
        else:
            chirp(e + "_chirp", n0, n1)
    elif e == "screen":
        out.add(("row", "screen", "c2c", "f64", p["ny"]))
        cols("screen", "f64", p["nx"], "plain")
    elif e == "intensity":
        out.add(("row", "intensity_reduce", "c2c", "f32", p["ny"]))
        out.add(("row", "intensity", "c2c", "f32", p["nx"]))
        cols("intensity", "f32", p["nx"], "plain")
    else:
        raise ValueError(e)
    return out


def reachable_loads(entry, R):
    """Load paths an input shape can reach at column length R (NF = 2 np2(nf) for
    calc_sspec, PF = np2(2 nf) for calc_acf: nf in (R/4, R/2] either way)."""
    return {col_load(nf, R) for nf in range(R // 4 + 1, R // 2 + 1)}


def required_templates():
    req = set()
    for n in ROW_LENGTHS:
        for key in (("sspec", "r2c", "f32"), ("acf", "r2c", "f32"), ("acf", "c2r", "f32"),
                    ("acf_sspec", "r2c", "f32"), ("cs", "r2c", "f32"), ("cs_chirp", "c2c", "f32"),
                    ("ifft2", "c2c", "f32"), ("ifft2_chirp", "c2c", "f32"),
                    ("intensity_reduce", "c2c", "f32"), ("intensity", "c2c", "f32")):
            req.add(("row",) + key + (n,))
        if n <= 8192:             # fp64 rows of 16384 points do not fit shared memory
            for key in (("sspec_prewhite", "r2c", "f64"), ("gs", "c2c", "f64"),
                        ("screen", "c2c", "f64")):
                req.add(("row",) + key + (n,))
    req.add(("row", "gs", "c2c", "f32", 16384))
    for r in COL_LENGTHS:
        for tag in ("sspec", "acf"):
            req.update(("col", tag, "f32", r, load) for load in reachable_loads(tag, r))
        req.add(("col", "sspec_prewhite", "f64", r, "plain"))
        req.add(("col", "cs", "f32", r, "tma"))
        req.add(("col", "screen", "f64", r, "plain"))
        if r >= 8:                # chirp-z: M = np2(2 n - 1) >= 8
            req.add(("col", "cs_chirp", "f32", r, "plain"))
            req.add(("col", "ifft2_chirp", "f32", r, "plain"))
            req.add(("col", "ifft2", "f32", r, "plain"))
        if 8 <= r <= 16384:
            req.add(("col", "intensity", "f32", r, "plain"))
    for L in TILE_LENGTHS:
        req.update({("tile", "f32", L), ("tile", "f64", L)})
    for tag in ("cs_chirp", "ifft2_chirp", "gs_chirp"):
        req.update({("chirp_table", tag, "row"), ("chirp_table", tag, "col")})
    return req


def missing_coverage(cases):
    got = set()
    for c in cases:
        got |= templates(c)
    return sorted(required_templates() - got, key=str)


# --------------------------------------------------------------------------
# the case table
# --------------------------------------------------------------------------
Case = namedtuple("Case", "entry p")


def _c(entry, **p):
    return Case(entry, p)


def case_size(c):
    p = c.p
    return p.get("nf", 1) * p.get("nt", 1) * p.get("n0", 1) * p.get("n1", 1) * \
        p.get("nx", 1) * p.get("ny", 1)


def case_id(c):
    return c.entry + "-" + "-".join("%s%s" % (k, int(v) if isinstance(v, bool) else v)
                                    for k, v in sorted(c.p.items()))


PADS = (0.375, None, -1.25)      # constant pads (exact in fp32); None = the device mean


def _build_cases():
    C = []
    # calc_sspec, fp32: rows N = np2(nt), columns NF = 2 np2(nf)
    for i, n in enumerate(ROW_LENGTHS):
        C.append(_c("sspec", nf=3 + i % 2, nt=n if i % 2 else n - 3, window=i % 2 == 0,
                    halve=1, prewhite=0))
    for i, r in enumerate(COL_LENGTHS):
        C.append(_c("sspec", nf=r // 2, nt=6, window=i % 2 == 1, halve=i % 2, prewhite=0))
        if r >= 8:                # odd nf: the live rows are no whole R2 groups -> plain loads
            C.append(_c("sspec", nf=r // 2 - 1, nt=8, window=i % 2 == 0, halve=1 - i % 2,
                        prewhite=0))
    # calc_sspec(prewhite=True), fp64 rows (<= 8192) and tiles
    for i, n in enumerate(ROW_LENGTHS[:-1]):
        C.append(_c("sspec", nf=5, nt=n if i % 2 == 0 else n - 3, window=i % 2 == 0,
                    halve=1, prewhite=1))
    for i, r in enumerate(COL_LENGTHS):
        C.append(_c("sspec", nf=max(r // 2 - i % 2, 2), nt=7, window=i % 2 == 1, halve=1,
                    prewhite=1))
    # calc_acf(method='direct'): PT = np2(2 nt), PF = np2(2 nf)
    for i, n in enumerate(ROW_LENGTHS):
        C.append(_c("acf", nf=3, nt=n if i % 2 else n - 3, normalise=i % 2))
    for i, r in enumerate(COL_LENGTHS):
        C.append(_c("acf", nf=r // 2, nt=5 + i % 4, normalise=1 - i % 2))
        if r >= 8:
            C.append(_c("acf", nf=r // 2 - 1, nt=6, normalise=i % 2))
    # calc_acf(method='sspec')
    for i, n in enumerate(ROW_LENGTHS):
        C.append(_c("acf_sspec", nf=3, nt=n - i % 2, window=i % 2 == 0, normalise=1 - i % 2))
    for r in (4, 256, 65536):
        C.append(_c("acf_sspec", nf=r // 2, nt=6, window=True, normalise=1))
    # conjugate spectrum, power-of-two padding
    for i, n in enumerate(ROW_LENGTHS):
        npad = i % 2
        half = i % 4 >= 2
        C.append(_c("cs", nf=4 // (npad + 1), nt=2 * n // (npad + 1), npad=npad, pad=PADS[i % 3],
                    half=half, keep=3 if half and i % 3 == 0 else 0, mask=i % 3 == 1))
    for i, r in enumerate(COL_LENGTHS):
        npad = i % 2
        half = i % 4 < 2
        C.append(_c("cs", nf=r // (npad + 1), nt=16 // (npad + 1), npad=npad, pad=PADS[i % 3],
                    half=half, keep=5 if half and i % 3 == 0 else 0, mask=i % 3 == 2))
    # fewer live rows than R2: plain loads
    C.append(_c("cs", nf=16, nt=1, npad=63, pad=None, half=True, keep=5, mask=True))
    C.append(_c("cs", nf=32, nt=1, npad=127, pad=0.375, half=False, keep=0, mask=False))
    # conjugate spectrum, chirp-z: MT = np2(2 NT - 1), MF = np2(2 NF - 1)
    for i, m in enumerate(ROW_LENGTHS):
        C.append(_c("cs", nf=6, nt=m // 2 - 1 if m > 8 else 3, npad=0, pad=PADS[i % 3],
                    half=False, keep=0, mask=i % 2 == 1))
    for i, m in enumerate(COL_LENGTHS[1:]):      # M = 4 has no row transform for its table
        C.append(_c("cs", nf=m // 2 - 1, nt=5, npad=0, pad=PADS[i % 3],
                    half=False, keep=0, mask=i % 2 == 0))
    C += [_c("cs", nf=10007, nt=13, npad=0, pad=0.375, half=False, keep=0, mask=True),   # primes
          _c("cs", nf=5, nt=7, npad=2, pad=None, half=False, keep=0, mask=False),
          _c("cs", nf=4, nt=4, npad=0, pad=-1.25, half=False, keep=0, mask=False),      # NT/2 < 8
          _c("cs", nf=6, nt=8192, npad=0, pad=0.375, half=False, keep=0, mask=False),   # largest NT
          _c("cs", nf=32768, nt=5, npad=0, pad=-1.25, half=False, keep=0, mask=True)]   # largest NF
    # ifft2, powers of two
    for i, n in enumerate(ROW_LENGTHS):
        n0 = 8 << (i % 3)
        C.append(_c("ifft2", n0=n0, n1=n, centred=i % 2, crop0=0 if i % 3 else n0 // 2 + 1,
                    crop1=0 if i % 4 else n - 3, real=i % 4 == 3))
    for i, r in enumerate(COL_LENGTHS[1:]):
        n1 = 8 << (i % 2)
        C.append(_c("ifft2", n0=r, n1=n1, centred=(i + 1) % 2, crop0=0 if i % 4 else r // 2 + 1,
                    crop1=0 if i % 3 else n1 - 3, real=i % 3 == 2))
    # ifft2, chirp-z
    for i, m in enumerate(ROW_LENGTHS):
        C.append(_c("ifft2", n0=6, n1=m // 2 - 1 if m > 8 else 3, centred=i % 2, crop0=0,
                    crop1=0 if i % 3 else 2, real=i % 4 == 1))
    for i, m in enumerate(COL_LENGTHS[1:]):
        C.append(_c("ifft2", n0=m // 2 - 1, n1=5, centred=i % 2,
                    crop0=0 if i % 3 else 1, crop1=0, real=i % 4 == 2))
    C += [_c("ifft2", n0=6, n1=8192, centred=1, crop0=0, crop1=0, real=False),
          _c("ifft2", n0=32768, n1=5, centred=0, crop0=0, crop1=0, real=False),
          _c("ifft2", n0=256, n1=600, centred=1, crop0=64, crop1=150, real=False)]
    # Gerchberg-Saxton: fp64 iterations up to 8192 columns, fp32 at 16384, chirp-z otherwise
    for n in ROW_LENGTHS:
        C.append(_c("gs", n0=16 if n <= 4096 else 8, n1=n))
    C += [_c("gs", n0=65536, n1=8), _c("gs", n0=1024, n1=32),
          _c("gs", n0=12, n1=10), _c("gs", n0=48, n1=150), _c("gs", n0=9000, n1=6),
          _c("gs", n0=6, n1=8192), _c("gs", n0=32768, n1=5)]
    # Simulation screen (fp64) and intensity (fp32)
    for i, n in enumerate(ROW_LENGTHS[:-1]):
        C.append(_c("screen", nx=4 << (i % 3), ny=n))
    for r in COL_LENGTHS[1:]:     # nx = 4: the first row case
        C.append(_c("screen", nx=r, ny=8))
    for i, n in enumerate(ROW_LENGTHS):
        C.append(_c("intensity", nx=8 << (i % 2), ny=n, nf=2))
        C.append(_c("intensity", nx=n, ny=16 >> (i % 2), nf=2))
    return C


CASES = _build_cases()

# (what, rejected call, words of the message, the largest accepted case)
LIMITS = [
    ("sspec nt", _c("sspec", nf=2, nt=16385, window=False, halve=1, prewhite=0), "nt 5..16384",
     _c("sspec", nf=4, nt=16384, window=False, halve=1, prewhite=0)),
    ("sspec nf", _c("sspec", nf=32769, nt=5, window=False, halve=1, prewhite=0), "nf 2..32768",
     _c("sspec", nf=32768, nt=6, window=False, halve=0, prewhite=0)),
    ("sspec prewhite nt", _c("sspec", nf=3, nt=8193, window=False, halve=1, prewhite=1),
     "nt <= 8192", _c("sspec", nf=5, nt=8192, window=True, halve=1, prewhite=1)),
    ("acf nt", _c("acf", nf=3, nt=16385, normalise=1), "nt 5..16384",
     _c("acf", nf=3, nt=16384, normalise=1)),
    ("acf nf", _c("acf", nf=32769, nt=5, normalise=1), "nf 2..32768",
     _c("acf", nf=32768, nt=7, normalise=1)),
    ("cs cols", _c("cs", nf=4, nt=65536, npad=0, pad=0.375, half=False, keep=0, mask=False),
     "cols <= 32768", _c("cs", nf=2, nt=16384, npad=1, pad=-1.25, half=True, keep=0, mask=False)),
    ("cs rows", _c("cs", nf=131072, nt=16, npad=0, pad=0.375, half=False, keep=0, mask=False),
     "rows <= 65536", _c("cs", nf=65536, nt=16, npad=0, pad=-1.25, half=False, keep=0,
                         mask=True)),
    ("cs chirp cols", _c("cs", nf=3, nt=8193, npad=0, pad=0.375, half=False, keep=0, mask=False),
     "cols 3..8192", _c("cs", nf=6, nt=8192, npad=0, pad=0.375, half=False, keep=0, mask=False)),
    ("cs chirp rows", _c("cs", nf=32769, nt=5, npad=0, pad=0.375, half=False, keep=0, mask=False),
     "rows 3..32768", _c("cs", nf=32768, nt=5, npad=0, pad=-1.25, half=False, keep=0, mask=True)),
    ("cs chirp rows, low", _c("cs", nf=2, nt=5, npad=0, pad=0.375, half=False, keep=0,
                              mask=False),
     "rows 3..32768", _c("cs", nf=3, nt=5, npad=0, pad=0.375, half=False, keep=0, mask=True)),
    ("ifft2 n1", _c("ifft2", n0=8, n1=32768, centred=0, crop0=0, crop1=0, real=False),
     "8..65536 x 8..16384", _c("ifft2", n0=32, n1=16384, centred=1, crop0=0, crop1=0,
                               real=True)),
    ("ifft2 n0", _c("ifft2", n0=131072, n1=8, centred=0, crop0=0, crop1=0, real=False),
     "8..65536 x 8..16384", _c("ifft2", n0=65536, n1=16, centred=0, crop0=0, crop1=0,
                               real=False)),
    ("ifft2 chirp n1", _c("ifft2", n0=6, n1=8193, centred=0, crop0=0, crop1=0, real=False),
     "3..32768 x 3..8192", _c("ifft2", n0=6, n1=8192, centred=1, crop0=0, crop1=0, real=False)),
    ("ifft2 chirp n0", _c("ifft2", n0=32769, n1=5, centred=0, crop0=0, crop1=0, real=False),
     "3..32768 x 3..8192", _c("ifft2", n0=32768, n1=5, centred=0, crop0=0, crop1=0,
                              real=False)),
    ("ifft2 chirp n0, low", _c("ifft2", n0=2, n1=5, centred=0, crop0=0, crop1=0, real=False),
     "3..32768 x 3..8192", _c("ifft2", n0=3, n1=5, centred=0, crop0=1, crop1=0, real=False)),
    ("gs n1", _c("gs", n0=8, n1=32768), "8..65536 x 8..16384", _c("gs", n0=8, n1=16384)),
    ("gs n0", _c("gs", n0=131072, n1=8), "8..65536 x 8..16384", _c("gs", n0=65536, n1=8)),
    ("gs chirp n1", _c("gs", n0=6, n1=8193), "3..32768 x 3..8192", _c("gs", n0=6, n1=8192)),
    ("gs chirp n0", _c("gs", n0=32769, n1=5), "3..32768 x 3..8192", _c("gs", n0=32768, n1=5)),
    ("screen ny", _c("screen", nx=4, ny=16384), "nx 4..65536, ny 8..8192",
     _c("screen", nx=8, ny=8192)),
    ("screen nx", _c("screen", nx=131072, ny=8), "nx 4..65536, ny 8..8192",
     _c("screen", nx=65536, ny=8)),
    ("intensity nx", _c("intensity", nx=32768, ny=8, nf=2), "8..16384",
     _c("intensity", nx=16384, ny=8, nf=2)),
    ("intensity ny", _c("intensity", nx=8, ny=32768, nf=2), "8..16384",
     _c("intensity", nx=16, ny=16384, nf=2)),
]


# --------------------------------------------------------------------------
# checks
# --------------------------------------------------------------------------
def _record(family, metric, err, bound):
    key = (family, metric)
    if key not in MEASURED or err > MEASURED[key][0]:
        MEASURED[key] = (float(err), bound)


def check_norms(family, got, ref, norm_bound, max_bound=MAX_FP32):
    got = np.asarray(got)
    ref = np.asarray(ref)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert np.isfinite(got).all(), "%s: non-finite output" % family
    d = got.astype(np.complex128) - ref
    en = float(np.linalg.norm(d) / np.linalg.norm(ref))
    em = float(np.abs(d).max() / np.abs(ref).max())
    _record(family, "normwise", en, norm_bound)
    _record(family, "max-norm", em, max_bound)
    assert en <= norm_bound, "%s: normwise error %.3g > %.3g" % (family, en, norm_bound)
    assert em <= max_bound, "%s: max-norm error %.3g > %.3g at %s" % (
        family, em, max_bound, np.unravel_index(np.abs(d).argmax(), d.shape))


def check_bins(family, got, ref, bound, floor=1.0):
    """Every bin on its own: |got - ref| <= bound * max(floor, |ref|)."""
    got = np.asarray(got)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert np.isfinite(got).all(), "%s: non-finite output" % family
    e = np.abs(got.astype(np.complex128) - ref) / np.maximum(floor, np.abs(ref))
    worst = float(e.max())
    _record(family, "per-bin", worst, bound)
    assert worst <= bound, "%s: bin %s off by %.3g (bound %.3g)" % (
        family, np.unravel_index(e.argmax(), e.shape), worst, bound)


def to_complex(a):
    return a[..., 0].astype(np.float64) + 1j * a[..., 1].astype(np.float64)


def phase_ramp(shape, pos, sign):
    """exp(sign 2 pi i (k r / n0 + l c / n1)): the DFT of a unit impulse at pos, with
    the phase reduced exactly in integers."""
    n0, n1 = shape
    k = (np.arange(n0)[:, None] * pos[0]) % n0
    l_ = (np.arange(n1)[None, :] * pos[1]) % n1
    return np.exp(sign * 2j * np.pi * (k / n0 + l_ / n1))


def _rng(case):
    return np.random.default_rng(zlib.crc32(case_id(case).encode()))


def _dev():
    from scintools_b200 import _device as D, _lib
    D.device()
    return D, _lib


# --------------------------------------------------------------------------
# entry points: inputs, device call, reference check
# --------------------------------------------------------------------------
def sspec_power(dyn, wt, wf, prewhite, halve, shift=True):
    """Linear-power calc_sspec (dynspec.py:3664-3721) in float64 from the float32
    inputs and windows the device receives."""
    nf, nt = dyn.shape
    NF, NT = DO.fft_lengths(nf, nt)
    x = dyn.astype(np.float64)
    x = x - x.mean()
    if wt is not None:
        x = x * wt.astype(np.float64)[None, :] * wf.astype(np.float64)[:, None]
    x = x - x.mean()
    if prewhite:
        x = x[1:, 1:] - x[1:, :-1] - x[:-1, 1:] + x[:-1, :-1]
    F = np.fft.fft2(x, s=[NF, NT])
    P = F.real ** 2 + F.imag ** 2
    if not shift:
        return P
    P = np.fft.fftshift(P)
    if halve:
        P = P[NF // 2:]
    if prewhite:
        v1 = np.sin(np.pi / NT * np.arange(-NT // 2, NT // 2)) ** 2
        v2 = np.sin(np.pi / NF * np.arange(NF // 2)) ** 2
        pd = np.outer(v2, v1)
        pd[:, NT // 2] = 1
        pd[0, :] = 1
        P = P / pd
    return P


def _dyn_inputs(case, window):
    rng = _rng(case)
    nf, nt = case.p["nf"], case.p["nt"]
    x = {"dyn": rng.exponential(1.0, (nf, nt)).astype(np.float32), "wt": None, "wf": None}
    if window:
        wt, wf = DO.get_window(nt, nf, "hanning", 0.3)
        x["wt"], x["wf"] = wt.astype(np.float32), wf.astype(np.float32)
    return x


def _windows(D, x):
    if x["wt"] is None:
        return None, None, 0.0, 0.0
    return (D.upload(x["wt"]), D.upload(x["wf"]), float(x["wt"].sum(dtype=np.float64)),
            float(x["wf"].sum(dtype=np.float64)))


def sspec_inputs(case):
    return _dyn_inputs(case, case.p["window"])


def sspec_device(case, x):
    import torch
    D, L = _dev()
    p = case.p
    nf, nt = x["dyn"].shape
    NF, NT = DO.fft_lengths(nf, nt)
    wt, wf, swt, swf = _windows(D, x)
    pd1 = pd2 = None
    if p["prewhite"]:             # required by the ABI; the fp64 path makes its own
        pd1, pd2 = D.upload(np.ones(NT, np.float32)), D.upload(np.ones(NF // 2, np.float32))
    out = D.empty((NF // 2 if p["halve"] else NF, NT), torch.float32)
    L.check(L.lib.sb_sspec_f32(D.upload(x["dyn"]).data_ptr(), nf, nt, D.ptr(wt), D.ptr(wf),
                               swt, swf, p["prewhite"], p["halve"], 0, D.ptr(pd1), D.ptr(pd2),
                               out.data_ptr(), D.stream_ptr()))
    return out.cpu().numpy()


def sspec_check(case, x, got):
    p = case.p
    ref = sspec_power(x["dyn"], x["wt"], x["wf"], p["prewhite"], p["halve"])
    if p["prewhite"]:
        # the Hann taper ends at zero, which makes the fd = 0 column (and the tau = 0 row)
        # of the differenced spectrum zero in exact arithmetic: those bins are held to
        # 1e-6 of a floor of 1e-12 of the mean power before post-darkening
        floor = 1e-12 * sspec_power(x["dyn"], x["wt"], x["wf"], True, True, shift=False).mean()
        check_bins("sspec prewhite (fp64)", got, ref, BIN_PREWHITE, floor=floor)
    else:
        check_norms("sspec", got, ref, NORM_FP32_POWER)


def acf_inputs(case):
    return _dyn_inputs(case, False)


def acf_device(case, x):
    import torch
    D, L = _dev()
    nf, nt = x["dyn"].shape
    out = D.empty((2 * nf, 2 * nt), torch.float32)
    L.check(L.lib.sb_acf_f32(D.upload(x["dyn"]).data_ptr(), nf, nt, 1, case.p["normalise"],
                             out.data_ptr(), D.stream_ptr()))
    return out.cpu().numpy()


def acf_check(case, x, got):
    ref = DO.calc_acf(x["dyn"].astype(np.float64), normalise=bool(case.p["normalise"]))
    check_norms("acf", got, ref, NORM_FP32_POWER)


def acf_sspec_inputs(case):
    return _dyn_inputs(case, case.p["window"])


def acf_sspec_device(case, x):
    import torch
    D, L = _dev()
    nf, nt = x["dyn"].shape
    NF, NT = DO.fft_lengths(nf, nt)
    wt, wf, swt, swf = _windows(D, x)
    out = D.empty((NF, NT), torch.float32)
    L.check(L.lib.sb_acf_sspec_f32(D.upload(x["dyn"]).data_ptr(), nf, nt, D.ptr(wt), D.ptr(wf),
                                   swt, swf, case.p["normalise"], out.data_ptr(),
                                   D.stream_ptr()))
    return out.cpu().numpy()


def acf_sspec_check(case, x, got):
    # dynspec.py:3798-3807: real(fftshift(fft2(linear, un-shifted secondary spectrum)))
    P = sspec_power(x["dyn"], x["wt"], x["wf"], False, False, shift=False)
    ref = np.real(np.fft.fftshift(np.fft.fft2(P)))
    if case.p["normalise"]:
        ref = ref / ref.max()
    check_norms("acf_sspec", got, ref, NORM_FP32_POWER)


def cs_inputs(case):
    rng = _rng(case)
    p = case.p
    NF = (p["npad"] + 1) * p["nf"]
    x = {"dspec": rng.normal(0.3, 1.0, (p["nf"], p["nt"])).astype(np.float32),
         "mask": (rng.random(NF) < 0.25).astype(np.uint8) if p["mask"] else None}
    return x


def cs_device(case, x, dspec=None):
    import torch
    D, L = _dev()
    p = case.p
    dspec = x["dspec"] if dspec is None else dspec
    nf, nt, npad = p["nf"], p["nt"], p["npad"]
    NF, NT = (npad + 1) * nf, (npad + 1) * nt
    pitch = NT // 2 + 4 if p["half"] else NT
    out = D.zeros((NF, pitch, 2), torch.float32)
    mask = D.upload(x["mask"]) if x["mask"] is not None else None
    pad = np.float32(np.nan if p["pad"] is None else p["pad"])
    L.check(L.lib.sb_cs_f32(D.upload(dspec).data_ptr(), nf, nt, npad, float(pad), D.ptr(mask),
                            int(p["half"]), pitch, p["keep"], out.data_ptr(), D.stream_ptr()))
    return to_complex(out.cpu().numpy())


def cs_layout(case, x, CS):
    """CS: unshifted fft2 of the padded chunk -> the layout sb_cs_f32 writes."""
    p = case.p
    CS = np.fft.fftshift(CS)
    if x["mask"] is not None:
        CS[x["mask"].astype(bool)] = 0
    if p["half"]:
        NT = (p["npad"] + 1) * p["nt"]
        CS = np.fft.ifftshift(CS, axes=1)[:, :p["keep"] or NT // 2 + 1]
    return CS


def cs_crop(case, got):
    p = case.p
    if p["half"]:
        NT = (p["npad"] + 1) * p["nt"]
        return got[:, :p["keep"] or NT // 2 + 1]
    return got


def cs_check(case, x, got):
    p = case.p
    npad = p["npad"]
    family = "cs" if cs_pow2(p["nf"], p["nt"], npad) else "cs chirp-z"
    d = x["dspec"].astype(np.float64)
    pad = d.mean() if p["pad"] is None else p["pad"]   # ththmod.py:781 / dynspec.py:1575
    padded = np.pad(d, ((0, npad * d.shape[0]), (0, npad * d.shape[1])), mode="constant",
                    constant_values=pad)
    check_norms(family, cs_crop(case, got), cs_layout(case, x, np.fft.fft2(padded)), NORM_FP32)
    if p["pad"] is None:
        return
    # dyn = p + unit impulse, padded with p: a phase ramp plus p NF NT at DC
    NF, NT = (npad + 1) * p["nf"], (npad + 1) * p["nt"]
    for pos in ((p["nf"] - 1, p["nt"] - 1), (0, 0)):
        imp = np.full(d.shape, p["pad"], np.float32)
        imp[pos] += 1
        ref = phase_ramp((NF, NT), pos, -1)
        ref[0, 0] += p["pad"] * NF * NT
        got_i = cs_crop(case, cs_device(case, x, imp))
        check_bins(family + " impulse", got_i, cs_layout(case, x, ref), BIN_IMPULSE)


def ifft2_inputs(case):
    rng = _rng(case)
    n0, n1 = case.p["n0"], case.p["n1"]
    return {"X": (rng.normal(size=(n0, n1)) + 1j * rng.normal(size=(n0, n1))).astype(np.complex64)}


def _crops(p):
    return p["crop0"] or p["n0"], p["crop1"] or p["n1"]


def ifft2_device(case, x, X=None, scale=3.0):
    import torch
    D, L = _dev()
    p = case.p
    X = x["X"] if X is None else X
    c0, c1 = _crops(p)
    out = D.empty((c0, c1) if p["real"] else (c0, c1, 2), torch.float32)
    L.check(L.lib.sb_ifft2_c2c_f32(D.upload(X).data_ptr(), p["n0"], p["n1"], p["centred"],
                                   p["crop0"], p["crop1"], scale, int(p["real"]), out.data_ptr(),
                                   D.stream_ptr()))
    a = out.cpu().numpy()
    return a.astype(np.float64) if p["real"] else to_complex(a)


def ifft2_check(case, x, got):
    p = case.p
    n0, n1 = p["n0"], p["n1"]
    family = "ifft2" if is_pow2(n0) and is_pow2(n1) else "ifft2 chirp-z"
    c0, c1 = _crops(p)
    X = x["X"].astype(np.complex128)
    ref = 3.0 * np.fft.ifft2(np.fft.ifftshift(X) if p["centred"] else X)[:c0, :c1]
    check_norms(family, got, ref.real if p["real"] else ref, NORM_FP32)
    # unit impulse, scaled by n0 n1: a unit phase ramp
    for pos in ((n0 - 1, n1 - 1), (0, 0)):
        imp = np.zeros((n0, n1), np.complex64)
        imp[pos] = 1
        src = ((pos[0] - n0 // 2) % n0, (pos[1] - n1 // 2) % n1) if p["centred"] else pos
        ref = phase_ramp((n0, n1), src, +1)[:c0, :c1]
        got_i = ifft2_device(case, x, imp, float(n0 * n1))
        check_bins(family + " impulse", got_i, ref.real if p["real"] else ref, BIN_IMPULSE)


def gs_fp64(p):
    return is_pow2(p["n0"]) and is_pow2(p["n1"]) and p["n1"] <= 8192


def gs_inputs(case):
    rng = _rng(case)
    n0, n1 = case.p["n0"], case.p["n1"]
    W = (rng.normal(size=(n0, n1)) + 1j * rng.normal(size=(n0, n1))).astype(np.complex64)
    amp = np.sqrt(rng.exponential(1.0, (n0, n1))).astype(np.float32)
    amp[rng.random((n0, n1)) < 0.05] = np.nan
    rowmask = (np.fft.fftfreq(n0) < 0).astype(np.uint8)     # tau < 0, unshifted rows
    return {"W": W, "amp": amp, "rowmask": rowmask,
            "niter": 10 if gs_fp64(case.p) else 1}


def gs_device(case, x, niter=None):
    D, L = _dev()
    p = case.p
    # the device copies stay referenced until the call returns: a temporary freed while
    # its data pointer is in flight would be handed to the next upload
    w, amp, rowmask = D.upload(x["W"]), D.upload(x["amp"]), D.upload(x["rowmask"])
    L.check(L.lib.sb_gerchberg_saxton_f32(w.data_ptr(), amp.data_ptr(),
                                          rowmask.data_ptr(), p["n0"], p["n1"],
                                          x["niter"] if niter is None else niter,
                                          D.stream_ptr()))
    return to_complex(w.cpu().numpy())


def gs_loop(W, amp, rowmask, niter):
    """The loop of TO.gerchberg_saxton (dynspec.py:1883-1896) on the wavefield and
    amplitude passed to the call; fftshift / ifftshift cancel, so the mask is
    applied to the unshifted rows.  Returns the wavefield and, of the last
    iteration, the wavefield before the amplitude step."""
    W = W.astype(np.complex128)
    amp = amp.astype(np.float64)
    known = ~np.isnan(amp)
    pre = W
    for _ in range(niter):
        C = np.fft.fft2(W)
        C[rowmask.astype(bool)] = 0
        pre = np.fft.ifft2(C)
        W = pre.copy()
        W[known] = amp[known] * np.exp(1j * np.angle(W[known]))
    return W, pre


def gs_check(case, x, got):
    p = case.p
    ref, pre = gs_loop(x["W"], x["amp"], x["rowmask"], x["niter"])
    if gs_fp64(p):
        check_norms("gs fp64 (10 iterations)", got, ref, GS_FP64, GS_FP64)
        return
    # fp32 iterations.  The amplitude step keeps only the phase w / |w|, whose error is
    # the transform's error divided by |w|: a max-norm bound would fail wherever |w|
    # happens to be small (on random input the smallest |w| of n elements is about
    # rms / sqrt(n), so the error grows with the size).  Each element is therefore held to
    # the fp32 transform bound t = 1e-5 max|w| carried through that step:
    #   known amplitude a:  |got - ref| <= a t / |w| + 1e-6 a
    #   elsewhere:          |got - ref| <= t
    assert np.isfinite(got).all()
    t = MAX_FP32 * np.abs(pre).max()
    amp = x["amp"].astype(np.float64)
    known = ~np.isnan(amp)
    bound = np.full(got.shape, t)
    bound[known] = amp[known] * (t / np.abs(pre[known]) + 1e-6)
    ratio = np.abs(got - ref) / bound
    family = "gs fp32" if is_pow2(p["n0"]) and is_pow2(p["n1"]) else "gs chirp-z"
    _record(family + " (error / conditioned bound)", "per-element", ratio.max(), 1.0)
    assert ratio.max() <= 1.0, "%s: element %s at %.3g of its bound" % (
        family, np.unravel_index(ratio.argmax(), ratio.shape), ratio.max())


def screen_inputs(case):
    rng = _rng(case)
    shape = (case.p["nx"], case.p["ny"])
    return {"w": rng.uniform(0.5, 1.5, shape), "n1": rng.normal(size=shape),
            "n2": rng.normal(size=shape)}


def screen_device(case, x):
    import torch
    D, L = _dev()
    nx, ny = case.p["nx"], case.p["ny"]
    out = D.empty((nx, ny), torch.float64)
    w, n1, n2 = D.upload(x["w"]), D.upload(x["n1"]), D.upload(x["n2"])
    L.check(L.lib.sb_sim_screen(nx, ny, w.data_ptr(), n1.data_ptr(), n2.data_ptr(), 0,
                                out.data_ptr(), D.stream_ptr()))
    return out.cpu().numpy()


def screen_check(case, x, got):
    # SimOracle.get_screen: xyp = real(fft2(w * (n1 + i n2)))
    ref = np.real(np.fft.fft2(x["w"] * (x["n1"] + 1j * x["n2"])))
    check_norms("sim screen (fp64)", got, ref, NORM_FP64_SCREEN, NORM_FP64_SCREEN)
    nx, ny = case.p["nx"], case.p["ny"]
    for pos in ((nx - 1, ny - 1), (0, 0)):
        imp = {"w": np.ones((nx, ny)), "n1": np.zeros((nx, ny)), "n2": np.zeros((nx, ny))}
        imp["n1"][pos] = 1.0
        check_bins("sim screen impulse (fp64)", screen_device(case, imp),
                   phase_ramp((nx, ny), pos, -1).real, NORM_FP64_SCREEN)


def intensity_inputs(case):
    rng = _rng(case)
    nx, ny, nf = case.p["nx"], case.p["ny"], case.p["nf"]
    dx = dy = 0.01
    return {"xyp": rng.normal(0.0, 3.0, (nx, ny)),
            "scales": 1 / (1.0 + 0.25 * (-0.5 + np.arange(nf) / nf)),    # scint_sim.py:218-224
            "ffconx": 2.0 / (nx * dx) ** 2 * np.pi ** 2,
            "ffcony": 2.0 / (ny * dy) ** 2 * np.pi ** 2}


def intensity_device(case, x):
    import torch
    D, L = _dev()
    nx, ny, nf = case.p["nx"], case.p["ny"], case.p["nf"]
    spe = D.empty((nf, nx, 2), torch.float32)
    xyi = D.empty((nx, ny), torch.float32)
    scales = np.ascontiguousarray(x["scales"], dtype=np.float64)
    L.check(L.lib.sb_sim_intensity(nx, ny, nf, D.upload(x["xyp"]).data_ptr(), scales.ctypes.data,
                                   x["ffconx"], x["ffcony"], spe.data_ptr(), xyi.data_ptr(),
                                   D.stream_ptr()))
    return to_complex(spe.cpu().numpy()), xyi.cpu().numpy()


def intensity_check(case, x, got):
    nx, ny = case.p["nx"], case.p["ny"]
    sim = SimpleNamespace(nx=nx, ny=ny, ffconx=x["ffconx"], ffcony=x["ffcony"])
    spe = []
    for s in x["scales"]:                                  # SimOracle.get_intensity
        xye = np.fft.fft2(np.exp(1j * x["xyp"] * s))
        xye = SO.SimOracle.frfilt3(sim, xye, s)
        xye = np.fft.ifft2(xye)
        spe.append(xye[:, ny // 2])
    check_norms("sim intensity spe", got[0], np.array(spe), NORM_FP32)
    check_norms("sim intensity xyi", got[1], np.abs(xye) ** 2, NORM_FP32_POWER)


ENTRIES = {
    "sspec": (sspec_inputs, sspec_device, sspec_check),
    "acf": (acf_inputs, acf_device, acf_check),
    "acf_sspec": (acf_sspec_inputs, acf_sspec_device, acf_sspec_check),
    "cs": (cs_inputs, cs_device, cs_check),
    "ifft2": (ifft2_inputs, ifft2_device, ifft2_check),
    "gs": (gs_inputs, gs_device, gs_check),
    "screen": (screen_inputs, screen_device, screen_check),
    "intensity": (intensity_inputs, intensity_device, intensity_check),
}


def run_device(case):
    inputs, device, _ = ENTRIES[case.entry]
    return device(case, inputs(case))


def run_case(case):
    inputs, device, check = ENTRIES[case.entry]
    x = inputs(case)
    check(case, x, device(case, x))


# --------------------------------------------------------------------------
# tests
# --------------------------------------------------------------------------
def test_case_table_coverage():
    """Every row length, column length and load path, and tile length 256 in
    both precisions, is reached by some case."""
    assert missing_coverage(CASES) == []
    assert len({case_id(c) for c in CASES}) == len(CASES)


def test_limits_accepted_side_in_table():
    ids = {case_id(c) for c in CASES}
    for what, _, _, ok in LIMITS:
        assert case_id(ok) in ids, what


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_fft_length(case):
    run_case(case)


@pytest.mark.gpu
@pytest.mark.parametrize("what,bad,words,ok", LIMITS, ids=[x[0] for x in LIMITS])
def test_size_limit(what, bad, words, ok):
    """One past the largest size raises, says what the limit is, and leaves the
    library usable (the largest size itself is a case of test_fft_length)."""
    inputs, device, _ = ENTRIES[bad.entry]
    with pytest.raises(RuntimeError) as err:
        device(bad, inputs(bad))
    assert words in str(err.value), str(err.value)
    run_case(min((c for c in CASES if c.entry == bad.entry), key=case_size))


# TMA-eligible shapes: the fetch path and the row-thread layout must not change a bit
BITWISE_CASES = [
    _c("sspec", nf=64, nt=4096, window=False, halve=1, prewhite=0),
    _c("sspec", nf=2048, nt=100, window=False, halve=0, prewhite=0),
    _c("acf", nf=64, nt=2048, normalise=0),
    _c("acf", nf=1024, nt=60, normalise=0),
    _c("cs", nf=128, nt=512, npad=1, pad=0.375, half=False, keep=0, mask=True),
    _c("cs", nf=64, nt=256, npad=3, pad=-1.25, half=True, keep=0, mask=False),
]


@pytest.mark.gpu
def test_load_paths_bit_identical(tmp_path):
    """The fp32 transforms round every operation explicitly (fft_core.cuh), so the
    TMA and plain-load column passes and the N/16 and N/8 row-thread layouts
    compute the same bits.  Both switches are read once per process."""
    for c in BITWISE_CASES:
        assert any(t[0] == "col" and t[-1] == "tma" for t in templates(c)), case_id(c)
    here = [run_device(c) for c in BITWISE_CASES]
    out = tmp_path / "alt.npz"
    env = dict(os.environ, SB_FFT_NO_TMA="1", SB_ROW_DIV="8",
               PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--device-outputs", str(out)],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    alt = np.load(out)
    for i, c in enumerate(BITWISE_CASES):
        assert np.array_equal(here[i], alt["arr_%d" % i]), case_id(c)


@pytest.mark.gpu
def test_column_chunks_bit_identical(monkeypatch):
    """SB_COL_CHUNK_MB=1 at 512 x 1024: five column chunks, the last one column
    wide, give the same bits as one pass."""
    c = _c("sspec", nf=512, nt=1024, window=False, halve=1, prewhite=0)
    x = sspec_inputs(c)
    whole = sspec_device(c, x)
    monkeypatch.setenv("SB_COL_CHUNK_MB", "1")
    chunked = sspec_device(c, x)
    monkeypatch.delenv("SB_COL_CHUNK_MB")
    assert np.array_equal(whole, chunked)
    sspec_check(c, x, chunked)


if __name__ == "__main__":
    # device outputs of BITWISE_CASES for test_load_paths_bit_identical (fresh process)
    dest = sys.argv[sys.argv.index("--device-outputs") + 1]
    np.savez(dest, *[run_device(c) for c in BITWISE_CASES])
