"""Wavefield mosaic fit on the CPU: the float64 oracle (oracle/mosaic_oracle.py) against the
unmodified reference's rotInit ... fullMosHess (tests/golden/mosaic_*.npz, made by
oracle/make_golden_mosaic.py), the device code of csrc/mosaic.cu (all five tile modes and
the four reductions) under the SIMT emulator (tests/host_emu/mosaic_emu.cpp) against the
oracle, the argument errors of the port raised before any device call, and the new C
symbols."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import mosaic_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emu")
U = 2.0 ** -24

CASES = [("mosaic_sample", ""), ("mosaic_synth", ""), ("mosaic_synth", "b2_")]


def _case(golden_dir, name, pre):
    f = np.load(os.path.join(golden_dir, name + ".npz"))
    return {k[len(pre):]: f[k] for k in f.files if k.startswith(pre) and
            (pre or not k.startswith("b2_"))}


def _close(got, ref, mag, tol):
    got, ref, mag = np.asarray(got), np.asarray(ref), np.asarray(mag)
    assert got.shape == ref.shape
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref)
    assert (np.abs(got - ref)[fin] <= tol * mag[fin] + 1e-300).all()


@pytest.mark.parametrize("name,pre", CASES)
def test_oracle_matches_reference(golden_dir, name, pre):
    """Every function to 1e-12 of sum|terms|, except the Hessian (1e-8): the oracle follows
    the reference's complex64 roundings (in-place scaling of chunk copies, products of two
    complex64 arrays, a float32 N ** 2), but 1.4e-9 .. 3.2e-9 of sum|terms| remain on the
    three cases and are not traced to a further rounding of the reference.  The NaN pattern
    exactly; rotInit to 1e-12 rad away from the all-zero chunk."""
    c = _case(golden_dir, name, pre)
    ch, x, p, D, N = c["chunks"], c["x"], c["p"], c["dspec"], c["N"]
    if "rotMos" not in c:       # case a stores one copy: p = (x, ones) there
        P = ch.shape[0] * ch.shape[1]
        assert np.array_equal(p, np.concatenate([x, np.ones(P)]))
        c["rotMos"] = c["fullMos"]
    nF, nT = c["fullMos"].shape
    _close(*MO.rot_mos(ch, x)[:1], c["rotMos"], MO.rot_mos(ch, x)[1], 1e-12)
    _close(*MO.full_mos(ch, p)[:1], c["fullMos"], MO.full_mos(ch, p)[1], 1e-12)
    v, a = MO.rot_fit(ch, x)
    _close(v, c["rotFit"], a, 1e-12)
    v, a = MO.rot_der(ch, x)
    _close(v, c["rotDer"], a, 1e-12)
    v, a = MO.full_fit(ch, p, D, N)
    _close(v, c["fullMosFit"], a, 1e-12)
    v, a = MO.full_grad(ch, p, D[:nF, :nT], N)
    _close(v, c["fullMosGrad"], a, 1e-12)
    v, a = MO.full_hess(ch, p, D[:nF, :nT], N)
    _close(v, c["fullMosHess"], a, 1e-8)
    assert np.array_equal(c["fullMosHess"], c["fullMosHess"].T, equal_nan=True)
    xi, _ = MO.rot_init(ch)
    nz = np.abs(ch).reshape(-1, ch.shape[2] * ch.shape[3]).max(1)[1:] > 0
    assert np.abs(np.angle(np.exp(1j * (xi - c["rotInit"])))[nz]).max() <= 1e-12
    if "mosaic" in c:
        W, _ = MO.rot_mos(ch, c["rotInit"])
        assert np.abs(W - c["mosaic"]).max() <= 1e-12 * np.abs(c["mosaic"]).max()


def _emu_lib():
    src = os.path.join(EMU, "mosaic_emu.cpp")
    out = os.path.join(EMU, "_build", "mosaic_emu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    csrc = os.path.join(ROOT, "scintools_b200", "csrc")
    newest = max([os.path.getmtime(os.path.join(csrc, f)) for f in os.listdir(csrc)] +
                 [os.path.getmtime(src), os.path.getmtime(os.path.join(EMU, "simt.h"))])
    if not os.path.exists(out) or os.path.getmtime(out) < newest:
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                        "-x", "c++", src, "-o", out], check=True)
    lib = ctypes.CDLL(out)
    vp, ci = ctypes.c_void_p, ctypes.c_int
    lib.emu_mosaic.argtypes = [ci, vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.emu_mosaic.restype = ci
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _emu(lib, mode, ch, phi=None, amp=None, W=None, D=None, N=None, out0=None, out1=None,
         rows=None, cols=None):
    ncf, nct, cwf, cwt = ch.shape
    c32 = np.ascontiguousarray(ch, np.complex64)
    rc = lib.emu_mosaic(mode, _ptr(c32), ncf, nct, cwf, cwt, _ptr(phi), _ptr(amp), _ptr(W),
                        _ptr(D), _ptr(N), _ptr(out0), _ptr(out1), _ptr(rows), _ptr(cols))
    assert rc == 0


@pytest.mark.parametrize("name,pre", CASES)
def test_kernels_on_host_against_oracle(golden_dir, name, pre):
    """mosaic_tile_kernel in every mode and the reductions, run under the SIMT emulator on
    each fixture case (the tutorial chunks; the all-zero chunk and NaN pixels; the single
    chunk axis of odd width 7), within the float32 bounds derived in tests/test_gpu_mosaic.py."""
    c = _case(golden_dir, name, pre)
    ch, x, p, D, N = c["chunks"], c["x"], c["p"], c["dspec"], c["N"]
    P = ch.shape[0] * ch.shape[1]
    nF, nT = c["fullMos"].shape
    lib = _emu_lib()
    Dm = np.ascontiguousarray(D[:nF, :nT], np.float32)
    Nm = np.ascontiguousarray(N[:nF, :nT], np.float32)
    # rotMos / rotFit / rotDer: phases x, amplitudes NULL
    phi = np.concatenate([[0.0], x[:P - 1]])
    W = np.zeros((nF, nT), np.complex64)
    _emu(lib, 0, ch, phi=phi, W=W)
    ref, mag = MO.rot_mos(ch, x)
    _close(W.astype(complex), ref, 12 * U * mag, 1.0)
    power, der = np.zeros(1), np.zeros(P)
    _emu(lib, 1, ch, phi=phi, W=W, out0=power, out1=der)
    v, a = MO.rot_fit(ch, x)
    _close(-power[0], v, 24 * U * a, 1.0)
    v, a = MO.rot_der(ch, x)
    _close(der[1:], v[:P - 1], 24 * U * a[:P - 1], 1.0)
    # rotInit overlaps
    C = np.zeros((P, 4, 2))
    _emu(lib, 2, ch, out0=C)
    ref, mag = MO.overlaps(ch)
    _close(C[..., 0] + 1j * C[..., 1], ref, 9 * U * mag, 1.0)
    # fullMos / fullMosFit / fullMosGrad / fullMosHess at p
    phi = np.concatenate([[0.0], p[:P - 1]])
    amp = np.ascontiguousarray(p[P - 1:2 * P - 1])
    _emu(lib, 0, ch, phi=phi, amp=amp, W=W)
    ref, mag = MO.full_mos(ch, p)
    _close(W.astype(complex), ref, 12 * U * mag, 1.0)
    fit, grad = np.zeros(1), np.zeros((P, 2))
    _emu(lib, 3, ch, phi=phi, amp=amp, W=W, D=Dm, N=Nm, out0=fit, out1=grad)
    v, a = MO.full_fit(ch, p, D, N)
    _close(fit[0], v, 56 * U * a, 1.0)
    v, a = MO.full_grad(ch, p, Dm, N)
    _close(grad[:, 0], v[P - 1:2 * P - 1], 56 * U * a[P - 1:2 * P - 1], 1.0)
    _close(grad[1:, 1], v[:P - 1], 56 * U * a[:P - 1], 1.0)
    rows, cols = np.zeros(40 * P, np.int64), np.zeros(40 * P, np.int64)
    vals = np.zeros(40 * P)
    _emu(lib, 4, ch, phi=phi, amp=amp, W=W, D=Dm, N=Nm, out0=vals, rows=rows, cols=cols)
    keep = rows >= 0
    pairs = set(zip(rows[keep].tolist(), cols[keep].tolist()))
    assert len(pairs) == keep.sum()                     # every entry once
    H = np.zeros((len(p), len(p)))
    H[rows[keep], cols[keep]] = vals[keep]
    v, a = MO.full_hess(ch, p, Dm, N)
    _close(H, v, 56 * U * a, 1.0)


def test_synthetic_case_layout(golden_dir):
    """Case b holds what the GPU tests rely on: an all-zero chunk, NaN pixels, a long p, N
    larger than the mosaic; b2 is one chunk of odd width 7 in frequency."""
    c = _case(golden_dir, "mosaic_synth", "")
    assert (c["chunks"][1, 2] == 0).all() and np.isnan(c["dspec"]).sum() >= 3
    P = 12
    assert c["p"].shape[0] == 2 * P - 1 + 3 and c["N"].shape[0] > c["fullMos"].shape[0]
    assert np.isnan(c["fullMosHess"]).any() and np.isfinite(c["fullMosFit"])
    b2 = _case(golden_dir, "mosaic_synth", "b2_")
    assert b2["chunks"].shape == (1, 3, 7, 8) and b2["fullMos"].shape == (7, 16)


def test_port_argument_errors_before_device(golden_dir):
    """The reference's exceptions (case c) for odd widths, short x / p and mismatched dspec
    are raised by the port before it touches a device."""
    from scintools_b200 import ththmod as T
    e = np.load(os.path.join(golden_dir, "mosaic_errors.npz"))
    rng = np.random.default_rng(3)
    odd = (rng.normal(size=(2, 2, 7, 8)) + 0j).astype(np.complex64)
    ch = (rng.normal(size=(2, 3, 8, 8)) + 1j * rng.normal(size=(2, 3, 8, 8))).astype(np.complex64)
    P = 6
    good = np.ones((12, 16), np.float32)
    calls = dict(
        rotMos_odd=lambda: T.rotMos(odd, np.zeros(3)),
        rotInit_odd=lambda: T.rotInit(odd),
        fullMosFit_odd=lambda: T.fullMosFit(np.ones(7), odd, good, good),
        rotMos_short=lambda: T.rotMos(ch, np.zeros(P - 2)),
        rotDer_short=lambda: T.rotDer(np.zeros(P - 2), ch),
        fullMos_short=lambda: T.fullMos(ch, np.ones(2 * P - 2)),
        fullMosGrad_short=lambda: T.fullMosGrad(np.ones(2 * P - 2), ch, good, good),
        fullMosHess_short=lambda: T.fullMosHess(np.ones(2 * P - 2), ch, good, good),
        fullMosGrad_dspec=lambda: T.fullMosGrad(np.ones(2 * P - 1), ch, np.ones((13, 16)), good),
        fullMosHess_dspec=lambda: T.fullMosHess(np.ones(2 * P - 1), ch, np.ones((12, 15)), good),
        fullMosGrad_N=lambda: T.fullMosGrad(np.ones(2 * P - 1), ch, good, np.ones((11, 16))),
        fullMosFit_small=lambda: T.fullMosFit(np.ones(2 * P - 1), ch, np.ones((11, 16)), good),
    )
    assert set(calls) == set(e.files)
    for name, f in calls.items():
        want = {"ValueError": ValueError, "IndexError": IndexError}[str(e[name])]
        with pytest.raises(want):
            f()


def test_library_exports_mosaic_symbols():
    import __graft_entry__ as g
    g.build()
    from scintools_b200 import _lib, ththmod
    for n in ("build", "rot", "overlap", "fit", "hess"):
        assert "sb_mosaic_" + n in _lib.EXPORTS
    assert _lib.lib.sb_abi_version() >= 6
    for n in ("rotInit", "rotMos", "rotFit", "rotDer", "fullMos", "fullMosFit", "fullMosGrad",
              "fullMosHess", "MosaicModel"):
        assert callable(getattr(ththmod, n))
