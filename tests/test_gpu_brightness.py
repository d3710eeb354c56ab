"""scint_sim.Brightness on the device (csrc/brightness.cu) against the unmodified
reference's fixtures (oracle/make_golden_brightness.py) at the bars of
tests/test_brightness_cpu.py (check_against_fixture): the axes, thetax, thetay and the
Jacobian bit-equal; acf_efield within 4 ulp of its maximum; B within 1e-12 max B; SS with the
same NaNs and within 1e-12 max B max jacobian (x2 after the flip); LSS within 1e-9 dB where
SS > 0; acf within 1e-12.  brightness_batch is bit-identical to single calls in any order and
on repeat, and sb_brightness_f64 gets the library-state cases of
tests/test_gpu_library_state.py."""
import importlib
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CPU = importlib.import_module("test_brightness_cpu")
LS = importlib.import_module("test_gpu_library_state")
grown = LS.grown
ATTRS = ("x", "X", "Y", "acf_efield", "B", "fd", "td", "thetax", "thetay", "jacobian", "SS",
         "LSS", "acf")
SMALL = dict(nx=4, dx=0.1, nf=1, df=0.02, nt=8, dt=0.16)


def _attrs(b):
    return {k: getattr(b, k) for k in ATTRS}


@pytest.mark.parametrize("fn", CPU.FIXTURES, ids=CPU.IDS)
def test_fixture(fn):
    from scintools_b200.scint_sim import Brightness
    z = np.load(fn)
    b = Brightness(**json.loads(str(z["kwargs"])))
    assert b.SS.dtype == np.float64 and b.SS.shape == (len(b.td), len(b.fd))
    CPU.check_against_fixture(z, _attrs(b))


def _same(a, b):
    for k in ATTRS:
        assert np.array_equal(a[k], b[k], equal_nan=True), k
        assert np.asarray(a[k]).dtype == np.asarray(b[k]).dtype, k


def _sets(rng, m):
    return [dict(ar=float(rng.uniform(1, 4)), psi=float(rng.uniform(-90, 90)),
                 alpha=float(rng.choice([1.67, 2.0, 1.0, rng.uniform(1, 2)])),
                 thetagx=float(rng.uniform(-0.3, 0.3)), thetagy=float(rng.uniform(-0.3, 0.3)),
                 thetarx=float(rng.uniform(-0.3, 0.3)), thetary=float(rng.uniform(-0.3, 0.3)))
            for _ in range(m)]


def test_batch_equals_single_calls(monkeypatch):
    from scintools_b200 import scint_sim as S
    sets = _sets(np.random.default_rng(7), 9)
    single = [_attrs(S.Brightness(**p, **SMALL)) for p in sets]
    batch = S.brightness_batch(sets, **SMALL)
    for a, b in zip(batch, single):
        _same(_attrs(a), b)
    order = [4, 0, 8, 2, 6, 1, 7, 3, 5]
    for k, a in zip(order, S.brightness_batch([sets[k] for k in order], **SMALL)):
        _same(_attrs(a), single[k])
    # groups of two sets: the same bits as one group
    monkeypatch.setattr(S, "_BRIGHT_GROUP_BYTES", 2 * 8 * (2 * 80 ** 2 + 8 * 100 * 100) +
                        16 * (100 * 100 * 2))
    for a, b in zip(S.brightness_batch(sets, **SMALL), single):
        _same(_attrs(a), b)


def test_batch_against_oracle():
    from oracle import brightness_oracle as BO
    from scintools_b200.scint_sim import brightness_batch
    sets = _sets(np.random.default_rng(11), 6)
    for p, b in zip(sets, brightness_batch(sets, **SMALL)):
        ref = BO.model(**p, **SMALL)
        CPU.check_against_fixture({k: ref[k] for k in CPU.EXACT + (
            "acf_efield", "B", "SS", "LSS", "acf")}, _attrs(b))


def test_stages_on_their_own():
    """calc_brightness, calc_SS and calc_acf re-read the attributes; calc_acf without
    calc_sspec raises AttributeError on SS as the reference does."""
    from oracle import brightness_oracle as BO
    from scintools_b200.scint_sim import Brightness
    with pytest.raises(AttributeError):
        Brightness(calc_sspec=False, **SMALL)
    b = Brightness(calc_sspec=False, calc_acf=False, **SMALL)
    assert not hasattr(b, "SS")
    full = _attrs(Brightness(**SMALL))
    b.calc_SS()
    b.calc_acf()
    _same(_attrs(b), full)
    b.B = b.B * 2.0                                   # calc_SS reads B
    b.calc_SS()
    assert np.array_equal(b.SS, full["SS"] * 2.0)
    b.SS = full["SS"][::-1].copy()                    # calc_acf reads SS
    b.calc_acf()
    ref = BO.acf(full["SS"][::-1].copy())
    assert np.max(np.abs(b.acf - ref)) <= 1e-12


def test_sizes_at_the_limits():
    """A 1024-point lattice and 4096 delays run; one more of either raises ValueError."""
    from oracle import brightness_oracle as BO
    from scintools_b200.scint_sim import Brightness
    b = Brightness(nx=51.2, dx=0.1, nf=0.04, df=0.02, nt=0.4, dt=0.1)
    assert b.B.shape == (1024, 1024)
    ref = BO.efield(nx=51.2, dx=0.1)[4]
    assert np.max(np.abs(b.B - ref)) <= 1e-12 * ref.max()
    c = Brightness(nx=2, dx=0.1, nf=0.02, df=0.02, nt=204.8, dt=0.1, thetagx=0.5)
    assert c.SS.shape == (4096, 2)
    ref = BO.model(nx=2, dx=0.1, nf=0.02, df=0.02, nt=204.8, dt=0.1, thetagx=0.5)
    fin = np.isfinite(ref["SS"])
    assert np.array_equal(np.isfinite(c.SS), fin)
    assert fin.any()
    assert np.max(np.abs(c.SS - ref["SS"])[fin]) <= 2e-12 * ref["B"].max() * 100
    for kw in (dict(nx=51.25, dx=0.1), dict(nx=2, dx=0.1, nt=204.85, dt=0.1)):
        with pytest.raises(ValueError):
            Brightness(**kw)


# ---- library state: the cases of tests/test_gpu_library_state.py for sb_brightness_f64 -------
def run_brightness(size):
    from oracle import brightness_oracle as BO
    from scintools_b200.scint_sim import brightness_batch
    grid = SMALL if size == "small" else dict(nx=12, dx=0.1, nf=3, df=0.02, nt=16, dt=0.08)
    sets = _sets(np.random.default_rng(3), 2)
    out = []
    for p, b in zip(sets, brightness_batch(sets, **grid)):
        ref = BO.model(**p, **grid)
        CPU.check_against_fixture({k: ref[k] for k in CPU.EXACT + (
            "acf_efield", "B", "SS", "LSS", "acf")}, _attrs(b))
        out += [b.acf_efield, b.B, b.SS, b.LSS, b.acf]
    return out


CASE = LS.Case("brightness", ("sb_brightness_f64",), True, run_brightness)


def test_cold():
    from scintools_b200 import _lib
    LS._sb()
    _lib.check(_lib.lib.sb_release())
    LS.same(CASE, CASE.run("small"), run_brightness("small"), "cold vs repeat")


def test_after_others(grown):
    a = CASE.run("small")
    from scintools_b200 import _lib
    _lib.check(_lib.lib.sb_release())
    LS.same(CASE, a, CASE.run("small"), "after others vs cold")


def test_small_large_small():
    a = CASE.run("small")
    CASE.run("large")
    LS.same(CASE, CASE.run("small"), a, "small, large, small")


def test_side_stream():
    import torch
    ref = CASE.run("small")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = CASE.run("small")
    torch.cuda.synchronize()
    LS.same(CASE, got, ref, "side stream vs default stream")
