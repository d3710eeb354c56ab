"""CPU: the library's internal plumbing in scintools_b200/csrc stays in one place each.
Every workspace request names its slot (the slot table and nesting rule are in common.cuh),
and each parameter struct the C API hands to a driver has one definition (drivers.cuh)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "scintools_b200", "csrc")


def _sources():
    out = {}
    for fn in sorted(os.listdir(CSRC)):
        if fn.endswith((".cu", ".cuh")):
            with open(os.path.join(CSRC, fn)) as f:
                out[fn] = f.read()
    return out


def test_workspace_slots_are_named():
    bad = []
    for fn, txt in _sources().items():
        for m in re.finditer(r"\bworkspace\(\s*\d|\bWsSlot\s*\)\s*\d|\bWsSlot>\(\s*\d", txt):
            bad.append("%s:%d" % (fn, txt.count("\n", 0, m.start()) + 1))
    assert not bad, "workspace slot given as an integer at " + ", ".join(bad)


@pytest.mark.parametrize("name", ["SimParams", "ThinGeom"])
def test_driver_struct_defined_once(name):
    where = [fn for fn, txt in _sources().items()
             for _ in re.finditer(r"\bstruct\s+%s\s*\{" % name, txt)]
    assert len(where) == 1, "struct %s defined in %s" % (name, where)
