"""Instruction budget of the radix-sort scatter kernel in the built library (no GPU: cuobjdump reads the sm_90a SASS).

The sort is bound by instruction issue, and the scatter kernel is most of it.  A compiler or source change that makes
its code longer, or makes it spill, costs time on every pass of every column without changing any result, so no
other test notices.  The budgets are the SASS lengths at the current tuning + 5 %."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# mangled name -> (max SASS instructions, NOPs excluded; local-memory accesses (LDL / STL) the chosen tuning has)
BUDGETS = {
    # sort_scatter_kernel<unsigned int>: 1469 with the asm ballots at 2 CTAs per SM (1518 before its parameter struct lost the
    # one-sweep fields, 2081 with the C++ ballots before that)
    "_ZN3anv19sort_scatter_kernelIjEEvNS_10SortParamsIT_EE": (1594, 0),
}


def _cuobjdump():
    for p in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if p and os.path.exists(p):
            return p
    return None


def _sass(lib, fun):
    out = subprocess.run([_cuobjdump(), "-sass", "-fun", fun, lib], capture_output=True, text=True, check=True).stdout
    ins = [re.sub(r"/\* 0x[0-9a-f]+ \*/", "", l).split("*/", 1)[1].strip()
           for l in out.split("\n") if re.match(r"^\s+/\*[0-9a-f]{4,6}\*/", l)]
    return [i for i in ins if not i.startswith("NOP")]


@pytest.mark.parametrize("fun", sorted(BUDGETS))
def test_scatter_kernel_stays_within_its_sass_budget(fun):
    if _cuobjdump() is None:
        pytest.skip("cuobjdump not found")
    from anovos_b200 import build
    lib = build.build()
    ins = _sass(lib, fun)
    assert ins, "no SASS for %s in %s" % (fun, lib)
    budget, local = BUDGETS[fun]
    assert len(ins) <= budget, "%s: %d SASS instructions, budget %d" % (fun, len(ins), budget)
    n_local = sum(1 for i in ins if re.search(r"\b(LDL|STL)\b", i))
    assert n_local <= local, "%s: %d local-memory accesses (spills), the tuned build has %d" % (fun, n_local, local)
