"""Instruction budget of the bucket count's direct kernel in the built library (no GPU: cuobjdump reads the sm_90a SASS),
next to the fine and hash count kernels' in test_sass_budget_bucket_cpu.py.

pc_direct_kernel counts most keys of float columns.  A compiler or source change that makes its code longer, or makes it
spill, costs time on every direct bucket without changing any result, so no other test notices.  The budget is the SASS
length of the current build + 5 %."""
import re

import pytest

from test_sass_budget_cpu import _cuobjdump, _sass

# mangled name -> (max SASS instructions, NOPs excluded; local-memory accesses (LDL / STL) the build has)
BUDGETS = {
    # pc_direct_kernel: 1836 with the stage fill inlined, the counter scan unrolled over 8 counters and the rank prefix's
    # rotated (conflict-free) reads
    "_ZN3anv16pc_direct_kernelENS_8PcParamsEiPd": (1928, 0),
}


@pytest.mark.parametrize("fun", sorted(BUDGETS))
def test_direct_count_kernel_stays_within_its_sass_budget(fun):
    if _cuobjdump() is None:
        pytest.skip("cuobjdump not found")
    from anovos_b200 import build
    lib = build.build()
    ins = _sass(lib, fun)
    assert ins, "no SASS for %s in %s" % (fun, lib)
    budget, local = BUDGETS[fun]
    assert len(ins) <= budget, "%s: %d SASS instructions, budget %d" % (fun, len(ins), budget)
    n_local = sum(1 for i in ins if re.search(r"\b(LDL|STL)\b", i))
    assert n_local <= local, "%s: %d local-memory accesses (spills), the build has %d" % (fun, n_local, local)
