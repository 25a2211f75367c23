"""Instruction budgets of the bucket count's fine and count kernels in the built library (no GPU: cuobjdump reads the
sm_90a SASS), next to the scatter kernel's in test_sass_budget_cpu.py.

The two kernels are most of the default exact-mode / distinct / percentile path.  A compiler or source change that makes
their code longer, or makes them spill, costs time on every bucket of every column without changing any result, so no
other test notices.  The budgets are the SASS lengths of the current build + 5 %."""
import re

import pytest

from test_sass_budget_cpu import _cuobjdump, _sass

# mangled name -> (max SASS instructions, NOPs excluded; local-memory accesses (LDL / STL) the build has)
BUDGETS = {
    # pc_group_kernel: 3377 with the shared-memory stage (its fill inlined at every call site) and the owner fold
    "_ZN3anv15pc_group_kernelENS_8PcParamsEiPd": (3546, 0),
    # pc_fine_kernel: 1806 with the cp.async gather
    "_ZN3anv14pc_fine_kernelENS_8PcParamsE": (1896, 0),
}


@pytest.mark.parametrize("fun", sorted(BUDGETS))
def test_bucket_count_kernel_stays_within_its_sass_budget(fun):
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
