"""The bucket count's coarse partition pass in the built library (no GPU: cuobjdump reads the sm_90a SASS), next to the
fine and count kernels' budgets in test_sass_budget_bucket_cpu.py.

The pass reads every row of every 32-bit column once.  It must load its rows as 128-bit words, keep 4 CTAs of 256
threads per SM (at most 64 registers) without spilling, and not grow: its budget is the SASS length of the current build
+ 5 %."""
import re
import subprocess

import pytest

from test_sass_budget_cpu import _cuobjdump, _sass

FUN = "_ZN3anv16pc_coarse_kernelENS_8PcParamsE"
BUDGET = 2139                      # 2037 with the 128-bit loads and the per-CTA (group, tile) table writes


@pytest.fixture(scope="module")
def lib():
    if _cuobjdump() is None:
        pytest.skip("cuobjdump not found")
    from anovos_b200 import build
    return build.build()


def test_coarse_pass_streams_without_spills(lib):
    ins = _sass(lib, FUN)
    assert ins, "no SASS for " + FUN
    assert not [i for i in ins if re.search(r"\b(LDL|STL)\b", i)]
    assert any(re.search(r"\bLDG\.E\.[A-Z0-9.]*\b128\b", i) for i in ins)
    assert len(ins) <= BUDGET, "%s: %d SASS instructions, budget %d" % (FUN, len(ins), BUDGET)


def test_coarse_pass_keeps_four_ctas_per_sm(lib):
    out = subprocess.run([_cuobjdump(), "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    m = re.search(r"Function %s:\s*\n\s*REG:(\d+)" % FUN, out)
    assert m, "no resource usage for " + FUN
    assert int(m.group(1)) <= 64
