"""The transform kernels in the built library (no GPU: cuobjdump reads the sm_90a SASS).  Both stream with 128-bit global
loads and stores; the main kernel (fdlibm, round, the exact ops) must not touch local memory.  The java.lang.Math kernel
may: CUDA's large-argument reduction of sin / cos / tan keeps its array there."""
import re

import pytest

from test_sass_budget_cpu import _cuobjdump, _sass

MAIN = "_ZN3anv16transform_kernelILb0EEEvPK12anv_column_tPK20anv_transform_spec_tPKPvPKPjPyl"
MATH = "_ZN3anv16transform_kernelILb1EEEvPK12anv_column_tPK20anv_transform_spec_tPKPvPKPjPyl"


@pytest.mark.parametrize("fun", [MAIN, MATH])
def test_transform_kernels_stream_128_bit(fun):
    if _cuobjdump() is None:
        pytest.skip("cuobjdump not found")
    from anovos_b200 import build
    ins = _sass(build.build(), fun)
    assert ins, "no SASS for " + fun
    if fun == MAIN:
        assert not [i for i in ins if re.search(r"\b(LDL|STL)\b", i)]
    assert any(re.match(r"LDG\.E\.[A-Z.]*128", i) for i in ins)
    assert any(re.match(r"STG\.E\.[A-Z.]*128", i) for i in ins)
