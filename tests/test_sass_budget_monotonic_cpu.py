"""The label-class histogram kernel in the built library (no GPU: cuobjdump reads the sm_90a SASS): a streaming pass, so
it must not spill to local memory and must load its rows with 128-bit global loads."""
import re

import pytest

from test_sass_budget_cpu import _cuobjdump, _sass

FUN = "_ZN3anv17class_hist_kernelEPK12anv_column_tPK21anv_class_hist_spec_tPKjS7_l"


def test_class_hist_streams_without_spills():
    if _cuobjdump() is None:
        pytest.skip("cuobjdump not found")
    from anovos_b200 import build
    ins = _sass(build.build(), FUN)
    assert ins, "no SASS for " + FUN
    assert not [i for i in ins if re.search(r"\b(LDL|STL)\b", i)]
    assert any(re.match(r"LDG\.E\.[A-Z.]*128", i) for i in ins)
