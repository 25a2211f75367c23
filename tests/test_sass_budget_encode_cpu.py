"""The encode kernels in the built library (no GPU: cuobjdump reads the sm_90a SASS): they are streaming passes, so they
must not spill to local memory and must move their rows with 128-bit global loads and stores."""
import re

import pytest

from test_sass_budget_cpu import _cuobjdump, _sass

FUNS = ["_ZN3anv15code_map_kernelEPK12anv_column_tPK19anv_code_map_spec_tPyl",
        "_ZN3anv14one_hot_kernelEPK12anv_column_tPK18anv_one_hot_spec_tl"]


@pytest.mark.parametrize("fun", FUNS)
def test_encode_kernels_stream_without_spills(fun):
    if _cuobjdump() is None:
        pytest.skip("cuobjdump not found")
    from anovos_b200 import build
    ins = _sass(build.build(), fun)
    assert ins, "no SASS for " + fun
    assert not [i for i in ins if re.search(r"\b(LDL|STL)\b", i)]
    assert any(re.match(r"LDG\.E\.[A-Z.]*128", i) for i in ins)
    assert any(re.match(r"STG\.E\.[A-Z.]*128", i) for i in ins)
