"""CPU checks of the C-ABI library: it is built, loads, and exports every symbol that
include/anovos_b200.h declares (no compute calls without a GPU)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    h = open(os.path.join(ROOT, "include", "anovos_b200.h")).read()
    h = re.sub(r"/\*.*?\*/", "", h, flags=re.S)
    return sorted(set(re.findall(r"\b(anv_[a-z0-9_]+)\s*\(", h)))


def test_library_builds_and_exports_every_declared_symbol():
    import __graft_entry__ as G
    G.build()
    from anovos_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 10
    for n in names:
        assert hasattr(lib, n), "missing export " + n
    assert sorted(names) == _lib.exported_symbols()      # the Python binding covers the whole header
    assert _lib.lib().anv_version() == 100


def test_column_block_limit_matches_header():
    from anovos_b200 import _lib
    h = open(os.path.join(ROOT, "include", "anovos_b200.h")).read()
    assert int(re.search(r"#define ANV_MAX_LAUNCH_COLS (\d+)", h).group(1)) == _lib.MAX_LAUNCH_COLS == 65535


def test_struct_layouts_match_header():
    from anovos_b200 import _lib, engine
    assert ctypes.sizeof(_lib.AnvColumn) == 24 and ctypes.sizeof(_lib.AnvMoments) == 64
    assert ctypes.sizeof(_lib.AnvBinspec) == 32 and ctypes.sizeof(_lib.AnvDrift) == 40
    assert engine._MOM_DT.itemsize == 64 and engine._SPEC_DT.itemsize == 32 and engine._DRIFT_DT.itemsize == 40


def test_product_fails_loudly_without_cuda():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    import pyarrow as pa
    from anovos_b200 import _lib, engine
    from anovos_b200.frame import ColumnFrame
    fr = ColumnFrame.from_arrow(pa.table({"a": [1.0, 2.0]}))
    with pytest.raises(_lib.AnvError):
        engine.moments(fr, ["a"])
