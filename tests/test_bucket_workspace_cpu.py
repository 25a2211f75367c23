"""CPU check of the two-level bucket count's workspace: per column it is no larger than the LSD sort's for 32-bit keys,
so switching the default path never shrinks a column batch (no compute calls without a GPU)."""
import pytest


@pytest.mark.parametrize("n_cols", [1, 7, 150])
def test_bucket_count_workspace_within_the_sort_workspace(n_cols):
    import __graft_entry__ as G
    G.build()
    from anovos_b200 import _lib
    L = _lib.lib()
    for n_rows in (65_536, 65_537, 300_007, 1_000_000, 4_194_305, 10_000_000, 40_000_000, 100_000_000, 2 ** 32 - 1):
        part = L.anv_mode_distinct_partition_workspace_bytes(n_cols, n_rows)
        lsd = L.anv_mode_distinct_workspace_bytes(n_cols, n_rows, 32)
        assert part <= lsd, (n_cols, n_rows, part, lsd)
