"""CPU check of the two-level bucket count's workspace: per column it is no larger than the LSD sort's workspace for
32-bit keys was when the bucket count became the default, so that switch never shrinks a column batch (no compute calls
without a GPU).

The bound is `anv_mode_distinct_workspace_bytes(n_cols, n_rows, 32)` of that build, written as a literal table.  The LSD
workspace has since shrunk (the buffers of the removed one-sweep passes left it), so the live figure is no longer the
bound; it is checked against the same table, because it may only shrink."""
import pytest

# n_cols -> n_rows -> bytes
LSD_WORKSPACE_BOUND = {
    1: {
        65_536: 583_936,
        65_537: 587_776,
        300_007: 2_640_128,
        1_000_000: 8_770_560,
        4_194_305: 36_746_752,
        10_000_000: 87_590_144,
        40_000_000: 350_323_712,
        100_000_000: 875_794_176,
        2 ** 32 - 1: 37_614_528_256,
    },
    7: {
        65_536: 4_083_456,
        65_537: 4_108_800,
        300_007: 18_475_520,
        1_000_000: 61_389_312,
        4_194_305: 257_221_632,
        10_000_000: 613_125_632,
        40_000_000: 2_452_261_632,
        100_000_000: 6_130_555_136,
        2 ** 32 - 1: 263_301_693_696,
    },
    150: {
        65_536: 87_491_328,
        65_537: 88_033_792,
        300_007: 395_891_456,
        1_000_000: 1_315_470_592,
        4_194_305: 5_511_880_192,
        10_000_000: 13_138_393_856,
        40_000_000: 52_548_448_256,
        100_000_000: 131_369_022_720,
        2 ** 32 - 1: 5_642_179_139_328,
    },
}


@pytest.mark.parametrize("n_cols", [1, 7, 150])
def test_bucket_count_workspace_within_the_recorded_sort_workspace(n_cols):
    import __graft_entry__ as G
    G.build()
    from anovos_b200 import _lib
    L = _lib.lib()
    for n_rows, bound in LSD_WORKSPACE_BOUND[n_cols].items():
        part = L.anv_mode_distinct_partition_workspace_bytes(n_cols, n_rows)
        assert part <= bound, (n_cols, n_rows, part, bound)
        lsd = L.anv_mode_distinct_workspace_bytes(n_cols, n_rows, 32)
        assert lsd <= bound, (n_cols, n_rows, lsd, bound)
