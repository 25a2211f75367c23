"""The bucket count's two partition passes (coarse: raw column -> keys grouped per tile; fine: chunks gathered from their
tile segments) against the LSD sort, cell for cell: mode, mode rows, distinct count, the summary ranks and the HLL++
registers, on columns built around the passes' edges - row counts that end mid-tile, mid-CTA span and mid-quad, nulls
across tile and bitmap-word edges, all-null and all-zero tiles, one group holding every key, coarse splitters crowded into
one lookup cell, NaN runs, and chunks spanning more than one 512-tile window."""
import numpy as np
import pyarrow as pa
import pytest

from test_gpu_bucket_count import _both, _check_equal, _summary_ranks

pytestmark = pytest.mark.gpu

TILE = 4096
N_ODD = TILE * 53 + 1236          # 54 tiles (a coarse CTA spans 16): the last CTA and the last tile are partial


def _edge_nulls(n, rng, rate):
    """Random nulls, plus nulls on both sides of every tile edge and of the 32-row bitmap words around it."""
    m = rng.random(n) < rate
    for e in range(TILE, n, TILE):
        m[e - 33:e + 33:31] = True
    return m


def _run(monkeypatch, t):
    from anovos_b200.frame import ColumnFrame
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    _check_equal(*_both(monkeypatch, fr, names, _summary_ranks(fr, names), 12), names)


def test_float_columns_at_the_tile_edges(monkeypatch):
    rng = np.random.default_rng(11)
    n = N_ODD
    normal = rng.normal(3.0, 2.0, n).astype(np.float32)
    holes = rng.uniform(-1e3, 1e3, n).astype(np.float32)
    holes[5 * TILE:7 * TILE] = 0.0                    # two all-zero tiles
    hmask = rng.random(n) < 0.05
    hmask[9 * TILE:10 * TILE] = True                  # an all-null tile
    nan_runs = rng.normal(0.0, 1.0, n).astype(np.float32)
    for s in range(100, n, 7919):
        nan_runs[s:s + 500] = np.nan
    t = pa.table({
        "normal": pa.array(normal, mask=_edge_nulls(n, rng, 0.1)),
        "holes": pa.array(holes, mask=hmask),
        "constant": pa.array(np.full(n, 2.5, np.float32)),
        "nan_runs": pa.array(nan_runs, mask=_edge_nulls(n, rng, 0.02)),
        "few_values": pa.array(rng.choice(np.array([-1.5, 0.0, 0.25, 7.0], np.float32), n)),
    })
    _run(monkeypatch, t)


def test_int_columns_with_crowded_coarse_splitters(monkeypatch):
    rng = np.random.default_rng(12)
    n = N_ODD + 1                  # also ends mid-quad (the coarse pass loads 4 rows per lane)
    t = pa.table({
        # every key shares its top 12 bits: all coarse splitters fall into one lookup cell
        "one_cell": pa.array(rng.integers(1, 1 << 20, n).astype(np.int32), mask=_edge_nulls(n, rng, 0.03)),
        "wide": pa.array(rng.integers(-2 ** 31, 2 ** 31 - 1, n).astype(np.int32)),
        "constant": pa.array(np.full(n, -7, np.int32)),
        "mostly_zero": pa.array(np.where(rng.random(n) < 0.9, 0, rng.integers(-100, 100, n)).astype(np.int32)),
    })
    _run(monkeypatch, t)


def test_sparse_groups_span_several_windows(monkeypatch):
    """95 % nulls at 3 M rows: ~6 keys of a group per tile, so a group's first chunk spans ~640 tiles."""
    rng = np.random.default_rng(13)
    n = 3_000_001
    t = pa.table({
        "f": pa.array(rng.normal(0.0, 1.0, n).astype(np.float32), mask=rng.random(n) < 0.95),
        "i": pa.array(rng.integers(-10 ** 6, 10 ** 6, n).astype(np.int32), mask=rng.random(n) < 0.97),
    })
    _run(monkeypatch, t)
