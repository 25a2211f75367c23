"""Fine buckets whose splitters are at most PC_DIRECT_RANGE key values apart are counted by pc_direct_kernel in 16-bit
counters indexed by the key; every other bucket by pc_group_kernel's hash table.  These inputs put buckets on both sides
of that rule inside one column (range PC_DIRECT_RANGE and PC_DIRECT_RANGE + 1), a direct bucket larger than a stage, a
narrow bucket holding one key 70 000 times that has to stay on the hash path (its 16-bit counter would wrap), a mode tie
inside a direct bucket, direct first and last buckets of int32 columns, and generator frames where the direct path
carries most keys.  Every column is compared with the LSD sort cell for cell (HLL++ registers bit for bit) and with
NumPy's exact counts and order statistics.

The columns are built as in test_gpu_bucket_stage.py: a background that every splitter is taken from, here with
background values placed a chosen number of key values apart, and the planted values on rows the splitter sample never
reads.  Each test asserts the ranges R and bucket sizes n it relies on."""
import numpy as np
import pyarrow as pa
import pytest

from test_gpu_bucket_count import _both, _check_equal, _sample_rows, _summary_ranks
from test_gpu_bucket_stage import Column, _check_numpy, _key, _ranks_at

pytestmark = pytest.mark.gpu

DIRECT_RANGE = 1 << 14       # PC_DIRECT_RANGE in sort.cu
STAGE_KEYS = 5120            # PC_SWEEP_KEYS
ZERO_KEY = 0x80000000


def _ikey(v):
    return (np.asarray(v, np.int64) + 2 ** 31).astype(np.uint64)


def _keys(x):
    return _ikey(x) if x.dtype == np.int32 else _key(x)


def _splitters(x, valid, c):
    """The fine splitters pc_sample_kernel / pc_split_kernel take for batch column c (float32 or int32 x)."""
    p, rows = _sample_rows(x.size, c)
    k = np.sort(_keys(x[rows][valid[rows]]))
    k = k[k != ZERO_KEY]
    idx = np.minimum((np.arange(1, p, dtype=np.int64) * k.size) // p, k.size - 1)
    s = k[idx]
    return np.insert(s, np.searchsorted(s, ZERO_KEY), np.uint64(ZERO_KEY))


def _buckets(x, valid, c):
    """-> (bucket of every valid non-splitter key (-1 otherwise), size n and range R of every bucket)"""
    s = _splitters(x, valid, c)
    k = _keys(x)
    b = np.searchsorted(s, k, "left")
    eq = (b < s.size) & (s[np.minimum(b, s.size - 1)] == k)
    bucket = np.where(valid & (k != ZERO_KEY) & ~eq, b, -1)
    lo = np.concatenate([[-1], s.astype(np.int64)])
    hi = np.concatenate([s.astype(np.int64), [2 ** 32]])
    return bucket, np.bincount(bucket[bucket >= 0], minlength=s.size + 1), hi - lo - 1


def _is_direct(n, r):
    return (n > 0) & (n < 2 ** 16) & (r <= DIRECT_RANGE)


def _after(v, ulps):
    """The float32 `ulps` representable values above positive v."""
    return (np.asarray(v, np.float32).view(np.uint32) + np.uint32(ulps)).view(np.float32)


def _bucket_of(col, values):
    bucket, sizes, ranges = _buckets(col.x, col.valid, col.c)
    b = np.unique(bucket[np.isin(col.x, values) & col.valid])
    assert b.size == 1 and b[0] >= 0
    return int(b[0]), int(sizes[b[0]]), int(ranges[b[0]])


def _float_column(c, seed, edges):
    """A Column whose background also holds the float32 values `edges`, which become adjacent splitters."""
    col = Column(1_000_003, c, seed)
    bg = np.concatenate([np.arange(1, 11), np.arange(50, 140)]).astype(np.float32)
    col.x = col.rng.choice(np.concatenate([bg, np.asarray(edges, np.float32)]), col.n)
    return col


def _edge_column(c, seed):
    """Buckets of range DIRECT_RANGE (20 000 keys: direct, several stages) and DIRECT_RANGE + 1 (6 000 keys: hash path)
    next to each other, and a bucket of range 1 000 holding one key 70 000 times (n >= 2^16: hash path), the column's
    mode."""
    e0 = np.float32(20)
    e1 = _after(e0, DIRECT_RANGE + 1)
    e2 = _after(e1, DIRECT_RANGE + 2)
    n0 = np.float32(30)
    n1 = _after(n0, 1001)
    col = _float_column(c, seed, [e0, e1, e2, n0, n1])
    a = _after(e0, 1 + col.rng.integers(0, DIRECT_RANGE, 20_000))
    a[:2] = [_after(e0, 1), _after(e0, DIRECT_RANGE)]              # the bucket's first and last key value
    b = _after(e1, 1 + col.rng.integers(0, DIRECT_RANGE + 1, 6_000))
    # 70 000 copies of one key at counter index 100 (the low half of a word: a 16-bit count that wrapped would carry into
    # counter 101, whose key never occurs) and 3 000 others: counted directly, its multiplicity and the distinct count
    # would come out wrong
    other = 1 + col.rng.integers(0, 1000, 3_000)
    d = _after(n0, np.concatenate([np.full(70_000, 101), other[(other != 101) & (other != 102)]]))
    d = col.rng.permutation(d)
    for v in (a, b, d):
        col.plant(v)
    ba, na, ra = _bucket_of(col, a)
    bb, nb, rb = _bucket_of(col, b)
    bd, nd, rd = _bucket_of(col, d)
    assert (ra, na) == (DIRECT_RANGE, a.size) and _is_direct(na, ra) and na > STAGE_KEYS
    assert (rb, nb) == (DIRECT_RANGE + 1, b.size) and bb > ba and not _is_direct(nb, rb)
    assert (rd, nd) == (1000, d.size) and nd >= 2 ** 16 and not _is_direct(nd, rd)
    assert np.unique(col.x[col.valid & ~np.isin(col.x, d)], return_counts=True)[1].max() < 70_000
    return col, [a, b, d]


def _tie_column(c, seed):
    """A direct bucket whose two most frequent keys tie, more often than any background value: the column's mode is
    the smaller one."""
    e0 = np.float32(20)
    col = _float_column(c, seed, [e0, _after(e0, 4001)])
    small, large = _after(e0, 1500), _after(e0, 2500)
    rest = _after(e0, 1 + col.rng.integers(0, 4000, 5_000))
    rest = rest[(rest != small) & (rest != large)]
    t = col.rng.permutation(np.concatenate([np.repeat([large, small], 15_000), rest]).astype(np.float32))
    col.plant(t)
    bt, nt, rt = _bucket_of(col, t)
    assert rt == 4000 and _is_direct(nt, rt) and nt == t.size
    assert np.unique(col.x[col.valid & ~np.isin(col.x, t)], return_counts=True)[1].max() < 15_000
    return col, [t]


def _columns_at(cols):
    from anovos_b200.frame import ColumnFrame
    names = ["d%d" % i for i in range(len(cols))]
    t = pa.table({nm: pa.array(col.x, mask=~col.valid) for nm, (col, _) in zip(names, cols)})
    rk = np.array([(_ranks_at(col.x, col.valid, sets) + [1, int(col.valid.sum())] + [0] * 16)[:16] for col, sets in cols],
                  dtype=np.int64)
    return t, ColumnFrame.from_arrow(t), names, rk


@pytest.mark.parametrize("p", [4, 9, 12])
def test_buckets_on_both_sides_of_the_direct_rule(p, monkeypatch):
    cols = [_edge_column(0, 31), _tie_column(1, 32), _edge_column(2, 33)]
    t, fr, names, rk = _columns_at(cols)
    got, ref = _both(monkeypatch, fr, names, rk, p)
    _check_equal(got, ref, names)
    _check_numpy(t, names, rk, got)
    assert got[0][1][0] == float(_after(np.float32(20), 1500)) and got[0][1][1] == 15_000
    for i in (0, 2):                                     # the 70 000-fold key of the narrow bucket
        assert got[0][i][0] == float(_after(np.float32(30), 101)) and got[0][i][1] == 70_000


def _int_edges_column(c, seed):
    """int32 values down to -2^31 below the lowest splitter and up to 2^31 - 1 above the top one: direct first and last
    buckets, each of range 10 000."""
    col = Column(1_000_003, c, seed)
    lo_edge, hi_edge = -2 ** 31 + 10_000, 2 ** 31 - 1 - 10_000
    bg = np.concatenate([[lo_edge, hi_edge], np.arange(-40, 60) * 1000]).astype(np.int32)
    col.x = col.rng.choice(bg, col.n).astype(np.int32)
    first = (-2 ** 31 + col.rng.integers(0, 10_000, 3_000)).astype(np.int32)
    last = (hi_edge + 1 + col.rng.integers(0, 10_000, 3_000)).astype(np.int32)
    first[0], last[0] = -2 ** 31, 2 ** 31 - 1
    col.plant(first)
    col.plant(last)
    bucket, sizes, ranges = _buckets(col.x, col.valid, c)
    bf, bl = _bucket_of(col, first)[0], _bucket_of(col, last)[0]
    assert bf == 0 and ranges[0] == 10_000 and _is_direct(sizes[0], ranges[0])
    assert bl == sizes.size - 1 and ranges[-1] == 10_000 and _is_direct(sizes[-1], ranges[-1])
    return col, [first, last]


def test_direct_first_and_last_buckets_of_int32_columns(monkeypatch):
    cols = [_int_edges_column(c, 40 + c) for c in range(2)]
    t, fr, names, rk = _columns_at(cols)
    for p in (4, 9, 12):
        got, ref = _both(monkeypatch, fr, names, rk, p)
        _check_equal(got, ref, names)
        _check_numpy(t, names, rk, got)
    # one column per batch: each batch samples its column as column 0
    from anovos_b200 import _lib, engine
    per_col = _lib.lib().anv_mode_distinct_partition_workspace_bytes(1, fr.n_rows)
    monkeypatch.setattr(engine, "SORT_WORKSPACE_BUDGET", per_col)
    assert engine._mode_distinct_batch_size(fr, len(names), per_col) == 1
    _check_equal(engine.sort_mode_distinct(fr, names, rk, hll_p=12), got, names)


def test_generator_frame_is_counted_mostly_direct(monkeypatch):
    """10 M rows of all four generator families: the direct path carries most keys, and the results match the sort."""
    from anovos_b200 import synth
    fr = synth.device_frame(10_000_000, 9, cat_every=4, seed=11)
    names = [n for n in fr.columns if fr.column(n).kind == "num"]
    t = fr.to_arrow()
    direct = total = 0
    for c, nm in enumerate(names):
        arr = t.column(nm).combine_chunks()
        x = np.asarray(arr.fill_null(0))
        valid = ~np.asarray(arr.is_null())
        bucket, sizes, ranges = _buckets(x, valid, c)
        direct += int(sizes[_is_direct(sizes, ranges)].sum())
        total += int(sizes.sum())
    assert direct > total // 2, (direct, total)
    rk = _summary_ranks(fr, names)
    for p in (9, 12):
        _check_equal(*_both(monkeypatch, fr, names, rk, p), names)
