"""The count pass of the two-level bucket count stages each fine bucket in shared memory before it counts it.  These
inputs put buckets exactly at the stage's size (5 120 keys) and one key over it, a bucket streamed in many pieces whose
hash classes have to be split several times, a group of more chunks than one window of its segment list, a bucket whose
keys sit in one chunk and empty buckets between full ones.  Every column is compared with the LSD sort cell for cell
(HLL++ registers bit for bit) and with NumPy's exact counts and order statistics.

The values are placed the way test_gpu_bucket_count.py places its dense run: a background of 100 integers that every
splitter is taken from, and the planted values on rows the splitter sample never reads, so that the buckets they fill
are known from the column alone.  Each test asserts the bucket sizes it relies on."""
import numpy as np
import pyarrow as pa
import pytest

from test_gpu_bucket_count import _both, _check_equal, _sample_rows

pytestmark = pytest.mark.gpu

STAGE_KEYS = 5120            # PC_SWEEP_KEYS in sort.cu
CHUNK = 4096                 # PC_CHUNK
WINDOW = 256                 # chunks per window of pc_stage_fill
BACKGROUND = np.concatenate([np.arange(1, 11), np.arange(50, 140)]).astype(np.float32)
ZERO_KEY = 0x80000000


def _key(v):
    b = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(b >> np.uint64(31), ~b & np.uint64(0xFFFFFFFF), b | np.uint64(ZERO_KEY))


def _float_of_key(k):
    return (np.asarray(k, np.uint64) & np.uint64(0x7FFFFFFF)).astype(np.uint32).view(np.float32)   # positive keys only


def _splitters(x, valid, c):
    """The fine splitters pc_sample_kernel / pc_split_kernel take for batch column c."""
    p, rows = _sample_rows(x.size, c)
    k = np.sort(_key(x[rows][valid[rows]]))
    k = k[k != ZERO_KEY]
    idx = np.minimum((np.arange(1, p, dtype=np.int64) * k.size) // p, k.size - 1)
    s = k[idx]
    return p, np.insert(s, np.searchsorted(s, ZERO_KEY), np.uint64(ZERO_KEY))


class Column:
    """A background column of n rows (some null) for batch column c, into which value sets are planted."""

    def __init__(self, n, c, seed):
        self.rng = np.random.default_rng(seed)
        self.n, self.c = n, c
        self.x = self.rng.choice(BACKGROUND, n)
        self.valid = self.rng.random(n) >= 0.03
        self.free = np.setdiff1d(np.arange(n), _sample_rows(n, c)[1])
        self.free = self.free[self.valid[self.free]]
        self.rng.shuffle(self.free)
        self.used = 0

    def plant(self, values, rows=None):
        if rows is None:
            rows = self.free[self.used:self.used + len(values)]
            self.used += len(values)
        assert len(rows) == len(values)
        self.x[rows] = values
        return rows

    def layout(self):
        """-> (fine bucket of every valid non-splitter key (-1 otherwise), coarse group of every valid key, P)"""
        p, s = _splitters(self.x, self.valid, self.c)
        k = _key(self.x)
        b = np.searchsorted(s, k, "left")
        eq = (b < s.size) & (s[np.minimum(b, s.size - 1)] == k)
        g = np.minimum(b // 32, p // 32 - 1)
        ok = self.valid & (k != ZERO_KEY)
        return np.where(ok & ~eq, b, -1), np.where(ok, g, -1), p

    def arrow(self):
        return pa.array(self.x, mask=~self.valid)


def _ranks_at(x, valid, sets):
    """1-based ranks (among the valid values) of the smallest, middle and largest value of each planted set."""
    srt = np.sort(x[valid].astype(np.float64))
    out = []
    for v in sets:
        lo, hi = np.searchsorted(srt, np.min(v), "left"), np.searchsorted(srt, np.max(v), "right")
        out += [lo + 1, (lo + hi + 1) // 2, hi]
    return out


def _check_numpy(t, names, rk, got):
    res, qv, _ = got
    for i, c in enumerate(names):
        x = np.asarray(t.column(c).drop_null())
        srt = np.sort(x.astype(np.float64))
        exp = [srt[r - 1] if r else np.nan for r in rk[i]]
        assert np.array_equal(qv[i], np.array(exp), equal_nan=True), c
        u, k = np.unique(x + np.float32(0.0), return_counts=True)
        assert res[i][2] == u.size and res[i][1] == int(k.max()), c
        assert res[i][0] == float(u[np.argmax(k)]), c


def _staged_column(c, seed):
    """n not a multiple of 4096.  A bucket of exactly STAGE_KEYS keys (with repeats), one of STAGE_KEYS + 1 distinct keys,
    and 200 keys above the top splitter, in one tile whose segment of the last group lies inside one chunk."""
    col = Column(1_000_003, c, seed)
    a = (np.float32(2) + np.float32(2 ** -22) * (1 + np.arange(STAGE_KEYS) % 4000)).astype(np.float32)
    b = (np.float32(4) + np.float32(2 ** -21) * (1 + np.arange(STAGE_KEYS + 1))).astype(np.float32)
    d = (np.float32(200) + np.float32(2 ** -16) * (1 + np.arange(200) % 64)).astype(np.float32)
    col.plant(a)
    col.plant(b)
    bucket, group, p = col.layout()
    last = group == p // 32 - 1
    # the last group's keys in group-major order: tile by tile; pick a tile whose segment (+ d) stays inside one chunk
    per_tile = np.bincount(np.nonzero(last)[0] // 4096, minlength=(col.n + 4095) // 4096)
    start = np.concatenate([[0], np.cumsum(per_tile)[:-1]])
    free_tile = col.free[col.used:] // 4096
    for t in col.rng.permutation(np.unique(free_tile)):
        rows = col.free[col.used:][free_tile == t]
        if rows.size >= d.size and start[t] // CHUNK == (start[t] + per_tile[t] + d.size - 1) // CHUNK:
            col.plant(d, np.sort(rows[:d.size]))
            break
    else:
        raise AssertionError("no tile keeps the planted keys inside one chunk")
    bucket, group, p = col.layout()
    sizes = np.bincount(bucket[bucket >= 0], minlength=p + 1)
    ka, kb, kd = (bucket[np.isin(col.x, v) & col.valid] for v in (a, b, d))
    assert np.unique(ka).size == 1 and sizes[ka[0]] == STAGE_KEYS
    assert np.unique(kb).size == 1 and sizes[kb[0]] == STAGE_KEYS + 1
    assert np.unique(kd).size == 1 and kd[0] == p, "the planted keys are above the top splitter"
    assert (sizes[ka[0] + 1:kb[0]] == 0).any(), "empty buckets between the full ones"
    assert sizes.sum() == 2 * STAGE_KEYS + 1 + d.size
    return col, [a, b, d]


def test_buckets_at_and_over_the_stage_size(monkeypatch):
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    cols = [_staged_column(c, 20 + c) for c in range(3)]
    names = ["s%d" % c for c in range(3)]
    t = pa.table({nm: col.arrow() for nm, (col, _) in zip(names, cols)})
    fr = ColumnFrame.from_arrow(t)
    rk = np.array([(_ranks_at(col.x, col.valid, sets) + [1, int(col.valid.sum())] + [0] * 16)[:16] for col, sets in cols],
                  dtype=np.int64)
    for p in (4, 12):
        got, ref = _both(monkeypatch, fr, names, rk, p)
        _check_equal(got, ref, names)
        _check_numpy(t, names, rk, got)
    # one column per batch: every batch samples its column as column 0, so the buckets differ; the results may not
    from anovos_b200 import _lib
    monkeypatch.setattr(engine, "SORT_WORKSPACE_BUDGET", _lib.lib().anv_mode_distinct_partition_workspace_bytes(1, fr.n_rows))
    assert engine._mode_distinct_batch_size(fr, len(names), _lib.lib().anv_mode_distinct_partition_workspace_bytes(1, fr.n_rows)) == 1
    _check_equal(engine.sort_mode_distinct(fr, names, rk, hll_p=12), got, names)


def _wide_column():
    """1.1 M keys in one bucket: many stage pieces, and 9 000 of its distinct keys share the top 10 bits of the class
    hash, so that class is split at levels 8, 9 and 10.  Its group spans more chunks than one window, and a bucket of
    that group small enough to be staged whole has its keys spread over all of them."""
    col = Column(3_000_017, 0, 5)
    lo, hi = int(_key(np.float32(10))[()]) + 1, int(_key(np.float32(50))[()])
    k = np.arange(lo, hi, dtype=np.uint64)
    cls = ((k * np.uint64(0x85EBCA6B)) & np.uint64(0xFFFFFFFF)) >> np.uint64(22)
    special = col.rng.choice(k[cls == 0], 9000, replace=False)
    filler = col.rng.choice(k, 220_000, replace=False)
    big = np.concatenate([special, np.repeat(filler, 5)])[:1_100_000]
    big = _float_of_key(col.rng.permutation(big))
    col.plant(big)
    _, split = _splitters(col.x, col.valid, 0)
    group_of = lambda v: int(np.searchsorted(split, _key(v), "left")) // 32
    small = None
    for a in (9, 50):                        # the keys just above a neighbouring background value, if in the same group
        v = (np.float32(a) + np.float32(2 ** -18) * (1 + np.arange(3000))).astype(np.float32)
        if group_of(v[0]) == group_of(big[0]):
            small = v
            break
    assert small is not None, "no neighbouring gap in the big bucket's group"
    col.plant(small)
    bucket, group, p = col.layout()
    sizes = np.bincount(bucket[bucket >= 0], minlength=p + 1)
    kb, ks = (bucket[np.isin(col.x, v) & col.valid] for v in (big, small))
    assert np.unique(kb).size == 1 and sizes[kb[0]] == big.size and sizes[kb[0]] > 100 * STAGE_KEYS
    assert np.unique(ks).size == 1 and sizes[ks[0]] == small.size and ks[0] // 32 == kb[0] // 32
    assert -(-int((group == kb[0] // 32).sum()) // CHUNK) > WINDOW
    return col, big, small


def test_streamed_bucket_with_class_splits_in_a_group_wider_than_one_window(monkeypatch):
    from anovos_b200.frame import ColumnFrame
    col, big, small = _wide_column()
    t = pa.table({"wide": col.arrow()})
    fr = ColumnFrame.from_arrow(t)
    rk = np.array([(_ranks_at(col.x, col.valid, [big, small, big[:1], big[-1:]]) + [0] * 16)[:16]], dtype=np.int64)
    got, ref = _both(monkeypatch, fr, ["wide"], rk, 12)
    _check_equal(got, ref, ["wide"])
    _check_numpy(t, ["wide"], rk, got)
