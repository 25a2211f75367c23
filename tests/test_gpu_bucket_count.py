"""The two-level bucket count (anv_mode_distinct_partition_hll, the default for F32 / I32 columns) against the LSD sort,
cell for cell: mode, mode_rows, distinct count, every requested rank and the HLL++ registers bit for bit - on generator
frames, int32 columns, inputs built to stress each level of the bucketing, and calls split into several batches."""
import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu


def _same(a, b):      # (mode, rows, distinct) tuples; the mode of a NaN-dominated column is NaN on both sides
    return a == b or (a[1:] == b[1:] and a[0] != a[0] and b[0] != b[0])


def _both(monkeypatch, fr, names, rk, p):
    from anovos_b200 import engine
    monkeypatch.setattr(engine, "sort_algorithm", "partition")
    got = engine.sort_mode_distinct(fr, names, rk, hll_p=p)
    monkeypatch.setattr(engine, "sort_algorithm", "lsd")
    ref = engine.sort_mode_distinct(fr, names, rk, hll_p=p)
    monkeypatch.setattr(engine, "sort_algorithm", "partition")
    return got, ref


def _check_equal(got, ref, names):
    (g, gq, gr), (r, rq, rr) = got, ref
    bad = [(n, a, b) for n, a, b in zip(names, g, r) if not _same(a, b)]
    assert not bad, bad
    assert np.array_equal(gq, rq, equal_nan=True)
    assert gr.dtype == rr.dtype and np.array_equal(gr, rr)


def _summary_ranks(fr, names):
    from anovos_b200 import engine
    from anovos_b200 import profile as P
    mom = engine.moments(fr, names)
    return np.array([engine.quantile_ranks(int(mom["n_valid"][i]), P.SUMMARY_PROBS, P.SUMMARY_EPS) for i in range(len(names))],
                    dtype=np.int64)


@pytest.mark.parametrize("p", [4, 9, 12])
def test_generator_frame_matches_the_sort(p, monkeypatch):
    """All four generator families (and their null rates) at 10 M rows."""
    from anovos_b200 import synth
    fr = synth.device_frame(10_000_000, 9, cat_every=4, seed=7)
    names = [n for n in fr.columns if fr.column(n).kind == "num"]
    assert len(names) >= 4
    _check_equal(*_both(monkeypatch, fr, names, _summary_ranks(fr, names), p), names)


def test_int32_columns_match_the_sort(monkeypatch):
    from anovos_b200.frame import ColumnFrame
    n = 3_000_017
    rng = np.random.default_rng(3)
    t = pa.table({
        "i_wide": pa.array(rng.integers(-2 ** 31, 2 ** 31 - 1, n).astype(np.int32), mask=rng.random(n) < 0.2),
        "i_small": pa.array(rng.integers(-3, 4, n).astype(np.int32)),
        "i_zipf": pa.array(np.minimum(rng.zipf(1.3, n), 2 ** 31 - 1).astype(np.int32), mask=rng.random(n) < 0.02),
        "i_mid": pa.array(rng.integers(-50_000, 50_000, n).astype(np.int32)),
        "i_extremes": pa.array(rng.choice(np.array([-2 ** 31, 2 ** 31 - 1, 0, -1, 1], np.int32), n)),
    })
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    for p in (4, 9, 12):
        _check_equal(*_both(monkeypatch, fr, names, _summary_ranks(fr, names), p), names)


def _sample_rows(n_rows, c=0):
    """Row positions pc_sample_kernel reads for batch column c (P fine splitters, 32 P samples)."""
    p = 256
    while p < 8192 and p * 4096 < n_rows:
        p <<= 1
    m = min(32 * p, n_rows)
    stride = max(n_rows // m, 1)
    i = np.arange(m, dtype=np.uint64)
    h = (i * np.uint64(0x9E3779B1) + np.uint64((c * 0x85EBCA6B) & 0xFFFFFFFF)) & np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(15)
    h = (h * np.uint64(0x2C1B3C6D)) & np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(12)
    rows = i.astype(np.int64) * stride + (h % np.uint64(stride)).astype(np.int64)
    return p, rows[rows < n_rows]


def test_adversarial_columns_match_numpy_and_the_sort(monkeypatch):
    from anovos_b200.frame import ColumnFrame
    n = 2_000_003
    rng = np.random.default_rng(11)
    p, sampled = _sample_rows(n)
    # a dense run of 150 000 distinct floats just above 1.0, on rows the splitter sample never reads: one fine bucket holds
    # them all, so its hash-table count takes many sweeps
    hidden = rng.normal(0, 100, n).astype(np.float32)
    free = np.setdiff1d(np.arange(n), sampled)
    at = rng.choice(free, 150_000, replace=False)
    hidden[at] = np.nextafter(np.float32(1.0), np.float32(2.0)) + np.arange(150_000, dtype=np.float32) * np.float32(2 ** -23)
    # one value just under the splitter frequency (n / P rows): it may stay out of the splitters and fill a bucket
    near = rng.normal(0, 1, n).astype(np.float32)
    near[rng.choice(n, int(0.9 * n / p), replace=False)] = np.float32(0.3125)
    heavy = rng.normal(5, 1, n).astype(np.float32)
    heavy[rng.random(n) < 0.25] = np.float32(-1.5)         # a splitter-equal run that the middle ranks land on
    runs = np.sort(np.repeat(rng.normal(0, 10, n // 50 + 1).astype(np.float32), 50)[:n])
    cols = {
        "hidden": pa.array(hidden),                        # first in the call: its sample rows are the ones above
        "near": pa.array(near, mask=rng.random(n) < 0.05),
        "heavy": pa.array(heavy),
        "sorted_runs": pa.array(runs),
        "nan_zero": pa.array(np.where(rng.random(n) < 0.4, np.float32(np.nan),
                                      np.where(rng.random(n) < 0.5, np.float32(-0.0), np.float32(2.5)))),
        "all_null": pa.array(np.zeros(n, np.float32), mask=np.ones(n, bool)),
    }
    t = pa.table(cols)
    fr = ColumnFrame.from_arrow(t)
    names = t.column_names
    rk = []
    for c in names:
        nv = n - t.column(c).null_count
        x = np.sort(np.asarray(t.column(c).drop_null()).astype(np.float64))
        extra = []
        if c == "heavy":                                  # first, middle and last rank of the -1.5 run
            lo, hi = np.searchsorted(x, -1.5, "left"), np.searchsorted(x, -1.5, "right")
            extra = [lo + 1, (lo + hi) // 2, hi]
        base = [1, nv, nv // 2, max(nv // 100, 1)] if nv else [0, 0, 0, 0]
        rk.append((base + extra + [0] * 16)[:12])
    rk = np.array(rk, dtype=np.int64)
    got, ref = _both(monkeypatch, fr, names, rk, 12)
    _check_equal(got, ref, names)
    res, qv, _ = got
    for i, c in enumerate(names):
        x = np.asarray(t.column(c).drop_null())
        if x.size == 0:
            assert res[i] == (None, None, 0) and np.isnan(qv[i]).all()
            continue
        srt = np.sort(x.astype(np.float64))               # NaN last
        exp = [srt[r - 1] if r else np.nan for r in rk[i]]
        assert np.array_equal(qv[i], np.array(exp), equal_nan=True), c
        u, k = np.unique(x + np.float32(0.0), return_counts=True)
        assert res[i][2] == u.size and res[i][1] == int(k.max()), c


def test_several_batches_match_one_batch(monkeypatch):
    from anovos_b200 import _lib, engine, synth
    fr = synth.device_frame(1_000_000, 10, cat_every=5, seed=3)
    names = [n for n in fr.columns if fr.column(n).kind == "num"]
    rk = _summary_ranks(fr, names)
    one = engine.sort_mode_distinct(fr, names, rk, hll_p=9)
    per_col = _lib.lib().anv_mode_distinct_partition_workspace_bytes(1, fr.n_rows)
    monkeypatch.setattr(engine, "SORT_WORKSPACE_BUDGET", 3 * per_col)    # 3 columns per batch
    assert engine._mode_distinct_batch_size(fr, len(names), per_col) == 3
    many = engine.sort_mode_distinct(fr, names, rk, hll_p=9)
    _check_equal(many, one, names)


def test_empty_frame():
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    t = pa.table({"f": pa.array([], pa.float32()), "i": pa.array([], pa.int32())})
    fr = ColumnFrame.from_arrow(t)
    res, qv, regs = engine.sort_mode_distinct(fr, ["f", "i"], np.zeros((2, 3), np.int64), hll_p=9)
    assert res == [(None, None, 0), (None, None, 0)]
    assert np.isnan(qv).all() and not regs.any()
