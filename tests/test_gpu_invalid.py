"""invalidEntries_detection on the GPU: anv_flag_members bit for bit against NumPy (np.isin on canonical bits plus per-entry
counts) on adversarial columns of every dtype, and the API against the oracle (tests/invalid_oracle.py) on the income
table, at 10 M rows, on chunked frames and on row slabs of two ranks, and against the notebook and unit-test pins."""
import json
import os
import socket
import warnings

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

import invalid_oracle as O
from test_invalid_cpu import UNIT_ROWS, entry_set, same_tables

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _words(valid):
    bits = np.packbits(np.asarray(valid, bool), bitorder="little")
    return np.concatenate([bits, np.zeros((-len(bits)) % 4, np.uint8)]).view(np.int32)


def _canon_bits(a):
    """Values -> integer bits with every NaN payload as the one quiet NaN (the kernel's equality)."""
    a = np.asarray(a)
    if a.dtype.kind != "f":
        return a.astype(np.int64)
    u = np.uint32 if a.itemsize == 4 else np.uint64
    b = a.view(u).copy()
    b[np.isnan(a)] = u(0x7FC00000) if a.itemsize == 4 else u(0x7FF8000000000000)
    return b.astype(np.uint64).view(np.int64)


def _expected(vals, valid, table):
    vb, tb = _canon_bits(vals), _canon_bits(table)
    hit = valid & np.isin(vb, tb)
    counts = np.array([int(np.sum(hit & (vb == t))) for t in tb], np.uint64) if len(tb) <= 4096 else None
    if counts is None:
        order = np.argsort(tb)
        pos = np.searchsorted(tb[order], vb[hit])
        counts = np.zeros(len(tb), np.uint64)
        np.add.at(counts, order[pos], 1)
    return counts, hit


def _table_and_values(kind, size, n, rng):
    from anovos_b200.shared.invalid_rules import sort_table
    if kind in ("i32", "code"):
        pool = np.concatenate([np.array([-(1 << 31), (1 << 31) - 1, -1, 0, 1], np.int32),
                               rng.integers(-(1 << 31), (1 << 31) - 1, size * 2 + 8, dtype=np.int64).astype(np.int32)])
        if kind == "code":
            pool = np.arange(size * 2 + 8, dtype=np.int32)
    elif kind == "i64":
        pool = np.concatenate([np.array([-(1 << 63), (1 << 63) - 1, -1, 0, 1], np.int64),
                               rng.integers(-(1 << 63), (1 << 63) - 1, size * 2 + 8, dtype=np.int64)])
    else:
        dt, u = (np.float32, np.uint32) if kind == "f32" else (np.float64, np.uint64)
        nan_payloads = (np.array([0x7FC00000, 0xFFC00001, 0x7F800001, 0x7FFFFFFF], np.uint32) if kind == "f32" else
                        np.array([0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000001, 0x7FFFFFFFFFFFFFFF],
                                 np.uint64)).astype(u).view(dt)
        special = np.array([0.0, -0.0, np.inf, -np.inf, 111.0, -1.5], dt)
        pool = np.concatenate([nan_payloads, special, (rng.standard_normal(size * 2 + 8) * 1e3).astype(dt)])
    table = sort_table(pool[rng.permutation(len(pool))])[:size]
    if kind in ("f32", "f64") and size >= 2 and not np.isnan(table).any():
        table = sort_table(np.concatenate([table[:-1], pool[:1]]))          # a NaN key in every float table of 2+
    vals = pool[rng.integers(0, len(pool), n)]
    if kind in ("f32", "f64"):
        nan_rows = rng.random(n) < 0.05
        vals[nan_rows] = pool[rng.integers(0, 4, int(nan_rows.sum()))]    # every NaN payload counts as one key
    return table, vals


@pytest.mark.parametrize("n", [1, 31, 33, 65_599, 100_001])
@pytest.mark.parametrize("size", ["1", "156", "332", "S-1", "S", "S+1", "100001"])
@pytest.mark.parametrize("kind", ["i32", "i64", "f32", "f64", "code"])
def test_flag_members_bit_exact(kind, size, n):
    import torch
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    S = engine.flag_smem_keys()
    size = {"S-1": S - 1, "S": S, "S+1": S + 1}.get(size) or int(size)
    rng = np.random.default_rng([n, size, len(kind)])
    table, vals = _table_and_values(kind, size, n, rng)
    valid = rng.random(n) > 0.2
    lead = valid.copy()
    lead[:min(n, 66_000)] = False                                  # leading all-null tiles
    dic = ["k%d" % i for i in range(size * 2 + 8)] if kind == "code" else None
    cols = {}
    for name, ok in (("some", valid), ("free", None), ("lead", lead), ("none", np.zeros(n, bool))):
        t = torch.from_numpy(np.ascontiguousarray(vals)).cuda()
        cols[name] = (t, None if ok is None else torch.from_numpy(_words(ok)).cuda()) + ((dic,) if dic else ())
    fr = ColumnFrame.from_tensors(cols)
    names = list(cols)
    for want in (False, True):
        counts, bitmaps = engine.flag_members(fr, names, [table] * len(names), want)
        for name, ok, cnt, bm in zip(names, (valid, None, lead, np.zeros(n, bool)), counts, bitmaps):
            ok = np.ones(n, bool) if ok is None else ok
            exp_counts, hit = _expected(vals, ok, table)
            assert np.array_equal(cnt, exp_counts), (name, want)
            if want:
                got = bm.cpu().numpy()
                assert np.array_equal(got, _words(ok & ~hit)[:len(got)]), name
            else:
                assert bm is None


def test_flag_members_column_blocks():
    import torch
    from anovos_b200 import _lib, engine
    from anovos_b200.frame import ColumnFrame
    n_cols = _lib.MAX_LAUNCH_COLS + 3
    n = 97
    rng = np.random.default_rng(7)
    vals = rng.integers(0, 50, n).astype(np.int32)
    t = torch.from_numpy(vals).cuda()
    fr = ColumnFrame.from_tensors({"c%d" % i: t for i in range(n_cols)})
    table = np.array([3, 11, 111], np.int32)
    counts, bitmaps = engine.flag_members(fr, fr.columns, [table] * n_cols, True)
    exp, hit = _expected(vals, np.ones(n, bool), table)
    assert len(counts) == n_cols and all(np.array_equal(c, exp) for c in counts)
    w = _words(~hit)
    assert np.array_equal(bitmaps[0].cpu().numpy(), w) and np.array_equal(bitmaps[-1].cpu().numpy(), w)


def test_empty_table_is_not_launched():
    import torch
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    fr = ColumnFrame.from_tensors({"a": torch.arange(10, dtype=torch.int32).cuda()})
    before = engine.launch_count
    counts, bitmaps = engine.flag_members(fr, ["a"], [np.zeros(0, np.int32)], True)
    assert engine.launch_count == before and len(counts[0]) == 0 and bitmaps == [None]


# ---- API against the oracle -------------------------------------------------------------------------

def _product(table_or_frame, **kw):
    from anovos.data_analyzer.quality_checker import invalidEntries_detection
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        odf, p = invalidEntries_detection(None, table_or_frame, **kw)
    if getattr(odf, "is_partitioned", False):
        odf = pa.concat_tables([ch.to_arrow() for ch in odf.chunks()])
    else:
        odf = odf.to_arrow()
    return odf, p.toPandas()


def _same_print(got, exp):
    assert got["attribute"].tolist() == exp["attribute"].tolist()
    assert got["invalid_count"].tolist() == exp["invalid_count"].tolist()
    assert got["invalid_pct"].tolist() == exp["invalid_pct"].tolist()
    assert [entry_set(s) for s in got["invalid_entries"]] == [entry_set(s) for s in exp["invalid_entries"]]


MODES = [dict(), dict(detection_type="manual", invalid_entries=["self-emp.*", "1[0-9]"]),
         dict(detection_type="manual", invalid_entries=["mar"], partial_match=True, valid_entries=["[a-z -]+"]),
         dict(detection_type="both", valid_entries=["self-emp.*", "[0-9]+"]),
         dict(list_of_cols=["age", "logfnl", "latitude", "workclass", "capital-gain"], detection_type="both",
              invalid_entries=["4.*"], partial_match=True)]


@pytest.mark.parametrize("kw", MODES)
def test_income_modes_match_oracle(income, kw):
    got_t, got = _product(income, **dict(kw))
    exp_t, exp, _ = O.invalidEntries_detection(income, **dict(kw))
    _same_print(got, exp)


@pytest.mark.parametrize("method", ["null_replacement", "column_removal", "MMM"])
@pytest.mark.parametrize("output_mode", ["replace", "append"])
@pytest.mark.parametrize("threshold", [None, 0.001])
def test_income_treatments_match_oracle(income, method, output_mode, threshold):
    import imputation_oracle as IO
    if method == "column_removal" and not threshold:
        pytest.skip("column_removal needs a threshold (tested on the CPU)")
    cols = ["age", "sex", "race", "workclass", "logfnl", "capital-gain", "empty"]
    cfg = {"treatment_threshold": threshold} if threshold else {}
    kw = dict(list_of_cols=cols, treatment=True, treatment_method=method, output_mode=output_mode)

    def impute(t, sub, **c):
        return IO.imputation_MMM(t, sub, **c)[0]
    if method == "MMM" and output_mode == "append" and not threshold:
        # <c>_invalid of a column without invalid rows was dropped again, and imputation_MMM is handed its name
        with pytest.raises(TypeError):
            O.invalidEntries_detection(income, impute=impute, **kw)
        with pytest.raises(TypeError):
            _product(income, **kw)
        return
    got_t, got = _product(income, treatment_configs=dict(cfg), **kw)
    exp_t, exp, _ = O.invalidEntries_detection(income, treatment_configs=dict(cfg), impute=impute, **kw)
    _same_print(got, exp)
    same_tables(got_t, exp_t)


def _big_frame(n):
    rng = np.random.default_rng(5)
    words = np.array(["ok", "?", "aaa", "abc", "Never", " n/a ", "x", "Z"], object)
    return pa.table({
        "i": pa.array(rng.choice(np.array([5, 111, -999, 123, 124, 77, 2 ** 31 - 1], np.int32), n),
                      mask=rng.random(n) < 0.1),
        "b": pa.array(rng.choice(np.array([1111111111111, 6, -6, 4567, 2 ** 62], np.int64), n)),
        "f": pa.array(rng.choice(np.array([np.nan, 0.0, -0.0, np.inf, -np.inf, 111.0, 2.5], np.float32), n),
                      mask=rng.random(n) < 0.05),
        "s": pa.array(rng.choice(words, n), mask=rng.random(n) < 0.1).dictionary_encode()})


def _distinct_oracle(table, cols):
    """The oracle's summary computed over distinct values (the row-by-row oracle at 10 M rows is too slow)."""
    rows = []
    for c in cols:
        groups = {}
        for v in table.column(c).to_pylist():
            if v is not None:
                groups.setdefault(repr(v) if isinstance(v, float) else v, [v, 0])[1] += 1
        flagged = [(v, k) for v, k in groups.values() if O.detect(v) == 1]
        cnt = sum(k for _, k in flagged)
        rows.append([c, "|".join(dict.fromkeys(str(v) for v, _ in flagged)), cnt, round(cnt / table.num_rows, 4)])
    return pd.DataFrame(rows, columns=O.PRINT_COLS)


def test_ten_million_rows_match_distinct_oracle():
    n = 10_000_000
    t = _big_frame(n)
    got_t, got = _product(t, list_of_cols=["i", "b", "f", "s"], treatment=True)
    _same_print(got, _distinct_oracle(t, ["i", "b", "f", "s"]))
    small = t.slice(0, 200_000)
    g2, p2 = _product(small, list_of_cols=["i", "b", "f", "s"], treatment=True)
    e2, ep2, _ = O.invalidEntries_detection(small, list_of_cols=["i", "b", "f", "s"], treatment=True)
    _same_print(p2, ep2)
    same_tables(g2, e2)
    assert got_t.column_names == ["i", "b", "f", "s"]
    for c in ("i", "b", "f", "s"):                 # null counts of the treated columns = old nulls + flagged rows
        row = got[got["attribute"] == c].iloc[0]
        assert got_t.column(c).null_count == t.column(c).null_count + row["invalid_count"]


@pytest.mark.parametrize("kw", [dict(treatment=True), dict(treatment=True, output_mode="append"),
                                dict(detection_type="both", valid_entries=["[a-z]+"], treatment=True)])
def test_chunked_frames_match_resident(income, kw):
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.partitioned import PartitionedFrame
    cols = ["age", "sex", "race", "workclass", "logfnl", "capital-gain"]
    fr = ColumnFrame.from_arrow(income)
    whole_t, whole = _product(fr, list_of_cols=cols, **kw)
    parts_t, parts = _product(PartitionedFrame.from_frame(fr, 4_096), list_of_cols=cols, **kw)
    pd.testing.assert_frame_equal(whole, parts)
    assert whole_t.equals(parts_t)


# ---- two ranks: row slabs -------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _slab_worker(rank, world, port, ret):
    import pyarrow.parquet as pq
    import torch.distributed as dist
    from anovos.data_analyzer.quality_checker import invalidEntries_detection
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.partitioned import PartitionedFrame
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    t = pq.read_table(os.path.join(GOLDEN, "income.parquet"))
    cut = 16_384
    # one dictionary in every slab: build the frame from the whole table's dictionaries
    whole = ColumnFrame.from_arrow(t)
    fr = whole.slice_rows(0, cut) if rank == 0 else whole.slice_rows(cut, t.num_rows)
    parts = PartitionedFrame.from_frame(fr, 4_096, group=True)
    cols = ["age", "sex", "race", "workclass", "capital-gain"]
    out = {}
    odf, p = invalidEntries_detection(None, parts, list_of_cols=cols, treatment=True)
    out["print"] = p.toPandas().to_dict("list")
    out["nulls"] = {c: sum(ch.n_rows - int(ch.valid_mask(c).sum()) for ch in odf.chunks()) for c in cols}
    try:
        invalidEntries_detection(None, parts, list_of_cols=["logfnl"])
        out["float"] = "ran"
    except NotImplementedError as e:
        out["float"] = "NotImplementedError" if "repartition_to_columns" in str(e) else str(e)
    ret[rank] = out
    dist.destroy_process_group()


def test_two_ranks_row_slabs(income):
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ret = mp.get_context("spawn").Manager().dict()
    mp.spawn(_slab_worker, args=(world, port, ret), nprocs=world, join=True)
    a, b = ret[0], ret[1]
    assert repr(a["print"]) == repr(b["print"])
    cols = ["age", "sex", "race", "workclass", "capital-gain"]
    _, exp, _ = O.invalidEntries_detection(income, list_of_cols=cols)
    _same_print(pd.DataFrame(a["print"]), exp)
    for c in cols:
        whole_nulls = income.column(c).null_count + int(exp.loc[exp["attribute"] == c, "invalid_count"].iloc[0])
        assert a["nulls"][c] + b["nulls"][c] == whole_nulls, c
    assert a["float"] == b["float"] == "NotImplementedError"


# ---- pins -----------------------------------------------------------------------------------------

def test_unit_test_pins():
    t = pa.table({"ifa": ["27520a", "10a", "10a", "11a", "1100b"], "age": pa.array([51, 42, 9999, 35, 23], pa.int64()),
                  "income": pa.array([9000, 7000, 7000, None, 6000], pa.int64()),
                  "education": ["HS-grad", "Postgrad", "Postgrad", ":", "HS-grad"]})
    assert t.num_rows == len(UNIT_ROWS)
    odf, p = _product(t, treatment=True)
    assert odf.num_rows == 5
    r = p.set_index("attribute")
    assert r.loc["age", "invalid_count"] == 1 and r.loc["age", "invalid_pct"] == 0.2
    assert r.loc["education", "invalid_count"] == 1 and r.loc["education", "invalid_pct"] == 0.2


def test_notebook_pins(income):
    quality = {t["code_cell"]: t for t in json.load(open(os.path.join(GOLDEN, "notebook_quality.json")))}
    shown = json.load(open(os.path.join(GOLDEN, "notebook_invalid.json")))
    _, p = _product(income)                                                   # example 1
    got = {r["attribute"]: r for r in p.to_dict("records")}
    for a, e, cnt, pct in quality[47]["rows"]:
        assert entry_set(got[a]["invalid_entries"]) == entry_set(e) and got[a]["invalid_count"] == int(cnt)
        assert abs(got[a]["invalid_pct"] - float(pct)) < 1e-12
    _, p = _product(income, list_of_cols="workclass", detection_type="both", valid_entries=["self-emp.*"])
    (a, e, cnt, pct), = shown[0]["rows"]                                      # example 4
    assert entry_set(p["invalid_entries"][0]) == entry_set(e) and p["invalid_count"][0] == int(cnt) == 28902
    assert p["invalid_pct"][0] == float(pct) == 0.8876
    cols = ["age", "sex", "race", "workclass", "logfnl"]                      # example 5, replace
    odf, _ = _product(income, list_of_cols=cols, treatment=True, print_impact=True)
    after = dict(zip(shown[3]["columns"], shown[3]["rows"][0]))
    for c in cols:
        assert odf.num_rows - odf.column(c).null_count == int(after[c]), c
    cols = ["sex", "race", "workclass"]                                       # example 5, append
    odf, _ = _product(income, list_of_cols=cols, treatment=True, output_mode="append")
    after = dict(zip(shown[6]["columns"], shown[6]["rows"][0]))
    for c in cols:
        assert odf.num_rows - odf.column(c + "_invalid").null_count == int(after[c + "_invalid"]), c


def test_default_config_runs(income):
    from anovos.data_analyzer.quality_checker import invalidEntries_detection
    odf, p = invalidEntries_detection(None, income, list_of_cols="all", drop_cols=["ifa"], treatment=True,
                                      output_mode="replace")
    assert len(p.toPandas()) == 17 and odf.count() == income.num_rows
