"""Row-level quality checks on the GPU (csrc/rows.cu): duplicate_detection and nullRows_detection against the notebook
tables, the reference unit tests and the oracle (oracle/row_checks.py), on seeded frames built to hit the kernels' edges."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from golden_util import shown_close
from oracle import api as O
from oracle import row_checks as RC

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import anovos.data_analyzer.quality_checker as qc          # noqa: E402
from anovos_b200 import engine, synth                      # noqa: E402
from anovos_b200.frame import ColumnFrame, _pack_validity   # noqa: E402
from anovos_b200.partitioned import PartitionedFrame       # noqa: E402
from anovos_b200.data_analyzer.quality_checker import _canonical_codes   # noqa: E402


def _bits(words, n):
    return np.unpackbits(words.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)


def _same_table(a, b):
    """Equal names, types, nulls and values (floats by their bits: NaN payloads included)."""
    assert a.column_names == b.column_names and a.num_rows == b.num_rows
    for name in a.column_names:
        x, y = a.column(name).combine_chunks(), b.column(name).combine_chunks()
        assert x.type == y.type, name
        vx, vy = np.asarray(x.is_valid()), np.asarray(y.is_valid())
        assert np.array_equal(vx, vy), name
        if pa.types.is_floating(x.type):
            bx = x.fill_null(0).to_numpy().view(np.uint32 if x.type == pa.float32() else np.uint64)
            by = y.fill_null(0).to_numpy().view(bx.dtype)
            assert np.array_equal(bx[vx], by[vy]), name
        else:
            assert x.to_pylist() == y.to_pylist(), name


def _check_table(got, cell):
    assert list(got.columns) == cell["columns"]
    assert len(got) == len(cell["rows"])
    for r, exp in zip(got.values.tolist(), cell["rows"]):
        for g, e in zip(r, exp):
            assert shown_close(g, e), (r, exp)


@pytest.mark.parametrize("cell,kw", [
    (7, {}), (8, dict(list_of_cols="all", drop_cols=["ifa"])),
    (9, dict(list_of_cols=["age", "sex", "race", "workclass", "fnlwgt"])),
    (10, dict(list_of_cols=["age", "sex", "race", "workclass", "fnlwgt"], treatment=True))])
def test_duplicate_detection_notebook(income, nb_quality, cell, kw):
    odf, stats = qc.duplicate_detection(None, income, print_impact=True, **kw)
    _check_table(stats.toPandas(), nb_quality[cell])
    if cell == 10:
        exp = RC.duplicate_detection(income, **kw)
        assert odf.count() == 30601
        _same_table(odf.to_arrow(), exp)


@pytest.mark.parametrize("cell,kw", [
    (12, {}), (13, dict(list_of_cols="all", drop_cols=["age"], treatment_threshold=0.4)),
    (14, dict(list_of_cols=["age", "sex", "race", "workclass", "fnlwgt"])),
    (15, dict(list_of_cols="all", treatment=True, treatment_threshold=0.75))])
def test_nullRows_detection_notebook(income, nb_quality, cell, kw):
    odf, stats = qc.nullRows_detection(None, income, **kw)
    _check_table(stats.toPandas(), nb_quality[cell])
    exp_odf, _ = RC.nullRows_detection(income, **kw)
    assert odf.count() == exp_odf.num_rows


def test_reference_unit_tests():
    t = O.table_from_rows([("27520a", 51, 9000, "HS-grad"), ("10a", 42, 7000, "Postgrad"), ("11a", 35, None, None),
                           ("1100b", 23, 6000, "HS-grad")], ["ifa", "age", "income", "education"])
    odf, st = qc.nullRows_detection(None, t, treatment=True, treatment_threshold=0.4)
    st = st.toPandas().set_index("null_cols_count")
    assert odf.count() == 3
    assert (st.loc[0, "row_count"], st.loc[0, "row_pct"], st.loc[0, "treated"]) == (3, 0.75, 0)
    assert (st.loc[2, "row_count"], st.loc[2, "row_pct"], st.loc[2, "treated"]) == (1, 0.25, 1)
    t1 = O.table_from_rows([("27520a", 51, 9000, "HS-grad"), ("10a", 42, 7000, "Postgrad"), ("10a", 42, 7000, "Postgrad"),
                            ("11a", 35, None, None), ("1100b", 23, 6000, "HS-grad")], ["ifa", "age", "income", "education"])
    odf, st = qc.duplicate_detection(None, t1, treatment=True, print_impact=True)
    v = dict(st.toPandas().values.tolist())
    assert odf.count() == 4
    assert (v["rows_count"], v["unique_rows_count"], v["duplicate_rows"], v["duplicate_pct"]) == (5, 4, 1, 0.20)


# ---- seeded frames -------------------------------------------------------------------------------------------------

_NAN_PAYLOADS32 = np.array([0x7fc00000, 0xffc00000, 0x7f800001, 0xff812345, 0x7fffffff], np.uint32).view(np.float32)
_NAN_PAYLOADS64 = np.array([0x7ff8000000000000, 0xfff8000000000000, 0x7ff0000000000001, 0xfff123456789abcd],
                           np.uint64).view(np.float64)


def _seeded(n, seed, null_rate, n_base=None, garbage_under_nulls=True):
    """A frame with all four dtypes and two string columns (one with a repeated dictionary string).  Rows are drawn
    from n_base base rows (planted duplicates); some copies differ in one column only; floats take NaN payloads, -0.0
    and 0.0.  -> (ColumnFrame, pyarrow Table holding the same values)."""
    rng = np.random.default_rng(seed)
    n_base = n_base or max(1, n // 3)
    base = {
        "f32": rng.choice(np.concatenate([rng.normal(0, 1, 6).astype(np.float32), _NAN_PAYLOADS32,
                                          np.float32([0.0, -0.0])]), n_base),
        "f64": rng.choice(np.concatenate([rng.normal(0, 1, 6), _NAN_PAYLOADS64, [0.0, -0.0]]), n_base),
        "i32": rng.integers(-3, 3, n_base).astype(np.int32),
        "i64": rng.integers(-(1 << 40), (1 << 40), n_base) // (1 << 38),
        "s": rng.integers(0, 5, n_base).astype(np.int32),
        "d": rng.integers(0, 4, n_base).astype(np.int32),
    }
    pick = rng.integers(0, n_base, n)
    vals = {k: v[pick].copy() for k, v in base.items()}
    one = rng.random(n) < 0.1                         # copies that differ in one column only
    col_of = rng.integers(0, len(vals), n)
    for j, k in enumerate(vals):
        m = one & (col_of == j)
        if k == "f32":
            vals[k][m] = np.float32(7.5)
        elif k == "f64":
            vals[k][m] = 7.5
        else:
            vals[k][m] = (vals[k][m] + 1) % (5 if k == "s" else 4) if k in ("s", "d") else vals[k][m] + 1
    valid = {k: rng.random(n) >= null_rate for k in vals}
    if null_rate > 0:
        valid["i32"][: min(n, 3)] = False                  # a null over 0 ...
        vals["i32"][: min(n, 3)] = 0
    if garbage_under_nulls:
        for k in vals:                                     # ... and nulls over arbitrary data
            g = ~valid[k]
            if k in ("s", "d"):
                vals[k][g] = rng.integers(0, 4, int(g.sum())).astype(np.int32)
            else:
                vals[k][g] = rng.integers(-9, 9, int(g.sum())).astype(vals[k].dtype)
    dic_s = ["a", "b", "c", "d", "e"]
    dic_d = ["x", "y", "x", "z"]                           # "x" twice: codes 0 and 2 are one value
    data = {}
    for k, v in vals.items():
        vw = None if valid[k].all() else _pack_validity(valid[k])
        if k == "s":
            data[k] = (torch.from_numpy(v).cuda(), None if vw is None else torch.from_numpy(vw).cuda(), dic_s)
        elif k == "d":
            data[k] = (torch.from_numpy(v).cuda(), None if vw is None else torch.from_numpy(vw).cuda(), dic_d)
        else:
            data[k] = (torch.from_numpy(v).cuda(), None if vw is None else torch.from_numpy(vw).cuda())
    fr = ColumnFrame.from_tensors(data)
    arrays = []
    for k, v in vals.items():
        mask = ~valid[k]
        if k in ("s", "d"):
            dic = dic_s if k == "s" else dic_d
            arrays.append(pa.array([dic[c] for c in v], pa.string(), mask=mask))
        else:
            arrays.append(pa.array(v, mask=mask))
    return fr, pa.table(arrays, names=list(vals))


SIZES = [1, 31, 32, 33, 4095, 4097, 400_003]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("null_rate", [0.0, 0.3, 1.0])
def test_row_distinct_matches_pandas(n, null_rate):
    fr, t = _seeded(n, seed=n + int(null_rate * 10), null_rate=null_rate)
    cols = fr.columns
    exp = RC.first_occurrence(t, cols)
    # hash widths of 1, 4 and 8 bits send (nearly) every row through the comparison path, whose rounds grow with the
    # distinct rows per hash prefix: the large frame keeps 8 bits (a few hundred per prefix)
    for hb in ((0, 1, 4, 8) if n < 10_000 else (0, 8)):
        nd, first = engine.row_distinct(_canonical_codes(fr, cols), cols, hash_bits=hb)
        assert nd == int(exp.sum()), (n, null_rate, hb)
        assert np.array_equal(_bits(first, n), exp), (n, null_rate, hb)


@pytest.mark.parametrize("n", [33, 4097, 400_003])
def test_row_distinct_mostly_unique_rows(n):
    rng = np.random.default_rng(n)
    x = rng.normal(0, 1, n)
    x[rng.integers(0, n, n // 10)] = x[0]
    y = rng.integers(0, 3, n)
    fr = ColumnFrame.from_tensors({"x": torch.from_numpy(x).cuda(), "y": torch.from_numpy(y).cuda()})
    t = pa.table({"x": x, "y": y})
    exp = RC.first_occurrence(t, ["x", "y"])
    for hb in ((0, 8) if n > 10_000 else (0, 1, 4, 8)):
        nd, first = engine.row_distinct(fr, ["x", "y"], hash_bits=hb)
        assert nd == int(exp.sum()) and np.array_equal(_bits(first, n), exp), hb


@pytest.mark.parametrize("n", [33, 4097, 400_003])
@pytest.mark.parametrize("null_rate", [0.0, 0.3, 1.0])
def test_treated_frames_equal_the_oracle(n, null_rate):
    fr, t = _seeded(n, seed=7 * n, null_rate=null_rate, garbage_under_nulls=False)
    cols = ["f64", "i32", "s", "d"]
    odf, st = qc.duplicate_detection(None, fr, list_of_cols=cols, treatment=True, print_impact=True)
    exp_odf, exp_st = RC.duplicate_detection(t, list_of_cols=cols, treatment=True, print_impact=True)
    assert st.toPandas().values.tolist() == exp_st.values.tolist()
    _same_table(odf.to_arrow(), exp_odf)
    for thr in (0.0, 0.3, 0.5, 1.0):
        odf, st = qc.nullRows_detection(None, fr, treatment=True, treatment_threshold=thr)
        exp_odf, exp_st = RC.nullRows_detection(t, treatment=True, treatment_threshold=thr)
        pd.testing.assert_frame_equal(st.toPandas(), exp_st, check_dtype=False)
        _same_table(odf.to_arrow(), exp_odf)


def test_nullRows_partitioned_equals_resident(income):
    whole = RC.nullRows_detection(income, treatment=True, treatment_threshold=0.3)
    pf = PartitionedFrame.from_frame(income, 4096)
    odf, st = qc.nullRows_detection(None, pf, treatment=True, treatment_threshold=0.3)
    pd.testing.assert_frame_equal(st.toPandas(), whole[1], check_dtype=False)
    assert odf.count() == whole[0].num_rows
    assert sum(ch.n_rows for ch in odf.chunks()) == whole[0].num_rows
    _, st2 = qc.nullRows_detection(None, income, treatment=True, treatment_threshold=0.3)
    pd.testing.assert_frame_equal(st.toPandas(), st2.toPandas())
    with pytest.raises(NotImplementedError):
        qc.duplicate_detection(None, pf, print_impact=True)


def test_row_distinct_20m_rows_four_byte_index():
    n = 20_000_000
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randint(0, 1000, (n,), device="cuda", dtype=torch.int32, generator=g)
    b = torch.randint(0, 50, (n,), device="cuda", dtype=torch.int64, generator=g)
    fr = ColumnFrame.from_tensors({"a": a, "b": b})
    exp_first = np.ones(n, bool)
    key = a.cpu().numpy().astype(np.int64) * 50 + b.cpu().numpy()
    _, idx = np.unique(key, return_index=True)
    exp_first[:] = False
    exp_first[idx] = True
    nd, first = engine.row_distinct(fr, ["a", "b"])
    assert nd == len(idx)
    assert np.array_equal(_bits(first, n), exp_first)
    hist, keep = engine.row_null_counts(fr, ["a", "b"], 0)
    assert hist.tolist() == [n, 0, 0] and _bits(keep, n).all()


def test_generator_frame_10m_x_12_with_planted_duplicates():
    n, c = 10_000_000, 12
    fr0 = synth.device_frame(n, c, cat_every=4)
    rng = np.random.default_rng(11)
    src = np.arange(n)
    dup = rng.random(n) < 0.3
    src[dup] = (rng.random(int(dup.sum())) * np.flatnonzero(dup)).astype(np.int64)   # an earlier row
    idx = torch.from_numpy(src).cuda()
    data, planes = {}, []
    for j, name in enumerate(fr0.columns):
        col = fr0.column(name)
        d, v = col.device()
        vb = None
        if v is not None:
            vb = _bits(v, n)[src]
        if col.dictionary is not None:
            hv, hm, dic = synth.host_codes(n, j, cat_every=4)
            hv = hv.astype(np.int32)
        else:
            hv, hm = synth.host_column(n, j, cat_every=4)
        assert np.array_equal(d.cpu().numpy(), hv) and (v is None or np.array_equal(_bits(v, n), hm))
        vw = None if vb is None else torch.from_numpy(_pack_validity(vb)).cuda()
        data[name] = (d[idx].contiguous(), vw, col.dictionary) if col.dictionary is not None else (d[idx].contiguous(), vw)
        # normalised image of the twin: null flag + value bits (0 under nulls; the generators make no NaN)
        hm = hm if v is not None else np.ones(n, bool)
        bits = hv.view(np.int32).astype(np.int64) if hv.dtype == np.float32 else hv.astype(np.int64)
        planes += [np.where(hm, bits, 0)[src], hm[src].astype(np.int64)]
    fr = ColumnFrame.from_tensors(data)
    exp = ~pd.DataFrame(np.stack(planes, axis=1)).duplicated(keep="first").to_numpy()
    nd, first = engine.row_distinct(fr, fr.columns)
    assert nd == int(exp.sum())
    assert np.array_equal(_bits(first, n), exp)
