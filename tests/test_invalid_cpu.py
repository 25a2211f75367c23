"""invalidEntries_detection without a GPU:
  - the oracle (tests/invalid_oracle.py) against the reference's unit test and the notebook tables of
    notebook_quality.json (code cells 47-49);
  - the rules of shared/invalid_rules.py against the reference's `detect`: the closed-form int32 / int64 tables over a
    dense range, around every member and at the dtype extremes; NaN / +-0.0 / +-inf verdicts;
  - the product's host layer (argument errors, the treatment_threshold pop, column order, summary table, treated frames
    and chunked frames) against the oracle, with anv_flag_members replaced by tests/invalid_stand_in.py."""
import json
import math
import os
import warnings

import numpy as np
import pyarrow as pa
import pytest

import invalid_oracle as O
import invalid_stand_in
from anovos_b200.shared import invalid_rules as R

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
UNIT_ROWS = [("27520a", 51, 9000, "HS-grad"), ("10a", 42, 7000, "Postgrad"), ("10a", 9999, 7000, "Postgrad"),
             ("11a", 35, None, ":"), ("1100b", 23, 6000, "HS-grad")]


def unit_table():
    """test_quality_checker.py:192-249: createDataFrame of Python ints gives bigint columns."""
    c = list(zip(*UNIT_ROWS))
    return pa.table({"ifa": list(c[0]), "age": pa.array(c[1], pa.int64()), "income": pa.array(c[2], pa.int64()),
                     "education": list(c[3])})


def entry_set(s):
    return set(s.split("|")) if s else set()


def same_tables(got, exp):
    assert got.column_names == exp.column_names
    for c in exp.column_names:
        g, e = got.column(c).combine_chunks(), exp.column(c).combine_chunks()
        if pa.types.is_dictionary(g.type):
            g = g.cast(g.type.value_type)
        if pa.types.is_dictionary(e.type):
            e = e.cast(e.type.value_type)
        if pa.types.is_large_string(e.type):
            e = e.cast(pa.string())
        assert g.type == e.type, (c, g.type, e.type)
        assert [repr(x) for x in g.to_pylist()] == [repr(x) for x in e.to_pylist()], c


# ---- the oracle against the pins ---------------------------------------------------------------------------------

def test_oracle_unit_test():
    odf, p, _ = O.invalidEntries_detection(unit_table(), treatment=True)
    assert odf.num_rows == 5
    r = p.set_index("attribute")
    assert (r.loc["age", "invalid_count"], r.loc["age", "invalid_pct"]) == (1, 0.2)
    assert (r.loc["education", "invalid_count"], r.loc["education", "invalid_pct"]) == (1, 0.2)


def _quality(cell):
    return {t["code_cell"]: t for t in json.load(open(os.path.join(GOLDEN, "notebook_quality.json")))}[cell]


def _kwargs_of(cell):
    return {47: dict(), 48: dict(list_of_cols=["age", "sex", "race", "workclass", "logfnl"]),
            49: dict(list_of_cols="workclass", detection_type="manual", invalid_entries=["self-emp.*"],
                     treatment_method="null_replacement")}[cell]


def check_print(got, table):
    rows = {r["attribute"]: r for r in got.to_dict("records")}
    assert set(rows) == {r[0] for r in table["rows"]}
    for a, e, cnt, pct in table["rows"]:
        assert entry_set(rows[a]["invalid_entries"]) == entry_set(e), a
        assert rows[a]["invalid_count"] == int(cnt), a
        assert abs(rows[a]["invalid_pct"] - float(pct)) < 1e-12, a


@pytest.mark.parametrize("cell", [47, 48, 49])
def test_oracle_notebook_tables(income, cell):
    _, p, _ = O.invalidEntries_detection(income, **_kwargs_of(cell))
    check_print(p, _quality(cell))


# ---- the rules against the reference's detect ---------------------------------------------------------------------

def _ref_flag(x):
    return O.detect(x) == 1


def test_closed_form_tables_sizes():
    assert len(R.AUTO_INT32) == 156 and len(R.AUTO_INT64) == 332
    assert np.all(np.diff(R.AUTO_INT64) > 0) and np.all(np.diff(R.AUTO_INT32.astype(np.int64)) > 0)


def test_closed_form_int_tables_dense_range():
    members = set(R.AUTO_INT_VALUES)
    bad = [x for x in range(-1_000_000, 1_000_001) if _ref_flag(x) != (x in members)]
    assert not bad, bad[:10]


def test_closed_form_int_tables_neighbours_and_extremes():
    members = set(R.AUTO_INT_VALUES)
    probe = set()
    for x in R.AUTO_INT_VALUES:
        probe |= {x - 1, x, x + 1, 10 * x, 10 * x + 1, -x}
    for lo, hi in ((-(1 << 31), (1 << 31) - 1), (-(1 << 63), (1 << 63) - 1)):
        probe |= set(range(lo, lo + 2000)) | set(range(hi - 2000, hi + 1))
    probe = {x for x in probe if -(1 << 63) <= x < (1 << 63)}
    bad = [x for x in probe if _ref_flag(x) != (x in members)]
    assert not bad, bad[:10]
    i32 = {int(x) for x in R.AUTO_INT32}
    assert i32 == {x for x in members if -(1 << 31) <= x < (1 << 31)}


@pytest.mark.parametrize("v,flag", [(float("nan"), True), (float("inf"), True), (float("-inf"), False), (0.0, False),
                                    (-0.0, False), (111.0, True), (-111.0, True), (1.5, False), (123.0, False),
                                    (1e16, False), (2.5e-05, False)])
def test_float_verdicts(v, flag):
    assert _ref_flag(v) == flag
    assert R.Rule()(R.value_str(v, True)) == flag


def test_float_keys_keep_signed_zero_and_one_nan():
    vals = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 1.0], np.float64)
    bits = vals.view(np.uint64).copy()
    bits[0] = 0xFFF8000000000001                       # another NaN payload
    vals = np.concatenate([vals, bits[:1].view(np.float64)])
    t = R.sort_table(vals)
    assert len(t) == 6 and np.isnan(t[-1]) and [str(x) for x in t[:-1]] == ["-inf", "-0.0", "0.0", "1.0", "inf"]
    assert [str(float(x)) for x in R.numeric_table(vals, R.Rule())] == ["inf", "nan"]


@pytest.mark.parametrize("kw", [dict(detection_type="manual", invalid_entries=["self-emp.*", "1[0-9]"]),
                                dict(detection_type="both", valid_entries=["[a-z -]+"], partial_match=True),
                                dict(detection_type="both", invalid_entries=["x"], valid_entries=["y"]),
                                dict(detection_type="nonsense", invalid_entries=[".*"])])
def test_rule_matches_detect_on_strings(kw):
    rule = R.Rule(kw.get("detection_type"), kw.get("invalid_entries", ()), kw.get("valid_entries", ()),
                  kw.get("partial_match", False))
    for s in ["", " ", "x", "y", " X ", "Self-emp-inc", "12", "abc", "aaa", "?", "n/a", "Never-worked", "mar-ried",
              "kkk k", "-111", "1a1", "xyz", "ÀÁÂ"]:
        assert rule(s) == (O.detect(s, **kw) == 1), s


# ---- the product's host layer against the oracle ---------------------------------------------------------------------

def product(table_or_frame, **kw):
    from anovos.data_analyzer.quality_checker import invalidEntries_detection
    with invalid_stand_in.installed(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        odf, p = invalidEntries_detection(None, table_or_frame, **kw)
        if getattr(odf, "is_partitioned", False):
            odf = pa.concat_tables([ch.to_arrow() for ch in odf.chunks()])
        else:
            odf = odf.to_arrow()
    return odf, p.toPandas()


def same_print(got, exp):
    assert got["attribute"].tolist() == exp["attribute"].tolist()
    assert got["invalid_count"].tolist() == exp["invalid_count"].tolist()
    assert got["invalid_pct"].tolist() == exp["invalid_pct"].tolist()
    assert [entry_set(s) for s in got["invalid_entries"]] == [entry_set(s) for s in exp["invalid_entries"]]


def test_product_unit_test():
    odf, p = product(unit_table(), treatment=True)
    _, exp, _ = O.invalidEntries_detection(unit_table(), treatment=True)
    same_print(p, exp)
    assert odf.num_rows == 5


@pytest.mark.parametrize("cell", [47, 48, 49])
def test_product_notebook_tables(income, cell):
    _, p = product(income, **_kwargs_of(cell))
    check_print(p, _quality(cell))


@pytest.mark.parametrize("kw", [dict(), dict(detection_type="manual", invalid_entries=["self-emp.*", "4[0-9]"]),
                                dict(detection_type="both", valid_entries=["[a-z -]+", "[0-9]+"], partial_match=True),
                                dict(list_of_cols="age|logfnl|latitude|sex", detection_type="both", invalid_entries=["3.*"]),
                                dict(detection_type="unknown", invalid_entries=[".*"])])
def test_product_modes_match_oracle(income, kw):
    _, p = product(income, **dict(kw))
    _, exp, _ = O.invalidEntries_detection(income, **dict(kw))
    same_print(p, exp)


@pytest.mark.parametrize("method", ["null_replacement", "column_removal"])
@pytest.mark.parametrize("output_mode", ["replace", "append"])
@pytest.mark.parametrize("threshold", [None, 0, 0.001])
def test_product_treatments_match_oracle(income, method, output_mode, threshold):
    cols = ["age", "sex", "race", "workclass", "logfnl", "capital-gain"]
    cfg = {} if threshold is None else {"treatment_threshold": threshold}
    kw = dict(list_of_cols=cols, treatment=True, treatment_method=method, output_mode=output_mode)
    if method == "column_removal" and not threshold:
        with pytest.raises(TypeError, match="column removal threshold"):
            product(income, treatment_configs=dict(cfg), **kw)
        with pytest.raises(TypeError, match="column removal threshold"):
            O.invalidEntries_detection(income, treatment_configs=dict(cfg), **kw)
        return
    got_t, got = product(income, treatment_configs=dict(cfg), **kw)
    exp_t, exp, _ = O.invalidEntries_detection(income, treatment_configs=dict(cfg), **kw)
    same_print(got, exp)
    same_tables(got_t, exp_t)


def test_product_column_order_and_append_drop(income):
    cols = ["sex", "age", "race"]
    t, _ = product(income, list_of_cols=cols, treatment=True)
    assert t.column_names[-3:] == cols                             # replace: treated columns move to the end
    t, _ = product(income, list_of_cols=cols, treatment=True, output_mode="append")
    assert t.column_names[-2:] == ["sex_invalid", "race_invalid"]  # age has no invalid rows: its _invalid is dropped


def test_product_chunked_frames_match_resident(income):
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.partitioned import PartitionedFrame
    cols = ["age", "sex", "race", "workclass", "logfnl", "capital-gain"]
    for kw in (dict(treatment=True), dict(treatment=True, output_mode="append"),
               dict(detection_type="both", valid_entries=["[a-z]+"], treatment=True)):
        wt, w = product(ColumnFrame.from_arrow(income), list_of_cols=cols, **kw)
        pt, p = product(PartitionedFrame.from_frame(ColumnFrame.from_arrow(income), 4096), list_of_cols=cols, **kw)
        assert w.equals(p)
        same_tables(pt, wt)


def test_treatment_threshold_is_popped(income):
    cfg = {"treatment_threshold": 0.01}
    product(income, list_of_cols="workclass", treatment=True, treatment_configs=cfg)
    assert cfg == {}


@pytest.mark.parametrize("kw,err", [(dict(list_of_cols=["nope"]), "Invalid input for Column"),
                                    (dict(output_mode="x"), "Invalid input for output_mode"),
                                    (dict(treatment="maybe"), "Non-Boolean input for treatment"),
                                    (dict(treatment_method="KNN"), "Invalid input for method_type"),
                                    (dict(treatment_method="column_removal"), "column removal threshold")])
def test_validation_errors(income, kw, err):
    with pytest.raises(TypeError, match=err):
        product(income, **kw)
    with pytest.raises(TypeError, match=err):
        O.invalidEntries_detection(income, **kw)


def test_empty_list_warns_and_returns_input(income):
    from anovos.data_analyzer.quality_checker import invalidEntries_detection
    with pytest.warns(UserWarning, match="No Invalid Entries Check"):
        odf, p = invalidEntries_detection(None, income, list_of_cols="age", drop_cols="age")
    assert list(p.toPandas().columns) == O.PRINT_COLS and len(p.toPandas()) == 0 and odf.columns == income.column_names


def test_other_kind_is_refused():
    t = pa.table({"flag": [True, False, None], "s": ["a", "b", "c"]})
    with pytest.raises(TypeError, match="boolean"):
        product(t, list_of_cols=["flag", "s"])


def test_all_takes_discrete_columns_only(income):
    _, p = product(income)
    assert "logfnl" not in p["attribute"].tolist() and "latitude" not in p["attribute"].tolist()
    assert p["attribute"].tolist() == [f.name for f in income.schema
                                       if str(f.type) in ("string", "int32", "int64")]
    assert not math.isnan(p["invalid_pct"].sum())
