"""Every table the transformers notebook stored for cat_to_num_unsupervised, cat_to_num_supervised and
outlier_categories (tests/golden/notebook_encoding.json, extracted by make_golden_encoding.py) against both the oracle
(tests/encoding_oracle.py) and the product's host layer on the NumPy kernel stand-ins of test_encoding_cpu.py, on the
income table the notebook read: the summary count / min / max tables, the printSchema blocks, the uniqueValues tables
and the encoded columns of the `toPandas().head(5)` tables."""
import json
import os
import warnings

import pyarrow as pa
import pytest

import encoding_oracle as E
from test_encoding_cpu import stand_ins

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _nb():
    return json.load(open(os.path.join(GOLDEN, "notebook_encoding.json")))


def _cell(cell, kind):
    return [t for t in _nb() if t["code_cell"] == cell and t["kind"] == kind]


def _run_product(name, table, **kw):
    import anovos.data_transformer.transformers as T
    with stand_ins(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return getattr(T, name)(None, table, **kw)


def _run_oracle(name, table, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return getattr(E, name)(table, **kw)


def _java(v, t):
    from anovos_b200.shared.utils import jvm_double_str
    if pa.types.is_floating(t):
        return jvm_double_str(v)
    return str(v)


def summary(table, cols):
    """`summary("count", "min", "max")` of a pyarrow table: {column: [count, min, max]} as Spark prints them (stripped,
    as the stored tables are)."""
    out = {}
    for c in cols:
        col = table.column(c)
        x = col.drop_null().to_pylist()
        if pa.types.is_string(col.type) or pa.types.is_large_string(col.type):
            x = sorted(x, key=lambda s: s.encode())
            lo, hi = (x[0], x[-1]) if x else ("null", "null")
        else:
            lo, hi = (_java(min(x), col.type), _java(max(x), col.type)) if x else ("null", "null")
        out[c] = [str(len(x)), lo.strip(), hi.strip()]
    return out


def _stored_summary(t):
    return {c: [r[j + 1] for r in t["rows"]] for j, c in enumerate(t["columns"][1:])}


def _product_summary(fr, cols):
    from anovos_b200.data_transformer.transformers import summary_count_min_max
    with stand_ins():
        df = summary_count_min_max(fr, cols).toPandas()
    return {c: [str(v).strip() for v in df[c].tolist()] for c in cols}


def _check_summaries(cell, before, after, src_cols, out_cols):
    """before / after = (product frame, oracle table) pairs."""
    tb, ta = _cell(cell, "show")
    exp_b, exp_a = _stored_summary(tb), _stored_summary(ta)
    assert sorted(exp_b) == sorted(src_cols) and sorted(exp_a) == sorted(out_cols)
    assert summary(before[1], src_cols) == exp_b
    assert summary(after[1], out_cols) == exp_a
    assert summary(_arrow(after[0]), out_cols) == exp_a
    assert _product_summary(before[0], src_cols) == exp_b
    assert _product_summary(after[0], out_cols) == exp_a


def _head_cell(v):
    return None if v in ("NaN", "None") else v


def _check_head(cell, table, outputs):
    """The encoded columns of the stored `toPandas().head(5)` table."""
    (t,) = _cell(cell, "pandas")
    checked = 0
    for j, c in enumerate(t["columns"]):
        if c not in outputs:
            continue
        got = table.column(c).to_pylist()[:len(t["rows"])]
        for r, g in zip(t["rows"], got):
            e = _head_cell(r[j])
            if e is None or g is None:
                assert e is None and g is None, (cell, c)
            elif isinstance(g, str):
                assert g.strip() == e, (cell, c)
            else:
                assert float(g) == float(e), (cell, c)
        checked += 1
    assert checked >= 5


def _unique_table(t):
    return {r[0]: int(r[1]) for r in t["rows"]}


def _distinct(table, cols):
    return {c: len(set(table.column(c).drop_null().to_pylist())) for c in cols}


@pytest.fixture(scope="module")
def cats(income):
    return [f.name for f in income.schema if pa.types.is_string(f.type)]


def test_cell18_label_encoding_summaries_and_head(income, cats):
    cols = [c for c in cats if c not in ("ifa", "geohash")]          # the default threshold 50 skips them
    odf = _run_product("cat_to_num_unsupervised", income)
    otab, _ = _run_oracle("cat_to_num_unsupervised", income)
    _check_summaries(18, (_frame(income), income), (odf, otab), cols, cols)
    _check_head(18, _arrow(odf), cols)
    _check_head(18, otab, cols)


def test_cell19_alphabet_order_head(income, cats):
    kw = dict(list_of_cols="all", drop_cols=["ifa"], index_order="alphabetAsc")
    outs = [c for c in cats if c not in ("ifa", "geohash")]
    _check_head(19, _arrow(_run_product("cat_to_num_unsupervised", income, **kw)), outs)
    _check_head(19, _run_oracle("cat_to_num_unsupervised", income, **kw)[0], outs)


def test_cells20_to_22_one_hot_schema_head_and_saved_model(income, tmp_path):
    from anovos_b200.data_transformer.transformers import print_schema
    kw = dict(list_of_cols=["race", "sex"], method_type="onehot_encoding")
    odf = _run_product("cat_to_num_unsupervised", income, **kw)
    otab, lab = _run_oracle("cat_to_num_unsupervised", income, **kw)
    before, after = _cell(20, "schema")
    new = ["%s_%d" % (c, j) for c in ("race", "sex") for j in range(len(lab[c]) + 1)]
    assert print_schema(_frame(income), ["race", "sex"]).splitlines()[1:] == before["lines"]
    assert print_schema(odf, new).splitlines()[1:] == after["lines"]
    assert [c for c in otab.column_names if c.startswith(("race_", "sex_"))] == new
    for cell in (20, 21, 22):
        _check_head(cell, otab, new)
    _check_head(20, _arrow(odf), new)
    mp = str(tmp_path)
    _check_head(21, _arrow(_run_product("cat_to_num_unsupervised", income, model_path=mp, **kw)), new)
    _check_head(22, _arrow(_run_product("cat_to_num_unsupervised", income, pre_existing_model=True, model_path=mp,
                                 **kw)), new)


def test_cells24_to_27_supervised_summaries(income, cats, tmp_path):
    cols = [c for c in cats if c not in ("ifa", "income")]
    kw = dict(list_of_cols="all", drop_cols="ifa", label_col="income", event_label=">50K")
    _check_summaries(24, (_frame(income), income),
                     (_run_product("cat_to_num_supervised", income, **kw), _run_oracle("cat_to_num_supervised", income, **kw)[0]),
                     cols, cols)
    two = ["relationship", "marital-status"]
    kw = dict(list_of_cols=two, label_col="income", event_label=">50K")
    app = dict(kw, output_mode="append")
    _check_summaries(25, (_frame(income), income),
                     (_run_product("cat_to_num_supervised", income, **app), _run_oracle("cat_to_num_supervised", income, **app)[0]),
                     two, [c + "_encoded" for c in two])
    mp = str(tmp_path)
    _run_product("cat_to_num_supervised", income, list_of_cols=two + ["workclass"], label_col="income", event_label=">50K",
                 model_path=mp, output_mode="append")
    _, models = _run_oracle("cat_to_num_supervised", income, **kw)
    _check_summaries(27, (_frame(income), income),
                     (_run_product("cat_to_num_supervised", income, pre_existing_model=True, model_path=mp, **kw),
                      _run_oracle("cat_to_num_supervised", income, models=models, **kw)[0]), two, two)


@pytest.mark.parametrize("cell,kw", [(96, dict(max_category=10)), (97, dict(coverage=0.9))])
def test_cells96_97_outlier_unique_counts(income, cell, kw):
    cols = ["education", "occupation", "native-country"]
    tb, ta = _cell(cell, "show")
    assert _distinct(income, cols) == _unique_table(tb)
    assert _distinct(_run_oracle("outlier_categories", income, list_of_cols=cols, **kw)[0], cols) == _unique_table(ta)
    odf = _run_product("outlier_categories", income, list_of_cols=cols, **kw)
    assert _product_unique(odf, cols) == _unique_table(ta)


def _product_unique(fr, cols):
    from anovos_b200.data_analyzer.stats_generator import uniqueCount_computation
    with stand_ins():
        df = uniqueCount_computation(None, fr, cols).toPandas()
    return dict(zip(df["attribute"], df["unique_values"].astype(int)))


def test_cells95_98_99_outliers_saved_model_and_whitespace(income, cats, tmp_path):
    income = income.drop_columns(["empty"])              # the notebook's frame of these cells has no `empty` column
    cols = [c for c in cats if c not in ("ifa", "empty")]
    kw = dict(drop_cols=["ifa"], max_category=15)
    app = _arrow(_run_product("outlier_categories", income, output_mode="append", **kw))
    _check_head(95, app, [c + "_outliered" for c in cols])
    _check_head(95, _run_oracle("outlier_categories", income, output_mode="append", **kw)[0], [c + "_outliered" for c in cols])
    mp = str(tmp_path)
    tb, ta = _cell(98, "show")
    assert _distinct(income, cols) == _unique_table(tb)
    fit = _run_product("outlier_categories", income, model_path=mp, **kw)
    otab, params = _run_oracle("outlier_categories", income, **kw)
    assert _product_unique(fit, cols) == _unique_table(ta) == _distinct(otab, cols)
    # cell 99: the saved model is trimmed, so " Private" / " State-gov" of the real table no longer match
    assert sum(1 for v in set(income.column("workclass").drop_null().to_pylist()) if v != v.strip()) == 2
    tb, ta = _cell(99, "show")
    again = _run_product("outlier_categories", income, drop_cols=["ifa"], pre_existing_model=True, model_path=mp)
    trimmed = {c: [k.strip() for k in ks] for c, ks in params.items()}
    oagain, _ = _run_oracle("outlier_categories", income, drop_cols=["ifa"], params=trimmed)
    assert _product_unique(again, cols) == _unique_table(ta) == _distinct(oagain, cols)
    assert _unique_table(ta)["workclass"] == 10 and _unique_table(tb)["workclass"] == 11


def _arrow(fr):
    with stand_ins():
        return fr.to_arrow()


def _frame(table):
    from anovos_b200.frame import ColumnFrame
    return ColumnFrame.from_arrow(table)
