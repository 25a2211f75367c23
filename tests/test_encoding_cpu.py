"""cat_to_num_unsupervised, cat_to_num_supervised and outlier_categories without a GPU:
  - the oracle (tests/encoding_oracle.py) against the reference's unit tests on part-00001 of its test dataset and the
    values its transformers notebook stored for the income table;
  - the product's host layer (argument handling, label orders, models, column order, partitioned frames, impact tables,
    the one-hot memory refusal) against the oracle, with anv_code_map / anv_one_hot replaced by NumPy images of one
    kernel call and the other kernels by tests/cpu_engine.py."""
import contextlib
import os
import warnings

import numpy as np
import pyarrow as pa
import pytest

import cpu_engine
import encoding_oracle as E
from anovos_b200 import engine

CATS = ["workclass", "education", "marital-status", "relationship", "race", "sex", "empty", "geohash"]


# ---- NumPy stand-ins of anv_code_map / anv_one_hot ------------------------------------------------------------------

def _slots(fr, n):
    vals, ok = cpu_engine._values(fr, n)
    size = len(fr.column(n).dictionary)
    return np.where(ok, np.minimum(vals.astype(np.int64) & 0xFFFFFFFF, size), size)


def code_map(fr, names, tables, entry_valid):
    import torch
    outs, valid, nulls = [], [], []
    for n, t, ev in zip(names, tables, entry_valid):
        s = _slots(fr, n)
        out = t[s]
        if ev is None:
            valid.append(None)
            nulls.append(0)
        else:
            keep = np.asarray(ev, bool)[s]
            out = np.where(keep, out, t.dtype.type(0))
            bits = np.packbits(keep, bitorder="little")
            bits = np.concatenate([bits, np.zeros((-len(bits)) % 4, np.uint8)])
            valid.append(torch.from_numpy(bits.view(np.int32).copy()))
            nulls.append(int((~keep).sum()))
        outs.append(torch.from_numpy(np.ascontiguousarray(out)))
    return outs, valid, np.array(nulls, np.int64)


def one_hot(fr, names, indexes, ks):
    import torch
    return [torch.from_numpy((ix[_slots(fr, n)][None, :] == np.arange(k)[:, None]).astype(np.int32))
            for n, ix, k in zip(names, indexes, ks)]


@contextlib.contextmanager
def stand_ins(free_bytes=1 << 40):
    from anovos_b200.data_transformer import transformers as T
    saved = engine.code_map, engine.one_hot, T._free_device_bytes
    try:
        engine.code_map, engine.one_hot, T._free_device_bytes = code_map, one_hot, lambda: free_bytes
        with cpu_engine.installed():
            yield
    finally:
        engine.code_map, engine.one_hot, T._free_device_bytes = saved


def _fn(name):
    import anovos.data_transformer.transformers as T
    return getattr(T, name)


def product(name, table_or_frame, **kw):
    with stand_ins():
        odf = _fn(name)(None, table_or_frame, **kw)
        if getattr(odf, "is_partitioned", False):
            return pa.concat_tables([ch.to_arrow() for ch in odf.chunks()])
        return odf.to_arrow()


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
        assert g.to_pylist() == e.to_pylist(), c


def _distinct(t, c):
    return len(set(t.column(c).to_pylist()))           # Spark's distinct() counts null as a value


def _minmax(t, c):
    x = t.column(c).drop_null().to_pylist()
    return min(x), max(x)


# ---- the oracle against the reference's unit tests (test_transformers.py:636-896) --------------------------------

def test_oracle_outlier_categories_unit_test(income_part1):
    cols5 = ["workclass", "education", "relationship", "race", "native-country"]
    odf, params = E.outlier_categories(income_part1, cols5, max_category=12)
    assert odf.num_columns == 17
    exp = {"workclass": 10, "education": 13, "relationship": 9, "native-country": 12, "race": 10, "occupation": 16,
           "sex": 4, "marital-status": 8}
    assert {c: _distinct(odf, c) for c in exp} == exp
    assert E.outlier_categories(income_part1, [], max_category=12)[0] is income_part1
    assert E.outlier_categories(income_part1, cols5, max_category=12, output_mode="append")[0].num_columns == 22


def test_oracle_unsupervised_unit_tests(income_part1):
    three = ["workclass", "relationship", "marital-status"]
    odf, _ = E.cat_to_num_unsupervised(income_part1, three, drop_cols=["ifa"], cardinality_threshold=100)
    assert odf.num_columns == 17
    assert {c: _minmax(odf, c) for c in three} == {"workclass": (0, 8), "relationship": (0, 7), "marital-status": (0, 6)}
    assert all(odf.schema.field(c).type == pa.int32() for c in three)
    assert odf.schema.field("education").type == pa.string()
    assert E.cat_to_num_unsupervised(income_part1, three, cardinality_threshold=100, output_mode="append")[0].num_columns == 20
    two = ["marital-status", "relationship"]
    odf, lab = E.cat_to_num_unsupervised(income_part1, two, method_type="onehot_encoding", cardinality_threshold=100)
    assert odf.num_columns == 32
    assert _minmax(odf, "marital-status_7") == (0, 1) and _minmax(odf, "relationship_8") == (0, 1)
    again, _ = E.cat_to_num_unsupervised(income_part1, two, method_type="onehot_encoding", labels=lab)
    same_tables(again, odf)


def test_oracle_supervised_unit_test(income_part1):
    three = ["workclass", "relationship", "marital-status"]
    odf, _ = E.cat_to_num_supervised(income_part1, three, drop_cols=["ifa"], label_col="income", event_label="<=50K")
    assert odf.num_columns == 17
    assert all(odf.schema.field(c).type == pa.float64() for c in three)
    ifa = income_part1.column("ifa").to_pylist()
    wc, inc = income_part1.column("workclass").to_pylist(), income_part1.column("income").to_pylist()
    for key, cat in (("27520a", "Private"), ("6144a", "Local-gov"), ("23710a", "Federal-gov")):
        lab = [y for w, y in zip(wc, inc) if w == cat]
        rate = lab.count("<=50K") / len(lab)
        assert round(odf.column("workclass")[ifa.index(key)].as_py()) == round(rate)
    assert E.cat_to_num_supervised(income_part1, three, label_col="income", event_label="<=50K",
                                   output_mode="append")[0].num_columns == 20


# ---- the oracle against the notebook's stored Spark outputs (income table) ------------------------------------------

def test_oracle_notebook_values(income):
    def head(order):
        return E.cat_to_num_unsupervised(income, ["workclass"], index_order=order)[0].column("workclass").to_pylist()[:5]
    assert head("frequencyDesc") == [10, 1, 0, 0, 0]
    assert head("alphabetAsc") == [1, 8, 6, 6, 6]
    oh, lab = E.cat_to_num_unsupervised(income, ["race"], method_type="onehot_encoding")
    assert len(lab["race"]) == 9 and [c for c in oh.column_names if c.startswith("race")] == ["race_%d" % j for j in range(10)]

    def uniq(c, **kw):
        return len(set(E.outlier_categories(income, [c], **kw)[0].column(c).drop_null().to_pylist()))
    assert [uniq(c, max_category=10) for c in ("education", "occupation", "native-country")] == [10, 10, 10]
    assert [uniq(c, coverage=0.9) for c in ("native-country", "occupation", "education")] == [3, 11, 9]
    assert uniq("geohash", max_category=15) == 38
    sup, models = E.cat_to_num_supervised(income, ["empty"], label_col="income", event_label=">50K")
    assert models["empty"] == [(None, 0.2408)]
    assert sup.column("empty").null_count == 0 and _minmax(sup, "empty") == (0.2408, 0.2408)


# ---- the product's host layer against the oracle --------------------------------------------------------------------

@pytest.mark.parametrize("method", ["label_encoding", "onehot_encoding"])
@pytest.mark.parametrize("order", ["frequencyDesc", "frequencyAsc", "alphabetDesc", "alphabetAsc"])
@pytest.mark.parametrize("output_mode", ["replace", "append"])
def test_unsupervised_host_layer_equals_oracle(income, method, order, output_mode):
    kw = dict(list_of_cols=CATS, method_type=method, index_order=order, cardinality_threshold=100, output_mode=output_mode)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        same_tables(product("cat_to_num_unsupervised", income, **kw), E.cat_to_num_unsupervised(income, **kw)[0])


@pytest.mark.parametrize("output_mode", ["replace", "append"])
@pytest.mark.parametrize("event", [">50K", "<=50K"])
def test_supervised_host_layer_equals_oracle(income, output_mode, event):
    kw = dict(list_of_cols="all", label_col="income", event_label=event, output_mode=output_mode)
    same_tables(product("cat_to_num_supervised", income, **kw), E.cat_to_num_supervised(income, **kw)[0])


@pytest.mark.parametrize("cov,mx", [(1.0, 50), (1.0, 10), (0.9, 50), (0.5, 3), (1.0, 2)])
@pytest.mark.parametrize("output_mode", ["replace", "append"])
def test_outlier_host_layer_equals_oracle(income, cov, mx, output_mode):
    kw = dict(list_of_cols="all", coverage=cov, max_category=mx, output_mode=output_mode)
    same_tables(product("outlier_categories", income, **kw), E.outlier_categories(income, **kw)[0])


def test_chunked_frames_equal_oracle(income):
    from anovos_b200.partitioned import PartitionedFrame
    with stand_ins():
        part = PartitionedFrame.from_frame(income, 4096)
    for name, kw in [("cat_to_num_unsupervised", dict(list_of_cols=CATS[:-1], method_type="onehot_encoding")),
                     ("cat_to_num_supervised", dict(label_col="income", event_label="<=50K")),
                     ("outlier_categories", dict(coverage=0.8))]:
        same_tables(product(name, part, **kw), getattr(E, name)(income, **kw)[0])


def test_unsorted_dictionary_and_nulls():
    """Orders come from a sort of the categories, never from code order; null rows stay null (label, outlier) or read
    the null group (supervised)."""
    from anovos_b200.frame import ColumnFrame
    codes = np.array([2, 0, 1, 1, 2, 2, 0, 0, 0, 1], np.int32)
    ok = np.array([1, 1, 1, 1, 1, 0, 1, 1, 1, 1], bool)
    words = np.packbits(ok, bitorder="little")
    words = np.concatenate([words, np.zeros((-len(words)) % 4, np.uint8)]).view(np.int32)
    lab = np.array([1, 0, 1, 0, 1, 1, 0, 0, 1, 1], np.int32)
    fr = ColumnFrame.from_tensors({"c": (codes, words, ["zz", "a", "é"]), "y": lab})
    table = pa.table({"c": pa.array(["é", "zz", "a", "a", "é", None, "zz", "zz", "zz", "a"]), "y": pa.array(lab)})
    for order in ("frequencyDesc", "alphabetAsc", "alphabetDesc", "frequencyAsc"):
        same_tables(product("cat_to_num_unsupervised", fr, index_order=order),
                    E.cat_to_num_unsupervised(table, index_order=order)[0])
    same_tables(product("cat_to_num_supervised", fr, label_col="y", event_label=1),
                E.cat_to_num_supervised(table, label_col="y", event_label=1)[0])
    same_tables(product("outlier_categories", fr, max_category=3), E.outlier_categories(table, max_category=3)[0])


# ---- models -----------------------------------------------------------------------------------------------------------

def test_unsupervised_model_round_trip(income, tmp_path):
    mp = str(tmp_path)
    kw = dict(list_of_cols=["race", "sex"], method_type="onehot_encoding", model_path=mp)
    first = product("cat_to_num_unsupervised", income, index_order="alphabetDesc", **kw)
    d = os.path.join(mp, "cat_to_num_unsupervised")
    assert sorted(os.listdir(os.path.join(d, "indexer"))) == ["data", "metadata"]
    assert os.path.exists(os.path.join(d, "encoder", "metadata", "part-00000"))
    for f in ("_SUCCESS", ".part-00000.crc"):                  # what Spark leaves next to its parts
        open(os.path.join(d, "indexer", "metadata", f), "w").close()
    again = product("cat_to_num_unsupervised", income, pre_existing_model=True, **kw)
    same_tables(again, first)
    # a model fitted on a subset: categories it lacks are unseen and go to the last column
    sub = income.filter(pa.compute.equal(income.column("race"), "White"))
    product("cat_to_num_unsupervised", sub, list_of_cols=["race"], model_path=mp)
    got = product("cat_to_num_unsupervised", income, list_of_cols=["race"], pre_existing_model=True, model_path=mp)
    exp = [None if v is None else (0 if v == "White" else 1) for v in income.column("race").to_pylist()]
    assert got.column("race").to_pylist() == exp
    with pytest.raises(ValueError, match="cannot resolve 'sex_index'"):
        product("cat_to_num_unsupervised", income, list_of_cols=["sex"], pre_existing_model=True, model_path=mp)


def test_supervised_model_round_trip(tmp_path):
    from anovos_b200.data_transformer import transformers as T
    mp = str(tmp_path)
    table = pa.table({"c": pa.array([" a", "b,c", None, "", 'q"x', "b,c", " a"] * 3),
                      "y": pa.array(["1", "0", "1", "0", "0", "1", "0"] * 3)})
    first = product("cat_to_num_supervised", table, label_col="y", event_label="1", model_path=mp)
    rows = open(os.path.join(mp, "cat_to_num_supervised", "c", "part-00000-c000.csv")).read().splitlines()
    assert rows[0] == "c,c_encoded" and rows[1] == ",1.0" and '" a",0.5' not in rows
    assert " a,0.5" in rows and '"b,c",0.5' in rows and '"",0.0' in rows and '"q\\"x",0.0' in rows
    assert T.load_supervised_model(mp, "c") == [(None, 1.0), ("", 0.0), (" a", 0.5), ("b,c", 0.5), ('q"x', 0.0)]
    same_tables(product("cat_to_num_supervised", table, label_col="y", event_label="1", pre_existing_model=True,
                        model_path=mp), first)
    tiny = pa.table({"c": pa.array(["u"] * 4 + [None]), "y": pa.array(["1"] + ["0"] * 4)})
    product("cat_to_num_supervised", tiny, label_col="y", event_label="1", model_path=mp)
    assert T.load_supervised_model(mp, "c") == [(None, 0.0), ("u", 0.25)]
    T.save_supervised_model(mp, "c", [("u", 1e-4)])
    assert open(os.path.join(mp, "cat_to_num_supervised", "c", "part-00000-c000.csv")).read().splitlines()[1] == "u,1.0E-4"
    got = product("cat_to_num_supervised", tiny, label_col="y", event_label="1", pre_existing_model=True, model_path=mp)
    assert got.column("c").to_pylist() == [1e-4] * 5          # one row: a cross join, nulls included


def test_outlier_model_trims_whitespace(income, tmp_path):
    from anovos_b200.data_transformer import transformers as T
    mp = str(tmp_path)
    t = income.select(["workclass", "geohash"])
    t = t.set_column(0, "workclass", pa.array([None if v is None else " " + v if v in ("Private", "State-gov") else v
                                               for v in t.column("workclass").to_pylist()]))
    fit = product("outlier_categories", t, list_of_cols=["workclass"], max_category=15, model_path=mp)
    before = _distinct_nonnull(fit, "workclass")
    again = product("outlier_categories", t, list_of_cols=["workclass", "geohash"], max_category=15, pre_existing_model=True,
                    model_path=mp)
    after = _distinct_nonnull(again, "workclass")
    assert after == before - 1                           # " Private" and " State-gov" no longer match once trimmed
    assert set(again.column("geohash").drop_null().to_pylist()) == {"outlier_categories"}
    assert "Private" in T.load_outlier_model(mp)["workclass"]


def _distinct_nonnull(t, c):
    return len(set(t.column(c).drop_null().to_pylist()))


# ---- refusals and argument errors -------------------------------------------------------------------------------------

def test_one_hot_refuses_more_than_free_memory(income):
    from anovos_b200 import _lib
    with stand_ins(free_bytes=1000):
        from anovos_b200.data_transformer import transformers as T
        with pytest.raises(_lib.AnvError, match="one-hot encoding of column 'race' needs 10 output columns"):
            T.cat_to_num_unsupervised(None, income, list_of_cols=["race"], method_type="onehot_encoding")
    # race alone (10 outputs, 1.30 MB) fits in 1.5 MB, race and sex together (14 outputs) do not: the refusal names sex
    with stand_ins(free_bytes=1_500_000):
        from anovos_b200.data_transformer import transformers as T
        T.cat_to_num_unsupervised(None, income, list_of_cols=["race"], method_type="onehot_encoding")
        with pytest.raises(_lib.AnvError, match="column 'sex' needs 4 output columns; with the columns before it"):
            T.cat_to_num_unsupervised(None, income, list_of_cols=["race", "sex"], method_type="onehot_encoding")


def test_argument_errors(income, tmp_path):
    from anovos_b200.data_transformer import transformers as T
    with stand_ins():
        for kw, msg in [(dict(list_of_cols=["age"]), "Invalid input for Column"),
                        (dict(method_type="x"), "Invalid input for method_type"),
                        (dict(index_order="x"), "Invalid input for Encoding Index Order"),
                        (dict(output_mode="x"), "Invalid input for output_mode")]:
            with pytest.raises(TypeError, match=msg):
                T.cat_to_num_unsupervised(None, income, **kw)
        with pytest.warns(UserWarning, match="high cardinality: geohash"):
            T.cat_to_num_unsupervised(None, income, list_of_cols=["geohash", "race"])
        with pytest.warns(UserWarning, match="No Encoding Computation"):
            assert T.cat_to_num_unsupervised(None, income, list_of_cols=["race"], drop_cols="race").columns == income.column_names
        with pytest.raises(TypeError, match="Invalid input for Column"):
            T.cat_to_num_supervised(None, income, list_of_cols=["age"], label_col="income")
        with pytest.raises(TypeError, match="Invalid input for Label Column"):
            T.cat_to_num_supervised(None, income, list_of_cols=["race"], label_col="nope")
        with pytest.warns(UserWarning, match="No Categorical Encoding"):
            T.cat_to_num_supervised(None, income, list_of_cols=[], label_col="income")
        with pytest.raises(ValueError, match="cannot resolve '1'"):
            T.cat_to_num_supervised(None, income, list_of_cols=["race"], label_col="income", event_label="nope")
        with pytest.raises(TypeError, match="Invalid input for Column"):
            T.outlier_categories(None, income, list_of_cols=["age"])
        with pytest.warns(UserWarning, match="No Outlier Categories Computation"):
            T.outlier_categories(None, income, list_of_cols=[])
        for kw, msg in [(dict(coverage=0), "Coverage"), (dict(coverage=1.5), "Coverage"),
                        (dict(max_category=1), "Maximum No. of Categories"), (dict(output_mode="x"), "output_mode")]:
            with pytest.raises(TypeError, match=msg):
                T.outlier_categories(None, income, list_of_cols=["race"], **kw)
        stats = tmp_path / "u.csv"
        stats.write_text("attribute,unique_values\nrace,99\nsex,2\n")
        with pytest.warns(UserWarning, match="high cardinality: race"):
            out = T.cat_to_num_unsupervised(None, income, list_of_cols=["race", "sex"],
                                            stats_unique={"file_path": str(stats), "file_type": "csv"})
        assert dict(out.dtypes)["race"] == "string" and dict(out.dtypes)["sex"] == "int"


def test_dispatcher(income):
    from anovos_b200.data_transformer import transformers as T
    with stand_ins():
        out = T.cat_to_num_transformer(None, income, ["race"], [], "supervised", "label_encoding", "income", ">50K")
        assert dict(out.dtypes)["income"] == "int" and dict(out.dtypes)["race"] == "double"
        exp = [int(v == ">50K") for v in income.column("income").to_pylist()]
        assert out.to_arrow().column("income").to_pylist() == exp
        assert T.cat_to_num_transformer(None, income, "all", [], "unsupervised", "label_encoding", "income", 1) is None
        out = T.cat_to_num_transformer(None, income, "race|sex", [], "unsupervised", "onehot_encoding", None, None)
        assert "race_9" in out.columns
        with pytest.raises(TypeError, match="Invalid input for Column"):
            T.cat_to_num_transformer(None, income, ["age"], [], "unsupervised", "label_encoding", None, None)


def test_print_impact(income, capsys):
    product("cat_to_num_unsupervised", income, list_of_cols=["race"], print_impact=True)
    out = capsys.readouterr().out
    keys = sorted(set(income.column("race").drop_null().to_pylist()), key=lambda k: k.encode())
    before, after = out.split("After")
    assert keys[0] in before and keys[-1] in before and str(income.column("race").drop_null().__len__()) in before
    assert " %d\n" % (len(keys) - 1) in after
    product("cat_to_num_unsupervised", income, list_of_cols=["sex"], method_type="onehot_encoding", print_impact=True)
    out = capsys.readouterr().out
    assert " |-- sex: string (nullable = true)" in out and " |-- sex_2: integer (nullable = true)" in out
    product("outlier_categories", income, list_of_cols=["education"], max_category=10, print_impact=True)
    out = capsys.readouterr().out
    assert "uniqueValues_before" in out and "uniqueValues_after" in out
    product("cat_to_num_supervised", income, list_of_cols=["empty"], label_col="income", event_label=">50K",
            print_impact=True)
    out = capsys.readouterr().out
    assert "0.2408" in out and "32561" in out
