"""monotonic_binning and the monotonicity check of IV / IG on the GPU: anv_class_hist bit for bit against NumPy on
adversarial columns of every dtype, its per-model sums against K2 (engine.histogram) on the masked class views, the
ladder cutoffs against compute_cutoffs, and the API against the oracle (tests/monotonic_oracle.py) on the income table
with its Spark partitions, at 10 M rows and on chunked frames."""
import json
import os
import warnings

import numpy as np
import pyarrow as pa
import pytest

import monotonic_oracle as MO
from test_monotonic_cpu import NB, CELLS, ENC, stand_in_counts

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _words(valid):
    bits = np.packbits(np.asarray(valid, bool), bitorder="little")
    return np.concatenate([bits, np.zeros((-len(bits)) % 4, np.uint8)]).view(np.int32)


def _values(kind, n, rng):
    if kind == "i32":
        v = rng.integers(-40, 40, n).astype(np.int32)
        v[rng.random(n) < 0.01] = np.iinfo(np.int32).min
        v[rng.random(n) < 0.01] = np.iinfo(np.int32).max
        return v
    if kind == "i64":
        v = rng.integers(-40, 40, n).astype(np.int64) + (1 << 62) * (rng.random(n) < 0.1)
        v[rng.random(n) < 0.01] = np.iinfo(np.int64).min
        v[rng.random(n) < 0.01] = np.iinfo(np.int64).max
        return v
    dt, u = (np.float32, np.uint32) if kind == "f32" else (np.float64, np.uint64)
    v = (rng.standard_normal(n) * 20).round(1).astype(dt)
    nan = (np.array([0x7FC00000, 0xFFC00001, 0x7F800001], np.uint32) if kind == "f32" else
           np.array([0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000001], np.uint64)).astype(u).view(dt)
    sp = np.concatenate([nan, np.array([0.0, -0.0, np.inf, -np.inf], dt)])
    pick = rng.random(n) < 0.05
    v[pick] = sp[rng.integers(0, len(sp), int(pick.sum()))]
    return v


def _thresholds(kind, rng):
    from anovos_b200 import _lib
    from anovos_b200.shared import monotonic as M
    anv = {"i32": _lib.ANV_I32, "i64": _lib.ANV_I64, "f32": _lib.ANV_F32, "f64": _lib.ANV_F64}[kind]
    cuts = {n: sorted((rng.standard_normal(n - 1) * 20).round(0).tolist()) for n in M.LADDER}
    cuts[20][0], cuts[19][-1] = -np.inf, np.inf
    if kind == "i64":
        cuts[18] = [float((1 << 62) + 1024 * j) for j in range(-8, 9)]   # doubles 1024 apart: 17 distinct thresholds
    return M.UnionModel(cuts, anv), cuts, anv


@pytest.mark.parametrize("n", [0, 1, 31, 33, 1025, 100_003])
@pytest.mark.parametrize("kind", ["i32", "i64", "f32", "f64"])
def test_class_hist_bit_exact(kind, n):
    import torch
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    rng = np.random.default_rng([n, len(kind), ord(kind[0])])
    um, _, _ = _thresholds(kind, rng)
    vals = _values(kind, n, rng)
    if n > 8:
        vals[:8] = um.thresholds[:8]                               # values equal to thresholds
    valid = rng.random(n) > 0.2
    lab = rng.integers(0, 3, n).astype(np.float64)                 # 1 = event, 0 / 2 = non-event
    lab_ok = rng.random(n) > 0.1
    cols = {"some": (torch.from_numpy(vals).cuda(), torch.from_numpy(_words(valid)).cuda()),
            "free": (torch.from_numpy(vals.copy()).cuda(), None),
            "none": (torch.from_numpy(vals.copy()).cuda(), torch.from_numpy(_words(np.zeros(n, bool))).cuda()),
            "label": (torch.from_numpy(lab).cuda(), torch.from_numpy(_words(lab_ok)).cuda())}
    fr = ColumnFrame.from_tensors(cols)
    names = ["some", "free", "none"]
    got = engine.class_hist(fr, names, [um.thresholds] * 3, "label", 1)
    for name, ok, g in zip(names, (valid, np.ones(n, bool), np.zeros(n, bool)), got):
        exp = stand_in_counts(vals, ok, (lab == 1).astype(np.int64), lab_ok, um)
        assert np.array_equal(g, exp), name


def test_class_hist_column_blocks():
    import torch
    from anovos_b200 import _lib, engine
    from anovos_b200.frame import ColumnFrame
    n_cols, n = _lib.MAX_LAUNCH_COLS + 3, 97
    rng = np.random.default_rng(5)
    vals = rng.integers(0, 50, n).astype(np.int32)
    t = torch.from_numpy(vals).cuda()
    cols = {"c%d" % i: t for i in range(n_cols)}
    cols["label"] = torch.from_numpy(rng.integers(0, 2, n).astype(np.int32)).cuda()
    fr = ColumnFrame.from_tensors(cols)
    thr = np.array([3, 11, 40], np.int32)
    got = engine.class_hist(fr, ["c%d" % i for i in range(n_cols)], [thr] * n_cols, "label", 1)
    assert len(got) == n_cols and np.array_equal(got[0], got[-1]) and np.array_equal(got[0], got[n_cols // 2])
    assert int(got[0].sum()) == n


@pytest.mark.parametrize("kind", ["i32", "i64", "f32", "f64"])
def test_class_hist_models_equal_k2(kind):
    """Slots summed per model equal engine.histogram on the masked event / non-event views, for every n."""
    import torch
    from anovos_b200 import engine
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.shared import monotonic as M
    from anovos_b200.shared.label_classes import label_bitmaps, masked
    rng = np.random.default_rng(len(kind) + ord(kind[-1]))
    um, cuts, _ = _thresholds(kind, rng)
    n = 50_001
    vals = _values(kind, n, rng)
    valid = rng.random(n) > 0.1
    fr = ColumnFrame.from_tensors({"x": (torch.from_numpy(vals).cuda(), torch.from_numpy(_words(valid)).cuda()),
                                   "label": torch.from_numpy(rng.integers(0, 2, n).astype(np.int64)).cuda()})
    (h,) = engine.class_hist(fr, ["x"], [um.thresholds], "label", 1)
    ev, nev, _ = label_bitmaps(fr, "label", 1)
    for m, cut in cuts.items():
        a, e, ne = M.model_table(um, h, m)
        for view, want in ((fr, a), (masked(fr, ["x"], ev), e), (masked(fr, ["x"], nev), ne)):
            k2 = engine.histogram(view, engine.BinModel(view, ["x"], [cut]))[0, :m + 1].astype(np.int64)
            assert np.array_equal(k2[1:], want[1:]), (kind, m)


def _spark_frame(table):
    from anovos_b200.partitioned import PartitionedFrame
    rpp = json.load(open(os.path.join(GOLDEN, "income_partitions.json")))["rows_per_partition"]
    return PartitionedFrame.from_arrow_partitions(table, rpp)


def _arrow(odf):
    if getattr(odf, "is_partitioned", False):
        return pa.concat_tables([ch.to_arrow() for ch in odf.chunks()])
    return odf.to_arrow()


@pytest.mark.parametrize("layout", ["spark_partitions", "resident"])
@pytest.mark.parametrize("method", ["equal_range", "equal_frequency"])
def test_ladder_cutoffs_equal_compute_cutoffs(income, method, layout):
    """Both quantile routes: the GK sketches of Spark's partitions and the exact ranks of a resident frame."""
    from anovos_b200.data_transformer.transformers import compute_cutoffs
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.shared import monotonic as M
    fr = _spark_frame(income) if layout == "spark_partitions" else ColumnFrame.from_arrow(income)
    cols = ["age", "fnlwgt", "education-num", "hours-per-week", "logfnl", "capital-gain"]
    cuts, _ = M.ladder_cutoffs(fr, cols, method)
    for n in M.LADDER:
        _, ref, _ = compute_cutoffs(fr, cols, method, n)
        for c, r in zip(cols, ref):
            assert np.array_equal(np.array(cuts[c][n]), np.array(r), equal_nan=True), (c, n)


@pytest.mark.parametrize("bin_dtype", ["numerical", "categorical"])
@pytest.mark.parametrize("output_mode", ["replace", "append"])
@pytest.mark.parametrize("method", ["equal_range", "equal_frequency"])
def test_api_matches_oracle_on_income(income_spark, income, method, output_mode, bin_dtype):
    from anovos.data_transformer.transformers import monotonic_binning
    cols = ["age", "fnlwgt", "education-num", "hours-per-week", "logfnl", "capital-gain"]
    kw = dict(list_of_cols=cols, label_col="income", event_label=">50K", bin_method=method, bin_dtype=bin_dtype,
              output_mode=output_mode)
    exp = MO.monotonic_binning(income_spark, **kw)
    got = _arrow(monotonic_binning(None, _spark_frame(income), **kw))
    assert got.column_names == exp.column_names
    for c in exp.column_names:
        assert got.column(c).to_pylist() == exp.column(c).to_pylist(), c


def test_api_on_a_resident_frame_bins_with_the_chosen_models(income):
    """equal_frequency on a resident frame (exact-rank quantiles): each column binned as attribute_binning bins it with
    the chosen n, in one call."""
    from anovos.data_transformer.transformers import attribute_binning, monotonic_binning
    from anovos_b200.data_transformer.transformers import monotonic_models
    from anovos_b200.frame import ColumnFrame
    fr = ColumnFrame.from_arrow(income)
    cols = ["age", "fnlwgt", "education-num", "hours-per-week", "logfnl"]
    models, _ = monotonic_models(fr, fr, cols, "income", ">50K", "equal_frequency", 10)
    got = _arrow(monotonic_binning(None, fr, cols, label_col="income", event_label=">50K", bin_method="equal_frequency"))
    for c in cols:
        ref = _arrow(attribute_binning(None, fr, [c], method_type="equal_frequency", bin_size=models[c][0]))
        assert got.column(c).to_pylist() == ref.column(c).to_pylist(), c


@pytest.mark.parametrize("cell", sorted(CELLS))
def test_api_matches_notebook(income, cell):
    from anovos.data_transformer.transformers import monotonic_binning
    odf = _arrow(monotonic_binning(None, _spark_frame(income), list_of_cols=["education-num", "hours-per-week"],
                                   label_col="income", event_label=">50K", **CELLS[cell]))
    for c, exp in NB[cell]["columns"].items():
        assert [float(v) for v in odf.column(c).slice(0, 5).to_pylist()] == exp, (cell, c)


def test_api_reference_unit_test(income_part1):
    from anovos.data_transformer.transformers import monotonic_binning
    kw = dict(list_of_cols=["age", "fnlwgt", "hours-per-week"], label_col="income", event_label="<=50K",
              bin_method="equal_range", bin_size=10)
    odf = _arrow(monotonic_binning(None, income_part1, **kw))
    assert len(odf.column_names) == 17
    for c in kw["list_of_cols"]:
        v = [x for x in odf.column(c).to_pylist() if x is not None]
        assert (min(v), max(v)) == (1, 10)
    assert odf.column("logfnl").to_pylist() == income_part1.column("logfnl").to_pylist()
    same = _arrow(monotonic_binning(None, income_part1, **dict(kw, list_of_cols=[])))
    assert same.column("age").to_pylist() == income_part1.column("age").to_pylist()
    assert len(_arrow(monotonic_binning(None, income_part1, **dict(kw, output_mode="append"))).column_names) == 20


def test_api_refuses_an_all_null_equal_range_column():
    from anovos.data_transformer.transformers import monotonic_binning
    t = pa.table({"x": pa.array([None] * 40, pa.float64()), "y": np.arange(40.0), "label": [1, 0] * 20})
    with pytest.raises(ValueError, match="no non-null"):
        monotonic_binning(None, t, ["x", "y"])


@pytest.mark.parametrize("cell", [23, 30])
def test_iv_ig_example_6(income, nb_assoc, cell):
    from anovos.data_analyzer.association_evaluator import IG_calculation, IV_calculation
    fn, col = (IV_calculation, "iv") if cell == 23 else (IG_calculation, "ig")
    got = fn(None, _spark_frame(income), ["age", "sex", "race", "workclass", "fnlwgt"], label_col="income",
             event_label=">50K", encoding_configs=ENC).to_pandas()
    exp = {r[0]: r[1] for r in nb_assoc[cell]["rows"]}
    assert set(got["attribute"]) == set(exp)
    for a, v in zip(got["attribute"], got[col]):
        assert "%.6f" % v == exp[a], (cell, a, v, exp[a])


@pytest.mark.parametrize("bin_size", [10, 25, 300])
def test_iv_ig_match_oracle(income_spark, income, bin_size):
    from anovos.data_analyzer.association_evaluator import IG_calculation, IV_calculation
    # fnlwgt accepts no n under equal_frequency (IV Example 6): bin_size 300 takes the K2 fallback outside 3 .. 20
    cols = ["age", "fnlwgt", "education-num", "hours-per-week", "logfnl", "sex"]
    for method in ("equal_range", "equal_frequency"):
        enc = {"bin_method": method, "bin_size": bin_size, "monotonicity_check": 1}
        for fn, ofn, col in ((IV_calculation, MO.IV_calculation, "iv"), (IG_calculation, MO.IG_calculation, "ig")):
            got = fn(None, _spark_frame(income), cols, label_col="income", event_label=">50K",
                     encoding_configs=enc).to_pandas()
            exp = ofn(income_spark, cols, label_col="income", event_label=">50K", encoding_configs=enc)
            assert got["attribute"].tolist() == exp["attribute"].tolist()
            assert np.allclose(got[col].astype(float), exp[col].astype(float), rtol=1e-12, atol=0), (method, col)


def _scale_table(n, seed):
    """x rising event rate: P(event) = sigmoid((x - 50) / 10), a float32 column with nulls, a second int column."""
    rng = np.random.default_rng(seed)
    x = (rng.random(n) * 100).astype(np.float32)
    y = rng.integers(0, 1000, n).astype(np.int32)
    lab = (rng.random(n) < 1 / (1 + np.exp(-(x.astype(np.float64) - 50) / 10))).astype(np.int32)
    xv = rng.random(n) > 0.05
    return pa.table({"x": pa.array(x, mask=~xv), "y": y, "label": lab})


def test_scale_10m_matches_cpu_twin_and_attribute_binning():
    from anovos.data_transformer.transformers import attribute_binning, monotonic_binning
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.shared import monotonic as M
    t = _scale_table(10_000_000, 11)
    fr = ColumnFrame.from_arrow(t)
    odf = monotonic_binning(None, fr, ["x", "y"], label_col="label", event_label=1)
    from anovos_b200.data_transformer.transformers import monotonic_models
    models, lad = monotonic_models(fr, fr, ["x", "y"], "label", 1, "equal_range", 10)
    # the CPU twin: the same union model counted by NumPy, and the oracle's groupBy with real averages
    lab = t.column("label").to_numpy()
    for c in ("x", "y"):
        vals = t.column(c).to_numpy(zero_copy_only=False)
        valid = ~np.asarray(t.column(c).is_null())
        vals = np.where(valid, vals, 0).astype(vals.dtype if c == "y" else np.float32)
        twin = stand_in_counts(vals, valid, lab, np.ones(len(lab), bool), lad[c].um)
        assert np.array_equal(twin, lad[c].counts), c
        assert M.choose(lad[c].um, twin) == lad[c].n
    assert lad["x"].n is not None
    assert MO.chosen_bins(t, ["x"], "label", 1, "equal_range") == {"x": lad["x"].n}
    for c in ("x", "y"):
        n = models[c][0]
        ref = attribute_binning(None, fr, [c], method_type="equal_range", bin_size=n)
        assert np.array_equal(odf.column(c).device()[0].cpu().numpy(), ref.column(c).device()[0].cpu().numpy()), c


def test_chunked_frames_match_the_single_frame():
    from anovos.data_transformer.transformers import monotonic_binning
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.partitioned import PartitionedFrame
    t = _scale_table(300_001, 3)
    for bin_dtype in ("numerical", "categorical"):
        kw = dict(list_of_cols=["x", "y"], label_col="label", event_label=1, bin_dtype=bin_dtype, output_mode="append")
        whole = _arrow(monotonic_binning(None, ColumnFrame.from_arrow(t), **kw))
        parts = _arrow(monotonic_binning(None, PartitionedFrame.from_frame(ColumnFrame.from_arrow(t), 65_536), **kw))
        assert whole.column_names == parts.column_names
        for c in whole.column_names:
            assert whole.column(c).to_pylist() == parts.column(c).to_pylist(), (bin_dtype, c)
