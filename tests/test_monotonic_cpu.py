"""CPU checks of monotonic_binning and the monotonicity check of IV / IG: the row-by-row oracle (tests/monotonic_oracle.py)
against the reference's unit test and notebooks, and the product's host layer (shared/monotonic.py: union slots, bin
tables, decision) against direct binning and the oracle, with a NumPy stand-in of the anv_class_hist pass."""
import json
import math
import os
import warnings

import numpy as np
import pyarrow as pa
import pytest

from oracle import api as O
from oracle import spark_semantics as S
from anovos_b200 import _lib
from anovos_b200.shared import monotonic as M
import monotonic_oracle as MO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NB = {t["cell"]: t for t in json.load(open(os.path.join(GOLDEN, "notebook_monotonic.json")))}
CELLS = {19: dict(bin_method="equal_range", output_mode="append"), 21: dict(bin_method="equal_frequency")}
IV_IG_CELLS = {23: ("iv", MO.IV_calculation), 30: ("ig", MO.IG_calculation)}
ENC = {"bin_method": "equal_frequency", "bin_size": 10, "monotonicity_check": 1}
_NP = {_lib.ANV_F32: np.float32, _lib.ANV_F64: np.float64, _lib.ANV_I32: np.int32, _lib.ANV_I64: np.int64}


def stand_in_counts(values, valid, label01, label_valid, um: M.UnionModel):
    """NumPy restatement of anv_class_hist for one column (include/anovos_b200.h)."""
    u = len(um.thresholds)
    out = np.zeros(3 * um.n_slots + 2, np.uint64)
    x = np.asarray(values)
    isnan = np.isnan(x) if x.dtype.kind == "f" else np.zeros(len(x), bool)
    slot = np.where(~valid, 0, np.where(isnan, u + 2, 1 + np.searchsorted(um.thresholds, x, side="left")))
    cls = np.where(label_valid & (label01 == 1), 0, np.where(label_valid, 1, 2))
    np.add.at(out, cls * um.n_slots + slot, np.uint64(1))
    if x.dtype.kind == "f":
        out[3 * um.n_slots] = np.count_nonzero(valid & (x == -np.inf))
        out[3 * um.n_slots + 1] = np.count_nonzero(valid & (x == np.inf))
    return out


# ---- the oracle against the reference -----------------------------------------------------------------------------------

def test_oracle_reference_unit_test(income_part1):
    t = income_part1
    kw = dict(list_of_cols=["age", "fnlwgt", "hours-per-week"], label_col="income", event_label="<=50K",
              bin_method="equal_range", bin_size=10)
    assert MO.chosen_bins(t, kw["list_of_cols"], "income", "<=50K", "equal_range") == \
        {"age": None, "fnlwgt": None, "hours-per-week": None}
    odf = MO.monotonic_binning(t, **kw)
    assert len(odf.column_names) == 17
    for c in kw["list_of_cols"]:
        v = [x for x in odf.column(c).to_pylist() if x is not None]
        assert (min(v), max(v)) == (1, 10)
    assert odf.column("logfnl").equals(t.column("logfnl"))
    assert MO.monotonic_binning(t, **dict(kw, list_of_cols=[])).equals(t)
    assert len(MO.monotonic_binning(t, **dict(kw, output_mode="append")).column_names) == 20


@pytest.mark.parametrize("cell", sorted(CELLS))
def test_oracle_matches_notebook(income_spark, cell):
    odf = MO.monotonic_binning(income_spark, list_of_cols=["education-num", "hours-per-week"], label_col="income",
                               event_label=">50K", **CELLS[cell])
    for c, exp in NB[cell]["columns"].items():
        assert [float(v) for v in odf.column(c).slice(0, 5).to_pylist()] == exp, (cell, c)


def test_oracle_chooses_the_notebooks_bin_counts(income_spark):
    cols = ["education-num", "hours-per-week"]
    assert MO.chosen_bins(income_spark, cols, "income", ">50K", "equal_range") == {"education-num": 7, "hours-per-week": 3}
    assert MO.chosen_bins(income_spark, cols, "income", ">50K", "equal_frequency") == \
        {"education-num": 18, "hours-per-week": 6}


@pytest.mark.parametrize("cell", sorted(IV_IG_CELLS))
def test_oracle_iv_ig_example_6(income_spark, nb_assoc, cell):
    col, fn = IV_IG_CELLS[cell]
    got = fn(income_spark, ["age", "sex", "race", "workclass", "fnlwgt"], label_col="income", event_label=">50K",
             encoding_configs=ENC)
    exp = {r[0]: r[1] for r in nb_assoc[cell]["rows"]}
    assert set(got["attribute"]) == set(exp)
    for a, v in zip(got["attribute"], got[col]):
        assert "%.6f" % v == exp[a], (cell, a, v, exp[a])


def test_oracle_refuses_an_all_null_equal_range_column():
    t = pa.table({"x": pa.array([None, None, None], pa.float64()), "label": [1, 0, 1]})
    with pytest.raises(ValueError, match="no non-null"):
        MO.monotonic_binning(t, ["x"])


# ---- the decision -----------------------------------------------------------------------------------------------------

def _monotone(k):
    count = np.array([0] + [10] * k)
    return count, np.array([0] + list(range(1, k + 1)))


@pytest.mark.parametrize("k", range(2, 21))
def test_perfectly_monotone_tables_follow_scipy(k):
    # scipy 1.18.1 gives 0.9999999999999999 for 2, 5 and 10 groups: those are rejected, as the reference rejects them
    count, events = _monotone(k)
    assert M.accepts(count, events) == (k not in (2, 5, 10))
    assert M.accepts(count, events) == (M.spearman_r(np.arange(k), events[1:] / 10) == 1.0)


def test_decreasing_ties_single_group_and_empty_bins():
    count, events = _monotone(4)
    assert not M.accepts(count, events[::-1].copy())                 # decreasing event rate: r = -1
    assert not M.accepts(count, np.array([0, 1, 2, 2, 3]))          # a tie
    assert math.isnan(M.spearman_r([1.0], [0.5]))                   # one group: NaN, rejected
    assert not M.accepts(np.array([0, 10, 0, 0, 0]), np.array([0, 3, 0, 0, 0]))
    # empty bins are skipped: bins 1, 3, 4, 6 hold rows and rise -> 4 groups, accepted
    assert M.accepts(np.array([0, 10, 0, 10, 10, 0, 10]), np.array([0, 1, 0, 2, 3, 0, 4]))
    # dropping bin 4 leaves 1, 3, 6 -> 3 groups, accepted; a falling bin that is dropped no longer counts
    assert M.accepts(np.array([0, 10, 0, 10, 10, 0, 10]), np.array([0, 1, 0, 2, 9, 0, 4]), drop={4})


def test_nan_and_infinity_bins():
    um = M.UnionModel({n: [float(j) for j in range(1, n)] for n in M.LADDER}, _lib.ANV_F64)
    x = np.array([0.5, 1.5, np.nan, 2.5])
    c = stand_in_counts(x, np.ones(4, bool), np.array([0, 1, 1, 1]), np.ones(4, bool), um)
    assert M.nan_mean_bins(um, c, 5) == {5}
    # -inf and +inf fall into bins 1 and n: apart, their bins average to -inf / +inf and stay
    x = np.array([-np.inf, np.inf, 3.5])
    c = stand_in_counts(x, np.ones(3, bool), np.array([0, 1, 1]), np.ones(3, bool), um)
    assert M.nan_mean_bins(um, c, 7) == set()
    # every cutoff +inf: no threshold is below +inf, so both infinities share bin 1 -> NaN
    um = M.UnionModel({n: [math.inf] * (n - 1) for n in M.LADDER}, _lib.ANV_F64)
    c = stand_in_counts(x, np.ones(3, bool), np.array([0, 1, 1]), np.ones(3, bool), um)
    assert M.nan_mean_bins(um, c, 9) == {1}


# ---- union slots against direct binning ---------------------------------------------------------------------------------

def _values(rng, dtype, n):
    if dtype == _lib.ANV_I32:
        return np.concatenate([rng.integers(-50, 50, n), [np.iinfo(np.int32).min, np.iinfo(np.int32).max]]).astype(np.int32)
    if dtype == _lib.ANV_I64:
        big = 1 << 62
        return np.concatenate([rng.integers(-60, 60, n), [-(1 << 63), (1 << 63) - 1, big, big + 1, big - 1,
                                                          (1 << 53) + 1]]).astype(np.int64)
    T = np.float32 if dtype == _lib.ANV_F32 else np.float64
    return np.concatenate([rng.normal(0, 30, n), [np.inf, -np.inf, np.nan, 0.0, -0.0]]).astype(T)


def _adversarial_cuts(rng, dtype, kind):
    out = {}
    for n in M.LADDER:
        if kind == "random":
            c = sorted(rng.normal(0, 30, n - 1).tolist())
        elif kind == "duplicates":                     # equal_frequency on a few distinct values
            c = sorted(rng.integers(-3, 3, n - 1).astype(float).tolist())
        elif kind == "nan":
            c = [float("nan")] * (n - 1)
        elif kind == "inf":
            c = [-math.inf] + [float(j) for j in range(1, n - 2)] + [math.inf]
        elif kind == "fractional":                     # int floors
            c = [j + 0.5 - n // 2 for j in range(n - 1)]
        else:                                          # bigint beyond 2^53
            c = [float((1 << 62) + j * 4096) for j in range(n - 1)]
        out[n] = c
    return out


@pytest.mark.parametrize("dtype", [_lib.ANV_F32, _lib.ANV_F64, _lib.ANV_I32, _lib.ANV_I64])
@pytest.mark.parametrize("kind", ["random", "duplicates", "nan", "inf", "fractional", "bigint"])
def test_union_slots_equal_direct_binning(dtype, kind):
    rng = np.random.default_rng([dtype, len(kind), ord(kind[0]), ord(kind[-1])])
    cuts = _adversarial_cuts(rng, dtype, kind)
    x = _values(rng, dtype, 400)
    if kind == "bigint" and dtype == _lib.ANV_I64:
        x = np.concatenate([x, np.array([(1 << 62) + j * 1024 for j in range(-8, 80000, 997)], np.int64)])
    valid = rng.random(len(x)) > 0.1
    lab = rng.integers(0, 2, len(x))
    lab_valid = rng.random(len(x)) > 0.1
    um = M.UnionModel(cuts, dtype)
    assert len(um.thresholds) <= 189 and np.all(um.thresholds[1:] > um.thresholds[:-1])
    counts = stand_in_counts(x, valid, lab, lab_valid, um)
    for n, cut in cuts.items():
        # each model on its own, as K2 bins it: 1 + #(native threshold < x), NaN in bin n
        th = np.sort(M.typed_thresholds(cut, dtype))
        ids = 1 + np.searchsorted(th, x, side="left")
        if x.dtype.kind == "f":
            ids = np.where(np.isnan(x), n, ids)
        if kind != "nan" and not (kind == "inf" and x.dtype.kind == "i"):
            # bucket_label itself, where the native thresholds carry it exactly (a NaN cutoff becomes the lowest value,
            # and -inf on an integer column its minimum, which the minimum itself is not above)
            assert np.array_equal(np.where(valid, ids, 0), S.assign_bins(x, valid, cut, n)), (n, kind)
        ids = np.where(valid, ids, 0)
        a, e, ne = M.model_table(um, counts, n)
        ev = lab_valid & (lab == 1)
        nev = lab_valid & (lab != 1)
        assert a.tolist() == np.bincount(ids, minlength=n + 1).tolist(), (n, kind)
        assert e.tolist() == np.bincount(ids[ev], minlength=n + 1).tolist()
        assert ne.tolist() == np.bincount(ids[nev], minlength=n + 1).tolist()


# ---- the host decision chain against the oracle ---------------------------------------------------------------------------

@pytest.mark.parametrize("method", ["equal_range", "equal_frequency"])
def test_host_chain_chooses_what_the_oracle_chooses(income_spark, method):
    """Oracle cutoffs -> UnionModel -> stand-in counts -> choose(), against the oracle's groupBy with the real avg(x)."""
    cols = ["age", "fnlwgt", "education-num", "hours-per-week", "capital-gain", "logfnl"]
    exp = MO.chosen_bins(income_spark, cols, "income", ">50K", method)
    label01 = MO._label01(income_spark, "income", ">50K")
    _, lab_valid = S.column_values(income_spark, "income")
    for c in cols:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            cuts = {n: O.binning_cutoffs(income_spark, [c], method, n)[1][0] for n in M.LADDER}
        vals, valid = S.column_values(income_spark, c)
        anv = {"float": _lib.ANV_F32, "double": _lib.ANV_F64, "int": _lib.ANV_I32}.get(
            S.spark_dtype(income_spark.schema.field(c).type), _lib.ANV_I64)
        x = np.where(valid, vals, 0).astype(_NP[anv])
        um = M.UnionModel(cuts, anv)
        assert M.choose(um, stand_in_counts(x, valid, label01, lab_valid, um)) == exp[c], c
