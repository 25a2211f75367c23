"""bigint columns beyond 2^53 through the public API, product vs oracle cell for cell.

A double holds every int64 only up to 2^53, so a comparison through float64 cannot see a bigint result that is off in its
low digits.  Here the mode, the distinct counts and the treated outlier columns of bigint columns are compared as exact
integers or strings (Spark returns the mode of a bigint column as a long and renders it with Long.toString), while the
values Spark itself computes through double - percentiles, moments, the reference's outlier compare `v.astype(float)` -
are compared as doubles.  Column families: epoch-nanosecond timestamps (doubles are 256 apart there), odd values
straddling +-2^53, the int64 extremes, a mode tie between 2^53 and 2^53 + 1 (one double, two keys) and a column with one
non-null value."""
import math
import os
import socket
import warnings

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu

from oracle import api as O
from oracle import row_checks as RC

N = 200_003
TWO53 = 1 << 53
TS0 = 1_600_000_000_000_000_000
TS_MODE = TS0 + 123_457                    # odd, so not a double: neighbouring doubles are 256 apart at 1.6e18
SINGLE = (1 << 62) + 3                     # not a double either (1 024 apart)
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
BIG = ["ts_ns", "straddle", "extremes", "tie", "single"]


def bigint_table(n=N, seed=5):
    rng = np.random.default_rng(seed)
    nulls = lambda: rng.random(n) < 0.05
    ts = TS0 + rng.integers(0, 1 << 22, n)
    ts[rng.random(n) < 0.01] = TS_MODE
    k = rng.integers(0, 3000, n)
    strad = np.where(rng.random(n) < 0.5, 1, -1) * (TWO53 + 2 * k + 1)
    ext = np.array([(1 << 62) + 1, -(1 << 62) - 1, I64_MAX, I64_MAX - 1, I64_MIN, I64_MIN + 1], np.int64)
    a = 2 * n // 5
    tie = rng.permutation(np.concatenate([np.full(a, TWO53), np.full(a, TWO53 + 1), 10 + np.arange(n - 2 * a)]))
    single = np.zeros(n, np.int64)
    one = int(rng.integers(0, n))
    single[one] = SINGLE
    return pa.table({
        "ts_ns": pa.array(ts.astype(np.int64), mask=nulls()),
        "straddle": pa.array(strad.astype(np.int64), mask=nulls()),
        "extremes": pa.array(ext[rng.integers(0, ext.size, n)]),                       # the null-free column
        "tie": pa.array(tie.astype(np.int64), mask=(tie < TWO53) & (rng.random(n) < 0.5)),   # nulls off the tie
        "single": pa.array(single, mask=np.arange(n) != one),
        "f32": pa.array(rng.normal(0, 10, n).astype(np.float32), mask=nulls()),
    })


@pytest.fixture(scope="module")
def table():
    return bigint_table()


def _native(t, c):
    a = t.column(c).combine_chunks()
    return np.asarray(a.fill_null(0)), np.asarray(a.is_valid())


def _exact_mode(x):
    """(mode, rows, distinct) of the non-null values: smallest value among ties (the product's documented rule)."""
    u, k = np.unique(x, return_counts=True)
    return u[np.argmax(k)].item(), int(k.max()), int(u.size)


def test_tables_are_what_they_claim(table):
    """The planted values sit where the tests need them: a double cannot tell them from their neighbours."""
    ts, v = _native(table, "ts_ns")
    assert float(TS_MODE) != TS_MODE and float(SINGLE) != SINGLE and float(TWO53 + 1) == float(TWO53)
    assert _exact_mode(ts[v])[0] == TS_MODE
    assert np.unique(ts[v]).size > np.unique(ts[v].astype(np.float64)).size         # neighbours collide as doubles
    x, v = _native(table, "tie")
    assert _exact_mode(x[v])[:2] == (TWO53, 2 * N // 5) and (x[v] == TWO53 + 1).sum() == 2 * N // 5
    assert int(np.asarray(table.column("single").is_valid()).sum()) == 1
    assert table.column("extremes").null_count == 0
    with pytest.raises(AssertionError):
        assert str(int(float(TS_MODE))) == str(TS_MODE)


# ---- engine level -----------------------------------------------------------------------------------------------

@pytest.fixture(params=["partition", "lsd"])
def sort_algorithm(request):
    from anovos_b200 import engine
    old, engine.sort_algorithm = engine.sort_algorithm, request.param
    yield request.param
    engine.sort_algorithm = old


def _check_engine_modes(t, fr, names):
    from anovos_b200 import engine
    rk = []
    for c in names:
        nv = int(np.asarray(t.column(c).is_valid()).sum())
        rk.append([1, max(1, nv // 2), nv] if nv else [0, 0, 0])
    got, qv = engine.sort_mode_distinct(fr, names, np.array(rk, np.int64))
    for i, c in enumerate(names):
        x, v = _native(t, c)
        x = x[v]
        if t.schema.field(c).type == pa.int64():
            mode, rows, nd = _exact_mode(x)
            assert type(got[i][0]) is int, (c, got[i])                              # an exact int, not a float
            assert got[i] == (mode, rows, nd), (c, got[i], (mode, rows, nd))
        else:
            mode, rows, nd = _exact_mode(x.astype(np.float64) + 0.0)
            assert type(got[i][0]) is float and got[i] == (mode, rows, nd), (c, got[i])
        srt = np.sort(x)                                                           # exact order, then rounded: Spark's
        exp = [float(srt[r - 1]) for r in rk[i]]                                   # percentiles of a bigint are doubles
        assert qv[i].dtype == np.float64 and np.array_equal(qv[i], exp), (c, qv[i], exp)


def test_engine_mode_distinct_exact(table, sort_algorithm):
    """Exact int64 modes next to float32 columns in one call: the int64 group takes the LSD sort, the float32 group the
    bucket count under "partition", and both must come back right."""
    from anovos_b200.frame import ColumnFrame
    _check_engine_modes(table, ColumnFrame.from_arrow(table), table.column_names)


def test_engine_mode_distinct_exact_over_a_million_rows(sort_algorithm):
    """Over a million rows the LSD sort works through many tiles and the merge folds their run summaries."""
    from anovos_b200.frame import ColumnFrame
    t = bigint_table(1_048_576 + 4099, seed=9).select(["ts_ns", "straddle", "tie", "f32"])
    _check_engine_modes(t, ColumnFrame.from_arrow(t), t.column_names)


# ---- the public API, resident and chunked ---------------------------------------------------------------------------

def _same(got, exp, what):
    """Cell-wise equality: exact for numbers and strings (an int never equals a float that rounded it), NaN == None."""
    got = got.toPandas() if hasattr(got, "toPandas") else got
    assert list(got.columns) == list(exp.columns) and len(got) == len(exp), (what, got, exp)
    for c in got.columns:
        for a, b in zip(got[c].tolist(), exp[c].tolist()):
            assert (pd.isna(a) and pd.isna(b)) or a == b, (what, c, a, b)


# ts_ns holds 19-digit values with a spread of 7 digits: its second moment cancels 12 digits of each value, and the FP64
# moments of the kernels keep its stddev to about 1e-7 (Spark's own double accumulation keeps less).  Every other column
# is held to 1e-9.
RTOL = {"ts_ns": 1e-6}


def _close(got, exp, what, cols):
    got = got.toPandas() if hasattr(got, "toPandas") else got
    assert list(got["attribute"]) == list(exp["attribute"]), what
    rtol = np.array([RTOL.get(a, 1e-9) for a in got["attribute"]])
    for c in cols:
        g, e = got[c].to_numpy(np.float64, na_value=np.nan), exp[c].to_numpy(np.float64, na_value=np.nan)
        ok = np.isclose(g, e, rtol=rtol, atol=1.01e-4, equal_nan=True)     # atol: shown values are rounded to 4 decimals
        assert ok.all(), (what, c, g, e)


def _frame(table, kind):
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.partitioned import PartitionedFrame
    if kind == "resident":
        return ColumnFrame.from_arrow(table)
    return PartitionedFrame.from_frame(table, 12_000)          # 375 * 32 rows: not a multiple of the 4 096-row sort tile


@pytest.mark.parametrize("kind", ["resident", "chunked"])
def test_stats_exact_against_oracle(table, kind, tmp_path):
    import anovos.data_analyzer.quality_checker as qc
    import anovos.data_analyzer.stats_generator as sg
    from anovos.data_report.report_preprocessing import save_stats
    fr = _frame(table, kind)
    if kind == "chunked":
        assert fr.n_chunks == -(-N // 12_000)
    mode = sg.mode_computation(None, fr).toPandas()
    exp = O.mode_computation(table)
    _same(mode, exp, "mode_computation")
    by = dict(zip(mode["attribute"], mode["mode"]))
    assert by["ts_ns"] == str(TS_MODE) and by["tie"] == str(TWO53) and by["single"] == str(SINGLE), by
    ct = sg.measures_of_centralTendency(None, fr).toPandas()
    ect = O.measures_of_centralTendency(table)
    _same(ct[["attribute", "mode", "mode_rows", "mode_pct", "median"]],
          ect[["attribute", "mode", "mode_rows", "mode_pct", "median"]], "measures_of_centralTendency")
    _close(ct, ect, "measures_of_centralTendency", ["mean"])
    save_stats(None, sg.measures_of_centralTendency(None, fr), str(tmp_path), "central")
    back = pd.read_csv(tmp_path / "central.csv", dtype={"mode": str})
    assert back["mode"].tolist() == ect["mode"].tolist()
    _same(sg.uniqueCount_computation(None, fr).toPandas(), O.uniqueCount_computation(table), "uniqueCount_computation")
    for kw in ({}, {"rsd": 0.02}):
        _same(sg.measures_of_cardinality(None, fr, **kw).toPandas(), O.measures_of_cardinality(table, **kw),
              ("measures_of_cardinality", kw))
    _same(sg.measures_of_counts(None, fr).toPandas(), O.measures_of_counts(table), "measures_of_counts")
    _same(sg.measures_of_percentiles(None, fr).toPandas(), O.measures_of_percentiles(table), "measures_of_percentiles")
    _close(sg.measures_of_dispersion(None, fr), O.measures_of_dispersion(table), "measures_of_dispersion",
           ["stddev", "variance", "cov", "IQR", "range"])
    _close(sg.measures_of_shape(None, fr), O.measures_of_shape(table), "measures_of_shape", ["skewness", "kurtosis"])
    # the quality checks take the discrete columns: every bigint one, not the float32 one
    card = O.measures_of_cardinality(table, BIG)
    _, idn = qc.IDness_detection(None, fr)
    _same(idn.toPandas()[["attribute", "unique_values", "IDness"]], card, "IDness_detection")
    _, bias = qc.biasedness_detection(None, fr)
    _same(bias.toPandas()[["attribute", "mode", "mode_rows", "mode_pct"]],
          ect[ect["attribute"].isin(BIG)].reset_index(drop=True)[["attribute", "mode", "mode_rows", "mode_pct"]],
          "biasedness_detection")


@pytest.mark.parametrize("bin_method", ["equal_range", "equal_frequency"])
def test_drift_statistics_against_oracle(table, bin_method, tmp_path):
    import anovos.drift_stability.drift_detector as dd
    tgt = bigint_table(N - 777, seed=6)
    cols = ["ts_ns", "straddle", "extremes", "tie"]
    kw = dict(list_of_cols=cols, method_type="all", bin_method=bin_method, use_sampling=False)
    got = dd.statistics(None, tgt, table, source_path=str(tmp_path / "g"), **kw).toPandas()
    exp = O.statistics(tgt, table, source_path=str(tmp_path / "o"), **kw)
    assert got["attribute"].tolist() == exp["attribute"].tolist()
    for m in ("PSI", "HD", "JSD", "KS"):
        assert np.allclose(got[m].to_numpy(float), np.asarray(exp[m], float), rtol=1e-9, atol=1e-12), (bin_method, m)
    assert got["flagged"].tolist() == exp["flagged"].tolist()


def test_duplicates_that_differ_below_double_precision():
    """Rows equal as doubles but not as int64 are distinct rows."""
    import anovos.data_analyzer.quality_checker as qc
    rng = np.random.default_rng(13)
    n = 50_000
    a = TS0 + rng.integers(0, 64, n)                 # 64 keys, all within one double of each other (256 apart)
    b = np.where(rng.random(n) < 0.5, TWO53, TWO53 + 1)
    t = pa.table({"a": pa.array(a.astype(np.int64)), "b": pa.array(b.astype(np.int64), mask=rng.random(n) < 0.05)})
    assert np.unique(a.astype(np.float64)).size <= 2
    odf, stats = qc.duplicate_detection(None, t, print_impact=True)
    eodf, estats = RC.duplicate_detection(t, print_impact=True)
    assert stats.toPandas().values.tolist() == estats.values.tolist()
    assert estats["value"][1] > 64 * 2                # more distinct rows than there are distinct doubles
    assert odf.count() == eodf.num_rows
    for c in ("a", "b"):
        d, v = odf.column(c).device()
        e = eodf.column(c).combine_chunks()
        valid = np.asarray(e.is_valid())
        assert np.array_equal(d.cpu().numpy()[valid], np.asarray(e.fill_null(0))[valid]), c


# ---- outlier flags: the reference rounds each value to double before it compares -----------------------------------

def _ref_flags(x, lo, hi):
    """The reference's compare (`v.astype(float)`, then `v - lower < 0` / `v - upper > 0`) -> (low, up) bool arrays."""
    f = x.astype(np.float64)
    with np.errstate(invalid="ignore"):
        return ((f - lo) < 0) if lo is not None else np.zeros(x.size, bool), ((f - hi) > 0) if hi is not None else np.zeros(x.size, bool)


def _check_outliers(got_t, got_p, exp_t, exp_p, what):
    from anovos_b200.frame import ColumnFrame
    gp = got_p.toPandas()
    assert gp.values.tolist() == exp_p.values.tolist(), (what, gp, exp_p)
    assert got_t.count() == exp_t.num_rows and got_t.columns == exp_t.column_names, what
    for c in exp_t.column_names:
        e = exp_t.column(c).combine_chunks()
        valid = np.asarray(e.is_valid())
        d, v = got_t.column(c).device()
        g = d.cpu().numpy()
        ev = np.asarray(e.fill_null(0))
        assert g.dtype == ev.dtype, (what, c, g.dtype, ev.dtype)                  # bigint stays bigint: exact compare
        assert np.array_equal(g[valid], ev[valid]), (what, c)
        gv = np.ones(len(g), bool) if v is None else ColumnFrame({c: got_t.column(c)}, got_t.count()).valid_mask(c).cpu().numpy()
        assert np.array_equal(gv, valid), (what, c)


GAP_BOUNDS = {  # [lower, upper] doubles >= 2^53: the exact compare and the compare through double disagree next to them
    "ts_ns": [float(TS0 + 1_000_000), float(TS0 + 3_000_000)],
    "straddle": [float(TWO53 + 2), float(TWO53 + 4000)],
}


def _gap_table():
    """bigint_table's ts_ns / straddle with rows planted in the gaps of GAP_BOUNDS: v = upper + 1 rounds down to upper (not
    an outlier in the reference), and v just below lower rounds down to the double below lower (an outlier there)."""
    t = bigint_table(50_000, seed=7).select(["ts_ns", "straddle"])
    cols = {}
    for c, (lo, hi) in GAP_BOUNDS.items():
        x, v = _native(t, c)
        x = x.copy()
        x[:40] = int(hi) + 1
        x[40:80] = int(lo) - (200 if c == "ts_ns" else 1)    # 200 of 256: nearer the double below lower
        cols[c] = pa.array(x, mask=~v)
    return pa.table(cols)


def test_outlier_planted_rows_fall_in_the_gap():
    """The test below fails on an exact int64 compare, for the reason it is there: on the planted rows the reference's
    flags differ from `v > floor(upper)` / `v <= floor(prev_double(lower))`."""
    t = _gap_table()
    for c, (lo, hi) in GAP_BOUNDS.items():
        x, v = _native(t, c)
        low, up = _ref_flags(x, lo, hi)
        exact_up = x > math.floor(hi)
        exact_low = x <= math.floor(np.nextafter(lo, -np.inf))
        assert (exact_up[:40] & ~up[:40] & v[:40]).sum() >= 30, c           # exact: flagged; reference: not
        assert (low[40:80] & ~exact_low[40:80] & v[40:80]).sum() >= 30, c  # reference: flagged; exact: not


@pytest.mark.parametrize("side", ["upper", "lower", "both"])
def test_outlier_flags_through_double_with_a_saved_model(side, tmp_path):
    import anovos.data_analyzer.quality_checker as qc
    from anovos_b200.data_analyzer.quality_checker import _save_outlier_model
    t = _gap_table()
    cols = list(GAP_BOUNDS)
    params = [[b[0] if side != "upper" else None, b[1] if side != "lower" else None] for b in GAP_BOUNDS.values()]
    _save_outlier_model(str(tmp_path), cols, params)
    for method in ("value_replacement", "null_replacement", "row_removal"):
        for mode in ("replace", "append"):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                got_t, got_p = qc.outlier_detection(None, t, detection_side=side, treatment_method=method, output_mode=mode,
                                                    pre_existing_model=True, model_path=str(tmp_path), print_impact=True)
            exp_t, exp_p = O.outlier_detection(t, detection_side=side, treatment_method=method, output_mode=mode,
                                               params=(cols, params, []))
            _check_outliers(got_t, got_p, exp_t, exp_p, (side, method, mode))
    # the histogram path of a chunked frame counts the same flags
    _, hp = qc.outlier_detection(None, _frame(t, "chunked"), detection_side=side, treatment=False, pre_existing_model=True,
                                 model_path=str(tmp_path), print_impact=True)
    assert hp.toPandas().values.tolist() == exp_p.values.tolist(), side


@pytest.mark.parametrize("side", ["upper", "lower", "both"])
def test_outlier_detection_against_oracle(table, side, tmp_path):
    """Bounds from the data (percentiles, mean +- 3 sd, IQR), every treatment and output mode, then the saved model's
    round trip: written with model_path, read back with pre_existing_model=True."""
    import anovos.data_analyzer.quality_checker as qc
    from anovos_b200.data_analyzer.quality_checker import _load_outlier_model
    t = table.select(["ts_ns", "straddle", "extremes", "tie", "f32"])
    for method in ("value_replacement", "null_replacement", "row_removal"):
        for mode in ("replace", "append"):
            got_t, got_p = qc.outlier_detection(None, t, detection_side=side, treatment_method=method, output_mode=mode,
                                                print_impact=True)
            exp_t, exp_p = O.outlier_detection(t, detection_side=side, treatment_method=method, output_mode=mode)
            _check_outliers(got_t, got_p, exp_t, exp_p, (side, method, mode))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        qc.outlier_detection(None, t, detection_side=side, treatment=False, model_path=str(tmp_path))
        model = _load_outlier_model(str(tmp_path))
        got_t, got_p = qc.outlier_detection(None, t, detection_side=side, treatment_method="null_replacement",
                                            pre_existing_model=True, model_path=str(tmp_path), print_impact=True)
    kept = [c for c in t.column_names if c in model and "skewed_attribute" not in model[c]]
    skewed = [c for c in t.column_names if c in model and "skewed_attribute" in model[c]]
    params = [[float(v) if v else None for v in model[c]] for c in kept]
    exp_t, exp_p = O.outlier_detection(t, kept, detection_side=side, treatment_method="null_replacement",
                                       params=(kept, params, skewed))
    _check_outliers(got_t, got_p, exp_t, exp_p, (side, "saved model"))


# ---- two ranks with gloo on one GPU: the mode travels through the summary all_gather -----------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


SLAB0 = 90_000 // 32 * 32


def _rank_worker(rank, world, port, ret):
    import torch.distributed as dist
    import anovos.data_analyzer.stats_generator as sg
    from anovos_b200.partitioned import PartitionedFrame
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    t = bigint_table()
    r0, r1 = (0, SLAB0) if rank == 0 else (SLAB0, N)
    parts = PartitionedFrame.from_frame(t.slice(r0, r1 - r0), 16_384, group=True)
    ret[rank] = {fn: getattr(sg, fn)(None, parts).toPandas().to_dict("list")
                 for fn in ("mode_computation", "measures_of_centralTendency", "uniqueCount_computation")}
    dist.destroy_process_group()


def test_two_ranks_row_slabs_exact_bigint_mode(table):
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ret = mp.get_context("spawn").Manager().dict()
    mp.spawn(_rank_worker, args=(world, port, ret), nprocs=world, join=True)
    a, b = ret[0], ret[1]
    assert repr(a) == repr(b)
    _same(pd.DataFrame(a["mode_computation"]), O.mode_computation(table), "mode_computation")
    ect = O.measures_of_centralTendency(table)
    cols = ["attribute", "mode", "mode_rows", "mode_pct", "median"]
    _same(pd.DataFrame(a["measures_of_centralTendency"])[cols], ect[cols], "measures_of_centralTendency")
    _same(pd.DataFrame(a["uniqueCount_computation"]), O.uniqueCount_computation(table), "uniqueCount_computation")
