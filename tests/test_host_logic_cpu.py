"""Host-side arithmetic of the product that has a scalar definition and a vectorised fast path: the fast path must be
bit-identical.  CPU only (no kernel is launched)."""
import numpy as np
import pandas as pd
import pytest

from anovos_b200 import engine, parallel
from anovos_b200.data_analyzer import stats_generator as sg
from anovos_b200.shared.utils import jvm_double_str, spark_round, spark_round_array
from oracle import spark_semantics as S


def test_spark_round_array_equals_scalar_half_up():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.normal(0, 100, 20000), rng.normal(0, 1e6, 5000), np.round(rng.normal(0, 10, 5000), 4) + 0.00005,
                        [0.12345, 1.00005, 2.5e-5, -0.00005, 1e12, -1e15, 0.0, np.nan, np.inf]])
    got = spark_round_array(x)
    exp = np.array([np.nan if v != v else spark_round(v) for v in x.tolist()])
    assert np.array_equal(got, exp, equal_nan=True)
    assert spark_round(0.12345) == S.round_half_up(0.12345) == 0.1235      # HALF_UP on the shortest repr, not half-even
    assert np.array_equal(spark_round_array(np.array([[0.00005, np.nan]])), np.array([[0.0001, np.nan]]), equal_nan=True)


def test_float32_display_shortcut_is_exact():
    """Float.toString round trip of FloatType values is skipped when it cannot change round(x, 4): same result as
    always converting, for single values and for differences (IQR, range)."""
    rng = np.random.default_rng(1)
    for scale in (1e-3, 1.0, 30.0, 1e3, 1e5):
        x = rng.normal(0, scale, 50000).astype(np.float32).astype(np.float64)
        full = spark_round_array(sg._f32_trip(x))
        need = sg._near_tie(x, np.abs(x) * sg._F32_EPS)
        y = x.copy()
        y[need] = sg._f32_trip(y[need])
        assert np.array_equal(full, spark_round_array(y)), scale
        a = rng.normal(0, scale, 50000).astype(np.float32).astype(np.float64)
        b = (a + np.abs(rng.normal(0, scale, 50000))).astype(np.float32).astype(np.float64)
        d = b - a
        nd = sg._near_tie(d, (np.abs(a) + np.abs(b)) * sg._F32_EPS)
        d[nd] = sg._f32_trip(b[nd]) - sg._f32_trip(a[nd])
        assert np.array_equal(spark_round_array(sg._f32_trip(b) - sg._f32_trip(a)), spark_round_array(d)), scale
    assert sg._f32_trip(np.array([np.float64(np.float32(0.1))]))[0] == 0.1


def test_hll_estimates_rows_equal_scalar():
    rng = np.random.default_rng(2)
    for p in (4, 9, 12, 14):
        R = rng.integers(0, 25, (30, 1 << p)).astype(np.uint32)
        R[:5] = 0
        R[5:10] = (rng.random((5, 1 << p)) < 0.02) * 3
        R[10:15] = (rng.random((5, 1 << p)) < 0.6) * rng.integers(1, 4, (5, 1 << p))
        assert engine.hll_estimates_from_register_rows(R, p) == [engine.hll_estimate_from_registers(R[i], p) for i in range(30)]
        assert engine.hll_estimate_from_registers(R[0], p) == (0, False)


def test_jvm_double_strings():
    for x, s in ((1.0, "1.0"), (5.093362141, "5.093362141"), (1e7, "1.0E7"), (12345678.9, "1.23456789E7"), (0.001, "0.001"),
                 (0.0001, "1.0E-4"), (-0.0, "-0.0"), (float("nan"), "NaN"), (float("inf"), "Infinity"), (100.0, "100.0")):
        assert jvm_double_str(x) == s, (x, jvm_double_str(x))
        assert S.java_double_to_string(x) == s


def test_frames_to_matrix_mixed_dtypes():
    f1 = pd.DataFrame({"attribute": ["a", "b"], "mean": [1.5, None], "mode": ["x", None], "mode_rows": [3, None]})
    f2 = pd.DataFrame({"attribute": ["a", "b"], "count": np.array([4, 5], dtype=np.int64),
                       "nullable": pd.array([1, None], dtype="Int64")})
    m, names = parallel.frames_to_matrix([f1, f2])
    assert names == ["mean", "mode_rows", "count", "nullable"]
    assert np.array_equal(m, np.array([[1.5, 3, 4, 1], [np.nan, np.nan, 5, np.nan]]), equal_nan=True)


def test_drift_argument_normalisers_contract():
    """validations.py:8-94 as behaviour: keyword-only reading, "all" = num + cat of the target, '|' strings, drops,
    first-seen de-duplication, error types (reference test_validations.py:13-20 checks the ValueErrors)."""
    import pyarrow as pa
    import pytest
    from anovos_b200.drift_stability.validations import check_distance_method, check_list_of_columns
    t = pa.table({"a": [1.0, 2.0], "b": ["x", "y"], "c": [1, 2], "d": pa.array([True, False])})

    @check_distance_method
    @check_list_of_columns
    def f(spark, idf_target, idf_source, *, list_of_cols="all", drop_cols=None, method_type="PSI"):
        return list_of_cols, drop_cols, method_type

    assert f(None, t, t) == (["a", "c", "b"], [], ["PSI"])                       # bool column is neither num nor cat
    assert f(None, t, t, list_of_cols="a| b |a", drop_cols="b") == (["a"], [], ["PSI"])
    assert f(None, idf_target=t, idf_source=t, list_of_cols=["c", "a", "c"], method_type="all") == (["c", "a"], [], ["PSI", "JSD", "HD", "KS"])
    assert f(None, t, t, method_type="KS|HD")[2] == ["KS", "HD"]
    with pytest.raises(ValueError):
        f(None, t, t, list_of_cols=["a"], drop_cols=["a"])
    with pytest.raises(ValueError):
        f(None, t, t, list_of_cols="zz")
    with pytest.raises(TypeError):
        f(None, t, t, list_of_cols=3)
    with pytest.raises(TypeError):
        f(None, t, t, drop_cols=3)
    with pytest.raises(TypeError):
        f(None, t, t, method_type="XYZ")

    @check_list_of_columns(columns="cols", drop="drops")
    def g(spark, idf_target, *, cols="all", drops=None):
        return cols, drops
    assert g(None, t, cols="b|c") == (["b", "c"], [])


def test_frames_to_matrix_aligns_frames_of_different_row_counts():
    """Mixed frames (the default bench workload): counts / centralTendency / cardinality cover string columns, the
    numeric-only functions do not - the summary matrix of the N > 1 exchange is aligned on `attribute`, NaN where a
    function has no row for a column."""
    import pandas as pd
    from anovos_b200 import parallel
    f1 = pd.DataFrame({"attribute": ["a", "s", "b"], "fill_count": [3, 2, 3], "mode": ["1", "x", None]})
    f2 = pd.DataFrame({"attribute": ["a", "b"], "stddev": [0.5, None], "range": [1.0, 2.0]})
    m, names = parallel.frames_to_matrix([f1, f2])
    assert names == ["fill_count", "stddev", "range"] and m.shape == (3, 3)
    assert m[:, 0].tolist() == [3.0, 2.0, 3.0]
    assert m[0, 1] == 0.5 and np.isnan(m[1, 1]) and np.isnan(m[2, 1])
    assert m[0, 2] == 1.0 and np.isnan(m[1, 2]) and m[2, 2] == 2.0


def test_result_frames_equal_the_plain_pandas_constructor():
    """ResultFrame.from_columns builds its frame through pandas' array constructor: values AND dtypes must be the ones
    pd.DataFrame(dict) infers; every toPandas() hands out an independent frame."""
    import numpy as np
    import pandas as pd
    from anovos_b200.result import ResultFrame, build_frame
    cases = [
        {"attribute": ["a", "b", "c"], "n": np.array([1, 2, 3], dtype=np.int64), "x": np.array([0.5, np.nan, 2.0]),
         "mode": ["1.0", None, "x"], "none": [None, None, None], "mixed": [1.5, None, 2.0]},
        {"attribute": [], "x": np.zeros(0)},
        {"attribute": ["only"], "flag": np.array([True]), "s": ["v"]},
    ]
    for cols in cases:
        exp = pd.DataFrame({k: (v.copy() if isinstance(v, np.ndarray) else list(v)) for k, v in cols.items()})
        got = build_frame(cols)
        assert list(got.columns) == list(exp.columns) and got.dtypes.tolist() == exp.dtypes.tolist(), (got.dtypes, exp.dtypes)
        assert got.equals(exp)
        rf = ResultFrame.from_columns(cols, attrs={"k": [1]})
        a, b = rf.toPandas(), rf.toPandas()
        assert a.equals(exp) and a.attrs == {"k": [1]} and rf.columns == list(cols) and rf.count() == len(exp)
        if len(a):
            a.iloc[0, 0] = "changed"
            assert b.equals(exp) and rf.toPandas().equals(exp)
            assert rf.where({"attribute": cols["attribute"][0]}).count() == 1


def _f32(x):
    return np.float32(x)


def _fma_f32(a, b, c):
    """round-to-nearest float32 of a * b + c (a, b, c float32): the product is exact in float64 / longdouble."""
    return np.float32(np.longdouble(np.float64(a) * np.float64(b)) + np.longdouble(c))


@pytest.mark.parametrize("seed", range(6))
def test_folded_bin_guess_stays_within_one_bin_of_the_exact_slot(seed):
    """NumPy restatement of the device's folded equal_range guess (csrc/scan_impl.cuh, FastF32::counter_addr<FOLD> and
    fold_ok): v = sat(x * (-c) + k), k = 1 + lo * c, r' = round(v * (B-1)), r = B-1-r', slot = r + !(x <= S[r]).  The exact
    threshold compare only repairs a guess that is at most one bin off, so the property to hold wherever fold_ok lets the
    fold run is: the exact 0-based bin b = #(theta_i < x) lies in {r-1, r}.  Ranges at the edge of the fold_ok bound (|lo| / w
    close to 2^18), values on and next to every threshold, the ends of the range, values outside it, NaN and infinities."""
    from anovos_b200 import _lib, engine
    rng = np.random.default_rng(seed)
    checked = 0
    for B in (2, 3, 10, 20, 39):
        for ratio in (0.0, 1.0, 977.0, 2.0 ** 12, 2.0 ** 17, 2.0 ** 18 - 2.0 * (B - 1) - 1.0, -(2.0 ** 18 - 2.0 * (B - 1) - 1.0)):
            w_target = float(rng.uniform(0.01, 50.0))
            mn = float(np.float32(ratio * w_target))                   # |lo| / w ~ ratio
            mx = float(np.float32(mn + B * w_target))
            w = (mx - mn) / B
            if not w > 0:
                continue
            cuts = [mn + j * w for j in range(1, B)]                   # the host's cutoffs (transformers.py:229-231)
            theta = engine.native_thresholds(cuts, _lib.ANV_F32).astype(np.uint32).view(np.float32)
            ulp = float(np.spacing(np.float32(max(abs(mn), abs(mx)))))
            if not (np.all(np.diff(theta) > 0) and w >= 8 * ulp):      # BinModel's own condition for mode 1
                continue
            inv_w = 1.0 / w
            if not (2.0 * (B - 1) + abs(mn) * inv_w <= 262144.0):      # fold_ok
                continue
            bm1 = _f32(B - 1)
            negc = _f32(-(_f32(inv_w) / bm1))
            lo = _f32(mn)
            k = _f32(1.0 - float(lo) * float(negc))
            xs = [theta, np.nextafter(theta, _f32(np.inf)), np.nextafter(theta, _f32(-np.inf)),
                  np.array([mn, mx, np.nextafter(_f32(mn), _f32(np.inf)), np.nextafter(_f32(mx), _f32(-np.inf)),
                            mn - 3 * w, mx + 3 * w, np.inf, -np.inf, np.nan], np.float32),
                  rng.uniform(mn, mx, 2000).astype(np.float32)]
            for x in np.concatenate(xs):
                v = _fma_f32(x, negc, k)
                v = _f32(0.0) if not v > 0 else min(v, _f32(1.0))      # .sat: NaN -> 0
                t = _fma_f32(v, bm1, _f32(12582912.0))
                r = (B - 1) - (int(np.float32(t).view(np.uint32)) - 0x4B400000)
                assert 0 <= r <= B - 1
                b = B - 1 if np.isnan(x) else int(np.sum(theta < x))   # bucket_label - 1; NaN: last bin
                assert b in (r - 1, r), (B, ratio, float(x), r, b)
                # what the kernel then does: one exact compare against S[r] (S[0] = NaN, S[r] = theta[r-1])
                s_r = np.float32(np.nan) if r == 0 else theta[r - 1]
                assert r + (0 if x <= s_r else 1) == b + 1
                checked += 1
    assert checked > 20000


def test_with_columns_replaces_in_place_appends_in_order_and_drop_moves_to_the_end():
    from anovos_b200.frame import Column, ColumnFrame
    fr = ColumnFrame.from_pandas(pd.DataFrame({"a": [1, 2], "b": [3, 4], "c": [5, 6]}))

    def col(name):
        return Column(name, "int", 2, host=np.array([7, 8], np.int32))
    made = {"z": col("z"), "b": col("b"), "y": col("y")}
    out = fr.with_columns(made)
    assert out.columns == ["a", "b", "c", "z", "y"] and out.n_rows == 2
    assert out.column("b") is made["b"] and out.column("a") is fr.column("a")
    assert fr.columns == ["a", "b", "c"] and fr.column("b") is not made["b"]          # the input frame is unchanged
    assert fr.with_columns(made, drop=["b", "a"]).columns == ["c", "z", "b", "y"]
