"""feature_transformation and boxcox_transformation without a GPU:
  - the oracle's fdlibm restatement (tests/transform_oracle.py) against mpmath: no result more than 1 ulp from the
    correctly rounded value, fdlibm's documented bound;
  - round(x, N) as HALF_UP of the shortest decimal, on constructed ties;
  - the product's host layer (argument handling, types, nulls, naming, column order, partitioned frames) against the
    oracle, with anv_transform_columns replaced by the oracle's image of one kernel column and the other kernels by
    tests/cpu_engine.py."""
import contextlib
import math
import struct
import warnings

import mpmath
import numpy as np
import pyarrow as pa
import pytest

import cpu_engine
import transform_oracle as TO
from anovos_b200 import engine

mpmath.mp.prec = 200


# ---- fdlibm against mpmath -------------------------------------------------------------------------------------------

def _ord(x):
    i = struct.unpack("<q", struct.pack("<d", x))[0]
    return i if i >= 0 else -(i & 0x7fffffffffffffff)


def _ulps(got, exact):
    """Distance in ulps between got and the correctly rounded exact value (an mpf)."""
    if mpmath.isnan(exact):
        return 0 if math.isnan(got) else 1 << 62
    ref = float(exact) if abs(exact) < mpmath.mpf(2) ** 1024 else math.copysign(math.inf, float(mpmath.sign(exact)))
    if math.isinf(ref) or math.isinf(got):
        return 0 if ref == got else 1 << 62
    return abs(_ord(got) - _ord(ref))


def _sweep(rng, lo_exp, hi_exp, n):
    return [float(s * 2.0 ** e) for s, e in zip(rng.uniform(1, 2, n), rng.integers(lo_exp, hi_exp, n))]


SUBNORMALS = [5e-324, 1e-320, 2.2250738585072e-308, 2.2250738585072014e-308, 4.9e-310]


def _check(fn, exact, xs):
    worst, one = 0, 0
    for x in xs:
        u = _ulps(fn(*x), exact(*x))
        worst = max(worst, u)
        one += u == 1
        assert u <= 1, (x, fn(*x), exact(*x))
    return worst, one


def test_log_and_log10_within_one_ulp():
    rng = np.random.default_rng(1)
    xs = _sweep(rng, -1074, 1024, 3000) + SUBNORMALS + [1.0, 2.0, 10.0, 1e22, 1.7976931348623157e308]
    xs += [1.0 + k * 2.0 ** -52 for k in range(-40, 40)] + list(rng.uniform(0.7, 1.5, 2000))
    for fn, ex in ((TO.fd_log, mpmath.log), (TO.fd_log10, mpmath.log10)):
        worst, one = _check(fn, ex, [(x,) for x in xs])
        print(fn.__name__, "1-ulp results:", one, "of", len(xs))
    assert TO.fd_log(0.0) == -math.inf and TO.fd_log(-0.0) == -math.inf and math.isnan(TO.fd_log(-1.0))
    assert TO.fd_log(math.inf) == math.inf and math.isnan(TO.fd_log(math.nan))
    assert [TO.fd_log10(10.0 ** k) for k in range(23)] == [float(k) for k in range(23)]


def test_exp_within_one_ulp_and_its_edges():
    rng = np.random.default_rng(2)
    xs = list(rng.uniform(-745.2, 709.8, 3000)) + list(rng.uniform(-1, 1, 1000)) + [
        7.09782712893383973096e+02, -7.45133219101941108420e+02, 709.78, -745.13, -708.4, -708.5, -720.0, 1e-300, -1e-300,
        2.0 ** -28, 0.5 * math.log(2), 1.5 * math.log(2), 0.0, -0.0]
    worst, one = _check(TO.fd_exp, mpmath.exp, [(x,) for x in xs])
    print("exp 1-ulp results:", one, "of", len(xs))
    assert TO.fd_exp(710.0) == math.inf and TO.fd_exp(-746.0) == 0.0 and TO.fd_exp(-math.inf) == 0.0
    assert math.isnan(TO.fd_exp(math.nan))


def _mp_pow(x, y):
    if math.isnan(x) or math.isnan(y):
        return mpmath.mpf("nan") if not (y == 0) else mpmath.mpf(1)
    if x < 0 and y != int(y):
        return mpmath.mpf("nan")
    if x == 0:
        return mpmath.mpf(0) if y > 0 else mpmath.mpf("inf") * (-1 if (y == int(y) and int(y) % 2 and math.copysign(1, x) < 0) else 1)
    r = mpmath.power(mpmath.mpf(abs(x)), mpmath.mpf(y))
    return -r if x < 0 and int(y) % 2 else r


def test_pow_within_one_ulp():
    rng = np.random.default_rng(3)
    pairs = [(x, y) for x, y in zip(_sweep(rng, -60, 60, 2000), rng.uniform(-20, 20, 2000))]
    pairs += [(x, y) for x, y in zip(rng.uniform(0, 3, 1000), rng.uniform(-600, 600, 1000))]
    pairs += [(x, float(k)) for x, k in zip(-np.abs(rng.normal(0, 10, 500)), rng.integers(-30, 30, 500))]   # negative bases
    pairs += [(x, s) for x in _sweep(rng, -1074, 1024, 400) for s in (0.5, -0.5)]
    pairs += [(2.0, y) for y in (-1074.0, -1074.5, -1075.0, -1022.5, 1023.0, 1023.999, 1024.0, -1060.3)]
    pairs += [(10.0, float(k)) for k in range(-330, 310, 7)] + [(x, 2.0) for x in SUBNORMALS]
    pairs += [(1.5, 2.0 ** 31 + 0.5), (1.0 - 2 ** -40, 2.0 ** 40), (1.0 + 2 ** -30, 2.0 ** 35)]
    worst, one = _check(TO.fd_pow, _mp_pow, pairs)
    print("pow 1-ulp results:", one, "of", len(pairs))
    assert TO.fd_pow(-8.0, 1.0 / 3) != TO.fd_pow(-8.0, 1.0 / 3)          # (x<0)**non-int is NaN
    assert TO.fd_pow(-2.0, 3.0) == -8.0 and TO.fd_pow(0.0, -1.0) == math.inf and TO.fd_pow(-0.0, -1.0) == -math.inf
    assert math.isnan(TO.fd_pow(1.0, math.inf)) and TO.fd_pow(math.nan, 0.0) == 1.0 and TO.fd_pow(-0.0, 0.5) == 0.0


def test_pow_near_one_with_huge_exponent_keeps_fdlibm_error():
    """For |y| > 2^31 and |1 - x| <= 2^-20, fdlibm takes log2(x) from a short series on t = x - 1 and assumes t has 20
    trailing zero bits; when it does not, the product loses bits.  StrictMath keeps that answer, and so do we: it is
    within 2^-40 relative, not within 1 ulp."""
    for x, y in ((0.9999999, 3e9), (1.0000001, 1e9)):
        got, exact = TO.fd_pow(x, y), _mp_pow(x, y)
        assert abs(mpmath.mpf(got) / exact - 1) < mpmath.mpf(2) ** -40


# ---- round(x, N) -----------------------------------------------------------------------------------------------------

ROUND_TIES = [(1.005, 2, 1.01), (2.675, 2, 2.68), (0.125, 2, 0.13), (-2.5, 0, -3.0), (-0.5, 0, -1.0), (1.0005, 3, 1.001),
              (0.285, 2, 0.29), (1.45, 1, 1.5), (8.345, 2, 8.35), (1234.5, -1, 1230.0), (1235.0, -1, 1240.0),
              (-0.004, 2, 0.0), (1e300, 2, 1e300), (4503599627370495.5, 0, 4503599627370496.0), (0.049999999999999996, 1, 0.0)]


@pytest.mark.parametrize("x,n,want", ROUND_TIES)
def test_round_half_up_of_the_shortest_decimal(x, n, want):
    got = TO.round_half_up(x, n)
    assert got == want and math.copysign(1, got) == math.copysign(1, want)


def test_round_integers_wrap_like_bigdecimal():
    assert TO.round_integer(15, -1, 32) == 20 and TO.round_integer(-15, -1, 32) == -20 and TO.round_integer(14, -1, 32) == 10
    assert TO.round_integer(2147483647, -1, 32) == TO._wrap(2147483650, 32)
    assert TO.round_integer(6 * 10 ** 18, -19, 64) == TO._wrap(10 ** 19, 64) and TO.round_integer(7, 3, 64) == 7


# ---- the host layer on a NumPy stand-in of the kernel ----------------------------------------------------------------

def transform_columns(fr, names, specs):
    import torch
    outs, valid, nulls = [], [], []
    for n, sp in zip(names, specs):
        vals, ok = cpu_engine._values(fr, n)
        out, keep = TO.transform_reference(vals, ok, fr.column(n).anv_dtype, sp)
        outs.append(torch.from_numpy(out))
        nulls.append(int((~keep).sum()))
        if sp[0] in TO.MAKES_NULLS:
            bits = np.packbits(keep, bitorder="little")
            n_words = (fr.n_rows + 31) // 32
            valid.append(torch.from_numpy(np.concatenate([bits, np.zeros(n_words * 4 - len(bits), np.uint8)]).view(np.int32)))
        else:
            valid.append(None)
    return outs, valid, np.array(nulls, np.int64)


@contextlib.contextmanager
def stand_ins():
    saved = engine.transform_columns
    try:
        engine.transform_columns = transform_columns
        with cpu_engine.installed():
            yield
    finally:
        engine.transform_columns = saved


def product(name, table, **kw):
    import anovos.data_transformer.transformers as T
    with stand_ins():
        odf = getattr(T, name)(table, **kw)
        if getattr(odf, "is_partitioned", False):
            return pa.concat_tables([ch.to_arrow() for ch in odf.chunks()])
        return odf.to_arrow() if hasattr(odf, "to_arrow") else odf


COLS3 = ["age", "fnlwgt", "hours-per-week"]


def _row(t, ifa, col):
    i = t.column("ifa").to_pylist().index(ifa)
    return t.column(col)[i].as_py()


def test_reference_unit_tests(income):
    """test_transformers.py:603-633."""
    for name, kw in (("feature_transformation", {}), ("boxcox_transformation", {"boxcox_lambda": 0.5})):
        odf = product(name, income, list_of_cols=COLS3, **kw)
        assert odf.num_columns == 21        # the reference's fixture has 17 columns, this table 21: all are replaced
        assert odf.column_names == income.column_names
        for c, want in zip(COLS3, (7.14142842854285, 399.6936326738268, 4.47213595499958)):
            assert _row(odf, "27520a", c) == pytest.approx(want)
        assert product(name, income, list_of_cols=COLS3, output_mode="append", **kw).num_columns == 24


def test_capital_loss_ln_pins_the_null_rule(income_spark):
    """The notebook's capital-loss_ln count is 1 519: log of x <= 0 is null."""
    odf = product("feature_transformation", income_spark, list_of_cols=["capital-loss"], method_type="ln", output_mode="append")
    assert odf.column("capital-loss_ln").null_count == odf.num_rows - 1519
    assert odf.schema.field("capital-loss_ln").type == pa.float64()


def _table(n=257, seed=7):
    rng = np.random.default_rng(seed)
    mask = rng.random(n) < 0.2
    return pa.table({
        "f32": pa.array(rng.normal(3, 4, n).astype(np.float32), mask=mask),
        "f64": pa.array(rng.normal(0, 30, n), mask=np.roll(mask, 1)),
        "i32": pa.array(rng.integers(-30, 40, n).astype(np.int32), mask=np.roll(mask, 2)),
        "i64": pa.array(rng.integers(-10 ** 6, 10 ** 6, n).astype(np.int64)),
        "s": pa.array(["a"] * n)})


NUM = ["f32", "f64", "i32", "i64"]


def _expect(t, method, N, c):
    from anovos_b200.data_transformer.transformers import transform_spec
    from anovos_b200.frame import as_frame
    sp = transform_spec(method, N, as_frame(t).column(c).anv_dtype)
    col = t.column(c)
    vals = np.asarray(col.fill_null(0).to_numpy(zero_copy_only=False))
    ok = ~np.asarray(col.is_null().to_numpy(zero_copy_only=False))
    if sp[0] is None:
        return np.zeros(len(vals), TO.NP_OF[sp[1]]), np.zeros(len(vals), bool)
    return TO.transform_reference(vals, ok, as_frame(t).column(c).anv_dtype, sp)


@pytest.mark.parametrize("method,N", [(m, None) for m in TO.METHODS if m not in ("powOfN", "toPowerN", "remainderDivByN", "roundN")]
                         + [("powOfN", 3), ("toPowerN", 0.5), ("remainderDivByN", 7), ("remainderDivByN", 2.5),
                            ("remainderDivByN", 0), ("roundN", 1), ("roundN", -1)])
def test_host_layer_types_nulls_and_names(method, N):
    t = _table()
    odf = product("feature_transformation", t, list_of_cols="all", method_type=method, N=N, output_mode="append")
    suffix = "_" + (method[:-1] + str(N) if N is not None else method)
    assert odf.column_names == t.column_names + [c + suffix for c in NUM]
    for c in NUM:
        exp, keep = _expect(t, method, N, c)
        got = odf.column(c + suffix)
        assert got.type == pa.from_numpy_dtype(exp.dtype), (c, got.type, exp.dtype)
        g = np.asarray(got.fill_null(0).to_numpy(zero_copy_only=False))
        assert np.array_equal(np.asarray(got.is_valid().to_numpy(zero_copy_only=False)), keep), c
        assert np.array_equal(g.view(np.uint8), exp.view(np.uint8)), (c, g[:5], exp[:5])


def test_remainder_and_round_types_follow_spark():
    t = _table()
    types = lambda odf: [odf.schema.field(c).type for c in NUM]         # noqa: E731
    odf = product("feature_transformation", t, method_type="remainderDivByN", N=10)
    assert types(odf) == [pa.float32(), pa.float64(), pa.int32(), pa.int64()]
    odf = product("feature_transformation", t, method_type="remainderDivByN", N=10.0)
    assert types(odf) == [pa.float64()] * 4
    odf = product("feature_transformation", t, method_type="remainderDivByN", N=1 << 40)
    assert types(odf) == [pa.float32(), pa.float64(), pa.int64(), pa.int64()]
    odf = product("feature_transformation", t, method_type="roundN", N=2)
    assert types(odf) == [pa.float32(), pa.float64(), pa.int32(), pa.int64()]
    for m in ("floor", "ceil", "factorial"):
        assert types(product("feature_transformation", t, method_type=m)) == [pa.int64()] * 4


def test_argument_errors():
    t = _table()
    with pytest.raises(TypeError, match="Invalid input for Column"):
        product("feature_transformation", t, list_of_cols=["s"])
    with pytest.raises(TypeError, match="Invalid input for Column"):
        product("feature_transformation", t, list_of_cols="f32", drop_cols="f32")
    with pytest.raises(TypeError, match="Invalid input method_type"):
        product("feature_transformation", t, method_type="log3")
    with pytest.raises(TypeError):
        product("feature_transformation", t, method_type="roundN")
    for m in ("powOfN", "toPowerN", "remainderDivByN"):         # F.pow(None, x), x ** None, x % None: all null
        odf = product("feature_transformation", t, list_of_cols=["f32", "i32"], method_type=m, output_mode="append")
        suffix = "_" + m[:-1] + "None"
        assert [odf.column(c + suffix).null_count for c in ("f32", "i32")] == [t.num_rows] * 2
        assert odf.schema.field("i32" + suffix).type == (pa.int32() if m == "remainderDivByN" else pa.float64())
    with pytest.raises(ValueError, match="N <= 22"):
        product("feature_transformation", t, method_type="roundN", N=23)
    with pytest.raises(ValueError, match="Data must be positive"):
        product("boxcox_transformation", t, list_of_cols=["f64"], boxcox_lambda=2)
    pos = pa.table({"a": pa.array([1.0, 2.0, 4.0]), "b": pa.array([3, 4, 5], pa.int32())})
    for bad in ([1], [1, "x"], "x"):
        with pytest.raises(TypeError, match="Invalid input for boxcox_lambda"):
            product("boxcox_transformation", pos, boxcox_lambda=bad)


def test_boxcox_lambdas_names_and_untouched_columns():
    pos = pa.table({"a": pa.array([1.0, 2.0, 4.0, None]), "b": pa.array([3, 4, 5, 6], pa.int32()), "c": pa.array([0.5, 1.5, 9.0, 2.0])})
    odf = product("boxcox_transformation", pos, boxcox_lambda=[0, 1, -0.5], output_mode="append")
    assert odf.column_names == ["a", "b", "c", "a_bxcx_0", "c_bxcx_-0.5"]
    assert odf.column("a_bxcx_0").to_pylist() == [TO.fd_log(1.0), TO.fd_log(2.0), TO.fd_log(4.0), None]
    assert odf.column("c_bxcx_-0.5").to_pylist() == [TO.fd_pow(v, -0.5) for v in (0.5, 1.5, 9.0, 2.0)]
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        assert product("boxcox_transformation", pos, boxcox_lambda=1) is pos
    assert "lambdaVal for all columns are 1" in str(w[-1].message)


def test_partitioned_frames_transform_per_chunk(income_spark):
    from anovos_b200.partitioned import PartitionedFrame
    whole = product("feature_transformation", income_spark, list_of_cols=COLS3, method_type="log10")
    with stand_ins():
        import anovos.data_transformer.transformers as T
        n = income_spark.num_rows
        pf = PartitionedFrame.from_arrow_partitions(income_spark, [5000] * (n // 5000) + [n % 5000])
        odf = T.feature_transformation(pf, list_of_cols=COLS3, method_type="log10")
        got = pa.concat_tables([ch.to_arrow() for ch in odf.chunks()])
    for c in COLS3:
        assert got.column(c).to_pylist() == whole.column(c).to_pylist()


def test_print_impact(income, capsys):
    product("boxcox_transformation", income, list_of_cols=COLS3, boxcox_lambda=0.5, print_impact=True)
    out = capsys.readouterr().out
    assert "Best BoxCox Parameter(s):  [0.5, 0.5, 0.5]" in out and out.count("skewness") == 2
