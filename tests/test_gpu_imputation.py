"""imputation_MMM on the GPU: anv_impute_fill / anv_valid_not_nan bit for bit against exact NumPy references on
adversarial columns, and the public function against the oracle (tests/imputation_oracle.py)."""
import numpy as np
import pyarrow as pa
import pytest

import imputation_oracle as IO
from test_imputation_cpu import _nb, _same_tables, _synthetic, _table, _tiny

pytestmark = pytest.mark.gpu

I64_MAX, I64_MIN = (1 << 63) - 1, -(1 << 63)


def _words(valid):
    valid = np.asarray(valid, bool)
    bits = np.packbits(valid, bitorder="little")
    pad = (-len(bits)) % 4
    return np.concatenate([bits, np.zeros(pad, np.uint8)]).view(np.int32)


def _frame(cols):
    """name -> (values ndarray, bool valid | None) -> device-resident ColumnFrame."""
    import torch
    from anovos_b200.frame import ColumnFrame
    data = {}
    for n, (v, ok) in cols.items():
        dv = torch.from_numpy(np.ascontiguousarray(v)).cuda()
        data[n] = (dv, None if ok is None else torch.from_numpy(_words(ok)).cuda())
    return ColumnFrame.from_tensors(data)


_NP = {0: np.float32, 1: np.float64, 2: np.int32, 3: np.int64}


def _run_and_check(cols, specs):
    """specs: name -> (out anv dtype, flags, fill value)."""
    from anovos_b200 import _lib, engine
    fr = _frame(cols)
    names = list(specs)
    outs = engine.impute_fill(fr, names, [specs[n][0] for n in names], [specs[n][1] for n in names],
                              [engine.fill_bits(specs[n][2], specs[n][0]) for n in names])
    for n, t in zip(names, outs):
        v, ok = cols[n]
        od, fl, fv = specs[n]
        exp = IO.fill_reference(v, np.ones(len(v), bool) if ok is None else ok, _NP[od], bool(fl & _lib.IMPUTE_NAN_MISSING),
                                bool(fl & _lib.IMPUTE_ROUND_DOUBLE), np.array([fv], _NP[od])[0])
        got = t.cpu().numpy()
        assert got.dtype == exp.dtype and got.shape == exp.shape, n
        assert np.array_equal(got.view(np.uint8), exp.view(np.uint8)), (n, got[:8], exp[:8])


@pytest.mark.parametrize("n", [1, 31, 33, 130, 1027, 70_001])
def test_fill_kernel_bit_exact(n):
    from anovos_b200 import _lib
    rng = np.random.default_rng(n)
    nan_pos = np.array([0x7fc00000, 0xffc00001, 0x7f800001, 0xff812345], np.uint32).view(np.float32)
    f32 = rng.normal(0, 1, n).astype(np.float32)
    idx = rng.random(n) < 0.2
    f32[idx] = nan_pos[rng.integers(0, 4, int(idx.sum()))]
    f32[:min(n, 3)] = np.array([-0.0, np.inf, -np.inf], np.float32)[:min(n, 3)]
    f64 = rng.normal(0, 1, n)
    idx = rng.random(n) < 0.2
    f64[idx] = np.array([0x7ff8000000000001, 0xfff8000000000000], np.uint64).view(np.float64)[rng.integers(0, 2, int(idx.sum()))]
    f64[:min(n, 3)] = np.array([-0.0, np.inf, -np.inf])[:min(n, 3)]
    i64 = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64)
    special = np.array([(1 << 53) - 1, 1 << 53, (1 << 53) + 1, I64_MAX, -I64_MAX, I64_MIN], np.int64)
    i64[:min(n, 6)] = special[:min(n, 6)]
    i32 = rng.integers(-(1 << 31), (1 << 31) - 1, n, dtype=np.int64).astype(np.int32)
    i32[:min(n, 2)] = np.array([2 ** 31 - 1, -2 ** 31], np.int32)[:min(n, 2)]
    some = rng.random(n) > 0.3
    lead_null = np.ones(n, bool)
    lead_null[:min(n, 66_000)] = False                        # the first tiles are all null
    cols = {"f32": (f32, some), "f32_free": (f32, None), "f64": (f64, some), "i64": (i64, some), "i64_all_null": (i64, np.zeros(n, bool)),
            "i32": (i32, lead_null), "i32_full": (i32, np.ones(n, bool)), "codes": (rng.integers(0, 5, n).astype(np.int32), some)}
    A = _lib
    specs = {"f32": (A.ANV_F32, A.IMPUTE_NAN_MISSING, 1.5), "f32_free": (A.ANV_F32, 0, -2.0),
             "f64": (A.ANV_F64, A.IMPUTE_NAN_MISSING, -0.0), "i64": (A.ANV_I64, A.IMPUTE_ROUND_DOUBLE, -5),
             "i64_all_null": (A.ANV_F64, 0, 3.25), "i32": (A.ANV_I32, A.IMPUTE_ROUND_DOUBLE, 2 ** 31 - 1),
             "i32_full": (A.ANV_F64, 0, 0.0), "codes": (A.ANV_I32, 0, 5)}
    _run_and_check(cols, specs)
    # the same bigint column without the round trip (mode: to double) and kept as is
    _run_and_check({"i64": (i64, some)}, {"i64": (A.ANV_F64, 0, 7.0)})
    _run_and_check({"i64": (i64, some)}, {"i64": (A.ANV_I64, 0, I64_MIN)})


@pytest.mark.parametrize("n", [1, 31, 33, 4099, 70_001])
def test_valid_not_nan_exact(n):
    from anovos_b200 import engine
    rng = np.random.default_rng(7 + n)
    f32 = rng.normal(0, 1, n).astype(np.float32)
    f32[rng.random(n) < 0.3] = np.float32(np.nan)
    f64 = rng.normal(0, 1, n)
    f64[rng.random(n) < 0.1] = -np.nan
    ok = rng.random(n) > 0.25
    cols = {"a": (f32, ok), "b": (f64, None), "c": (f64, ok), "d": (rng.integers(0, 3, n).astype(np.int32), ok)}
    fr = _frame(cols)
    words, n_nan = engine.valid_not_nan(fr, list(cols))
    w = words.cpu().numpy()
    for i, (name, (v, vk)) in enumerate(cols.items()):
        vk = np.ones(n, bool) if vk is None else vk
        isn = np.isnan(v) if v.dtype.kind == "f" else np.zeros(n, bool)
        exp = _words(vk & ~isn)[:(n + 31) // 32]
        assert np.array_equal(w[i], exp), name
        assert n_nan[i] == int((vk & isn).sum()), name


def test_fill_beyond_65535_columns_runs_in_blocks():
    from anovos_b200 import _lib, engine
    n = 37
    v = np.arange(n, dtype=np.float64)
    v[::3] = np.nan
    ok = np.arange(n) % 5 != 0
    fr = _frame({"x": (v, ok)})
    k = _lib.MAX_LAUNCH_COLS + 3
    fills = list(range(k))
    outs = engine.impute_fill(fr, ["x"] * k, [_lib.ANV_F64] * k, [_lib.IMPUTE_NAN_MISSING] * k,
                              [engine.fill_bits(float(f), _lib.ANV_F64) for f in fills])
    assert len(outs) == k
    for j in (0, _lib.MAX_LAUNCH_COLS - 1, _lib.MAX_LAUNCH_COLS, k - 1):
        exp = IO.fill_reference(v, ok, np.float64, True, False, float(fills[j]))
        assert np.array_equal(outs[j].cpu().numpy(), exp)
    words, n_nan = engine.valid_not_nan(fr, ["x"] * k)
    assert words.shape[0] == k and (n_nan == n_nan[0]).all()


# ---- the public function against the oracle ------------------------------------------------------------------------

def _gpu(table_or_frame, **kw):
    import anovos.data_transformer.transformers as T
    return T.imputation_MMM(None, table_or_frame, **kw)


def test_notebook_calls_on_spark_partitioned_income(income_spark, capsys):
    from anovos_b200.result import ResultFrame
    calls = [dict(print_impact=True), dict(list_of_cols="all", method_type="mean", output_mode="append"),
             dict(list_of_cols=["marital-status", "sex", "occupation", "age"], print_impact=True),
             dict(list_of_cols="all", method_type="median"), dict(list_of_cols="all", method_type="mode")]
    for kw in calls:
        odf = _gpu(income_spark, **kw)
        printed = capsys.readouterr().out
        exp, imp = IO.imputation_MMM(income_spark, **{k: v for k, v in kw.items() if k != "print_impact"})
        got = odf.materialize().to_arrow() if getattr(odf, "is_partitioned", False) else odf.to_arrow()
        _same_tables(got, exp, rel=1e-12 if kw.get("method_type") == "mean" else 0.0)
        if kw.get("print_impact"):
            ResultFrame(imp).show(100)
            assert printed == capsys.readouterr().out
    nb = _nb()
    _gpu(income_spark, print_impact=True)
    rows = [line.split() for line in capsys.readouterr().out.strip().splitlines()[1:]]
    assert rows == _table(nb, "transformers", 44)["rows"]


def _synthetic_frames():
    rng = np.random.default_rng(11)
    out = []
    for rate in (0.0, 0.01, 0.5, 1.0):
        n = 50_007
        f32 = rng.normal(5, 3, n).astype(np.float32)
        f32[rng.random(n) < 0.02] = np.nan
        f64 = rng.exponential(2, n)
        if rate < 1.0:
            f64[rng.random(n) < 0.05] = np.nan
        t = pa.table({"f32": pa.array(f32, mask=rng.random(n) < max(rate, 0.001) if rate < 1 else None),
                      "f64": pa.array(f64, mask=rng.random(n) < rate),
                      "i32": pa.array(rng.integers(-9, 99, n).astype(np.int32), mask=rng.random(n) < rate),
                      "i64": pa.array(rng.integers(-(1 << 60), 1 << 60, n), mask=rng.random(n) < min(rate, 0.9)),
                      "cat": pa.array(rng.choice(["x", "yy", "zzz", "w"], n), mask=rng.random(n) < rate)})
        out.append((rate, t))
    return out


@pytest.mark.parametrize("method_type", ["mean", "median", "mode"])
def test_synthetic_frames_equal_oracle(method_type):
    from anovos_b200.frame import ColumnFrame
    for rate, t in _synthetic_frames():
        for mode in ("replace", "append"):
            kw = dict(list_of_cols="all", method_type=method_type, output_mode=mode)
            try:
                exp, _ = IO.imputation_MMM(t, **kw)
            except ValueError:
                with pytest.raises(ValueError, match="surrogate cannot be computed"):
                    _gpu(ColumnFrame.from_arrow(t), **kw)
                continue
            _same_tables(_gpu(ColumnFrame.from_arrow(t), **kw).to_arrow(), exp, rel=1e-12 if method_type == "mean" else 0.0)
    t = _synthetic()
    for mt in ("mean", "median", "mode"):
        _same_tables(_gpu(ColumnFrame.from_arrow(t), list_of_cols="all", method_type=mt).to_arrow(),
                     IO.imputation_MMM(t, list_of_cols="all", method_type=mt)[0], rel=1e-12 if mt == "mean" else 0.0)
    _same_tables(_gpu(ColumnFrame.from_arrow(_tiny())).to_arrow(), IO.imputation_MMM(_tiny())[0])


def test_chunked_frame_equals_resident():
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.partitioned import PartitionedFrame
    t = _synthetic(n=100_003)
    for mt in ("median", "mean", "mode"):
        res = _gpu(ColumnFrame.from_arrow(t), method_type=mt, output_mode="append").to_arrow()
        odf = _gpu(PartitionedFrame.from_frame(ColumnFrame.from_arrow(t), 8192 * 4), method_type=mt, output_mode="append")
        got = odf.materialize().to_arrow()
        for c in res.column_names:
            if c.endswith("_imputed") and mt != "median":       # the median of a chunked frame is exact, not one sketch
                _same_tables(got.select([c]), res.select([c]), rel=1e-12 if mt == "mean" else 0.0)
        assert got.column_names == res.column_names


def test_null_columns_detection_mmm_reproduces_notebook(income_spark, capsys):
    import anovos.data_analyzer.quality_checker as qc
    nb = _nb()
    for cell, cfg in [(22, {"method_type": "median"}), (23, {"method_type": "mean"}),
                      (25, {"method_type": "mean", "output_mode": "append"})]:
        odf, _ = qc.nullColumns_detection(None, income_spark, list_of_cols="all", treatment=True, treatment_method="MMM",
                                          treatment_configs=cfg, print_impact=True)
        rows = [line.split() for line in capsys.readouterr().out.strip().splitlines()[1:]]
        assert rows == _table(nb, "quality_checker", cell)["rows"], cell
        exp, _ = IO.nullColumns_detection_MMM(income_spark, "all", treatment_configs=cfg)
        got = odf.materialize().to_arrow() if getattr(odf, "is_partitioned", False) else odf.to_arrow()
        _same_tables(got, exp, rel=1e-12)
