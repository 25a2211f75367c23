"""The scalers on the GPU: anv_scale_columns bit for bit against its exact NumPy image (scaling_oracle.scale_reference)
on adversarial columns, and z_standardization / IQR_standardization / normalization against the oracle and the
notebook's stored Spark outputs."""
import contextlib

import numpy as np
import pyarrow as pa
import pytest

import scaling_oracle as SO
from test_scaling_cpu import check_notebook, same_tables, synthetic

pytestmark = pytest.mark.gpu

I64_MAX, I64_MIN = (1 << 63) - 1, -(1 << 63)


def _words(valid):
    bits = np.packbits(np.asarray(valid, bool), bitorder="little")
    return np.concatenate([bits, np.zeros((-len(bits)) % 4, np.uint8)]).view(np.int32)


def _frame(cols):
    """name -> (values ndarray, bool valid | None) -> device-resident ColumnFrame."""
    import torch
    from anovos_b200.frame import ColumnFrame
    return ColumnFrame.from_tensors({n: (torch.from_numpy(np.ascontiguousarray(v)).cuda(),
                                         None if ok is None else torch.from_numpy(_words(ok)).cuda())
                                     for n, (v, ok) in cols.items()})


def _check(cols, names, specs):
    from anovos_b200 import engine
    fr = _frame(cols)
    outs, valid, nulls = engine.scale_columns(fr, names, specs)
    n_rows = fr.n_rows
    for i, (n, sp) in enumerate(zip(names, specs)):
        v, ok = cols[n]
        exp, keep = SO.scale_reference(v, np.ones(len(v), bool) if ok is None else ok, sp)
        got = outs[i].cpu().numpy()
        assert got.dtype == exp.dtype and np.array_equal(got.view(np.uint8), exp.view(np.uint8)), (n, sp, got[:8], exp[:8])
        assert nulls[i] == int((~keep).sum()), (n, sp)
        if sp[2] & SO.NAN_TO_NULL:
            assert np.array_equal(valid[i].cpu().numpy(), _words(keep)[:(n_rows + 31) // 32]), (n, sp)
        else:
            assert valid[i] is None


def _columns(n):
    rng = np.random.default_rng(n)
    nan_pos = np.array([0x7fc00000, 0xffc00001, 0x7f800001, 0xff812345], np.uint32).view(np.float32)
    f32 = rng.normal(0, 1e3, n).astype(np.float32)
    idx = rng.random(n) < 0.15
    f32[idx] = nan_pos[rng.integers(0, 4, int(idx.sum()))]
    f32[:min(n, 4)] = np.array([-0.0, np.inf, -np.inf, 0.0], np.float32)[:min(n, 4)]
    f64 = rng.normal(0, 1, n) * 10.0 ** rng.integers(-300, 300, n)
    idx = rng.random(n) < 0.15
    f64[idx] = np.array([0x7ff8000000000001, 0xfff8000000000000], np.uint64).view(np.float64)[rng.integers(0, 2, int(idx.sum()))]
    f64[:min(n, 4)] = np.array([-0.0, np.inf, -np.inf, 5e-324])[:min(n, 4)]
    i64 = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64)
    special = np.array([(1 << 53) - 1, 1 << 53, (1 << 53) + 1, -(1 << 53) - 1, I64_MAX, I64_MIN], np.int64)
    i64[:min(n, 6)] = special[:min(n, 6)]
    i32 = rng.integers(-(1 << 31), (1 << 31) - 1, n, dtype=np.int64).astype(np.int32)
    i32[:min(n, 2)] = np.array([2 ** 31 - 1, -2 ** 31], np.int32)[:min(n, 2)]
    some = rng.random(n) > 0.3
    lead_null = np.ones(n, bool)
    lead_null[:min(n, 66_000)] = False                          # the first row tiles are all null
    return {"f32": (f32, some), "f32_free": (f32, None), "f64": (f64, some), "f64_free": (f64, None),
            "i32": (i32, lead_null), "i32_free": (i32, None), "i64": (i64, some), "i64_free": (i64, None)}


@pytest.mark.parametrize("n", [1, 31, 33, 130, 1027, 70_001])
def test_scale_kernel_bit_exact(n):
    cols = _columns(n)
    params = [(SO.DIV, 3.25, 0.1), (SO.DIV, -7.0, -0.0), (SO.DIV, 1e300, 1e-300), (SO.AFFINE, -1.5, 1 / 3),
              (SO.AFFINE, np.inf, 2.0), (SO.AFFINE, 0.0, 1e308), (SO.CONST, 0.0, 0.0)]
    names, specs = [], []
    for name in cols:
        for k, (mode, a, b) in enumerate(params):
            for od in (SO.F32, SO.F64):
                for fl in (0, SO.NAN_TO_NULL):
                    names.append(name)
                    specs.append((mode, od, fl, a, b, 0.25 * k - 0.5))
    _check(cols, names, specs)


def test_scale_beyond_65535_columns_runs_in_blocks():
    from anovos_b200 import _lib, engine
    n = 37
    v = np.arange(n, dtype=np.float64)
    v[::3] = np.nan
    ok = np.arange(n) % 5 != 0
    fr = _frame({"x": (v, ok)})
    k = _lib.MAX_LAUNCH_COLS + 3
    specs = [(SO.AFFINE, SO.F32 if j % 2 else SO.F64, SO.NAN_TO_NULL if j % 3 else 0, float(j), 0.5, 1.0) for j in range(k)]
    outs, valid, nulls = engine.scale_columns(fr, ["x"] * k, specs)
    assert len(outs) == len(valid) == len(nulls) == k
    for j in (0, 1, 2, _lib.MAX_LAUNCH_COLS - 1, _lib.MAX_LAUNCH_COLS, k - 1):
        exp, keep = SO.scale_reference(v, ok, specs[j])
        assert np.array_equal(outs[j].cpu().numpy().view(np.uint8), exp.view(np.uint8)), j
        assert nulls[j] == int((~keep).sum())
        assert (valid[j] is None) == (not specs[j][2])


# ---- the public functions against the oracle -----------------------------------------------------------------------

def _gpu(name, table_or_frame, **kw):
    import anovos.data_transformer.transformers as T
    args = () if name == "normalization" else (None,)
    odf = getattr(T, name)(*args, table_or_frame, **kw)
    return odf.materialize().to_arrow() if getattr(odf, "is_partitioned", False) else odf.to_arrow()


NAMES = ["z_standardization", "IQR_standardization", "normalization"]


def test_income_equals_oracle_and_notebook(income_spark, tmp_path):
    check_notebook(_gpu, income_spark)
    for name in NAMES:
        for mode in ("replace", "append"):
            kw = dict(list_of_cols="all", output_mode=mode)
            got, exp = _gpu(name, income_spark, **kw), SO.__dict__[name](income_spark, **kw)[0]
            if name == "z_standardization":            # FP64 moments vs the oracle's pairwise sums: a few ulps
                assert got.column_names == exp.column_names
                for c in exp.column_names:
                    if pa.types.is_floating(exp.schema.field(c).type):
                        assert np.allclose(got.column(c).to_numpy(zero_copy_only=False),
                                           exp.column(c).to_numpy(zero_copy_only=False), rtol=1e-13, atol=1e-12, equal_nan=True)
            else:
                same_tables(got, exp)


@pytest.mark.parametrize("name", NAMES)
def test_synthetic_equals_oracle(name, tmp_path):
    from anovos_b200.frame import ColumnFrame
    t = synthetic(n=50_021)
    for mode in ("replace", "append"):
        kw = dict(list_of_cols="all", output_mode=mode, model_path=str(tmp_path))
        with pytest.warns(UserWarning) if name != "normalization" else contextlib.nullcontext():
            got = _gpu(name, ColumnFrame.from_arrow(t), **kw)
        exp = SO.__dict__[name](t, **dict(kw, model_path="NA"))[0]
        if name == "z_standardization":
            for c in exp.column_names:
                if pa.types.is_floating(exp.schema.field(c).type):
                    assert np.allclose(got.column(c).to_numpy(zero_copy_only=False), exp.column(c).to_numpy(zero_copy_only=False),
                                       rtol=1e-13, atol=1e-12, equal_nan=True), c
        else:
            same_tables(got, exp)
        same_tables(_gpu(name, ColumnFrame.from_arrow(t.slice(7, 9000)), list_of_cols="all", output_mode=mode,
                         pre_existing_model=True, model_path=str(tmp_path)),
                    SO.__dict__[name](t.slice(7, 9000), list_of_cols="all", output_mode=mode, pre_existing_model=True,
                                      model_path=str(tmp_path))[0])


def test_ten_million_rows_synthetic():
    """synth.device_frame at 10 M rows against its host twin: the kernel on the oracle's parameters bit for bit, the
    API end to end within 1e-13 relative (z: its mean and stddev come from the FP64 moments pass, so values next to the
    mean also get 1e-12 absolute)."""
    import torch
    from anovos_b200 import engine, synth
    rows, ncol = 10_000_000, 4
    fr = synth.device_frame(rows, ncol)
    t = synth.host_table(rows, ncol)
    cols = list(t.column_names)
    specs = []
    for c in cols:
        mn, mx = SO.minmax(t, c)
        rng = mx - mn
        specs.append((SO.AFFINE, SO.F32, SO.NAN_TO_NULL, mn, 1.0 / rng, 0.0))
        x = t.column(c).drop_null().to_numpy().astype(np.float64)
        specs.append((SO.DIV, SO.F64, 0, float(np.mean(x)), float(np.std(x, ddof=1)), 0.0))
    names = [c for c in cols for _ in range(2)]
    outs, valid, nulls = engine.scale_columns(fr, names, specs)
    for i, (n, sp) in enumerate(zip(names, specs)):
        v, ok = SO._values(t, n)
        exp, keep = SO.scale_reference(v, ok, sp)
        assert torch.equal(outs[i].cpu(), torch.from_numpy(exp)), (n, sp)
        assert nulls[i] == int((~keep).sum())
    del outs, valid
    for name in NAMES:
        got = _gpu(name, fr, list_of_cols=cols)
        exp = SO.__dict__[name](t, list_of_cols=cols)[0]
        for c in cols:
            g, e = got.column(c), exp.column(c)
            assert g.type == e.type and np.array_equal(np.asarray(g.is_valid()), np.asarray(e.is_valid())), (name, c)
            gv, ev = g.fill_null(0).to_numpy().astype(np.float64), e.fill_null(0).to_numpy().astype(np.float64)
            assert np.allclose(gv, ev, rtol=1e-13, atol=1e-12), (name, c, float(np.max(np.abs(gv - ev))))


def test_partitioned_equals_resident():
    from anovos_b200.frame import ColumnFrame
    from anovos_b200.partitioned import PartitionedFrame
    t = synthetic(n=100_003)
    for name in NAMES:
        for mode in ("replace", "append"):
            res = _gpu(name, ColumnFrame.from_arrow(t), list_of_cols="all", output_mode=mode)
            par = _gpu(name, PartitionedFrame.from_frame(ColumnFrame.from_arrow(t), 8192 * 4), list_of_cols="all",
                       output_mode=mode)
            if name != "z_standardization":             # exact quartiles and min / max on both
                same_tables(par, res)
            else:                                       # merged moments: mean / stddev may differ in the last bits
                assert par.column_names == res.column_names
                for c in res.column_names:
                    if pa.types.is_floating(res.schema.field(c).type):
                        assert np.allclose(par.column(c).to_numpy(zero_copy_only=False),
                                           res.column(c).to_numpy(zero_copy_only=False), rtol=1e-13, atol=1e-12, equal_nan=True)
