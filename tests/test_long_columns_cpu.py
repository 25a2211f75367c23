"""The closed-form references of the long-column tests (closed_form.py), pinned against the brute-force expanded column.

At a short period (M = 251, P = 7) the columns are expanded on the host below, at and past whole periods, with marked
rows, and every reference the GPU tests use - per-value counts, exact moments, extrema, ranks, mode, distinct count,
histogram, HLL++ registers and the per-row output tables - must equal the existing oracle helpers on the expanded
column.  The counts are also checked at the default period.  And frame.pack_bits_device, which builds the bitmaps of
materialized frames, must equal the host packing bit for bit."""
import collections
import math

import numpy as np
import pytest

import closed_form as CF
from oracle import exact as X
from oracle import spark_semantics as S

torch = pytest.importorskip("torch")

from anovos_b200 import engine                              # noqa: E402
from anovos_b200 import frame as F                          # noqa: E402

SMALL = (251, 7, 100, 17)             # (M, P, A, B): 251 is prime, 7 coprime to it
MP = 251 * 7
AT = (400, 1200)                      # where the small columns carry the marks of rows 2^31 and 2^32
SIZES = (MP - 1, MP, MP + 1, 3 * MP + 5)
TABLES = {"f32_special": (lambda: CF.table_f32_special(3, 251), "f32", "float"),
          "f32_finite": (lambda: CF.table_f32_finite(4, 251), "f32", "float"),
          "i32": (lambda: CF.table_i32(5, 251), "i32", "int"),
          "i32_narrow": (lambda: CF.table_i32(6, 251, narrow=True), "i32", "int"),
          "f64_special": (lambda: CF.table_f64_special(7, 251), "f64", "double"),
          "i64": (lambda: CF.table_i64(8, 251), "i64", "bigint")}


def _mark_values(name, kind):
    return CF.MARK_I32_NARROW if name == "i32_narrow" else \
        {"f32": CF.MARK_F32, "f64": CF.MARK_F32, "i32": CF.MARK_I32, "i64": CF.MARK_I64}[kind]


def _column(name, n):
    make, kind, _ = TABLES[name]
    return CF.LongColumn(make(), n, nulls=(2, 5), marks=CF.marks(kind, n, at=AT, run=40, values=_mark_values(name, kind)),
                         period=SMALL)


def _key(v):
    """Grouping key of the exact mode / distinct count: -0.0 is 0.0 and every NaN one value."""
    v = float(v) if isinstance(v, (float, np.floating)) else int(v)
    return "nan" if v != v else v + 0 if isinstance(v, int) else v + 0.0


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("name", sorted(TABLES))
def test_closed_form_equals_expanded_column(name, n):
    col = _column(name, n)
    vals, valid = col.expand()
    x = vals[valid]
    w, n_null = col.counts()
    assert n_null == int((~valid).sum()) and w.sum() + n_null + sum(v is not None for v in col.marks.values()) == n
    dv, dw, dn = col.distribution()
    assert dn == n_null and int(dw.sum()) == x.size

    # moments, extrema, counts
    ref = CF.moments_ref(dv, dw)
    assert ref["n_valid"] == x.size and ref["n_nonzero"] == int(np.count_nonzero(x != 0))
    f = x[~np.isnan(x)] if x.dtype.kind == "f" else x
    assert ref["min"] == float(f.min()) and ref["max"] == float(f.max())
    assert ref["finite"] == bool(np.isfinite(x.astype(np.float64)).all())
    if ref["finite"]:
        en, mean, m2, m3, m4 = X.exact_central(x)
        assert (ref["mean"], ref["m2"], ref["m3"], ref["m4"]) == (float(mean), float(m2), float(m3), float(m4))

    # mode (ties to the smallest value, NaN last) and distinct count
    cnt = collections.Counter(_key(v) for v in x.tolist())
    top = max(cnt.values())
    best = sorted((k for k, c in cnt.items() if c == top), key=lambda k: (k == "nan", 0 if k == "nan" else k))[0]
    mode, rows, nd = CF.mode_ref(dv, dw)
    assert rows == top and nd == len(cnt)
    assert (best == "nan" and math.isnan(mode)) or mode == best

    # order statistics at Spark's ranks, the ends and both sides of the marks
    srt = np.sort(x.astype(np.float64))
    rk = list(engine.quantile_ranks(x.size, [0.0, 0.01, 0.25, 0.5, 0.75, 0.99, 1.0])) + [1, 2, x.size - 1, x.size, 0]
    got = CF.rank_values(dv, dw, rk)
    exp = [srt[r - 1] if r else np.nan for r in rk]
    assert np.array_equal(got, np.array(exp), equal_nan=True)

    # histogram and per-row bin ids
    fin = f[np.isfinite(f.astype(np.float64))].astype(np.float64)
    cuts = sorted(set(np.quantile(fin, [0.1, 0.3, 0.5, 0.7, 0.9]).tolist()) | {2.0e30})
    ids = X.exact_bins(vals, valid, cuts)
    assert np.array_equal(CF.histogram_ref(dv, dw, n_null, cuts),
                          np.bincount(ids, minlength=len(cuts) + 2).astype(np.uint64))
    table = torch.from_numpy(CF.bin_table(col.T, cuts).astype(np.int32))
    mk = {r: int(CF.bin_table(np.array([v], col.T.dtype), cuts)[0]) if v is not None else 0 for r, v in col.marks.items()}
    for r0 in (0, 96, n // 2 // 32 * 32):
        blk = col.block(torch, r0, n, table, 0, mk).numpy()
        assert np.array_equal(blk, ids[r0:]), (name, n, r0)

    # HLL++ registers: the distribution's distinct values give the registers of every value
    sd = TABLES[name][2]
    for p in (9, 14):
        assert np.array_equal(CF.registers_ref(dv, sd, p), S.hll_registers(S.hll_hashes(x, sd), p))


def test_counts_at_the_default_period():
    """One default period (M P = 6 355 537 rows) and a few rows past it, expanded."""
    for n in (CF.M * CF.P - 1, CF.M * CF.P + 3):
        col = CF.LongColumn(np.arange(CF.M, dtype=np.int32), n, marks={n - 1: None, 7: 123456})
        vals, valid = col.expand()
        w, n_null = col.counts()
        assert np.array_equal(w, np.bincount(vals[valid & (np.arange(n) != 7)], minlength=CF.M)) and n_null == (~valid).sum()


def test_marks_are_unique_values():
    for name, (make, kind, _) in TABLES.items():
        T = make()
        mk = _mark_values(name, kind)
        assert not np.isin(T, np.array(list(mk.values()), T.dtype)).any()
    narrow = np.concatenate([CF.table_i32(6, narrow=True), list(CF.MARK_I32_NARROW.values())])
    assert narrow.max() - narrow.min() < 1 << 14                              # direct buckets span the whole column
    assert math.isnan(CF.MARK_NAN64) and not np.isin(np.float64(CF.MARK_NAN64).view(np.uint64), CF.NAN64.view(np.uint64))
    assert np.isin(CF.table_i64(8), [2 ** 53 + 1, 2 ** 53 - 1]).any()         # integers a double cannot tell apart
    assert math.isnan(CF.MARK_NAN32) and not np.isin(np.float32(CF.MARK_NAN32).view(np.uint32), CF.NAN32.view(np.uint32))
    assert all(np.float32(v) == v for v in CF.MARK_F32.values())
    m = CF.marks("f32", (1 << 32) + 4099)
    assert m[(1 << 31) - 1] == CF.MARK_F32["lo"] and m[(1 << 32) + 4098] == CF.MARK_F32["tail"]
    assert all(m[r] is None for r in range((1 << 31) + 2, (1 << 31) + 64))        # bitmap words 2^26 and 2^26 + 1
    assert m[1 << 32] is None and m[(1 << 32) - 1] == CF.MARK_F32["hi2"]


@pytest.mark.parametrize("n", (0, 1, 31, 32, 33, 10 ** 6 + 7))
@pytest.mark.parametrize("fill", ("random", "all_true"))
def test_pack_bits_device_matches_pack_validity(n, fill):
    m = np.random.default_rng(n).random(n) < 0.5 if fill == "random" else np.ones(n, bool)
    got = F.pack_bits_device(torch.from_numpy(m))
    assert got.dtype == torch.int32 and got.numel() == (n + 31) // 32
    assert np.array_equal(got.numpy(), F._pack_validity(m)[:(n + 31) // 32])


def test_pack_bits_device_across_steps(monkeypatch):
    """Steps of 64 rows: a mask of several steps and a ragged last one packs as one piece."""
    monkeypatch.setattr(F, "_PACK_BLOCK_ROWS", 64)
    rng = np.random.default_rng(1)
    for n in (63, 64, 65, 129, 1000, 4099):
        m = rng.random(n) < 0.3
        assert np.array_equal(F.pack_bits_device(torch.from_numpy(m)).numpy(), F._pack_validity(m)[:(n + 31) // 32]), n
