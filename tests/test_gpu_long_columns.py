"""Columns of 2^31 rows and more against closed-form references.

Every C entry point takes int64 row counts, and between 2^31 and 2^32 rows the kernels keep row-scale quantities in
32-bit words: the sort's run summaries and mode candidates, the bucket count's counters, the row-distinct verifier's row
numbers and positions.  NumPy cannot hold or sort a reference copy of such a column in reasonable time, so these columns
are closed-form (closed_form.py): row r holds T[(A r + B) mod 65521] and is null when r mod 97 is in a fixed set, so the
multiset of a column's values follows from per-residue counts, and per-row outputs from a table gathered by the same
index.  Marked rows sit at 2^31 - 1, 2^31 and 2^31 + 1 (a unique low value, a unique high value, a unique NaN or a
null), a null run covers bitmap words 2^26 and 2^26 + 1, the last row is marked, and past 2^32 rows 2^32 - 1 and 2^32
are marked too.  Row counts are 2^31 + 4 099, 2^32 - 1 (the most one exact mode / distinct call counts) and
2^32 + 4 099: none is a multiple of 4 or 4 096.

Columns are generated on the device in blocks of 2^26 rows; full-length outputs are compared bit for bit in blocks.
Each test states the device memory it needs and skips, naming it, when that much is not free: the GPU may be shared."""
import gc
import math

import numpy as np
import pytest

import closed_form as CF

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import anovos.data_analyzer.stats_generator as sg            # noqa: E402
from anovos_b200 import _lib, engine                          # noqa: E402
from anovos_b200.frame import Column, ColumnFrame, pack_bits_device   # noqa: E402
from anovos_b200.partitioned import PartitionedFrame          # noqa: E402

N_A = (1 << 31) + 4099
N_B = (1 << 32) - 1
N_C = (1 << 32) + 4099
GB = 1e9
PROBS = [0.0, 0.01, 0.25, 0.5, 0.75, 0.99, 1.0]
_TD = {"f32": torch.float32, "i32": torch.int32, "f64": torch.float64, "i64": torch.int64}
_NPT = {"f32": np.float32, "i32": np.int32, "f64": np.float64, "i64": np.int64}
_SD = {"f32": "float", "i32": "int", "f64": "double", "i64": "bigint"}


def _int_view(kind):
    return (np.int32, torch.int32) if _NPT[kind]().itemsize == 4 else (np.int64, torch.int64)


def need(gb):
    """Skip unless gb GB (+ 2 GB margin) of device memory are free."""
    gc.collect()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < (gb + 2) * GB:
        pytest.skip("needs %.1f GB of free device memory (+ 2 GB margin); %.1f GB free" % (gb, free / GB))


@pytest.fixture(autouse=True)
def _release():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _bits(v, kind):
    """A value of the column as the integer bits it is stored as."""
    return int(np.array([v], _NPT[kind]).view(_int_view(kind)[0])[0])


def build(col, kind):
    """-> (data tensor, validity words | None) of a LongColumn on the device, block by block."""
    n = col.n
    npi, ti = _int_view(kind)
    data = torch.empty((n + 3) // 4 * 4, dtype=ti, device="cuda")
    words = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda") if col.has_bitmap else None
    table = torch.from_numpy(col.T.view(npi)).cuda()
    ones = torch.ones(col.M, dtype=torch.bool, device="cuda")
    vmarks = {r: _bits(v, kind) for r, v in col.marks.items() if v is not None}
    bmarks = {r: v is not None for r, v in col.marks.items()}
    for r0 in range(0, n, CF.BLOCK):
        r1 = min(n, r0 + CF.BLOCK)
        data[r0:r1] = col.block(torch, r0, r1, table, 0, vmarks)
        if words is not None:
            words[r0 // 32:(r1 + 31) // 32] = pack_bits_device(col.block(torch, r0, r1, ones, False, bmarks))
    return data.view(_TD[kind])[:n], words


def frame_of(cols):
    """{name: (LongColumn, kind)} -> ColumnFrame."""
    n = {c.n for c, _ in cols.values()}.pop()
    return ColumnFrame.from_tensors({nm: build(c, k) for nm, (c, k) in cols.items()}, n_rows=n)


def check_rows(got, col, table, null_value, marks, what):
    """got (CUDA tensor [n], any 4- or 8-byte type) == table[index(r)] / null_value / marks, compared as integers."""
    it = torch.int32 if got.element_size() == 4 else torch.int64
    g = got.view(it)
    tdev = torch.from_numpy(np.ascontiguousarray(table)).cuda().view(it)
    for r0 in range(0, col.n, CF.BLOCK):
        r1 = min(col.n, r0 + CF.BLOCK)
        bad = torch.nonzero(g[r0:r1] != col.block(torch, r0, r1, tdev, null_value, marks))
        assert bad.numel() == 0, (what, "first bad row", r0 + int(bad[0]))


def check_words(got, col, table_bool, null_bit, marks, what):
    """A bitmap (int32 words) == the packed per-row bits table_bool[index(r)] / null_bit / marks."""
    tdev = torch.from_numpy(np.ascontiguousarray(table_bool)).cuda()
    for r0 in range(0, col.n, CF.BLOCK):
        r1 = min(col.n, r0 + CF.BLOCK)
        exp = pack_bits_device(col.block(torch, r0, r1, tdev, null_bit, marks))
        bad = torch.nonzero(got[r0 // 32:(r1 + 31) // 32] != exp)
        assert bad.numel() == 0, (what, "first bad word", r0 // 32 + int(bad[0]))


def _cast(vals, kind):
    return np.asarray(vals, _NPT[kind])


def _special(n, nulls=CF.NULLS):
    return CF.LongColumn(CF.table_f32_special(11), n, nulls, CF.marks("f32", n)), "f32"


def _finite(n, nulls=CF.NULLS):
    return CF.LongColumn(CF.table_f32_finite(12), n, nulls, CF.marks("f32", n)), "f32"


def _int(n, narrow=False):
    """The narrow column's marks stay inside its range, so it keeps fewer than 2^14 distinct values (direct buckets)."""
    mk = CF.marks("i32", n, values=CF.MARK_I32_NARROW if narrow else None)
    return CF.LongColumn(CF.table_i32(14 if narrow else 13, narrow=narrow), n, CF.NULLS, mk), "i32"


def _wide(n, kind):
    """64-bit columns: doubles with the special values, or int64 around 2^53 and 2^62."""
    T = CF.table_f64_special(16) if kind == "f64" else CF.table_i64(17)
    return CF.LongColumn(T, n, CF.NULLS, CF.marks(kind, n)), kind


def _ranks(n_valid):
    """Spark's ranks of PROBS, the ends, and ranks just below and above 2^31 and 2^32 where they exist."""
    rk = list(engine.quantile_ranks(n_valid, PROBS)) + [1, n_valid]
    rk += [r for r in ((1 << 31) - 1, 1 << 31, (1 << 31) + 1, (1 << 32) - 1, 1 << 32, (1 << 32) + 1) if r <= n_valid]
    return np.array(rk, np.int64)


def _cuts(T):
    fin = T[np.isfinite(T.astype(np.float64))].astype(np.float64)
    return sorted(set(np.quantile(fin, np.linspace(0.1, 0.9, 9)).tolist()) | {2.0e30})


# ---- per-column scans at 2^31 + 4 099 rows ---------------------------------------------------------------------------

SCAN_COLS = {"f32_special": lambda n: _special(n), "f32_finite": lambda n: _finite(n), "i32": lambda n: _int(n)}


@pytest.mark.parametrize("name", sorted(SCAN_COLS))
def test_scans_past_2_31_rows(name):
    """moments, moments + histogram, histogram (equal-range on the finite column), bin ids, ranks, HLL++ registers."""
    need(17.5)
    col, kind = SCAN_COLS[name](N_A)
    fr = frame_of({"x": (col, kind)})
    vals, ws, n_null = col.distribution()
    ref = CF.moments_ref(vals, ws)
    CF.check_moments(engine.moments(fr, ["x"])[0], ref, name)
    cuts = _cuts(col.T)
    lo_hi = None
    if name == "f32_finite":          # equal-range binning: the cutoffs split [min, max] into 10 equal bins
        lo_hi = [(ref["min"], ref["max"])]
        cuts = [ref["min"] + (ref["max"] - ref["min"]) / 10 * k for k in range(1, 10)]
    model = engine.BinModel(fr, ["x"], [cuts], lo_hi)
    if lo_hi:
        assert model.specs_host[0]["mode"] == 1                 # the equal-range guess is taken
    h = CF.histogram_ref(vals, ws, n_null, cuts)
    assert np.array_equal(engine.histogram(fr, model)[0, :h.size], h)
    mom, hist = engine.moments_histogram(fr, model)
    CF.check_moments(mom[0], ref, name + " fused")
    assert np.array_equal(hist[0, :h.size], h)
    rk = _ranks(ref["n_valid"])
    got = engine.select_ranks(fr, ["x"], rk[None, :])[0]
    assert np.array_equal(got, CF.rank_values(vals, ws, rk), equal_nan=True), (got, rk)
    for p in (9, 14, 18):
        assert np.array_equal(engine.hll_registers(fr, ["x"], p)[0], CF.registers_ref(vals, _SD[kind], p)), p
    ids = engine.bin_assign(fr, model)[0]
    mk = {r: (0 if v is None else int(CF.bin_table(_cast([v], kind), cuts)[0])) for r, v in col.marks.items()}
    check_rows(ids, col, CF.bin_table(col.T, cuts).astype(np.int32), 0, mk, "bin ids")


def test_code_counts_past_2_31_rows():
    need(9.5)
    card = 300
    T = np.random.default_rng(15).integers(0, card, CF.M).astype(np.int32)
    col = CF.LongColumn(T, N_A, CF.NULLS, {(1 << 31) - 1: 0, 1 << 31: None, N_A - 1: card - 1})
    d, w = build(col, "i32")
    fr = ColumnFrame.from_tensors({"s": (d, w, ["v%03d" % i for i in range(card)])})
    vals, ws, n_null = col.distribution()
    exp = np.zeros(card + 1, np.int64)
    np.add.at(exp, vals.astype(np.int64) + 1, ws)
    exp[0] = n_null
    assert np.array_equal(engine.code_counts(fr, ["s"])[0], exp.astype(np.uint64))


# ---- exact mode / distinct / ranks / registers through the bucket count and the LSD sort ------------------------------

def _heavy(n, zeros=False):
    """7.5 (or alternating -0.0 / +0.0) on every row but r = 0 mod 2^20, which holds 1 + r / 2^20: a heavy hitter of
    more than 2^31 - 1 rows; zeros test the zero run the sort keeps out of the keys."""
    k = (n - 1 >> 20) + 1
    data = torch.empty((n + 3) // 4 * 4, dtype=torch.float32, device="cuda")
    for r0 in range(0, n, CF.BLOCK):
        r1 = min(n, r0 + CF.BLOCK)
        blk = data[r0:r1]
        blk.fill_(0.0 if zeros else 7.5)
        if zeros:
            blk[(1 - r0 % 2)::2] = -0.0
        blk[0::1 << 20] = torch.arange(r0 >> 20, (r1 - 1 >> 20) + 1, dtype=torch.float32, device="cuda") + 1
    if zeros:
        vals, ws = [0.0, -0.0] + list(range(1, k + 1)), [(n + 1) // 2 - k, n // 2] + [1] * k
    else:
        vals, ws = [7.5] + list(range(1, k + 1)), [n - k] + [1] * k
    return data, CF.runs(np.array(vals, np.float32), ws)


def _constant(n):
    data = torch.full(((n + 3) // 4 * 4,), 7.5, dtype=torch.float32, device="cuda")
    return data, CF.runs(np.array([7.5], np.float32), [n])


def _sort_case(kind, n):
    """-> (ColumnFrame with column "x", (values, multiplicities, nulls), Spark dtype)."""
    if kind in ("f32_special", "i32_narrow", "i32", "f64_special", "i64"):
        col, k = _special(n) if kind == "f32_special" else _wide(n, kind[:3]) if kind[1:3] == "64" else \
            _int(n, narrow=kind == "i32_narrow")
        return frame_of({"x": (col, k)}), col.distribution(), _SD[k]
    data, dist = _heavy(n, zeros=kind == "zeros") if kind in ("heavy", "zeros") else _constant(n)
    return ColumnFrame.from_tensors({"x": data[:n]}), dist, "float"


def _check_sort(fr, dist, sd, algo, monkeypatch, what):
    monkeypatch.setattr(engine, "sort_algorithm", algo)
    vals, ws, _ = dist
    rk = _ranks(int(ws.sum()))
    assert rk.size <= 16                                        # the bucket count takes up to 16 ranks
    res, rv, regs = engine.sort_mode_distinct(fr, ["x"], rk[None, :], hll_p=9)
    exp = CF.mode_ref(vals, ws, as_int=sd == "bigint")          # a bigint mode is an exact Python int
    got = res[0]
    assert type(got[0]) is type(exp[0]), (what, got, exp)
    assert got[1:] == exp[1:] and (got[0] == exp[0] or (math.isnan(got[0]) and math.isnan(exp[0]))), (what, got, exp)
    assert np.array_equal(rv[0], CF.rank_values(vals, ws, rk), equal_nan=True), (what, rv[0], rk)
    assert np.array_equal(regs[0], CF.registers_ref(vals, sd, 9)), what


@pytest.mark.parametrize("algo", ("partition", "lsd"))
@pytest.mark.parametrize("kind", ("f32_special", "i32_narrow", "heavy", "zeros"))
def test_mode_distinct_past_2_31_rows(kind, algo, monkeypatch):
    """The bucket count (hash buckets for the special column, direct buckets for the narrow one) and the LSD sort."""
    need(28.0)
    fr, dist, sd = _sort_case(kind, N_A)
    if kind in ("heavy", "zeros"):
        assert CF.mode_ref(*dist[:2])[1] > (1 << 31) - 1       # the premise: a multiplicity past INT_MAX
    _check_sort(fr, dist, sd, algo, monkeypatch, (kind, algo))


@pytest.mark.parametrize("kind", ("f64_special", "i64"))
def test_mode_distinct_64_bit_past_2_31_rows(kind, monkeypatch):
    """The 64-bit LSD sort: doubles with the special values, and int64 beyond 2^53 with the mode as an exact int."""
    need(54.0)
    fr, dist, sd = _sort_case(kind, N_A)
    _check_sort(fr, dist, sd, "lsd", monkeypatch, kind)


@pytest.mark.parametrize("algo", ("partition", "lsd"))
@pytest.mark.parametrize("kind", ("f32_special", "i32", "heavy", "constant"))
def test_mode_distinct_at_the_row_limit(kind, algo, monkeypatch):
    """2^32 - 1 rows, the most one call counts: a constant column's mode_rows is 2^32 - 1, and a heavy hitter of
    2^32 - 4 097 rows fills one coarse group of the bucket count with more than 2^32 - 4 096 keys."""
    need(55.0)
    fr, dist, sd = _sort_case(kind, N_B)
    _check_sort(fr, dist, sd, algo, monkeypatch, (kind, algo))


# ---- impute / scale past 2^31 rows ----------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ("f32_n_A", "i32_n_A", "f32_n_C"))
def test_impute_and_scale_long_columns(case):
    """impute_fill (and valid_not_nan of the float columns); scale_columns DIV (float out), AFFINE (double out, NaN to
    null) and CONST."""
    kind, n = case[:3], N_A if case.endswith("A") else N_C
    need(26.0 if n == N_A else 36.0)
    col, kind = (_special(n) if kind == "f32" else _int(n)) if n == N_A else _finite(n, nulls=())
    fr = frame_of({"x": (col, kind)})
    isf, anv = kind == "f32", _lib.ANV_F32 if kind == "f32" else _lib.ANV_I32
    fill = _NPT[kind](-123.25 if isf else -123)
    nan_t = np.isnan(col.T) if isf else np.zeros(col.M, bool)
    mark_f = {r: (fill if v is None or v != v else v) for r, v in col.marks.items()}
    out = engine.impute_fill(fr, ["x"], [anv], [_lib.IMPUTE_NAN_MISSING if isf else 0], [engine.fill_bits(fill, anv)])[0]
    check_rows(out, col, np.where(nan_t, fill, col.T).astype(_NPT[kind]).view(np.int32), _bits(fill, kind),
               {r: _bits(v, kind) for r, v in mark_f.items()}, "impute")
    del out
    vals, ws, _ = col.distribution()
    if isf:
        words, n_nan = engine.valid_not_nan(fr, ["x"])
        assert n_nan[0] == int(ws[np.isnan(vals)].sum())
        check_words(words[0], col, ~nan_t, False, {r: v is not None and v == v for r, v in col.marks.items()},
                    "valid_not_nan")
        del words

    a, b, c = 3.5, 0.1, -2.0
    aff_f32 = n > N_A                                   # a double output of 2^32 rows would need 34 GB more
    with np.errstate(all="ignore"):
        div = lambda x: ((np.asarray(x, np.float64) - a) / b).astype(np.float32)
        aff = lambda x: ((np.asarray(x, np.float64) - a) * b + c).astype(np.float32 if aff_f32 else np.float64)
        cases = [((_lib.SCALE_DIV, _lib.ANV_F32, 0, a, b, 0.0), div),
                 ((_lib.SCALE_AFFINE, _lib.ANV_F32 if aff_f32 else _lib.ANV_F64, _lib.SCALE_NAN_TO_NULL, a, b, c), aff),
                 ((_lib.SCALE_CONST, _lib.ANV_F32, 0, 0.0, 0.0, c), lambda x: np.full(np.shape(x), c, np.float32))]
        for spec, f in cases:
            outs, valid, nulls = engine.scale_columns(fr, ["x"], [spec])
            nan_to_null = bool(spec[2] & _lib.SCALE_NAN_TO_NULL)
            table = np.asarray(f(col.T))
            out_nan = np.isnan(table)
            if nan_to_null:
                table = np.where(out_nan, 0, table).astype(table.dtype)
            it = np.int32 if table.dtype == np.float32 else np.int64
            mk = {}
            for r, v in col.marks.items():
                e = np.asarray(f(np.array([0 if v is None else v], col.T.dtype)))
                if v is None or (nan_to_null and np.isnan(e[0])):
                    e[:] = 0
                mk[r] = int(e.view(it)[0])
            check_rows(outs[0], col, table.view(it), 0, mk, ("scale", spec))
            n_null = col.distribution()[2]
            if nan_to_null:
                assert nulls[0] == n_null + int(ws[np.isnan(vals)].sum()), (nulls, n_null)
                check_words(valid[0], col, ~out_nan, False, {r: v is not None and v == v for r, v in col.marks.items()},
                            "scale bitmap")
            else:
                assert nulls[0] == n_null and valid[0] is None
            del outs, valid


# ---- row checks -----------------------------------------------------------------------------------------------------

def test_row_distinct_past_2_31_rows():
    """(r mod 65521, r mod 97) has period L = 6 355 537, so rows >= L repeat; one unique row past 2^31 and its copy in
    the last row.  The first-occurrence bitmap is rows < L and the unique row."""
    need(54.0)
    n, L, uniq = N_A, 65521 * 97, (1 << 31) + 5
    cols = {}
    for nm, m in (("a", 65521), ("b", 97)):
        d = torch.empty((n + 3) // 4 * 4, dtype=torch.int32, device="cuda")
        for r0 in range(0, n, CF.BLOCK):
            r1 = min(n, r0 + CF.BLOCK)
            d[r0:r1] = (torch.arange(r0, r1, device="cuda") % m).to(torch.int32)
        d[uniq] = d[n - 1] = -1
        cols[nm] = d[:n]
    fr = ColumnFrame.from_tensors(cols)
    nd, first = engine.row_distinct(fr, ["a", "b"])
    assert nd == L + 1
    for r0 in range(0, n, CF.BLOCK):
        r1 = min(n, r0 + CF.BLOCK)
        r = torch.arange(r0, r1, device="cuda")
        exp = pack_bits_device((r < L) | (r == uniq))
        assert torch.equal(first[r0 // 32:(r1 + 31) // 32], exp), r0


def test_row_null_counts_past_2_32_rows():
    """Three bitmaps of n_C rows (no data): count slots and the keep bitmap of rows with at most one null."""
    need(3.0)
    n = N_C
    sets = [(1, 2, 3), (2, 3, 50), (3, 60)]
    extra = {(1 << 31): (0, 1, 2), (1 << 32): (0, 2)}               # marked rows: these columns are null there
    nulls_of = np.zeros(97, np.int64)
    for s in sets:
        nulls_of[list(s)] += 1
    cols, cnt_of = {}, {}
    for j, s in enumerate(sets):
        col = CF.LongColumn(np.arange(97, dtype=np.int32), n, s, {r: None for r, js in extra.items() if j in js},
                            period=(97, 97, 1, 0))
        ones = torch.ones(97, dtype=torch.bool, device="cuda")
        w = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")
        for r0 in range(0, n, CF.BLOCK):
            r1 = min(n, r0 + CF.BLOCK)
            w[r0 // 32:(r1 + 31) // 32] = pack_bits_device(col.block(torch, r0, r1, ones, False,
                                                                      {r: False for r in col.marks}))
        cols["c%d" % j] = Column("c%d" % j, "float", n, dev=torch.zeros(4, device="cuda"), dev_valid=w, anv_dtype=_lib.ANV_F32)
    fr = ColumnFrame(dict(cols), n)
    t = np.arange(97)
    per_t = (n - 1 - t) // 97 + 1
    exp = np.bincount(nulls_of, weights=per_t, minlength=4).astype(np.int64)
    for r, js in extra.items():
        exp[nulls_of[r % 97]] -= 1
        exp[len(set(js) | {j for j, s in enumerate(sets) if r % 97 in s})] += 1
    counts, keep = engine.row_null_counts(fr, list(cols), max_keep=1)
    assert np.array_equal(counts, exp.astype(np.uint64)), (counts, exp)
    kcol = CF.LongColumn(np.arange(97, dtype=np.int32), n, (), None, period=(97, 97, 1, 0))
    km = {r: len(set(js) | {j for j, s in enumerate(sets) if r % 97 in s}) <= 1 for r, js in extra.items()}
    check_words(keep, kcol, nulls_of <= 1, False, km, "keep")


# ---- past 2^32 rows: scans, and the refusal of exact mode / distinct ----------------------------------------------------

def test_scans_past_2_32_rows():
    """n_valid and n_nonzero past 2^32, one histogram bin of more than 2^32 rows, ranks past 2^32, registers, bin ids."""
    need(35.0)
    col, kind = _finite(N_C, nulls=())
    fr = frame_of({"x": (col, kind)})
    vals, ws, n_null = col.distribution()
    ref = CF.moments_ref(vals, ws)
    assert ref["n_valid"] > (1 << 32) and ref["n_nonzero"] > (1 << 32)
    CF.check_moments(engine.moments(fr, ["x"])[0], ref, "n_C")
    cuts = [-1.0e6, 2.0e30]
    model = engine.BinModel(fr, ["x"], [cuts], None)
    h = CF.histogram_ref(vals, ws, n_null, cuts)
    assert h[2] > (1 << 32)
    assert np.array_equal(engine.histogram(fr, model)[0, :h.size], h)
    rk = _ranks(ref["n_valid"])
    assert rk.max() > (1 << 32)
    assert np.array_equal(engine.select_ranks(fr, ["x"], rk[None, :])[0], CF.rank_values(vals, ws, rk), equal_nan=True)
    for p in (9, 14, 18):
        assert np.array_equal(engine.hll_registers(fr, ["x"], p)[0], CF.registers_ref(vals, "float", p)), p
    ids = engine.bin_assign(fr, model)[0]
    mk = {r: (0 if v is None else int(CF.bin_table(_cast([v], kind), cuts)[0])) for r, v in col.marks.items()}
    check_rows(ids, col, CF.bin_table(col.T, cuts).astype(np.int32), 0, mk, "bin ids")


def test_exact_mode_and_distinct_refuse_2_32_rows():
    """sort_mode_distinct, row_distinct and the API's exact mode / distinct count raise AnvError on n_C rows, resident
    or partitioned, before any workspace is allocated."""
    need(18.0)
    col, kind = _finite(N_C, nulls=())
    fr = frame_of({"x": (col, kind)})
    pf = PartitionedFrame.from_frame(fr, 1 << 30)
    for frame in (fr, pf):
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        for algo in ("partition", "lsd"):
            engine.sort_algorithm = algo
            try:
                with pytest.raises(_lib.AnvError, match="2\\^32 rows"):
                    engine.sort_mode_distinct(frame, ["x"])
            finally:
                engine.sort_algorithm = "partition"
        assert torch.cuda.memory_allocated() == before and torch.cuda.max_memory_allocated() == before
        with pytest.raises(_lib.AnvError, match="2\\^32 rows"):
            sg.mode_computation(None, frame, ["x"])
        with pytest.raises(_lib.AnvError, match="2\\^32 rows"):
            sg.measures_of_cardinality(None, frame, ["x"], use_approx_unique_count=False)
    with pytest.raises(_lib.AnvError, match="2\\^32 rows"):
        engine.row_distinct(fr, ["x"])


# ---- a partitioned frame past 2^31 rows ---------------------------------------------------------------------------

def test_partitioned_frame_past_2_31_rows():
    """Chunks of 2^27 rows: merged moments / histogram / ranks / registers, and the exact mode through materialize(),
    equal the closed form and the resident frame."""
    need(40.0)
    col, kind = _special(N_A)
    fr = frame_of({"x": (col, kind)})
    pf = PartitionedFrame.from_frame(fr, 1 << 27)
    vals, ws, n_null = col.distribution()
    ref = CF.moments_ref(vals, ws)
    CF.check_moments(engine.moments(pf, ["x"])[0], ref, "partitioned")
    cuts = _cuts(col.T)
    model = engine.BinModel(fr, ["x"], [cuts], None)
    h = CF.histogram_ref(vals, ws, n_null, cuts)
    assert np.array_equal(engine.histogram(pf, model)[0, :h.size], h)
    rk = _ranks(ref["n_valid"])
    assert np.array_equal(engine.select_ranks(pf, ["x"], rk[None, :])[0], CF.rank_values(vals, ws, rk), equal_nan=True)
    assert np.array_equal(engine.hll_registers(pf, ["x"], 14)[0], CF.registers_ref(vals, "float", 14))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    res = engine.sort_mode_distinct(pf, ["x"])
    peak = torch.cuda.max_memory_allocated() - base
    exp = CF.mode_ref(vals, ws)
    assert res[0][1:] == exp[1:] and res[0][0] == exp[0], (res, exp)
    assert res == engine.sort_mode_distinct(fr, ["x"])
    # materialize: the column, a bool mask per chunk and their concatenation, the bitmap, the sort workspace
    ws_bytes = _lib.lib().anv_mode_distinct_partition_workspace_bytes(1, N_A)
    assert peak <= 4 * N_A + 2 * N_A + N_A // 8 + ws_bytes + 6 * (1 << 27) * 8, (peak, ws_bytes)
    print("partitioned sort_mode_distinct peak above the frame: %.2f GB" % (peak / GB))
