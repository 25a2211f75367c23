"""Wide frames: thousands of columns in one launch, and more columns than one launch takes (ANV_MAX_LAUNCH_COLS).

Several code paths depend on the column count alone: the column of a CTA beyond the first (32 columns per CTA in the
drift reduce, 128 in the bucket count's final kernel), tile sizes picked from the number of columns (8 tiles per SM over
the whole launch), the row null counts' shared-memory histogram (up to 6 143 columns) and bit planes, the row hash and
comparison loops over every column, the code histograms grouped by cardinality class, and the split of a frame wider
than 65 535 columns into column blocks.

How the columns are built, so that the references stay cheap at tens of thousands of columns and no column can be
mistaken for another:
* column j holds pattern j mod 97 (97 is prime: a result shifted by 1, 32, 128, 1 024 or 65 535 columns lands on a
  different pattern).  The pattern fixes the dtype, which rotates, so the descriptor array mixes types everywhere;
* the patterns hold the special cases of the kernel-edge tests: all-null columns, columns without a bitmap, a single
  valid value, constant columns, NaN payloads, -0.0 and subnormals, integer extremes, int64 beyond 2^53, heavy hitters,
  and null rates from 0 to 1;
* every column but the all-null and constant ones carries a mark in its last row: the value 10^6 + j (exact in float32)
  or, for strings, its own dictionary entry.  Its maximum, distinct count, order statistics, bins and registers then
  name the column;
* each reference is computed once per pattern from the other rows and then extended by the mark: exact power sums
  (oracle.exact) are additive, a sorted list takes one insertion, a histogram or a register array one update.
Every input is built from a seed; each test asserts the premise it relies on."""
import bisect
import math
from fractions import Fraction

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from golden_util import assert_frames_match
from oracle import api as O
from oracle import exact as X
from oracle import row_checks as RC
from oracle import spark_semantics as S

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import anovos.data_analyzer.quality_checker as qc          # noqa: E402
import anovos.data_analyzer.stats_generator as sg          # noqa: E402
from anovos_b200 import _lib, engine                       # noqa: E402
from anovos_b200.frame import ColumnFrame, _pack_validity  # noqa: E402
from anovos_b200.partitioned import PartitionedFrame       # noqa: E402

N_PAT = 97
KINDS = ("spread", "all_null", "no_bitmap", "single", "constant", "nan_payloads", "zero_subnormal", "extremes", "heavy",
         "beyond_2_53")
UNMARKED = ("all_null", "constant")
CARDS = (3, 20, 38, 39, 300, 5000, 10238, 10239, 12000, 20000)   # string patterns: every cardinality class
_NP = {"f32": np.float32, "f64": np.float64, "i32": np.int32, "i64": np.int64, "str": np.int32}
_SD = {"f32": "float", "f64": "double", "i32": "int", "i64": "bigint", "str": "string"}
NAN32 = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x7FC00123], np.uint32).view(np.float32)
NAN64 = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF], np.uint64).view(np.float64)
MARK = 10 ** 6
SMEM_SLOTS = 6144           # NC_SMEM_SLOTS in rows.cu: shared-memory histogram up to 6 143 columns


def _mark(j):
    return MARK + j


# ---- patterns ----------------------------------------------------------------------------------------------------

class Pattern:
    """Rows of pattern k: `body` rows from the seed, then (marked patterns) one row for the column's mark."""

    def __init__(self, k, n_rows, dts, cards=CARDS):
        rng = np.random.default_rng(9000 + k)
        self.k, self.dt = k, dts[k % len(dts)]
        self.kind = KINDS[(k // len(dts)) % len(KINDS)]
        self.marked = self.kind not in UNMARKED
        m = n_rows - 1 if self.marked else n_rows
        rate = ((k * 7) % 11) / 10.0
        T = _NP[self.dt]
        isf = self.dt in ("f32", "f64")
        self.card = cards[(k // len(dts)) % len(cards)] if self.dt == "str" else 0
        if self.dt == "str":
            v = rng.integers(0, self.card, m)
            if self.kind == "heavy":
                v = np.where(rng.random(m) < 0.9, 0, v)
        elif self.kind in ("spread", "all_null", "no_bitmap", "single", "heavy") or (self.kind == "nan_payloads" and not isf):
            v = rng.normal(0.0, 1000.0, m) if isf else rng.integers(-10 ** 5, 10 ** 5, m)
            if self.kind in ("heavy", "nan_payloads"):
                v = np.where(rng.random(m) < 0.9, 42, v)
        elif self.kind == "constant":
            v = np.full(m, 3.25 if isf else -7)
        elif self.kind == "nan_payloads":
            v = rng.normal(5.0, 2.0, m).astype(T)
            nans = NAN32 if self.dt == "f32" else NAN64
            v = np.where(rng.random(m) < 0.3, nans[rng.integers(0, nans.size, m)], v)
        elif self.kind == "zero_subnormal":
            if isf:
                cat = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, 1.5], np.float32) if self.dt == "f32" else \
                    np.array([0.0, -0.0, 5e-324, -5e-324, 1e-310, 1.5])
            else:
                cat = np.array([-1, 0, 1])
            v = cat[rng.integers(0, cat.size, m)]
        elif self.kind == "extremes":
            if isf:
                f = np.finfo(T)
                cat = np.array([f.max, -f.max, np.inf, -np.inf, f.tiny, 0.0, 1.0], T)
            else:
                i = np.iinfo(T)
                cat = np.array([i.min, i.max, i.min + 1, 0, -1], T)
            v = cat[rng.integers(0, cat.size, m)]
        else:                                                  # beyond_2_53 (or the edge of the type's exact range)
            base = {"f32": 2 ** 24, "f64": 2 ** 53, "i32": 2 ** 31 - 20, "i64": 2 ** 53}[self.dt]
            v = np.array([base + int(d) for d in rng.integers(-9, 10, m) * (2 if self.dt == "f32" else 1)], dtype=object)
            if self.dt == "i64":
                v = np.where(rng.random(m) < 0.1, 2 ** 62 + 1, v)
        self.body = np.asarray(v).astype(T)
        if self.kind in ("all_null", "single"):
            self.valid = np.zeros(m, bool)
        elif self.kind == "no_bitmap":
            self.valid = np.ones(m, bool)
        else:
            self.valid = rng.random(m) >= rate
        self.dic = ["v%06d" % i for i in range(self.card)]
        self.full = np.concatenate([self.body, np.zeros(1, T)]) if self.marked else self.body
        self.full_valid = np.concatenate([self.valid, [True]]) if self.marked else self.valid
        self._summary()

    def mark_value(self, j):
        """The mark as the column's value (strings: code 0, the entry "m<j>" that sorts before every "v..." entry)."""
        return 0 if self.dt == "str" else _mark(j)

    def column(self, j):
        """(values, valid) of column j on the host."""
        v = self.full.copy()
        if self.dt == "str" and self.marked:
            v = v + 1
        if self.marked:
            v[-1] = self.mark_value(j)
        return v, self.full_valid

    def dictionary(self, j):
        return (["m%07d" % j] + self.dic) if self.marked else self.dic

    def _summary(self):
        x = self.body[self.valid]
        self.n = int(x.size)
        if self.dt == "str":
            self.codes = np.bincount(x, minlength=self.card).astype(np.uint64)
            self.nulls = int((~self.valid).sum())
            return
        isf = x.dtype.kind == "f"
        self.nz = int(np.count_nonzero(x != 0))
        nn = x[~np.isnan(x)] if isf else x
        self.mn = None if nn.size == 0 else nn.min().item()
        self.mx = None if nn.size == 0 else nn.max().item()
        self.finite = not isf or bool(np.isfinite(x).all())
        if self.finite:
            N, E = X._scaled_ints(x)
            sc = Fraction(2) ** E
            self.sums = [Fraction(sum(v ** p for v in N)) * sc ** p for p in (1, 2, 3, 4)]
        self.srt = np.sort(x.astype(np.float64)) if isf else np.sort(x)        # NaN last, int64 exact
        with np.errstate(invalid="ignore"):
            xn = x.astype(np.float64) + 0.0 if isf else x    # -0.0 -> 0.0
        if isf:
            xn[np.isnan(xn)] = np.nan                        # every payload one NaN
        self.u, self.c = np.unique(xn, return_counts=True)
        # bins: cutoffs from the pattern's finite values, and one between the marks of the first and last columns
        fin = x[np.isfinite(x)].astype(np.float64) if isf else x.astype(np.float64)
        cut = set(np.quantile(fin, np.linspace(0.1, 0.9, 9)).tolist()) if fin.size else set()
        self.cuts = sorted(cut | {MARK + 1500.5})
        self.ids = X.exact_bins(self.body, self.valid, self.cuts)
        self._regs = {}

    # ---- references of column j (the pattern's rows + the mark) ----
    def mark_bin(self, j):
        return 1 + bisect.bisect_left(self.cuts, _mark(j))

    def bins(self, j):
        return np.concatenate([self.ids, [self.mark_bin(j)]]) if self.marked else self.ids

    def hist(self, j):
        return np.bincount(self.bins(j), minlength=len(self.cuts) + 2).astype(np.uint64)

    def rank_value(self, j, r):
        """Value of 1-based rank r among the non-null values of column j, as float64."""
        if not self.marked:
            return float(self.srt[r - 1])
        pos = int(np.searchsorted(self.srt, _mark(j)))
        return float(self.srt[r - 1]) if r - 1 < pos else (float(_mark(j)) if r - 1 == pos else float(self.srt[r - 2]))

    def n_valid(self):
        return self.n + self.marked

    def mode(self, j):
        """-> (mode, mode_rows, n_distinct) with ties to the smallest value, NaN ranked last; (None, None, 0) if empty."""
        ints = self.dt == "i64"
        conv = (lambda v: int(v)) if ints else (lambda v: float(v))
        if self.u.size == 0:
            return (conv(_mark(j)), 1, 1) if self.marked else (None, None, 0)
        best = int(self.c.max())
        top = conv(self.u[self.c == best][0])
        if not self.marked:
            return top, best, int(self.u.size)
        if best > 1:
            return top, best, int(self.u.size) + 1
        v0 = conv(self.u[0])
        return (v0 if (v0 == v0 and v0 < _mark(j)) else conv(_mark(j))), 1, int(self.u.size) + 1

    def registers(self, j, p):
        if p not in self._regs:
            x = self.body[self.valid]
            if self.dt == "str":
                x = np.array(self.dic, dtype=object)[x]
            self._regs[p] = S.hll_registers(S.hll_hashes(x, _SD[self.dt]), p)
        r = self._regs[p]
        if not self.marked:
            return r
        mv = np.array(["m%07d" % j], dtype=object) if self.dt == "str" else np.array([_mark(j)], _NP[self.dt])
        return np.maximum(r, S.hll_registers(S.hll_hashes(mv, _SD[self.dt]), p))

    def code_counts(self, j):
        if self.marked:
            return np.concatenate([[self.nulls, 1], self.codes]).astype(np.uint64)
        return np.concatenate([[self.nulls], self.codes]).astype(np.uint64)

    def check_moments(self, rec, j, name):
        n = self.n_valid()
        mk = _mark(j) if self.marked else None
        assert rec["n_valid"] == n, name
        assert rec["n_nonzero"] == self.nz + self.marked, name
        if n == 0:
            assert math.isnan(rec["min"]) and math.isnan(rec["max"]), name
            return
        mn = self.mn if mk is None else (mk if self.mn is None else min(self.mn, mk))
        mx = self.mx if mk is None else (mk if self.mx is None else max(self.mx, mk))
        if mn is None:                                     # nothing but NaN
            assert math.isnan(rec["min"]) and math.isnan(rec["max"]), name
        else:
            assert rec["min"] == float(mn) and rec["max"] == float(mx), (name, rec["min"], rec["max"], mn, mx)
        if not self.finite:
            for f in ("mean", "m2", "m3", "m4"):
                assert not math.isfinite(rec[f]), (name, f, rec[f])
            return
        s = list(self.sums)
        if mk is not None:
            s = [s[p - 1] + Fraction(mk) ** p for p in (1, 2, 3, 4)]
        a = s[0] / n
        m2 = s[1] - a * s[0]
        m3 = s[2] - 3 * a * s[1] + 2 * a * a * s[0]
        m4 = s[3] - 4 * a * s[2] + 6 * a * a * s[1] - 3 * a * a * a * s[0]
        mean, m2, m3, m4 = float(a), float(m2), float(m3), float(m4)
        sd = math.sqrt(m2 / n)
        assert abs(rec["mean"] - mean) <= 1e-9 * max(abs(mean), sd) + n * 2.0 ** -1074, (name, rec["mean"], mean)
        if m2 == 0.0:                                      # constant column: exactly zero
            assert rec["m2"] == 0.0 and rec["m3"] == 0.0 and rec["m4"] == 0.0, name
            return
        for k, (g, e) in enumerate(((rec["m2"], m2), (rec["m3"], m3), (rec["m4"], m4))):
            assert abs(g - e) <= 1e-6 * abs(e) + 1e-9 * n * sd ** (k + 2), (name, "M%d" % (k + 2), g, e)


class WideFrame:
    """n_cols columns of n_rows rows; column j = pattern j mod 97 (+ its mark).  Columns of one pattern share one
    device allocation (rows of a 2-D tensor) and one validity bitmap."""

    def __init__(self, n_cols, n_rows, dts, cards=CARDS):
        assert n_rows % 4 == 0                             # every row of the 2-D tensors stays 16-byte aligned
        self.n_cols, self.n_rows = n_cols, n_rows
        self.pats = [Pattern(k, n_rows, dts, cards) for k in range(N_PAT)]
        self.names = ["c%05d" % j for j in range(n_cols)]
        data = {}
        for P in self.pats:
            js = np.arange(P.k, n_cols, N_PAT)
            if js.size == 0:
                continue
            M = np.tile(P.full + (1 if (P.dt == "str" and P.marked) else 0), (js.size, 1)).astype(_NP[P.dt])
            if P.marked:
                M[:, -1] = [P.mark_value(j) for j in js]
            dev = torch.from_numpy(M).cuda()
            vw = None if P.full_valid.all() else torch.from_numpy(_pack_validity(P.full_valid)).cuda()
            for i, j in enumerate(js.tolist()):
                data[j] = (dev[i], vw, P.dictionary(j)) if P.dt == "str" else (dev[i], vw)
        self.fr = ColumnFrame.from_tensors({self.names[j]: data[j] for j in range(n_cols)})

    def pat(self, j):
        return self.pats[j % N_PAT]

    def of(self, *dts):
        return [j for j in range(self.n_cols) if self.pat(j).dt in dts]

    def table(self, js):
        arrays = []
        for j in js:
            P = self.pat(j)
            v, valid = P.column(j)
            if P.dt == "str":
                dic = P.dictionary(j)
                arrays.append(pa.array([dic[c] for c in v.tolist()], pa.string(), mask=~valid))
            else:
                arrays.append(pa.array(v, mask=~valid))
        return pa.table(arrays, names=[self.names[j] for j in js])


def _sample(n_cols, every=37):
    """Every `every`-th column, the first and last, and both sides of 32, 128, 1 056 and 65 535."""
    s = set(range(0, n_cols, every)) | {n_cols - 1}
    for b in (32, 128, 1056, 6144, 65534, 65535, 65536):
        s |= {c for c in (b - 2, b - 1, b, b + 1) if 0 <= c < n_cols}
    return sorted(s)


def _ranks(n_valid, n_ranks):
    if n_valid == 0:
        return [0] * n_ranks
    r = [1, n_valid, 2, n_valid - 1] + [max(1, int(n_valid * q)) for q in np.linspace(0.01, 0.99, n_ranks - 4)]
    return [min(max(1, v), n_valid) for v in r]


def _same_float(a, b):
    return np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64), equal_nan=True)


def _same_results(a, b):
    """Equal lists of (mode, mode_rows, n_distinct), a NaN mode equal to a NaN mode."""
    return len(a) == len(b) and all(x[1:] == y[1:] and type(x[0]) is type(y[0]) and
                                    (x[0] == y[0] or (x[0] != x[0] and y[0] != y[0])) for x, y in zip(a, b))


# ---- about 3 000 columns in one launch ------------------------------------------------------------------------------

WIDE_COLS, WIDE_ROWS = 3000, 3004


@pytest.fixture(scope="module")
def wide():
    w = WideFrame(WIDE_COLS, WIDE_ROWS, ("f32", "f64", "i32", "i64", "str"))
    assert w.n_cols > 1056 > 128 > 32                      # past the first CTA of 32 / 128 columns, >= 8 tiles per SM
    return w


def _model(w, js):
    return engine.BinModel(w.fr, [w.names[j] for j in js], [w.pat(j).cuts for j in js], None)


def test_moments_of_3000_columns(wide):
    js = wide.of("f32", "f64", "i32", "i64")
    got = engine.moments(wide.fr, [wide.names[j] for j in js])
    for i, j in enumerate(js):
        wide.pat(j).check_moments(got[i], j, wide.names[j])


def test_histograms_and_bin_ids_of_3000_columns(wide, monkeypatch):
    js = wide.of("f32", "f64", "i32", "i64")
    model = _model(wide, js)
    got = {"hist": engine.histogram(wide.fr, model)}
    moms = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("ANV_FUSED_STAGED", flag)
        moms[flag], got["moments_hist staged=" + flag] = engine.moments_histogram(wide.fr, model)
    ids = engine.bin_assign(wide.fr, model).cpu().numpy()
    for i, j in enumerate(js):
        P = wide.pat(j)
        h = P.hist(j)
        for label, g in got.items():
            assert np.array_equal(g[i, :h.size], h), (wide.names[j], label)
        assert np.array_equal(ids[i], P.bins(j)), wide.names[j]
        for flag, m in moms.items():
            P.check_moments(m[i], j, (wide.names[j], flag))


def test_code_counts_of_every_cardinality_class(wide):
    js = wide.of("str")
    card = {j: len(wide.pat(j).dictionary(j)) for j in js}
    cls = [0 if c + 1 <= 40 else (1 if c + 1 <= 10240 else 2) for c in card.values()]
    assert min(cls.count(0), cls.count(1), cls.count(2)) >= 10 and sum(c > 10240 for c in card.values()) >= 2
    got = engine.code_counts(wide.fr, [wide.names[j] for j in js])
    for i, j in enumerate(js):
        assert np.array_equal(got[i], wide.pat(j).code_counts(j)), wide.names[j]


def test_select_20_ranks_of_3000_columns(wide):
    js = wide.of("f32", "f64", "i32", "i64")
    rk = np.array([_ranks(wide.pat(j).n_valid(), 20) for j in js])
    assert rk.shape[1] > 16                                # two selections per column group
    got = engine.select_ranks(wide.fr, [wide.names[j] for j in js], rk)
    for i, j in enumerate(js):
        exp = [wide.pat(j).rank_value(j, r) if r else np.nan for r in rk[i]]
        assert _same_float(got[i], exp), (wide.names[j], got[i], exp)


def _check_mode_distinct(w, js, got, qv=None, rk=None, regs=None, p=None):
    for i, j in enumerate(js):
        P = w.pat(j)
        mode, rows, nd = P.mode(j)
        g = got[i]
        assert g[2] == nd and g[1] == rows, (w.names[j], g, (mode, rows, nd))
        if mode is not None:
            assert type(g[0]) is type(mode), (w.names[j], g)
            assert g[0] == mode or (math.isnan(g[0]) and math.isnan(mode)), (w.names[j], g, mode)
        if qv is not None:
            assert _same_float(qv[i], [P.rank_value(j, r) if r else np.nan for r in rk[i]]), w.names[j]
        if regs is not None:
            assert np.array_equal(regs[i], P.registers(j, p)), (w.names[j], p)


@pytest.mark.parametrize("algo", ["partition", "lsd"])
def test_mode_distinct_and_registers_of_3000_columns(wide, algo, monkeypatch):
    monkeypatch.setattr(engine, "sort_algorithm", algo)
    js = wide.of("f32", "f64", "i32", "i64")
    names = [wide.names[j] for j in js]
    rk = np.array([_ranks(wide.pat(j).n_valid(), 16) for j in js])
    got, qv = engine.sort_mode_distinct(wide.fr, names, rk)
    _check_mode_distinct(wide, js, got, qv, rk)
    for p in (9, 12):
        got, _, regs = engine.sort_mode_distinct(wide.fr, names, None, hll_p=p)
        _check_mode_distinct(wide, js, got, regs=regs, p=p)


def test_sort_batches_split_at_arbitrary_columns(wide, monkeypatch):
    """A workspace budget of 250 columns per batch: batch boundaries fall at columns that are no multiple of 97."""
    js = wide.of("f32", "f64", "i32", "i64")
    names = [wide.names[j] for j in js]
    rk = np.array([_ranks(wide.pat(j).n_valid(), 5) for j in js])
    for algo in ("partition", "lsd"):
        monkeypatch.setattr(engine, "sort_algorithm", algo)
        monkeypatch.setattr(engine, "SORT_WORKSPACE_BUDGET", 24 << 30)
        whole = engine.sort_mode_distinct(wide.fr, names, rk, hll_p=9)
        _check_mode_distinct(wide, js, *whole[:2], rk, whole[2], 9)
        for kb, dts in ((32, ("f32", "i32")), (64, ("f64", "i64"))):
            if algo == "lsd" or kb == 64:
                per = engine._lib.lib().anv_mode_distinct_workspace_bytes(1, wide.n_rows, kb)
            else:
                per = engine._lib.lib().anv_mode_distinct_partition_workspace_bytes(1, wide.n_rows)
            monkeypatch.setattr(engine, "SORT_WORKSPACE_BUDGET", 250 * per)
            n = len(wide.of(*dts))
            assert engine._mode_distinct_batch_size(wide.fr, n, per) == 250 < n and 250 % N_PAT
            got = engine.sort_mode_distinct(wide.fr, names, rk, hll_p=9)
            assert _same_results(got[0], whole[0]) and _same_float(got[1], whole[1]), (algo, kb)
            assert np.array_equal(got[2], whole[2]), (algo, kb)


@pytest.mark.parametrize("p", [9, 14, 15, 18])
def test_hll_registers(wide, p):
    """p <= 14 keeps the registers in shared memory; 15..18 take the global-register kernel (approx_count_distinct at
    rsd < 0.00864).  At p 15 and 18 the first 400 columns (3.3 GB of registers for all 3 000)."""
    assert (S.hll_precision(0.008), S.hll_precision(0.005), S.hll_precision(0.0025)) == (15, 16, 18)
    js = wide.of("f32", "f64", "i32", "i64")
    if p > 14:
        js = [j for j in js if j < 400]
    got = engine.hll_registers(wide.fr, [wide.names[j] for j in js], p)
    for i, j in enumerate(js):
        assert np.array_equal(got[i], wide.pat(j).registers(j, p)), (wide.names[j], p)


@pytest.mark.parametrize("rsd,p", [(0.008, 15), (0.0025, 18)])
def test_approx_unique_count_at_high_precision(wide, rsd, p):
    assert S.hll_precision(rsd) == p
    js = list(range(400))
    names = [wide.names[j] for j in js]
    got = sg.uniqueCount_computation(None, wide.fr, list_of_cols=names, compute_approx_unique_count=True, rsd=rsd).toPandas()
    exp = O.uniqueCount_computation(wide.table(js), list_of_cols=names, compute_approx_unique_count=True, rsd=rsd)
    assert got["attribute"].tolist() == exp["attribute"].tolist()
    assert got["unique_values"].astype(int).tolist() == exp["unique_values"].astype(int).tolist()


# ---- many columns, several tiles each -------------------------------------------------------------------------------

TILED_COLS, TILED_ROWS = 1100, 300_032


@pytest.fixture(scope="module")
def tiled():
    from anovos_b200 import synth
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_col = -(-8 * sms // TILED_COLS)                    # pick_tile_rows: >= 8 tiles per SM over the launch ...
    t = 16384
    while t < TILED_ROWS // per_col and t < 262144:       # ... of at most 256 Ki rows
        t <<= 1
    assert TILED_COLS >= 8 * sms and t == 262144 and TILED_ROWS > t   # the largest tile, and more than one per column
    js = _sample(TILED_COLS)
    return synth.device_frame(TILED_ROWS, TILED_COLS, cat_every=8), synth.host_table(TILED_ROWS, TILED_COLS, cat_every=8,
                                                                                     columns=js)


@pytest.mark.parametrize("fn", ["measures_of_counts", "measures_of_centralTendency", "measures_of_percentiles",
                                "measures_of_shape", "measures_of_cardinality"])
def test_stats_of_1100_columns_of_two_tiles(tiled, fn):
    """The whole frame in one call; the oracle on its NumPy twin, on every 37th column and those next to 32, 128, 1 056."""
    fr, t = tiled
    got = getattr(sg, fn)(None, fr).toPandas()
    numeric_only = fn in ("measures_of_percentiles", "measures_of_shape")
    assert len(got) == (sum(c % 8 != 7 for c in range(TILED_COLS)) if numeric_only else TILED_COLS)
    exp = getattr(O, fn)(t)
    assert_frames_match(got.set_index("attribute").loc[exp["attribute"]].reset_index(), exp)


# ---- drift ---------------------------------------------------------------------------------------------------------

def _drift_tables(wide_keys, seed):
    rng = np.random.default_rng(seed)
    cards = (5, 40, 95, 97, 150, 400) if wide_keys else (5, 20, 40, 60, 80, 85)
    out = []
    for shift in (0, 1):
        n = 5000 + 17 * shift
        cols = {}
        for j in range(300):
            dt = ("f32", "f64", "i32", "i64")[j % 4]
            v = rng.normal(j % 7 + 0.15 * shift * (j % 5), 1.0 + j % 3, n)
            v = v.astype(_NP[dt]) if dt in ("f32", "f64") else np.round(v * 10).astype(_NP[dt])
            cols["x%03d" % j] = pa.array(v, mask=rng.random(n) < 0.05 * (j % 3))
        for j in range(40):
            card = cards[j % len(cards)]
            k = np.minimum(rng.geometric(4.0 / card, n) - 1 + shift * (j % 3), card + 2)
            cols["s%02d" % j] = pa.array(["k%04d" % c for c in k.tolist()], mask=rng.random(n) < 0.03 * (j % 2))
        out.append(pa.table(cols))
    return out, cards


@pytest.mark.parametrize("wide_keys", [False, True])
@pytest.mark.parametrize("bin_method", ["equal_range", "equal_frequency"])
def test_drift_of_340_columns(tmp_path, bin_method, wide_keys):
    """300 numeric and 40 string columns: the reduce kernel maps 32 columns to a CTA; with a string table wider than
    96 keys every column goes through the wide kernel, where the narrow ones return early."""
    import anovos.drift_stability.drift_detector as dd
    (src, tgt), cards = _drift_tables(wide_keys, 340 + wide_keys)
    width = [len(set(src.column("s%02d" % j).to_pylist()) | set(tgt.column("s%02d" % j).to_pylist())) for j in range(40)]
    assert (max(width) > 96) == wide_keys and min(width) <= 96
    kw = dict(method_type="all", bin_method=bin_method, use_sampling=False)
    got = dd.statistics(None, tgt, src, source_path=str(tmp_path / "g"), **kw).toPandas()
    exp = O.statistics(tgt, src, source_path=str(tmp_path / "o"), **kw)
    again = dd.statistics(None, tgt, None, pre_existing_source=True, source_path=str(tmp_path / "g"), **kw).toPandas()
    assert got["attribute"].tolist() == exp["attribute"].tolist() == again["attribute"].tolist() and len(got) == 340
    for m in ("PSI", "HD", "JSD", "KS"):
        e = np.array([0.0 if v is None else v for v in exp[m].tolist()], float)
        for label, g in (("source", got), ("saved model", again)):
            assert np.allclose(g[m].values.astype(float), e, rtol=1e-9, atol=1e-12), (m, label)
    assert got["flagged"].tolist() == exp["flagged"].tolist()


# ---- row checks ----------------------------------------------------------------------------------------------------

def _null_frame(n_cols, n_rows, seed):
    """Float32 columns whose rows have every null count from 0 (row 0) to the number of columns with a bitmap (last
    row); every 101st column has no bitmap.  -> (ColumnFrame, pyarrow Table, columns with a bitmap)"""
    rng = np.random.default_rng(seed)
    p = np.arange(n_rows) / (n_rows - 1)
    null = rng.random((n_cols, n_rows)) < p[None, :]
    null[::101] = False
    words = torch.from_numpy(np.stack([_pack_validity(~r) for r in null])).cuda()
    zeros = torch.zeros(n_rows, dtype=torch.float32, device="cuda")
    names = ["n%05d" % j for j in range(n_cols)]
    fr = ColumnFrame.from_tensors({nm: (zeros, None if j % 101 == 0 else words[j]) for j, nm in enumerate(names)})
    z = np.zeros(n_rows, np.float32)
    t = pa.table([pa.array(z, mask=null[j]) for j in range(n_cols)], names=names)
    return fr, t, n_cols - len(range(0, n_cols, 101))


@pytest.mark.parametrize("n_cols", [6143, 6144, 20000, 70000])
def test_null_rows_of_wide_frames(n_cols):
    """6 143 columns keep the histogram in shared memory, 6 144 do not; 20 000 bitmaps need 15 bit planes per row count,
    70 000 need all 17 (beyond ANV_MAX_LAUNCH_COLS: the null counts run over rows only)."""
    fr, t, n_bm = _null_frame(n_cols, 96, n_cols)
    assert (n_cols + 1 <= SMEM_SLOTS) == (n_cols == 6143)
    assert n_bm.bit_length() == {6143: 13, 6144: 13, 20000: 15, 70000: 17}[n_cols]
    for kw in (dict(), dict(treatment=True, treatment_threshold=0.5)):
        odf, st = qc.nullRows_detection(None, fr, **kw)
        exp_odf, exp_st = RC.nullRows_detection(t, **kw)
        assert int(exp_st["null_cols_count"].max()) == n_bm
        pd.testing.assert_frame_equal(st.toPandas(), exp_st, check_dtype=False)
        assert odf.count() == exp_odf.num_rows


def test_duplicate_rows_of_2600_columns():
    """Copies of earlier rows, and rows that differ from an earlier row only in the last column, in one column beyond
    2 048, or by a null against a value (all distinct); copies whose only difference is another NaN payload or -0.0
    against 0.0 (duplicates).  row_distinct at hash widths 1-8 sends every row through the comparison."""
    rng = np.random.default_rng(2600)
    n_cols, n_base, n = 2600, 300, 1200
    dts = ("f32", "f64", "i32", "i64")
    nan = {"f32": NAN32, "f64": NAN64}
    vals, valid = [], []
    pick = np.concatenate([np.arange(n_base), rng.integers(0, n_base, n - n_base)])
    for c in range(n_cols):
        dt = dts[c % 4]
        T = _NP[dt]
        cat = np.array([1.5, nan[dt][0], 0.0], T) if dt in nan else np.array([-5, 0, 7], T)
        base = cat[rng.integers(0, 3, n_base)]
        vals.append(base[pick].copy())
        valid.append((rng.random(n_base) >= 0.1)[pick].copy())
    rows = np.arange(n_base, n)
    kinds = rng.integers(0, 5, rows.size)
    distinct, dup = [], []
    for r, kind in zip(rows.tolist(), kinds.tolist()):
        if kind == 0:                                      # the last column only
            c = n_cols - 1
            vals[c][r], valid[c][r] = 10 ** 6 + r, True
            distinct.append(r)
        elif kind == 1:                                    # one column beyond 2 048
            c = int(rng.integers(2049, n_cols - 1))
            vals[c][r], valid[c][r] = (10 ** 6 + r), True
            distinct.append(r)
        elif kind == 2:                                    # null against a value
            c = int(rng.integers(0, n_cols))
            if valid[c][r]:
                valid[c][r] = False
                distinct.append(r)
        elif kind == 3:                                    # another NaN payload, or -0.0 for 0.0: still a duplicate
            c = int(rng.integers(0, n_cols // 4)) * 4 + int(rng.integers(0, 2))   # f32 / f64 columns
            T = _NP[dts[c % 4]]
            v = vals[c][r]
            if valid[c][r] and np.isnan(v):
                vals[c][r] = nan[dts[c % 4]][1 + r % (len(nan[dts[c % 4]]) - 1)]
                dup.append(r)
            elif valid[c][r] and v == 0:
                vals[c][r] = T(-0.0)
                dup.append(r)
        else:
            dup.append(r)
    names = ["d%04d" % c for c in range(n_cols)]
    garbage = [np.where(valid[c], vals[c], _NP[dts[c % 4]](3)) for c in range(n_cols)]   # data under nulls is ignored
    fr = ColumnFrame.from_tensors({names[c]: (torch.from_numpy(garbage[c]).cuda(),
                                              None if valid[c].all() else torch.from_numpy(_pack_validity(valid[c])).cuda())
                                   for c in range(n_cols)})
    t = pa.table([pa.array(vals[c], mask=~valid[c]) for c in range(n_cols)], names=names)
    exp = RC.first_occurrence(t, names)
    assert exp[distinct].all() and not exp[dup].any() and len(distinct) > 100 and len(dup) > 100
    for hb in range(0, 9):
        nd, first = engine.row_distinct(fr, names, hash_bits=hb)
        bits = np.unpackbits(first.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)
        assert nd == int(exp.sum()) and np.array_equal(bits, exp), hb
    odf, st = qc.duplicate_detection(None, fr, treatment=True, print_impact=True)
    exp_odf, exp_st = RC.duplicate_detection(t, treatment=True, print_impact=True)
    assert st.toPandas().values.tolist() == exp_st.values.tolist()
    assert odf.count() == exp_odf.num_rows


# ---- more columns than one launch takes -----------------------------------------------------------------------------

HUGE_COLS, HUGE_ROWS = 70000, 1000


@pytest.fixture(scope="module")
def huge():
    w = WideFrame(HUGE_COLS, HUGE_ROWS, ("f32", "i64"))
    assert w.n_cols > _lib.MAX_LAUNCH_COLS == 65535
    assert len(w.of("f32")) > 1000 and len(w.of("i64")) > 1000   # the bucket count (float32) and the LSD sort (int64)
    return w


def test_engine_entry_points_beyond_65535_columns(huge):
    w = huge
    names = w.names
    js = range(w.n_cols)
    m = engine.moments(w.fr, names)
    for j in js:
        w.pat(j).check_moments(m[j], j, names[j])
    model = _model(w, js)
    h = engine.histogram(w.fr, model)
    m2, h2 = engine.moments_histogram(w.fr, model)
    ids = engine.bin_assign(w.fr, model).cpu().numpy()
    assert h.shape == h2.shape == (w.n_cols, model.max_bins + 1) and ids.shape == (w.n_cols, w.n_rows)
    for j in js:
        P = w.pat(j)
        exp = P.hist(j)
        assert np.array_equal(h[j, :exp.size], exp) and np.array_equal(h2[j, :exp.size], exp), names[j]
        assert np.array_equal(ids[j], P.bins(j)), names[j]
    for j in _sample(w.n_cols):
        w.pat(j).check_moments(m2[j], j, (names[j], "moments_hist"))
    rk = np.array([_ranks(w.pat(j).n_valid(), 20) for j in js])
    sel = engine.select_ranks(w.fr, names, rk)
    part = PartitionedFrame.from_frame(w.fr, 512).select_ranks(names, rk[:, :3])
    for j in js:
        exp = [w.pat(j).rank_value(j, r) if r else np.nan for r in rk[j]]
        assert _same_float(sel[j], exp) and _same_float(part[j], exp[:3]), names[j]
    regs = engine.hll_registers(w.fr, names, 9)
    for j in js:
        assert np.array_equal(regs[j], w.pat(j).registers(j, 9)), names[j]


@pytest.mark.parametrize("algo", ["partition", "lsd"])
def test_mode_distinct_beyond_65535_columns(huge, algo, monkeypatch):
    monkeypatch.setattr(engine, "sort_algorithm", algo)
    js = list(range(huge.n_cols))
    rk = np.array([_ranks(huge.pat(j).n_valid(), 4) for j in js])
    got, qv, regs = engine.sort_mode_distinct(huge.fr, huge.names, rk, hll_p=9)
    _check_mode_distinct(huge, js, got, qv, rk, regs, 9)


def test_code_counts_beyond_65535_columns():
    w = WideFrame(66000, 64, ("str",), cards=(3, 20, 30))
    assert all(len(w.pat(j).dictionary(j)) + 1 <= 40 for j in range(N_PAT))    # one cardinality class: one launch
    got = engine.code_counts(w.fr, w.names)
    assert len(got) == w.n_cols
    for j in range(w.n_cols):
        assert np.array_equal(got[j], w.pat(j).code_counts(j)), w.names[j]


@pytest.mark.parametrize("fn", ["measures_of_counts", "measures_of_percentiles", "mode_computation",
                                "measures_of_cardinality"])
def test_stats_beyond_65535_columns(huge, fn):
    js = _sample(huge.n_cols, 211)
    assert {0, 65534, 65535, 65536, huge.n_cols - 1} <= set(js)
    got = getattr(sg, fn)(None, huge.fr).toPandas()
    assert len(got) == huge.n_cols - (fn == "mode_computation") * sum(huge.pat(j).n_valid() == 0 for j in range(huge.n_cols))
    exp = getattr(O, fn)(huge.table(js))
    got = got.set_index("attribute").loc[exp["attribute"]].reset_index()
    if fn == "measures_of_percentiles":
        # min / max of a column that mixes NaN and numbers skip the NaN, where Spark ranks NaN largest (DESIGN.md
        # section 1, pinned in test_gpu_kernel_edges.py): those two cells are left out here
        mixed = exp["attribute"].isin([huge.names[j] for j in js if huge.pat(j).kind == "nan_payloads"
                                       and huge.pat(j).dt == "f32"]).to_numpy()
        assert mixed.sum() >= 3
        for t in (got, exp):
            t.loc[mixed, ["min", "max"]] = None
    assert_frames_match(got, exp)


def test_duplicate_rows_beyond_65535_columns_are_refused(huge):
    with pytest.raises(NotImplementedError, match="65535"):
        qc.duplicate_detection(None, huge.fr, print_impact=True)
