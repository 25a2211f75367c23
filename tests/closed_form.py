"""Closed-form long columns: columns of billions of rows whose every statistic is known without holding the column.

Row r of a column holds T[(A r + B) mod M] and is null when r mod P is in `nulls`; a few marked rows are overwritten.
M is prime and P = 97 is coprime to it, so by the Chinese remainder theorem the pair (value index, null) of row r depends
on t = r mod M P alone, and the rows of [0, n) with residue t number floor((n - 1 - t) / (M P)) + 1.  Summing those
counts per value index gives the multiset of the column's values (`LongColumn.distribution`): a few tens of thousands of
(value, multiplicity) pairs from which the moments (exactly, as oracle.exact does), extrema, order statistics, mode,
distinct count, histogram and HLL++ registers follow.  Per-row outputs (bin ids, imputed and scaled values, bitmaps) are
a per-value-index table gathered by the same index, which `LongColumn.block` evaluates on the device block by block.

The heavy, zeros and constant columns of the sort tests are not of that form: `runs` describes them directly."""
from fractions import Fraction

import numpy as np

from oracle import exact as X
from oracle import spark_semantics as S

M = 65521                   # the largest prime below 2^16: length of a value table
P = 97                      # null period
A, B = 40503, 12345         # row r -> value index (A r + B) mod M; A is coprime to M
NULLS = (5, 31, 64)         # r mod P in NULLS -> null: 3 rows in 97
BLOCK = 1 << 26             # rows per device block: an int64 row index of one block is 512 MiB


class LongColumn:
    """n rows: T[(A r + B) mod M], null where r mod P is in `nulls`; `marks` {row: value, or None for a null} override."""

    def __init__(self, T, n, nulls=NULLS, marks=None, period=(M, P, A, B)):
        self.M, self.P, self.A, self.B = period
        self.T = np.asarray(T)
        assert self.T.size == self.M
        self.n = int(n)
        self.nulls = tuple(nulls)
        self.marks = {int(r): v for r, v in (marks or {}).items() if int(r) < self.n}
        self.has_bitmap = bool(self.nulls) or any(v is None for v in self.marks.values())

    def index(self, r):
        return (self.A * r + self.B) % self.M

    def pattern_null(self, r):
        return (r % self.P) in self.nulls

    def counts(self):
        """-> (int64 [M]: non-null pattern rows holding T[k], number of null rows), markers included."""
        MP = self.M * self.P
        t = np.arange(MP, dtype=np.int64)
        c = np.where(t < self.n, (self.n - 1 - t) // MP + 1, 0)
        k = self.index(t % self.M)
        null = np.isin(t % self.P, self.nulls)
        w = np.bincount(k[~null], weights=c[~null], minlength=self.M).astype(np.int64)   # float64 sums: exact below 2^53
        n_null = int(c[null].sum())
        for r, v in self.marks.items():
            if self.pattern_null(r):
                n_null -= 1
            else:
                w[self.index(r)] -= 1
            n_null += v is None
        return w, n_null

    def distribution(self):
        """-> (values, multiplicities, number of nulls): the non-null values of the column as a multiset."""
        w, n_null = self.counts()
        mv = [v for v in self.marks.values() if v is not None]
        vals = np.concatenate([self.T, np.array(mv, self.T.dtype)])
        ws = np.concatenate([w, np.ones(len(mv), np.int64)])
        keep = ws > 0
        return vals[keep], ws[keep], n_null

    def expand(self):
        """The whole column on the host (values, valid) - small n only: the brute-force twin the CPU tests compare with."""
        r = np.arange(self.n, dtype=np.int64)
        vals = self.T[self.index(r)].copy()
        valid = ~np.isin(r % self.P, self.nulls)
        for row, v in self.marks.items():
            valid[row] = v is not None
            if v is not None:
                vals[row] = v
        return vals, valid

    def block(self, torch, r0, r1, table, null_value, marks):
        """Rows [r0, r1) of a per-row output on the device: table[index(r)] (a CUDA tensor of M entries), null_value on
        pattern-null rows, and marks {row: value} on the marked rows."""
        r = torch.arange(r0, r1, device=table.device, dtype=torch.int64)
        out = table[(r * self.A + self.B) % self.M]
        if self.nulls:
            nl = torch.isin(r % self.P, torch.tensor(self.nulls, device=table.device))
            out = torch.where(nl, torch.full((), null_value, dtype=out.dtype, device=out.device), out)
        for row, v in marks.items():
            if r0 <= row < r1:
                out[row - r0] = v
        return out


# ---- value tables and marked rows -------------------------------------------------------------------------------

NAN32 = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFA00001, 0x7FC00123], np.uint32).view(np.float32)
F32_MAX = float(np.finfo(np.float32).max)
MARK_F32 = {"lo": -3.0e30, "hi": 3.0e30, "hi2": 2.5e30, "tail": 1234.5625}     # exact in float32; outside the tables
MARK_NAN32 = float(np.array([0xFF800123], np.uint32).view(np.float32)[0])     # sign set, signalling: no table holds it
MARK_I32 = {"lo": -2147480000, "hi": 2147480000, "hi2": 2147470000, "tail": 777777777}
MARK_I32_NARROW = {"lo": -8100, "hi": 8100, "hi2": 8090, "tail": 8050}   # keeps the narrow column under 2^14 values
NAN64 = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF4000000000001],
                 np.uint64).view(np.float64)
F64_MAX = float(np.finfo(np.float64).max)
MARK_NAN64 = float(np.array([0xFFF0000000000123], np.uint64).view(np.float64)[0])   # sign set, signalling
MARK_I64 = {"lo": -(1 << 62) - 7, "hi": (1 << 62) + 9, "hi2": (1 << 62) + 5, "tail": (1 << 53) + 1000001}


def _without(T, marks):
    """T with every entry equal to a mark moved off it (so the marks stay unique values)."""
    for v in marks:
        T[T == v] = T[T == v] + 1
    return T


def table_f32_special(seed, m=M):
    """Quarter steps of a normal spread (repeated values, so the mode has a margin) with -0.0 / +0.0, NaN payloads
    (sign set, signalling), subnormals and +-FLT_MAX / +-inf at the front."""
    rng = np.random.default_rng(seed)
    T = _without((np.round(rng.normal(0.0, 400.0, m)) / 4).astype(np.float32), MARK_F32.values())
    sp = np.concatenate([np.array([-0.0, 0.0, 1e-45, -1e-45, 1e-40, F32_MAX, -F32_MAX, np.inf, -np.inf], np.float32), NAN32])
    T[:sp.size] = sp
    return T


def table_f32_finite(seed, m=M):
    """Finite, nonzero eighths of a normal spread and one subnormal: moments, scaling, and n_nonzero = n_valid."""
    rng = np.random.default_rng(seed)
    T = (np.round(rng.normal(5.0, 100.0, m) * 8) / 8).astype(np.float32)
    T[T == 0] = 0.125
    T[0] = 1e-45
    return _without(T, MARK_F32.values())


def table_f64_special(seed, m=M):
    """table_f32_special in double: -0.0 / +0.0, NaN payloads, subnormals and +-DBL_MAX / +-inf at the front."""
    rng = np.random.default_rng(seed)
    T = _without(np.round(rng.normal(0.0, 400.0, m)) / 4, MARK_F32.values())
    sp = np.concatenate([np.array([-0.0, 0.0, 5e-324, -5e-324, 1e-310, F64_MAX, -F64_MAX, np.inf, -np.inf]), NAN64])
    T[:sp.size] = sp
    return T


def table_i64(seed, m=M):
    """int64 around 2^53 (where a double no longer holds every integer), near 2^62 and at the type's extremes."""
    rng = np.random.default_rng(seed)
    T = (1 << 53) + rng.integers(-40000, 40000, m)
    far = rng.random(m) < 0.1
    T[far] = (1 << 62) + rng.integers(-1000, 1000, int(far.sum()))
    T[:4] = (-(1 << 63), (1 << 63) - 1, -(1 << 53) - 1, 0)
    return _without(T.astype(np.int64), MARK_I64.values())


def table_i32(seed, m=M, narrow=False):
    """int32 over the whole range with INT_MIN / INT_MAX at the front, or (narrow) fewer than 2^14 distinct values."""
    rng = np.random.default_rng(seed)
    if narrow:
        return rng.integers(-8000, 8000, m).astype(np.int32)
    T = rng.integers(-(1 << 31), 1 << 31, m).astype(np.int64)
    T[:5] = (-(1 << 31), (1 << 31) - 1, -(1 << 31) + 1, 0, -1)
    return _without(T, MARK_I32.values()).astype(np.int32)


def marks(kind, n, at=(1 << 31, 1 << 32), run=68, values=None):
    """Marked rows of a column of n rows: at[0] - 1 holds a unique low value, at[0] a unique high one, at[0] + 1 a
    unique NaN payload (float) or a null (int), then `run` nulls cover the bitmap word of row at[0] and the next one;
    n - 1 holds a unique tail value.  Past at[1]: at[1] - 1 another unique value, at[1] a null."""
    mk = values or {"f32": MARK_F32, "f64": MARK_F32, "i32": MARK_I32, "i64": MARK_I64}[kind]
    a, b = at
    out = {a - 1: mk["lo"], a: mk["hi"], a + 1: {"f32": MARK_NAN32, "f64": MARK_NAN64}.get(kind)}
    out.update({r: None for r in range(a + 2, a + 2 + run)})
    if n > b:
        out.update({b - 1: mk["hi2"], b: None})
    out[n - 1] = mk["tail"]
    return {r: v for r, v in out.items() if r < n}


def runs(values, counts):
    """(values, multiplicities, 0): the distribution of a column without nulls given as its distinct values."""
    return np.asarray(values), np.asarray(counts, np.int64), 0


# ---- references of a distribution (values, multiplicities, n_null) --------------------------------------------------

def canonical(vals, ws):
    """-> (sorted distinct values, multiplicities): -0.0 counts as 0.0 and every NaN as one NaN, sorted last, as the
    exact mode / distinct count group them.  Integer columns stay integers (int64 beyond 2^53 stays exact)."""
    vals = np.asarray(vals)
    if vals.dtype.kind == "f":
        with np.errstate(invalid="ignore"):
            x = vals.astype(np.float64) + 0.0
        x[np.isnan(x)] = np.nan
    else:
        x = vals.astype(np.int64)
    u, inv = np.unique(x, return_inverse=True)
    cnt = np.zeros(u.size, np.int64)
    np.add.at(cnt, inv.reshape(-1), np.asarray(ws, np.int64))
    return u, cnt


def exact_central_weighted(vals, ws):
    """oracle.exact.exact_central of the multiset: (n, mean, M2, M3, M4) as Fractions from weighted exact power sums."""
    N, E = X._scaled_ints(np.asarray(vals))
    s = [0, 0, 0, 0, 0]
    for v, w in zip(N, np.asarray(ws, np.int64).tolist()):
        p = w
        for k in range(5):
            s[k] += p
            p *= v
    n, s1, s2, s3, s4 = s
    if n == 0:
        return 0, None, Fraction(0), Fraction(0), Fraction(0)
    a = Fraction(s1, n)
    m2 = s2 - a * s1
    m3 = s3 - 3 * a * s2 + 2 * a * a * s1
    m4 = s4 - 4 * a * s3 + 6 * a * a * s2 - 3 * a * a * a * s1
    sc = Fraction(2) ** E
    return n, a * sc, m2 * sc ** 2, m3 * sc ** 3, m4 * sc ** 4


def moments_ref(vals, ws):
    """-> dict n_valid, n_nonzero, min, max (NaN-free extrema; NaN when only NaN or nothing), finite, and the rounded
    exact mean / M2..M4 of finite columns."""
    vals, ws = np.asarray(vals), np.asarray(ws, np.int64)
    isf = vals.dtype.kind == "f"
    nn = ~np.isnan(vals) if isf else np.ones(vals.size, bool)
    out = {"n_valid": int(ws.sum()), "n_nonzero": int(ws[vals != 0].sum()),
           "min": float(vals[nn].min()) if nn.any() else float("nan"),
           "max": float(vals[nn].max()) if nn.any() else float("nan"),
           "finite": not isf or bool(np.isfinite(vals).all())}
    if out["finite"]:
        n, mean, m2, m3, m4 = exact_central_weighted(vals, ws)
        out.update(mean=float(mean) if n else float("nan"), m2=float(m2), m3=float(m3), m4=float(m4))
    return out


def check_moments(rec, ref, name):
    """One moments record against moments_ref, on the contract of test_gpu_kernel_edges._check_moments: counts and
    extrema exact, mean to 1e-9, M2..M4 to 1e-6 + 1e-9 n sd^k; a NaN / inf value makes every moment non-finite."""
    n = ref["n_valid"]
    assert rec["n_valid"] == n and rec["n_nonzero"] == ref["n_nonzero"], (name, rec, ref)
    for f in ("min", "max"):
        assert rec[f] == ref[f] or (ref[f] != ref[f] and rec[f] != rec[f]), (name, f, rec[f], ref[f])
    if not ref["finite"]:
        for f in ("mean", "m2", "m3", "m4"):
            assert not np.isfinite(rec[f]), (name, f, rec[f])
        return
    mean, m2 = ref["mean"], ref["m2"]
    sd = (m2 / n) ** 0.5
    assert abs(rec["mean"] - mean) <= 1e-9 * max(abs(mean), sd) + n * 2.0 ** -1074, (name, rec["mean"], mean)
    for k, f in enumerate(("m2", "m3", "m4")):
        assert abs(rec[f] - ref[f]) <= 1e-6 * abs(ref[f]) + 1e-9 * n * sd ** (k + 2), (name, f, rec[f], ref[f])


def mode_ref(vals, ws, as_int=False):
    """-> (mode, mode_rows, n_distinct) with ties to the smallest value; (None, None, 0) when empty."""
    u, cnt = canonical(vals, ws)
    if u.size == 0:
        return None, None, 0
    i = int(np.argmax(cnt))                  # the first maximum: the smallest value (NaN sorts last)
    return (int(u[i]) if as_int else float(u[i])), int(cnt[i]), int(u.size)


def rank_values(vals, ws, ranks):
    """Order statistics at 1-based ranks among the non-null values (NaN last), as float64; rank 0 -> NaN."""
    u, cnt = canonical(vals, ws)
    cum = np.cumsum(cnt)
    out = []
    for r in np.asarray(ranks, np.int64).tolist():
        out.append(float("nan") if r == 0 else float(u[int(np.searchsorted(cum, r, side="left"))]))
    return np.array(out, np.float64)


def bin_table(T, cuts):
    """bin id of every table entry (oracle.exact.exact_bins): 1 + #(c < v), NaN -> len(cuts) + 1."""
    return X.exact_bins(np.asarray(T), np.ones(len(T), bool), cuts)


def histogram_ref(vals, ws, n_null, cuts):
    """uint64 [len(cuts) + 2]: slot 0 = nulls, slot b = rows in bin b."""
    ids = bin_table(vals, cuts)
    h = np.zeros(len(cuts) + 2, np.int64)
    np.add.at(h, ids, np.asarray(ws, np.int64))
    h[0] = n_null
    return h.astype(np.uint64)


def registers_ref(vals, sdtype, p):
    """HLL++ registers of the distinct values (a maximum over the values: multiplicities do not matter)."""
    return S.hll_registers(S.hll_hashes(np.asarray(vals), sdtype), p)
