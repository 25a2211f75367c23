"""Behavioural restatement of the Apache Spark primitives the Anovos hot path
bottoms out in.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Third-party dependency restated here: Apache Spark SQL / MLlib (un-vendored;
the reference supports 2.4.8, 3.1.3, 3.2.2 - .github/workflows/unit.yml:19-40).
Reference call sites (relative to /root/reference/src/main/anovos):
  data_analyzer/stats_generator.py:163,241,310,488,607,611,813,908,993
  data_transformer/transformers.py:215,219,248-271
  drift_stability/drift_detector.py:253-334
Pins: src/test/anovos/data_analyzer/{test_stats_generator,test_quality_checker,test_association_evaluator}.py,
src/test/anovos/drift_stability/{test_drift_detector,test_stability}.py and the stored outputs of
examples/notebooks/{data_analyzer__stats_generator,data_analyzer__quality_checker,data_analyzer__association_evaluator,
data_transformer__transformers,drift_stability}.ipynb.
"""
from __future__ import annotations

import decimal
import math

import numpy as np
import pyarrow as pa

# ----------------------------------------------------------------------------
# dtype mapping (shared/utils.py:64-72 works on Spark dtype strings)
# ----------------------------------------------------------------------------


def spark_dtype(t: pa.DataType) -> str:
    """Arrow type -> the Spark SQL dtype string `idf.dtypes` would show."""
    if pa.types.is_dictionary(t):
        return spark_dtype(t.value_type)
    if pa.types.is_string(t) or pa.types.is_large_string(t):
        return "string"
    if pa.types.is_int32(t):
        return "int"
    if pa.types.is_int64(t) or pa.types.is_uint32(t):
        return "bigint"
    if pa.types.is_float32(t):
        return "float"
    if pa.types.is_float64(t):
        return "double"
    if pa.types.is_decimal(t):
        return "decimal(%d,%d)" % (t.precision, t.scale)
    if pa.types.is_int16(t) or pa.types.is_uint8(t):
        return "smallint"
    if pa.types.is_int8(t):
        return "tinyint"
    if pa.types.is_boolean(t):
        return "boolean"
    if pa.types.is_date(t):
        return "date"
    if pa.types.is_timestamp(t):
        return "timestamp"
    if pa.types.is_null(t):
        return "void"
    return str(t)


def segregate(table: pa.Table):
    """attributeType_segregation (shared/utils.py:48-73)."""
    num, cat, other = [], [], []
    for f in table.schema:
        d = spark_dtype(f.type)
        if d == "string":
            cat.append(f.name)
        elif d in ("double", "int", "bigint", "float", "long") or d.startswith("decimal"):
            num.append(f.name)
        else:
            other.append(f.name)
    return num, cat, other


def column_values(table: pa.Table, name: str):
    """-> (values ndarray [native dtype or object for strings], valid bool ndarray)."""
    col = table.column(name)
    if isinstance(col, pa.ChunkedArray):
        col = col.combine_chunks() if col.num_chunks != 1 else col.chunk(0)
    t = col.type
    if pa.types.is_dictionary(t):
        col = col.dictionary_decode()
        t = col.type
    n = len(col)
    valid = np.ones(n, dtype=bool) if col.null_count == 0 else ~np.asarray(col.is_null())
    if pa.types.is_string(t) or pa.types.is_large_string(t):
        vals = np.asarray(col.to_pylist(), dtype=object)
        return vals, valid
    if pa.types.is_decimal(t):
        vals = np.array([float(v) if v is not None else 0.0 for v in col.to_pylist()], dtype=np.float64)
        return vals, valid
    if pa.types.is_null(t):
        return np.zeros(n, dtype=np.float64), np.zeros(n, dtype=bool)
    filled = col.fill_null(0) if col.null_count else col
    vals = filled.to_numpy(zero_copy_only=False)
    return vals, valid


# ----------------------------------------------------------------------------
# rounding / string forms
# ----------------------------------------------------------------------------

_Q = {}


def round_half_up(x, scale: int = 4):
    """Spark `round(double, scale)`: BigDecimal(Double.toString(d)).setScale(scale, HALF_UP)
    (catalyst Round; used at stats_generator.py:169,243,313,319,499,506,521,728,818-822,
    912,1005-1006).  None -> None, NaN/inf pass through.  Parity unpinned vs HALF_EVEN:
    no reference vector separates the two modes (SURVEY 8a item 6)."""
    if x is None:
        return None
    x = float(x)
    if math.isnan(x) or math.isinf(x):
        return x
    q = _Q.get(scale)
    if q is None:
        q = _Q[scale] = decimal.Decimal(1).scaleb(-scale)
    # BigDecimal has no digit limit: the context must hold all ~309 integer digits of a double and the scale
    return float(decimal.Decimal(repr(x)).quantize(q, rounding=decimal.ROUND_HALF_UP, context=_WIDE))


_WIDE = decimal.Context(prec=340)


def java_double_to_string(x: float) -> str:
    """java.lang.Double.toString: plain decimal for 1e-3 <= |x| < 1e7, else
    computerised scientific notation `d.dddE[-]n` (SURVEY 8a item 6b; pinned only for
    the plain range by notebook cell 'measures_of_centralTendency': "5.093362141")."""
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "Infinity" if x > 0 else "-Infinity"
    if x == 0:
        return "-0.0" if math.copysign(1.0, x) < 0 else "0.0"
    r = repr(float(x))
    sign = ""
    if r[0] == "-":
        sign, r = "-", r[1:]
    # decompose the shortest repr into digits and a decimal exponent
    if "e" in r or "E" in r:
        mant, exp = r.lower().split("e")
        exp = int(exp)
    else:
        mant, exp = r, 0
    if "." in mant:
        ip, fp = mant.split(".")
    else:
        ip, fp = mant, ""
    digits = (ip + fp).lstrip("0")
    # position of the decimal point relative to the first significant digit
    lead = len(ip.lstrip("0")) if ip.strip("0") else -(len(fp) - len(fp.lstrip("0")))
    point = lead + exp  # value = 0.digits * 10**point
    digits = digits.rstrip("0") or "0"
    a = abs(x)
    if 1e-3 <= a < 1e7:
        if point <= 0:
            s = "0." + "0" * (-point) + digits
        elif point >= len(digits):
            s = digits + "0" * (point - len(digits)) + ".0"
        else:
            s = digits[:point] + "." + digits[point:]
        return sign + s
    e = point - 1
    m = digits[0] + "." + (digits[1:] or "0")
    return "%s%sE%d" % (sign, m, e)


def mode_to_string(value, sdtype: str) -> str:
    """mode is cast to StringType via the JVM's toString of the unpickled Python
    value (stats_generator.py:405-411; pin test_stats_generator.py:225-229 -> "42")."""
    if sdtype == "string":
        return str(value)
    if sdtype in ("int", "bigint", "long"):
        return str(int(value))
    return java_double_to_string(float(value))


def float32_via_string(v) -> float:
    """`summary()` renders min/max/percentiles of a FloatType column with
    Float.toString and Anovos casts the string back to double (stats_generator.py:
    818-822, 910-912).  Parity unpinned: no golden vector has a float32 column."""
    return float(str(np.float32(v)))


# ----------------------------------------------------------------------------
# moments (SURVEY Appendix B.1; pins test_stats_generator.py:292-339,451-504,570-605)
# ----------------------------------------------------------------------------


def central_moments(x64: np.ndarray):
    """x64: float64 non-null values. -> n, mean, M2, M3, M4 with M_k = sum (x-mean)^k.
    Two-pass, pairwise summation: the accuracy reference for the GPU kernels."""
    n = int(x64.size)
    if n == 0:
        return 0, None, 0.0, 0.0, 0.0
    mean = float(np.sum(x64) / n)
    d = x64 - mean
    # second-order mean correction keeps the two-pass result exact to ~1ulp
    corr = float(np.sum(d) / n)
    mean = mean + corr
    d = d - corr
    d2 = d * d
    return n, mean, float(np.sum(d2)), float(np.sum(d2 * d)), float(np.sum(d2 * d2))


def stddev_samp(n, m2):
    """sqrt(M2/(n-1)); n<=1 -> null (Spark >= 3.1 default; parity unpinned)."""
    if n is None or n <= 1:
        return None
    return math.sqrt(m2 / (n - 1))


def skewness(n, m2, m3):
    """sqrt(n)*M3/M2^1.5 (population); M2 == 0 -> null (Spark >= 3.1; unpinned)."""
    if not n or m2 == 0:
        return None
    return math.sqrt(n) * m3 / math.sqrt(m2 * m2 * m2)


def kurtosis(n, m2, m4):
    """n*M4/M2^2 - 3 (population, excess); M2 == 0 -> null."""
    if not n or m2 == 0:
        return None
    return n * m4 / (m2 * m2) - 3.0


# ----------------------------------------------------------------------------
# quantiles (Appendix B.2; pins test_stats_generator.py:328-333,493-498, drift
# equal_frequency vector, 81 notebook percentiles)
# ----------------------------------------------------------------------------


def quantile_rank(p: float, n: int) -> int:
    """1-based rank max(1, ceil(p*n)); p*n evaluated in float64 as written."""
    return max(1, int(math.ceil(p * n)))


def quantile_sorted(sorted_vals: np.ndarray, p: float):
    n = int(sorted_vals.size)
    if n == 0:
        return None
    return sorted_vals[quantile_rank(p, n) - 1]


# ---------------------------------------------------------------------------
# Spark's Greenwald-Khanna sketch (org.apache.spark.sql.catalyst.util.QuantileSummaries, Spark >= 3.1;
# un-vendored third-party code: restated from its published algorithm) as it behaves for ONE partition of
# fewer than 50 000 non-null values - the situation of every unit test of the reference.  All values then sit
# in the head buffer (defaultHeadSize = 50 000) until the final compress(): they are sorted and inserted in one
# batch with g = 1 and delta_k = floor(2*eps*k) (0 for the first and the last), compressed once from the tail with
# mergeThreshold = 2*eps*n, and queried with targetError = max(g + delta) / 2.  The surviving sample POSITIONS
# and the queried position depend on (n, eps, p) only - never on the values - so approxQuantile / summary()
# percentiles reduce to "the order statistic at a shifted rank".  Pinned by the 13 outlier counts / clamp values
# of test_quality_checker.py:526-637 (eps = 0.01), which the exact rank ceil(p*n) does NOT reproduce.
# Larger or multi-partition inputs make Spark's answer depend on arrival order and partitioning (any element
# within eps*n ranks): there the exact rank is used.
# ---------------------------------------------------------------------------

GK_HEAD_SIZE = 50000


def gk_single_batch_summary(n: int, eps: float):
    """-> list of (position in the sorted values [0-based], g, delta) after withHeadBufferInserted + compress."""
    if n <= 0:
        return []
    delta = [0] * n
    for k in range(1, n - 1):                    # currentCount after the increment = k + 1
        delta[k] = int(math.floor(2 * eps * (k + 1)))
    thr = 2 * eps * n                            # mergeThreshold of compressImmut
    res = []
    head = [n - 1, 1, delta[n - 1]]              # the last element is always kept
    for i in range(n - 2, 0, -1):                # the first element is never compressed
        if 1 + head[1] + head[2] < thr:          # sample1.g + head.g + head.delta < mergeThreshold
            head[1] += 1
        else:
            res.append(tuple(head))
            head = [i, 1, delta[i]]
    res.append(tuple(head))
    if n > 1:
        res.append((0, 1, 0))                    # "if necessary, add the minimum element"
    res.reverse()
    return res


def gk_query_position(summary, n: int, eps: float, p: float) -> int:
    """QuantileSummaries.query -> 0-based position in the sorted values."""
    if p <= eps:
        return summary[0][0]
    if p >= 1 - eps:
        return summary[-1][0]
    target_error = max(g + d for _, g, d in summary) / 2.0
    rank = int(math.ceil(p * n))
    min_rank = summary[0][1]
    i = 0
    while i < len(summary) - 1:
        pos, g, d = summary[i]
        max_rank = min_rank + d
        if max_rank - target_error <= rank <= min_rank + target_error:
            return pos
        i += 1
        min_rank += summary[i][1]
    return summary[-1][0]


# --- the full sketch (arrival order, several partitions): what Dataset.summary() / approxQuantile return in general.
# Pinned by the 81 stored summary() percentiles of the reference notebook on the income CSV, which Spark read as TWO
# partitions (Hadoop split of the 5.9 MB file at 4 MiB = spark.sql.files.openCostInBytes): tests/test_oracle_golden.py.

GK_COMPRESS_THRESHOLD = 10000


def gk_compress(samples, merge_threshold):
    """QuantileSummaries.compressImmut on a list of (value, g, delta)."""
    if not samples:
        return []
    res = []
    head = list(samples[-1])
    for i in range(len(samples) - 2, 0, -1):
        v, g, d = samples[i]
        if g + head[1] + head[2] < merge_threshold:
            head[1] += g
        else:
            res.append(tuple(head))
            head = [v, g, d]
    res.append(tuple(head))
    if samples[0][0] <= head[0] and len(samples) > 1:
        res.append(tuple(samples[0]))
    res.reverse()
    return res


def gk_insert_batch(samples, count, batch_sorted, eps):
    """withHeadBufferInserted: merge one sorted head buffer into the sample list -> (samples, count)."""
    out, si, cur = [], 0, count
    m = len(batch_sorted)
    for oi, x in enumerate(batch_sorted):
        while si < len(samples) and samples[si][0] <= x:
            out.append(samples[si])
            si += 1
        cur += 1
        first_or_last = (not out) or (si == len(samples) and oi == m - 1)
        out.append((float(x), 1, 0 if first_or_last else int(math.floor(2 * eps * cur))))
    out.extend(samples[si:])
    return out, cur


def gk_sketch(values, eps):
    """One partition: values in ARRIVAL order -> (compressed samples, count), flushing the head buffer every 50 000
    insertions (and compressing when >= 10 000 samples are held) exactly like QuantileSummaries.insert, then the
    final compress()."""
    samples, count = [], 0
    vals = np.asarray(values, dtype=np.float64)
    for b0 in range(0, len(vals), GK_HEAD_SIZE):
        batch = np.sort(vals[b0:b0 + GK_HEAD_SIZE], kind="stable")
        full = len(batch) == GK_HEAD_SIZE
        samples, count = gk_insert_batch(samples, count, batch.tolist(), eps)
        if full and len(samples) >= GK_COMPRESS_THRESHOLD:
            samples = gk_compress(samples, 2 * eps * count)
    return gk_compress(samples, 2 * eps * count), count


def gk_merge(a, na, b, nb, eps):
    """QuantileSummaries.merge (Spark >= 3.0: deltas of interleaved samples grow by the other side's 2*eps*count)."""
    if nb == 0:
        return list(a), na
    if na == 0:
        return list(b), nb
    add_self, add_other = int(math.floor(2 * eps * nb)), int(math.floor(2 * eps * na))
    out, i, j = [], 0, 0
    while i < len(a) and j < len(b):
        if a[i][0] < b[j][0]:
            s, ad = a[i], (add_self if j > 0 else 0)
            i += 1
        else:
            s, ad = b[j], (add_other if i > 0 else 0)
            j += 1
        out.append((s[0], s[1], s[2] + ad))
    out.extend(a[i:])
    out.extend(b[j:])
    return gk_compress(out, 2 * eps * (na + nb)), na + nb


def gk_query_value(samples, n, eps, p):
    if not samples:
        return None
    if p <= eps:
        return samples[0][0]
    if p >= 1 - eps:
        return samples[-1][0]
    target_error = max(g + d for _, g, d in samples) / 2.0
    rank = int(math.ceil(p * n))
    min_rank, i = samples[0][1], 0
    while i < len(samples) - 1:
        if min_rank + samples[i][2] - target_error <= rank <= min_rank + target_error:
            return samples[i][0]
        i += 1
        min_rank += samples[i][1]
    return samples[-1][0]


def gk_partitioned_quantiles(partitions, probs, eps):
    """partitions: list of value arrays (non-null, arrival order), merged in partition order -> list of quantiles."""
    samples, n = [], 0
    for part in partitions:
        s, c = gk_sketch(part, eps)
        samples, n = gk_merge(samples, n, s, c, eps)
    return [gk_query_value(samples, n, eps, p) for p in probs]


def approx_quantile_rank(p: float, n: int, eps) -> int:
    """1-based rank Spark returns for quantile p of n non-null values of one partition: the sketch position
    when the single-batch model applies (eps given, n < 50 000), else the exact rank max(1, ceil(p*n))."""
    if eps is None or n >= GK_HEAD_SIZE or n <= 0:
        return quantile_rank(p, n)
    return gk_query_position(gk_single_batch_summary(n, eps), n, eps, p) + 1


def approx_quantile_sorted(sorted_vals: np.ndarray, p: float, eps):
    n = int(sorted_vals.size)
    if n == 0:
        return None
    return sorted_vals[approx_quantile_rank(p, n, eps) - 1]


SUMMARY_EPS = 1e-4       # Dataset.summary(): ApproximatePercentile accuracy 10000
APPROX_QUANTILE_EPS = 0.01   # every approxQuantile(..., 0.01) call of the reference

SUMMARY_PCTS = {"1%": 0.01, "5%": 0.05, "10%": 0.1, "25%": 0.25, "50%": 0.5,
                "75%": 0.75, "90%": 0.9, "95%": 0.95, "99%": 0.99}


def spark_sort_key(x: np.ndarray) -> np.ndarray:
    """Spark orders NaN above +inf (parity unpinned).  np.sort already does."""
    return np.sort(x, kind="stable")


# ----------------------------------------------------------------------------
# binning (Appendix B.3; transformers.py:210-232,248-271)
# ----------------------------------------------------------------------------


def equal_range_cutoffs(mn: float, mx: float, bin_size: int):
    """transformers.py:229-231 in Python float64, same operation order."""
    mn, mx = float(mn), float(mx)
    w = (mx - mn) / bin_size
    return [mn + j * w for j in range(1, bin_size)]


def equal_frequency_cutoffs(sorted_x64: np.ndarray, bin_size: int):
    """transformers.py:210-215: approxQuantile(cols, [j*(1/bin_size)], 0.01): the GK sketch position for one
    partition of < 50 000 values, the exact rank ceil(p*n) element otherwise (inside Spark's own error band)."""
    w = 1 / bin_size
    n = int(sorted_x64.size)
    if n >= GK_HEAD_SIZE:
        return [float(quantile_sorted(sorted_x64, j * w)) for j in range(1, bin_size)]
    sm = gk_single_batch_summary(n, APPROX_QUANTILE_EPS)
    return [float(sorted_x64[gk_query_position(sm, n, APPROX_QUANTILE_EPS, j * w)]) for j in range(1, bin_size)]


def assign_bins(x: np.ndarray, valid: np.ndarray, cutoffs, bin_size: int) -> np.ndarray:
    """bucket_label (transformers.py:248-271), bin_dtype="numerical":
    null -> 0 here (None in the reference); first i with v <= cut[i] -> i+1; else
    len(cutoffs)+1.  == 1 + #(cutoffs strictly below v); NaN lands in the last bin.
    x holds the column's own values: an integer column compares exactly, as Python compares an int with a
    float (c < v <=> floor(c) < v), where float64(v) would round above 2^53."""
    x = np.asarray(x)
    if x.dtype.kind in "iu":
        info = np.iinfo(np.int64)
        below, th = 0, []                            # cutoffs below every int64, int64 floors of the others
        for c in map(float, cutoffs):
            if c == -math.inf:
                below += 1
            elif math.isfinite(c):
                t = math.floor(c)
                if t < info.min:
                    below += 1
                elif t < info.max:                   # floor(c) >= INT64_MAX is below no int64
                    th.append(t)
        th = np.sort(np.array(th, dtype=np.int64))
        idx = (np.searchsorted(th, x.astype(np.int64), side="left") + 1 + below).astype(np.int32)
    else:
        x64 = x.astype(np.float64)
        cut = np.asarray(cutoffs, dtype=np.float64)
        idx = np.searchsorted(cut, x64, side="left").astype(np.int32) + 1
        idx[np.isnan(x64)] = len(cut) + 1
    idx[~valid] = 0
    return idx


# ----------------------------------------------------------------------------
# drift (Appendix B.4; drift_detector.py:243-356)
# ----------------------------------------------------------------------------


def drift_from_groups(src_groups, tgt_groups, n_src: int, n_tgt: int, ordered_keys, null_rows: int = 0):
    """src_groups / tgt_groups: dict key -> count of NON-NULL rows in the group
    (the null group is present with count 0 when the column has nulls).
    ordered_keys: every key present on either side, in `orderBy(i)` order.
    null_rows: string columns keep their null group key as SQL NULL, which never
    matches in the full-outer join (:266): each side's null group becomes its own row
    (p or q = 0 -> 1e-4, other side missing -> 1e-4), sorted first (NULLS FIRST).
    Returns PSI, HD, JSD, KS (no rounding)."""
    psi = hd = pm = qm = 0.0
    cp = cq = 0.0
    ks = 0.0
    any_row = null_rows > 0
    for _ in range(null_rows):
        p = q = 0.0001
        psi += (p - q) * math.log(p / q)
        hd += (math.sqrt(p) - math.sqrt(q)) ** 2
        m = (p + q) / 2
        pm += p * math.log(p / m)
        qm += q * math.log(q / m)
        cp += p
        cq += q
        ks = max(ks, abs(cp - cq))
    for k in ordered_keys:
        ps = src_groups.get(k)
        qs = tgt_groups.get(k)
        if ps is None and qs is None:
            continue
        p = 0.0001 if ps is None else ps / n_src       # :253-254, fillna :268
        q = 0.0001 if qs is None else qs / n_tgt       # :264
        if p == 0:
            p = 0.0001                                  # .replace(0, 0.0001) :269
        if q == 0:
            q = 0.0001
        any_row = True
        psi += (p - q) * math.log(p / q)               # :274-282
        hd += (math.sqrt(p) - math.sqrt(q)) ** 2       # :286-294
        m = (p + q) / 2                                # :298-309
        pm += p * math.log(p / m)
        qm += q * math.log(q / m)
        cp += p                                        # :313-334
        cq += q
        ks = max(ks, abs(cp - cq))
    if not any_row:
        return None, None, None, None
    return psi, math.sqrt(hd / 2), (pm + qm) / 2, ks


# ----------------------------------------------------------------------------
# HyperLogLog++ as used by approx_count_distinct (Appendix B.5; pins notebook
# cells measures_of_cardinality rsd 0.05 / 0.02)
# ----------------------------------------------------------------------------

_M64 = (1 << 64) - 1
P1, P2, P3, P4, P5 = (0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9,
                      0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5)
HLL_SEED = 42
HLL_THRESHOLDS = {4: 10, 5: 20, 6: 40, 7: 80, 8: 220, 9: 400, 10: 900, 11: 1800, 12: 3100,
                  13: 6500, 14: 11500, 15: 20000, 16: 50000, 17: 120000, 18: 350000}


def _rotl_np(x, r):
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def _fmix_np(h):
    h = h ^ (h >> np.uint64(33))
    h = h * np.uint64(P2)
    h = h ^ (h >> np.uint64(29))
    h = h * np.uint64(P3)
    h = h ^ (h >> np.uint64(32))
    return h


def xxh64_int_np(i32: np.ndarray, seed: int = HLL_SEED) -> np.ndarray:
    """XXH64.hashInt over an int32 array (vectorised)."""
    with np.errstate(over="ignore"):
        h = np.uint64((seed + P5 + 4) & _M64)
        v = i32.astype(np.int64).astype(np.uint64) & np.uint64(0xFFFFFFFF)
        h = h ^ (v * np.uint64(P1))
        h = _rotl_np(h, 23) * np.uint64(P2) + np.uint64(P3)
        return _fmix_np(h)


def xxh64_long_np(i64: np.ndarray, seed: int = HLL_SEED) -> np.ndarray:
    """XXH64.hashLong over an int64/uint64 array (vectorised)."""
    with np.errstate(over="ignore"):
        h = np.uint64((seed + P5 + 8) & _M64)
        l = i64.view(np.uint64) if i64.dtype != np.uint64 else i64
        h = h ^ (_rotl_np(l * np.uint64(P2), 31) * np.uint64(P1))
        h = _rotl_np(h, 27) * np.uint64(P1) + np.uint64(P4)
        return _fmix_np(h)


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M64


def xxh64_bytes(b: bytes, seed: int = HLL_SEED) -> int:
    """Standard XXH64 over a byte string (Spark hashUnsafeBytes for UTF8String)."""
    n = len(b)
    off = 0
    if n >= 32:
        v1 = (seed + P1 + P2) & _M64
        v2 = (seed + P2) & _M64
        v3 = seed & _M64
        v4 = (seed - P1) & _M64
        while off + 32 <= n:
            for k in range(4):
                w = int.from_bytes(b[off + 8 * k: off + 8 * k + 8], "little")
                if k == 0:
                    v1 = (_rotl((v1 + w * P2) & _M64, 31) * P1) & _M64
                elif k == 1:
                    v2 = (_rotl((v2 + w * P2) & _M64, 31) * P1) & _M64
                elif k == 2:
                    v3 = (_rotl((v3 + w * P2) & _M64, 31) * P1) & _M64
                else:
                    v4 = (_rotl((v4 + w * P2) & _M64, 31) * P1) & _M64
            off += 32
        h = (_rotl(v1, 1) + _rotl(v2, 7) + _rotl(v3, 12) + _rotl(v4, 18)) & _M64
        for v in (v1, v2, v3, v4):
            h = ((h ^ ((_rotl((v * P2) & _M64, 31) * P1) & _M64)) * P1 + P4) & _M64
    else:
        h = (seed + P5) & _M64
    h = (h + n) & _M64
    while off + 8 <= n:
        w = int.from_bytes(b[off: off + 8], "little")
        h ^= (_rotl((w * P2) & _M64, 31) * P1) & _M64
        h = (_rotl(h, 27) * P1 + P4) & _M64
        off += 8
    if off + 4 <= n:
        w = int.from_bytes(b[off: off + 4], "little")
        h ^= (w * P1) & _M64
        h = (_rotl(h, 23) * P2 + P3) & _M64
        off += 4
    while off < n:
        h ^= (b[off] * P5) & _M64
        h = (_rotl(h, 11) * P1) & _M64
        off += 1
    h ^= h >> 33
    h = (h * P2) & _M64
    h ^= h >> 29
    h = (h * P3) & _M64
    h ^= h >> 32
    return h


def hll_precision(rsd) -> int:
    rsd = 0.05 if rsd is None else rsd
    return int(math.ceil(2.0 * math.log(1.106 / rsd) / math.log(2.0)))


def hll_hashes(values: np.ndarray, sdtype: str) -> np.ndarray:
    """Spark's per-type XXH64 encoding of non-null values -> uint64 hashes."""
    if sdtype == "string":
        # the registers are a max over the values: hashing every DISTINCT string once gives the same registers
        return np.array([xxh64_bytes(str(s).encode("utf-8")) for s in set(values.tolist())], dtype=np.uint64)
    if sdtype == "int":
        return xxh64_int_np(values.astype(np.int32))
    if sdtype in ("bigint", "long"):
        return xxh64_long_np(values.astype(np.int64))
    if sdtype == "float":  # hashInt(floatToIntBits) - parity unpinned
        v = values.astype(np.float32).copy()
        v[v == 0] = 0.0
        v[np.isnan(v)] = np.float32(np.nan)
        return xxh64_int_np(v.view(np.int32))
    v = values.astype(np.float64).copy()
    v[v == 0] = 0.0  # -0.0 normalised
    v[np.isnan(v)] = np.nan
    return xxh64_long_np(v.view(np.int64))


def hll_registers(hashes: np.ndarray, p: int) -> np.ndarray:
    m = 1 << p
    regs = np.zeros(m, dtype=np.uint8)
    if hashes.size == 0:
        return regs
    idx = (hashes >> np.uint64(64 - p)).astype(np.int64)
    with np.errstate(over="ignore"):
        w = (hashes << np.uint64(p)) | np.uint64(1 << (p - 1))
    # rho = clz64(w) + 1
    wf = w.copy()
    lz = np.zeros(w.shape, dtype=np.int64)
    for shift in (32, 16, 8, 4, 2, 1):
        mask = (wf >> np.uint64(64 - shift)) == 0
        lz[mask] += shift
        wf[mask] = wf[mask] << np.uint64(shift)
    rho = (lz + 1).astype(np.uint8)
    np.maximum.at(regs, idx, rho)
    return regs


def hll_estimate(regs: np.ndarray, p: int):
    """-> (estimate:int, in_bias_band:bool).  Bias tables are not available offline:
    in the band (threshold(p), 5m) the raw estimate is returned uncorrected and the
    flag is set ("HLL bias band, parity unpinned")."""
    m = 1 << p
    z = float(np.sum(np.exp2(-regs.astype(np.float64))))
    v = int(np.count_nonzero(regs == 0))
    alpha_mm = (0.7213 / (1.0 + 1.079 / m)) * m * m if p >= 7 else \
        {4: 0.673, 5: 0.697, 6: 0.709}[p] * m * m
    e = alpha_mm / z
    if v > 0:
        h = m * math.log(m / v)
        if h <= HLL_THRESHOLDS[p]:
            return int(round(h)), False
    if e >= 5.0 * m:
        return int(round(e)), False
    return int(round(e)), True


def approx_count_distinct(values: np.ndarray, sdtype: str, rsd=None):
    p = hll_precision(rsd)
    regs = hll_registers(hll_hashes(values, sdtype), p)
    return hll_estimate(regs, p)


# ----------------------------------------------------------------------------
# Spark's row samplers (data_sampling.py:122-149 -> Dataset.sample / stat.sampleBy).  Un-vendored classes
# org.apache.spark.util.random.{XORShiftRandom, BernoulliCellSampler} and catalyst Rand (Spark 3.x), restated from
# their published algorithm.  PARITY UNPINNED for the kept row set: the reference holds no vector (its test checks
# count ranges on data/data_sample/test_data_sample.csv only, tests/test_data_sampling_cpu.py).
# ----------------------------------------------------------------------------

_M32 = 0xFFFFFFFF
_M64 = 0xFFFFFFFFFFFFFFFF


def _murmur3_bytes(data: bytes, seed: int) -> int:
    """scala.util.hashing.MurmurHash3.bytesHash (len % 4 == 0 is all XORShiftRandom needs)."""
    h = seed & _M32
    for i in range(0, len(data) - len(data) % 4, 4):
        k = int.from_bytes(data[i:i + 4], "little")
        k = (k * 0xcc9e2d51) & _M32
        k = ((k << 15) | (k >> 17)) & _M32
        k = (k * 0x1b873593) & _M32
        h ^= k
        h = ((h << 13) | (h >> 19)) & _M32
        h = (h * 5 + 0xe6546b64) & _M32
    h ^= len(data)
    h ^= h >> 16
    h = (h * 0x85ebca6b) & _M32
    h ^= h >> 13
    h = (h * 0xc2b2ae35) & _M32
    h ^= h >> 16
    return h


def xorshift_hash_seed(seed: int) -> int:
    """XORShiftRandom.hashSeed: MurmurHash3 of the 8 big-endian bytes of the (Java long) seed, twice."""
    b = (seed & _M64).to_bytes(8, "big")
    low = _murmur3_bytes(b, 0x3c074a61)
    high = _murmur3_bytes(b, low)
    return ((high << 32) | low) & _M64


def xorshift_uniform53(seed: int, n: int) -> np.ndarray:
    """The first n nextDouble() draws of XORShiftRandom(seed) as 53-bit integers k (the double is k * 2^-53)."""
    s = xorshift_hash_seed(seed)
    out = np.empty(n, dtype=np.uint64)

    def nxt(s):
        s ^= (s << 21) & _M64
        s ^= s >> 35
        s ^= (s << 4) & _M64
        return s
    for i in range(n):
        s = nxt(s)
        hi = s & ((1 << 26) - 1)
        s = nxt(s)
        out[i] = (hi << 27) + (s & ((1 << 27) - 1))
    return out


def bernoulli_keep(n: int, seed: int, fractions) -> np.ndarray:
    """bool[n]: row i of ONE partition is kept when draw_i < fractions[i] (scalar fraction or per-row array)."""
    x = xorshift_uniform53(seed, n).astype(np.float64) * 2.0 ** -53     # exact: k < 2^53
    return x < np.asarray(fractions, dtype=np.float64)
