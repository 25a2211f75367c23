"""`data_sample` of anovos.data_ingest.data_sampling (reference /root/reference/src/main/anovos/data_ingest/
data_sampling.py:8-149): random and stratified (population / balanced) under-sampling, reproducing WHICH rows Spark
keeps.  Spark draws one `nextDouble()` per row from `XORShiftRandom(seed + partitionIndex)` and keeps the row when
x < fraction (`Dataset.sample`) or x < fractions[stratum] (`stat.sampleBy`, evaluated on the rows that survive
`na.drop(subset=strata_cols)`); the generator is restated in csrc/sample.cu and runs on the device, one launch per
partition.  A ColumnFrame is one partition (index 0); a Spark-partitioned PartitionedFrame keeps its partitions.

Parity: the sampler follows the published algorithm of the un-vendored Spark classes (XORShiftRandom,
BernoulliCellSampler, Rand); the reference holds no vector that pins individual kept rows (its test checks count
ranges only, tests/test_data_sampling_cpu.py reproduces it through the oracle) - "parity unpinned" for the row set.
"""
from __future__ import annotations

import ctypes as C
import warnings
from fractions import Fraction

import numpy as np

from .. import _lib, profile
from ..frame import ColumnFrame, as_frame
from ..shared.utils import names, unique


def fraction_threshold(fraction: float) -> int:
    """x < fraction with x = k * 2^-53  <=>  k < ceil(fraction * 2^53) (exact rational arithmetic)."""
    f = Fraction(float(fraction)) * (1 << 53)
    k = -((-f.numerator) // f.denominator)
    return int(min(max(k, 0), 1 << 53))


def _require(ok, message):
    """The reference signals every bad argument of data_sample with a TypeError (data_sampling.py:72-118)."""
    if not ok:
        raise TypeError(message)


def sample_mask(n_rows: int, seed: int, thresholds, strata=None):
    """-> bool CUDA tensor [n_rows] of the rows Spark keeps in ONE partition seeded with `seed` (already seed + index).
    thresholds: ceil(fraction * 2^53) per stratum; strata: int32 CUDA tensor of stratum ids or None."""
    torch = _lib.require_cuda()
    L = _lib.lib()
    words = (n_rows + 31) // 32
    keep = torch.zeros(max(words, 1), dtype=torch.int32, device="cuda")
    thr = torch.from_numpy(np.asarray(thresholds, dtype=np.uint64).view(np.int64)).cuda()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    # Java long arithmetic wraps: seed + partitionIndex is taken modulo 2^64 as a signed value
    seed = ((int(seed) + (1 << 63)) % (1 << 64)) - (1 << 63)
    _lib.check(L.anv_spark_sample_mask(n_rows, seed, strata.data_ptr() if strata is not None else None, thr.data_ptr(),
                                       len(thresholds), keep.data_ptr(), st), "anv_spark_sample_mask")
    rows = torch.arange(n_rows, device="cuda")
    return ((keep[rows >> 5] >> (rows & 31).to(torch.int32)) & 1).bool()


def _value_strings(fr: ColumnFrame, name, values):
    """Spark's cast-to-string of the distinct `values` (numpy) of column `name` - what F.concat sees."""
    col = fr.column(name)
    if col.dictionary is not None:
        return [col.dictionary[int(v)] for v in values]
    if col.sdtype in ("int", "bigint", "long"):
        return [str(int(v)) for v in values]
    from ..shared.utils import jvm_double_str
    if col.sdtype == "float":      # Float.toString prints the shortest float32 repr
        return [jvm_double_str(float(str(np.float32(v)))) for v in values]
    return [jvm_double_str(float(v)) for v in values]


def _strata_ids(fr: ColumnFrame, cols):
    """-> (int32 CUDA tensor of stratum ids per row, counts per stratum as numpy int64).  Strata are the distinct
    values of F.concat(*cols): value tuples whose concatenated strings coincide share a stratum, like in Spark."""
    torch = _lib.require_cuda()
    per_col = []
    for c in cols:
        d, _ = fr.column(c).device()
        u, inv = torch.unique(d, return_inverse=True)
        per_col.append((u.cpu().numpy(), inv))
    comp = torch.zeros(fr.n_rows, dtype=torch.int64, device=per_col[0][1].device)
    for u, inv in per_col:
        comp = comp * max(len(u), 1) + inv
    combos, inv = torch.unique(comp, return_inverse=True)
    combos = combos.cpu().numpy()
    parts, rem = [], combos.copy()
    for (u, _), c in reversed(list(zip(per_col, cols))):
        k = max(len(u), 1)
        parts.append(_value_strings(fr, c, u[rem % k]))
        rem = rem // k
    merged = ["".join(t) for t in zip(*reversed(parts))] if parts else []
    ids = {}
    remap = np.empty(len(merged), np.int64)
    for i, s in enumerate(merged):
        remap[i] = ids.setdefault(s, len(ids))
    strata = torch.from_numpy(remap).to(inv.device)[inv].to(torch.int32)
    counts = np.bincount(remap[inv.cpu().numpy()] if len(ids) != len(merged) else inv.cpu().numpy(), minlength=len(ids))
    return strata, counts.astype(np.int64), list(ids)


def data_sample(idf, strata_cols="all", drop_cols=[], fraction=0.1, method_type="random", stratified_type="population",
                seed_value=12, unique_threshold=0.5, partition_index=0):
    """Same arguments, checks, warnings and results as the reference (:8-149).  `partition_index` (extra): the Spark
    partition a ColumnFrame stands for (default 0 - a frame is one partition)."""
    _require(type(fraction) in (float, int), "Invalid input for fraction")
    _require(0 < fraction <= 1, "Invalid input for fraction: fraction value is between 0 and 1")
    _require(type(seed_value) is int, "Invalid input for seed_value")
    _require(method_type in ("stratified", "random"), "Invalid input for data_sample method_type")
    fr = as_frame(idf)
    if getattr(fr, "is_partitioned", False):
        return _sample_partitions(fr, strata_cols, drop_cols, fraction, method_type, stratified_type, seed_value, unique_threshold)
    if method_type == "random":
        return fr.filter_rows(sample_mask(fr.n_rows, seed_value + partition_index, [fraction_threshold(fraction)]))
    strata_cols = _checked_strata(fr, strata_cols, drop_cols, stratified_type, unique_threshold)
    if not strata_cols:
        return fr
    return _stratified(fr, strata_cols, fraction, stratified_type, seed_value + partition_index, None)


def _checked_strata(fr, strata_cols, drop_cols, stratified_type, unique_threshold):
    _require(type(unique_threshold) in (float, int), "Invalid input for unique_threshold")
    _require(unique_threshold <= 1 or type(unique_threshold) is int,
             "Invalid input for unique_threshold: unique_threshold can only be integer if larger than 1")
    _require(unique_threshold > 0,
             "Invalid input for unique_threshold: unique_threshold value is either between 0 and 1, or an integer > 1")
    _require(stratified_type in ("population", "balanced"), "Invalid input for stratified_type")
    if isinstance(strata_cols, str) and strata_cols == "all":
        strata_cols = fr.columns
    strata_cols = unique(names(strata_cols), names(drop_cols))
    _require(strata_cols, "Missing strata_cols value")
    for col in strata_cols:
        _require(col in fr.columns, "Invalid input for strata_cols: " + col + " does not exist")
        _require(fr.column(col).kind != "other", "Invalid input for strata_cols: dtype of %s is not numerical/categorical" % col)
    # `select(col).distinct().count()` counts the null group as one value; `select(col).count()` is the row count
    md = profile.mode_distinct(fr, strata_cols)
    nv = profile.n_valid(fr, strata_cols)
    N = fr.count()
    skip = []
    for col in strata_cols:
        distinct = md[col][2] + (1 if nv[col] < N else 0)
        limit = unique_threshold * float(N) if unique_threshold <= 1 else unique_threshold
        if float(distinct) > limit:
            skip.append(col)
    if skip:
        warnings.warn("Columns dropped from strata due to high cardinality: " + ",".join(skip))
    strata_cols = [e for e in strata_cols if e not in skip]
    if len(strata_cols) == 0:
        warnings.warn("No Stratified Sampling Computation - No strata column(s) to sample")
    return strata_cols


def _stratified(fr, strata_cols, fraction, stratified_type, seed, global_counts):
    """na.drop(subset) -> merge key -> sampleBy (:122-146) on ONE partition.  global_counts: {merge string: rows} over
    ALL partitions (balanced fractions are computed on the whole frame), None = this frame is the whole frame."""
    sub = fr.dropna(subset=strata_cols)
    if sub.n_rows == 0:
        return sub
    strata, counts, keys = _strata_ids(sub, strata_cols)
    if stratified_type == "population":
        thr = [fraction_threshold(fraction)] * len(keys)
    else:
        cnt = {k: int(v) for k, v in zip(keys, counts)} if global_counts is None else global_counts
        smallest = min(cnt.values())
        thr = [fraction_threshold(float(fraction * smallest / cnt[k])) for k in keys]
    keep = sample_mask(sub.n_rows, seed, thr, strata)
    return sub.filter_rows(keep)


def _sample_partitions(pf, strata_cols, drop_cols, fraction, method_type, stratified_type, seed_value, unique_threshold):
    """Every chunk of a Spark-partitioned frame is one partition: seed + chunk index, the partitions stay partitions."""
    from ..partitioned import PartitionedFrame
    if pf.group is not None:
        raise NotImplementedError("data_sample on row slabs spread over ranks")
    chunks = [pf._chunk_fn(i) for i in range(pf.n_chunks)]
    if method_type == "random":
        out = [ch.filter_rows(sample_mask(ch.n_rows, seed_value + i, [fraction_threshold(fraction)])) for i, ch in enumerate(chunks)]
    else:
        whole = pf.materialize()
        cols = _checked_strata(whole, strata_cols, drop_cols, stratified_type, unique_threshold)
        if not cols:
            return pf
        gc = None
        if stratified_type == "balanced":
            sub = whole.dropna(subset=cols)
            _, counts, keys = _strata_ids(sub, cols) if sub.n_rows else (None, [], [])
            gc = {k: int(v) for k, v in zip(keys, counts)}
        out = [_stratified(ch, cols, fraction, stratified_type, seed_value + i, gc) for i, ch in enumerate(chunks)]
    res = PartitionedFrame.from_frames(out)
    res.spark_partitions = pf.spark_partitions
    return res
