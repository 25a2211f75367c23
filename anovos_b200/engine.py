"""Host driver of the CUDA kernels: turns ColumnFrames + binning models into C-ABI calls.

All device work goes through libanovos_b200.so (include/anovos_b200.h) on torch's
current CUDA stream.  torch is plumbing only: device buffers and streams.
"""
from __future__ import annotations

import copy
import ctypes as C
import math

import numpy as np

from . import _lib
from .frame import ColumnFrame
from .shared import gk as _gk

_NP_OF_ANV = {_lib.ANV_F32: np.float32, _lib.ANV_F64: np.float64, _lib.ANV_I32: np.int32, _lib.ANV_I64: np.int64}

MOMENT_FIELDS = ("n_valid", "n_nonzero", "min", "max", "mean", "m2", "m3", "m4")
_MOM_DT = np.dtype([("n_valid", "<i8"), ("n_nonzero", "<i8"), ("min", "<f8"), ("max", "<f8"),
                    ("mean", "<f8"), ("m2", "<f8"), ("m3", "<f8"), ("m4", "<f8")])
_DRIFT_DT = np.dtype([("psi", "<f8"), ("hd", "<f8"), ("jsd", "<f8"), ("ks", "<f8"), ("n_rows", "<i4"), ("r", "<i4")])
_SPEC_DT = np.dtype([("n_bins", "<i4"), ("mode", "<i4"), ("lo", "<f8"), ("inv_w", "<f8"), ("cut_offset", "<i8")])

launch_count = 0  # kernels launched through this module (bench.py reports it)


class KernelTimer:
    """Optional CUDA-event timing of every C-ABI call (on the launching stream), per entry point."""

    def __init__(self):
        self.spans = []

    def totals(self):
        import torch
        torch.cuda.synchronize()
        out = {}
        for name, e0, e1, nbytes in self.spans:
            t = out.setdefault(name, [0.0, 0, 0])
            t[0] += e0.elapsed_time(e1)
            t[1] += 1
            t[2] += nbytes
        return {k: {"ms": v[0], "calls": v[1], "input_bytes": v[2]} for k, v in out.items()}


timer = None  # set to a KernelTimer() to collect per-call device times
d2h_bytes = 0  # bytes read back from the device by this module


def _host(t, nbytes=None):
    """device uint8 tensor -> numpy (counts the D2H bytes)."""
    global d2h_bytes
    a = t.cpu().numpy()
    d2h_bytes += a.nbytes if nbytes is None else nbytes
    return a


def _call(fn, name, *args, nbytes=0):
    """nbytes: bytes of column data (+ validity bitmaps) one read of the call's input columns moves - the
    algorithmic bytes of SURVEY.md 8(d), recorded with the device time so bench.py can quote GB/s per call."""
    if timer is None:
        _lib.check(fn(*args), name)
        return
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    rc = fn(*args)
    e1.record()
    timer.spans.append((name, e0, e1, nbytes))
    _lib.check(rc, name)


def input_bytes(frame, names) -> int:
    """One read of `names`: n_rows * itemsize (+ n_rows / 8 where a validity bitmap exists)."""
    if timer is None:
        return 0
    tot = 0
    for n in names:
        col = frame.column(n)
        tot += frame.n_rows * (4 if col.anv_dtype in (_lib.ANV_F32, _lib.ANV_I32) else 8)
        if col.has_validity:
            tot += (frame.n_rows + 7) // 8
    return tot


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev_bytes(nbytes):
    import torch
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device="cuda")


def _to_dev(arr: np.ndarray):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(-1)).cuda()


def _in_column_blocks(call, n_cols):
    """call(lo, hi) over consecutive column blocks [lo, hi) of at most _lib.MAX_LAUNCH_COLS columns, the most one launch
    of a per-column pass takes, with the per-block results joined along the column axis: NumPy arrays and CUDA tensors
    concatenated, lists chained, tuples joined element by element.  Up to that many columns it is call(0, n_cols) itself.
    Every per-column result depends on its own column only, so the blocks give the results of one wide call."""
    if n_cols <= _lib.MAX_LAUNCH_COLS:
        return call(0, n_cols)
    parts = [call(lo, min(lo + _lib.MAX_LAUNCH_COLS, n_cols)) for lo in range(0, n_cols, _lib.MAX_LAUNCH_COLS)]

    def join(xs):
        if isinstance(xs[0], list):
            return [v for x in xs for v in x]
        if isinstance(xs[0], tuple):
            return tuple(join(list(t)) for t in zip(*xs))
        if isinstance(xs[0], np.ndarray):
            return np.concatenate(xs)
        import torch
        return torch.cat(xs)
    return join(parts)


# ---- K1 ---------------------------------------------------------------------------------

def moments(frame: ColumnFrame, names):
    """-> structured ndarray (one row per name) with MOMENT_FIELDS.  One fused pass."""
    if getattr(frame, "is_partitioned", False):
        return frame.moments(names)
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: moments(frame, names[lo:hi]), len(names))
    if not names:
        return np.zeros(0, dtype=_MOM_DT)
    desc, keep = frame.descriptors(names)
    ws_bytes = L.anv_moments_workspace_bytes(len(names), frame.n_rows)
    ws = _dev_bytes(ws_bytes)
    out = _dev_bytes(len(names) * _MOM_DT.itemsize)
    _call(L.anv_moments, "anv_moments", desc.data_ptr(), len(names), frame.n_rows, out.data_ptr(), ws.data_ptr(), ws_bytes,
                             _stream(), nbytes=input_bytes(frame, names))
    launch_count += 2
    return _host(out).view(_MOM_DT).copy()


# ---- binning model -> device specs ---------------------------------------------------------

def native_thresholds(cutoffs, anv_dtype) -> np.ndarray:
    """float64 cutoffs -> native-type thresholds theta with (double(v) <= c) == (v <= theta), as uint64 slots.
    NaN cutoffs (`v <= NaN` is False for every v) become the lowest value: "below" everything."""
    cut = np.asarray(cutoffs, dtype=np.float64)
    raw = np.zeros(cut.size, dtype=np.uint64)
    nan = np.isnan(cut)
    if anv_dtype == _lib.ANV_F32:
        with np.errstate(over="ignore", invalid="ignore"):
            th = cut.astype(np.float32)
            up = th.astype(np.float64) > cut                      # rounded up: step one float32 down
            th = np.where(up, np.nextafter(th, np.float32(-np.inf)), th).astype(np.float32)
        th[nan] = -np.inf
        raw[:] = th.view(np.uint32).astype(np.uint64)
    elif anv_dtype == _lib.ANV_F64:
        th = np.where(nan, -np.inf, cut)
        raw[:] = th.view(np.uint64)
    else:
        lo, hi = (-(1 << 31), (1 << 31) - 1) if anv_dtype == _lib.ANV_I32 else (-(1 << 63), (1 << 63) - 1)
        vals = []
        for c in cut.tolist():
            if c != c or c == -math.inf:
                v = lo
            elif c == math.inf:
                v = hi
            else:
                v = min(max(math.floor(c), lo), hi)
            vals.append(v)
        if anv_dtype == _lib.ANV_I32:
            raw[:] = np.array(vals, dtype=np.int64).astype(np.int32).view(np.uint32).astype(np.uint64)
        else:
            raw[:] = np.array(vals, dtype=np.int64).view(np.uint64)
    return raw


I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def i64_at_most(c) -> int:
    """The largest int64 x whose double is <= c, as a Python int: `float(x) <= c` <=> `x <= i64_at_most(c)` for every int64
    x, where float(x) is x rounded to the nearest double (ties to even), as NumPy's astype(float64) and the JVM's long ->
    double conversion round.  I64_MIN - 1 when no int64 qualifies (c < -2^63, or NaN)."""
    c = float(c)
    if c != c or c < -2.0 ** 63:
        return I64_MIN - 1
    if c >= 2.0 ** 63:
        return I64_MAX
    x = math.floor(c)                       # exact: float(x) == x <= c
    if x == c:                              # c is an integer: the ints up to the midpoint to the next double may round to c
        nxt = math.nextafter(c, math.inf)
        mid = x + (int(nxt) - x) // 2
        x = mid if float(mid) <= c else mid - 1
    return min(x, I64_MAX)


class BinModel:
    """Host description of the binning of a set of columns + its device image.
    exact: optional per-column list of the native thresholds themselves, as Python ints (None: derive them from the
    float64 cutoffs), for ANV_I64 columns whose thresholds a double cannot hold; value v goes to bin 1 + #(thresholds < v)."""

    def __init__(self, frame: ColumnFrame, names, cutoffs, lo_hi=None, exact=None):
        self.names = list(names)
        self.cutoffs = [list(map(float, c)) for c in cutoffs]
        self.exact = list(exact) if exact is not None else [None] * len(self.names)
        self.max_bins = max((len(c) + 1 for c in self.cutoffs), default=2)
        specs = np.zeros(len(self.names), dtype=_SPEC_DT)
        raws, off = [], 0
        for i, (nme, cut) in enumerate(zip(self.names, self.cutoffs)):
            col = frame.column(nme)
            if self.exact[i] is not None:
                if col.anv_dtype != _lib.ANV_I64 or len(self.exact[i]) != len(cut):
                    raise ValueError("exact thresholds are for bigint columns, one per cutoff (column %r)" % nme)
                raw = np.array([int(t) for t in self.exact[i]], dtype=np.int64).view(np.uint64)   # out of range: OverflowError
            else:
                raw = native_thresholds(cut, col.anv_dtype)
            mode, lo, inv_w = 0, 0.0, 0.0
            if lo_hi is not None and lo_hi[i] is not None and col.anv_dtype in (_lib.ANV_F32, _lib.ANV_F64):
                mn, mx = lo_hi[i]
                nb = len(cut) + 1
                w = (mx - mn) / nb
                th = raw.astype(np.uint32).view(np.float32).astype(np.float64) if col.anv_dtype == _lib.ANV_F32 \
                    else raw.view(np.float64)
                ulp = np.spacing(np.float32(max(abs(mn), abs(mx)))) if col.anv_dtype == _lib.ANV_F32 \
                    else np.spacing(max(abs(mn), abs(mx)))
                ok = (w > 0 and math.isfinite(w) and np.all(np.isfinite(th)) and np.all(np.diff(th) > 0)
                      and w >= 8 * float(ulp) and nb < (1 << 20))
                # the guess runs in the column's type: x - lo over the range and the scales 1/w and 1/(w (B-1)) must be
                # finite normal numbers of it (a range wider than FLT_MAX overflows; a subnormal width overflows 1/w)
                T = np.float32 if col.anv_dtype == _lib.ANV_F32 else np.float64
                with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
                    scales = np.array([1.0 / w, 1.0 / (w * max(nb - 1, 1))]).astype(T) if ok else np.zeros(2, T)
                    ok = ok and bool(np.isfinite(T(mx) - T(mn)) and np.all(np.isfinite(scales))
                                     and np.all(scales >= np.finfo(T).tiny))
                if ok:
                    mode, lo, inv_w = 1, mn, 1.0 / w
            specs[i] = (len(cut) + 1, mode, lo, inv_w, off)
            raws.append(raw)
            off += len(raw)
        self.specs_host = specs
        self.cuts_host = np.concatenate(raws) if raws else np.zeros(1, np.uint64)
        self._dev = None

    def block(self, lo, hi):
        """The model of columns [lo, hi): their specs with the same thresholds (cut_offset indexes the whole `cuts`) and
        the same max_bins, so the count strides of the blocks agree."""
        sub = copy.copy(self)
        sub.names, sub.cutoffs, sub.exact = self.names[lo:hi], self.cutoffs[lo:hi], self.exact[lo:hi]
        sub.specs_host = self.specs_host[lo:hi]
        sub._dev = None
        return sub

    def device(self):
        if self._dev is None:
            self._dev = (_to_dev(self.specs_host), _to_dev(self.cuts_host if self.cuts_host.size else np.zeros(1, np.uint64)))
        return self._dev


# ---- K2 / fused / assign ---------------------------------------------------------------------

def histogram(frame: ColumnFrame, model: BinModel):
    """-> uint64 ndarray [n_cols, max_bins + 1]: slot 0 = nulls, slot b = rows in bin b."""
    if getattr(frame, "is_partitioned", False):
        return frame.histogram(model)
    global launch_count
    _lib.require_cuda()
    L = _lib.lib()
    n = len(model.names)
    if n > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: histogram(frame, model.block(lo, hi)), n)
    stride = model.max_bins + 1
    if n == 0:
        return np.zeros((0, stride), np.uint64)
    desc, keep = frame.descriptors(model.names)
    specs, cuts = model.device()
    counts = _dev_bytes(n * stride * 8)
    _call(L.anv_hist, "anv_hist", desc.data_ptr(), specs.data_ptr(), cuts.data_ptr(), n, frame.n_rows, counts.data_ptr(),
                          stride, _stream(), nbytes=input_bytes(frame, model.names))
    launch_count += 1
    return _host(counts).view(np.uint64).reshape(n, stride).copy()


def moments_histogram(frame: ColumnFrame, model: BinModel):
    """Moments AND histogram of `model.names` in ONE read of the frame."""
    if getattr(frame, "is_partitioned", False):
        return frame.moments_histogram(model)
    global launch_count
    _lib.require_cuda()
    L = _lib.lib()
    n = len(model.names)
    if n > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: moments_histogram(frame, model.block(lo, hi)), n)
    stride = model.max_bins + 1
    if n == 0:
        return np.zeros(0, dtype=_MOM_DT), np.zeros((0, stride), np.uint64)
    desc, keep = frame.descriptors(model.names)
    specs, cuts = model.device()
    counts = _dev_bytes(n * stride * 8)
    ws_bytes = L.anv_moments_workspace_bytes(n, frame.n_rows)
    ws = _dev_bytes(ws_bytes)
    out = _dev_bytes(n * _MOM_DT.itemsize)
    _call(L.anv_moments_hist, "anv_moments_hist", desc.data_ptr(), specs.data_ptr(), cuts.data_ptr(), n, frame.n_rows, out.data_ptr(),
                                  counts.data_ptr(), stride, ws.data_ptr(), ws_bytes, _stream(),
          nbytes=input_bytes(frame, model.names))
    launch_count += 2
    return (_host(out).view(_MOM_DT).copy(),
            _host(counts).view(np.uint64).reshape(n, stride).copy())


def bin_assign(frame: ColumnFrame, model: BinModel):
    """-> int32 CUDA tensor [n_cols, stride] of bin ids (0 = null row); stride >= n_rows."""
    if getattr(frame, "is_partitioned", False):
        return frame.bin_assign(model)
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    n = len(model.names)
    if n > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: bin_assign(frame, model.block(lo, hi)), n)
    stride = (frame.n_rows + 3) // 4 * 4
    out = torch.empty((max(n, 1), max(stride, 4)), dtype=torch.int32, device="cuda")
    if n == 0 or frame.n_rows == 0:
        return out[:n, :frame.n_rows]
    desc, keep = frame.descriptors(model.names)
    specs, cuts = model.device()
    _call(L.anv_bin_assign, "anv_bin_assign", desc.data_ptr(), specs.data_ptr(), cuts.data_ptr(), n, frame.n_rows, model.max_bins,
                                out.data_ptr(), out.stride(0), _stream(), nbytes=input_bytes(frame, model.names))
    launch_count += 1
    return out[:, :frame.n_rows]


def code_counts(frame: ColumnFrame, names):
    """Dictionary-code histograms of string columns -> list of uint64 arrays [cardinality + 1]
    (slot 0 = nulls).  Columns are grouped by cardinality class so each launch sizes its
    shared-memory histogram for its own group."""
    if getattr(frame, "is_partitioned", False):
        return frame.code_counts(list(names))
    global launch_count
    _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: code_counts(frame, names[lo:hi]), len(names))
    out = {}
    groups = {}
    for nme in names:
        card = max(len(frame.column(nme).dictionary), 1)
        cls = 0 if card + 1 <= 40 else (1 if card + 1 <= 10240 else 2)
        groups.setdefault(cls, []).append(nme)
    for cls, grp in groups.items():
        cards = np.array([max(len(frame.column(g).dictionary), 1) for g in grp], dtype=np.int32)
        stride = int(cards.max()) + 1
        desc, keep = frame.descriptors(grp)
        dcards = _to_dev(cards)
        counts = _dev_bytes(len(grp) * stride * 8)
        _call(L.anv_hist_codes, "anv_hist_codes", desc.data_ptr(), dcards.data_ptr(), len(grp), frame.n_rows, counts.data_ptr(),
                                    stride, _stream(), nbytes=input_bytes(frame, grp))
        launch_count += 1
        h = _host(counts).view(np.uint64).reshape(len(grp), stride)
        for i, g in enumerate(grp):
            out[g] = h[i, :cards[i] + 1].copy()
    return [out[n] for n in names]


# ---- K3 ---------------------------------------------------------------------------------

def drift_reduce(src_counts, tgt_counts, kinds, n_src, n_tgt, src_p=None):
    """Lists (per column) of aligned uint64 count arrays (slot 0 = nulls) -> structured array
    with psi/hd/jsd/ks/n_rows.  src_p: list of float64 arrays (NaN = key absent) instead of
    src_counts when the source comes from a saved model."""
    global launch_count
    _lib.require_cuda()
    L = _lib.lib()
    n = len(tgt_counts)
    if n == 0:
        return np.zeros(0, dtype=_DRIFT_DT)
    n_slots = np.array([len(t) for t in tgt_counts], dtype=np.int32)
    stride = int(n_slots.max())
    T = np.zeros((n, stride), np.uint64)
    for i, t in enumerate(tgt_counts):
        T[i, :len(t)] = t
    dT = _to_dev(T)
    if src_p is None:
        S = np.zeros((n, stride), np.uint64)
        for i, s in enumerate(src_counts):
            S[i, :len(s)] = s
        dS, dP, is_p = _to_dev(S), None, 0
    else:
        Pm = np.full((n, stride), np.nan, np.float64)
        for i, s in enumerate(src_p):
            Pm[i, :len(s)] = s
        dS, dP, is_p = None, _to_dev(Pm), 1
    dslots, dkind = _to_dev(n_slots), _to_dev(np.asarray(kinds, dtype=np.int32))
    out = _dev_bytes(n * _DRIFT_DT.itemsize)
    _call(L.anv_drift_reduce, "anv_drift_reduce", dS.data_ptr() if dS is not None else None, dT.data_ptr(),
                                  dP.data_ptr() if dP is not None else None, is_p, dslots.data_ptr(), dkind.data_ptr(),
                                  n, stride, int(n_src), int(n_tgt), out.data_ptr(), _stream())
    launch_count += 1
    return _host(out).view(_DRIFT_DT).copy()


# ---- K4 ---------------------------------------------------------------------------------

def quantile_ranks(n_valid: int, probs, eps=None):
    """1-based ranks of the order statistics Spark returns for `probs` over n_valid non-null values.
    eps None: the exact rule max(1, ceil(p * n)) with p * n in float64 (SURVEY B.2).  eps = the relativeError of
    the Spark call being replaced (1e-4 for summary(), 0.01 for approxQuantile): the Greenwald-Khanna sketch
    position for one partition of < 50 000 values, the exact rule beyond (shared/gk.py; frames tagged with their
    Spark partitioning go through PartitionedFrame.gk_quantiles instead, any partition size)."""
    return _gk.spark_ranks(int(n_valid), probs, eps)


def select_ranks(frame: ColumnFrame, names, ranks):
    """ranks: int64 array [n_cols, n_ranks] of 1-based ranks among non-null values (0 = skip).
    -> float64 array [n_cols, n_ranks] of the exact order statistics (NaN where skipped)."""
    if getattr(frame, "is_partitioned", False):
        return frame.select_ranks(names, ranks)
    global launch_count
    _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    ranks = np.ascontiguousarray(ranks, dtype=np.int64).reshape(len(names), -1)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: select_ranks(frame, names[lo:hi], ranks[lo:hi]), len(names))
    out = np.full(ranks.shape, np.nan, np.float64)
    if not names or ranks.shape[1] == 0:
        return out
    groups = {}
    for i, nme in enumerate(names):
        kb = 32 if frame.column(nme).anv_dtype in (_lib.ANV_F32, _lib.ANV_I32) else 64
        groups.setdefault(kb, []).append(i)
    for kb, idx in groups.items():
        for r0 in range(0, ranks.shape[1], 16):
            rk = np.ascontiguousarray(ranks[idx, r0:r0 + 16])
            grp = [names[i] for i in idx]
            desc, keep = frame.descriptors(grp)
            ws_bytes = L.anv_select_workspace_bytes(len(grp), rk.shape[1])
            ws = _dev_bytes(ws_bytes)
            drk = _to_dev(rk)
            dout = _dev_bytes(rk.size * 8)
            _call(L.anv_select_ranks, "anv_select_ranks", desc.data_ptr(), len(grp), frame.n_rows, drk.data_ptr(), rk.shape[1], kb,
                                          dout.data_ptr(), ws.data_ptr(), ws_bytes, _stream(), nbytes=input_bytes(frame, grp))
            launch_count += 2 * (3 if kb == 32 else 7)
            out[np.asarray(idx)[:, None], np.arange(r0, r0 + rk.shape[1])[None, :]] = \
                _host(dout).view(np.float64)[:rk.size].reshape(rk.shape)
    return out


# ---- sort-based exact mode / distinct --------------------------------------------------------

EXACT_MAX_ROWS = (1 << 32) - 1    # rows one exact mode / distinct call counts: multiplicities and row numbers are 32-bit
SORT_WORKSPACE_BUDGET = 24 << 30  # bytes of scratch one sort batch may use
sort_algorithm = "partition"      # "partition": F32 / I32 columns with <= 16 ranks take the bucket count; "lsd": every column sorts
FUSED_HLL = True                  # sort_mode_distinct(..., hll_p=p) also returns the HLL++ registers (one hash per distinct value)


def refuse_exact_rows(n_rows, what):
    """AnvError for frames of 2^32 rows or more, which the exact mode / distinct counts of one call cannot count."""
    if n_rows > EXACT_MAX_ROWS:
        raise _lib.AnvError("%s: frames of 2^32 rows or more are not supported (%d rows): the exact mode and distinct "
                            "counts are 32-bit; use the approximate distinct count (HLL++) instead" % (what, n_rows))


def _mode_distinct_batch_size(frame, n_cols, per_col_bytes):
    """Columns per sort launch: at most _lib.MAX_LAUNCH_COLS, and the scratch of a batch stays under SORT_WORKSPACE_BUDGET and
    under 80 % of the memory that is not held by live tensors (torch's allocator statistics: no driver call - cudaMemGetInfo
    costs ~7 ms)."""
    torch = _lib.require_cuda()
    budget = SORT_WORKSPACE_BUDGET
    if per_col_bytes * n_cols > (2 << 30):
        total = torch.cuda.get_device_properties(torch.cuda.current_device()).total_memory
        budget = min(budget, int((total - torch.cuda.memory_allocated()) * 0.8))
    return max(1, min(n_cols, _lib.MAX_LAUNCH_COLS, budget // max(per_col_bytes, 1)))


def sort_mode_distinct(frame: ColumnFrame, names, ranks=None, hll_p=None):
    """-> list of (mode value | None, mode_rows | None, n_distinct) for NUMERIC columns.  The mode of a bigint (ANV_I64)
    column is an exact Python int, every other mode a float; rank values are float64 for every column, as in Spark.
    hll_p (4..12): additionally returns the HyperLogLog++ registers uint32 [n_cols, 2**hll_p] as a by-product of the
    counting (one hash per DISTINCT value instead of a separate pass over every value) - the result then is
    (list, rank values | None, registers).
    ranks: optional int64 [n_cols, n_ranks] of 1-based ranks among the non-null values (0 = skip);
    then returns (list, float64 [n_cols, n_ranks]) with the exact order statistics.
    F32 / I32 columns with at most 16 ranks go through the two-level bucket count (anv_mode_distinct_partition_hll: no
    sort, ~4 words of traffic per key - DESIGN.md section 3); 64-bit columns, longer rank lists and sort_algorithm = "lsd"
    take the batched LSD radix sort (anv_mode_distinct).  All column batches of a call are enqueued back to back on the
    stream into one workspace (stream order makes the reuse safe) and the results come back in ONE device-to-host copy.
    Frames of more than EXACT_MAX_ROWS rows raise AnvError before anything is allocated."""
    refuse_exact_rows(frame.n_rows, "sort_mode_distinct")
    if getattr(frame, "is_partitioned", False):
        return frame.sort_mode_distinct(names, ranks)
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    n_ranks = 0
    if ranks is not None:
        ranks = np.ascontiguousarray(ranks, dtype=np.int64).reshape(len(names), -1)
        n_ranks = ranks.shape[1]
    rvals = np.full((len(names), n_ranks), np.nan, np.float64)
    want_hll = hll_p is not None and 4 <= hll_p <= 12
    hll_m = (1 << hll_p) if want_hll else 0
    hregs = np.zeros((len(names), hll_m), np.uint32) if want_hll else None
    res = {}
    groups = {}
    for i, nme in enumerate(names):
        kb = 32 if frame.column(nme).anv_dtype in (_lib.ANV_F32, _lib.ANV_I32) else 64
        groups.setdefault(kb, []).append(i)

    def run(kb, idxs, partition):
        global launch_count
        n_all = len(idxs)
        if partition:
            ws_of = lambda n: L.anv_mode_distinct_partition_workspace_bytes(n, frame.n_rows)
        else:
            ws_of = lambda n: L.anv_mode_distinct_workspace_bytes(n, frame.n_rows, kb)
        batch = _mode_distinct_batch_size(frame, n_all, ws_of(1))
        ws_bytes = ws_of(min(batch, n_all))
        ws = _dev_bytes(ws_bytes)
        # one result block for the whole call: [mode_value | mode_rows | n_distinct | rank_values], 8 bytes per cell
        out = torch.empty((3 + n_ranks) * n_all, dtype=torch.int64, device="cuda")
        base = out.data_ptr()
        dregs = torch.empty(max(n_all * hll_m, 1), dtype=torch.int32, device="cuda") if want_hll else None
        drk = _to_dev(ranks[idxs]) if n_ranks else None
        for b0 in range(0, n_all, batch):
            sub = [names[i] for i in idxs[b0:b0 + batch]]
            n = len(sub)
            desc, keep = frame.descriptors(sub)
            common = (drk.data_ptr() + b0 * n_ranks * 8 if n_ranks else None, n_ranks,
                      base + (3 * n_all + b0 * n_ranks) * 8 if n_ranks else None, ws.data_ptr(), ws_bytes, _stream())
            mv, mr, nd = base + b0 * 8, base + (n_all + b0) * 8, base + (2 * n_all + b0) * 8
            if partition:
                _call(L.anv_mode_distinct_partition_hll, "anv_mode_distinct_partition", desc.data_ptr(), n, frame.n_rows, mv, mr,
                      nd, *common[:3], hll_p if dregs is not None else 0,
                      dregs.data_ptr() + b0 * hll_m * 4 if dregs is not None else None, *common[3:], nbytes=input_bytes(frame, sub))
                launch_count += 11 + 16
            else:
                _call(L.anv_mode_distinct_hll, "anv_mode_distinct", desc.data_ptr(), n, frame.n_rows, kb, mv, mr, nd,
                      *common[:3], hll_p if dregs is not None else 0,
                      dregs.data_ptr() + b0 * hll_m * 4 if dregs is not None else None, *common[3:], nbytes=input_bytes(frame, sub))
                launch_count += 3 + 4 * (kb // 8)
        host = _host(out.view(torch.uint8))
        hv = host[:n_all * 8].view(np.float64)
        hv64 = host[:n_all * 8].view(np.int64)        # the mode slot of an ANV_I64 column holds the int64 itself
        hr = host[n_all * 8:2 * n_all * 8].view(np.int64)
        hd = host[2 * n_all * 8:3 * n_all * 8].view(np.int64)
        hrv = host[3 * n_all * 8:].view(np.float64).reshape(n_all, n_ranks) if n_ranks else None
        if dregs is not None:
            hregs[np.asarray(idxs)] = _host(dregs.view(torch.uint8)).view(np.uint32)[:n_all * hll_m].reshape(n_all, hll_m)
        del ws
        for j, i in enumerate(idxs):
            if hr[j] == -3:
                raise _lib.AnvError("anv_mode_distinct: a one-sweep look-back gave up waiting for a preceding tile (column %r); "
                                    "unset ANV_SORT_ONESWEEP to use the three-kernel passes" % names[i])
            if n_ranks:
                rvals[i] = hrv[j]
            if hr[j] <= 0:
                res[names[i]] = (None, None, 0)
                continue
            mode = int(hv64[j]) if frame.column(names[i]).anv_dtype == _lib.ANV_I64 else float(hv[j])
            res[names[i]] = (mode, int(hr[j]), int(hd[j]))

    for kb, idxs in groups.items():
        run(kb, idxs, kb == 32 and n_ranks <= 16 and sort_algorithm == "partition")
    out = [res[n] for n in names]
    if hll_p is not None:
        return out, (rvals if ranks is not None else None), hregs
    return (out, rvals) if ranks is not None else out


# ---- row-level checks ----------------------------------------------------------------------------

def row_null_counts(frame: ColumnFrame, names, max_keep=None):
    """-> (uint64 ndarray [len(names) + 1]: slot k = rows with k null columns among `names`,
    int32 CUDA tensor of keep-bitmap words (bit set where the count <= max_keep) or None when max_keep is None).
    Columns without a validity bitmap add nothing and are not handed to the kernel; the kernel reads the bitmaps only."""
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    ptrs, keepalive, nbytes = [], [], 0
    for nme in names:
        col = frame.column(nme)
        if not col.has_validity:
            continue
        d, v = col.device()
        if v is None:
            continue
        ptrs.append(v.data_ptr())
        keepalive.append(v)
        nbytes += (frame.n_rows + 7) // 8
    dptrs = _to_dev(np.asarray(ptrs or [0], dtype=np.uint64))
    counts = _dev_bytes((len(names) + 1) * 8)
    keep = None
    if max_keep is not None:
        keep = torch.empty(max((frame.n_rows + 31) // 32, 1), dtype=torch.int32, device="cuda")
    _call(L.anv_row_null_counts, "anv_row_null_counts", dptrs.data_ptr(), len(ptrs), len(names), frame.n_rows,
          -1 if max_keep is None else int(max_keep), counts.data_ptr(), keep.data_ptr() if keep is not None else None,
          _stream(), nbytes=nbytes if timer is not None else 0)
    launch_count += 1
    return _host(counts).view(np.uint64)[:len(names) + 1].copy(), keep


def row_distinct(frame: ColumnFrame, names, hash_bits=0):
    """-> (n_distinct, int32 CUDA tensor of first-occurrence bitmap words in row order).  Exact: rows are compared
    after the hash sort, whatever the hash width (hash_bits 0 = the full width; small widths exercise the comparisons).
    String columns compare by dictionary code: the caller maps repeated dictionary strings to one code first."""
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    if frame.n_rows >= (1 << 32):
        raise _lib.AnvError("row_distinct: frames of 2^32 rows or more are not supported")
    if len(names) > _lib.MAX_LAUNCH_COLS:
        raise NotImplementedError("distinct rows over more than %d columns are not supported: rows are compared whole, so "
                                  "the columns cannot be split into blocks" % _lib.MAX_LAUNCH_COLS)
    desc, keep = frame.descriptors(names) if names else (_dev_bytes(16), None)
    ws_bytes = L.anv_row_distinct_workspace_bytes(frame.n_rows)
    ws = _dev_bytes(ws_bytes)
    nd = torch.zeros(1, dtype=torch.int64, device="cuda")
    first = torch.empty(max((frame.n_rows + 31) // 32, 1), dtype=torch.int32, device="cuda")
    _call(L.anv_row_distinct, "anv_row_distinct", desc.data_ptr(), len(names), frame.n_rows, int(hash_bits), nd.data_ptr(),
          first.data_ptr(), ws.data_ptr(), ws_bytes, _stream(), nbytes=input_bytes(frame, names))
    launch_count += 12
    return int(nd.item()), first


def bitmap_to_bool(words, n_rows):
    """int32 bitmap words (LSB-first) on the device -> bool CUDA tensor [n_rows] (plumbing for frame.filter_rows)."""
    torch = _lib.require_cuda()
    rows = torch.arange(n_rows, device=words.device)
    return ((words[rows >> 5] >> (rows & 31).to(torch.int32)) & 1).bool()


# ---- HLL++ -------------------------------------------------------------------------------------

_HLL_T = {4: 10, 5: 20, 6: 40, 7: 80, 8: 220, 9: 400, 10: 900, 11: 1800, 12: 3100, 13: 6500, 14: 11500,
          15: 20000, 16: 50000, 17: 120000, 18: 350000}


def hll_estimate_from_registers(regs: np.ndarray, p: int):
    """HyperLogLogPlusPlusHelper.query restated: linear counting below the threshold, raw
    estimate above 5m; in between Spark subtracts an empirical bias (tables not available
    offline) -> returned with band=True so the caller can fall back."""
    m = 1 << p
    z = float(np.sum(np.ldexp(1.0, -regs.astype(np.int64))))
    v = int(np.count_nonzero(regs == 0))
    alpha = {4: 0.673, 5: 0.697, 6: 0.709}.get(p, 0.7213 / (1.0 + 1.079 / m))
    e = alpha * m * m / z
    if v > 0:
        h = m * math.log(m / v)
        if h <= _HLL_T[p]:
            return int(math.floor(h + 0.5)), False
    if e >= 5.0 * m:
        return int(math.floor(e + 0.5)), False
    return int(math.floor(e + 0.5)), True


_POW2_NEG = np.ldexp(1.0, -np.arange(128))


def hll_estimates_from_register_rows(R: np.ndarray, p: int):
    """hll_estimate_from_registers for every row of R [n_cols, 2**p] at once -> list of (estimate, in_bias_band)."""
    m = 1 << p
    z = _POW2_NEG[R].sum(axis=1)             # 2^-register, exact (registers are <= 64 - p + 1)
    v = m - np.count_nonzero(R, axis=1)
    alpha = {4: 0.673, 5: 0.697, 6: 0.709}.get(p, 0.7213 / (1.0 + 1.079 / m))
    e = alpha * m * m / z
    out = []
    for ei, vi in zip(e.tolist(), v.tolist()):
        if vi > 0:
            h = m * math.log(m / vi)
            if h <= _HLL_T[p]:
                out.append((int(math.floor(h + 0.5)), False))
                continue
        out.append((int(math.floor(ei + 0.5)), not (ei >= 5.0 * m)))
    return out


_DICT_HLL = {}   # (id(dictionary), p) -> (dictionary, register index per entry, rho per entry)


def _dictionary_hll(dic, p: int):
    """HLL++ (register index, rho) of every entry of a string dictionary: Spark's XXH64 (seed 42) over the UTF-8 bytes
    (anv_xxh64_utf8, host helper of the library), idx = top p bits, rho = clz(rest) + 1.  Cached per dictionary object."""
    key = (id(dic), p)
    hit = _DICT_HLL.get(key)
    if hit is not None and hit[0] is dic:
        return hit[1], hit[2]
    L = _lib.lib()
    enc = [s.encode("utf-8") for s in dic]
    hs = np.zeros(len(enc), np.uint64)
    if enc:
        offs = np.zeros(len(enc) + 1, np.int64)
        np.cumsum([len(b) for b in enc], out=offs[1:])
        blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
        _lib.check(L.anv_xxh64_utf8(blob.ctypes.data, offs.ctypes.data, len(enc), hs.ctypes.data), "anv_xxh64_utf8")
    idx = (hs >> np.uint64(64 - p)).astype(np.int64)
    w = (hs << np.uint64(p)) | np.uint64(1 << (p - 1))
    # clz64(w) + 1 without a Python loop: position of the highest set bit from the float64 exponent is unsafe for 64-bit
    # values, so split into halves (each < 2^32 is exact in float64)
    hi, lo = (w >> np.uint64(32)).astype(np.float64), (w & np.uint64(0xFFFFFFFF)).astype(np.float64)
    with np.errstate(divide="ignore"):
        bl_hi = np.where(hi > 0, np.floor(np.log2(np.maximum(hi, 1))) + 33, 0)
        bl_lo = np.where(lo > 0, np.floor(np.log2(np.maximum(lo, 1))) + 1, 0)
    bitlen = np.where(hi > 0, bl_hi, bl_lo).astype(np.int64)
    rho = (64 - bitlen + 1).astype(np.uint32)
    if len(_DICT_HLL) > 256:
        _DICT_HLL.clear()
    _DICT_HLL[key] = (dic, idx, rho)
    return idx, rho


def hll_registers(frame: ColumnFrame, names, p: int):
    """-> uint32 [n_cols, 2**p] HLL++ registers of NUMERIC columns (max-mergeable across row partitions)."""
    if getattr(frame, "is_partitioned", False):
        return frame.hll_registers(list(names), p)
    global launch_count
    _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: hll_registers(frame, names[lo:hi], p), len(names))
    m = 1 << p
    desc, keep = frame.descriptors(names)
    regs = _dev_bytes(len(names) * m * 4)
    _call(L.anv_hll_registers, "anv_hll_registers", desc.data_ptr(), len(names), frame.n_rows, p, regs.data_ptr(), _stream(), nbytes=input_bytes(frame, names))
    launch_count += 1
    return _host(regs).view(np.uint32)[:len(names) * m].reshape(len(names), m).copy()


def hll_estimates(frame: ColumnFrame, names, p: int):
    """-> list of (estimate, in_bias_band) matching Spark's approx_count_distinct."""
    global launch_count
    _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    m = 1 << p
    out = {}
    num = [n for n in names if frame.column(n).kind == "num"]
    cat = [n for n in names if frame.column(n).kind == "cat"]
    if num:
        R = hll_registers(frame, num, p)
        for n, r in zip(num, hll_estimates_from_register_rows(R, p)):
            out[n] = r
    if cat:
        # per-row work (the code histogram) runs on the device; every dictionary entry is hashed on the host ONCE per
        # dictionary (cached: register index and rho of each entry), so a step only takes a masked maximum
        cc = code_counts(frame, cat)
        R = np.zeros((len(cat), m), np.uint32)
        for i, (n, h) in enumerate(zip(cat, cc)):
            idx, rho = _dictionary_hll(frame.column(n).dictionary, p)
            present = np.flatnonzero(h[1:])
            if present.size:
                np.maximum.at(R[i], idx[present], rho[present])
        for n, r in zip(cat, hll_estimates_from_register_rows(R, p)):
            out[n] = r
    return [out[n] for n in names]


# ---- imputation --------------------------------------------------------------------------------

_IMPUTE_SPEC_DT = np.dtype([("out_dtype", "<i4"), ("flags", "<i4"), ("fill", "<u8")])
_FILL_PAIRS = {(_lib.ANV_F32, _lib.ANV_F32), (_lib.ANV_F64, _lib.ANV_F64), (_lib.ANV_I32, _lib.ANV_I32),
               (_lib.ANV_I64, _lib.ANV_I64), (_lib.ANV_I32, _lib.ANV_F64), (_lib.ANV_I64, _lib.ANV_F64)}
_TORCH_OF_ANV = {_lib.ANV_F32: "float32", _lib.ANV_F64: "float64", _lib.ANV_I32: "int32", _lib.ANV_I64: "int64"}


def java_cast(x, anv_dtype):
    """A double cast to the column type the way the JVM casts it (Spark's `cast` of a double): (float) rounds to nearest,
    d2i / d2l truncate toward zero, saturate at the type's range and map NaN to 0.  -> Python float or int."""
    x = float(x)
    if anv_dtype == _lib.ANV_F64:
        return x
    if anv_dtype == _lib.ANV_F32:
        with np.errstate(over="ignore"):
            return float(np.float32(x))
    lo, hi = (-(1 << 31), (1 << 31) - 1) if anv_dtype == _lib.ANV_I32 else (I64_MIN, I64_MAX)
    if x != x:
        return 0
    if x >= hi:            # hi + 1 is a power of two: every double at or above hi saturates
        return hi
    if x <= lo:
        return lo
    return int(x)          # truncation toward zero; exact, |x| < 2^63


def fill_bits(value, anv_dtype) -> int:
    """The fill value's bits in an output column of `anv_dtype` (the `fill` slot of anv_impute_spec_t): value must be
    representable (java_cast it first)."""
    if anv_dtype == _lib.ANV_F32:
        return int(np.array([value], np.float32).view(np.uint32)[0])
    if anv_dtype == _lib.ANV_F64:
        return int(np.array([value], np.float64).view(np.uint64)[0])
    if anv_dtype == _lib.ANV_I32:
        return int(np.array([value], np.int32).view(np.uint32)[0])
    return int(np.array([value], np.int64).view(np.uint64)[0])


def impute_fill(frame: ColumnFrame, names, out_dtypes, flags, fills):
    """-> list of dense CUDA tensors [n_rows] (one per name, no nulls): anv_impute_fill with per-column output dtype, flags
    (_lib.IMPUTE_*) and fill bits (fill_bits).  One streaming pass over the columns."""
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: impute_fill(frame, names[lo:hi], out_dtypes[lo:hi], flags[lo:hi], fills[lo:hi]),
                                 len(names))
    if not names:
        return []
    specs = np.zeros(len(names), _IMPUTE_SPEC_DT)
    outs, ptrs = [], np.zeros(len(names), np.uint64)
    padded = (frame.n_rows + 3) // 4 * 4
    for i, (n, od, fl, fv) in enumerate(zip(names, out_dtypes, flags, fills)):
        ind = frame.column(n).anv_dtype
        if (ind, od) not in _FILL_PAIRS or (fl & _lib.IMPUTE_NAN_MISSING and ind not in (_lib.ANV_F32, _lib.ANV_F64)):
            raise ValueError("impute_fill: column %r: no fill from dtype %d to %d with flags %d" % (n, ind, od, fl))
        specs[i] = (od, fl, fv)
        t = torch.empty(max(padded, 4), dtype=getattr(torch, _TORCH_OF_ANV[od]), device="cuda")
        outs.append(t)
        ptrs[i] = t.data_ptr()
    if frame.n_rows:
        desc, keep = frame.descriptors(names)
        dspecs, dptrs = _to_dev(specs), _to_dev(ptrs)
        nbytes = input_bytes(frame, names)
        if timer is not None:
            nbytes += sum(frame.n_rows * t.element_size() for t in outs)
        _call(L.anv_impute_fill, "anv_impute_fill", desc.data_ptr(), dspecs.data_ptr(), dptrs.data_ptr(), len(names),
              frame.n_rows, _stream(), nbytes=nbytes)
        launch_count += 1
    return [t[:frame.n_rows] for t in outs]


def valid_not_nan(frame: ColumnFrame, names):
    """-> (int32 CUDA tensor [n_cols, ceil(n_rows/32)] of "non-null and not NaN" bitmap words, int64 ndarray of NaN counts
    per column).  The Imputer's mean and median are the moments / selection of a view of the column with this bitmap."""
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names = list(names)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: valid_not_nan(frame, names[lo:hi]), len(names))
    n_words = (frame.n_rows + 31) // 32
    words = torch.zeros((max(len(names), 1), max(n_words, 1)), dtype=torch.int32, device="cuda")
    if not names:
        return words[:0, :n_words], np.zeros(0, np.int64)
    desc, keep = frame.descriptors(names)
    n_nan = _dev_bytes(len(names) * 8)
    _call(L.anv_valid_not_nan, "anv_valid_not_nan", desc.data_ptr(), len(names), frame.n_rows, words.data_ptr(),
          n_nan.data_ptr(), _stream(), nbytes=input_bytes(frame, names))
    launch_count += 1
    return words[:, :n_words], _host(n_nan).view(np.int64)[:len(names)].copy()


# ---- scaling -------------------------------------------------------------------------------------

_SCALE_SPEC_DT = np.dtype([("mode", "<i4"), ("out_dtype", "<i4"), ("flags", "<i4"), ("reserved", "<i4"),
                           ("a", "<f8"), ("b", "<f8"), ("c", "<f8")])


def scale_columns(frame: ColumnFrame, names, specs):
    """anv_scale_columns: specs = one (mode, out anv dtype, flags, a, b, c) per name (_lib.SCALE_*).
    -> (list of CUDA tensors [n_rows] in the output dtype, list of int32 bitmap tensors [ceil(n_rows/32)] for the
    NAN_TO_NULL columns and None for the others (which keep the source's validity), int64 ndarray of null counts)."""
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names, specs = list(names), list(specs)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: scale_columns(frame, names[lo:hi], specs[lo:hi]), len(names))
    sp = np.zeros(len(names), _SCALE_SPEC_DT)
    outs, ptrs = [], np.zeros(len(names), np.uint64)
    padded = (frame.n_rows + 3) // 4 * 4
    for i, (n, (mode, od, fl, a, b, c)) in enumerate(zip(names, specs)):
        if mode not in (_lib.SCALE_DIV, _lib.SCALE_AFFINE, _lib.SCALE_CONST) or od not in (_lib.ANV_F32, _lib.ANV_F64) \
                or frame.column(n).anv_dtype not in _NP_OF_ANV or fl & ~_lib.SCALE_NAN_TO_NULL:
            raise ValueError("scale_columns: column %r: no scale mode %r to dtype %r with flags %r" % (n, mode, od, fl))
        sp[i] = (mode, od, fl, 0, a, b, c)
        t = torch.empty(max(padded, 4), dtype=getattr(torch, _TORCH_OF_ANV[od]), device="cuda")
        outs.append(t)
        ptrs[i] = t.data_ptr()
    n_words = (frame.n_rows + 31) // 32
    flagged = [bool(s[2] & _lib.SCALE_NAN_TO_NULL) for s in specs]
    words = torch.zeros((max(len(names), 1), max(n_words, 1)), dtype=torch.int32, device="cuda") if any(flagged) else None
    if not names or not frame.n_rows:
        return [t[:frame.n_rows] for t in outs], [None if words is None else words[i, :n_words] if f else None
                                                  for i, f in enumerate(flagged)], np.zeros(len(names), np.int64)
    nulls = _dev_bytes(len(names) * 8)
    desc, keep = frame.descriptors(names)
    nbytes = input_bytes(frame, names)
    if timer is not None:
        nbytes += sum(frame.n_rows * t.element_size() + (n_words * 4 if f else 0) for t, f in zip(outs, flagged))
    dspecs, dptrs = _to_dev(sp), _to_dev(ptrs)          # held until the launch is enqueued
    _call(L.anv_scale_columns, "anv_scale_columns", desc.data_ptr(), dspecs.data_ptr(), dptrs.data_ptr(),
          None if words is None else words.data_ptr(), nulls.data_ptr(), len(names), frame.n_rows, _stream(), nbytes=nbytes)
    launch_count += 1
    valid = [words[i, :n_words] if f else None for i, f in enumerate(flagged)]
    return [t[:frame.n_rows] for t in outs], valid, _host(nulls).view(np.int64)[:len(names)].copy()


# ---- feature transformation ----------------------------------------------------------------------

_TRANSFORM_SPEC_DT = np.dtype([("op", "<i4"), ("out_dtype", "<i4"), ("n", "<i8"), ("a", "<f8")])
_FLOATS = (_lib.ANV_F32, _lib.ANV_F64)


def transform_spec_ok(op, in_dtype, out_dtype, n):
    """The (op, input, output) combinations of the header's ANV_TF_* table."""
    if op in (_lib.TF_FLOOR, _lib.TF_CEIL, _lib.TF_FACTORIAL):
        return out_dtype == _lib.ANV_I64
    if op == _lib.TF_REMAINDER:
        return {_lib.ANV_F64: True, _lib.ANV_F32: in_dtype == _lib.ANV_F32, _lib.ANV_I32: in_dtype == _lib.ANV_I32 and n != 0,
                _lib.ANV_I64: in_dtype in (_lib.ANV_I32, _lib.ANV_I64) and n != 0}.get(out_dtype, False)
    if op == _lib.TF_ROUND:
        return out_dtype == in_dtype and (in_dtype not in _FLOATS or -22 <= n <= 22)
    return _lib.TF_LN <= op <= _lib.TF_MUL_INV and out_dtype == _lib.ANV_F64


def transform_columns(frame: ColumnFrame, names, specs):
    """anv_transform_columns: specs = one (op, out anv dtype, n, a) per name (_lib.TF_*).
    -> (list of CUDA tensors [n_rows] in the output dtype, list of int32 bitmap tensors [ceil(n_rows/32)] for the ops that
    make nulls (_lib.TF_MAKES_NULLS) and None for the others (which keep the source's validity), int64 ndarray of null
    counts)."""
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names, specs = list(names), list(specs)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: transform_columns(frame, names[lo:hi], specs[lo:hi]), len(names))
    sp = np.zeros(len(names), _TRANSFORM_SPEC_DT)
    outs, ptrs = [], np.zeros(len(names), np.uint64)
    padded = (frame.n_rows + 3) // 4 * 4
    for i, (n, (op, od, k, a)) in enumerate(zip(names, specs)):
        ind = frame.column(n).anv_dtype
        if ind not in _NP_OF_ANV or not transform_spec_ok(op, ind, od, k):
            raise ValueError("transform_columns: column %r: no op %r from dtype %r to %r with n = %r" % (n, op, ind, od, k))
        sp[i] = (op, od, k, a)
        t = torch.empty(max(padded, 4), dtype=getattr(torch, _TORCH_OF_ANV[od]), device="cuda")
        outs.append(t)
        ptrs[i] = t.data_ptr()
    n_words = (frame.n_rows + 31) // 32
    flagged = [s[0] in _lib.TF_MAKES_NULLS for s in specs]
    valid = [torch.zeros(max(n_words, 1), dtype=torch.int32, device="cuda")[:n_words] if f else None for f in flagged]
    vptrs = np.array([0 if v is None else v.data_ptr() for v in valid], np.uint64)
    if not names or not frame.n_rows:
        return [t[:frame.n_rows] for t in outs], valid, np.zeros(len(names), np.int64)
    nulls = _dev_bytes(len(names) * 8)
    desc, keep = frame.descriptors(names)
    nbytes = input_bytes(frame, names)
    if timer is not None:
        nbytes += sum(frame.n_rows * t.element_size() + (n_words * 4 if f else 0) for t, f in zip(outs, flagged))
    dspecs, dptrs = _to_dev(sp), _to_dev(ptrs)          # held until the launch is enqueued
    dvptrs = _to_dev(vptrs) if any(flagged) else None
    _call(L.anv_transform_columns, "anv_transform_columns", desc.data_ptr(), dspecs.data_ptr(), dptrs.data_ptr(),
          None if dvptrs is None else dvptrs.data_ptr(), nulls.data_ptr(), len(names), frame.n_rows, _stream(), nbytes=nbytes)
    launch_count += 1
    return [t[:frame.n_rows] for t in outs], valid, _host(nulls).view(np.int64)[:len(names)].copy()


def ks_candidates(frame: ColumnFrame, name, lambdas, n_null):
    """anv_ks_candidates on one column (values > 0 where valid, n_null null rows): -> (float64 ndarray of len(lambdas) + 1 statistics over the
    valid rows, for pow(x, lambda) then log(x); the count of valid values below 1)."""
    global launch_count
    _lib.require_cuda()
    L = _lib.lib()
    n = frame.n_rows
    desc, keep = frame.descriptors([name])
    lam = (C.c_double * max(len(lambdas), 1))(*[float(v) for v in lambdas])
    d_out, below = _dev_bytes(8 * (len(lambdas) + 1)), _dev_bytes(8)
    ws = _dev_bytes(L.anv_ks_candidates_workspace_bytes(n))
    _call(L.anv_ks_candidates, "anv_ks_candidates", desc.data_ptr(), 0, n, int(n_null), lam, len(lambdas),
          d_out.data_ptr(), below.data_ptr(), ws.data_ptr(), ws.numel(), _stream(), nbytes=input_bytes(frame, [name]))
    launch_count += 1
    return _host(d_out).view(np.float64)[:len(lambdas) + 1].copy(), int(_host(below).view(np.int64)[0])


# ---- categorical encoding ------------------------------------------------------------------------

_CODE_MAP_SPEC_DT = np.dtype([("size", "<i4"), ("out_dtype", "<i4"), ("table", "<u8"), ("table_valid", "<u8"),
                              ("out", "<u8"), ("out_valid", "<u8")])
_ONE_HOT_SPEC_DT = np.dtype([("size", "<i4"), ("k", "<i4"), ("index", "<u8"), ("out", "<u8"), ("stride", "<i8")])


def _tables_to_dev(arrays):
    """Host arrays -> one device buffer holding each at a 16-byte aligned offset; -> (buffer, device address of each)."""
    offs, pos = [], 0
    for a in arrays:
        offs.append(pos)
        pos += (a.nbytes + 15) // 16 * 16
    host = np.zeros(max(pos, 16), np.uint8)
    for a, o in zip(arrays, offs):
        host[o:o + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    dev = _to_dev(host)
    return dev, [dev.data_ptr() + o for o in offs]


def code_map(frame: ColumnFrame, names, tables, entry_valid):
    """anv_code_map: tables = per name, a host array of len(dictionary) + 1 entries (int32 or float64; the last is the null
    slot); entry_valid = per name, a bool array of the same length or None.
    -> (list of CUDA tensors [n_rows] in the table's dtype, list of int32 bitmap tensors [ceil(n_rows/32)] for the names
    with entry_valid and None for the others (which keep the source's validity), int64 ndarray of null counts)."""
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names, tables, entry_valid = list(names), list(tables), list(entry_valid)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: code_map(frame, names[lo:hi], tables[lo:hi], entry_valid[lo:hi]), len(names))
    n_words = (frame.n_rows + 31) // 32
    padded = max((frame.n_rows + 3) // 4 * 4, 4)
    host, outs, valid = [], [], []
    for n, t, ev in zip(names, tables, entry_valid):
        col = frame.column(n)
        size = len(col.dictionary) if col.dictionary is not None else -1
        if col.anv_dtype != _lib.ANV_I32 or size < 0 or t.dtype not in (np.int32, np.float64) or len(t) != size + 1 \
                or (ev is not None and len(ev) != size + 1):
            raise ValueError("code_map: column %r needs a string column and a table of its dictionary size + 1" % n)
        host.append(t)
        if ev is not None:
            host.append(np.packbits(np.asarray(ev, bool), bitorder="little"))
        outs.append(torch.empty(padded, dtype=torch.int32 if t.dtype == np.int32 else torch.float64, device="cuda"))
        valid.append(torch.zeros(max(n_words, 1), dtype=torch.int32, device="cuda") if ev is not None else None)
    if not names or not frame.n_rows:
        return [t[:frame.n_rows] for t in outs], [None if v is None else v[:n_words] for v in valid], \
            np.zeros(len(names), np.int64)
    buf, addr = _tables_to_dev(host)
    sp = np.zeros(len(names), _CODE_MAP_SPEC_DT)
    a = iter(addr)
    for i, (n, t, ev) in enumerate(zip(names, tables, entry_valid)):
        od = _lib.ANV_I32 if t.dtype == np.int32 else _lib.ANV_F64
        sp[i] = (len(t) - 1, od, next(a), next(a) if ev is not None else 0, outs[i].data_ptr(),
                 valid[i].data_ptr() if valid[i] is not None else 0)
    nulls = _dev_bytes(len(names) * 8)
    desc, keep = frame.descriptors(names)
    nbytes = input_bytes(frame, names)
    if timer is not None:
        nbytes += sum(frame.n_rows * t.element_size() + (n_words * 4 if v is not None else 0) for t, v in zip(outs, valid))
    dspecs = _to_dev(sp)                                # held until the launch is enqueued
    _call(L.anv_code_map, "anv_code_map", desc.data_ptr(), dspecs.data_ptr(), nulls.data_ptr(), len(names), frame.n_rows,
          _stream(), nbytes=nbytes)
    launch_count += 1
    return [t[:frame.n_rows] for t in outs], [None if v is None else v[:n_words] for v in valid], \
        _host(nulls).view(np.int64)[:len(names)].copy()


def one_hot_stride(n_rows):
    """Elements between the output columns of one_hot: n_rows rounded up to a multiple of 4 (16-byte aligned columns)."""
    return max((int(n_rows) + 3) // 4 * 4, 4)


def one_hot(frame: ColumnFrame, names, indexes, ks):
    """anv_one_hot: indexes = per name, a host int32 array of len(dictionary) + 1 entries (the last is the null slot) in
    [0, k); ks = output columns per name.  -> list of int32 CUDA tensors [k, n_rows], row j = (index == j), each row a
    16-byte aligned view of one [k, one_hot_stride(n_rows)] allocation."""
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names, indexes, ks = list(names), list(indexes), [int(k) for k in ks]
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: one_hot(frame, names[lo:hi], indexes[lo:hi], ks[lo:hi]), len(names))
    stride = one_hot_stride(frame.n_rows)
    outs = []
    for n, ix, k in zip(names, indexes, ks):
        col = frame.column(n)
        size = len(col.dictionary) if col.dictionary is not None else -1
        if col.anv_dtype != _lib.ANV_I32 or size < 0 or ix.dtype != np.int32 or len(ix) != size + 1 or k < 1:
            raise ValueError("one_hot: column %r needs a string column, an int32 index of its dictionary size + 1 and k >= 1"
                             % n)
        outs.append(torch.empty((k, stride), dtype=torch.int32, device="cuda"))
    if not names or not frame.n_rows:
        return [o[:, :frame.n_rows] for o in outs]
    buf, addr = _tables_to_dev(indexes)
    sp = np.zeros(len(names), _ONE_HOT_SPEC_DT)
    for i in range(len(names)):
        sp[i] = (len(indexes[i]) - 1, ks[i], addr[i], outs[i].data_ptr(), stride)
    desc, keep = frame.descriptors(names)
    nbytes = input_bytes(frame, names)
    if timer is not None:
        nbytes += sum(frame.n_rows * 4 * k for k in ks)
    dspecs = _to_dev(sp)
    _call(L.anv_one_hot, "anv_one_hot", desc.data_ptr(), dspecs.data_ptr(), len(names), frame.n_rows, _stream(),
          nbytes=nbytes)
    launch_count += 1
    return [o[:, :frame.n_rows] for o in outs]


# ---- table membership (invalidEntries_detection) --------------------------------------------------

_FLAG_SPEC_DT = np.dtype([("keys", "<u8"), ("n_keys", "<i8"), ("counts", "<u8"), ("out_valid", "<u8")])


def flag_smem_keys() -> int:
    """Largest table anv_flag_members searches in shared memory (larger ones are searched in global memory)."""
    return int(_lib.lib().anv_flag_members_smem_keys())


def flag_members(frame: ColumnFrame, names, tables, want_bitmap):
    """anv_flag_members: tables = per name, a host array of the column's own dtype (int32 codes for string columns) holding
    distinct values in ascending key order (shared/invalid_rules.sort_table).  A valid row holding a table value is a hit.
    -> (list of uint64 ndarrays of per-entry row counts, list of int32 bitmap tensors [ceil(n_rows/32)] with the hits
    nulled, or None where want_bitmap is False or the table is empty: an empty table is never launched and leaves the
    column's own validity)."""
    if getattr(frame, "is_partitioned", False):
        if want_bitmap:
            raise ValueError("flag_members: a row-partitioned frame counts only; map_chunks gives the treated chunks")
        return frame.flag_members(list(names), list(tables)), [None] * len(list(names))
    from .shared.invalid_rules import ordered_keys
    global launch_count
    torch = _lib.require_cuda()
    L = _lib.lib()
    names, tables = list(names), list(tables)
    if len(names) > _lib.MAX_LAUNCH_COLS:
        return _in_column_blocks(lambda lo, hi: flag_members(frame, names[lo:hi], tables[lo:hi], want_bitmap), len(names))
    n_words = (frame.n_rows + 31) // 32
    keys = []
    for n, t in zip(names, tables):
        col = frame.column(n)
        want = _NP_OF_ANV.get(col.anv_dtype)
        if want is None or np.asarray(t).dtype != want:
            raise ValueError("flag_members: column %r needs a table of %s values" % (n, want))
        k = ordered_keys(np.asarray(t))
        if len(k) > 1 and not bool(np.all(k[1:] > k[:-1])):
            raise ValueError("flag_members: the table of column %r is not distinct values in key order" % n)
        keys.append(k)
    launch = [i for i, k in enumerate(keys) if len(k) and frame.n_rows]
    counts = [np.zeros(len(k), np.uint64) for k in keys]
    valid = [None] * len(names)
    if not launch:
        return counts, valid
    if want_bitmap:
        for i in launch:
            valid[i] = torch.empty(max(n_words, 1), dtype=torch.int32, device="cuda")
    offs = np.cumsum([0] + [len(keys[i]) for i in launch])
    dcounts = torch.zeros(max(int(offs[-1]), 1), dtype=torch.int64, device="cuda")
    buf, addr = _tables_to_dev([keys[i] for i in launch])
    sp = np.zeros(len(launch), _FLAG_SPEC_DT)
    for j, i in enumerate(launch):
        sp[j] = (addr[j], len(keys[i]), dcounts.data_ptr() + 8 * int(offs[j]),
                 valid[i].data_ptr() if valid[i] is not None else 0)
    lnames = [names[i] for i in launch]
    desc, keep = frame.descriptors(lnames)
    nbytes = input_bytes(frame, lnames)
    if timer is not None and want_bitmap:
        nbytes += len(launch) * n_words * 4
    dspecs = _to_dev(sp)                                # held until the launch is enqueued
    _call(L.anv_flag_members, "anv_flag_members", desc.data_ptr(), dspecs.data_ptr(), len(launch), frame.n_rows, _stream(),
          nbytes=nbytes)
    launch_count += 1
    flat = _host(dcounts).view(np.uint64)
    for j, i in enumerate(launch):
        counts[i] = flat[offs[j]:offs[j + 1]].copy()
    return counts, [None if v is None else v[:n_words] for v in valid]
