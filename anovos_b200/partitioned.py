"""Row-partitioned frames (SURVEY.md 8(e) "row-sharded variant", BASELINE.json configs C4/C5).

A `PartitionedFrame` is a frame whose ROWS are split into partitions: row chunks streamed one
after the other through this GPU (a frame larger than HBM, or a host table uploaded chunk by
chunk with the next chunk's H2D copy in flight), and / or row slabs held by the other ranks of
a torch.distributed group.  Every pass of the hot path has an exact merge over row partitions:

  moments           Pebay/Chan merge of (n, mean, M2, M3, M4) in partition order (chunks, then
                    ranks) + integer sums + min/max              -> one all_gather of 64 B/column
  histograms        integer sums of the per-partition counts     -> one all_reduce(sum)
  HLL++ registers   element-wise max                             -> one all_reduce(max)
  exact percentiles the radix select one pass at a time: every partition adds its digit
                    histogram (anv_select_accumulate), then ONE all_reduce(sum) of the uint64
                    histogram region in device memory per refinement round (anv_select_advance
                    afterwards takes the same decision on every rank)

so the data itself never moves between GPUs.  Equal-range binning is the 2-step protocol the
survey names: pass 1 merges min/max, the cutoffs are computed on the host (identically on every
rank), pass 2 histograms every partition against them.  The reference functions
(stats_generator, attribute_binning, drift statistics) accept a PartitionedFrame wherever they
accept a frame.  The exact mode / exact distinct count of NUMERIC columns needs a global group-by,
the one thing row partitions cannot merge: there the partitions are turned into whole columns
first - local chunks are concatenated on the device, row slabs are exchanged with
`repartition_to_columns` (all-to-all over NVLink, every rank ends up with whole columns of its
block), each rank sorts its block and the per-column results are all-gathered.
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np

from . import _lib
from .frame import ColumnFrame


# ---- merge operators (host, deterministic) ------------------------------------------------------

def merge_moments(parts):
    """Merge per-partition moment records (engine._MOM_DT arrays, one row per column) in the order
    given.  The same algebra as the device-side tile merge (csrc/common.cuh merge_central) and as
    Spark's CentralMomentAgg.merge; min/max follow Spark's NaN-is-largest ordering, except that a partition of
    nothing but NaN (min = max = NaN, as finalize_moments reports it) adds no extrema: a frame split into row
    partitions then has the extrema of the same frame held whole.  Both sides all-NaN give NaN."""
    acc = np.array(parts[0], copy=True)
    for b in parts[1:]:
        a = acc
        na, nb = a["n_valid"].astype(np.float64), b["n_valid"].astype(np.float64)
        both, only_b = (na > 0) & (nb > 0), (na == 0) & (nb > 0)
        with np.errstate(all="ignore"):
            n = na + nb
            d = b["mean"] - a["mean"]
            dn = d / n
            dn2 = dn * dn
            ab = na * nb
            mean = a["mean"] + dn * nb
            m2 = a["m2"] + b["m2"] + d * dn * ab
            m3 = a["m3"] + b["m3"] + d * dn2 * ab * (na - nb) + 3.0 * dn * (na * b["m2"] - nb * a["m2"])
            m4 = (a["m4"] + b["m4"] + d * dn * dn2 * ab * (na * na - ab + nb * nb)
                  + 6.0 * dn2 * (na * na * b["m2"] + nb * nb * a["m2"]) + 4.0 * dn * (na * b["m3"] - nb * a["m3"]))
            mn = np.fmin(a["min"], b["min"])           # NaN only when both sides are all-NaN
            mx = np.maximum(a["max"], b["max"])        # NaN (largest in Spark's order) propagates
            a_nan, b_nan = np.isnan(a["min"]) & np.isnan(a["max"]), np.isnan(b["min"]) & np.isnan(b["max"])
            mx = np.where(a_nan, b["max"], np.where(b_nan, a["max"], mx))   # all-NaN partitions add no extrema
        out = np.array(a, copy=True)
        for f, v in (("mean", mean), ("m2", m2), ("m3", m3), ("m4", m4), ("min", mn), ("max", mx)):
            out[f] = np.where(both, v, np.where(only_b, b[f], a[f]))
        out["n_valid"] = a["n_valid"] + b["n_valid"]
        out["n_nonzero"] = a["n_nonzero"] + b["n_nonzero"]
        acc = out
    return acc


# ---- collectives over the row slabs of a group ----------------------------------------------------

class _Group:
    """Thin wrapper: numpy in / numpy out collectives on the group's backend device."""

    def __init__(self, group):
        import torch.distributed as dist
        self.dist = dist
        self.group = None if group is True else group
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.device = "cuda" if dist.get_backend(self.group) == "nccl" else "cpu"

    def all_reduce(self, arr: np.ndarray, op="sum"):
        import torch
        signed = arr.view(np.int64) if arr.dtype == np.uint64 else (arr.astype(np.int64) if arr.dtype == np.uint32 else arr)
        t = torch.from_numpy(np.ascontiguousarray(signed)).to(self.device)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM if op == "sum" else self.dist.ReduceOp.MAX, group=self.group)
        out = t.cpu().numpy()
        return out.view(np.uint64) if arr.dtype == np.uint64 else out.astype(arr.dtype)

    def all_reduce_device(self, t):
        """In-place sum of a DEVICE tensor: NCCL reduces it where it lies (NVLink / NVSwitch); a
        gloo group (CPU tests, or several ranks sharing one GPU) stages it through the host."""
        if self.device == "cuda":
            self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM, group=self.group)
        else:
            h = t.cpu()
            self.dist.all_reduce(h, op=self.dist.ReduceOp.SUM, group=self.group)
            t.copy_(h)

    def all_gather_records(self, rec: np.ndarray):
        import torch
        t = torch.from_numpy(np.ascontiguousarray(rec).view(np.uint8).reshape(-1).copy()).to(self.device)
        out = [torch.empty_like(t) for _ in range(self.world)]
        self.dist.all_gather(out, t, group=self.group)
        return [o.cpu().numpy().view(rec.dtype) for o in out]


def _side_stream():
    """The device's persistent side stream (frame.side_stream); the CPU engine stand-in of the tests has no streams."""
    from . import frame as _frame
    return _frame.side_stream()


class PartitionedFrame:
    """Frame-like object over row partitions.  `schema` is a ColumnFrame (any row count, usually
    the first chunk or an empty frame) that supplies column names, dtypes and dictionaries;
    `chunk_fn(i)` returns the ColumnFrame of local chunk i (it may re-create the chunk on every
    call - a pass calls it once per chunk); `group` (True = default group) adds the row slabs of
    the other ranks.  String columns must use the SAME dictionary in every partition."""

    is_partitioned = True

    spark_partitions = False   # True: the chunks ARE the partitions Spark would scan (see gk_quantiles)

    def __init__(self, schema: ColumnFrame, chunk_rows, chunk_fn, group=None, release=True):
        self._schema = schema
        self.chunk_rows = [int(r) for r in chunk_rows]
        self._chunk_fn = chunk_fn
        self._release = release
        self._cache = {}
        self.group = _Group(group) if group is not None and group is not False else None
        self.n_rows_local = sum(self.chunk_rows)
        self.n_rows = self.n_rows_local
        if self.group is not None:
            self.n_rows = int(self.group.all_reduce(np.array([self.n_rows_local], np.int64))[0])
        self.passes = 0  # full reads of the local partitions so far (reported by the bench)

    # ---- constructors ---------------------------------------------------------------------------
    @staticmethod
    def from_frames(frames, group=None) -> "PartitionedFrame":
        frames = list(frames)
        return PartitionedFrame(frames[0], [f.n_rows for f in frames], lambda i: frames[i], group=group, release=False)

    @staticmethod
    def from_frame(frame, chunk_rows: int, group=None) -> "PartitionedFrame":
        """Row chunks of a (host- or device-resident) frame / pyarrow table / pandas frame.
        Host-resident chunks are uploaded while the previous chunk is being processed and freed
        afterwards, so device memory holds two chunks, not the frame."""
        from .frame import as_frame
        fr = as_frame(frame)
        chunk_rows = max(32, int(chunk_rows) // 32 * 32)
        starts = list(range(0, fr.n_rows, chunk_rows)) or [0]
        return PartitionedFrame(fr.slice_rows(0, 0), [min(chunk_rows, fr.n_rows - s) for s in starts],
                                lambda i: fr.slice_rows(starts[i], starts[i] + chunk_rows), group=group)

    @staticmethod
    def from_arrow_partitions(table, rows_per_partition, spark=True) -> "PartitionedFrame":
        """A pyarrow table cut into the row ranges Spark scanned as partitions (in order).  String columns are
        dictionary-encoded once so that every partition shares the dictionary."""
        import pyarrow as pa
        import pyarrow.compute as pc
        rows = [int(k) for k in rows_per_partition]
        if sum(rows) != table.num_rows:
            raise ValueError("rows_per_partition does not add up to the table's rows")
        cols = []
        for f in table.schema:
            c = table.column(f.name)
            if pa.types.is_string(f.type) or pa.types.is_large_string(f.type):
                c = pc.dictionary_encode(c.combine_chunks())
            cols.append(c)
        table = pa.table(cols, names=table.column_names)
        frames, r0 = [], 0
        for k in rows:
            frames.append(ColumnFrame.from_arrow(table.slice(r0, k)))
            r0 += k
        out = PartitionedFrame(frames[0], rows, lambda i: frames[i], release=True)
        out.spark_partitions = bool(spark)
        return out

    # ---- Spark-DataFrame-like surface -----------------------------------------------------------
    @property
    def columns(self):
        return self._schema.columns

    @property
    def dtypes(self):
        return self._schema.dtypes

    @property
    def n_chunks(self):
        return len(self.chunk_rows)

    def count(self):
        return self.n_rows

    def column(self, name):
        return self._schema.column(name)

    def __contains__(self, name):
        return name in self._schema

    def _project(self, schema, fn):
        out = PartitionedFrame.__new__(PartitionedFrame)
        out.__dict__.update(self.__dict__)
        out._schema, out._chunk_fn, out._cache, out.passes = schema, fn, {}, 0
        return out

    def select(self, names):
        names = [names] if isinstance(names, str) else list(names)
        base = self._chunk_fn
        return self._project(self._schema.select(names), lambda i: base(i).select(names))

    def drop(self, *names):
        names = set(names[0]) if len(names) == 1 and isinstance(names[0], (list, tuple, set)) else set(names)
        return self.select([c for c in self.columns if c not in names])

    def map_chunks(self, schema, fn):
        """Lazy per-chunk transform (e.g. attribute_binning with a fixed model)."""
        base = self._chunk_fn
        return self._project(schema, lambda i: fn(base(i)))

    def dropna(self, subset=None):
        raise NotImplementedError("dropna is not defined on a row-partitioned frame; filter the chunks instead")

    def descriptors(self, names):
        raise _lib.AnvError("a PartitionedFrame has no single device image; kernels run per chunk")

    # ---- chunk iteration with the next chunk's H2D copy in flight ---------------------------------
    def chunks(self, names=None):
        torch = _lib.require_cuda()
        self.passes += 1
        copy = None
        nxt = self._chunk_fn(0) if self.n_chunks else None
        for i in range(self.n_chunks):
            cur = nxt
            nxt = None
            if i + 1 < self.n_chunks:
                nxt = self._chunk_fn(i + 1)
                for n in (names or nxt.columns):
                    c = nxt.column(n)
                    if c.kind == "other" or c._dev is not None:
                        continue
                    if c._host is not None:
                        if copy is None:
                            copy = _side_stream()
                        c.upload_async(copy)
                    elif c._loader is not None:
                        # generated chunks (synthetic frames): run the generator of chunk i+1 on the side stream while the
                        # scan kernels of chunk i run - the generator is ALU-bound, the scans HBM-bound
                        if copy is None:
                            copy = _side_stream()
                        c.generate_async(copy)
            yield cur
            if self._release:
                for n in cur.columns:
                    cur.column(n).drop_device()
            del cur

    # ---- merged passes (called by engine.* when handed a PartitionedFrame) -----------------------
    def moments(self, names):
        from . import engine
        names = list(names)
        parts = [engine.moments(ch, names) for ch in self.chunks(names)]
        acc = merge_moments(parts) if parts else np.zeros(len(names), dtype=engine._MOM_DT)
        if self.group is not None:
            acc = merge_moments(self.group.all_gather_records(acc))
        return acc

    def histogram(self, model):
        from . import engine
        acc = None
        for ch in self.chunks(model.names):
            h = engine.histogram(ch, model)
            acc = h if acc is None else acc + h
        if acc is None:
            acc = np.zeros((len(model.names), model.max_bins + 1), np.uint64)
        return self.group.all_reduce(acc) if self.group is not None else acc

    def moments_histogram(self, model):
        from . import engine
        parts, acc = [], None
        for ch in self.chunks(model.names):
            m, h = engine.moments_histogram(ch, model)
            parts.append(m)
            acc = h if acc is None else acc + h
        mom = merge_moments(parts) if parts else np.zeros(len(model.names), dtype=engine._MOM_DT)
        if acc is None:
            acc = np.zeros((len(model.names), model.max_bins + 1), np.uint64)
        if self.group is not None:
            mom = merge_moments(self.group.all_gather_records(mom))
            acc = self.group.all_reduce(acc)
        return mom, acc

    def code_counts(self, names):
        from . import engine
        names = list(names)
        acc = None
        for ch in self.chunks(names):
            h = engine.code_counts(ch, names)
            acc = h if acc is None else [a + b for a, b in zip(acc, h)]
        if acc is None:
            acc = [np.zeros(max(len(self.column(n).dictionary), 1) + 1, np.uint64) for n in names]
        if self.group is not None and names:
            flat = self.group.all_reduce(np.concatenate(acc))
            offs = np.cumsum([0] + [len(a) for a in acc])
            acc = [flat[offs[i]:offs[i + 1]] for i in range(len(acc))]
        return acc

    def flag_members(self, names, tables):
        """Per-entry row counts of engine.flag_members summed over the chunks and, for row slabs, over the ranks (one
        all_reduce).  The treated chunks come from map_chunks with engine.flag_members per chunk."""
        from . import engine
        names, tables = list(names), list(tables)
        acc = [np.zeros(len(t), np.uint64) for t in tables]
        for ch in self.chunks(names):
            counts, _ = engine.flag_members(ch, names, tables, False)
            acc = [a + c for a, c in zip(acc, counts)]
        if self.group is not None and names:
            flat = self.group.all_reduce(np.concatenate(acc + [np.zeros(1, np.uint64)]))
            offs = np.cumsum([0] + [len(a) for a in acc])
            acc = [flat[offs[i]:offs[i + 1]].copy() for i in range(len(acc))]
        return acc

    def hll_registers(self, names, p):
        from . import engine
        names = list(names)
        acc = np.zeros((len(names), 1 << p), np.uint32)
        for ch in self.chunks(names):
            np.maximum(acc, engine.hll_registers(ch, names, p), out=acc)
        return self.group.all_reduce(acc, op="max") if self.group is not None else acc

    def select_ranks(self, names, ranks):
        """Exact order statistics at global 1-based `ranks` [n_cols, n_ranks]: one read of every
        partition and one all_reduce per radix pass."""
        import ctypes as C
        from . import engine
        torch = _lib.require_cuda()
        L = _lib.lib()
        names = list(names)
        ranks = np.ascontiguousarray(ranks, dtype=np.int64).reshape(len(names), -1)
        if len(names) > _lib.MAX_LAUNCH_COLS:
            return engine._in_column_blocks(lambda lo, hi: self.select_ranks(names[lo:hi], ranks[lo:hi]), len(names))
        out = np.full(ranks.shape, np.nan, np.float64)
        if not names or ranks.shape[1] == 0:
            return out
        groups = {}
        for i, nme in enumerate(names):
            kb = 32 if self.column(nme).anv_dtype in (_lib.ANV_F32, _lib.ANV_I32) else 64
            groups.setdefault(kb, []).append(i)
        for kb, idx in groups.items():
            grp = [names[i] for i in idx]
            for r0 in range(0, ranks.shape[1], 16):
                rk = np.ascontiguousarray(ranks[idx, r0:r0 + 16])
                nr = rk.shape[1]
                ws_bytes = L.anv_select_workspace_bytes(len(grp), nr)
                ws = engine._dev_bytes(ws_bytes)
                drk = engine._to_dev(rk)
                dout = engine._dev_bytes(rk.size * 8)
                engine._call(L.anv_select_begin, "anv_select_begin", len(grp), nr, ws.data_ptr(), ws_bytes, engine._stream())
                sdesc = None
                for ps in range(L.anv_select_passes(kb)):
                    for ch in self.chunks(grp):
                        desc, keep = ch.descriptors(grp)
                        sdesc = (desc, keep) if sdesc is None else sdesc
                        engine._call(L.anv_select_accumulate, "anv_select_accumulate", desc.data_ptr(), len(grp), ch.n_rows, nr, kb,
                                     ps, ws.data_ptr(), ws_bytes, engine._stream())
                        engine.launch_count += 1
                        torch.cuda.current_stream().synchronize()   # the chunk may be released / re-created next
                    if self.group is not None:
                        off, nb = C.c_size_t(), C.c_size_t()
                        _lib.check(L.anv_select_hist_region(len(grp), nr, ps, C.byref(off), C.byref(nb)), "anv_select_hist_region")
                        self.group.all_reduce_device(ws[off.value:off.value + nb.value].view(torch.int64))
                    d0 = sdesc[0] if sdesc is not None else self._schema.descriptors(grp)[0]
                    engine._call(L.anv_select_advance, "anv_select_advance", d0.data_ptr(), len(grp), drk.data_ptr(), nr, kb, ps,
                                 dout.data_ptr(), ws.data_ptr(), ws_bytes, engine._stream())
                    engine.launch_count += 1
                out[np.asarray(idx)[:, None], np.arange(r0, r0 + nr)[None, :]] = \
                    engine._host(dout).view(np.float64)[:rk.size].reshape(rk.shape)
        return out

    def bin_assign(self, model):
        raise NotImplementedError("bin ids of a row-partitioned frame are produced per chunk: use attribute_binning(), "
                                  "which returns a PartitionedFrame")

    def gk_quantiles(self, names, probs, eps):
        """Spark-partitioned frames (`spark_partitions=True`: every chunk is one Spark partition, in order): the
        quantiles Dataset.summary() / approxQuantile return - one Greenwald-Khanna sketch per partition, merged in
        partition order (shared/gk.py).  A partition of fewer than 50 000 non-null values keeps the order statistics at
        data-independent positions, so the sort kernel supplies just those few thousand samples.  A LARGER partition makes
        Spark flush its 50 000-value head buffer as the rows arrive: every batch of 50 000 consecutive non-null values is
        sorted on the device (one "column" per batch) and the strictly sequential merge / compress runs in the library's
        host helper (anv_gk_partition_sketch).  -> dict name -> [value | None per prob]."""
        from . import engine
        from .shared import gk
        names = [n for n in names]
        sketch = {n: ([], 0) for n in names}
        for ch in self.chunks(names):
            mom = engine.moments(ch, names)
            nv = [int(m["n_valid"]) for m in mom]
            small = [i for i, k in enumerate(nv) if k < gk.HEAD_SIZE]
            if small:
                sub = [names[i] for i in small]
                pos = [gk.sample_positions(nv[i], eps) for i in small]
                width = max((len(q) for q in pos), default=0)
                if width:
                    rk = np.zeros((len(sub), width), np.int64)
                    for j, q in enumerate(pos):
                        rk[j, :len(q)] = q + 1
                    _, vals = engine.sort_mode_distinct(ch, sub, rk)
                    for j, i in enumerate(small):
                        s = gk.partition_samples(vals[j, :len(pos[j])], nv[i], eps)
                        sketch[names[i]] = gk.merge_samples(sketch[names[i]][0], sketch[names[i]][1], s, nv[i], eps)
            for i, k in enumerate(nv):
                if k >= gk.HEAD_SIZE:
                    s = _large_partition_sketch(ch, names[i], k, eps)
                    sketch[names[i]] = gk.merge_samples(sketch[names[i]][0], sketch[names[i]][1], s, k, eps)
        return {n: [gk.query_samples(sketch[n][0], sketch[n][1], eps, p) for p in probs] for n in names}

    def materialize(self, names=None) -> ColumnFrame:
        """Concatenate the local chunks of `names` into one device-resident ColumnFrame (for the passes that need
        whole columns - the exact mode / distinct count sort).  Only sensible when the columns fit in HBM."""
        torch = _lib.require_cuda()
        from .frame import Column, pack_bits_device
        names = [n for n in (names or self.columns) if self.column(n).kind != "other"]
        data = {n: [] for n in names}
        valid = {n: [] for n in names}
        any_null = {n: False for n in names}
        for ch in self.chunks(names):
            for n in names:
                d, v = ch.column(n).device()
                data[n].append(d)
                valid[n].append(ch.valid_mask(n))
                any_null[n] |= v is not None
        out = OrderedDict()
        for n in names:
            c = self.column(n)
            d = torch.cat(data[n]) if data[n] else torch.empty(0, device="cuda")
            v = pack_bits_device(torch.cat(valid[n])) if any_null[n] else None
            out[n] = Column(n, c.sdtype, self.n_rows_local, dev=d, dev_valid=v, anv_dtype=c.anv_dtype, dictionary=c.dictionary)
        return ColumnFrame(out, self.n_rows_local)

    def sort_mode_distinct(self, names, ranks=None):
        """Exact mode / distinct count of numeric columns needs whole columns.  Local chunks are concatenated on the
        device; row slabs on several ranks are first exchanged (repartition_to_columns: every rank receives whole
        columns of its block over NVLink), each rank sorts its block and the small per-column results are
        all-gathered, so every rank returns the full answer."""
        from . import engine
        engine.refuse_exact_rows(self.n_rows, "sort_mode_distinct")     # before anything is materialized
        torch = _lib.require_cuda()
        names = list(names)
        need = sum(self.n_rows * (8 if self.column(n).anv_dtype in (_lib.ANV_F64, _lib.ANV_I64) else 4) for n in names)
        if 3 * need // (self.group.world if self.group is not None else 1) > torch.cuda.mem_get_info()[0]:
            raise NotImplementedError(
                "exact mode / exact distinct count of numeric columns needs whole columns in HBM, which this frame "
                "does not fit: use the approximate distinct count (HLL++) or fewer columns per call")
        local = self.materialize(names)
        if self.group is None:
            return engine.sort_mode_distinct(local, names, ranks)
        if self.group.group is not None:
            raise NotImplementedError("row-slab exchange is implemented on the default process group only")
        from . import parallel
        block = repartition_to_columns(local, True, names)
        del local
        mine = block.columns
        n_ranks = 0 if ranks is None else np.asarray(ranks).reshape(len(names), -1).shape[1]
        rk = None if ranks is None else np.asarray(ranks, dtype=np.int64).reshape(len(names), -1)[[names.index(n) for n in mine]]
        # [mode of a bigint column | mode_rows (-1: no value) | n_distinct] as int64, so a bigint mode stays exact;
        # [mode of any other column | rank values] as float64
        imat = np.zeros((len(mine), 3), np.int64)
        fmat = np.full((len(mine), 1 + n_ranks), np.nan, np.float64)
        if mine:
            res = engine.sort_mode_distinct(block, mine, rk)
            modes, rvals = res if ranks is not None else (res, None)
            for i, (mv, mr, nd) in enumerate(modes):
                imat[i] = (mv if isinstance(mv, int) else 0, -1 if mr is None else mr, nd)
                if isinstance(mv, float):
                    fmat[i, 0] = mv
            if n_ranks:
                fmat[:, 1:] = rvals
        dev = "cuda" if self.group.device == "cuda" else None
        ifull = np.concatenate(parallel.gather_summaries(imat, device=dev))
        ffull = np.concatenate(parallel.gather_summaries(fmat, device=dev))
        order = [n for r in range(self.group.world) for n in parallel.shard_columns(names, r, self.group.world)]
        at = {n: i for i, n in enumerate(order)}
        out = []
        for n in names:
            mv, mr, nd = (int(x) for x in ifull[at[n]])
            if mr < 0:
                out.append((None, None, 0))
            else:
                out.append((mv if self.column(n).anv_dtype == _lib.ANV_I64 else float(ffull[at[n], 0]), mr, nd))
        if ranks is None:
            return out
        return out, np.array([ffull[at[n], 1:] for n in names], dtype=np.float64).reshape(len(names), n_ranks)


# ---- row slabs -> column blocks (the one real exchange step) ---------------------------------------

def _large_partition_sketch(ch: ColumnFrame, name: str, n_valid: int, eps: float, batches_per_call: int = 128):
    """Spark's sketch of ONE partition with >= 50 000 non-null values of column `name` -> [(value, g, delta)].
    Device: the non-null values in arrival order, cut into head-buffer batches of 50 000; each batch goes through the
    radix sort as one column and comes back fully ordered through its rank outputs.  Host: anv_gk_partition_sketch."""
    import ctypes as C
    from . import engine
    from .shared import gk
    L = _lib.lib()
    H = gk.HEAD_SIZE
    d, v = ch.column(name).device()
    vals = d if v is None else d[ch.valid_mask(name)]          # arrival order, nulls dropped (a gather: plumbing)
    n = int(vals.shape[0])
    assert n == n_valid, (n, n_valid)
    parts = []
    nb, rem = n // H, n % H
    full_ranks = np.arange(1, H + 1, dtype=np.int64)
    for b0 in range(0, nb, batches_per_call):
        b1 = min(nb, b0 + batches_per_call)
        cols = {"b%06d" % j: vals[j * H:(j + 1) * H] for j in range(b0, b1)}
        bf = ColumnFrame.from_tensors(cols, n_rows=H)
        _, sv = engine.sort_mode_distinct(bf, list(cols), np.tile(full_ranks, (b1 - b0, 1)))
        parts.append(np.ascontiguousarray(sv, dtype=np.float64).reshape(-1))
    if rem:
        bf = ColumnFrame.from_tensors({"rest": vals[nb * H:]}, n_rows=rem)
        _, sv = engine.sort_mode_distinct(bf, ["rest"], np.arange(1, rem + 1, dtype=np.int64).reshape(1, -1))
        parts.append(np.ascontiguousarray(sv, dtype=np.float64).reshape(-1))
    sb = np.concatenate(parts) if parts else np.zeros(0)
    cap = n + 8
    ov, og, od = np.zeros(cap), np.zeros(cap, np.int64), np.zeros(cap, np.int64)
    k = L.anv_gk_partition_sketch(sb.ctypes.data_as(C.c_void_p), n, H, float(eps), gk.COMPRESS_THRESHOLD, ov.ctypes.data_as(C.c_void_p),
                                  og.ctypes.data_as(C.c_void_p), od.ctypes.data_as(C.c_void_p), cap)
    if k < 0:
        _lib.check(int(k), "anv_gk_partition_sketch")
    return list(zip(ov[:k].tolist(), og[:k].tolist(), od[:k].tolist()))


def repartition_to_columns(frame: ColumnFrame, group=True, names=None) -> ColumnFrame:
    """All-to-all over the group (NCCL over NVLink on GPUs): every rank holds a row slab of ALL
    columns on entry and whole columns of ITS contiguous column block (parallel.shard_columns) on
    exit, after which the column-sharded path applies with no further exchange.  Slabs are
    concatenated in rank order; every slab except the last must have a multiple of 32 rows so the
    validity bitmaps concatenate on word boundaries."""
    import torch
    import torch.distributed as dist
    from .frame import Column
    from .parallel import shard_columns
    pg = None if group is True else group
    world, rank = dist.get_world_size(pg), dist.get_rank(pg)
    on_gpu = dist.get_backend(pg) == "nccl"
    dev = "cuda" if on_gpu else "cpu"
    names = [n for n in (names or frame.columns) if frame.column(n).kind != "other"]
    rows = torch.tensor([frame.n_rows], dtype=torch.int64, device=dev)
    all_rows = [torch.zeros_like(rows) for _ in range(world)]
    dist.all_gather(all_rows, rows, group=pg)
    slab = [int(r.item()) for r in all_rows]
    if any(r % 32 for r in slab[:-1]):
        raise ValueError("repartition_to_columns: every row slab except the last needs a multiple of 32 rows")
    total = sum(slab)
    words = [(r + 31) // 32 for r in slab]
    # which columns carry a validity bitmap anywhere in the group (a slab without nulls sends all-ones)
    has_v = torch.tensor([1 if frame.column(n).has_validity else 0 for n in names], dtype=torch.int32, device=dev)
    dist.all_reduce(has_v, op=dist.ReduceOp.MAX, group=pg)
    has_v = has_v.cpu().tolist()
    owner = {}
    for r in range(world):
        for n in shard_columns(names, r, world):
            owner[n] = r
    mine = shard_columns(names, rank, world)

    def local(n):
        c = frame.column(n)
        if on_gpu:
            return c.device()
        if c._host is None:  # device-resident frame on a gloo group: stage through the host
            d, v = c.device()
            return d.cpu(), (v.cpu() if v is not None else None)
        h = c._host if c.dictionary is None else np.asarray(c._host).astype(np.int32, copy=False)   # narrow host codes
        return (torch.from_numpy(np.ascontiguousarray(h)),
                torch.from_numpy(np.ascontiguousarray(c._host_valid)) if c._host_valid is not None else None)

    # grouped point-to-point transfers (NCCL fuses the batch into one all-to-all over NVLink; gloo,
    # which has no alltoall, runs them as plain sends): slab column -> its owner, in rank order
    peer = (lambda r: r) if pg is None else (lambda r: dist.get_global_rank(pg, r))
    ops, recv = [], {}
    for ci, n in enumerate(names):
        d, v = local(n)
        o = owner[n]
        if has_v[ci]:
            if v is None:
                v = torch.full((words[rank],), -1, dtype=torch.int32, device=dev)
            elif v.dtype != torch.int32:
                v = v.view(torch.int32)
        else:
            v = None
        if o == rank:
            rd = [d if r == rank else torch.empty(slab[r], dtype=d.dtype, device=dev) for r in range(world)]
            rv = None if v is None else [v if r == rank else torch.empty(words[r], dtype=torch.int32, device=dev)
                                         for r in range(world)]
            for r in range(world):
                if r != rank and slab[r]:
                    ops.append(dist.P2POp(dist.irecv, rd[r], peer(r), group=pg))
                    if rv is not None:
                        ops.append(dist.P2POp(dist.irecv, rv[r], peer(r), group=pg))
            recv[n] = (rd, rv)
        elif slab[rank]:
            ops.append(dist.P2POp(dist.isend, d.contiguous(), peer(o), group=pg))
            if v is not None:
                ops.append(dist.P2POp(dist.isend, v.contiguous(), peer(o), group=pg))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    out = OrderedDict()
    for n in mine:
        c = frame.column(n)
        rd, rv = recv[n]
        data = torch.cat(rd)
        valid = torch.cat(rv)[:(total + 31) // 32] if rv is not None else None
        if on_gpu:
            out[n] = Column(n, c.sdtype, total, dev=data, dev_valid=valid, anv_dtype=c.anv_dtype, dictionary=c.dictionary)
        else:
            out[n] = Column(n, c.sdtype, total, host=data.numpy(), host_valid=valid.numpy() if valid is not None else None,
                            anv_dtype=c.anv_dtype, dictionary=c.dictionary)
    return ColumnFrame(OrderedDict((n, out[n]) for n in mine), total)
