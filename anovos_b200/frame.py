"""Columnar frame: the `idf` of the GPU path.

The reference passes Spark DataFrames (`idf`) into every function of the hot path;
here `idf` is a ColumnFrame: column-major device buffers (one contiguous torch CUDA
tensor per column + optional Arrow validity bitmap), dictionary codes for string
columns, and the Spark dtype string of every column so that
`attributeType_segregation` (reference shared/utils.py:48-73) behaves identically.

`as_frame(x)` accepts a ColumnFrame, a pyarrow Table, a pandas DataFrame or a dict of
torch tensors / numpy arrays.
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np

from . import _lib

_NUMERIC_SPARK = ("double", "int", "bigint", "float", "long")

h2d_bytes = 0  # bytes uploaded to the device by Column.device()

_SIDE_STREAMS = {}


def side_stream():
    """ONE side stream per device for asynchronous uploads / chunk generation.  torch's caching allocator keeps a pool per
    stream: a fresh stream per pass would cudaMalloc every chunk again (measured: the streamed c4 step went from 0.36 s to 1.3 s)."""
    torch = _lib.require_cuda()
    if not hasattr(torch.cuda, "current_device"):      # the CPU engine stand-in of the tests: no streams
        return torch.cuda.Stream()
    dev = torch.cuda.current_device()
    st = _SIDE_STREAMS.get(dev)
    if st is None:
        st = _SIDE_STREAMS[dev] = torch.cuda.Stream()
    return st


def spark_dtype_of_arrow(t) -> str:
    """Arrow type -> Spark SQL dtype string as `idf.dtypes` would print it."""
    import pyarrow as pa
    if pa.types.is_dictionary(t):
        return spark_dtype_of_arrow(t.value_type)
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


def kind_of(sdtype: str) -> str:
    """'num' | 'cat' | 'other' exactly as shared/utils.py:64-72 decides."""
    if sdtype == "string":
        return "cat"
    if sdtype in _NUMERIC_SPARK or sdtype.startswith("decimal"):
        return "num"
    return "other"


_NP_TO_ANV = {np.dtype("float32"): (_lib.ANV_F32, "float"), np.dtype("float64"): (_lib.ANV_F64, "double"),
              np.dtype("int32"): (_lib.ANV_I32, "int"), np.dtype("int64"): (_lib.ANV_I64, "bigint")}


def _pack_validity(valid_bool: np.ndarray) -> np.ndarray:
    """bool[n] -> Arrow LSB-first bitmap as int32 words (padded with zeros)."""
    bits = np.packbits(valid_bool, bitorder="little")
    pad = (-len(bits)) % 4
    if pad:
        bits = np.concatenate([bits, np.zeros(pad, np.uint8)])
    return bits.view(np.int32)


_PACK_BLOCK_ROWS = 1 << 26      # rows packed per step of pack_bits_device: bounds its scratch at about 2 bytes per row of a step


def pack_bits_device(bits):
    """bool tensor [n] -> Arrow LSB-first validity bitmap as int32 words, on the tensor's device.  Every 8 rows become one
    byte (a sum of the rows weighted by 1, 2, ..., 128 in uint8) and four bytes one little-endian word, step by step, so a
    mask of billions of rows needs about n / 8 bytes of output and a few bytes per row of one step, not an int64 per row."""
    import torch
    n = int(bits.numel())
    words = (n + 31) // 32
    out = torch.zeros(max(words, 1) * 4, dtype=torch.uint8, device=bits.device)
    weights = torch.tensor([1 << i for i in range(8)], dtype=torch.uint8, device=bits.device)
    flat = bits.reshape(-1)
    for r0 in range(0, n, _PACK_BLOCK_ROWS):
        r1 = min(r0 + _PACK_BLOCK_ROWS, n)
        blk = flat[r0:r1].to(torch.uint8)
        if (r1 - r0) % 8:
            blk = torch.cat([blk, blk.new_zeros(8 - (r1 - r0) % 8)])
        out[r0 // 8:r0 // 8 + blk.numel() // 8] = (blk.view(-1, 8) * weights).sum(dim=1, dtype=torch.uint8)
    return out.view(torch.int32)[:words]


def _arrow_validity_words(arr):
    """Arrow array -> int32 bitmap words (None when the array has no nulls)."""
    if arr.null_count == 0:
        return None
    n = len(arr)
    buf = arr.buffers()[0]
    if buf is not None and arr.offset == 0:
        nbytes = (n + 7) // 8
        raw = np.frombuffer(buf, dtype=np.uint8, count=nbytes).copy()
        if n % 8:
            raw[-1] &= (1 << (n % 8)) - 1  # bits past n_rows must read as 0
        pad = (-len(raw)) % 4
        if pad:
            raw = np.concatenate([raw, np.zeros(pad, np.uint8)])
        return raw.view(np.int32)
    return _pack_validity(np.asarray(arr.is_valid()))


def narrow_code_dtype(cardinality: int):
    """Host storage type of the dictionary codes of a string column: the narrowest of uint8 / int16 / int32 that holds
    every code (the way Parquet and Arrow keep dictionary indices).  Fewer bytes cross PCIe; the device copy is widened to
    the int32 the kernels read right after the upload, on the upload's stream."""
    if cardinality <= 256:
        return np.uint8
    if cardinality <= 32768:
        return np.int16
    return np.int32


def narrow_codes(codes: np.ndarray, cardinality: int) -> np.ndarray:
    dt = narrow_code_dtype(cardinality)
    return codes if codes.dtype == dt else codes.astype(dt)


_CODE_DTYPES = (np.dtype(np.uint8), np.dtype(np.int16), np.dtype(np.int32))


class Column:
    __slots__ = ("name", "sdtype", "kind", "anv_dtype", "n_rows", "null_count", "dictionary",
                 "_host", "_host_valid", "_dev", "_dev_valid", "_ready", "_loader")

    def __init__(self, name, sdtype, n_rows, host=None, host_valid=None, dev=None, dev_valid=None,
                 anv_dtype=None, null_count=None, dictionary=None, loader=None):
        self.name, self.sdtype, self.kind = name, sdtype, kind_of(sdtype)
        self.n_rows = int(n_rows)
        self._host, self._host_valid, self._dev, self._dev_valid = host, host_valid, dev, dev_valid
        self.anv_dtype = anv_dtype
        self.null_count = null_count
        self.dictionary = dictionary
        self._ready = None  # CUDA event of an in-flight asynchronous upload
        self._loader = loader  # () -> (device data, device validity | None): materialised on first use (lazy chunks)

    def upload_async(self, stream):
        """Enqueue the H2D copy of this column on `stream` (pinned host memory makes it truly
        asynchronous); consumers wait on the recorded event, not on the host."""
        global h2d_bytes
        torch = _lib.require_cuda()
        if self._dev is not None or self.kind == "other" or self._host is None:
            return
        h = self._host if self._host.flags.writeable else self._host.copy()
        th = torch.from_numpy(h)
        dv = None
        consumer = torch.cuda.current_stream()
        with torch.cuda.stream(stream):
            # allocate from the copy stream's pool (blocks are reused by the next upload without a
            # cudaMalloc) and tell the allocator that the compute stream uses them too
            dev = torch.empty(th.shape, dtype=th.dtype, device="cuda")
            dev.copy_(th, non_blocking=True)
            h2d_bytes += h.nbytes
            if self.dictionary is not None and dev.dtype != torch.int32:
                dev = dev.to(torch.int32)      # narrow host codes -> the int32 codes the kernels read
            if self._host_valid is not None:
                tv = torch.from_numpy(self._host_valid)
                dv = torch.empty(tv.shape, dtype=tv.dtype, device="cuda")
                dv.copy_(tv, non_blocking=True)
                h2d_bytes += self._host_valid.nbytes
            ev = torch.cuda.Event()
            ev.record(stream)
        dev.record_stream(consumer)
        if dv is not None:
            dv.record_stream(consumer)
        self._dev, self._dev_valid, self._ready = dev, dv, ev

    def generate_async(self, stream):
        """Run this lazy column's generator on `stream` (a side stream) and leave an event for the consumers - the
        counterpart of upload_async for columns that are produced on the device."""
        torch = _lib.require_cuda()
        if self._dev is not None or self._loader is None or stream is None:
            return
        consumer = torch.cuda.current_stream()
        with torch.cuda.stream(stream):
            dev, dv = self._loader()
            ev = torch.cuda.Event()
            ev.record(stream)
        dev.record_stream(consumer)
        if dv is not None:
            dv.record_stream(consumer)
        self._dev, self._dev_valid, self._ready = dev, dv, ev

    @property
    def has_validity(self):
        if self._loader is not None and self._dev is None:
            return self.null_count is None or self.null_count > 0
        return self._host_valid is not None or self._dev_valid is not None

    def device(self):
        """-> (data tensor, validity tensor|None) on the current CUDA device (uploads once)."""
        torch = _lib.require_cuda()
        if self.kind == "other":
            raise _lib.AnvError("column %r has dtype %s which the hot path does not process" % (self.name, self.sdtype))
        if self._ready is not None:  # asynchronous upload in flight: order the current stream after it
            torch.cuda.current_stream().wait_event(self._ready)
            self._ready = None
        if self._dev is None and self._loader is not None:
            self._dev, self._dev_valid = self._loader()
        if self._dev is None:
            global h2d_bytes
            h = self._host if self._host.flags.writeable else self._host.copy()
            t = torch.from_numpy(h)
            # pinned host buffers upload asynchronously on the current stream (stream-ordered with the kernels)
            self._dev = t.cuda(non_blocking=t.is_pinned())
            h2d_bytes += h.nbytes
            if self.dictionary is not None and self._dev.dtype != torch.int32:
                self._dev = self._dev.to(torch.int32)
            if self._host_valid is not None:
                tv = torch.from_numpy(self._host_valid)
                self._dev_valid = tv.cuda(non_blocking=tv.is_pinned())
                h2d_bytes += self._host_valid.nbytes
        return self._dev, self._dev_valid

    def drop_device(self):
        if self._host is not None or self._loader is not None:
            self._dev = self._dev_valid = None


class ColumnFrame:
    """Immutable column-major frame; `columns` / `dtypes` / `count()` mirror the Spark API
    the reference uses."""

    def __init__(self, cols: "OrderedDict[str, Column]", n_rows: int):
        self._cols = cols
        self.n_rows = int(n_rows)
        self._cache = {}

    # ---- Spark-DataFrame-like surface used by the reference code ------------------------
    @property
    def columns(self):
        return list(self._cols)

    @property
    def dtypes(self):
        return [(c.name, c.sdtype) for c in self._cols.values()]

    def count(self):
        return self.n_rows

    def select(self, names):
        if isinstance(names, str):
            names = [names]
        return ColumnFrame(OrderedDict((n, self._cols[n]) for n in names), self.n_rows)

    def column(self, name) -> Column:
        return self._cols[name]

    def drop(self, *names) -> "ColumnFrame":
        """`idf.drop(*cols)`."""
        names = set(names[0]) if len(names) == 1 and isinstance(names[0], (list, tuple, set)) else set(names)
        return ColumnFrame(OrderedDict((n, c) for n, c in self._cols.items() if n not in names), self.n_rows)

    def with_columns(self, cols, drop=()) -> "ColumnFrame":
        """The frame without `drop`, then with `cols` (an ordered name -> Column mapping): a name the frame still has is
        replaced in place, a new one is appended in the order of `cols` (Spark's withColumn, one call per column)."""
        drop = set(drop)
        out = OrderedDict((n, c) for n, c in self._cols.items() if n not in drop)
        out.update(cols)
        return ColumnFrame(out, self.n_rows)

    def valid_mask(self, name):
        """bool CUDA tensor [n_rows]: True where column `name` is non-null (frame transforms only)."""
        torch = _lib.require_cuda()
        d, v = self._cols[name].device()
        if v is None:
            return torch.ones(self.n_rows, dtype=torch.bool, device=d.device)
        rows = torch.arange(self.n_rows, device=d.device)
        return ((v[rows >> 5] >> (rows & 31).to(torch.int32)) & 1).bool()

    def filter_rows(self, keep) -> "ColumnFrame":
        """`idf.where(cond)`: keep the rows where the bool CUDA tensor `keep` is True (frame transform on the
        device with torch indexing: plumbing, not a hot path)."""
        torch = _lib.require_cuda()
        idx = torch.nonzero(keep).flatten()
        m = int(idx.numel())
        out = OrderedDict()
        for n, c in self._cols.items():
            if c.kind == "other":
                out[n] = Column(n, c.sdtype, m)
                continue
            d, v = c.device()
            nv = None
            if v is not None:
                bits = ((v[idx >> 5] >> (idx & 31).to(torch.int32)) & 1).bool()
                if not bool(bits.all()):
                    nv = pack_bits_device(bits)
            out[n] = Column(n, c.sdtype, m, dev=d.index_select(0, idx), dev_valid=nv, anv_dtype=c.anv_dtype,
                            dictionary=c.dictionary)
        return ColumnFrame(out, m)

    def dropna(self, subset=None) -> "ColumnFrame":
        """`idf.dropna(subset=cols)`: keep the rows whose `subset` columns are all non-null."""
        torch = _lib.require_cuda()
        subset = list(subset) if subset is not None else self.columns
        keep = None
        for n in subset:
            if self._cols[n].kind != "other" and self._cols[n].device()[1] is not None:
                m = self.valid_mask(n)
                keep = m if keep is None else keep & m
        return self if keep is None else self.filter_rows(keep)

    def slice_rows(self, r0: int, r1: int) -> "ColumnFrame":
        """Zero-copy view of rows [r0, r1): r0 must be a multiple of 32 so that the validity
        bitmap (and the 16-byte alignment of the values) slices on a word boundary.  Host-resident
        columns stay on the host (each slice uploads on first use): the row chunks of a
        PartitionedFrame are made this way."""
        r0, r1 = int(r0), min(int(r1), self.n_rows)
        if r0 % 32 or r0 < 0 or r1 < r0:
            raise ValueError("slice_rows: r0 must be a non-negative multiple of 32 and r1 >= r0")
        m = r1 - r0
        w0, w1 = r0 // 32, (r1 + 31) // 32
        out = OrderedDict()
        for n, c in self._cols.items():
            if c.kind == "other":
                out[n] = Column(n, c.sdtype, m)
                continue
            if c._dev is None and c._host is None and c._loader is not None:
                c.device()   # a lazy column has to exist before it can be sliced
            host = c._host[r0:r1] if c._host is not None else None
            hv = c._host_valid[w0:w1] if c._host_valid is not None else None
            dev = c._dev[r0:r1] if c._dev is not None else None
            dv = c._dev_valid[w0:w1] if c._dev_valid is not None else None
            if c._ready is not None and dev is not None:  # slice of an in-flight upload: wait for it first
                c.device()
            out[n] = Column(n, c.sdtype, m, host=host, host_valid=hv, dev=dev, dev_valid=dv, anv_dtype=c.anv_dtype,
                            dictionary=c.dictionary)
        return ColumnFrame(out, m)

    def __contains__(self, name):
        return name in self._cols

    def to_arrow(self):
        """-> pyarrow Table (D2H of values and validity; string columns decoded through their dictionary).  Columns of
        "other" kind carry no data on this path and come back as all-null columns."""
        import pyarrow as pa
        arrays = []
        for n, c in self._cols.items():
            if c.kind == "other":
                arrays.append(pa.nulls(self.n_rows))
                continue
            if c._host is not None and c._dev is None:
                vals, words = np.asarray(c._host), c._host_valid
            else:
                d, v = c.device()
                vals, words = d.cpu().numpy(), (None if v is None else v.cpu().numpy())
            mask = None
            if words is not None:
                bits = np.unpackbits(np.ascontiguousarray(words).view(np.uint8), bitorder="little")[:self.n_rows]
                mask = bits == 0
            if c.dictionary is not None:
                idx = pa.array(np.asarray(vals[:self.n_rows]).astype(np.int32, copy=False), type=pa.int32(), mask=mask)
                arrays.append(pa.DictionaryArray.from_arrays(idx, pa.array(c.dictionary, type=pa.string())).cast(pa.string()))
            else:
                arrays.append(pa.array(vals[:self.n_rows], mask=mask))
        return pa.table(arrays, names=list(self._cols))

    def to_pandas(self):
        return self.to_arrow().to_pandas()

    # ---- constructors -----------------------------------------------------------------
    @staticmethod
    def from_arrow(table) -> "ColumnFrame":
        import pyarrow as pa
        import pyarrow.compute as pc
        cols = OrderedDict()
        n = table.num_rows
        for field in table.schema:
            arr = table.column(field.name)
            arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
            if isinstance(arr, pa.ChunkedArray):  # zero chunks
                arr = pa.array([], type=field.type)
            t = arr.type
            sd = spark_dtype_of_arrow(t)
            k = kind_of(sd)
            if k == "other":
                cols[field.name] = Column(field.name, sd, n)
                continue
            if k == "cat":
                if not pa.types.is_dictionary(t):
                    arr = pc.dictionary_encode(arr)
                dic = arr.dictionary.to_pylist()
                idx = arr.indices
                codes = (idx.fill_null(0) if idx.null_count else idx).to_numpy(zero_copy_only=False).astype(np.int32)
                order = sorted(range(len(dic)), key=lambda i: dic[i].encode("utf-8"))  # Spark: UTF-8 byte order
                remap = np.empty(max(len(dic), 1), dtype=np.int32)
                remap[np.asarray(order, dtype=np.int64)] = np.arange(len(dic), dtype=np.int32)
                codes = remap[codes] if len(dic) else codes
                cols[field.name] = Column(field.name, "string", n, host=np.ascontiguousarray(narrow_codes(codes, len(dic))),
                                          host_valid=_arrow_validity_words(idx), anv_dtype=_lib.ANV_I32,
                                          null_count=idx.null_count, dictionary=[dic[i] for i in order])
                continue
            if pa.types.is_decimal(t):
                arr = arr.cast(pa.float64())
            elif pa.types.is_uint32(t):
                arr = arr.cast(pa.int64())
            vals = (arr.fill_null(0) if arr.null_count else arr).to_numpy(zero_copy_only=False)
            vals = np.ascontiguousarray(vals)
            anv_dt = _NP_TO_ANV[vals.dtype][0]
            cols[field.name] = Column(field.name, sd, n, host=vals, host_valid=_arrow_validity_words(arr),
                                      anv_dtype=anv_dt, null_count=arr.null_count)
        return ColumnFrame(cols, n)

    @staticmethod
    def from_pandas(df) -> "ColumnFrame":
        import pyarrow as pa
        return ColumnFrame.from_arrow(pa.Table.from_pandas(df, preserve_index=False))

    @staticmethod
    def from_tensors(data: dict, n_rows=None) -> "ColumnFrame":
        """dict name -> tensor | (tensor, validity_words) | (codes, validity_words, dictionary).
        Tensors may be torch (CUDA or CPU) or numpy; dtype float32/float64/int32/int64; HOST dictionary codes may also be
        uint8 / int16 (narrow_code_dtype).
        validity_words: int32 Arrow bitmap words (ceil(n/32)) or None."""
        import torch
        cols = OrderedDict()
        for name, v in data.items():
            dic = None
            valid = None
            if isinstance(v, tuple):
                if len(v) == 3:
                    v, valid, dic = v
                else:
                    v, valid = v
            is_torch = isinstance(v, torch.Tensor)
            npdt = np.dtype(str(v.dtype).replace("torch.", "")) if is_torch else np.asarray(v).dtype
            if dic is not None and npdt in _CODE_DTYPES and not (is_torch and v.is_cuda):
                anv_dt, sd = _lib.ANV_I32, "string"     # host codes may be narrow (narrow_code_dtype): widened on upload
            elif npdt not in _NP_TO_ANV:
                raise TypeError("column %r: unsupported dtype %s" % (name, npdt))
            else:
                anv_dt, sd = _NP_TO_ANV[npdt]
            n = int(v.shape[0])
            if n_rows is None:
                n_rows = n
            if n != n_rows:
                raise ValueError("column %r has %d rows, expected %d" % (name, n, n_rows))
            if dic is not None:
                sd = "string"
                if anv_dt != _lib.ANV_I32:
                    raise TypeError("dictionary codes must be int32 (uint8 / int16 are accepted for host buffers)")
            if is_torch and v.is_cuda:
                if v.data_ptr() % 16 or not v.is_contiguous():
                    v = v.contiguous().clone()
                col = Column(name, sd, n, dev=v, dev_valid=valid, anv_dtype=anv_dt, dictionary=dic)
            else:
                hv = v.numpy() if is_torch else np.ascontiguousarray(v)
                hvalid = None
                if valid is not None:
                    hvalid = valid.numpy() if isinstance(valid, torch.Tensor) else np.ascontiguousarray(valid)
                col = Column(name, sd, n, host=hv, host_valid=hvalid, anv_dtype=anv_dt, dictionary=dic)
            cols[name] = col
        return ColumnFrame(cols, n_rows or 0)

    # ---- device descriptors -----------------------------------------------------------
    def descriptors(self, names):
        """Device array of anv_column_t for `names` (kept alive by the returned tensor)."""
        torch = _lib.require_cuda()
        key = ("desc", tuple(names))
        hit = self._cache.get(key)
        if hit is not None:
            # valid only while every column still holds the buffers the descriptors point at: a chunk released with
            # drop_device() (and re-uploaded later) must not be kept alive - or addressed - through this cache
            if all(self._cols[n]._dev is d and self._cols[n]._dev_valid is v for n, (d, v) in zip(names, hit[1])):
                return hit
            del self._cache[key]
        arr = (_lib.AnvColumn * max(len(names), 1))()
        keep = []
        for i, nme in enumerate(names):
            col = self._cols[nme]
            d, v = col.device()
            if d.data_ptr() % 16:
                raise _lib.AnvError("column %r is not 16-byte aligned" % nme)
            arr[i].data = d.data_ptr()
            arr[i].validity = v.data_ptr() if v is not None else None
            arr[i].dtype = col.anv_dtype
            keep.append((d, v))
        host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
        dev = host.cuda()
        self._cache[key] = (dev, keep)
        return dev, keep


def as_frame(idf) -> ColumnFrame:
    if isinstance(idf, ColumnFrame) or getattr(idf, "is_partitioned", False):
        return idf
    mod = type(idf).__module__
    if mod.startswith("pyarrow"):
        md = idf.schema.metadata or {}
        if b"spark_partition_rows" in md:   # the table says how Spark partitioned it: percentiles follow Spark's sketch
            import json
            from .partitioned import PartitionedFrame
            return PartitionedFrame.from_arrow_partitions(idf, json.loads(md[b"spark_partition_rows"]))
        return ColumnFrame.from_arrow(idf)
    if mod.startswith("pandas"):
        return ColumnFrame.from_pandas(idf)
    if isinstance(idf, dict):
        return ColumnFrame.from_tensors(idf)
    if hasattr(idf, "toPandas"):  # a Spark DataFrame, when pyspark is installed
        return ColumnFrame.from_pandas(idf.toPandas())
    raise TypeError("unsupported frame type %r: pass a ColumnFrame, pyarrow Table, pandas DataFrame or dict of tensors"
                    % type(idf))
