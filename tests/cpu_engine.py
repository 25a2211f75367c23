"""TEST INFRASTRUCTURE: a NumPy stand-in for `anovos_b200.engine` so that the product's host layer (argument handling,
binning models, key alignment of drift, saved artefacts, partition merges, outlier thresholds) can be exercised under
`-m "not gpu"`.  Every function has the signature and result layout of the engine function it replaces and is written
from the oracle's primitives; the kernels themselves are tested against the oracle on the GPU (`-m gpu`).

    with cpu_engine.installed():      # monkeypatches engine.*, Column.device / upload_async and _lib.require_cuda
        dd.statistics(None, target, source, ...)
"""
import contextlib

import numpy as np

from anovos_b200 import _lib, engine, frame as framemod
from oracle import spark_semantics as S


def _values(fr, name):
    """(float64-or-native values, bool valid) of a HOST-resident column."""
    col = fr.column(name)
    if col._host is not None:
        vals, words = np.asarray(col._host), col._host_valid
        if col.dictionary is not None:
            vals = vals.astype(np.int32, copy=False)      # host codes are stored narrow (frame.narrow_code_dtype)
    else:                                  # a column produced by a frame transform: CPU tensors under this stand-in
        vals = col._dev.numpy()
        words = None if col._dev_valid is None else col._dev_valid.numpy()
    if words is None:
        valid = np.ones(fr.n_rows, dtype=bool)
    else:
        bits = np.unpackbits(np.ascontiguousarray(words).view(np.uint8), bitorder="little")
        valid = bits[:fr.n_rows].astype(bool)
    return vals[:fr.n_rows], valid


def moments(fr, names):
    if getattr(fr, "is_partitioned", False):
        return fr.moments(names)
    out = np.zeros(len(list(names)), dtype=engine._MOM_DT)
    for i, n in enumerate(names):
        vals, valid = _values(fr, n)
        x = vals[valid].astype(np.float64)
        out[i]["n_valid"], out[i]["n_nonzero"] = x.size, int(np.count_nonzero(x))
        if x.size:
            cnt, mean, m2, m3, m4 = S.central_moments(x)
            out[i]["min"], out[i]["max"], out[i]["mean"] = x.min(), x.max(), mean
            out[i]["m2"], out[i]["m3"], out[i]["m4"] = m2, m3, m4
        else:
            out[i]["min"] = out[i]["max"] = out[i]["mean"] = np.nan
    return out


def _bin_ids(fr, model, i):
    """Bin ids of column i of `model` (0 = null): from the exact int64 thresholds when the model has them
    (bin 1 + #(thresholds < v), the kernels' compare), else from the float64 cutoffs."""
    vals, valid = _values(fr, model.names[i])
    ex = getattr(model, "exact", [None] * len(model.names))[i]
    if ex is None:
        return S.assign_bins(vals, valid, model.cutoffs[i], len(model.cutoffs[i]) + 1)
    ids = 1 + np.searchsorted(np.array(ex, dtype=np.int64), vals.astype(np.int64), side="left")
    return np.where(valid, ids, 0).astype(np.int32)


def histogram(fr, model):
    if getattr(fr, "is_partitioned", False):
        return fr.histogram(model)
    h = np.zeros((len(model.names), model.max_bins + 1), np.uint64)
    for i, n in enumerate(model.names):
        ids = _bin_ids(fr, model, i)
        h[i, :len(model.cutoffs[i]) + 2] = np.bincount(ids, minlength=len(model.cutoffs[i]) + 2)
    return h


def moments_histogram(fr, model):
    if getattr(fr, "is_partitioned", False):
        return fr.moments_histogram(model)
    return moments(fr, model.names), histogram(fr, model)


def code_counts(fr, names):
    if getattr(fr, "is_partitioned", False):
        return fr.code_counts(list(names))
    out = []
    for n in names:
        vals, valid = _values(fr, n)
        card = max(len(fr.column(n).dictionary), 1)
        h = np.zeros(card + 1, np.uint64)
        h[0] = int((~valid).sum())
        h[1:] = np.bincount(vals[valid].astype(np.int64), minlength=card)[:card]
        out.append(h)
    return out


def drift_reduce(src_counts, tgt_counts, kinds, n_src, n_tgt, src_p=None):
    n = len(tgt_counts)
    out = np.zeros(n, dtype=engine._DRIFT_DT)
    for i in range(n):
        t = np.asarray(tgt_counts[i], dtype=np.float64)
        if src_p is None:
            s = np.asarray(src_counts[i], dtype=np.float64)
            present_s, p = s > 0, s / n_src
        else:
            sp = np.asarray(src_p[i], dtype=np.float64)
            present_s, p = ~np.isnan(sp), np.nan_to_num(sp)
        rows = []
        s_null, t_null = bool(present_s[0]), bool(t[0] > 0)
        if kinds[i] == 0:
            if s_null or t_null:
                rows.append((1e-4, 1e-4))
        else:
            rows += [(1e-4, 1e-4)] * (int(s_null) + int(t_null))
        for k in range(1, len(t)):
            ps, pt = bool(present_s[k]), bool(t[k] > 0)
            if ps or pt:
                rows.append((p[k] if ps else 1e-4, t[k] / n_tgt if pt else 1e-4))
        psi = hd = pm = qm = cp = cq = ks = 0.0
        for a, b in rows:
            a, b = (a or 1e-4), (b or 1e-4)
            psi += (a - b) * np.log(a / b)
            hd += (np.sqrt(a) - np.sqrt(b)) ** 2
            m = (a + b) / 2
            pm += a * np.log(a / m)
            qm += b * np.log(b / m)
            cp += a
            cq += b
            ks = max(ks, abs(cp - cq))
        out[i]["n_rows"] = len(rows)
        if rows:
            out[i]["psi"], out[i]["hd"], out[i]["jsd"], out[i]["ks"] = psi, np.sqrt(hd / 2), (pm + qm) / 2, ks
        else:
            out[i]["psi"] = out[i]["hd"] = out[i]["jsd"] = out[i]["ks"] = np.nan
    return out


def _sorted_valid(fr, names):
    """name -> sorted float64 non-null values (chunks of a partitioned frame concatenated)."""
    names = list(names)
    if getattr(fr, "is_partitioned", False):
        parts = {n: [] for n in names}
        for ch in fr.chunks(names):
            for n in names:
                vals, valid = _values(ch, n)
                parts[n].append(vals[valid].astype(np.float64))
        return {n: np.sort(np.concatenate(parts[n])) if parts[n] else np.zeros(0) for n in names}
    return {n: np.sort(_values(fr, n)[0][_values(fr, n)[1]].astype(np.float64)) for n in names}


def select_ranks(fr, names, ranks):
    names = list(names)
    whole = _sorted_valid(fr, names)
    ranks = np.asarray(ranks, dtype=np.int64).reshape(len(names), -1)
    out = np.full(ranks.shape, np.nan)
    for i, n in enumerate(names):
        for j, r in enumerate(ranks[i]):
            if r > 0:
                out[i, j] = whole[n][r - 1]
    return out


def sort_mode_distinct(fr, names, ranks=None):
    """Modes of bigint columns are exact Python ints (engine.sort_mode_distinct's contract), every other mode a float."""
    names = list(names)
    whole = _sorted_valid(fr, names)
    res = []
    for n in names:
        if fr.column(n).anv_dtype == _lib.ANV_I64:
            if getattr(fr, "is_partitioned", False):
                x = np.concatenate([_values(ch, n)[0][_values(ch, n)[1]] for ch in fr.chunks([n])] or [np.zeros(0, np.int64)])
            else:
                x = _values(fr, n)[0][_values(fr, n)[1]]
            x = x.astype(np.int64)
        else:
            x = whole[n] + 0.0
        if x.size == 0:
            res.append((None, None, 0))
            continue
        u, k = np.unique(x, return_counts=True)
        res.append((u[np.argmax(k)].item(), int(k.max()), int(u.size)))
    if ranks is None:
        return res
    return res, select_ranks(fr, names, ranks)


def hll_registers(fr, names, p):
    if getattr(fr, "is_partitioned", False):
        return fr.hll_registers(list(names), p)
    out = np.zeros((len(list(names)), 1 << p), np.uint32)
    for i, n in enumerate(names):
        vals, valid = _values(fr, n)
        out[i] = S.hll_registers(S.hll_hashes(vals[valid], fr.column(n).sdtype), p)
    return out


def bin_assign(fr, model):
    """-> int32 torch (CPU) tensor [n_cols, n_rows] of bin ids, 0 = null row (the layout anv_bin_assign fills)."""
    import torch
    out = np.zeros((max(len(model.names), 1), fr.n_rows), np.int32)
    for i, n in enumerate(model.names):
        out[i] = _bin_ids(fr, model, i)
    return torch.from_numpy(out)[:len(model.names)]


class _Cuda:
    @staticmethod
    def Stream():
        return None


class _TorchProxy:
    """What the host layer asks of torch when no kernel runs: tensor ops on the CPU, and a stream object for the chunk
    prefetcher (uploads are no-ops here)."""
    cuda = _Cuda

    def __getattr__(self, name):
        import torch
        return getattr(torch, name)


def _host_device(self):
    """Column.device() without a GPU: the host arrays as CPU tensors."""
    import torch
    if self.kind == "other":
        raise _lib.AnvError("column %r has dtype %s which the hot path does not process" % (self.name, self.sdtype))
    if self._dev is None:
        h = np.ascontiguousarray(self._host)
        if self.dictionary is not None:
            h = h.astype(np.int32, copy=False)
        self._dev = torch.from_numpy(h.copy() if not h.flags.writeable else h)
        if self._host_valid is not None:
            self._dev_valid = torch.from_numpy(np.ascontiguousarray(self._host_valid).copy())
    return self._dev, self._dev_valid


def sample_mask(n_rows, seed, thresholds, strata=None):
    """Stand-in of data_sampling.sample_mask (csrc/sample.cu): the oracle's sequential XORShiftRandom stream."""
    import torch
    x = S.xorshift_uniform53(seed, n_rows)
    thr = np.asarray(thresholds, dtype=np.uint64)
    if strata is None:
        keep = x < thr[0]
    else:
        g = strata.numpy().astype(np.int64)
        ok = (g >= 0) & (g < len(thr))
        keep = ok & (x < thr[np.where(ok, g, 0)])
    return torch.from_numpy(keep)


@contextlib.contextmanager
def installed():
    names = ["moments", "histogram", "moments_histogram", "code_counts", "drift_reduce", "select_ranks", "sort_mode_distinct",
             "hll_registers", "bin_assign"]
    saved = {n: getattr(engine, n) for n in names}
    saved_req, saved_up, saved_dev = _lib.require_cuda, framemod.Column.upload_async, framemod.Column.device
    saved_fused, engine.FUSED_HLL = engine.FUSED_HLL, False
    from anovos_b200.data_ingest import data_sampling
    saved_mask = data_sampling.sample_mask
    try:
        data_sampling.sample_mask = sample_mask
        for n in names:
            setattr(engine, n, globals()[n])
        proxy = _TorchProxy()
        _lib.require_cuda = lambda: proxy
        framemod.Column.upload_async = lambda self, stream: None
        framemod.Column.device = _host_device
        yield
    finally:
        for n, f in saved.items():
            setattr(engine, n, f)
        _lib.require_cuda, framemod.Column.upload_async, framemod.Column.device = saved_req, saved_up, saved_dev
        data_sampling.sample_mask = saved_mask
        engine.FUSED_HLL = saved_fused
