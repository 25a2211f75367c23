"""Multi-GPU plumbing of the hot path (SURVEY.md 8e): columns are independent in every
function of the path, so they shard across ranks with NO data-path collective; the only
exchange is one all_gather of the small per-column summary table at the end of a pass
(NCCL over NVLink on GPUs, gloo in the CPU tests)."""
from __future__ import annotations

import numpy as np


def shard_columns(names, rank: int, world: int):
    """Contiguous column blocks, ceil(C / world) per rank (source and target of a column stay
    on the same rank, so drift needs no exchange)."""
    names = list(names)
    per = (len(names) + world - 1) // world
    return names[rank * per:(rank + 1) * per]


_NON_NUMERIC = {"attribute", "mode", "metric", "value"}


def frames_to_matrix(frames):
    """Result frames (pandas) -> float64 matrix [n_attributes, n_numeric_fields] + the field names, aligned on
    `attribute` (mixed frames: the numeric-only functions - dispersion, percentiles, shape - return fewer rows than the
    functions that also cover string columns; the missing cells are NaN).  Non-numeric fields (attribute, mode) stay
    local to the rank; they are re-attached by name."""
    import pandas as pd
    order = {}
    for df in frames:
        if "attribute" in df.columns:
            for a in df["attribute"].tolist():
                order.setdefault(a, len(order))
    n = len(order) if order else max((len(df) for df in frames), default=0)
    cols, names = [], []
    for df in frames:
        rows = np.fromiter((order[a] for a in df["attribute"].tolist()), dtype=np.int64, count=len(df)) \
            if "attribute" in df.columns else np.arange(len(df))
        for c in df.columns:
            if c in _NON_NUMERIC:
                continue
            a = df[c]._values
            if isinstance(a, np.ndarray) and a.dtype != object:
                a = a.astype(np.float64, copy=False)
            else:                       # object columns (None for "not applicable"), pandas extension arrays
                a = pd.to_numeric(df[c], errors="coerce").to_numpy(dtype=np.float64, na_value=np.nan)
            full = np.full(n, np.nan)
            full[rows] = a
            cols.append(full)
            names.append(c)
    return np.ascontiguousarray(np.stack(cols, axis=1)), names


class PendingGather:
    """Handle of an asynchronous summary all_gather: `.result()` waits and returns the per-rank matrices."""

    def __init__(self, work, out, n_rows):
        self.work, self.out, self.n_rows = work, out, n_rows

    def result(self):
        self.work.wait()
        return [o[:n].cpu().numpy() for o, n in zip(self.out, self.n_rows)]


def gather_summaries_async(matrix: np.ndarray, n_max: int, device=None) -> PendingGather:
    """Non-blocking all_gather of fixed-shape [n_max, n_fields] padded summaries (every rank passes the same
    n_max, e.g. ceil(C / world)): ranks do not wait for each other inside a step, only when the result is
    consumed.  Rows beyond a rank's own column count are NaN."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size()
    t = torch.from_numpy(np.ascontiguousarray(matrix, dtype=np.float64))
    pad = torch.full((n_max, t.shape[1]), float("nan"), dtype=torch.float64)
    pad[:t.shape[0]] = t
    if device is not None:
        pad = pad.to(device)
    out = [torch.empty_like(pad) for _ in range(world)]
    work = dist.all_gather(out, pad, async_op=True)
    return PendingGather(work, out, [n_max] * world)


def gather_summaries(matrix: np.ndarray, device=None):
    """all_gather of each rank's [n_local_cols, n_fields] summary matrix -> list over ranks.
    Ranks may own different numbers of columns: matrices are padded to the largest.  An int64 matrix is gathered as
    int64 (exact 64-bit integers, e.g. the mode of a bigint column); anything else as float64."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size()
    exact = np.asarray(matrix).dtype == np.int64
    t = torch.from_numpy(np.ascontiguousarray(matrix, dtype=np.int64 if exact else np.float64))
    if device is not None:
        t = t.to(device)
    n_local = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    counts = [torch.zeros_like(n_local) for _ in range(world)]
    dist.all_gather(counts, n_local)
    n_max = int(max(int(c.item()) for c in counts))
    pad = torch.full((n_max, t.shape[1]), 0 if exact else float("nan"), dtype=t.dtype, device=t.device)
    pad[:t.shape[0]] = t
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad)
    return [o[:int(c.item())].cpu().numpy() for o, c in zip(out, counts)]


def bind_numa(device_index: int):
    """Pin this process to the CPUs of the NUMA node the GPU hangs off (sysfs: /sys/bus/pci/devices/<bdf>/numa_node), so
    that pinned host buffers allocated afterwards are local to the GPU's PCIe root: torchrun does not bind its workers, and
    a rank that lands on the other socket uploads at a fraction of the PCIe rate.  Call BEFORE the first pinned allocation.
    -> dict describing what was done (bench.py reports it)."""
    import os
    info = {"bound": False}
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        idx = device_index
        if vis:
            ent = vis.split(",")[device_index].strip()
            h = pynvml.nvmlDeviceGetHandleByUUID(ent) if ent.startswith(("GPU-", "MIG-")) else pynvml.nvmlDeviceGetHandleByIndex(int(ent))
        else:
            h = pynvml.nvmlDeviceGetHandleByIndex(idx)
        bdf = pynvml.nvmlDeviceGetPciInfo(h).busId
        bdf = bdf.decode() if isinstance(bdf, bytes) else bdf
        bdf = bdf.lower()
        if len(bdf.split(":")[0]) == 8:          # nvml prints an 8-digit domain, sysfs a 4-digit one
            bdf = bdf[4:]
        node = int(open("/sys/bus/pci/devices/%s/numa_node" % bdf).read().strip())
        info.update(pci=bdf, node=node)
        if node < 0:
            return info
        cpus = set()
        for part in open("/sys/devices/system/node/node%d/cpulist" % node).read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        cpus &= os.sched_getaffinity(0)
        if cpus:
            os.sched_setaffinity(0, cpus)
            info.update(bound=True, cpus=len(cpus))
    except Exception as ex:   # best effort: an unbound process still works, only slower over PCIe
        info["error"] = repr(ex)
    return info
