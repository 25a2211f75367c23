"""TEST INFRASTRUCTURE: a NumPy stand-in of engine.flag_members (one anv_flag_members call: np.isin plus per-entry counts
on the ordered keys), installed with tests/cpu_engine.py, so the host layer of invalidEntries_detection runs without a
GPU."""
import contextlib

import numpy as np

import cpu_engine
from anovos_b200 import engine
from anovos_b200.shared.invalid_rules import ordered_keys


def pack_bits(keep):
    bits = np.packbits(np.asarray(keep, bool), bitorder="little")
    return np.concatenate([bits, np.zeros((-len(bits)) % 4, np.uint8)]).view(np.int32)


def flag_rows(vals, valid, table):
    """-> (per-entry counts uint64, bool hit per row): the kernel's contract on host arrays."""
    keys, tk = ordered_keys(np.asarray(vals)), ordered_keys(np.asarray(table))
    pos = np.minimum(np.searchsorted(tk, keys), max(len(tk) - 1, 0))
    hit = valid & (tk[pos] == keys) if len(tk) else np.zeros(len(keys), bool)
    counts = np.bincount(pos[hit], minlength=len(tk)).astype(np.uint64)[:len(tk)]
    return counts, hit


def flag_members(fr, names, tables, want_bitmap):
    import torch
    if getattr(fr, "is_partitioned", False):
        return fr.flag_members(list(names), list(tables)), [None] * len(list(names))
    counts, valid = [], []
    for n, t in zip(names, tables):
        t = np.asarray(t)
        vals, ok = cpu_engine._values(fr, n)
        if len(t) == 0 or fr.n_rows == 0:
            counts.append(np.zeros(len(t), np.uint64))
            valid.append(None)
            continue
        cnt, hit = flag_rows(vals, ok, t)
        counts.append(cnt)
        valid.append(torch.from_numpy(pack_bits(ok & ~hit).copy()) if want_bitmap else None)
    return counts, valid


@contextlib.contextmanager
def installed():
    saved = engine.flag_members
    try:
        engine.flag_members = flag_members
        with cpu_engine.installed():
            yield
    finally:
        engine.flag_members = saved
