"""Timing of invalidEntries_detection's table-membership pass (anv_flag_members, csrc/invalid.cu) on a frame built from
synth.device_frame's Philox columns (default 40 M rows x 32 columns):
  16 int32 columns   round(x * 37) of float32 Philox columns, auto table (AUTO_INT32, 156 entries, shared memory)
   8 int64 columns   round(x * 1e4) of float32 Philox columns, auto table (AUTO_INT64, 332 entries, shared memory)
   8 string columns  Zipf dictionary codes (cardinalities 2, 12, 100, 10 000), manual tables: codes 1-3 of every column
                     and, on the 10 000-entry columns, every other code as well (5 000 entries: the global-memory path)
  count_pass         anv_flag_members without output bitmaps (treatment=False)
  bitmap_pass        anv_flag_members with the nulled output bitmaps (null_replacement)
  torch              the same membership as a torch composite: torch.isin on the ordered keys, searchsorted + bincount
                     for the per-entry counts, the bitmap packed from the mask; counts and bitmaps compared bit for bit
  host_dictionary    the rule (shared/invalid_rules.py) over a 10^6-entry dictionary, auto and manual
  host_float         distinct values of one 40 M-row float32 column (torch.unique on the device) and the rule over them
Algorithmic bytes of a pass: one read of every column and bitmap, plus one write of the output bitmaps; TB/s against the
3.35 TB/s data-sheet HBM3 figure.  Prints the card and its power limit (read-only nvidia-smi query) and one JSON line.
Usage: python scripts/prof_invalid.py [rows] [reps]"""
import json
import subprocess
import sys
import time
from collections import OrderedDict

import numpy as np
import torch

sys.path.insert(0, ".")
from anovos_b200 import _lib, engine, synth  # noqa: E402
from anovos_b200.data_analyzer import quality_checker as QC  # noqa: E402
from anovos_b200.frame import Column, ColumnFrame  # noqa: E402
from anovos_b200.shared import invalid_rules as R  # noqa: E402

rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 40_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
HBM_PEAK = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def build_frame():
    src = synth.device_frame(rows, 32, cat_every=4)
    cats = [n for n in src.columns if src.column(n).dictionary is not None]
    nums = [n for n in src.columns if src.column(n).dictionary is None]
    cols = OrderedDict()
    for i, n in enumerate(nums[:24]):
        d, v = src.column(n).device()
        if i < 16:
            x, dt, sd = torch.round(d * 37).to(torch.int32), _lib.ANV_I32, "int"
        else:
            x, dt, sd = torch.round(d.double() * 1e4).to(torch.int64), _lib.ANV_I64, "bigint"
        cols["n%02d" % i] = Column("n%02d" % i, sd, rows, dev=x, dev_valid=v, anv_dtype=dt)
    for n in cats:
        c = src.column(n)
        cols[n] = c
    return ColumnFrame(cols, rows)


def tables_of(fr):
    out = []
    for n in fr.columns:
        c = fr.column(n)
        if c.dictionary is not None:
            size = len(c.dictionary)
            codes = set(range(1, min(4, size)))
            if size >= 10_000:
                codes |= set(range(0, size, 2))
            out.append(np.array(sorted(codes), np.int32))
        else:
            out.append(R.int_auto_table(engine._NP_OF_ANV[c.anv_dtype]))
    return out


def kernel_ms(fn):
    engine.timer = engine.KernelTimer()
    fn()
    engine.timer = engine.KernelTimer()
    for _ in range(reps):
        fn()
    t = engine.timer.totals()["anv_flag_members"]
    engine.timer = None
    return t["ms"] / t["calls"]


def events(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _bits(words, n):
    r = torch.arange(n, device="cuda")
    return ((words[r >> 5] >> (r & 31).to(torch.int32)) & 1).bool()


def _pack(mask):
    n = mask.numel()
    m = torch.cat([mask, torch.zeros((-n) % 32, dtype=torch.bool, device="cuda")]).view(-1, 32).to(torch.int64)
    w = (m << torch.arange(32, device="cuda", dtype=torch.int64)).sum(1)
    return ((w + (1 << 31)) % (1 << 32) - (1 << 31)).to(torch.int32)


def torch_flags(fr, names, tables):
    """-> (counts, bitmaps) of the torch composite.  Keys: the integers themselves (string codes, int32, int64)."""
    counts, bms = [], []
    for n, t in zip(names, tables):
        d, v = fr.column(n).device()
        tab = torch.from_numpy(t.astype(np.int64)).cuda()
        x = d.to(torch.int64)
        hit = torch.isin(x, tab)
        valid = _bits(v, fr.n_rows) if v is not None else torch.ones(fr.n_rows, dtype=torch.bool, device="cuda")
        hit &= valid
        counts.append(torch.bincount(torch.searchsorted(tab, x[hit]), minlength=len(t)))
        bms.append(_pack(valid & ~hit))
    return counts, bms


def main():
    print("card:", card())
    fr = build_frame()
    names, tables = fr.columns, tables_of(fr)
    torch.cuda.synchronize()
    nbytes = sum(rows * (8 if fr.column(n).anv_dtype == _lib.ANV_I64 else 4) +
                 ((rows + 7) // 8 if fr.column(n).has_validity else 0) for n in names)
    bm_bytes = len(names) * ((rows + 31) // 32) * 4
    count_ms = kernel_ms(lambda: engine.flag_members(fr, names, tables, False))
    bitmap_ms = kernel_ms(lambda: engine.flag_members(fr, names, tables, True))
    torch_ms = events(lambda: torch_flags(fr, names, tables))
    counts, bms = engine.flag_members(fr, names, tables, True)
    tc, tb = torch_flags(fr, names, tables)
    same = all(np.array_equal(c, x.cpu().numpy().astype(np.uint64)) for c, x in zip(counts, tc)) and \
        all(torch.equal(a, b) for a, b in zip(bms, tb))
    hits = int(sum(int(c.sum()) for c in counts))

    dic = ["w%07d" % i if i % 7 else "%03d" % (i % 1000) for i in range(1_000_000)]
    t0 = time.perf_counter()
    R.dictionary_table(dic, R.Rule())
    host_dict_auto = time.perf_counter() - t0
    t0 = time.perf_counter()
    R.dictionary_table(dic, R.Rule("manual", invalid_entries=["w00.*"], valid_entries=["w.*"]))
    host_dict_manual = time.perf_counter() - t0

    f32 = synth.device_frame(rows, 1)
    name = f32.columns[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    distinct = QC._distinct_numeric(f32, name)
    t1 = time.perf_counter()
    table = R.numeric_table(distinct, R.Rule())
    t2 = time.perf_counter()

    res = {"rows": rows, "columns": len(names), "card": card(), "hits": hits,
           "count_pass_ms": round(count_ms, 3), "count_pass_tbs": round(nbytes / count_ms / 1e9, 3),
           "count_pass_of_peak": round(nbytes / count_ms / 1e9 / (HBM_PEAK / 1e12), 3),
           "bitmap_pass_ms": round(bitmap_ms, 3), "bitmap_pass_tbs": round((nbytes + bm_bytes) / bitmap_ms / 1e9, 3),
           "bitmap_pass_of_peak": round((nbytes + bm_bytes) / bitmap_ms / 1e9 / (HBM_PEAK / 1e12), 3),
           "torch_ms": round(torch_ms, 3), "bit_identical": bool(same),
           "host_dictionary_1e6_auto_s": round(host_dict_auto, 3),
           "host_dictionary_1e6_manual_s": round(host_dict_manual, 3),
           "float32_distinct_values": int(len(distinct)), "float32_distinct_s": round(t1 - t0, 3),
           "float32_rule_s": round(t2 - t1, 3), "float32_invalid_values": int(len(table))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
