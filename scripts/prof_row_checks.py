"""Timing of the row-level quality checks at the c3 shape: synth.device_frame(40 M, 200, cat_every=4).
Three calls, each timed with CUDA events after a warm-up call, then a torch.profiler kernel breakdown in a separate run:
  null_rows   nullRows_detection on all 200 columns (reads the validity bitmaps only)
  dup_all     duplicate_detection(print_impact=True, treatment=False) on all 200 columns: nearly every row is unique, the
              work is the hash pass, the sort of the hash bytes and the prefix collisions
  dup_cat4    the same call on 4 string columns, one of each cardinality: duplicates are heavy, the work is the verify path
Prints the card and its power limit (read-only nvidia-smi query), the hash pass's algorithmic GB/s against the 3.35 TB/s
data-sheet figure, and one JSON line.  Usage: python scripts/prof_row_checks.py [rows] [reps]"""
import collections
import contextlib
import io
import json
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, ".")
import anovos.data_analyzer.quality_checker as qc   # noqa: E402
from anovos_b200 import engine, synth               # noqa: E402

rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 40_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
HBM_PEAK = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    fr = synth.device_frame(rows, 200, cat_every=4)
    cat = [c for c in fr.columns if fr.column(c).kind == "cat"]
    by_card = {}
    for c in cat:
        by_card.setdefault(len(fr.column(c).dictionary), c)
    cat4 = [by_card[k] for k in sorted(by_card)][:4]
    calls = {
        "null_rows": lambda: qc.nullRows_detection(None, fr),
        "dup_all": lambda: qc.duplicate_detection(None, fr, print_impact=True, treatment=False),
        "dup_cat4": lambda: qc.duplicate_detection(None, fr, list_of_cols=cat4, print_impact=True, treatment=False),
    }
    out = {"card": card(), "rows": rows, "cols": 200, "cat4": cat4, "ms": {}, "kernels_ms": {}}
    quiet = contextlib.redirect_stdout(io.StringIO())
    for name, fn in calls.items():
        with quiet:
            fn()                                   # warm-up: module load, allocator pools
        torch.cuda.synchronize()
        times = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            with quiet:
                res = fn()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        out["ms"][name] = times
        if name.startswith("dup"):
            out.setdefault("unique_rows", {})[name] = float(res[1].toPandas()["value"][1])
    # the hash pass alone: algorithmic bytes = one read of every column (+ bitmaps) + the 8-byte keys written
    engine.timer = engine.KernelTimer()
    for name in ("dup_all", "dup_cat4"):
        with quiet:
            calls[name]()
    tot = engine.timer.totals()
    engine.timer = None
    out["anv_row_distinct_calls"] = tot.get("anv_row_distinct")
    # separate profiled run: per-kernel device time
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, fn in calls.items():
            with quiet:
                fn()
        torch.cuda.synchronize()
    per = collections.defaultdict(float)
    for ev in prof.key_averages():
        if ev.device_type is not None and "cuda" in str(ev.device_type).lower():
            per[ev.key] += ev.device_time_total / 1000.0 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1000.0
    out["kernels_ms"] = {k: round(v, 3) for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:25]}
    hash_ms = sum(v for k, v in per.items() if "row_hash_kernel" in k)
    hash_bytes = engine_bytes(fr, fr.columns) + engine_bytes(fr, cat4) + 8 * rows * 2
    out["hash_pass"] = {"ms_both_calls": hash_ms, "bytes": hash_bytes,
                        "GBps": hash_bytes / (hash_ms * 1e-3) / 1e9 if hash_ms else None,
                        "share_of_3.35TBps": hash_bytes / (hash_ms * 1e-3) / HBM_PEAK if hash_ms else None}
    print(json.dumps(out))


def engine_bytes(fr, names):
    tot = 0
    for n in names:
        col = fr.column(n)
        tot += fr.n_rows * 4 + ((fr.n_rows + 7) // 8 if col.has_validity else 0)
    return tot


if __name__ == "__main__":
    main()
