"""Kernel breakdown of one sort_mode_distinct call (exact mode, distinct count, percentiles and HLL++ registers) at the
default bench shape: the numeric columns of synth.device_frame(rows, cols, cat_every=4), with the summary ranks and hll_p
the stats_generator step passes, so the column batching matches the step.  algo: "partition" (the default two-level bucket
count for 32-bit columns) or "lsd" (the radix sort for every column).
torch.profiler with CUDA activities; prints ms per call for each kernel family next to the HBM bytes the family needs at
these shapes (computed from the column sizes, not measured) and the rate that implies, the card and its power limit, and
one JSON line.  hll_p = 0 leaves the HLL++ registers out and ranks = 0 the percentile ranks, so that a stage's time can
be split into counting, hashing and selection.
Usage: python scripts/prof_sort.py [rows] [cols] [calls] [tag] [algo] [hll_p] [ranks: 1 | 0]"""
import collections
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, ".")
from anovos_b200 import engine, synth
from anovos_b200 import profile as anv_profile

rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 40_000_000
cols = int(sys.argv[2]) if len(sys.argv) > 2 else 200
calls = int(sys.argv[3]) if len(sys.argv) > 3 else 2
tag = sys.argv[4] if len(sys.argv) > 4 else "default"
algo = sys.argv[5] if len(sys.argv) > 5 else "partition"
hll_p = int(sys.argv[6]) if len(sys.argv) > 6 else anv_profile.DEFAULT_HLL_P
with_ranks = (sys.argv[7] != "0") if len(sys.argv) > 7 else True
engine.sort_algorithm = algo

FAMILIES = ["pack_kernel", "sort_bases_kernel", "sort_hist_kernel", "sort_totals_kernel", "sort_scan_kernel",
            "sort_scatter_kernel", "sort_onesweep_kernel", "run_tile_kernel", "run_merge_kernel",
            "pc_sample_kernel", "pc_split_kernel", "pc_coarse_kernel", "pc_chunks_kernel", "pc_fine_kernel", "pc_cum_kernel",
            "pc_group_kernel", "pc_direct_kernel", "pc_final_kernel", "pc_partition_kernel", "pc_count_kernel"]


def family(name):
    for f in FAMILIES:
        if f in name:
            return f.replace("_kernel", "").replace("sort_", "")
    return "other"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
        name, plim = [s.strip() for s in q.split(",")]
        return name, plim
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


fr = synth.device_frame(rows, cols, cat_every=4)
num = [n for n in fr.columns if fr.column(n).kind == "num"]
mom = engine.moments(fr, num)
n_valid = np.array([int(mom["n_valid"][i]) for i in range(len(num))], dtype=np.int64)
keys = int(np.array([int(mom["n_nonzero"][i]) for i in range(len(num))], dtype=np.int64).sum())   # nonzero non-null values
raw = sum(fr.n_rows * 4 + (fr.n_rows + 7) // 8 * bool(fr.column(n).has_validity) for n in num)   # 32-bit columns + bitmaps
# HBM bytes per family at these shapes (the keys equal to a fine splitter are counted as moved: an upper bound).  The count
# stage reads every key once, split between pc_group (hash buckets) and pc_direct (direct buckets) by the data: its 4 bytes
# per key are set against each kernel alone and against the two together ("count").
if algo == "partition":
    BYTES = {"pc_coarse": raw + 4 * keys, "pc_fine": 8 * keys, "pc_group": 4 * keys, "pc_direct": 4 * keys, "count": 4 * keys}
else:
    BYTES = {"pack": raw + 4 * keys, "hist": 4 * 4 * keys, "scatter": 4 * 8 * keys, "run_tile": 4 * keys}
ranks = np.array([engine.quantile_ranks(int(mom["n_valid"][i]), anv_profile.SUMMARY_PROBS, anv_profile.SUMMARY_EPS)
                  for i in range(len(num))], dtype=np.int64)


def run():
    return engine.sort_mode_distinct(fr, num, ranks if with_ranks else None, hll_p=hll_p or None)


run()                                   # warm-up: module load, workspace
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(calls):
        run()
    torch.cuda.synchronize()

with tempfile.TemporaryDirectory() as d:   # the kernel records of the chrome trace: name + duration in us
    prof.export_chrome_trace(os.path.join(d, "trace.json"))
    with open(os.path.join(d, "trace.json")) as f:
        trace = json.load(f)
ms = collections.Counter()
launches = collections.Counter()
for ev in trace["traceEvents"]:
    if ev.get("cat") == "kernel":
        f = family(ev["name"])
        ms[f] += ev["dur"] / 1e3 / calls
        launches[f] += 1
total = sum(ms.values())
if algo == "partition":
    ms["count"] = ms["pc_group"] + ms["pc_direct"]   # not a kernel: left out of the total
gpu, plim = card()
print("%s, power limit %s; %s path, %d rows x %d numeric columns, %.2f G nonzero keys, hll_p %d, %s ranks, per call:"
      % (gpu, plim, algo, rows, len(num), keys / 1e9, hll_p, "with" if with_ranks else "no"))
for f, t in sorted(ms.items(), key=lambda kv: -kv[1]):
    b = BYTES.get(f)
    rate = ("  %6.1f GB  %6.0f GB/s" % (b / 1e9, b / 1e6 / t)) if b and t > 0 else ""
    print("  %-12s %8.2f ms  %5.1f %%  (%d launches per call)%s" % (f, t, 100 * t / total, launches[f] // calls, rate))
    if f == "count":
        print("  %-12s (pc_group + pc_direct, not in the total)" % "")
print("  %-12s %8.2f ms" % ("total", total))
print(json.dumps({"tag": tag, "algo": algo, "gpu": gpu, "power_limit": plim, "rows": rows, "numeric_cols": len(num),
                  "hll_p": hll_p, "ranks": with_ranks,
                  "calls": calls, "kernel_ms_per_call": round(total, 3), "ms_per_call": {f: round(t, 3) for f, t in ms.items()},
                  "hbm_gb": {f: round(b / 1e9, 2) for f, b in BYTES.items()}}))
