"""Timing + result checksum of the LSD radix sort path (anv_mode_distinct with ranks and HLL++ registers) on synthetic
float32 columns resident in HBM; key_bits 64 sorts the same columns as float64 (the 64-bit instantiation).  Run once per
library variant (ANOVOS_B200_LIB) and compare the checksums.  Prints one JSON line.
Usage: python scripts/sort_ab.py [rows] [cols] [tag] [key_bits: 32 | 64]"""
import hashlib
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from anovos_b200 import engine, profile, synth
from anovos_b200.frame import ColumnFrame

rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
cols = int(sys.argv[2]) if len(sys.argv) > 2 else 12
tag = sys.argv[3] if len(sys.argv) > 3 else "default"
key_bits = int(sys.argv[4]) if len(sys.argv) > 4 else 32
engine.sort_algorithm = "lsd"      # float32 columns would otherwise take the two-level bucket count
fr = synth.device_frame(rows, cols)
names = fr.columns
if key_bits == 64:
    fr = ColumnFrame.from_tensors({n: (fr.column(n).device()[0].double(), fr.column(n).device()[1]) for n in names})
mom = engine.moments(fr, names)
ranks = np.array([engine.quantile_ranks(int(mom["n_valid"][i]), profile.SUMMARY_PROBS) for i in range(cols)])


def run():
    return engine.sort_mode_distinct(fr, names, ranks=ranks, hll_p=9)


res = run()
torch.cuda.synchronize()
engine.timer = engine.KernelTimer()
for _ in range(4):
    run()
tot = engine.timer.totals()
engine.timer = None
h = hashlib.sha1()
h.update(repr(res[0]).encode()); h.update(np.ascontiguousarray(res[1]).tobytes()); h.update(np.ascontiguousarray(res[2]).tobytes())
k = tot["anv_mode_distinct"]
print(json.dumps({"tag": tag, "rows": rows, "cols": cols, "key_bits": key_bits, "ms_per_call": k["ms"] / k["calls"], "ms_per_column": k["ms"] / k["calls"] / cols * (k["calls"] / 4),
                  "calls": k["calls"], "checksum": h.hexdigest()}))
