"""Timing of monotonic_binning's label-class histogram (anv_class_hist, csrc/classhist.cu) on a frame built from
synth.device_frame's Philox columns (default 40 M rows x 60 float32 columns) plus a label whose event rate rises with the
first column (P(event) = sigmoid(x0 / 2), drawn from torch's Philox generator with a fixed seed):
  class_hist       one anv_class_hist pass over every column: the 18 candidate models (n = 20 .. 3, equal_range) of a
                   column merged into one threshold union, counted per (union slot, label class)
  k2_composite     the same tables from K2 (engine.histogram), one model at a time: 18 models x the all / event /
                   non-event views, 54 passes; every model's (rows, events, non-events) compared bit for bit
  k2_union         the cheapest K2 route: the three views binned once over each column's threshold union (3 passes;
                   K2 folds NaN into the last slot, so a torch count of the NaN rows per class completes the table);
                   compared bit for bit with the class-histogram slots
  monotonic_call   the whole monotonic_binning call (cutoffs, histogram, decision, final bin_assign)
Algorithmic bytes of a pass: one read of every column, its bitmap and the two class bitmaps; TB/s against the 3.35 TB/s
data-sheet HBM3 figure.  Prints the card and its power limit (read-only nvidia-smi query) and one JSON line.
Usage: python scripts/prof_monotonic.py [rows] [cols] [reps]"""
import json
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from anovos_b200 import _lib, engine, synth  # noqa: E402
from anovos_b200.data_transformer.transformers import monotonic_binning  # noqa: E402
from anovos_b200.frame import Column, ColumnFrame  # noqa: E402
from anovos_b200.shared import monotonic as M  # noqa: E402
from anovos_b200.shared.label_classes import label_bitmaps, masked  # noqa: E402

rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 40_000_000
ncols = int(sys.argv[2]) if len(sys.argv) > 2 else 60
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
HBM_PEAK = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def build_frame():
    src = synth.device_frame(rows, ncols)
    names = [n for n in src.columns if src.column(n).dictionary is None][:ncols]
    cols = {n: src.column(n) for n in names}
    x0, _ = src.column(names[0]).device()
    g = torch.Generator(device="cuda").manual_seed(1234)
    p = torch.sigmoid(torch.nan_to_num(x0.double(), nan=0.0) / 2)
    lab = (torch.rand(rows, generator=g, device="cuda", dtype=torch.float64) < p).to(torch.int32)
    cols["label"] = Column("label", "int", rows, dev=lab, anv_dtype=_lib.ANV_I32)
    return ColumnFrame(cols, rows), names


def timed(fn):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return out, float(np.median(ts))


def main():
    fr, names = build_frame()
    cuts, _ = M.ladder_cutoffs(fr, names, "equal_range")
    ums = [M.UnionModel(cuts[c], fr.column(c).anv_dtype) for c in names]
    thr = [u.thresholds for u in ums]
    ev, nev, _ = label_bitmaps(fr, "label", 1)
    hist, t_hist = timed(lambda: engine._class_hist_words(fr, names, thr, ev, nev))

    views = (fr, masked(fr, names, ev), masked(fr, names, nev))

    def k2():
        out = {}
        for n in M.LADDER:
            out[n] = [engine.histogram(v, engine.BinModel(v, names, [cuts[c][n] for c in names])) for v in views]
        return out
    k2_out, t_k2 = timed(k2)
    same = True
    for i, c in enumerate(names):
        for n in M.LADDER:
            tab = M.model_table(ums[i], hist[i], n)
            for t, h in zip(tab, k2_out[n]):
                same &= bool(np.array_equal(t[1:], h[i, 1:n + 1].astype(np.int64)))
    idx = torch.arange(rows, device="cuda")
    shift = (idx & 31).to(torch.int32)

    def bits(words):
        return ((words[idx >> 5] >> shift) & 1).bool()
    evb, nevb = bits(ev), bits(nev)

    def k2_union():
        h = [engine.histogram(v, engine.BinModel(v, names, [u.thresholds.astype(np.float64) for u in ums]))
             for v in views]
        nan = []
        for c in names:
            d, v = fr.column(c).device()
            isnan = torch.isnan(d) if v is None else torch.isnan(d) & bits(v)
            nan.append([int((isnan & w).sum().item()) for w in (evb, nevb)])
        return h, nan
    (k2u, k2u_nan), t_k2u = timed(k2_union)
    for i in range(len(names)):
        u = len(ums[i].thresholds)
        c = hist[i][:3 * ums[i].n_slots].astype(np.int64).reshape(3, ums[i].n_slots)
        for j, want in enumerate((c.sum(0), c[0], c[1])):
            got = k2u[j][i, 1:u + 2].astype(np.int64)
            slots = want[1:u + 2].copy()
            slots[-1] += want[u + 2]                               # K2's last slot holds the NaN rows too
            same &= bool(np.array_equal(got, slots))
            if j:
                same &= k2u_nan[i][j - 1] == int(want[u + 2])
    _, t_call = timed(lambda: monotonic_binning(None, fr, names, label_col="label", event_label=1))
    nbytes = sum(rows * 4 + ((rows + 7) // 8 if fr.column(c).has_validity else 0) for c in names) \
        + len(names) * 2 * ((rows + 31) // 32) * 4
    res = {"card": card(), "rows": rows, "cols": len(names), "class_hist_ms": round(t_hist, 3),
           "class_hist_TBps": round(nbytes / t_hist / 1e9, 3), "k2_composite_ms": round(t_k2, 3),
           "speedup": round(t_k2 / t_hist, 2),
           "k2_union_ms": round(t_k2u, 3), "speedup_vs_union": round(t_k2u / t_hist, 2), "monotonic_call_ms": round(t_call, 3), "tables_identical": same,
           "chosen_n_first_cols": [M.choose(ums[i], hist[i]) for i in range(min(4, len(names)))]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
