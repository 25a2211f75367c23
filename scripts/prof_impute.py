"""Timing of imputation_MMM at the c3 shape: synth.device_frame(40 M, 200, cat_every=4).
  api_cold   imputation_MMM(method_type="median") on a fresh frame: missing counts, moments, medians, modes, then the fill
  api_warm   the same call again on the same frame: the statistics come from the frame's cache, the fill runs again
  fill       anv_impute_fill alone over the columns that have nulls, CUDA events over repeated launches
  torch      the same fill as a torch.where composite (unpack the bitmap, select, cast): the comparison arm; its outputs
             are compared with the kernel's bit for bit
Algorithmic bytes of the fill: one read of the values and bitmaps and one write of the outputs of the columns with nulls;
GB/s against the 3.35 TB/s data-sheet HBM3 figure.  Prints the card and its power limit (read-only nvidia-smi query) and
one JSON line.  Usage: python scripts/prof_impute.py [rows] [reps]"""
import contextlib
import io
import json
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")
import anovos.data_transformer.transformers as T   # noqa: E402
from anovos_b200 import _lib, engine, synth          # noqa: E402

rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 40_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
HBM_PEAK = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def events(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def torch_fill(fr, names, fills):
    """The fill as torch ops: bitmap -> bool per row, where(valid, x, fill)."""
    out = []
    rows_ = torch.arange(fr.n_rows, device="cuda")
    shift = (rows_ & 31).to(torch.int32)
    for n, f in zip(names, fills):
        d, v = fr.column(n).device()
        if v is None:
            out.append(d.clone())
            continue
        keep = ((v[rows_ >> 5] >> shift) & 1).bool()
        out.append(torch.where(keep, d, torch.tensor(f, dtype=d.dtype, device="cuda")))
    return out


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    out = {"card": card(), "rows": rows, "cols": 200}
    quiet = contextlib.redirect_stdout(io.StringIO())
    fr = synth.device_frame(rows, 200, cat_every=4)
    torch.cuda.synchronize()
    odf = None
    for key in ("api_cold_ms", "api_warm_ms"):
        odf = None                                 # free the previous outputs first
        t0 = time.perf_counter()
        with quiet:
            odf = T.imputation_MMM(None, fr, method_type="median")
        torch.cuda.synchronize()
        out[key] = (time.perf_counter() - t0) * 1e3
    out["out_cols"] = len(odf.columns)
    odf = None
    names = [c for c in fr.columns if fr.column(c).has_validity]
    out["imputed_cols"] = len(names)
    fills = [1 if fr.column(c).kind == "cat" else 0.5 for c in names]
    od = [fr.column(c).anv_dtype for c in names]
    bits = [engine.fill_bits(engine.java_cast(f, d), d) for f, d in zip(fills, od)]
    for c in names:
        fr.column(c).device()
    ms = events(lambda: engine.impute_fill(fr, names, od, [0] * len(names), bits), reps)
    nbytes = sum(fr.n_rows * (4 if d in (_lib.ANV_F32, _lib.ANV_I32) else 8) * 2 + (fr.n_rows + 7) // 8 for d in od)
    out["fill_ms"] = ms
    out["fill_bytes"] = nbytes
    out["fill_GBps"] = nbytes / ms / 1e6
    out["fill_pct_of_datasheet_3.35TBps"] = 100 * nbytes / (ms * 1e-3) / HBM_PEAK
    tfills = [engine.java_cast(f, d) for f, d in zip(fills, od)]
    out["torch_where_ms"] = events(lambda: torch_fill(fr, names, tfills), reps)
    a = engine.impute_fill(fr, names, od, [0] * len(names), bits)
    same = True
    for i, n in enumerate(names):                  # one torch column at a time: both arms at once would not fit
        b = torch_fill(fr, [n], tfills[i:i + 1])[0]
        same = same and torch.equal(a[i].contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))
        a[i] = None
    out["bit_identical"] = bool(same)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
