"""Timing of anv_transform_columns on synth.device_frame(rows, cols) float columns (default 40 M x 60).
  <op>_pass     the transform pass alone, CUDA events over repeated launches, for ln, toPowerN with N = 0.5 (fdlibm pow
                returns sqrt(x) for y = 0.5), toPowerN with N = 0.3 (the full fdlibm pow), roundN with N = 2, and sqrt,
                floor and mul_inv
  <op>_torch    the same op as a torch composite (torch.log / torch.pow are CUDA's, not fdlibm's: a speed reference only);
                sqrt, floor and mul_inv are exact in both, so those outputs are compared bit for bit
  ks_candidates  the Box-Cox search's one sort + candidate pass per column (engine.ks_candidates), 8 columns; the
                synthetic columns are not all positive, which changes no work the kernels do
Algorithmic bytes of a pass: one read of the values and bitmaps, one write of the outputs (and of the bitmaps of ln and
mul_inv).  The FP64 operations of a pow pass are not counted here: pow is reported against the HBM bound, and its time
above that bound is the FP64 pipe's.  Prints the card and its power limit (read-only nvidia-smi query) and one JSON
line.  Usage: python scripts/prof_transform.py [rows] [cols] [reps]"""
import json
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from anovos_b200 import _lib, engine, synth  # noqa: E402

rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 40_000_000
ncols = int(sys.argv[2]) if len(sys.argv) > 2 else 60
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
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


def keep_mask(fr, name):
    d, v = fr.column(name).device()
    if v is None:
        return torch.ones(fr.n_rows, dtype=torch.bool, device="cuda")
    r = torch.arange(fr.n_rows, device="cuda")
    return ((v[r >> 5] >> (r & 31).to(torch.int32)) & 1).bool()


TORCH = {"ln": lambda x: torch.log(x), "pow05": lambda x: torch.pow(x, 0.5), "pow03": lambda x: torch.pow(x, 0.3),
         "round2": lambda x: torch.round(x, decimals=2), "sqrt": lambda x: torch.sqrt(x),
         "floor": lambda x: torch.floor(x).to(torch.int64), "mul_inv": lambda x: 1.0 / x}
SPECS = {"ln": (_lib.TF_LN, _lib.ANV_F64, 0, 0.0), "pow05": (_lib.TF_POW, _lib.ANV_F64, 0, 0.5),
         "pow03": (_lib.TF_POW, _lib.ANV_F64, 0, 0.3), "round2": (_lib.TF_ROUND, _lib.ANV_F32, 2, 0.0),
         "sqrt": (_lib.TF_SQRT, _lib.ANV_F64, 0, 0.0), "floor": (_lib.TF_FLOOR, _lib.ANV_I64, 0, 0.0),
         "mul_inv": (_lib.TF_MUL_INV, _lib.ANV_F64, 0, 0.0)}
EXACT = ("sqrt", "floor", "mul_inv")


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    out = {"card": card(), "rows": rows, "cols": ncols}
    fr = synth.device_frame(rows, ncols)
    torch.cuda.synchronize()
    names = list(fr.columns)
    in_bytes = sum(rows * 4 + ((rows + 7) // 8 if fr.column(c).has_validity else 0) for c in names)
    same = True
    for key, spec in SPECS.items():
        specs = [spec] * len(names)
        ob = 4 if spec[1] == _lib.ANV_F32 else 8
        ms = events(lambda: engine.transform_columns(fr, names, specs), reps)
        nbytes = in_bytes + len(names) * rows * ob + (len(names) * ((rows + 31) // 32) * 4 if spec[0] in _lib.TF_MAKES_NULLS else 0)
        out[key + "_pass_ms"] = ms
        out[key + "_pass_GBps"] = nbytes / ms / 1e6
        out[key + "_pass_pct_of_datasheet_3.35TBps"] = 100 * nbytes / (ms * 1e-3) / HBM_PEAK
        f = TORCH[key]
        out[key + "_torch_ms"] = events(lambda: [f(fr.column(c).device()[0].double() if key != "round2" else
                                                   fr.column(c).device()[0]).data_ptr() for c in names], reps)
        if key in EXACT:
            data, _, _ = engine.transform_columns(fr, names, specs)
            for i, c in enumerate(names):
                keep = keep_mask(fr, c)
                if spec[0] == _lib.TF_MUL_INV:
                    keep = keep & (fr.column(c).device()[0] != 0)
                y = f(fr.column(c).device()[0].double())
                y = torch.where(keep, y, torch.zeros((), dtype=y.dtype, device="cuda"))
                same = same and torch.equal(data[i].view(torch.uint8), y.view(torch.uint8))
                data[i] = None
            del data
    out["exact_ops_bit_identical_to_torch"] = bool(same)
    # the Box-Cox lambda search: one sort + one candidate pass per column (8 columns: the sort dominates)
    from anovos_b200.data_transformer.transformers import BOXCOX_LAMBDAS
    del fr
    pos = synth.device_frame(rows, 8)
    ks_names = list(pos.columns)
    n_null = {c: rows - int(r["n_valid"]) for c, r in zip(ks_names, engine.moments(pos, ks_names))}
    ms = events(lambda: [engine.ks_candidates(pos, c, BOXCOX_LAMBDAS, n_null[c]) for c in ks_names], 1)
    out["ks_candidates_ms_per_column"] = ms / len(ks_names)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
