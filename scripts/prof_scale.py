"""Timing of the scalers on synth.device_frame(rows, cols) float columns (default 40 M x 60: the inputs and 60 double
outputs fit in 80 GB together).
  api_cold / api_warm  z_standardization, IQR_standardization and normalization on a fresh frame, then again on the same
                       frame (statistics from the frame's cache; the scale pass runs again)
  z_pass / norm_pass   anv_scale_columns alone with the z specs (DIV, double out) and the normalization specs (AFFINE,
                       float out, NaN to null), CUDA events over repeated launches
  torch                the same formulas as torch composites (true division by a device scalar, so no reciprocal
                       multiply); outputs compared with the kernel's bit for bit, one column at a time
Algorithmic bytes of a pass: one read of the values and bitmaps, one write of the outputs (and of the bitmaps the
normalization pass writes); GB/s against the 3.35 TB/s data-sheet HBM3 figure.  Prints the card and its power limit
(read-only nvidia-smi query) and one JSON line.  Usage: python scripts/prof_scale.py [rows] [cols] [reps]"""
import contextlib
import io
import json
import subprocess
import sys
import time
import warnings

import torch

sys.path.insert(0, ".")
import anovos.data_transformer.transformers as T   # noqa: E402
from anovos_b200 import _lib, engine, profile, synth  # noqa: E402
from anovos_b200.data_transformer import transformers as TB  # noqa: E402

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


def torch_scale(fr, name, spec):
    """One column of anv_scale_columns as torch ops -> (values, keep mask)."""
    mode, od, fl, a, b, c = spec
    d, v = fr.column(name).device()
    r = torch.arange(fr.n_rows, device="cuda")
    keep = torch.ones(fr.n_rows, dtype=torch.bool, device="cuda") if v is None else ((v[r >> 5] >> (r & 31).to(torch.int32)) & 1).bool()
    x = d.double()
    A, B, Cc = (torch.tensor(z, dtype=torch.float64, device="cuda") for z in (a, b, c))
    if mode == _lib.SCALE_DIV:
        y = (x - A) / B
    elif mode == _lib.SCALE_AFFINE:
        y = (x - A) * B + Cc
    else:
        y = Cc.expand_as(x)
    if fl & _lib.SCALE_NAN_TO_NULL:
        keep = keep & ~torch.isnan(x) & ~torch.isnan(y)
    y = y.float() if od == _lib.ANV_F32 else y
    return torch.where(keep, y, torch.zeros((), dtype=y.dtype, device="cuda")), keep


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    out = {"card": card(), "rows": rows, "cols": ncols}
    quiet = contextlib.redirect_stdout(io.StringIO())
    fr = synth.device_frame(rows, ncols)
    torch.cuda.synchronize()
    names = list(fr.columns)
    calls = {"z": lambda: T.z_standardization(None, fr, list_of_cols=names),
             "iqr": lambda: T.IQR_standardization(None, fr, list_of_cols=names),
             "norm": lambda: T.normalization(fr, list_of_cols=names)}
    for key, call in calls.items():
        for phase in ("cold", "warm"):
            odf = None                                 # free the previous outputs first
            t0 = time.perf_counter()
            with quiet, warnings.catch_warnings():
                warnings.simplefilter("ignore")
                odf = call()
            torch.cuda.synchronize()
            out["api_%s_%s_ms" % (key, phase)] = (time.perf_counter() - t0) * 1e3
        odf = None
    mom = profile.moments(fr, names)
    z_specs, n_specs = [], []
    for c in names:
        r = mom[c]
        z_specs.append((_lib.SCALE_DIV, _lib.ANV_F64, 0, float(r["mean"]), TB._stddev(r), 0.0))
        n_specs.append(TB.minmax_spec(float(r["min"]), float(r["max"])))
    in_bytes = sum(rows * 4 + ((rows + 7) // 8 if fr.column(c).has_validity else 0) for c in names)
    same = True
    for key, specs, ob in (("z", z_specs, 8), ("norm", n_specs, 4)):
        ms = events(lambda: engine.scale_columns(fr, names, specs), reps)
        nbytes = in_bytes + len(names) * rows * ob + (len(names) * ((rows + 31) // 32) * 4 if key == "norm" else 0)
        out[key + "_pass_ms"] = ms
        out[key + "_pass_bytes"] = nbytes
        out[key + "_pass_GBps"] = nbytes / ms / 1e6
        out[key + "_pass_pct_of_datasheet_3.35TBps"] = 100 * nbytes / (ms * 1e-3) / HBM_PEAK
        out[key + "_torch_ms"] = events(lambda: [torch_scale(fr, c, s)[0].data_ptr() for c, s in zip(names, specs)], reps)
        data, valid, _ = engine.scale_columns(fr, names, specs)
        for i, (c, s) in enumerate(zip(names, specs)):
            y, keep = torch_scale(fr, c, s)
            same = same and torch.equal(data[i].view(torch.uint8), y.view(torch.uint8))
            if valid[i] is not None:
                r = torch.arange(rows, device="cuda")
                bits = ((valid[i][r >> 5] >> (r & 31).to(torch.int32)) & 1).bool()
                same = same and torch.equal(bits, keep)
            data[i] = None
        del data, valid
    out["bit_identical"] = bool(same)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
