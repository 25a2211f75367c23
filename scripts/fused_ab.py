"""A/B of the fused moments + histogram pass: cp.async-staged loop (ANV_FUSED_STAGED=1) vs register-staged loop (=0), same
process, alternating, on synthetic float32 columns resident in HBM (null rates as in bench.py's c3).  Prints one JSON line.
Usage: python scripts/fused_ab.py [rows] [cols] [null_mode] [tag]"""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from anovos_b200 import _lib, engine
from anovos_b200.frame import ColumnFrame

rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
cols = int(sys.argv[2]) if len(sys.argv) > 2 else 40
null_mode = sys.argv[3] if len(sys.argv) > 3 else "mixed"
tag = sys.argv[4] if len(sys.argv) > 4 else "default"
L = _lib.lib()
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
data = {}
for c in range(cols):
    x = torch.empty(rows, dtype=torch.float32, device="cuda")
    fam = c % 4
    rate = {"none": 0.0, "all": 0.02, "mixed": [0.0, 0.001, 0.02, 0.3][c % 4]}[null_mode]
    v = torch.zeros((rows + 31) // 32, dtype=torch.int32, device="cuda") if rate > 0 else None
    a, b = [(5.0 + c, 1.0 + 0.1 * c), (0.0, 0.75), (-3.0 - c, 7.0 + c), (0.0, 2.0)][fam]
    _lib.check(L.anv_synth_f32(x.data_ptr(), v.data_ptr() if v is not None else None, rows, 42, c, fam, a, b, rate, st))
    data["c%03d" % c] = (x, v) if v is not None else x
torch.cuda.synchronize()
fr = ColumnFrame.from_tensors(data)
names = fr.columns
mom = engine.moments(fr, names)
cuts = [[float(mom["min"][i]) + j * ((float(mom["max"][i]) - float(mom["min"][i])) / 10) for j in range(1, 10)] for i in range(cols)]
model = engine.BinModel(fr, names, cuts, [(float(mom["min"][i]), float(mom["max"][i])) for i in range(cols)])
nbytes = rows * cols * 4 + sum((rows + 7) // 8 for c in range(cols) if isinstance(data["c%03d" % c], tuple))
desc, keep = fr.descriptors(names)
specs, dcuts = model.device()
ws_bytes = L.anv_moments_workspace_bytes(cols, rows)
ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")


def run(flag):
    os.environ["ANV_FUSED_STAGED"] = flag
    out = torch.zeros(cols * 64, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(cols * 11 * 8, dtype=torch.uint8, device="cuda")
    fn = lambda: _lib.check(L.anv_moments_hist(desc.data_ptr(), specs.data_ptr(), dcuts.data_ptr(), cols, rows, out.data_ptr(),
                                               counts.data_ptr(), 11, ws.data_ptr(), ws_bytes, st))
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(8):
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(np.min(ts)), out.cpu().numpy().tobytes(), counts.cpu().numpy().tobytes()


def sustained(flag, launches=80):
    """Enqueue `launches` back to back and sample NVML (SM clock, power, throttle reasons) while they run: the pass is
    FP64- and HBM-heavy, and a GPU under its power cap lowers the SM clock within a few hundred milliseconds."""
    import time
    import pynvml
    pynvml.nvmlInit()
    h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
    os.environ["ANV_FUSED_STAGED"] = flag
    out = torch.zeros(cols * 64, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(cols * 11 * 8, dtype=torch.uint8, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        _lib.check(L.anv_moments_hist(desc.data_ptr(), specs.data_ptr(), dcuts.data_ptr(), cols, rows, out.data_ptr(),
                                      counts.data_ptr(), 11, ws.data_ptr(), ws_bytes, st))
    e1.record()
    mhz, watts, reasons = [], [], set()
    while not e1.query():
        mhz.append(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM))
        watts.append(pynvml.nvmlDeviceGetPowerUsage(h) / 1e3)
        r = pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(h)
        for name in ("SwPowerCap", "HwSlowdown", "SwThermalSlowdown", "HwThermalSlowdown", "HwPowerBrakeSlowdown"):
            if r & getattr(pynvml, "nvmlClocksThrottleReason" + name, 0):
                reasons.add(name)
        time.sleep(0.02)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / launches
    return {"ms_per_launch": ms, "gbs": nbytes / ms / 1e6, "launches": launches, "sm_mhz_first": mhz[:3], "sm_mhz_median": float(np.median(mhz)) if mhz else None,
            "sm_mhz_min": min(mhz) if mhz else None, "sm_mhz_max": pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM),
            "power_w_max": max(watts) if watts else None, "reasons": sorted(reasons), "samples": len(mhz)}


res = {}
r0 = run("0"); r1 = run("1"); r0b = run("0"); r1b = run("1")
peak = 6566.7
try:
    peak = json.load(open("MEASURED_PEAKS.json")).get("hbm_gbs", peak)
except Exception:
    pass
line = {"tag": tag, "rows": rows, "cols": cols, "nulls": null_mode, "bytes": nbytes,
        "register_staged_ms": [r0[0], r0b[0]], "cp_async_staged_ms": [r1[0], r1b[0]],
        "register_staged_gbs": nbytes / min(r0[0], r0b[0]) / 1e6, "cp_async_staged_gbs": nbytes / min(r1[0], r1b[0]) / 1e6,
        "bit_identical": r0[2] == r1[2] and r0[3] == r1[3]}
if os.environ.get("FUSED_AB_SUSTAINED", "1") != "0":
    try:
        line["sustained_default_loop"] = sustained("1")
        line["sustained_register_staged"] = sustained("0")
    except Exception as e:   # no NVML on the box: the burst numbers stand alone
        line["sustained_error"] = repr(e)
print(json.dumps(line))
