"""Timing of the exact mode / distinct count (engine.sort_mode_distinct) on one float32 column of 40 M, 2^31 + 4 099 and
2^32 - 1 rows, through the two-level bucket count (sort_algorithm = "partition") and the LSD radix sort ("lsd").

The column is the closed-form column of tests/test_gpu_long_columns.py without nulls: row r holds T[(A r + B) mod 65521],
T the "special" table (quarter steps of a normal spread, -0.0 / +0.0, NaN payloads, subnormals, +-FLT_MAX, +-inf).  About
49 k distinct values, so a fine bucket of the bucket count holds about n / 8 192 keys and on long columns takes many
hash-class sweeps.  The two algorithms run alternately, after one warm-up call each; both workspaces stay cached, except
at 2^32 - 1 rows, where the two together do not fit in 80 GB: there each algorithm runs its calls back to back and the
cache is emptied in between.  A call is timed by the host clock around the call and a device synchronise (the result
comes back to the host inside the call).  The two algorithms' results are compared.  Prints the card and its power
limit (read-only nvidia-smi query), one line per call and one JSON line.
Usage: python scripts/prof_long_columns.py [reps] [rows ...]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import closed_form as CF                                  # noqa: E402
from anovos_b200 import _lib, engine                      # noqa: E402
from anovos_b200.frame import ColumnFrame                 # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
sizes = [int(float(a)) for a in sys.argv[2:]] or [40_000_000, (1 << 31) + 4099, (1 << 32) - 1]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def column(n):
    T = torch.from_numpy(CF.table_f32_special(11)).cuda()
    data = torch.empty((n + 3) // 4 * 4, dtype=torch.float32, device="cuda")
    for r0 in range(0, n, CF.BLOCK):
        r = torch.arange(r0, min(n, r0 + CF.BLOCK), device="cuda")
        data[r0:r0 + r.numel()] = T[(r * CF.A + CF.B) % CF.M]
    return ColumnFrame.from_tensors({"x": data[:n]})


def call(fr, algo):
    engine.sort_algorithm = algo
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = engine.sort_mode_distinct(fr, ["x"])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, res[0]


def main():
    _lib.require_cuda()
    out = {"card": card(), "reps": reps, "sizes": {}}
    print(out["card"], flush=True)
    for n in sizes:
        fr = column(n)
        both = 2 * 4 * n + _lib.lib().anv_mode_distinct_partition_workspace_bytes(1, n) + \
            _lib.lib().anv_mode_distinct_workspace_bytes(1, n, 32)
        alternate = both < torch.cuda.mem_get_info()[0] * 0.9
        times = {"partition": [], "lsd": []}
        results = {}
        order = [a for _ in range(reps) for a in ("partition", "lsd")] if alternate else \
            ["partition"] * reps + ["lsd"] * reps
        warmed = set()
        for algo in order:
            if algo not in warmed:
                if not alternate:
                    torch.cuda.empty_cache()
                _, results[algo] = call(fr, algo)
                warmed.add(algo)
            ms, res = call(fr, algo)
            assert res == results[algo]
            times[algo].append(ms)
            print("rows %d  %-9s  %.1f ms" % (n, algo, ms), flush=True)
        assert results["partition"] == results["lsd"], results
        med = {a: float(np.median(t)) for a, t in times.items()}
        out["sizes"][str(n)] = {"alternating": alternate, "ms": times, "median_ms": med,
                                "lsd_over_partition": med["lsd"] / med["partition"],
                                "keys_per_s": {a: n / (m * 1e-3) for a, m in med.items()}, "result": list(results["lsd"])}
        print("rows %d  median  partition %.1f ms  lsd %.1f ms  (lsd / partition %.2f)  result %s"
              % (n, med["partition"], med["lsd"], med["lsd"] / med["partition"], results["lsd"]), flush=True)
        del fr
        torch.cuda.empty_cache()
    engine.sort_algorithm = "partition"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
