"""ncu launch list (--metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --csv) of a
`bench.py --steps S --warmup W --no-extras` run -> profiles/<name>.json (DRAM bytes per C call per step: bench.py reads it
for `roofline.traffic`) and profiles/<name>.md (per-kernel time share, DRAM bytes, GB/s).

    python scripts/traffic_summary.py gpurun_out/traffic_c3.csv profiles/r2_traffic_c3 --rows 100000000 --cols 200 --cat-every 4 --steps 2
"""
import argparse
import collections
import csv
import json
import re

CALL_OF = [  # first match wins
    (r"pc_", "anv_mode_distinct_partition"),
    (r"pack_kernel|run_tile|run_merge", "anv_mode_distinct"),
    (r"sort_hist|sort_totals|sort_scan|sort_scatter", "SORT"),      # LSD passes: the full sort, or the sample sort of the partition path
    (r"hll_kernel", "anv_hll_registers"),
    (r"scan_kernel<\(bool\)1, \(int\)-1|scan_kernel<1, *\(?i?n?t?\)?-1|finalize_moments", "anv_moments"),
    (r"scan_kernel<\(bool\)1|scan_kernel<1", "anv_moments_hist"),
    (r"scan_kernel<\(bool\)0|scan_kernel<0", "anv_hist_codes"),
    (r"select_", "anv_select_ranks"),
    (r"drift_reduce", "anv_drift_reduce"),
    (r"synth_", "generator (not part of the step)"),
]


# one launch of these kernels = one C call (to turn the capture into bytes per CALL, whatever the number of calls per step)
CALL_MARK = {"anv_moments": r"finalize_moments", "anv_mode_distinct": r"run_merge", "anv_mode_distinct_partition": r"pc_final",
             "anv_hll_registers": r"hll_kernel", "anv_hist_codes": r"scan_kernel<\(bool\)0|scan_kernel<0", "anv_moments_hist": r"finalize_moments",
             "anv_select_ranks": None, "anv_drift_reduce": r"drift_reduce"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("out")
    ap.add_argument("--rows", type=int, required=True)
    ap.add_argument("--cols", type=int, required=True)
    ap.add_argument("--cat-every", type=int, default=0)
    ap.add_argument("--steps", type=int, required=True, help="steps + warm-up steps the capture covers")
    ap.add_argument("--command", default="")
    a = ap.parse_args()
    lines = open(a.csv).readlines()
    start = [i for i, l in enumerate(lines) if l.startswith('"ID"')][0]
    per = collections.defaultdict(lambda: collections.defaultdict(float))
    launches = collections.Counter()
    for r in csv.DictReader(lines[start:]):
        k = re.sub(r"\(anv::.*", "", r["Kernel Name"]).replace("void ", "").strip()
        v = float(r["Metric Value"].replace(",", ""))
        u, m = r["Metric Unit"], r["Metric Name"]
        if m.startswith("dram"):
            per[k][m] += v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[u]
        else:
            per[k]["ms"] += v * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(u, 1e-6)
            launches[k] += 1
    partition = any("pc_" in k for k in per)
    calls = collections.defaultdict(lambda: collections.defaultdict(float))
    rows = []
    total_ms = sum(v["ms"] for k, v in per.items() if "synth" not in k and "at::" not in k)
    for k, v in sorted(per.items(), key=lambda kv: -kv[1]["ms"]):
        call = next((c for pat, c in CALL_OF if re.search(pat, k)), "other")
        if call == "SORT":
            call = "anv_mode_distinct_partition" if partition else "anv_mode_distinct"
        tr = v["dram__bytes_read.sum"] + v["dram__bytes_write.sum"]
        calls[call]["bytes"] += tr
        calls[call]["ms"] += v["ms"]
        rows.append((k, call, launches[k], v["ms"], tr))
    n_calls = {}
    for call, pat in CALL_MARK.items():
        if pat and call in calls:
            n_calls[call] = sum(n for k, n in launches.items() if re.search(pat, k)) or None
    out = {"workload_rows": a.rows, "rows": a.rows, "cols": a.cols, "cat_every": a.cat_every, "steps_captured": a.steps,
           "calls_captured": n_calls,
           "dram_bytes_per_launch": {c: calls[c]["bytes"] / n for c, n in n_calls.items() if n},
           "source": a.csv + " (ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none; "
                     + (a.command or "bench.py --no-extras") + "); bytes of every kernel a C call launches, per step; times are ncu's "
                     "serialised cold-cache times: compare shares, not absolutes",
           "dram_bytes_per_step": {c: v["bytes"] / a.steps for c, v in calls.items() if not c.startswith(("generator", "other"))},
           "ncu_ms_per_step": {c: v["ms"] / a.steps for c, v in calls.items() if not c.startswith(("generator", "other"))}}
    json.dump(out, open(a.out + ".json", "w"), indent=1)
    with open(a.out + ".md", "w") as f:
        f.write("# ncu launch list: %s\n\n%d rows x %d cols (cat_every=%d), %d steps captured; kernel time of the steps %.1f ms "
                "(generator and torch fill kernels excluded from the share)\n\n" % (a.csv, a.rows, a.cols, a.cat_every, a.steps, total_ms))
        f.write("| kernel | C call | launches | ms | share | DRAM GB | GB/s |\n|---|---|---|---|---|---|---|\n")
        for k, call, n, ms, tr in rows:
            if "at::" in k:
                continue
            f.write("| `%s` | %s | %d | %.2f | %.1f %% | %.2f | %.0f |\n" % (k[:70], call, n, ms, 100 * ms / total_ms if "synth" not in k else 0.0,
                                                                             tr / 1e9, tr / 1e6 / max(ms, 1e-9)))
    print(json.dumps(out["dram_bytes_per_step"], indent=1))


if __name__ == "__main__":
    main()
