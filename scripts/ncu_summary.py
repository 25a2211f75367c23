"""Turn ncu captures into the summaries committed under profiles/.

    python scripts/ncu_summary.py full   gpurun_out/r1_full.ncu-rep  profiles/r1_ncu_kernels   [rows cols]
    python scripts/ncu_summary.py launch gpurun_out/launches.csv     profiles/r1_launches_c2

`full`  : one row per profiled kernel of an `ncu --set full` report (time, DRAM bytes, pipe utilisation,
          stall picture) as .md + .json, and profiles/r1_traffic.json (dram bytes per launch of the scan
          kernels, read by bench.py for roofline.traffic).
`launch`: the `--metrics gpu__time_duration.sum` launch list aggregated per kernel (.md + the raw .csv).
Runs where ncu is installed (the build container); needs no GPU."""
import csv
import io
import json
import os
import re
import subprocess
import sys

METRICS = [
    ("time_us", "gpu__time_duration.sum"),
    ("dram_read_MB", "dram__bytes_read.sum"),
    ("dram_write_MB", "dram__bytes_write.sum"),
    ("dram_pct_of_peak", "FBSP.TriageCompute.dram__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("warp_inst", "smsp__inst_executed.sum"),
    ("issue_active_pct", "smsp__issue_active.avg.pct_of_peak_sustained_active"),
    ("alu_pct", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active"),
    ("fma_pct", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active"),
    ("fp64_pct", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active"),
    ("lsu_pct", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active"),
    ("xu_pct", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active"),
    ("warps_active_pct", "sm__warps_active.avg.pct_of_peak_sustained_active"),
    ("regs", "launch__registers_per_thread"),
    ("grid", "launch__grid_size"),
    ("smem_bank_conflicts", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"),
    ("stall_long_scoreboard", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio"),
    ("stall_short_scoreboard", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio"),
    ("stall_mio_throttle", "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio"),
    ("stall_barrier", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio"),
    ("stall_math_pipe", "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio"),
]

FRIENDLY = [
    (r"scan_kernel<1, \(int\)-1, 0>", "K1 moments `scan_kernel<MOM>` (anv_moments)"),
    (r"scan_kernel<0, (\(int\))?0, 0>", "K2 histogram `scan_kernel<HIST private>` (anv_hist)"),
    (r"scan_kernel<1, (\(int\))?0, 0>", "K1+K2 fused `scan_kernel<MOM,HIST>` (anv_moments_hist)"),
    (r"scan_kernel<0, (\(int\))?\d, 1>", "bin assign `scan_kernel<ASSIGN>` (anv_bin_assign)"),
    (r"hll_kernel", "K6 HLL++ registers `hll_kernel`"),
    (r"select_pass_kernel<1>", "K4 select pass 0 `select_pass_kernel<FIRST>`"),
    (r"select_pass_kernel<0>", "K4 select refinement pass `select_pass_kernel`"),
    (r"select_scan_kernel", "K4 `select_scan_kernel`"),
    (r"pack_kernel", "sort: pack keys `sort_pack_kernel`"),
    (r"sort_hist", "sort: tile digit histogram `sort_hist_kernel`"),
    (r"sort_totals", "sort: digit totals `sort_totals_kernel`"),
    (r"sort_scan", "sort: digit/tile scan `sort_scan_kernel`"),
    (r"pc_", "partition path: small kernels (opt-in)"),
    (r"spark_sample", "Spark Bernoulli sampler `spark_sample_kernel`"),
    (r"sort_scatter", "sort: stable scatter `sort_scatter_kernel`"),
    (r"run_tile", "sort: run summaries `run_tile_kernel`"),
    (r"run_merge", "sort: run merge `run_merge_kernel`"),
    (r"finalize", "moments finalize (Pebay merge of tile partials)"),
]
TRAFFIC_KEYS = {"K1 moments": "anv_moments", "K2 histogram": "anv_hist", "K1+K2 fused": "anv_moments_hist"}


def friendly(name):
    for pat, nice in FRIENDLY:
        if re.search(pat, name):
            return nice
    return name[:70]


def to_float(cell):
    try:
        return float(cell.replace(",", ""))
    except ValueError:
        return None


def full(rep, out, rows=None, cols=None):
    if rep.endswith(".csv"):     # `ncu -i <rep> --page raw --csv` already run on the GPU box (a full report can exceed the 64 MiB pull limit)
        raw = open(rep).read()
    else:
        raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows_csv = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows_csv[0], rows_csv[1]
    idx = {m: hdr.index(m) for _, m in METRICS if m in hdr}
    kname = hdr.index("Kernel Name")
    recs = []
    for r in rows_csv[2:]:
        rec = {"kernel": friendly(r[kname]), "raw_name": r[kname]}
        for key, m in METRICS:
            if m not in idx:
                continue
            v, u = to_float(r[idx[m]]), units[idx[m]]
            if v is None:
                continue
            if key == "time_us":
                v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(u, 1.0)
            if key.endswith("_MB"):
                v *= {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}.get(u, 1.0)
            rec[key] = v
        if rec.get("time_us"):
            rec["dram_GBps"] = (rec.get("dram_read_MB", 0.0) + rec.get("dram_write_MB", 0.0)) / rec["time_us"] * 1e3
        recs.append(rec)
    json.dump(recs, open(out + ".json", "w"), indent=1)
    cols_md = ["time_us", "dram_read_MB", "dram_write_MB", "dram_GBps", "issue_active_pct", "fp64_pct", "alu_pct", "fma_pct",
               "lsu_pct", "xu_pct", "regs", "warps_active_pct", "warp_inst", "stall_long_scoreboard", "stall_mio_throttle",
               "stall_math_pipe"]
    with open(out + ".md", "w") as fh:
        fh.write("# ncu --set full: per-kernel summary\n\n")
        fh.write("Source report: `%s` (`ncu --set full --clock-control none --import-source on --profile-from-start off "
                 "python scripts/prof_kernels.py`%s). Times under ncu are cold-cache and serialised; the bench numbers "
                 "come from CUDA events. DRAM bytes are `dram__bytes_read.sum` / `dram__bytes_write.sum` per launch.\n\n"
                 % (os.path.basename(rep), " on %s rows x %s float32 columns" % (rows, cols) if rows else ""))
        fh.write("| kernel | " + " | ".join(cols_md) + " |\n|---|" + "---|" * len(cols_md) + "\n")
        for r in recs:
            fh.write("| %s | " % r["kernel"] + " | ".join(
                ("%.4g" % r[c]) if isinstance(r.get(c), float) else str(r.get(c, "")) for c in cols_md) + " |\n")
    print("wrote", out + ".md", len(recs), "kernels")


def launch(csv_path, out):
    lines = [ln for ln in open(csv_path) if ln.startswith('"')]
    rd = list(csv.reader(io.StringIO("".join(lines))))
    hdr = rd[0]
    kn, mv, mu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg = {}
    for r in rd[1:]:
        v = to_float(r[mv])
        if v is None:
            continue
        v *= {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(r[mu], 1e-6)
        a = agg.setdefault(friendly(r[kn]), [0, 0.0])
        a[0] += 1
        a[1] += v
    tot = sum(a[1] for a in agg.values())
    with open(out + ".md", "w") as fh:
        fh.write("# ncu launch list, round 1: `python bench.py --steps 2 --warmup 1 --no-extras` (c2: 10M x 50 f32, full stats_generator)\n\n")
        fh.write("Command: `ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/launches.csv "
                 "python bench.py --steps 2 --warmup 1 --no-extras` (warm-up + timed steps + frame generation captured). "
                 "Per-launch times are cold-cache and serialised: compare SHARES with bench.py's `kernels` object.\n\n")
        fh.write("| kernel | launches | total ms | ms / launch | share |\n|---|---|---|---|---|\n")
        for k, (n, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            fh.write("| %s | %d | %.3f | %.4f | %.1f%% |\n" % (k, n, ms, ms / n, 100 * ms / tot))
    if os.path.abspath(csv_path) != os.path.abspath(out + ".csv"):
        open(out + ".csv", "w").write("".join(lines))
    print("wrote", out + ".md", len(agg), "kernels, total %.1f ms" % tot)


CALL_OF = [(r"scan_kernel<1, \(int\)-1, 0>|finalize", "anv_moments"), (r"hll_kernel", "anv_hll_registers"),
           (r"pack_kernel|sort_hist|sort_scan|sort_scatter|run_tile|run_merge", "anv_mode_distinct"),
           (r"scan_kernel<0, (\(int\))?0, 0>", "anv_hist"), (r"scan_kernel<1, (\(int\))?0, 0>", "anv_moments_hist"),
           (r"select_pass|select_scan", "anv_select_ranks")]
CALL_MARK = {"anv_moments": r"finalize", "anv_hll_registers": r"hll_kernel", "anv_mode_distinct": r"run_merge",
             "anv_hist": r"scan_kernel<0", "anv_moments_hist": r"finalize", "anv_select_ranks": None}


def traffic(csv_path, out_json, rows, cols):
    """`ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum --csv` launch list of a bench run -> DRAM bytes per
    C call (all kernels the call launches), written to profiles/r1_traffic.json for bench.py's roofline.traffic."""
    lines = [ln for ln in open(csv_path) if ln.startswith('"')]
    rd = list(csv.reader(io.StringIO("".join(lines))))
    hdr = rd[0]
    kn, mn, mv, mu = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    iid = hdr.index("ID")
    bytes_of, marks, seen = {}, {}, set()
    for r in rd[1:]:
        if not r[mn].startswith("dram__bytes"):
            continue
        v = to_float(r[mv])
        if v is None:
            continue
        v *= {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(r[mu], 1.0)
        for pat, call in CALL_OF:
            if re.search(pat, r[kn]):
                bytes_of[call] = bytes_of.get(call, 0.0) + v
                mk = CALL_MARK.get(call)
                if mk and re.search(mk, r[kn]) and (call, r[iid]) not in seen:
                    seen.add((call, r[iid]))
                    marks[call] = marks.get(call, 0) + 1
                break
    per_call = {c: b / max(marks.get(c, 1), 1) for c, b in bytes_of.items()}
    json.dump({"workload": "c2", "rows": int(rows), "cols": int(cols), "source": os.path.basename(csv_path) +
               " (ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum on `bench.py --steps 1 --warmup 1 --no-extras`; "
               "bytes of every kernel a C call launches, per call)", "calls_captured": marks,
               "dram_bytes_per_launch": per_call}, open(out_json, "w"), indent=1)
    print("wrote", out_json, per_call, marks)


if __name__ == "__main__":
    if sys.argv[1] == "traffic":
        traffic(sys.argv[2], sys.argv[3], sys.argv[4], sys.argv[5])
    elif sys.argv[1] == "full":
        full(sys.argv[2], sys.argv[3], *(sys.argv[4:6]))
    else:
        launch(sys.argv[2], sys.argv[3])
