"""ncu `--page raw --csv` export -> profiles/<tag>_ncu.json (per kernel: time, DRAM bytes, issue utilisation, stalls, ...)
and profiles/traffic.json (DRAM bytes per launch of the composite stages, read by bench.py for roofline.traffic).
usage: python tools/ncu_to_profiles.py prof_raw.csv r02_c3"""
import csv
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
rows = list(csv.reader(open(sys.argv[1])))
tag = sys.argv[2]
hdr, units, data = rows[0], rows[1], rows[2:]
ix = {h: i for i, h in enumerate(hdr)}
KEEP = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio"]


def num(s):
    try:
        return float(s.replace(",", ""))
    except Exception:
        return s


def to_bytes(v, unit):
    return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}.get(unit, 1)


out, traffic = [], {}
for r in data:
    name = r[ix["Kernel Name"]]
    rec = {"kernel": name}
    for k in KEEP:
        if k in ix:
            rec[k] = num(r[ix[k]])
            rec[k + " [unit]"] = units[ix[k]]
    rd = to_bytes(num(r[ix["dram__bytes_read.sum"]]), units[ix["dram__bytes_read.sum"]])
    wr = to_bytes(num(r[ix["dram__bytes_write.sum"]]), units[ix["dram__bytes_write.sum"]])
    rec["dram_bytes_total"] = rd + wr
    out.append(rec)
    stage = ("composite_fwd" if "composite_fwd" in name else
             "composite_bwd" if ("composite_bwd" in name or "feature_bwd" in name) else None)
    if stage:
        traffic.setdefault(stage, {}).setdefault(name.split("(")[0], []).append(rd + wr)
json.dump(out, open(os.path.join(ROOT, "profiles", f"{tag}_ncu.json"), "w"), indent=1)
summary = {"source": f"profiles/{tag}_ncu.json (ncu --set full --clock-control none, per launch; dram__bytes_read + dram__bytes_write)"}
for stage, ks in traffic.items():
    summary[stage] = int(sum(sum(v) / len(v) for v in ks.values()))  # kernels of one stage add up (two-kernel backward)
    summary[stage + "_kernels"] = {k: int(sum(v) / len(v)) for k, v in ks.items()}
json.dump(summary, open(os.path.join(ROOT, "profiles", "traffic.json"), "w"), indent=1)
print(json.dumps(summary, indent=1))
