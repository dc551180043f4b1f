#!/usr/bin/env python
"""Print the key raw-page metrics of every kernel launch in an .ncu-rep as a markdown table row set.

    summarize_ncu.py rep.ncu-rep [...]                       markdown on stdout
    summarize_ncu.py --traffic-json OUT SAMPLES rep.ncu-rep  also write {kernel: dram bytes per input sample} (first
                                                             launch of each kernel; SAMPLES = input samples per launch)"""
import csv
import subprocess
import sys

WANT = [
    ("gpu__time_duration.sum", "time"),
    ("dram__bytes_read.sum", "dram read"),
    ("dram__bytes_write.sum", "dram write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram %peak"),
    ("smsp__inst_executed.sum", "warp insts"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue active %"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
    ("launch__registers_per_thread", "regs"),
    ("launch__grid_size", "grid"),
    ("smsp__thread_inst_executed_per_inst_executed.ratio", "threads/inst"),
    ("sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active", "fp64 pipe %"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "alu pipe %"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "lsu pipe %"),
]
args = sys.argv[1:]
traffic_out, samples = None, None
if args and args[0] == "--traffic-json":
    traffic_out, samples, args = args[1], float(args[2]), args[3:]
traffic = {}
for rep in args:
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    print(f"\n### {rep}")
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")][:70]
        cells = []
        for key, label in WANT:
            if key in hdr:
                i = hdr.index(key)
                v = r[i]
                try:
                    v = f"{float(v):.4g}"
                except ValueError:
                    pass
                cells.append(f"{label} {v} {units[i]}")
        print(f"- `{name}`: " + "; ".join(cells))
        if traffic_out and "dram__bytes_read.sum" in hdr:
            def gb(key):
                i = hdr.index(key)
                v, u = float(r[i]), units[i]
                return v * {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "Tbyte": 1e12}.get(u, 1.0)
            full = r[hdr.index("Kernel Name")]
            plain = full.replace("(bool)", "").replace("(int)", "").replace("b2p::", "")
            key = plain.split("(")[0].split("<")[0].replace("void ", "").strip()
            if key == "range_lean_kernel":  # template <FN, FLAGS, GROUPED, UNI>
                targs = [x.strip() for x in plain.split("<", 1)[1].split(">")[0].split(",")]
                if len(targs) > 2 and targs[2] == "1":
                    key += "_grouped"
                if len(targs) > 3 and targs[3] == "1":
                    key += "_uniform"
            if key not in traffic:
                b = gb("dram__bytes_read.sum") + gb("dram__bytes_write.sum")
                traffic[key] = {"dram_bytes_per_launch": b, "dram_bytes_per_sample": b / samples,
                                "samples_per_launch": samples, "kernel": full, "source": rep}
if traffic_out:
    import json
    with open(traffic_out, "w") as f:
        json.dump(traffic, f, indent=1)
