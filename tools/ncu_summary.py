#!/usr/bin/env python
"""Summarise one kernel of an ncu report (.ncu-rep) into key = value text.
    python tools/ncu_summary.py x.ncu-rep "header comment lines..." > x.txt
Also prints a one-line JSON with DRAM traffic for bench.py's roofline.traffic (--json out.json)."""
import csv, io, json, subprocess, sys

KEEP = ["dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "gpu__time_duration.sum",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "launch__block_size", "launch__grid_size", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "sm__inst_issued.avg.per_cycle_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__average_warp_latency_per_inst_issued.ratio",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "sm__cycles_active.avg", "smsp__cycles_active.avg"]


def main():
    rep = sys.argv[1]
    comments = [a for a in sys.argv[2:] if not a.startswith("--json")]
    jout = None
    if "--json" in sys.argv:
        jout = sys.argv[sys.argv.index("--json") + 1]
        comments = [c for c in comments if c != jout]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, vals = rows[0], rows[1], rows[2]
    get = lambda k: next(((vals[i], units[i]) for i, h in enumerate(hdr) if h == k), (None, None))
    out = [f"# {c}" for c in comments]
    out.append(f"Kernel Name [] = {get('Kernel Name')[0]}")
    for k in KEEP:
        v, u = get(k)
        if v is not None:
            out.append(f"{k} [{u}] = {v}")
    for i, h in enumerate(hdr):
        if "issue_stalled" in h and h.endswith("per_issue_active.ratio"):
            out.append(f"{h} [{units[i]}] = {vals[i]}")
    print("\n".join(out))
    if jout:
        scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "Tbyte": 1e12}
        rd, ru = get("dram__bytes_read.sum"); wr, wu = get("dram__bytes_write.sum"); dur, du = get("gpu__time_duration.sum")
        dms = float(dur) * {"ms": 1.0, "us": 1e-3, "s": 1e3, "ns": 1e-6}[du]
        json.dump({"kernel": get("Kernel Name")[0], "jobs": int(float(get("launch__grid_size")[0])), "dram_bytes_read": float(rd) * scale[ru], "dram_bytes_write": float(wr) * scale[wu],
                   "duration_ms": dms, "source": jout.replace(".json", ".txt")}, open(jout, "w"), indent=1)


if __name__ == "__main__":
    main()
