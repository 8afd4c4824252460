"""Per-kernel limiter table from an `ncu --set full` report: duration, registers, achieved warps, issue-active, pipe utilisation, the
five largest warp-stall reasons, cache hit rates and DRAM bytes.

    python tools/ncu_stalls.py out/prof.ncu-rep [out.md]
"""
import csv
import io
import re
import subprocess
import sys


def main():
    rep = sys.argv[1]
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}

    def get(r, name, default=""):
        i = col.get(name)
        return r[i] if i is not None and i < len(r) else default

    def num(r, name):
        try:
            return float(get(r, name, "nan").replace(",", ""))
        except ValueError:
            return float("nan")

    stall_cols = [h for h in hdr if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
    if not stall_cols:
        stall_cols = [h for h in hdr if h.startswith("smsp__average_warp_latency_issue_stalled_") or (h.startswith("smsp__average_warps_issue_stalled") and "ratio" in h)]
    lines = ["| kernel | grid x block | us | regs | warps active % | issue active % | fma % | alu % | lsu % | tensor % | L1 hit % | L2 hit % | dram rd+wr MB | top stalls (warps per issue) |",
             "|---|---|---|---|---|---|---|---|---|---|---|---|---|---|"]
    seen = {}
    for r in data:
        name = get(r, "Kernel Name")
        m = re.search(r"(k_[a-z0-9_]+)", name)
        k = m.group(1) if m else name
        key = (k, get(r, "Grid Size"), get(r, "Block Size"))
        if key in seen:
            continue
        seen[key] = 1
        stalls = sorted(((num(r, c), c) for c in stall_cols), reverse=True)
        top = ", ".join("%s %.2f" % (c.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", ""), v) for v, c in stalls[:5] if v == v)
        dur = num(r, "gpu__time_duration.sum")
        unit = units[col["gpu__time_duration.sum"]] if "gpu__time_duration.sum" in col else ""
        us = dur / 1e3 if unit.startswith("ns") else (dur if unit.startswith("us") else dur * 1e3 if unit.startswith("ms") else dur)

        def mb(name):
            v = num(r, name)
            u = units[col[name]] if name in col else ""
            scale = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}.get(u, 1e-6)
            return v * scale

        lines.append("| %s | %s x %s | %.1f | %s | %.1f | %.1f | %.1f | %.1f | %.1f | %.1f | %.1f | %.1f | %.1f | %s |" % (
            k, get(r, "Grid Size"), get(r, "Block Size"), us, get(r, "launch__registers_per_thread"),
            num(r, "sm__warps_active.avg.pct_of_peak_sustained_active"), num(r, "sm__inst_issued.avg.pct_of_peak_sustained_active") if "sm__inst_issued.avg.pct_of_peak_sustained_active" in col else num(r, "smsp__issue_active.avg.pct_of_peak_sustained_active"),
            num(r, "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active"), num(r, "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active"),
            num(r, "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active"), num(r, "TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed"),
            num(r, "l1tex__t_sector_hit_rate.pct"), num(r, "lts__t_sector_hit_rate.pct"), mb("dram__bytes_read.sum") + mb("dram__bytes_write.sum"), top))
    text = "\n".join(lines)
    print(text)
    if len(sys.argv) > 2:
        open(sys.argv[2], "w").write(text + "\n")


if __name__ == "__main__":
    main()
