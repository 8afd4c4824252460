"""Summarise one ncu capture into profiles/<tag>_ncu_summary.md (+ <tag>_ncu_launches.csv, ncu_traffic.json).

    python tools/ncu_summary.py r01k out/launches.csv out/prof_r01k.ncu-rep

launches.csv : `ncu --metrics gpu__time_duration.sum --clock-control none --csv` launch list of `bench.py`
*.ncu-rep    : `ncu --set full --clock-control none --import-source on` capture of the step's kernels
"""
import csv
import io
import json
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEP = ["k_draw", "k_gather", "k_gather_tma", "k_tc_prep_weights", "k_front_fwd_tc", "k_front_fwd_tc2", "k_front_fwd", "k_gru_fwd", "k_gru_fwd2", "k_qhead", "k_mixer",
        "k_mix_hyper_fwd", "k_mix_core", "k_mix_hyper_bwd", "k_mid", "k_qhead_bwd", "k_gru_bwd", "k_gru_bwd2", "k_gru_wgrad", "k_front_bwd", "k_grad_reduce", "k_adam", "k_optim_fused", "k_polyak"]


def short(name):
    m = re.search(r"(k_[a-z0-9_]+)", name)
    return m.group(1) if m else name


def launch_table(path):
    rows = [r for r in csv.reader(l for l in open(path) if l.startswith('"'))]
    hdr = rows[0]
    ik, iv, ig, ib = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Grid Size"), hdr.index("Block Size")
    agg = {}
    for r in rows[1:]:
        k = (short(r[ik]), r[ig], r[ib])
        agg.setdefault(k, []).append(float(r[iv].replace(",", "")) / 1e3)     # ns -> us
    return agg


def full_table(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    return hdr, units, data


def main():
    tag, lpath, rep = sys.argv[1], sys.argv[2], sys.argv[3]
    prof = os.path.join(ROOT, "profiles")
    shutil.copy(lpath, os.path.join(prof, "%s_ncu_launches.csv" % tag))
    agg = launch_table(lpath)
    per_kernel = {}
    for (k, g, b), v in agg.items():
        per_kernel.setdefault(k, []).extend(v)
    step_total = sum(sum(v) / len(v) * (2 if k == "k_tc_prep_weights" and False else 1) for k, v in per_kernel.items() if k in STEP)
    md = ["# %s -- ncu evidence (qmix_3m: B=32, T=60, N=3)" % tag, "",
          "Commands (1 GPU): `ncu --metrics gpu__time_duration.sum --clock-control none -c 500 --csv python bench.py --steps 3 --warmup 3 --buffer 512`",
          "(launch list, copied to `%s_ncu_launches.csv`) and `ncu --set full --clock-control none --import-source on -k regex:... -s 36 -c 20` (report not committed: 32 MB)." % tag, "",
          "## Launch list (cold-cache, serialised: compare SHARES with bench.py's live per-kernel timing, not absolutes)", "",
          "| kernel | grid | block | launches | avg us | share of the step's kernels |", "|---|---|---|---|---|---|"]
    for (k, g, b), v in sorted(agg.items(), key=lambda kv: -sum(kv[1]) / len(kv[1])):
        if not k.startswith("k_"):
            continue            # torch fill kernels of the set-up phase
        avg = sum(v) / len(v)
        share = "%.1f%%" % (100 * avg / step_total) if k in STEP else "-"
        md.append("| %s | %s | %s | %d | %.2f | %s |" % (k, g, b, len(v), avg, share))
    hdr, units, data = full_table(rep)
    cols = [("gpu__time_duration.sum", "time us"), ("launch__grid_size", "grid"), ("launch__registers_per_thread", "regs"),
            ("launch__shared_mem_per_block_dynamic", "dyn smem KB"), ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
            ("sm__inst_issued.avg.pct_of_peak_sustained_active", "issue active %"), ("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "fma pipe %"),
            ("TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed", "tensor pipe % (cycles active)"),
            ("sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active", "hmma subpipe inst %"),
            ("sm__inst_executed_pipe_tmem.avg.pct_of_peak_sustained_active", "tmem inst %"),
            ("sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "tensor-memory (TMA) cycles %"),
            ("dram__bytes_read.sum", "dram rd"), ("dram__bytes_write.sum", "dram wr"),
            ("lts__t_sectors_op_read.sum", "L2 rd sectors"), ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smem bank conflicts"),
            ("sm__cycles_elapsed.max", "cycles")]
    cols = [(c, n) for c, n in cols if c in hdr]
    md += ["", "## `--set full` key metrics (first captured launch of each kernel)", "", "| kernel | " + " | ".join(n for _, n in cols) + " |",
           "|---|" + "---|" * len(cols)]
    ik = hdr.index("Kernel Name")
    seen, traffic = set(), {}
    for r in data:
        k = short(r[ik])
        if k in seen:
            continue
        seen.add(k)
        cells = []
        for c, n in cols:
            i = hdr.index(c)
            cells.append("%s %s" % (r[i], units[i]) if units[i] and n in ("dram rd", "dram wr") else r[i])
        md.append("| %s | " % k + " | ".join(cells) + " |")

        def to_bytes(c):
            i = hdr.index(c)
            u = units[i].lower()
            mul = 1e9 if u.startswith("g") else 1e6 if u.startswith("m") else 1e3 if u.startswith("k") else 1.0
            return float(r[i].replace(",", "")) * mul
        traffic[k] = dict(dram_bytes=to_bytes("dram__bytes_read.sum") + to_bytes("dram__bytes_write.sum"),
                          time_us=float(r[hdr.index("gpu__time_duration.sum")].replace(",", "")), source="%s --set full capture" % tag)
    notes = os.path.join(prof, "%s_ncu_reading.md" % tag)
    if os.path.exists(notes):
        md += ["", open(notes).read().rstrip()]
    open(os.path.join(prof, "%s_ncu_summary.md" % tag), "w").write("\n".join(md) + "\n")
    json.dump(traffic, open(os.path.join(prof, "ncu_traffic.json"), "w"), indent=1, sort_keys=True)
    print("\n".join(md))


if __name__ == "__main__":
    main()
