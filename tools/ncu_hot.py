"""Hot SASS instructions + stall-reason totals of one kernel from an ncu report (source page).
    python tools/ncu_hot.py out/prof.ncu-rep k_gru_fwd [top_n]"""
import csv, io, subprocess, sys
rep, kern = sys.argv[1], sys.argv[2]
top = int(sys.argv[3]) if len(sys.argv) > 3 else 25
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--kernel-name", "regex:" + kern, "--launch-count", "1"],
                     capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(out)))
hdr = rows[1]
data = []
for r in rows[2:]:
    if r and r[0] == "Kernel Name":
        break                     # only the first captured launch of the kernel
    if len(r) == len(hdr) and r[hdr.index("# Samples")].isdigit():
        data.append(r)
i_src, i_smp, i_exec = hdr.index("Source"), hdr.index("# Samples"), hdr.index("Instructions Executed")
stalls = [(i, h) for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h]
tot = sum(int(r[i_smp] or 0) for r in data)
print("kernel %s: %d SASS instructions, %d samples" % (rows[0][1], len(data), tot))
agg = sorted(((sum(int(r[i] or 0) for r in data), h) for i, h in stalls), reverse=True)
print("stall totals:", ", ".join("%s %.1f%%" % (h[6:], 100.0 * v / max(tot, 1)) for v, h in agg[:8]))
print("top instructions by samples:")
for n, r in sorted(enumerate(data), key=lambda nr: -int(nr[1][i_smp] or 0))[:top]:
    st = sorted(((int(r[i] or 0), h[6:]) for i, h in stalls), reverse=True)[:2]
    print("%5d %5.1f%% exec=%-7s %-60s %s" % (n, 100.0 * int(r[i_smp] or 0) / max(tot, 1), r[i_exec], r[i_src].strip()[:60], st))
