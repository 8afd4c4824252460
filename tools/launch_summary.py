"""Per-kernel average duration from an `ncu --metrics gpu__time_duration.sum --csv` launch list (second half of the launches of each kernel).
    python tools/launch_summary.py out/launches.csv"""
import collections
import csv
import sys
for f in sys.argv[1:]:
    rows = list(csv.reader(l for l in open(f) if not l.startswith("==")))
    hdr = rows[0]
    ik, iv, iu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    d = collections.OrderedDict()
    for r in rows[1:]:
        if len(r) <= iv:
            continue
        k = r[ik].split("(")[0].replace("void ", "")
        v = float(r[iv].replace(",", ""))
        v = v / 1000 if r[iu] == "ns" else (v * 1000 if r[iu] == "ms" else v)
        d.setdefault(k, []).append(v)
    print(f)
    tot = 0.0
    for k, v in d.items():
        if not k.startswith("k_"):
            continue
        v2 = v[len(v) // 2:]
        print("  %-28s n=%3d  %6.1f us" % (k, len(v), sum(v2) / len(v2)))
