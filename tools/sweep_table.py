"""Tabulate the `bench.py --quick` lines of an option sweep (one log file per sweep): one row per
(workload, options), steps/s and the ratio to the same workload's run without options (or with every option at 0).

    python tools/sweep_table.py out/sweep_*.log
"""
import glob
import json
import sys


def main(paths):
    rows = []
    for pat in paths:
        for p in sorted(glob.glob(pat)):
            for ln in open(p):
                ln = ln.strip()
                if not ln.startswith("{"):
                    continue
                try:
                    d = json.loads(ln)
                except ValueError:
                    continue
                if d.get("quick"):
                    rows.append((p, d["workload"], tuple(d.get("opts") or ()), float(d["value"]), float(d["ms_per_step"]), d.get("kernels_per_step")))
    base = {}
    for p, w, opts, v, ms, k in rows:
        if all(o.endswith("=0") for o in opts):
            base.setdefault((p, w), v)
    print("%-22s %-52s %12s %10s %8s %6s" % ("workload", "options", "steps/s", "us/step", "vs base", "kern"))
    for p, w, opts, v, ms, k in rows:
        b = base.get((p, w))
        print("%-22s %-52s %12.1f %10.1f %8s %6s" % (w, " ".join(opts) or "-", v, ms * 1e3, ("%.3f" % (v / b)) if b else "", k if k is not None else ""))


if __name__ == "__main__":
    main(sys.argv[1:] or ["out/sweep_*.log"])
