#!/usr/bin/env python
"""Summarise an .ncu-rep (read on the CPU box with `ncu -i`) into profiles/<name>.md.

    python benchmarks/ncu_summary.py <report>.ncu-rep <summary>.md
"""
import csv
import io
import subprocess
import sys

KEEP = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
    "launch__block_size", "launch__occupancy_limit_registers", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct",
    "smsp__cycles_active.avg", "dram__cycles_active.avg.pct_of_peak_sustained_elapsed",
]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    with open(out, "w") as f:
        f.write("# ncu summary of %s\n\n`ncu --set full --clock-control none --import-source on` on one H100; "
                "read here with `ncu -i ... --page raw --csv`.\n\n" % rep)
        for r in data:
            d = dict(zip(hdr, r))
            f.write("## %s  (grid %s, block %s)\n\n| metric | value | unit |\n|---|---|---|\n" % (
                d.get("Kernel Name", "?")[:120], d.get("launch__grid_size", "?"), d.get("launch__block_size", "?")))
            for k in KEEP:
                if k in d:
                    f.write("| %s | %s | %s |\n" % (k, d[k], units[hdr.index(k)]))
            try:
                rd, wr = float(d["dram__bytes_read.sum"].replace(",", "")), float(d["dram__bytes_write.sum"].replace(",", ""))
                t = float(d["gpu__time_duration.sum"].replace(",", ""))
                scale = {"byte": 1e-9, "Kbyte": 1e-6, "Mbyte": 1e-3, "Gbyte": 1.0}
                ru, wu = units[hdr.index("dram__bytes_read.sum")], units[hdr.index("dram__bytes_write.sum")]
                f.write("\nDRAM traffic %.2f GB read + %.2f GB write in %s %s.\n\n" % (
                    rd * scale.get(ru, 1.0), wr * scale.get(wu, 1.0), t, units[hdr.index("gpu__time_duration.sum")]))
            except Exception:  # noqa: BLE001
                f.write("\n")
    # ---- stall hot spots per distinct kernel (source page; needs `--import-source on` / -lineinfo)
    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    secs, cur = [], None
    for r in csv.reader(src.splitlines()):
        if r and r[0] == "Kernel Name":
            cur = {"name": r[1], "hdr": None, "rows": []}
            secs.append(cur)
        elif cur is not None and cur["hdr"] is None:
            cur["hdr"] = r
        elif cur is not None:
            cur["rows"].append(r)
    seen = set()
    with open(out, "a") as f:
        for sec in secs:
            if sec["name"] in seen or not sec["hdr"] or "Source" not in sec["hdr"]:
                continue
            seen.add(sec["name"])
            h = sec["hdr"]
            i_src, i_s = h.index("Source"), h.index("Warp Stall Sampling (All Samples)")
            tot = sum(int(r[i_s] or 0) for r in sec["rows"])
            f.write("\n## stall hot spots: %s\n\n%d samples over %d SASS instructions\n\n| SASS | samples | share | "
                    "dominant stall |\n|---|---|---|---|\n" % (sec["name"][:100], tot, len(sec["rows"])))
            for r in sorted(sec["rows"], key=lambda q: -int(q[i_s] or 0))[:8]:
                stalls = [(h[j], int(r[j] or 0)) for j in range(min(len(h), len(r))) if h[j].startswith("stall_")]
                dom = max(stalls, key=lambda t: t[1])[0].replace("stall_", "") if stalls else "?"
                f.write("| `%s` | %d | %.1f %% | %s |\n" % (r[i_src].strip()[:70], int(r[i_s] or 0),
                                                          100.0 * int(r[i_s] or 0) / max(tot, 1), dom))
    print(open(out).read()[:2500])


if __name__ == "__main__":
    main()
