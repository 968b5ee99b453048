#!/usr/bin/env python
"""Static resource table of every kernel in the built CUDA module (registers, stack, static shared memory,
local memory), from `cuobjdump --dump-resource-usage`.  Runs without a GPU.

    python benchmarks/resource_usage.py > profiles/resource_usage.md
"""
import glob
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    so = glob.glob(os.path.join(ROOT, "byteps_b200", "_cuda*.so"))
    if not so:
        sys.exit("build the CUDA module first (python __graft_entry__.py)")
    txt = subprocess.run(["cuobjdump", "--dump-resource-usage", so[0]], capture_output=True, text=True).stdout
    rows, cur = [], None
    for line in txt.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", line)
        if m and cur:
            rows.append((cur,) + tuple(int(x) for x in m.groups()))
            cur = None
    names = subprocess.run(["c++filt"] + [r[0] for r in rows], capture_output=True, text=True).stdout.splitlines()
    table = {}
    for (f, reg, stack, sh, loc), n in zip(rows, names):
        n = re.sub(r"bps::\(anonymous namespace\)::", "", n)
        n = re.sub(r"^void ", "", n)
        base = re.sub(r"<.*", "", re.sub(r"\(.*", "", n))
        tmpl = re.search(r"<(.*)>", re.sub(r"\(.*", "", n))
        t = table.setdefault(base, {"n": 0, "reg": [], "stack": 0, "shared": 0, "local": 0, "variants": []})
        t["n"] += 1
        t["reg"].append(reg)
        t["stack"] = max(t["stack"], stack)
        t["shared"] = max(t["shared"], sh)
        t["local"] = max(t["local"], loc)
        if tmpl:
            t["variants"].append((tmpl.group(1).replace("bps::", ""), reg))
    print("# Static resource usage of the sm_90a kernels\n")
    print("`python benchmarks/resource_usage.py` (cuobjdump --dump-resource-usage on the in-tree `_cuda` module; no GPU "
          "needed).  %d kernel instantiations of %d kernels.  `stack`/`local` > 0 would mean spills or dynamically "
          "indexed arrays in a hot loop; the 16 B (32 B) stack of the cross-rank kernels is the argument block of the barrier "
          "watchdog's `printf` (cold path).\n" % (len(rows), len(table)))
    print("| kernel | instantiations | registers (min-max) | max stack B | static smem B | local B |")
    print("|---|---|---|---|---|---|")
    for k in sorted(table):
        t = table[k]
        print("| `%s` | %d | %d-%d | %d | %d | %d |" % (k, t["n"], min(t["reg"]), max(t["reg"]), t["stack"], t["shared"],
                                                       t["local"]))
    print("\nDynamic shared memory (not in the table): TMA push-pull ring `stages x (world+1) x 4 KiB`, fused-optimizer "
          "ring `stages x streams x 256 x 16|32 B` (<= 96 KiB so that two CTAs share an SM), wgmma variant "
          "`6 x 16 KiB peer tiles + a 16 KiB output tile`.")


if __name__ == "__main__":
    main()
