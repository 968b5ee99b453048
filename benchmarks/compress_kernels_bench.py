#!/usr/bin/env python
"""Device time of the fused GPU compressor phases on ONE GPU (no peers: the push is a no-op).

For a 100 MB fp32 gradient it prints the producer (momentum + error feedback + compress), the push
and the consumer (decompress + "server" stage + output) times separately, next to the HBM bytes
each phase has to move, i.e. how far the passes are from the copy roofline in MEASURED_PEAKS.json.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


class _Ctx:
    def __init__(self, vc, r):
        self.cu, self.device, self.world, self.rank = vc.cu, vc.device, vc.world, r
        self.view, self.arena, self.data_bytes = vc.views[r], vc.arenas[r], vc.data_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=100)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops.compress import GpuCompressor

    n = args.mb * 1000 * 1000 // 4
    vc = VirtualCluster(1, "cuda:0", 64 << 20)
    g = torch.randn(n, device="cuda")
    out = torch.empty_like(g)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream()
    cases = [
        ("onebit+scaling+ef", dict(compressor_type="onebit", compressor_onebit_scaling="true", ef_type="vanilla")),
        ("onebit+scaling+ef+nesterov", dict(compressor_type="onebit", compressor_onebit_scaling="true",
                                            ef_type="vanilla", momentum_type="nesterov", momentum_mu="0.9")),
        ("topk1%+ef", dict(compressor_type="topk", compressor_k=0.01, ef_type="vanilla")),
        ("randomk1%+ef", dict(compressor_type="randomk", compressor_k=0.01, ef_type="vanilla", seed=7)),
        ("dithering4", dict(compressor_type="dithering", compressor_k=4, seed=7)),
    ]
    rows = []
    for name, kw in cases:
        comp = GpuCompressor(_Ctx(vc, 0), kw, n, torch.float32)
        tot = None
        for it in range(args.iters + 2):
            flush.fill_(it & 1)                       # evict the 50 MB L2 between iterations
            phases = comp.phases(g, out, True, s.cuda_stream)
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(len(phases) + 1)]
            evs[0].record()
            for i, ph in enumerate(phases):
                ph()
                evs[i + 1].record()
            torch.cuda.synchronize()
            ms = [evs[i].elapsed_time(evs[i + 1]) for i in range(len(phases))]
            if it >= 2:
                tot = ms if tot is None else [a + b for a, b in zip(tot, ms)]
        ms = [t / args.iters for t in tot]
        rows.append({"case": name, "producer_ms": ms[0], "push_ms": ms[1], "consumer_ms": ms[2], "total_ms": sum(ms),
                     "finite": bool(torch.isfinite(out).all().item())})
        print("%-28s producer %.3f  push %.3f  consumer %.3f  total %.3f ms" % (name, ms[0], ms[1], ms[2], sum(ms)),
              flush=True)
        del comp
    if args.out:
        json.dump({"gradient_bytes": n * 4, "rows": rows}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
