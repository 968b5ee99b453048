#!/usr/bin/env python
"""Synthetic all-gradients push-pull throughput (BASELINE.json metric, part 1).

Measures, on N GPUs of one box (launch with torchrun), device-timed with CUDA
events and max over ranks:

* our fused in-place kernel (P2P and, when available, NVLS) over a size sweep,
* the reference-style NCCL path (per-4MB ReduceScatter+AllGather, groups of 4, div_),
* a plain NCCL all_reduce for context,
* the three gradient sets BASELINE.json names: a 100 MB synthetic gradient,
  ResNet-50's 161 tensors (bf16) and BERT-large's tensors (bf16).

bus GB/s = 2*(N-1)/N * bytes / time, the NCCL-tests convention.  Roofline: the
P2P kernel moves 2*(N-1)/N*S bytes per GPU per direction -> bus GB/s is bounded
by the per-direction NVLink bandwidth (H100, NVLink 4: 450 GB/s nominal).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def timed(fn, iters, warm, device, flush=None):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize(device)
    dist.barrier()
    torch.cuda.synchronize(device)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    tot = 0.0
    for _ in range(iters):
        if flush is not None:
            flush()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize(device)
        tot += e0.elapsed_time(e1)
    ms = tot / iters
    t = torch.tensor([ms], device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--sizes", default="65536,1048576,4194304,16777216,104857600,536870912")
    ap.add_argument("--quick", action="store_true",
                    help="bf16 only, one grid per variant, no TMA/wgmma/reference-style sweeps (short GPU leases)")
    ap.add_argument("--skip-api", action="store_true", help="skip the per-tensor public-API gradient sets")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    import byteps_b200.torch as bps
    from byteps_b200 import _native
    from byteps_b200.comm.nccl_baseline import NcclReferencePath
    from byteps_b200.comm.symm import SymmContext, pick_blocks, wire_code
    from byteps_b200.common import engine

    bps.init()
    eng = engine()
    cu = _native.cuda()
    sizes = [int(s) for s in args.sizes.split(",")]
    arena_bytes = max(sizes) * 2 + (1 << 20)
    ctx = SymmContext(eng.group, device, arena_bytes, eng.cfg.symm_mode,
                      "try" if eng.cfg.use_nvls == "auto" else eng.cfg.use_nvls)   # measure NVLS at any world size
    stream = torch.cuda.current_stream(device)
    ref = NcclReferencePath()
    # L2 flush buffer (> the 50 MB L2)
    fl = torch.empty(256 << 20, dtype=torch.uint8, device=device)

    def flush():
        cu.l2_flush(fl.data_ptr(), fl.numel(), 1, stream.cuda_stream)

    rows = []
    factor = 2.0 * (world - 1) / world if world > 1 else 1.0
    for nbytes in sizes:
        for dt in ((torch.bfloat16,) if args.quick else (torch.bfloat16, torch.float32)):
            es = 2 if dt == torch.bfloat16 else 4
            n = nbytes // es // 8 * 8
            x = ctx.tensor(0, n, dt)
            x.fill_(1.0)
            shard = nbytes // world
            for mode in (["p2p"] + (["nvls"] if ctx.nvls else [])):
                best = None
                for cap in ((64,) if args.quick else (8, 16, 32, 64, 128)):
                    blocks = pick_blocks(shard, 512, 32, cap=cap)
                    if best is not None and blocks == best[1]:
                        continue
                    ms = timed(lambda: cu.pushpull_inplace(ctx.view, wire_code(dt), 0, n, 1.0 / world, blocks, 512, 0,
                                                           mode == "nvls", stream.cuda_stream),
                               args.iters, args.warmup, device, flush)
                    if best is None or ms < best[0]:
                        best = (ms, blocks)
                ms, blocks = best
                rows.append({"what": "ours_inplace_" + mode, "bytes": nbytes, "dtype": str(dt)[6:], "ms": ms,
                             "blocks": blocks, "alg_gbs": nbytes / ms / 1e6, "bus_gbs": factor * nbytes / ms / 1e6})
            best = None
            for cap in (() if args.quick else (16, 32, 64, 128)):
                blocks = pick_blocks(shard, 256, 16, cap=cap)
                if best is not None and blocks == best[1]:
                    continue
                ms = timed(lambda: cu.pushpull_inplace_tma(ctx.view, wire_code(dt), 0, n, 1.0 / world, blocks, 4, 0,
                                                           stream.cuda_stream), args.iters, args.warmup, device, flush)
                if best is None or ms < best[0]:
                    best = (ms, blocks)
            if best is not None:
                rows.append({"what": "ours_inplace_tma_p2p", "bytes": nbytes, "dtype": str(dt)[6:], "ms": best[0],
                             "blocks": best[1], "alg_gbs": nbytes / best[0] / 1e6,
                             "bus_gbs": factor * nbytes / best[0] / 1e6})
            if dt == torch.bfloat16 and world <= 8 and not args.quick:
                maps = cu.make_umma_maps(ctx.view, wire_code(dt), 0, n)
                best = None
                for cap in (8, 16, 32, 64, torch.cuda.get_device_properties(device).multi_processor_count):
                    blocks = max(1, min(cap, (shard + 16383) // 16384))
                    if best is not None and blocks == best[1]:
                        continue
                    ms = timed(lambda: cu.pushpull_inplace_umma(ctx.view, maps, wire_code(dt), 0, n, 1.0 / world,
                                                                blocks, 0, stream.cuda_stream),
                               args.iters, args.warmup, device, flush)
                    if best is None or ms < best[0]:
                        best = (ms, blocks)
                rows.append({"what": "ours_inplace_wgmma_tma", "bytes": nbytes, "dtype": str(dt)[6:], "ms": best[0],
                             "blocks": best[1], "alg_gbs": nbytes / best[0] / 1e6,
                             "bus_gbs": factor * nbytes / best[0] / 1e6})
            y = torch.ones(n, dtype=dt, device=device)
            if world > 1:
                ms = timed(lambda: dist.all_reduce(y), args.iters, args.warmup, device, flush)
                rows.append({"what": "nccl_all_reduce", "bytes": nbytes, "dtype": str(dt)[6:], "ms": ms,
                             "alg_gbs": nbytes / ms / 1e6, "bus_gbs": factor * nbytes / ms / 1e6})

                def ref_fn():
                    ev = ref.push_pull_([y], average=True)
                    stream.wait_event(ev)
                if not args.quick:
                    ms = timed(ref_fn, args.iters, args.warmup, device, flush)
                    rows.append({"what": "nccl_reference_style", "bytes": nbytes, "dtype": str(dt)[6:], "ms": ms,
                                 "alg_gbs": nbytes / ms / 1e6, "bus_gbs": factor * nbytes / ms / 1e6})
    # ---- whole-model gradient sets through the PUBLIC push_pull API vs the reference-style path
    from byteps_b200.models import get_model

    for mname in ("resnet50", "bert_large"):
        with torch.device("meta"):
            model = get_model(mname)
        shapes = [p.shape for p in model.parameters()]
        grads = [torch.ones(s, dtype=torch.bfloat16, device=device) for s in shapes]
        tot = sum(g.numel() * 2 for g in grads)

        def ours():
            hs = [eng.push_pull_async(g, g, True, "bench.%s.%d" % (mname, i), 0, -i, flush=False)
                  for i, g in enumerate(grads)]
            eng.flush()
            for h in hs:
                eng.synchronize(h)
        if tot <= eng.cfg.arena_bytes and not args.skip_api:
            ms = timed(ours, max(args.iters // 2, 3), 2, device, flush)
            rows.append({"what": "ours_api_all_grads", "model": mname, "bytes": tot, "ntensors": len(grads), "ms": ms,
                         "alg_gbs": tot / ms / 1e6, "bus_gbs": factor * tot / ms / 1e6})
        # the path DistributedOptimizer actually uses: gradients resident in the arena, one in-place
        # launch per 16 MB bucket, no per-tensor host work
        if tot <= ctx.data_bytes:
            bucket = 16 << 20
            spans, o = [], 0
            while o < tot:
                ln = min(bucket, tot - o)
                spans.append((o, ln // 2 // 8 * 8))
                o += ln

            def bucketed():
                for (bo, bn) in spans:
                    blocks = pick_blocks(bn * 2 // world, 512, 32, cap=64)
                    cu.pushpull_inplace(ctx.view, wire_code(torch.bfloat16), bo, bn, 1.0 / world, blocks, 512, 0,
                                        bool(ctx.nvls), stream.cuda_stream)
            ms = timed(bucketed, max(args.iters // 2, 3), 2, device, flush)
            rows.append({"what": "ours_bucketed_inplace_all_grads", "model": mname, "bytes": tot,
                         "ntensors": len(spans), "ms": ms, "alg_gbs": tot / ms / 1e6,
                         "bus_gbs": factor * tot / ms / 1e6})
            # the same buckets through ONE descriptor-ring launch: flags instead of two barriers per bucket,
            # no launch gaps, CTAs flow from bucket to bucket (csrc/kernels/pushpull_ring.cu)
            from byteps_b200.ops.ring import RingEntry, RingTable

            for part in (16 << 20, 4096000 // 256 * 256):
                pspans, o = [], 0
                while o < tot:
                    ln = min(part, tot - o)
                    pspans.append((o, ln // 2 // 8 * 8))
                    o += ln
                if len(pspans) > cu.RING_SLOTS:
                    continue
                table = RingTable([RingEntry(grad_off=bo, numel=bn, wire=wire_code(torch.bfloat16), slot=i,
                                             scale=1.0 / world, priority=-i) for i, (bo, bn) in enumerate(pspans)],
                                  device)
                for sched in (False, True):
                    best = None
                    for blocks in ((32,) if args.quick and sched else (16, 32, 64)):
                        ms = timed(lambda: table.launch(ctx.view, blocks, stream.cuda_stream, nvls=bool(ctx.nvls),
                                                        sched=sched), max(args.iters // 2, 3), 2, device, flush)
                        if best is None or ms < best[0]:
                            best = (ms, blocks)
                    rows.append({"what": "ours_ring_all_grads" + ("_sched" if sched else ""), "model": mname,
                                 "bytes": tot, "ntensors": len(pspans), "partition": part, "ms": best[0],
                                 "blocks": best[1], "alg_gbs": tot / best[0] / 1e6,
                                 "bus_gbs": factor * tot / best[0] / 1e6})
        if world > 1 and not args.quick:
            def refm():
                ev = ref.push_pull_(grads, average=True)
                stream.wait_event(ev)
            ms = timed(refm, max(args.iters // 2, 3), 2, device, flush)
            rows.append({"what": "nccl_reference_style_all_grads", "model": mname, "bytes": tot,
                         "ntensors": len(grads), "ms": ms, "alg_gbs": tot / ms / 1e6,
                         "bus_gbs": factor * tot / ms / 1e6})
    if rank == 0:
        res = {"n_gpus": world, "nvls": bool(ctx.nvls), "symm_mode": ctx.mem.mode, "rows": rows}
        print(json.dumps(res))
        if args.out:
            with open(args.out, "w") as f:
                json.dump(res, f, indent=1)
    torch.cuda.synchronize()
    dist.barrier()
    ctx.close()
    bps.shutdown()


if __name__ == "__main__":
    main()
