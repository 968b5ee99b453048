#!/usr/bin/env python
"""Synchronised batch norm (SyncBatchNormAct2d) against the rank-local fused passes, at the world size this
process can see (one GPU: world 1).

Per shape (the 12 distinct ResNet-50 batch-norm shapes at --batch images per rank, bf16 NHWC, BN + ReLU), CUDA
events over --iters launches time:

    local fwd   fwd_stats + fwd_apply
    sync fwd    fwd_stats_local + sync_stats + fwd_apply
    local bwd   bwd_reduce + bwd_apply
    sync bwd    bwd_reduce + sync_grad + bwd_apply (global count)

At world 1 the sync kernels exchange with their own rank only, so the difference is the cost of the two extra
small launches and the barrier on one GPU; the cost of the 106 cross-rank round trips of a ResNet-50 step over
NVLink needs a multi-GPU run and is printed as "not measured".  The whole-step rows time one ResNet-50 bf16
channels_last training step (forward, backward, SGD) with and without convert_sync_batchnorm at the same world.
The GPU name and power limit are printed with the table.

    python benchmarks/sync_bn_bench.py [--batch 64] [--iters 50] [--steps 30]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SHAPES = [(64, 112, 112), (64, 56, 56), (256, 56, 56), (128, 56, 56), (128, 28, 28), (512, 28, 28),
          (256, 28, 28), (256, 14, 14), (1024, 14, 14), (512, 14, 14), (512, 7, 7), (2048, 7, 7)]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def _time(torch, fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters   # us


def passes(torch, cu, vc, ctx, batch, iters):
    rows = []
    s = torch.cuda.current_stream().cuda_stream
    assert s == vc.streams[0].cuda_stream
    for c, h, w in SHAPES:
        m = batch * h * w
        dev, f32 = "cuda", dict(dtype=torch.float32, device="cuda")
        x = torch.randn(m, c, device=dev).to(torch.bfloat16)
        dy = torch.randn(m, c, device=dev).to(torch.bfloat16)
        y, dx = torch.empty_like(x), torch.empty_like(x)
        mask = torch.empty(m, c // 8, dtype=torch.uint8, device=dev)
        wt, bias = torch.ones(c, **f32), torch.zeros(c, **f32)
        rm, rv = torch.zeros(c, **f32), torch.ones(c, **f32)
        mean, invstd, total = torch.empty(c, **f32), torch.empty(c, **f32), torch.empty(1, **f32)
        local, sums, dw, db = torch.empty(2, c, **f32), torch.empty(2, c, **f32), torch.empty(c, **f32), torch.empty(c, **f32)
        nws, nctr = cu.bn_act_workspace(m, c)
        ws, ctr = torch.empty(nws, **f32), torch.zeros(nctr, dtype=torch.int32, device=dev)
        p = lambda t: t.data_ptr()  # noqa: E731

        def apply():
            cu.bn_act_fwd_apply(p(x), 0, 1, m, c, p(mean), p(invstd), p(wt), p(bias), True, p(y), p(mask), s)

        def local_fwd():
            cu.bn_act_fwd_stats(p(x), 1, m, c, 1e-5, 0.1, p(rm), p(rv), p(mean), p(invstd), p(ws), p(ctr), s)
            apply()

        def sync_fwd():
            cu.bn_act_fwd_stats_local(p(x), 1, m, c, p(local[0]), p(local[1]), p(ws), p(ctr), s)
            cu.bn_sync_stats(ctx.view, ctx.channel, 0, ctx.cmax, c, p(local[0]), p(local[1]), float(m), 1e-5, 0.1,
                             p(rm), p(rv), p(mean), p(invstd), p(total), s)
            apply()

        def local_bwd():
            cu.bn_act_bwd_reduce(p(dy), p(x), p(mask), 1, m, c, p(mean), p(invstd), p(dw), p(db), p(ws), p(ctr), s)
            cu.bn_act_bwd_apply(p(dy), p(x), p(mask), 1, m, c, p(mean), p(invstd), p(wt), p(dw), p(db), p(dx), 0, s)

        def sync_bwd():
            cu.bn_act_bwd_reduce(p(dy), p(x), p(mask), 1, m, c, p(mean), p(invstd), p(dw), p(db), p(ws), p(ctr), s)
            cu.bn_sync_grad(ctx.view, ctx.channel, 0, ctx.cmax, c, p(db), p(dw), p(sums[0]), p(sums[1]), s)
            cu.bn_act_bwd_apply(p(dy), p(x), p(mask), 1, m, c, p(mean), p(invstd), p(wt), p(sums[1]), p(sums[0]),
                                p(dx), 0, s, p(total))

        sync_fwd()   # mean / invstd for the backward timings
        rows.append(((c, h, w), _time(torch, local_fwd, iters), _time(torch, sync_fwd, iters),
                     _time(torch, local_bwd, iters), _time(torch, sync_bwd, iters)))
    return rows


def step_time(torch, sync_bn, batch, steps):
    import torch.nn.functional as F

    import byteps_b200.torch as bps
    from byteps_b200.models import resnet50

    torch.manual_seed(0)
    model = resnet50().cuda().to(memory_format=torch.channels_last).to(torch.bfloat16)
    for mod in model.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.float()
    if sync_bn:
        model = bps.convert_sync_batchnorm(model)
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    x = torch.randn(batch, 3, 224, 224, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device="cuda")

    def step():
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(model(x).float(), y).backward()
        opt.step()

    return _time(torch, step, steps) / 1e3   # ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()

    import torch

    import byteps_b200.torch as bps
    from byteps_b200 import _native
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops.bn_act import SyncBatchNormContext

    if not torch.cuda.is_available():
        raise SystemExit("sync_bn_bench.py needs a GPU")
    bps.init()
    world = bps.size()
    print("GPU: %s" % gpu_info())
    print("world size: %d" % world)
    cu = _native.cuda()
    vc = VirtualCluster(1, "cuda", SyncBatchNormContext.window_bytes(1, 2048))
    ctx = SyncBatchNormContext.from_virtual(vc, 0, 2048)
    with torch.cuda.stream(vc.streams[0]):
        rows = passes(torch, cu, vc, ctx, args.batch, args.iters)
    torch.cuda.synchronize()
    print("\nper-pass time, batch %d per rank, bf16 NHWC, BN + ReLU, world 1 (us)" % args.batch)
    print("%-14s %10s %10s %10s %10s" % ("C x H x W", "local fwd", "sync fwd", "local bwd", "sync bwd"))
    for (c, h, w), lf, sf, lb, sb in rows:
        print("%-14s %10.1f %10.1f %10.1f %10.1f" % ("%dx%dx%d" % (c, h, w), lf, sf, lb, sb))
    print("sum            %10.1f %10.1f %10.1f %10.1f" % tuple(sum(r[i] for r in rows) for i in range(1, 5)))
    print("sync passes at world > 1 over NVLink: not measured")

    base = step_time(torch, False, args.batch, args.steps)
    conv = step_time(torch, True, args.batch, args.steps)
    print("\nResNet-50 bf16 channels_last training step, batch %d, world %d: %.2f ms without, %.2f ms with "
          "convert_sync_batchnorm" % (args.batch, world, base, conv))
    if world == 1:
        print("(at world 1 the converted model takes the local path; the step at world > 1: not measured)")
    bps.shutdown()


if __name__ == "__main__":
    main()
