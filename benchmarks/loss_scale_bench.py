#!/usr/bin/env python
"""Dynamic loss scaling of the fused optimizer against the two ways the project offered fp16 training before it.

ResNet-50 in fp16 (batch-norm affine parameters in fp32), channels_last, batch --batch, SGD with momentum, one GPU.
Three arms, built once and timed in --rounds alternating rounds of --steps steps each (CUDA events around the steps,
ending in a device synchronise):

    static    HalfPrecisionDistributedOptimizer(loss_scale=1024): the fused update, whole step in one CUDA graph
    dynamic   DistributedOptimizer(fused_update=True, dynamic_loss_scale=True), whole step in one CUDA graph
    eager     HalfPrecisionDistributedOptimizer(dynamic_loss_scale=True): unfused exchange, an isfinite reduction
              per parameter, a host sync per step, torch.optim on fp32 masters, eager

Printed: ms/step per round and the median per arm, and the skipped-step count of the two dynamic arms.  The GPU name
and power limit are read in the same run.  The dynamic mode issues the update at the step instead of during
backward; what that costs at world > 1 (where the update overlapped with backward) needs several GPUs and is
printed as "not measured".

    python benchmarks/loss_scale_bench.py [--batch 64] [--steps 30] [--rounds 3] [--warmup 5]
"""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def build_arm(torch, name, batch, warmup):
    """(run one step, skipped-step count) of one arm."""
    import torch.nn.functional as F

    import byteps_b200.torch as bps
    from byteps_b200.models import resnet50
    from byteps_b200.torch.graph import GraphedStep
    from byteps_b200.torch.half_optimizer import HalfPrecisionDistributedOptimizer

    torch.manual_seed(0)
    model = resnet50().cuda().to(memory_format=torch.channels_last).to(torch.float16)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.float()
    inner = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    if name == "static":
        opt = HalfPrecisionDistributedOptimizer(inner, named_parameters=model.named_parameters(), loss_scale=1024.0)
    elif name == "dynamic":
        opt = bps.DistributedOptimizer(inner, named_parameters=model.named_parameters(), fused_update=True,
                                       dynamic_loss_scale=True)
    else:
        opt = HalfPrecisionDistributedOptimizer(inner, named_parameters=model.named_parameters(),
                                                dynamic_loss_scale=True)
    x = torch.randn(batch, 3, 224, 224, device="cuda").to(torch.float16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device="cuda")

    def step():
        opt.zero_grad()
        loss = F.cross_entropy(model(x).float(), y)
        opt.scale_loss(loss).backward()
        opt.step()
        return loss

    if name == "eager":
        for _ in range(warmup):
            step()
        return step, lambda: opt.skipped_steps
    g = GraphedStep(step, warmup=warmup, pre_replay=opt.refresh_hparams)
    skipped = (lambda: opt.skipped_steps) if name == "dynamic" else (lambda: None)
    return g, skipped


def time_steps(torch, fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch

    import byteps_b200.torch as bps

    if not torch.cuda.is_available():
        raise SystemExit("loss_scale_bench.py needs a GPU")
    torch.cuda.set_device(0)
    bps.init()
    print("GPU: %s" % gpu_info())
    print("world size: %d" % bps.size())
    names = ["static", "dynamic", "eager"]
    arms = {n: build_arm(torch, n, args.batch, args.warmup) for n in names}
    times = {n: [] for n in names}
    for r in range(args.rounds):
        for n in (names if r % 2 == 0 else names[::-1]):
            times[n].append(time_steps(torch, arms[n][0], args.steps))
    print("\nResNet-50 fp16 (BN affine fp32), channels_last, batch %d, SGD momentum, %d rounds x %d steps (ms/step)"
          % (args.batch, args.rounds, args.steps))
    for n in names:
        sk = arms[n][1]()
        print("%-8s median %7.2f  rounds %s  skipped steps %s" % (
            n, statistics.median(times[n]), " ".join("%.2f" % t for t in times[n]),
            "-" if sk is None else sk))
    print("cost of the deferred update at world > 1: not measured")
    bps.shutdown()


if __name__ == "__main__":
    main()
