#!/usr/bin/env python
"""LARS in the fused exchange against fused SGD with momentum, on ResNet-50, one GPU.

Part "buckets": ResNet-50's parameters as bench.py builds them (bf16, channels_last, batch-norm parameters in fp32),
the exchange's 16 MB buckets, one param group (so both optimizers bucket alike).  For every bucket, CUDA events around --iters back-to-back launches of its update on
the comm stream: the fused SGD kernel (the TMA variant, the one-GPU default) against the three LARS kernels.  Printed
per bucket size class: microseconds, bytes moved and the rate.  Bytes come from shapes (bf16 parameters and
gradients, fp32 master and momentum):

    fused SGD    read g (2) + w, v (8), write w, v (8) + the bf16 parameter (2)                     = 20 B/element
    fused LARS   lars_norms_partial: read g (2) + w (4)
                 lars_apply:         read g (2) + w, v (8), write w, v (8) + the bf16 parameter (2)  = 26 B/element
                 (plus the per-parameter float64 partial sums: 16 B per 32 wire units, and the norm windows)
    least        one pass over g, w, v and back: 20 B/element.  LARS cannot reach it: the trust ratio needs the
                 whole parameter's ||g|| and ||w|| before any element of it is written.

Part "step": a whole ResNet-50 training step in bench.py's configuration (bf16, batch --batch, channels_last), each
step captured in one CUDA graph.  Three arms, built once and timed in --rounds alternating rounds of --steps replays:

    sgd     DistributedOptimizer(SGD(lr=0.01, momentum=0.9), fused_update=True), bench.py's optimizer
    lars    DistributedOptimizer(Lars, fused_update=True), batch-norm parameters and biases in an adapt=False,
            weight_decay=0 group
    plain   the plain Lars, per tensor, on fp32 master copies (gradients copied in, weights copied back)

Printed: ms/step per round, the median and the spread (max - min) per arm, and fused LARS's device memory beyond
fused SGD's.  The GPU name, power limit and SM clock are read in the same run.  Everything at world > 1 (the two
extra barrier round trips per bucket, the descriptor ring LARS does not use) needs several GPUs and is not measured
here.

    python benchmarks/lars_bench.py [--part buckets|step|all] [--iters 20] [--batch 64] [--steps 10] [--rounds 5]
"""
import argparse
import gc
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

BYTES_PER_ELEMENT = {"sgd": 20, "lars": 26}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def lars_groups(params):
    params = list(params)
    return [dict(params=[p for p in params if p.dim() > 1], weight_decay=5e-5),
            dict(params=[p for p in params if p.dim() <= 1], weight_decay=0.0, adapt=False)]


def resnet50(torch):
    from byteps_b200.models import get_model

    torch.manual_seed(0)
    model = get_model("resnet50").cuda().to(memory_format=torch.channels_last).to(torch.bfloat16)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.float()
    return model.train()


def make_opt(torch, kind, model, one_group=False):
    """one_group: LARS with every parameter in one group, so its buckets are SGD's (a bucket holds one group)."""
    import byteps_b200.torch as bps

    if kind == "sgd":
        inner = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    else:
        inner = bps.Lars(model.parameters() if one_group else lars_groups(model.parameters()), lr=0.5, momentum=0.9,
                         weight_decay=5e-5)
    return bps.DistributedOptimizer(inner, named_parameters=model.named_parameters(), fused_update=True)


def bucket_times(torch, kind, iters):
    """[(elements, microseconds per update)] per bucket of ResNet-50's parameters."""
    model = resnet50(torch)
    opt = make_opt(torch, kind, model, one_group=True)
    sync = opt.grad_sync
    cs = sync.comm_stream
    out = []
    for b in sync.buckets:
        for _ in range(2):
            sync._launch(b)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(cs)
        for _ in range(iters):
            sync._launch(b)
        t1.record(cs)
        torch.cuda.synchronize()
        out.append((b.numel, str(b.dtype)[6:], t0.elapsed_time(t1) * 1000.0 / iters))
    if kind == "lars":
        print("fused LARS device memory beyond fused SGD's: %d bytes (%d buckets, %d parameters)"
              % (sync.lamb_device_bytes(), len(sync.buckets), sum(len(b.params) for b in sync.buckets)))
    sync._reset()
    sync.close()
    del opt, model, sync
    gc.collect()
    torch.cuda.empty_cache()
    return out


def part_buckets(torch, iters):
    res = {k: bucket_times(torch, k, iters) for k in ("sgd", "lars")}
    assert [n for n, _, _ in res["sgd"]] == [n for n, _, _ in res["lars"]], "the two optimizers bucket differently"
    print("per bucket (16 MB buckets, world 1; %d launches each; bytes per element of bf16 buckets, fp32 buckets "
          "move 2 x 2 B more):" % iters)
    print("  %10s %5s %10s %10s %9s %10s %10s" % ("elements", "dtype", "SGD us", "LARS us", "LARS/SGD", "SGD GB/s",
                                                 "LARS GB/s"))
    for (n, dt, ts), (_, _, tl) in zip(res["sgd"], res["lars"]):
        extra = 4 if dt == "float32" else 0
        bs, bl = n * (BYTES_PER_ELEMENT["sgd"] + extra), n * (BYTES_PER_ELEMENT["lars"] + 2 * extra)
        print("  %10d %5s %10.1f %10.1f %9.2f %10.0f %10.0f" % (n, dt[:5], ts, tl, tl / ts, bs / ts / 1e3,
                                                                bl / tl / 1e3))
    tot_n = sum(n for n, _, _ in res["sgd"])
    tot_s = sum(t for _, _, t in res["sgd"])
    tot_l = sum(t for _, _, t in res["lars"])
    print("  all %d buckets, %d elements: SGD %.0f us, LARS %.0f us (x%.2f)" % (len(res["sgd"]), tot_n, tot_s, tot_l,
                                                                             tot_l / tot_s))


def build_step(torch, name, batch):
    import torch.nn.functional as F

    import byteps_b200.torch as bps
    from byteps_b200.torch.graph import GraphedStep

    model = resnet50(torch)
    g = torch.Generator().manual_seed(1)
    x = torch.rand(batch, 3, 224, 224, generator=g).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last).cuda()
    y = torch.randint(0, 1000, (batch,), generator=g).cuda()
    if name == "plain":
        params = list(model.parameters())
        masters = [torch.nn.Parameter(p.detach().float()) for p in params]
        for m in masters:
            m.grad = torch.zeros_like(m)
        opt = bps.Lars(lars_groups(masters), lr=0.5, momentum=0.9)

        def step():
            for p in params:
                p.grad = None
            loss = F.cross_entropy(model(x).float(), y)
            loss.backward()
            with torch.no_grad():
                for m, p in zip(masters, params):
                    if p.grad is not None:
                        m.grad.copy_(p.grad)
                opt.step()
                torch._foreach_copy_(params, masters)
            return loss

        return GraphedStep(step, warmup=3)
    opt = make_opt(torch, name, model)

    def step():
        opt.zero_grad()
        loss = F.cross_entropy(model(x).float(), y)
        loss.backward()
        opt.step()
        return loss

    return GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams)


def part_step(torch, batch, steps, rounds):
    arms = {name: build_step(torch, name, batch) for name in ("sgd", "lars", "plain")}
    times = {name: [] for name in arms}
    for name, g in arms.items():         # one untimed replay each
        g()
    torch.cuda.synchronize()
    for r in range(rounds):
        for name, g in arms.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(steps):
                g()
            t1.record()
            torch.cuda.synchronize()
            times[name].append(t0.elapsed_time(t1) / steps)
        print("  round %d: %s" % (r, "  ".join("%s %.2f ms" % (n, t[-1]) for n, t in times.items())), flush=True)
    print("ResNet-50 step (bf16, batch %d, channels_last, one CUDA graph, world 1):" % batch)
    for name, t in times.items():
        print("  %-6s median %.2f ms/step, spread %.2f ms over %d rounds of %d steps"
              % (name, statistics.median(t), max(t) - min(t), rounds, steps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=("buckets", "step", "all"), default="all")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch

    import byteps_b200.torch as bps

    if not torch.cuda.is_available():
        raise SystemExit("lars_bench needs a GPU")
    print("GPU (name, power limit, max SM clock, SM clock):", gpu_info())
    bps.init()
    if args.part in ("buckets", "all"):
        part_buckets(torch, args.iters)
    if args.part in ("step", "all"):
        part_step(torch, args.batch, args.steps, args.rounds)
    print("GPU after the run:", gpu_info())
    bps.shutdown()


if __name__ == "__main__":
    main()
