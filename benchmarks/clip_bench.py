#!/usr/bin/env python
"""Global gradient-norm clipping in the fused exchange (max_grad_norm), one GPU.

Part "kernels": BERT-large's parameters in bf16, the exchange's 16 MB buckets, fused AdamW with max_grad_norm=1.0.
CUDA events around --iters back-to-back launches of each bucket's norm pass (clip_norm_partial) on the comm stream,
and of the per-step clip_norm_update.  The norm pass reads the bucket's bf16 gradients once: 2 B/element at world 1.
Also printed: the device memory clipping adds.

Part "bert": a whole BERT-large training step, bf16, batch --batch x --seq, fp8_linear + fused_norm + fused_loss.
Arms, built once and timed in --rounds alternating rounds of --steps steps, medians and spreads printed (the AdamW
arms and the LAMB arms in two sets):

    adamw, adamw_clip   DistributedOptimizer(AdamW, fused_update=True), without and with max_grad_norm=1.0; one
                        CUDA graph per step
    lamb, lamb_clip     the same with Lamb (BERT's two groups)
    unfused_clip        DistributedOptimizer(AdamW, fused_update=False, max_grad_norm=1.0): synchronize(),
                        clip_grad_norm_ and torch's AdamW on the bf16 parameters, eager (torch's non-capturable AdamW)

Part "resnet": ResNet-50 bf16 channels_last, batch --resnet-batch, fused SGD momentum, one CUDA graph per step,
without and with max_grad_norm=1.0, alternating rounds as above.

The GPU name, power limit and SM clock are read in the same run.  Nothing at world > 1 is measured here.

    python benchmarks/clip_bench.py [--part kernels|bert|resnet|all] [--iters 20] [--batch 64] [--seq 128]
                                    [--resnet-batch 64] [--steps 10] [--rounds 5]
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


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def lamb_groups(params):
    params = list(params)
    return [dict(params=[p for p in params if p.dim() > 1], weight_decay=0.01),
            dict(params=[p for p in params if p.dim() <= 1], weight_decay=0.0, adapt=False)]


def free(torch):
    gc.collect()
    torch.cuda.empty_cache()


def part_kernels(torch, iters):
    import byteps_b200.torch as bps
    from byteps_b200.models import bert_large

    model = bert_large().cuda().to(torch.bfloat16)
    opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01),
                                   named_parameters=model.named_parameters(), fused_update=True, max_grad_norm=1.0)
    sync = opt.grad_sync
    cu, cs = sync.ctx.cu, sync.comm_stream
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    total, elems = 0.0, 0
    for b in sync.buckets:
        for _ in range(2):
            sync._launch_norm(b)
        t0, t1 = ev(), ev()
        t0.record(cs)
        for _ in range(iters):
            sync._launch_norm(b, wait=False)
        t1.record(cs)
        torch.cuda.synchronize()
        total += t0.elapsed_time(t1) * 1000.0 / iters
        elems += b.numel

    def update():
        cu.clip_norm_update(sync.ctx.view, 0, sync.clip_win_off, sync._clip_scratch.data_ptr(), len(sync.buckets),
                            sync._clip_scratch.shape[1], 1.0, sync._grad_norm.data_ptr(), sync._hp_dev.data_ptr(),
                            len(sync.param_groups), cs.cuda_stream)

    for _ in range(2):
        update()
    t0, t1 = ev(), ev()
    t0.record(cs)
    for _ in range(iters):
        update()
    t1.record(cs)
    torch.cuda.synchronize()
    tu = t0.elapsed_time(t1) * 1000.0 / iters
    print("clipping kernels, BERT-large bf16, %d buckets, %d elements, world 1 (%d launches each):"
          % (len(sync.buckets), elems, iters))
    print("  clip_norm_partial over all buckets: %.1f us, %.1f MB read (2 B/element), %.0f GB/s"
          % (total, elems * 2 / 1e6, elems * 2 / total / 1e3))
    print("  clip_norm_update: %.1f us" % tu)
    print("  device memory added by clipping: %d bytes" % sync.clip_device_bytes())
    sync._reset()
    sync.close()
    del opt, model, sync
    free(torch)


def bert_arm(torch, name, batch, seq):
    import byteps_b200.torch as bps
    from byteps_b200.models import bert_large
    from byteps_b200.torch.graph import GraphedStep

    torch.manual_seed(0)
    model = bert_large(fp8_linear=True, fused_norm=True, fused_loss=True).cuda().to(torch.bfloat16).train()
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 30522, (batch, seq), generator=g).cuda()
    labels = torch.randint(0, 30522, (batch, seq), generator=g)
    labels[torch.rand(batch, seq, generator=g) > 0.15] = -100
    labels = labels.cuda()
    clip = 1.0 if name.endswith("_clip") else None
    if name.startswith("lamb"):
        inner = bps.Lamb(lamb_groups(model.parameters()), lr=1e-3)
    else:
        inner = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01)
    opt = bps.DistributedOptimizer(inner, named_parameters=model.named_parameters(),
                                   fused_update=name != "unfused_clip", max_grad_norm=clip)

    def step():
        opt.zero_grad()
        loss = model(ids, mlm_labels=labels)
        loss.backward()
        opt.step()
        return loss

    if name == "unfused_clip":
        return step
    return GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams)


def resnet_arm(torch, name, batch):
    import torch.nn.functional as F

    import byteps_b200.torch as bps
    from byteps_b200.models import resnet50
    from byteps_b200.torch.graph import GraphedStep

    torch.manual_seed(0)
    model = resnet50().cuda().to(memory_format=torch.channels_last).to(torch.bfloat16)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.float()
    opt = bps.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=5e-5),
                                   named_parameters=model.named_parameters(), fused_update=True,
                                   max_grad_norm=1.0 if name == "sgd_clip" else None)
    g = torch.Generator().manual_seed(1)
    x = torch.rand(batch, 3, 224, 224, generator=g).cuda().to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), generator=g).cuda()

    def step():
        opt.zero_grad()
        loss = F.cross_entropy(model(x).float(), y)
        loss.backward()
        opt.step()
        return loss

    return GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams)


def alternate(torch, arms, steps, rounds, title):
    times = {name: [] for name in arms}
    for g in arms.values():         # one untimed step each
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
    print(title)
    for name, t in times.items():
        print("  %-13s median %.2f ms/step, spread %.2f ms over %d rounds of %d steps"
              % (name, statistics.median(t), max(t) - min(t), rounds, steps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=("kernels", "bert", "resnet", "all"), default="all")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--resnet-batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch

    import byteps_b200.torch as bps

    if not torch.cuda.is_available():
        raise SystemExit("clip_bench needs a GPU")
    print("GPU (name, power limit, max SM clock, SM clock):", gpu_info())
    bps.init()
    if args.part in ("kernels", "all"):
        part_kernels(torch, args.iters)
    if args.part in ("bert", "all"):
        # two sets of arms, so that no more than three BERT-large models share the card
        for names in (("adamw", "adamw_clip", "unfused_clip"), ("lamb", "lamb_clip")):
            arms = {n: bert_arm(torch, n, args.batch, args.seq) for n in names}
            alternate(torch, arms, args.steps, args.rounds,
                      "BERT-large step (bf16, batch %d x %d, fp8_linear + fused_norm + fused_loss, world 1):"
                      % (args.batch, args.seq))
            del arms
            free(torch)
    if args.part in ("resnet", "all"):
        arms = {n: resnet_arm(torch, n, args.resnet_batch) for n in ("sgd", "sgd_clip")}
        alternate(torch, arms, args.steps, args.rounds,
                  "ResNet-50 step (bf16 channels_last, batch %d, fused SGD momentum, one CUDA graph, world 1):"
                  % args.resnet_batch)
    print("GPU after the run:", gpu_info())
    bps.shutdown()


if __name__ == "__main__":
    main()
