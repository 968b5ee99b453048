#!/usr/bin/env python
"""LAMB in the fused exchange against fused AdamW, on BERT-large, one GPU.

Part "buckets": BERT-large's parameters in bf16, the exchange's 16 MB buckets, one param group.  For every bucket,
CUDA events around --iters back-to-back launches of its update on the comm stream: the fused AdamW kernel (the TMA
variant, the one-GPU default) against the three LAMB kernels.  Printed per bucket size class: microseconds, bytes
moved and the least bytes, and the rate.  Bytes come from shapes (bf16 parameters and gradients, fp32 master and
moments):

    fused AdamW   read g (2) + w, m, v (12), write w, m, v (12) + the bf16 parameter (2)          = 28 B/element
    fused LAMB    lamb_moments: read g (2) + w, m, v (12), write m, v (8)
                  lamb_apply:   read w, m, v (12), write w (4) + the bf16 parameter (2)             = 40 B/element
                  (plus the per-parameter float64 partial sums: 16 B per 32 wire units, and the norm windows)
    least         one pass over g, w, m, v and back: 28 B/element.  LAMB cannot reach it: the trust ratio needs
                  the whole parameter's ||u|| before any element of it is written.

Part "step": a whole BERT-large training step, bf16, batch --batch x --seq, fp8_linear, fused_norm, fused_loss, each
step captured in one CUDA graph.  Three arms, built once and timed in --rounds alternating rounds of --steps replays:

    adamw   DistributedOptimizer(AdamW, fused_update=True)
    lamb    DistributedOptimizer(Lamb, fused_update=True), BERT's two groups (1-D parameters without decay and
            without the trust ratio)
    plain   the plain Lamb, per tensor, on fp32 master copies (gradients copied in, weights copied back).  On one
            GPU there is no exchange; the captured graph keeps the bias corrections of the step it captured, which
            does not change the work.

Printed: ms/step per round, the median and the spread (max - min) per arm.  The GPU name, power limit and SM clock
are read in the same run.  Everything at world > 1 (the two extra barrier round trips per bucket, the descriptor
ring LAMB does not use) needs several GPUs and is not measured here.

    python benchmarks/lamb_bench.py [--part buckets|step|all] [--iters 20] [--batch 64] [--seq 128]
                                    [--steps 10] [--rounds 5]
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

BYTES_PER_ELEMENT = {"adamw": 28, "lamb": 40}
LEAST_BYTES_PER_ELEMENT = 28


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


def bucket_times(torch, kind, iters):
    """[(elements, microseconds per update)] per bucket of BERT-large's bf16 parameters."""
    import byteps_b200.torch as bps
    from byteps_b200.models import bert_large

    model = bert_large().cuda().to(torch.bfloat16)
    inner = (torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01) if kind == "adamw"
             else bps.Lamb(model.parameters(), lr=1e-3, weight_decay=0.01))
    opt = bps.DistributedOptimizer(inner, named_parameters=model.named_parameters(), fused_update=True)
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
        out.append((b.numel, t0.elapsed_time(t1) * 1000.0 / iters))
    if kind == "lamb":
        print("fused LAMB device memory beyond fused Adam's: %d bytes (%d buckets, %d parameters)"
              % (sync.lamb_device_bytes(), len(sync.buckets), sum(len(b.params) for b in sync.buckets)))
    sync._reset()
    sync.close()
    del opt, model, sync
    gc.collect()
    torch.cuda.empty_cache()
    return out


def part_buckets(torch, iters):
    res = {k: bucket_times(torch, k, iters) for k in ("adamw", "lamb")}
    assert [n for n, _ in res["adamw"]] == [n for n, _ in res["lamb"]], "the two optimizers bucket differently"
    classes = {}
    for (n, ta), (_, tl) in zip(res["adamw"], res["lamb"]):
        classes.setdefault(n, []).append((ta, tl))
    print("per bucket (bf16 parameters, 16 MB buckets, world 1; %d launches each):" % iters)
    print("  %10s %4s %12s %12s %9s %9s %9s %11s %11s" % ("elements", "n", "AdamW us", "LAMB us", "LAMB/Adam",
                                                           "Adam MB", "LAMB MB", "Adam GB/s", "LAMB GB/s"))
    for n in sorted(classes, reverse=True):
        ta = statistics.median(t for t, _ in classes[n])
        tl = statistics.median(t for _, t in classes[n])
        ba, bl = n * BYTES_PER_ELEMENT["adamw"], n * BYTES_PER_ELEMENT["lamb"]
        print("  %10d %4d %12.1f %12.1f %9.2f %9.1f %9.1f %11.0f %11.0f" % (n, len(classes[n]), ta, tl, tl / ta,
                                                                          ba / 1e6, bl / 1e6, ba / ta / 1e3,
                                                                          bl / tl / 1e3))
    tot_n = sum(n for n, _ in res["adamw"])
    tot_a = sum(t for _, t in res["adamw"])
    tot_l = sum(t for _, t in res["lamb"])
    print("  all %d buckets, %d elements: AdamW %.0f us, LAMB %.0f us (x%.2f); least bytes %.0f MB, moved %.0f / %.0f MB"
          % (len(res["adamw"]), tot_n, tot_a, tot_l, tot_l / tot_a, tot_n * LEAST_BYTES_PER_ELEMENT / 1e6,
             tot_n * BYTES_PER_ELEMENT["adamw"] / 1e6, tot_n * BYTES_PER_ELEMENT["lamb"] / 1e6))


def build_step(torch, name, batch, seq):
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
    if name == "plain":
        params = list(model.parameters())
        masters = [torch.nn.Parameter(p.detach().float()) for p in params]
        for m in masters:
            m.grad = torch.zeros_like(m)
        opt = bps.Lamb(lamb_groups(masters), lr=1e-3)

        def step():
            for p in params:
                p.grad = None
            loss = model(ids, mlm_labels=labels)
            loss.backward()
            with torch.no_grad():
                for m, p in zip(masters, params):
                    if p.grad is not None:
                        m.grad.copy_(p.grad)
                opt.step()
                torch._foreach_copy_(params, masters)
            return loss

        return GraphedStep(step, warmup=3)
    inner = (torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01) if name == "adamw"
             else bps.Lamb(lamb_groups(model.parameters()), lr=1e-3))
    opt = bps.DistributedOptimizer(inner, named_parameters=model.named_parameters(), fused_update=True)

    def step():
        opt.zero_grad()
        loss = model(ids, mlm_labels=labels)
        loss.backward()
        opt.step()
        return loss

    return GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams)


def part_step(torch, batch, seq, steps, rounds):
    arms = {name: build_step(torch, name, batch, seq) for name in ("adamw", "lamb", "plain")}
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
    print("BERT-large step (bf16, batch %d x %d, fp8_linear + fused_norm + fused_loss, one CUDA graph, world 1):"
          % (batch, seq))
    for name, t in times.items():
        print("  %-6s median %.2f ms/step, spread %.2f ms over %d rounds of %d steps"
              % (name, statistics.median(t), max(t) - min(t), rounds, steps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=("buckets", "step", "all"), default="all")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch

    import byteps_b200.torch as bps

    if not torch.cuda.is_available():
        raise SystemExit("lamb_bench needs a GPU")
    print("GPU (name, power limit, max SM clock, SM clock):", gpu_info())
    bps.init()
    if args.part in ("buckets", "all"):
        part_buckets(torch, args.iters)
    if args.part in ("step", "all"):
        part_step(torch, args.batch, args.seq, args.steps, args.rounds)
    print("GPU after the run:", gpu_info())
    bps.shutdown()


if __name__ == "__main__":
    main()
