#!/usr/bin/env python
"""Fused softmax cross-entropy (ops/xent.py, kernels/xent.cu) against the stock loss of BERT's masked-LM head:
``F.cross_entropy(logits.float(), labels, ignore_index=-100)``.

Per pass: 8192 x 30522 bf16 logits (batch 64 x sequence 128 tokens over BERT's vocabulary), mean reduction, with
every row labelled (as bench.py --model bert_large draws its labels) and with 15 % of the rows labelled (MLM
masking; the others carry ignore_index).  Each timed pass runs on the next of enough copies of the logits that the
copies span more than --rotate-mb together, so no pass finds its input in the 50 MB L2; the launches of --iters
passes are captured in one CUDA graph and the graph's replays are timed with CUDA events, so host overhead does not
enter.  bwd is fwd + backward minus fwd.  Bytes are the least each path moves, computed from the shape (e = element
bytes, N = M V elements, f = share of labelled rows, per-row targets / lse / loss 16 M):

    fused fwd    read the labelled rows                                              f N e + 16 M
    fused bwd    read the labelled rows, write dlogits                              (1 + f) N e + 16 M
    stock fwd    cast: read x, write fp32 x; log_softmax: read it, write fp32 out     N (e + 12)
    stock bwd    nll_loss backward: write the fp32 one-hot gradient; log_softmax backward: read it and the
                 saved output, write fp32 dx; cast back: read it, write dx              N (20 + e)

Share of peak is against the H100 SXM data-sheet 3.35 TB/s.

Whole step: BERT-large bf16 with fused_norm=True, batch 64, sequence 128, every position labelled, AdamW through
DistributedOptimizer(fused_update=True), the whole step captured in one CUDA graph as bench.py builds it.  The stock
loss and fused_loss=True steps share one model and optimizer; each is captured once and the two graphs are timed
alternately, --rounds rounds of --steps replays each.  The GPU name, power limit and SM clock are read in the same
run.

    python benchmarks/xent_bench.py [--iters 20] [--rotate-mb 1200] [--steps 20] [--rounds 5] [--no-step] [--json f]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0
M, V = 8192, 30522
LABELLED = [1.0, 0.15]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def pass_bytes(path, kind, m, v, e, f):
    n = m * v
    if path == "fused":
        return int((f if kind == "fwd" else 1 + f) * n * e) + 16 * m
    return n * (e + 12) if kind == "fwd" else n * (20 + e)


def per_pass(args, torch, F, rows):
    from byteps_b200.ops.xent import softmax_cross_entropy

    dev = torch.device("cuda", 0)
    dt, e = torch.bfloat16, 2

    def graphed_us(fn, k):
        """us per call of fn(i), i over the k copies, --iters calls captured in one graph"""
        for i in range(k):
            fn(i)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(args.iters):
                fn(i % k)
        g.replay()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            g.replay()
        b.record()
        torch.cuda.synchronize()
        us = a.elapsed_time(b) * 1e3 / (args.reps * args.iters)
        del g
        return us

    print("%-12s %-8s %-6s %-4s %9s %9s %8s %6s" % ("M x V", "labelled", "path", "pass", "MB", "us", "GB/s", "%peak"))
    k = max(2, int(-(-args.rotate_mb * 1e6 // (M * V * e))))
    gen = torch.Generator(device=dev).manual_seed(0)
    X = [(torch.randn(M, V, device=dev, generator=gen, dtype=torch.float32) * 2).to(dt).requires_grad_(True)
         for _ in range(k)]
    for f in LABELLED:
        t = torch.randint(0, V, (M,), device=dev, generator=gen)
        t[torch.rand(M, device=dev, generator=gen) >= f] = -100
        fns = {
            "fused": lambda x: softmax_cross_entropy(x, t, ignore_index=-100),
            "stock": lambda x: F.cross_entropy(x.float(), t, ignore_index=-100),
        }
        for path, fn in fns.items():
            def fwd(i, fn=fn):
                fn(X[i])

            def both(i, fn=fn):
                torch.autograd.grad(fn(X[i]), [X[i]])

            us_f = graphed_us(fwd, k)
            us_b = graphed_us(both, k) - us_f
            for kind, us in (("fwd", us_f), ("bwd", us_b)):
                nbytes = pass_bytes(path, kind, M, V, e, f)
                gbs = nbytes / (us * 1e3)
                rows.append(dict(shape=[M, V], labelled=f, path=path, kind=kind, bytes=nbytes, us=us, gbs=gbs,
                                 peak_share=gbs / PEAK_GBS))
                print("%-12s %-8s %-6s %-4s %9.1f %9.1f %8.0f %5.0f%%" % (
                    "%dx%d" % (M, V), "%d %%" % round(100 * f), path, kind, nbytes / 1e6, us, gbs,
                    100 * gbs / PEAK_GBS))
    del X


def whole_step(args, torch, rows):
    import byteps_b200.torch as bps
    from byteps_b200.models import bert_large
    from byteps_b200.torch.graph import GraphedStep

    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = True
    bps.init()
    torch.manual_seed(0)
    model = bert_large(fused_norm=True).to(dev).to(torch.bfloat16).train()
    opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01),
                                   named_parameters=model.named_parameters(), fused_update=True)
    gen = torch.Generator().manual_seed(1234)
    ids = torch.randint(0, 30522, (args.batch, args.seq), generator=gen).to(dev)
    labels = torch.randint(0, 30522, (args.batch, args.seq), generator=gen).to(dev)

    def step():
        opt.zero_grad()
        loss = model(ids, mlm_labels=labels)
        loss.backward()
        opt.step()
        return loss

    graphs = {}
    for fused in (False, True):
        model.config.fused_loss = fused     # read at every forward, so each capture takes its own loss path
        graphs[fused] = GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams, device=dev)
    model.config.fused_loss = False

    def timed(g):
        for _ in range(3):
            g()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            g()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps

    ms = {False: [], True: []}
    for _ in range(args.rounds):
        for fused in (False, True):
            ms[fused].append(timed(graphs[fused]))
    info = gpu_info()
    for fused in (False, True):
        name = "fused_loss" if fused else "stock"
        best = min(ms[fused])
        rows.append(dict(step=name, ms=ms[fused], best_ms=best,
                         tokens_per_s=args.batch * args.seq / (best / 1e3)))
        print("BERT-large step %-10s ms per step over %d rounds: %s  (best %.2f ms, %.0f tokens/s)" % (
            name, args.rounds, " ".join("%.2f" % v for v in ms[fused]), best, args.batch * args.seq / (best / 1e3)))
    print("GPU after the step rounds: %s" % info)
    del graphs
    bps.shutdown()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="passes captured in one timed graph")
    ap.add_argument("--reps", type=int, default=5, help="replays of that graph")
    ap.add_argument("--rotate-mb", type=float, default=1200.0, help="bytes the logits copies span together")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20, help="timed replays of a whole step per round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-step", action="store_true", help="per-pass table only")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F

    from byteps_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("xent_bench.py needs a GPU")
    _native.cuda()
    torch.cuda.set_device(0)
    info = gpu_info()
    print("GPU: %s; bf16 logits, mean reduction" % info)
    rows = []
    per_pass(args, torch, F, rows)
    if not args.no_step:
        whole_step(args, torch, rows)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
