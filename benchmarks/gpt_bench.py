#!/usr/bin/env python
"""Causal fused self-attention (ops/attn.py with causal=True, kernels/attn_causal.cu) and a graphed GPT-2 small step.

Per call, in bf16 with D = 64, at (B, S, H) = (16, 512, 12), (8, 512, 16) and (64, 128, 12), p = 0.1 and p = 0,
fwd and fwd+bwd (torch.autograd.grad to qkv) of three arms: the causal fused kernels, the bidirectional fused kernels
(the work the causal ones skip is the difference), and SDPA with is_causal=True, whose backend is read from the
kernel names of one profiled fwd+bwd.  As in attn_bench.py, each timed call runs on the next of enough copies of qkv
and dout that they span more than --rotate-mb together, so no call finds its inputs in the 50 MB L2; --iters calls
are captured in one CUDA graph and its replays are timed with CUDA events.

Per junction of the pre-LN residual stream, bf16 8192 x 768 with bf16 gamma / beta and p = 0.1: fwd and fwd+bwd
(torch.autograd.grad to y, residual, gamma and beta, with gradients arriving at both the LayerNorm's output and the
sum z) of DropoutAddLayerNorm with return_sum=True against the stock z = residual + F.dropout(y), F.layer_norm(z);
rotated copies and graphed replays as above.

Whole step: gpt2_small (124 M) in bf16 at 16 x 512, fused AdamW through DistributedOptimizer(fused_update=True),
the whole step in one CUDA graph: stock (SDPA, F.cross_entropy), fused_attention + fused_loss, that with fused_norm,
and those two with fp8_linear.  The arms are separate models with the same initial weights, timed alternately over
--rounds rounds of --steps replays; medians and spreads.  The GPU name, power limit and SM clock are read in the
same run.

    python benchmarks/gpt_bench.py [--iters 20] [--rotate-mb 200] [--steps 20] [--rounds 5] [--no-step]
                                   [--no-call] [--no-junction] [--json f]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from benchmarks.attn_bench import gpu_info, sdpa_backend  # noqa: E402

D = 64
SHAPES = [(16, 512, 12), (8, 512, 16), (64, 128, 12)]


def graphed_us(args, torch, fn, k):
    """us per call of fn(i % k), --iters calls captured in one graph, timed over --reps replays"""
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


def per_call(args, torch, rows):
    from byteps_b200.ops.attn import _stock, self_attention

    dev = torch.device("cuda", 0)
    dt = torch.bfloat16

    print("%-12s %-4s %-14s %-8s %9s" % ("B x S x H", "p", "path", "pass", "us"))
    for (b, s, h) in SHAPES:
        e = h * D
        per_copy = b * s * e * 2 * 4
        k = max(2, int(-(-args.rotate_mb * 1e6 // per_copy)))
        gen = torch.Generator(device=dev).manual_seed(0)
        T = [((torch.randn(b, s, 3 * e, device=dev, generator=gen) * 1.5).to(dt).requires_grad_(True),
              torch.randn(b, s, e, device=dev, generator=gen).to(dt)) for _ in range(k)]
        for p in (0.1, 0.0):
            fns = {"causal_fused": lambda x, p=p: self_attention(x, h, None, p, True, causal=True),
                   "full_fused": lambda x, p=p: self_attention(x, h, None, p, True),
                   "causal_sdpa": lambda x, p=p: _stock(x, h, None, p, causal=True)}
            res = {}
            for path, f in fns.items():
                def fwd(i, f=f):
                    f(T[i][0])

                def both(i, f=f):
                    x, dout = T[i]
                    torch.autograd.grad(f(x), [x], dout)

                us_f, us_fb = graphed_us(args, torch, fwd, k), graphed_us(args, torch, both, k)
                res[path] = (us_f, us_fb)
                backend = sdpa_backend(torch, both) if path == "causal_sdpa" else "byteps_b200 attn kernels"
                for kind, us in (("fwd", us_f), ("fwd+bwd", us_fb)):
                    rows.append(dict(shape=[b, s, h], p=p, path=path, kind=kind, us=us, backend=backend))
                    print("%-12s %-4g %-14s %-8s %9.1f" % ("%dx%dx%d" % (b, s, h), p, path, kind, us))
                if path == "causal_sdpa":
                    print("             SDPA kernels: %s" % backend)
            c, f, sd = res["causal_fused"], res["full_fused"], res["causal_sdpa"]
            print("             causal / full fused: fwd %.2f, fwd+bwd %.2f;  SDPA / causal fused: fwd %.2fx, "
                  "fwd+bwd %.2fx" % (c[0] / f[0], c[1] / f[1], sd[0] / c[0], sd[1] / c[1]))
        del T


def per_junction(args, torch, rows, m=8192, h=768, p=0.1):
    import torch.nn.functional as F

    from byteps_b200.ops.ln import dropout_add_layer_norm

    dev = torch.device("cuda", 0)
    dt = torch.bfloat16
    per_copy = m * h * 2 * 4
    k = max(2, int(-(-args.rotate_mb * 1e6 // per_copy)))
    gen = torch.Generator(device=dev).manual_seed(0)
    T = [tuple(torch.randn(m, h, device=dev, generator=gen).to(dt) for _ in range(4)) for _ in range(k)]
    w = torch.ones(h, device=dev, dtype=dt, requires_grad=True)
    b = torch.zeros(h, device=dev, dtype=dt, requires_grad=True)
    leaves = [(y.requires_grad_(True), r.requires_grad_(True)) for y, r, _, _ in T]

    def fused(y, r):
        return dropout_add_layer_norm(y, r, w, b, p, 1e-5, True, return_sum=True)

    def stock(y, r):
        z = r + F.dropout(y, p, True)
        return F.layer_norm(z, (h,), w, b, 1e-5), z

    print("%-10s %-6s %-8s %9s" % ("M x H", "path", "pass", "us"))
    res = {}
    for path, f in (("fused", fused), ("stock", stock)):
        def fwd(i, f=f):
            f(*leaves[i])

        def both(i, f=f):
            y, r = leaves[i]
            torch.autograd.grad(f(y, r), [y, r, w, b], [T[i][2], T[i][3]])

        res[path] = (graphed_us(args, torch, fwd, k), graphed_us(args, torch, both, k))
        for kind, us in zip(("fwd", "fwd+bwd"), res[path]):
            rows.append(dict(junction=[m, h], p=p, path=path, kind=kind, us=us))
            print("%-10s %-6s %-8s %9.1f" % ("%dx%d" % (m, h), path, kind, us))
    print("           stock / fused: fwd %.2fx, fwd+bwd %.2fx" % (res["stock"][0] / res["fused"][0],
                                                                  res["stock"][1] / res["fused"][1]))
    del T, leaves


ARMS = {"stock": {}, "fused_attn_loss": dict(fused_attention=True, fused_loss=True),
        "fused_attn_loss_norm": dict(fused_attention=True, fused_loss=True, fused_norm=True),
        "fused_attn_loss_fp8": dict(fused_attention=True, fused_loss=True, fp8_linear=True),
        "fused_attn_loss_fp8_norm": dict(fused_attention=True, fused_loss=True, fp8_linear=True, fused_norm=True)}


def whole_step(args, torch, rows, batch, seq):
    import byteps_b200.torch as bps
    from byteps_b200.models import gpt2_small
    from byteps_b200.torch.graph import GraphedStep

    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(1234)
    ids = torch.randint(0, 50257, (batch, seq), generator=gen).to(dev)
    graphs = {}
    for name, flags in ARMS.items():
        torch.manual_seed(0)
        model = gpt2_small(**flags).to(dev).to(torch.bfloat16).train()
        opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01),
                                       named_parameters=model.named_parameters(), fused_update=True)

        def step(model=model, opt=opt):
            opt.zero_grad()
            loss = model(ids, ids)
            loss.backward()
            opt.step()
            return loss

        graphs[name] = GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams, device=dev)
        graphs[name]()
        torch.cuda.synchronize()

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

    ms = {name: [] for name in ARMS}
    for _ in range(args.rounds):
        for name in ARMS:
            ms[name].append(timed(graphs[name]))
    info = gpu_info()
    base = statistics.median(ms["stock"])
    for name in ARMS:
        med = statistics.median(ms[name])
        spread = max(ms[name]) - min(ms[name])
        rows.append(dict(step=name, batch=batch, seq=seq, ms=ms[name], median_ms=med, spread_ms=spread))
        print("gpt2_small step %dx%d %-20s ms over %d rounds: %s  (median %.2f, spread %.2f, %.3fx stock)" % (
            batch, seq, name, args.rounds, " ".join("%.2f" % v for v in ms[name]), med, spread, base / med))
    print("GPU after the step rounds: %s" % info)
    del graphs
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="calls captured in one timed graph")
    ap.add_argument("--reps", type=int, default=10, help="replays of that graph")
    ap.add_argument("--rotate-mb", type=float, default=200.0, help="bytes the input copies of a shape span together")
    ap.add_argument("--steps", type=int, default=20, help="timed replays of a whole step per round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-step", action="store_true", help="per-call table only")
    ap.add_argument("--no-call", action="store_true", help="no per-call attention table")
    ap.add_argument("--no-junction", action="store_true", help="no per-junction LayerNorm table")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()

    import torch

    from byteps_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("gpt_bench.py needs a GPU")
    _native.cuda()
    torch.cuda.set_device(0)
    info = gpu_info()
    print("GPU: %s; bf16, D = %d" % (info, D))
    rows = []
    if not args.no_call:
        per_call(args, torch, rows)
    if not args.no_junction:
        per_junction(args, torch, rows)
    if not args.no_step:
        import byteps_b200.torch as bps

        bps.init()
        whole_step(args, torch, rows, 16, 512)
        bps.shutdown()
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
