#!/usr/bin/env python
"""Fused dropout + residual add + LayerNorm (ops/ln.py, kernels/ln.cu) against the stock torch sequence of the BERT
encoder's junctions: ``layer_norm(residual + dropout(y, p))``.

Per pass: 8192 x 768 (BERT-base) and 8192 x 1024 (BERT-large) rows of bf16 activations with bf16 gamma / beta (the
models are cast to bf16 whole), batch 64 x sequence 128 tokens, p = 0.1, with and without the residual.  Each
timed pass runs through the public function (or the stock F.dropout / add / F.layer_norm) on the next of enough
copies of its tensors that a row's copies span more than --rotate-mb together, so no pass finds its inputs in the
50 MB L2; the launches of --iters passes are captured in one CUDA graph and the graph's replays are timed with CUDA
events, so host overhead does not enter.  bwd is fwd + backward minus fwd.  Bytes are the least each path moves,
computed from the shape (e = element bytes, N = elements, rows' mean and rstd 8 M):

    fused fwd    read y [, residual]; write z, out, 1-bit mask            N e (3 [+1]) + N / 8 + 8 M
    fused bwd    read dout, z, mask; write dy [, dres]                    N e (3 [+1]) + N / 8 + 8 M
    stock fwd    dropout: read y, write y' and a byte mask; [add: read y', residual, write z];
                 layer_norm: read z, write out                            N e (4 [+3]) + N + 8 M
    stock bwd    layer_norm backward: read dout, z, write dz; its gamma / beta reduction: read dout, z;
                 dropout backward: read dz, mask, write dy                 7 N e + N + 8 M

Share of peak is against the H100 SXM data-sheet 3.35 TB/s.

Whole step: BERT-large bf16, batch 64, sequence 128, AdamW through DistributedOptimizer(fused_update=True), the
whole step captured in one CUDA graph as bench.py builds it.  The stock and fused_norm=True steps share one model
and optimizer (the fused norms hold the stock norms' Parameters); each is captured once and the two graphs are
timed alternately, --rounds rounds of --steps replays each.  The GPU name, power limit and SM clock are read in the
same run.

    python benchmarks/ln_bench.py [--iters 40] [--rotate-mb 200] [--steps 20] [--rounds 3] [--no-step] [--json f]
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
SHAPES = [(8192, 768), (8192, 1024)]
P = 0.1


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def pass_bytes(path, kind, m, h, e, res):
    n = m * h
    if path == "fused":
        return n * e * (4 if res else 3) + n // 8 + 8 * m
    if kind == "fwd":
        return n * e * (7 if res else 4) + n + 8 * m
    return 7 * n * e + n + 8 * m


def per_pass(args, torch, F, rows):
    from byteps_b200.ops.ln import dropout_add_layer_norm

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

    print("%-11s %-8s %-6s %-4s %9s %9s %8s %6s" % ("M x H", "residual", "path", "pass", "MB", "us", "GB/s", "%peak"))
    for (m, h) in SHAPES:
        for res in (False, True):
            per_copy = m * h * e * (6 if res else 4)
            k = max(2, int(-(-args.rotate_mb * 1e6 // per_copy)))
            gen = torch.Generator(device=dev).manual_seed(0)
            T = []
            for _ in range(k):
                y = torch.randn(m, h, device=dev, generator=gen).to(dt).requires_grad_(True)
                r = torch.randn(m, h, device=dev, generator=gen).to(dt).requires_grad_(True) if res else None
                T.append((y, r, torch.randn(m, h, device=dev, generator=gen).to(dt)))
            w = torch.ones(h, device=dev, dtype=dt, requires_grad=True)
            bias = torch.zeros(h, device=dev, dtype=dt, requires_grad=True)
            fns = {
                "fused": lambda y, r: dropout_add_layer_norm(y, r, w, bias, P, 1e-12, True),
                "stock": lambda y, r: F.layer_norm((r + F.dropout(y, P, True)) if r is not None
                                                   else F.dropout(y, P, True), (h,), w, bias, 1e-12),
            }
            for path, f in fns.items():
                def fwd(i, f=f):
                    y, r, _ = T[i]
                    f(y, r)

                def both(i, f=f):
                    y, r, dout = T[i]
                    inputs = [y, w, bias] + ([r] if r is not None else [])
                    torch.autograd.grad(f(y, r), inputs, dout)

                us_f = graphed_us(fwd, k)
                us_b = graphed_us(both, k) - us_f
                for kind, us in (("fwd", us_f), ("bwd", us_b)):
                    nbytes = pass_bytes(path, kind, m, h, e, res)
                    gbs = nbytes / (us * 1e3)
                    rows.append(dict(shape=[m, h], residual=res, path=path, kind=kind, bytes=nbytes, us=us, gbs=gbs,
                                     peak_share=gbs / PEAK_GBS))
                    print("%-11s %-8s %-6s %-4s %9.1f %9.1f %8.0f %5.0f%%" % (
                        "%dx%d" % (m, h), "yes" if res else "no", path, kind, nbytes / 1e6, us, gbs,
                        100 * gbs / PEAK_GBS))
            del T


def whole_step(args, torch, rows):
    import byteps_b200.torch as bps
    from byteps_b200.models import bert_large
    from byteps_b200.ops.ln import DropoutAddLayerNorm
    from byteps_b200.torch.graph import GraphedStep

    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = True
    bps.init()
    torch.manual_seed(0)
    model = bert_large().to(dev).to(torch.bfloat16).train()
    opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01),
                                   named_parameters=model.named_parameters(), fused_update=True)
    gen = torch.Generator().manual_seed(1234)
    ids = torch.randint(0, 30522, (args.batch, args.seq), generator=gen).to(dev)
    labels = torch.randint(0, 30522, (args.batch, args.seq), generator=gen).to(dev)

    stock_norms = [(layer.norm1, layer.norm2) for layer in model.layers]

    def fused_twin(ln, p):
        f = DropoutAddLayerNorm(ln.normalized_shape, eps=ln.eps, p=p, device="meta")
        f.weight, f.bias = ln.weight, ln.bias      # the same Parameters: one optimizer serves both variants
        return f

    fused_norms = [(fused_twin(a, layer.p), fused_twin(b, layer.p)) for layer, (a, b) in zip(model.layers, stock_norms)]

    def use(fused):
        for layer, norms in zip(model.layers, fused_norms if fused else stock_norms):
            layer.norm1, layer.norm2 = norms
            layer.fused_norm = fused

    def step():
        opt.zero_grad()
        loss = model(ids, mlm_labels=labels)
        loss.backward()
        opt.step()
        return loss

    graphs = {}
    for fused in (False, True):
        use(fused)
        graphs[fused] = GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams, device=dev)
    use(False)

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
        name = "fused_norm" if fused else "stock"
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
    ap.add_argument("--iters", type=int, default=40, help="passes captured in one timed graph")
    ap.add_argument("--reps", type=int, default=10, help="replays of that graph")
    ap.add_argument("--rotate-mb", type=float, default=200.0, help="bytes the tensor copies of a row span together")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20, help="timed replays of a whole step per round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-step", action="store_true", help="per-pass table only")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F

    from byteps_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("ln_bench.py needs a GPU")
    _native.cuda()
    torch.cuda.set_device(0)
    info = gpu_info()
    print("GPU: %s; bf16 activations and parameters, p = %g" % (info, P))
    rows = []
    per_pass(args, torch, F, rows)
    if not args.no_step:
        whole_step(args, torch, rows)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
