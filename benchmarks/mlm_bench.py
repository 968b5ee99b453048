#!/usr/bin/env python
"""BERT's masked-LM head on the labelled positions only (max_predictions_per_seq, kernels/mlm_gather.cu) against the
dense head that runs on every token.

Labels mark 15 % of the real tokens, drawn from a seeded generator (the rest -100); token ids are random.  Nothing is
downloaded.  Sequence lengths and packing follow packed_bench.py.

Per call: the gather (fwd) and the scatter (bwd) at T = 8192 and 65536 tokens, H = 1024, bf16, C = ceil(0.15 T),
against the stock expression (ops.mlm._stock), fwd and fwd + bwd each captured in a CUDA graph of --iters calls (bwd =
their difference)
(timed eagerly, and marked so, where the stock expression does not capture).  The least bytes are
what the op must move: fwd reads T labels (8 B) and C rows and writes C rows, C labels and T slots (4 B); bwd reads T
slots and C rows and writes T rows.  Share = least bytes / time over 3.35 TB/s.

Head per call: mlm_dense -> GELU -> mlm_norm -> tied decoder -> fused loss, forward + backward, on BERT-large's head
(H = 1024, V = 30522) at 64 x 128: dense over 8192 rows, sparse over the gathered 64 k rows (k = 20).

Whole step: BERT-large bf16 with fp8_linear, fused_norm, fused_loss and fused_attention, fused AdamW, one CUDA graph
per step.  Rows (B x S, layout, k): 64 x 128 padded (k = 20), 64 x 128 packed (k = 20), 16 x 512 packed (k = 80); k is
raised where a prepared batch would drop a target, so that no timed batch drops one (the dropped count is checked).
Dense and sparse arms of a row are timed alternately over --rounds rounds of --steps replays; the table gives ms per
step (median and spread), real tokens per second and each arm's peak memory over what was allocated before its
warm-up and capture, and the GPU's name, power limit and SM clock, read in the same run.

    python benchmarks/mlm_bench.py [--steps 20] [--rounds 5] [--batches 4] [--iters 20] [--rows 0,1] [--json f]

The memory the earlier rows' graphs keep leaves too little for the 16 x 512 row in the same process on an 80 GB card:
run it on its own with --no-call --rows 2.
"""
import argparse
import json
import math
import os
import statistics
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from attn_bench import gpu_info   # noqa: E402
from packed_bench import make_inputs, packed_batches, padded_batches   # noqa: E402

HBM = 3.35e12
STEP_ROWS = [(64, 128, False, 20), (64, 128, True, 20), (16, 512, True, 80)]


def graphed_us(torch, fn, iters, reps):
    """us per call of fn, from a CUDA graph of `iters` calls replayed `reps` times; ("eager", us) over iters * reps
    eager calls when fn does not capture (as happens to the stock expression)"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    try:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(iters):
                fn()
    except RuntimeError:
        torch.cuda.synchronize()
        e0.record()
        for _ in range(iters * reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return "eager", e0.elapsed_time(e1) * 1e3 / (reps * iters)
    g.replay()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return "graph", e0.elapsed_time(e1) * 1e3 / (reps * iters)


def per_call(args, torch, rows):
    from byteps_b200.ops.mlm import _stock, gather_labelled

    dev = torch.device("cuda", 0)
    h = 1024
    for t in (8192, 65536):
        c = math.ceil(0.15 * t)
        gen = torch.Generator(device=dev).manual_seed(t)
        x = torch.randn(t, h, device=dev, generator=gen).to(torch.bfloat16).requires_grad_(True)
        lab = torch.where(torch.rand(t, device=dev, generator=gen) < 0.15, 7, -100)
        n = int((lab != -100).sum())
        c = max(c, n)
        drows = torch.randn(c, h, device=dev, generator=gen).to(torch.bfloat16)
        fwd_bytes = t * 8 + 2 * c * h * 2 + c * 8 + t * 4
        bwd_bytes = t * 4 + c * h * 2 + t * h * 2
        res = {}
        for name, fn in (("kernel", lambda: gather_labelled(x, lab, c)), ("stock", lambda: _stock(x, lab, c, -100))):
            mode_f, us_f = graphed_us(torch, fn, args.iters, args.reps)
            mode_fb, us_fb = graphed_us(torch, lambda fn=fn: torch.autograd.grad(fn()[0], [x], drows), args.iters,
                                        args.reps)
            us_b = us_fb - us_f
            res[name] = (us_f, us_b, mode_f, mode_fb)
            rows.append(dict(call=name, T=t, H=h, C=c, fwd_us=us_f, fwd_bwd_us=us_fb, bwd_us=us_b, fwd_mode=mode_f,
                             fwd_bwd_mode=mode_fb, fwd_hbm_share=fwd_bytes / (us_f * 1e-6) / HBM,
                             bwd_hbm_share=bwd_bytes / (us_b * 1e-6) / HBM))
        for name, (us_f, us_b, mode_f, mode_fb) in res.items():
            print("gather T=%-6d C=%-5d %-6s fwd %7.1f us %-5s (%4.1f %% of HBM)  bwd %7.1f us %-5s (%4.1f %% of HBM)"
                  "   stock / this: fwd %.2fx bwd %.2fx" % (
                      t, c, name, us_f, mode_f, 100 * fwd_bytes / (us_f * 1e-6) / HBM, us_b, mode_fb,
                      100 * bwd_bytes / (us_b * 1e-6) / HBM, res["stock"][0] / us_f, res["stock"][1] / us_b))


def head_call(args, torch, rows):
    import torch.nn.functional as F

    from byteps_b200.models import bert_large
    from byteps_b200.ops.mlm import gather_labelled
    from byteps_b200.ops.xent import softmax_cross_entropy

    dev = torch.device("cuda", 0)
    b, s, k = 64, 128, 20
    torch.manual_seed(0)
    m = bert_large(num_layers=1).to(dev).to(torch.bfloat16)
    gen = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(b, s, 1024, device=dev, generator=gen).to(torch.bfloat16).requires_grad_(True)
    lab = torch.where(torch.rand(b, s, device=dev, generator=gen) < 0.15,
                      torch.randint(0, 30522, (b, s), device=dev, generator=gen), -100)
    params = [x, m.mlm_dense.weight, m.mlm_dense.bias, m.mlm_norm.weight, m.mlm_norm.bias, m.embeddings.word.weight,
              m.mlm_bias]

    def head(sparse):
        hx, hl = (gather_labelled(x, lab, b * k)[:2]) if sparse else (x, lab)
        hh = m.mlm_norm(F.gelu(m.mlm_dense(hx)))
        logits = F.linear(hh, m.embeddings.word.weight, m.mlm_bias)
        loss = softmax_cross_entropy(logits.view(-1, logits.shape[-1]), hl.reshape(-1))
        return torch.autograd.grad(loss, params)

    res = {}
    for name in ("dense", "sparse"):
        mode, us = graphed_us(torch, lambda name=name: head(name == "sparse"), args.iters, args.reps)
        res[name] = us
        rows.append(dict(head=name, batch=b, seq=s, k=k, fwd_bwd_us=us, mode=mode))
        print("MLM head fwd+bwd 64x128 %-6s: %8.1f us (%s)  dense / this %.2fx" % (name, us, mode, res["dense"] / us))
    del m


def needed_k(batches, b):
    return max(int((x["labels"] != -100).sum()) for x in batches) / b


def whole_step(args, torch, rows, b, s, packed, k0):
    import byteps_b200.torch as bps
    from byteps_b200.models import bert_large
    from byteps_b200.torch.graph import GraphedStep

    dev = torch.device("cuda", 0)
    torch.cuda.empty_cache()   # the blocks cached by earlier rows would not fit beside a new model and its graphs
    cap = b * s // (s // 16) + 1
    rng = np.random.RandomState(2024)
    lens = (packed_batches if packed else padded_batches)(rng, b, s, args.batches)
    gen = torch.Generator().manual_seed(1234)
    host = [make_inputs(torch, ln, b, s, packed, cap, gen) for ln in lens]
    k = max(k0, math.ceil(needed_k(host, b)))
    torch.manual_seed(0)
    model = bert_large(fp8_linear=True, fused_norm=True, fused_loss=True, fused_attention=True)
    model = model.to(dev).to(torch.bfloat16).train()
    opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01),
                                   named_parameters=model.named_parameters(), fused_update=True)
    dev_in = [{kk: (v.to(dev) if torch.is_tensor(v) else v) for kk, v in x.items()} for x in host]
    arms = {}
    for sparse in (False, True):
        model.config.max_predictions_per_seq = k if sparse else 0   # read when each arm's step is captured
        static = {kk: v.clone() for kk, v in dev_in[0].items() if torch.is_tensor(v)}

        def step(static=static):
            opt.zero_grad()
            if packed:
                loss = model(static["ids"], cu_seqlens=static["extra"], max_seqlen=s, mlm_labels=static["labels"])
            else:
                loss = model(static["ids"], mask=static["extra"], mlm_labels=static["labels"])
            loss.backward()
            opt.step()
            return loss

        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        graph = GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams, device=dev)
        for i in range(4):
            for kk in static:
                static[kk].copy_(dev_in[i % len(dev_in)][kk])
            graph()
        torch.cuda.synchronize()
        arms[sparse] = dict(graph=graph, static=static, batches=dev_in, real=[x["real"] for x in host],
                            peak=torch.cuda.max_memory_allocated() - base)

    def timed(arm):
        g, st, bs = arm["graph"], arm["static"], arm["batches"]
        model.mlm_dropped_targets.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            for kk in st:
                st[kk].copy_(bs[i % len(bs)][kk], non_blocking=True)
            loss = g()
        e1.record()
        torch.cuda.synchronize()
        assert torch.isfinite(loss).item()
        assert int(model.mlm_dropped_targets) == 0, "a timed batch dropped a target"
        real = sum(arm["real"][i % len(bs)] for i in range(args.steps))
        return e0.elapsed_time(e1) / args.steps, real / args.steps

    ms = {False: [], True: []}
    real = {}
    for _ in range(args.rounds):
        for sparse in (False, True):
            t, r = timed(arms[sparse])
            ms[sparse].append(t)
            real[sparse] = r
    layout = "packed" if packed else "padded"
    for sparse in (False, True):
        name = "sparse k=%d" % k if sparse else "dense"
        med, spread = statistics.median(ms[sparse]), max(ms[sparse]) - min(ms[sparse])
        tps = real[sparse] / (med / 1e3)
        rows.append(dict(step=layout, head=name, batch=b, seq=s, k=k if sparse else 0, ms=ms[sparse], median_ms=med,
                         spread_ms=spread, real_tokens_per_s=tps, peak_gb=arms[sparse]["peak"] / 1e9))
        print("BERT-large step %dx%d %s %-12s: %6.2f ms (spread %.2f over %d rounds: %s), %8.0f real tokens/s, "
              "peak %.2f GB" % (b, s, layout, name, med, spread, args.rounds, " ".join("%.2f" % v for v in ms[sparse]),
                                tps, arms[sparse]["peak"] / 1e9))
    print("GPU after the step rounds: %s" % gpu_info())
    del arms, opt, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed replays of a whole step per round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batches", type=int, default=4, help="prepared batches each arm replays in turn")
    ap.add_argument("--iters", type=int, default=20, help="calls captured in one timed per-call graph")
    ap.add_argument("--reps", type=int, default=10, help="replays of that graph")
    ap.add_argument("--no-step", action="store_true", help="per-call tables only")
    ap.add_argument("--rows", default=None, help="comma-separated indices into the whole-step rows (default all)")
    ap.add_argument("--no-call", action="store_true", help="whole steps only")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()

    import torch

    from byteps_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("mlm_bench.py needs a GPU")
    _native.cuda()
    torch.cuda.set_device(0)
    info = gpu_info()
    print("GPU: %s; bf16" % info)
    rows = []
    if not args.no_call:
        per_call(args, torch, rows)
        head_call(args, torch, rows)
    if not args.no_step:
        import byteps_b200.torch as bps

        bps.init()
        pick = range(len(STEP_ROWS)) if args.rows is None else [int(i) for i in args.rows.split(",")]
        for b, s, packed, k in (STEP_ROWS[i] for i in pick):
            whole_step(args, torch, rows, b, s, packed, k)
        bps.shutdown()
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
