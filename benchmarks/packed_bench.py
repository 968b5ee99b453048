#!/usr/bin/env python
"""Packed variable-length BERT pre-training (cu_seqlens, kernels/attn_varlen.cu) against padded batches.

Sequence lengths are drawn from a seeded NumPy generator, uniform over the integers [S / 16, S] for a padded row
length S (so [32, 512] at S = 512, mean 272, and [8, 128] at S = 128); token ids and MLM labels (15 % of the real
tokens, the rest -100) are random.  Nothing is downloaded.

Whole step: BERT-large bf16 with fp8_linear, fused_norm, fused_loss and fused_attention, fused AdamW through
DistributedOptimizer(fused_update=True), one CUDA graph per step, at B x S = 16 x 512 and 64 x 128.
    padded  one sequence per row, a bool key-padding mask [B, 1, 1, S]
    packed  the same sequence stream, packed greedily in draw order into B S tokens (a sequence that does not fit
            starts the next step); cu_seqlens has a fixed capacity of B S / min_len + 1 slots, padded by repeating
            its last value, max_seqlen = S
Each arm captures once and replays over --batches prepared batches, copied into its static inputs before each
replay.  The two arms are timed alternately over --rounds rounds of --steps replays (CUDA events); the table gives
real (non-padding) tokens per second, ms per step, the median and spread over the rounds, and the GPU's name, power
limit and SM clock read in the same run.

Per call: self-attention at BERT-large's heads (H = 16, D = 64) in bf16 on one padded batch's B sequences, p = 0 and
0.1, fwd and fwd+bwd captured in CUDA graphs: the packed kernels on the sequences concatenated (T = sum of lengths),
the padded fused kernel with the bool mask, and stock SDPA with the same mask.  All three hold the same real tokens.

    python benchmarks/packed_bench.py [--steps 20] [--rounds 5] [--batches 4] [--iters 20] [--json f]
"""
import argparse
import json
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

H = 16
SHAPES = [(16, 512), (64, 128)]


def draw_lengths(rng, s, n):
    return rng.randint(s // 16, s + 1, size=n)


def padded_batches(rng, b, s, count):
    return [draw_lengths(rng, s, b) for _ in range(count)]


def packed_batches(rng, b, s, count):
    """greedy packing of the drawn stream into b * s tokens per step, in draw order"""
    t, out, cur, pending = b * s, [], [], None
    while len(out) < count:
        n = pending if pending is not None else int(draw_lengths(rng, s, 1)[0])
        pending = None
        if sum(cur) + n > t:
            out.append(cur)
            cur, pending = [], n
        else:
            cur.append(n)
    return out


def make_inputs(torch, lengths, b, s, packed, cap, gen):
    t = b * s
    ids = torch.randint(0, 30522, (t,), generator=gen)
    labels = torch.where(torch.rand(t, generator=gen) < 0.15, torch.randint(0, 30522, (t,), generator=gen),
                         torch.full((t,), -100))
    if packed:
        cu = np.concatenate([[0], np.cumsum(lengths)])
        real = int(cu[-1])
        cu = np.concatenate([cu, np.full(cap + 1 - len(cu), cu[-1])])
        labels[real:] = -100
        extra = torch.tensor(cu, dtype=torch.int32)
    else:
        attend = torch.arange(s)[None, :] < torch.tensor(lengths)[:, None]
        labels = torch.where(attend.reshape(-1), labels, torch.full_like(labels, -100))
        real = int(attend.sum())
        extra = attend.view(b, 1, 1, s)
    return dict(ids=ids.view(b, s), labels=labels.view(b, s), extra=extra, real=real)


def whole_step(args, torch, rows, b, s):
    import byteps_b200.torch as bps
    from byteps_b200.models import bert_large
    from byteps_b200.torch.graph import GraphedStep

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = bert_large(fp8_linear=True, fused_norm=True, fused_loss=True, fused_attention=True)
    model = model.to(dev).to(torch.bfloat16).train()
    opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01),
                                   named_parameters=model.named_parameters(), fused_update=True)
    cap = b * s // (s // 16) + 1
    gen = torch.Generator().manual_seed(1234)
    arms = {}
    for packed in (False, True):
        rng = np.random.RandomState(2024)   # both arms draw from the same sequence stream
        lens = (packed_batches if packed else padded_batches)(rng, b, s, args.batches)
        host = [make_inputs(torch, ln, b, s, packed, cap, gen) for ln in lens]
        dev_in = [{k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in x.items()} for x in host]
        static = {k: v.clone() for k, v in dev_in[0].items() if torch.is_tensor(v)}

        def step(static=static, packed=packed):
            opt.zero_grad()
            if packed:
                loss = model(static["ids"], cu_seqlens=static["extra"], max_seqlen=s, mlm_labels=static["labels"])
            else:
                loss = model(static["ids"], mask=static["extra"], mlm_labels=static["labels"])
            loss.backward()
            opt.step()
            return loss

        graph = GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams, device=dev)
        arms[packed] = dict(graph=graph, static=static, batches=dev_in, real=[x["real"] for x in host],
                            seqs=[len(ln) for ln in lens])

    def timed(arm):
        g, st, bs = arm["graph"], arm["static"], arm["batches"]

        def one(i):
            for k in st:
                st[k].copy_(bs[i % len(bs)][k], non_blocking=True)
            return g()

        for i in range(3):
            one(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            loss = one(i)
        e1.record()
        torch.cuda.synchronize()
        assert torch.isfinite(loss).item()
        real = sum(arm["real"][i % len(bs)] for i in range(args.steps))
        ms = e0.elapsed_time(e1) / args.steps
        return ms, real / args.steps

    ms = {False: [], True: []}
    real = {}
    for _ in range(args.rounds):
        for packed in (False, True):
            t, r = timed(arms[packed])
            ms[packed].append(t)
            real[packed] = r
    info = gpu_info()
    for packed in (False, True):
        name = "packed" if packed else "padded"
        med, spread = statistics.median(ms[packed]), max(ms[packed]) - min(ms[packed])
        tps = real[packed] / (med / 1e3)
        rows.append(dict(step=name, batch=b, seq=s, ms=ms[packed], median_ms=med, spread_ms=spread,
                         real_tokens_per_step=real[packed], real_tokens_per_s=tps,
                         sequences_per_step=statistics.mean(arms[packed]["seqs"])))
        print("BERT-large FP8 step %dx%d %-6s: %6.2f ms (spread %.2f over %d rounds: %s), %7.0f real tokens/step "
              "(%.1f sequences), %8.0f real tokens/s" % (
                  b, s, name, med, spread, args.rounds, " ".join("%.2f" % v for v in ms[packed]), real[packed],
                  statistics.mean(arms[packed]["seqs"]), tps))
    print("GPU after the step rounds: %s" % info)
    del arms, opt, model
    torch.cuda.empty_cache()


def per_call(args, torch, rows, b, s):
    from byteps_b200.ops.attn import _stock, self_attention

    dev = torch.device("cuda", 0)
    e = H * 64
    lengths = padded_batches(np.random.RandomState(7), b, s, 1)[0]
    real = int(lengths.sum())
    gen = torch.Generator(device=dev).manual_seed(0)
    qkv = (torch.randn(b, s, 3 * e, device=dev, generator=gen) * 1.5).to(torch.bfloat16)
    dout = torch.randn(b, s, e, device=dev, generator=gen).to(torch.bfloat16)
    attend = torch.arange(s, device=dev)[None, :] < torch.tensor(lengths, device=dev)[:, None]
    mask = attend.view(b, 1, 1, s)
    pq = qkv[attend].contiguous().requires_grad_(True)
    pdo = dout[attend].contiguous()
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lengths)]), dtype=torch.int32, device=dev)
    qkv.requires_grad_(True)

    def graphed_us(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(args.iters):
                fn()
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / (args.reps * args.iters)

    for p in (0.0, 0.1):
        paths = {
            "packed": (lambda p=p: self_attention(pq, H, p=p, cu_seqlens=cu, max_seqlen=s), pq, pdo),
            "padded": (lambda p=p: self_attention(qkv, H, mask, p, True), qkv, dout),
            "sdpa": (lambda p=p: _stock(qkv, H, mask, p), qkv, dout),
        }
        res = {}
        for name, (f, x, do) in paths.items():
            us_f = graphed_us(f)
            us_fb = graphed_us(lambda f=f, x=x, do=do: torch.autograd.grad(f(), [x], do))
            res[name] = (us_f, us_fb)
            rows.append(dict(call=name, batch=b, seq=s, real_tokens=real, p=p, fwd_us=us_f, fwd_bwd_us=us_fb))
        for name, (us_f, us_fb) in res.items():
            print("%dx%d (%d real tokens) p=%-3g %-6s fwd %8.1f us  fwd+bwd %8.1f us   vs packed: fwd %.2fx, "
                  "fwd+bwd %.2fx" % (b, s, real, p, name, us_f, us_fb, us_f / res["packed"][0],
                                     us_fb / res["packed"][1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed replays of a whole step per round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batches", type=int, default=4, help="prepared batches each arm replays in turn")
    ap.add_argument("--iters", type=int, default=20, help="calls captured in one timed per-call graph")
    ap.add_argument("--reps", type=int, default=10, help="replays of that graph")
    ap.add_argument("--no-step", action="store_true", help="per-call table only")
    ap.add_argument("--no-call", action="store_true", help="whole steps only")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()

    import torch

    from byteps_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("packed_bench.py needs a GPU")
    _native.cuda()
    torch.cuda.set_device(0)
    info = gpu_info()
    print("GPU: %s; bf16, H = %d, D = 64" % (info, H))
    rows = []
    if not args.no_call:
        for b, s in SHAPES:
            per_call(args, torch, rows, b, s)
    if not args.no_step:
        import byteps_b200.torch as bps

        bps.init()
        for b, s in SHAPES:
            whole_step(args, torch, rows, b, s)
        bps.shutdown()
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
