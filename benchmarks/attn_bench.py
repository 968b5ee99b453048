#!/usr/bin/env python
"""Fused self-attention (ops/attn.py, kernels/attn.cu) against the stock expression of the BERT encoder:
``qkv.view(b, s, 3, h, d).permute(...)``, ``F.scaled_dot_product_attention`` and ``transpose(1, 2).reshape(...)``,
with their backward.

Per call, at BERT-large's heads (H = 16, D = 64) in bf16, at (B, S) = (64, 128) (phase 1), (8, 512) (phase 2) and
(32, 200) (partial tiles), with p = 0.1 and p = 0, each without a mask and with a bool key-padding mask [B, 1, 1, S]
(random lengths).  Each timed call runs on the next of enough copies of qkv and dout that they span more than
--rotate-mb together, so no call finds its inputs in the 50 MB L2; --iters calls are captured in one CUDA graph and
its replays are timed with CUDA events.  fwd+bwd is one forward and its backward (torch.autograd.grad to qkv).  The
least bytes and FLOPs come from the shapes (e = 2 bytes, N = B S E elements, E = H D):

    fwd      read qkv, write the context and an fp32 log-sum-exp:      4 N e + 4 B H S bytes,   4 B H S^2 D FLOPs
    bwd      read qkv, context, dout, log-sum-exp; write d(qkv):       8 N e + 4 B H S bytes,   8 B H S^2 D FLOPs

Share of peak is the least time the H100 SXM data sheet allows (the larger of bytes / 3.35 TB/s and FLOPs / 989
TFLOP/s dense bf16; the bound names which) over the measured time.  The SDPA backend of the stock arm is read from the
kernel names of one profiled fwd+bwd per configuration.

Whole step: BERT-large bf16 with fp8_linear, fused_norm and fused_loss, fused AdamW through
DistributedOptimizer(fused_update=True), the whole step in one CUDA graph, at batch 64 x 128 and 16 x 512, no mask
(as examples/pytorch/train_bert_byteps.py trains).  fused_attention off and on are two captures of one model,
timed alternately over --rounds rounds of --steps replays; medians, spreads and the memory each capture adds at its
peak.  The GPU name, power limit and SM clock are read in the same run.

    python benchmarks/attn_bench.py [--iters 20] [--rotate-mb 200] [--steps 20] [--rounds 5] [--no-step] [--json f]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0
PEAK_TFLOPS = 989.0
H, D = 16, 64
SHAPES = [(64, 128), (8, 512), (32, 200)]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def least(kind, b, s):
    """(bytes, FLOPs) the computation needs at least"""
    n, stats = b * s * H * D, 4 * b * H * s
    flops = 4 * b * H * s * s * D
    if kind == "fwd":
        return 4 * n * 2 + stats, flops
    if kind == "bwd":
        return 8 * n * 2 + stats, 2 * flops
    return 12 * n * 2 + 2 * stats, 3 * flops


def least_us(nbytes, flops):
    tb, tf = nbytes / (PEAK_GBS * 1e3), flops / (PEAK_TFLOPS * 1e6)
    return (tb, "bytes") if tb >= tf else (tf, "flops")


def sdpa_backend(torch, fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(0)
        torch.cuda.synchronize()
    names = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA":
            names[ev.name] = names.get(ev.name, 0) + ev.device_time
    keys = [k for k in names if any(t in k.lower() for t in ("flash", "fmha", "efficient", "attention", "softmax"))]
    keys.sort(key=lambda k: -names[k])
    return "; ".join(k[:90] for k in keys[:2]) or "unknown"


def per_call(args, torch, rows):
    from byteps_b200.ops.attn import _stock, self_attention

    dev = torch.device("cuda", 0)
    dt = torch.bfloat16

    def graphed_us(fn, k):
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

    print("%-8s %-4s %-5s %-6s %-8s %9s %9s %8s %6s  %s" % (
        "B x S", "p", "mask", "path", "pass", "MB", "us", "least", "%peak", "bound"))
    for (b, s) in SHAPES:
        e = H * D
        per_copy = b * s * e * 2 * 4
        k = max(2, int(-(-args.rotate_mb * 1e6 // per_copy)))
        gen = torch.Generator(device=dev).manual_seed(0)
        T = [((torch.randn(b, s, 3 * e, device=dev, generator=gen) * 1.5).to(dt).requires_grad_(True),
              torch.randn(b, s, e, device=dev, generator=gen).to(dt)) for _ in range(k)]
        lengths = torch.randint(s // 2, s + 1, (b,), generator=torch.Generator().manual_seed(1))
        pad = (torch.arange(s)[None, :] < lengths[:, None]).view(b, 1, 1, s).to(dev)
        for p in (0.1, 0.0):
            for mask in (None, pad):
                fns = {"fused": lambda x, m=mask, p=p: self_attention(x, H, m, p, True),
                       "stock": lambda x, m=mask, p=p: _stock(x, H, m, p)}
                res = {}
                for path, f in fns.items():
                    def fwd(i, f=f):
                        f(T[i][0])

                    def both(i, f=f):
                        x, dout = T[i]
                        torch.autograd.grad(f(x), [x], dout)

                    us_f = graphed_us(fwd, k)
                    us_fb = graphed_us(both, k)
                    res[path] = (us_f, us_fb)
                    backend = sdpa_backend(torch, both) if path == "stock" else "attn_fwd / attn_bwd_dq / attn_bwd_dkv"
                    for kind, us in (("fwd", us_f), ("fwd+bwd", us_fb)):
                        nbytes, flops = least(kind if kind == "fwd" else "both", b, s)
                        t_min, bound = least_us(nbytes, flops)
                        rows.append(dict(shape=[b, s], heads=H, p=p, mask=mask is not None, path=path, kind=kind,
                                         us=us, least_bytes=nbytes, least_flops=flops, least_us=t_min, bound=bound,
                                         peak_share=t_min / us, backend=backend))
                        print("%-8s %-4g %-5s %-6s %-8s %9.1f %9.1f %8.1f %5.0f%%  %s" % (
                            "%dx%d" % (b, s), p, "pad" if mask is not None else "none", path, kind, nbytes / 1e6,
                            us, t_min, 100 * t_min / us, bound))
                    if path == "stock":
                        print("         stock SDPA kernels: %s" % backend)
                print("         fused / stock: fwd %.2fx, fwd+bwd %.2fx" % (
                    res["stock"][0] / res["fused"][0], res["stock"][1] / res["fused"][1]))
        del T


def whole_step(args, torch, rows, batch, seq):
    import byteps_b200.torch as bps
    from byteps_b200.models import bert_large
    from byteps_b200.torch.graph import GraphedStep

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = bert_large(fp8_linear=True, fused_norm=True, fused_loss=True).to(dev).to(torch.bfloat16).train()
    opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01),
                                   named_parameters=model.named_parameters(), fused_update=True)
    gen = torch.Generator().manual_seed(1234)
    ids = torch.randint(0, 30522, (batch, seq), generator=gen).to(dev)
    labels = torch.randint(0, 30522, (batch, seq), generator=gen).to(dev)

    def use(fused):
        for layer in model.layers:
            layer.fused_attention = fused

    def step():
        opt.zero_grad()
        loss = model(ids, mlm_labels=labels)
        loss.backward()
        opt.step()
        return loss

    graphs, extra_mb = {}, {}
    for fused in (False, True):
        use(fused)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        graphs[fused] = GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams, device=dev)
        graphs[fused]()
        torch.cuda.synchronize()
        extra_mb[fused] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
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
        name = "fused_attention" if fused else "stock_attention"
        med = statistics.median(ms[fused])
        spread = max(ms[fused]) - min(ms[fused])
        rows.append(dict(step=name, batch=batch, seq=seq, ms=ms[fused], median_ms=med, spread_ms=spread,
                         peak_extra_mb=extra_mb[fused]))
        print("BERT-large FP8 step %dx%d %-16s ms over %d rounds: %s  (median %.2f, spread %.2f, peak +%.0f MB)" % (
            batch, seq, name, args.rounds, " ".join("%.2f" % v for v in ms[fused]), med, spread, extra_mb[fused]))
    print("GPU after the step rounds: %s" % info)
    del graphs, opt, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="calls captured in one timed graph")
    ap.add_argument("--reps", type=int, default=10, help="replays of that graph")
    ap.add_argument("--rotate-mb", type=float, default=200.0, help="bytes the input copies of a shape span together")
    ap.add_argument("--steps", type=int, default=20, help="timed replays of a whole step per round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-step", action="store_true", help="per-call table only")
    ap.add_argument("--no-call", action="store_true", help="whole steps only")
    ap.add_argument("--step-shapes", default="64x128,16x512", help="batch x sequence of the whole steps")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()

    import torch

    from byteps_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("attn_bench.py needs a GPU")
    _native.cuda()
    torch.cuda.set_device(0)
    info = gpu_info()
    print("GPU: %s; bf16, H = %d, D = %d" % (info, H, D))
    rows = []
    if not args.no_call:
        per_call(args, torch, rows)
    if not args.no_step:
        import byteps_b200.torch as bps

        bps.init()
        for shape in args.step_shapes.split(","):
            batch, seq = map(int, shape.split("x"))
            whole_step(args, torch, rows, batch, seq)
        bps.shutdown()
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
