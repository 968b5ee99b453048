#!/usr/bin/env python
"""FP8 linear layers (ops/fp8.py, kernels/fp8.cu) against bf16 ``nn.Linear`` at BERT-large's encoder shapes.

Per layer: M = 8192 tokens (batch 64 x sequence 128) and (K, N) = (1024, 3072) qkv, (1024, 1024) proj,
(1024, 4096) fc1, (4096, 1024) fc2, with bias.  Rows:

    linear     nn.Linear bf16: forward, and backward (fwd + bwd minus fwd) with dx, dW and the bias gradient
    fp8        Fp8Linear: the same, every cast and GEMM included
    casts      the cast kernels alone, forward (x and W to E4M3 rows + transposed) and backward (dy to E5M2 rows +
               transposed with the bias gradient); bytes from the shape: read the bf16 tensor, write two FP8 copies
               (4 bytes per element moved), plus the bias
    gemm       the three FP8 GEMMs alone (_scaled_mm, no fast accumulation); 2 M N K FLOP forward, 4 M N K backward

Feed-forward block (fc1 -> GELU -> fc2 of BERT-large, M = 8192, K = 1024, I = 4096, with bias):

    mlp        composed fc2(F.gelu(fc1(x))) of two Fp8Linear, and fused ops.fp8.fp8_gelu_mlp: forward, and forward +
               backward with every gradient
    actcast    the fused casts alone at [M, I]: ACT_GELU z -> E4M3 rows + transposed (read z, write two FP8 copies:
               4 bytes per element) and ACT_DGELU (dh, z) -> E5M2 rows + transposed + the bias gradient (read dh
               and z, write two copies: 6 bytes per element, plus the bias)

Each timed call runs on the next of enough copies of its inputs that they span more than --rotate-mb, so no call finds
its input in the 50 MB L2; --iters calls are captured in one CUDA graph and its replays are timed with CUDA events.
Shares of peak are against the H100 SXM data sheet (3.35 TB/s; 1979 dense FP8 TFLOP/s and 989 bf16 TFLOP/s), figures
a card is not expected to reach.

Whole step: BERT-large bf16, batch 64 x 128, fused_norm=True, fused_loss=True, AdamW through
DistributedOptimizer(fused_update=True), the whole step captured in one CUDA graph.  One model and one optimizer:
the bf16 graph is captured first, then the encoder's qkv / proj / fc1 / fc2 become Fp8Linear (the same parameters, as
bert_large(fp8_linear=True) builds them) and the fp8 graph is captured; the two graphs are timed alternately,
--rounds rounds of --steps replays each.  Memory is the peak allocated while each graph is warmed up and captured,
above what was allocated before.  The GPU name, power limit and SM clock are read in the same run.  Then, the
same way, BERT-large with fp8_linear=True, fused_norm=True and fused_loss=True twice: its encoder MLPs through the
composition fc2(F.gelu(fc1(x))) and through fp8_gelu_mlp (the model as it ships), two graphs timed alternately.

    python benchmarks/fp8_bench.py [--iters 20] [--reps 5] [--rotate-mb 600] [--steps 20] [--rounds 5] [--no-step]
                                   [--only-mlp] [--json f]
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

PEAK_GBS, PEAK_FP8, PEAK_BF16 = 3350.0, 1979.0, 989.0
M = 8192
SHAPES = [("qkv", 1024, 3072), ("proj", 1024, 1024), ("fc1", 1024, 4096), ("fc2", 4096, 1024)]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def cast_bytes(kind, k, n):
    if kind == "fwd":
        return 4 * (M * k + n * k)
    return 4 * M * n + 2 * n


def _graphed_us(args, torch, fn, k):
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
    del g
    return a.elapsed_time(b) * 1e3 / (args.reps * args.iters)


def per_layer(args, torch, rows):
    import torch.nn as nn

    from byteps_b200.ops import fp8
    from byteps_b200.ops.fp8 import Fp8Linear

    dev = torch.device("cuda", 0)
    dt = torch.bfloat16

    def graphed_us(fn, k):
        return _graphed_us(args, torch, fn, k)

    def row(layer, k, n, path, kind, us, nbytes=None, flop=None):
        r = dict(layer=layer, K=k, N=n, path=path, kind=kind, us=us)
        extra = ""
        if nbytes is not None:
            r.update(bytes=nbytes, gbs=nbytes / (us * 1e3), peak_share=nbytes / (us * 1e3) / PEAK_GBS)
            extra = "%8.0f GB/s %5.1f%% of 3.35 TB/s" % (r["gbs"], 100 * r["peak_share"])
        if flop is not None:
            peak = PEAK_BF16 if path == "linear" else PEAK_FP8
            r.update(tflops=flop / (us * 1e6), peak_share=flop / (us * 1e6) / peak)
            extra = "%8.0f TFLOP/s %5.1f%% of %d" % (r["tflops"], 100 * r["peak_share"], peak)
        rows.append(r)
        print("%-5s %5d %5d %-7s %-4s %9.1f us  %s" % (layer, k, n, path, kind, us, extra))

    gen = torch.Generator(device=dev).manual_seed(0)
    for name, k, n in SHAPES:
        copies = max(2, int(-(-args.rotate_mb * 1e6 // (2 * M * max(k, n)))))
        X = [torch.randn(M, k, device=dev, generator=gen, dtype=dt).requires_grad_(True) for _ in range(copies)]
        DYs = [torch.randn(M, n, device=dev, generator=gen, dtype=dt) for _ in range(copies)]
        base = nn.Linear(k, n).to(dev).to(dt)
        lin8 = Fp8Linear(k, n).to(dev).to(dt)
        lin8.load_state_dict(base.state_dict())
        flop = 2 * M * n * k
        for path, layer in (("linear", base), ("fp8", lin8)):
            params = [layer.weight, layer.bias]

            def fwd(i, layer=layer):
                layer(X[i])

            def both(i, layer=layer, params=params):
                torch.autograd.grad(layer(X[i]), [X[i]] + params, DYs[i])

            us_f = graphed_us(fwd, copies)
            us_b = graphed_us(both, copies) - us_f
            row(name, k, n, path, "fwd", us_f, flop=flop)
            row(name, k, n, path, "bwd", us_b, flop=2 * flop)

        # the cast kernels and the GEMMs of Fp8Linear on their own
        st = fp8.ScalingState(dev)
        fp8.seed(X[0].detach(), st.row(fp8.X), fp8.E4M3)
        fp8.seed(lin8.weight.detach(), st.row(fp8.W), fp8.E4M3)
        fp8.seed(DYs[0], st.row(fp8.DY), fp8.E5M2)

        def cast_fwd(i):
            fp8.cast(X[i].detach(), st.row(fp8.X), fp8.E4M3, fp8.BOTH)
            fp8.cast(lin8.weight.detach(), st.row(fp8.W), fp8.E4M3, fp8.BOTH)

        def cast_bwd(i):
            fp8.cast(DYs[i], st.row(fp8.DY), fp8.E5M2, fp8.BOTH, dt)

        row(name, k, n, "casts", "fwd", graphed_us(cast_fwd, copies), nbytes=cast_bytes("fwd", k, n))
        row(name, k, n, "casts", "bwd", graphed_us(cast_bwd, copies), nbytes=cast_bytes("bwd", k, n))
        ops = []
        for i in range(copies):
            x8, xt8, ix, _ = fp8.cast(X[i].detach(), st.row(fp8.X), fp8.E4M3, fp8.BOTH)
            dy8, dyt8, idy, _ = fp8.cast(DYs[i], st.row(fp8.DY), fp8.E5M2, fp8.BOTH)
            ops.append((x8, xt8, ix, dy8, dyt8, idy))
        w8, wt8, iw, _ = fp8.cast(lin8.weight.detach(), st.row(fp8.W), fp8.E4M3, fp8.BOTH)

        def mm(a, b, sa, sb, bias=None):
            return torch._scaled_mm(a, b, sa, sb, bias=bias, out_dtype=dt, use_fast_accum=False)

        def gemm_fwd(i):
            x8, _, ix, _, _, _ = ops[i]
            mm(x8, w8.t(), ix, iw, lin8.bias.detach())

        def gemm_bwd(i):
            _, xt8, ix, dy8, dyt8, idy = ops[i]
            mm(dy8, wt8.t(), idy, iw)
            mm(dyt8, xt8.t(), idy, ix)

        row(name, k, n, "gemm", "fwd", graphed_us(gemm_fwd, copies), flop=flop)
        row(name, k, n, "gemm", "bwd", graphed_us(gemm_bwd, copies), flop=2 * flop)
        del X, DYs, ops


def per_block(args, torch, rows):
    """fc1 -> GELU -> fc2 composed and fused, and the two fused casts alone"""
    import copy

    import torch.nn.functional as F

    from byteps_b200.ops import fp8
    from byteps_b200.ops.fp8 import Fp8Linear, fp8_gelu_mlp

    dev = torch.device("cuda", 0)
    dt = torch.bfloat16
    k, i = 1024, 4096
    gen = torch.Generator(device=dev).manual_seed(0)
    copies = max(2, int(-(-args.rotate_mb * 1e6 // (2 * M * i))))
    X = [torch.randn(M, k, device=dev, generator=gen, dtype=dt).requires_grad_(True) for _ in range(copies)]
    DY = [torch.randn(M, k, device=dev, generator=gen, dtype=dt) for _ in range(copies)]
    torch.manual_seed(0)
    fc1, fc2 = Fp8Linear(k, i).to(dev).to(dt), Fp8Linear(i, k).to(dev).to(dt)
    mods = {"composed": (copy.deepcopy(fc1), copy.deepcopy(fc2)), "fused": (fc1, fc2)}
    paths = {"composed": lambda x, m1, m2: m2(F.gelu(m1(x))), "fused": fp8_gelu_mlp}
    res = {}
    for path in ("composed", "fused"):
        m1, m2 = mods[path]
        f = paths[path]
        params = list(m1.parameters()) + list(m2.parameters())

        def fwd(j, f=f, m1=m1, m2=m2):
            f(X[j], m1, m2)

        def both(j, f=f, m1=m1, m2=m2, params=params):
            torch.autograd.grad(f(X[j], m1, m2), [X[j]] + params, DY[j])

        res[path] = (_graphed_us(args, torch, fwd, copies), _graphed_us(args, torch, both, copies))
    for path in ("composed", "fused"):
        us_f, us_fb = res[path]
        rows.append(dict(block="mlp", K=k, I=i, path=path, fwd_us=us_f, fwd_bwd_us=us_fb))
        print("mlp   %5d %5d %-8s fwd %9.1f us   fwd+bwd %9.1f us" % (k, i, path, us_f, us_fb))
    print("mlp   fused saves %.1f us forward and %.1f us forward + backward per layer" % (
        res["composed"][0] - res["fused"][0], res["composed"][1] - res["fused"][1]))
    del X, DY

    Z = [torch.randn(M, i, device=dev, generator=gen, dtype=dt) for _ in range(copies)]
    DH = [torch.randn(M, i, device=dev, generator=gen, dtype=dt) for _ in range(copies)]
    st = fp8.ScalingState(dev)
    fp8.seed(F.gelu(Z[0]), st.row(fp8.X), fp8.E4M3)
    fp8.seed(torch.ops.aten.gelu_backward(DH[0], Z[0]), st.row(fp8.DY), fp8.E5M2)

    def gelu_cast(j):
        fp8.cast(Z[j], st.row(fp8.X), fp8.E4M3, fp8.BOTH, act=fp8.ACT_GELU)

    def dgelu_cast(j):
        fp8.cast(DH[j], st.row(fp8.DY), fp8.E5M2, fp8.BOTH, dt, act=fp8.ACT_DGELU, aux=Z[j])

    for kind, fn, nbytes in (("gelu", gelu_cast, 4 * M * i), ("dgelu", dgelu_cast, 6 * M * i + 2 * i)):
        us = _graphed_us(args, torch, fn, copies)
        gbs = nbytes / (us * 1e3)
        rows.append(dict(block="actcast", M=M, I=i, kind=kind, us=us, bytes=nbytes, gbs=gbs,
                         peak_share=gbs / PEAK_GBS))
        print("actcast [%d, %d] %-5s %9.1f us %8.0f GB/s %5.1f%% of 3.35 TB/s" % (M, i, kind, us, gbs,
                                                                                 100 * gbs / PEAK_GBS))
    del Z, DH


def mlp_step(args, torch, rows):
    """BERT-large fp8_linear step with the encoder MLPs composed vs fused, two graphs timed alternately"""
    import torch.nn.functional as F

    import byteps_b200.models.bert as bert
    import byteps_b200.torch as bps
    from byteps_b200.torch.graph import GraphedStep

    dev = torch.device("cuda", 0)
    bps.init()
    torch.manual_seed(0)
    model = bert.bert_large(fp8_linear=True, fused_norm=True, fused_loss=True).to(dev).to(torch.bfloat16).train()
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

    fused_mlp = bert.fp8_gelu_mlp
    graphs = {}
    for name in ("composed", "fused"):
        bert.fp8_gelu_mlp = (lambda x, fc1, fc2: fc2(F.gelu(fc1(x)))) if name == "composed" else fused_mlp
        try:
            graphs[name] = GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams, device=dev)
        finally:
            bert.fp8_gelu_mlp = fused_mlp

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

    ms = {"composed": [], "fused": []}
    for _ in range(args.rounds):
        for name in ("composed", "fused"):
            ms[name].append(timed(graphs[name]))
    info = gpu_info()
    for name in ("composed", "fused"):
        med = statistics.median(ms[name])
        spread = max(ms[name]) - min(ms[name])
        rows.append(dict(step="fp8_linear_mlp_" + name, ms=ms[name], median_ms=med, spread_ms=spread,
                         tokens_per_s=args.batch * args.seq / (med / 1e3)))
        print("BERT-large fp8_linear step, MLP %-8s ms per step over %d rounds: %s  (median %.2f ms, spread "
              "%.2f ms)" % (name, args.rounds, " ".join("%.2f" % v for v in ms[name]), med, spread))
    print("fused MLP saves %.2f ms per step (medians)" % (statistics.median(ms["composed"]) -
                                                          statistics.median(ms["fused"])))
    print("GPU after the step rounds: %s" % info)
    del graphs
    bps.shutdown()


def whole_step(args, torch, rows):
    import byteps_b200.torch as bps
    from byteps_b200.models import bert_large
    from byteps_b200.ops.fp8 import Fp8Linear
    from byteps_b200.torch.graph import GraphedStep

    dev = torch.device("cuda", 0)
    bps.init()
    torch.manual_seed(0)
    model = bert_large(fused_norm=True, fused_loss=True).to(dev).to(torch.bfloat16).train()
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

    graphs, mem = {}, {}
    for f8 in (False, True):
        if f8:
            for layer in model.layers:
                for name in ("qkv", "proj", "fc1", "fc2"):
                    lin = getattr(layer, name)
                    lin.__class__ = Fp8Linear
                    lin._fp8 = None
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        graphs[f8] = GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams, device=dev)
        mem[f8] = torch.cuda.max_memory_allocated(dev) - before

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
        for f8 in (False, True):
            ms[f8].append(timed(graphs[f8]))
    info = gpu_info()
    for f8 in (False, True):
        name = "fp8_linear" if f8 else "bf16"
        med = statistics.median(ms[f8])
        spread = max(ms[f8]) - min(ms[f8])
        rows.append(dict(step=name, ms=ms[f8], median_ms=med, spread_ms=spread, peak_mem_bytes=mem[f8],
                         tokens_per_s=args.batch * args.seq / (med / 1e3)))
        print("BERT-large step %-10s ms per step over %d rounds: %s  (median %.2f ms, spread %.2f ms, %.0f tokens/s, "
              "peak memory above the model %.2f GB)" % (
                  name, args.rounds, " ".join("%.2f" % v for v in ms[f8]), med, spread,
                  args.batch * args.seq / (med / 1e3), mem[f8] / 1e9))
    print("GPU after the step rounds: %s" % info)
    del graphs
    bps.shutdown()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="calls captured in one timed graph")
    ap.add_argument("--reps", type=int, default=5, help="replays of that graph")
    ap.add_argument("--rotate-mb", type=float, default=600.0, help="bytes the input copies span together")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20, help="timed replays of a whole step per round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-step", action="store_true", help="per-layer table only")
    ap.add_argument("--only-mlp", action="store_true", help="only the feed-forward block rows and its step")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()

    import torch

    from byteps_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench.py needs a GPU")
    _native.cuda()
    torch.cuda.set_device(0)
    info = gpu_info()
    print("GPU: %s; M = %d, bf16 inputs" % (info, M))
    rows = []
    if not args.only_mlp:
        per_layer(args, torch, rows)
    per_block(args, torch, rows)
    if not args.no_step:
        if not args.only_mlp:
            whole_step(args, torch, rows)
        mlp_step(args, torch, rows)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
