#!/usr/bin/env python
"""Where one training step of the bench configuration spends its GPU time.

Builds the model exactly as ``bench.py`` does (same model, dtype, channels_last, seeded weights and batch,
``DistributedOptimizer(fused_update=True)``), times the whole step captured in one CUDA graph with CUDA events,
then profiles a few eager steps with ``torch.profiler`` (CUDA activities) and sums kernel time per category:

    conv      convolution / GEMM kernels (cuDNN, cuBLAS, CUTLASS) and their layout transforms
    bn        batch-norm forward / backward, under whatever names torch picks (cuDNN or ATen)
    relu      ReLU forward and threshold-backward
    add       elementwise add: the residual add and autograd's gradient accumulation
    fused_opt our fused optimizer and stamp kernels (namespace bps)
    bn_act    our fused batch-norm / activation kernels (namespace bps, bn_act_*)
    other     everything else (pooling, loss, casts, memset, ...)

    python benchmarks/step_breakdown.py [--out-dir DIR]

The trace (Chrome JSON) and the per-kernel table go under --out-dir (default: a directory under the system's
temporary directory).  The GPU name and power limit are read in the
same run and printed with the result.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# first match wins; names are the demangled kernel names the profiler reports
CATEGORIES = [
    ("bn_act", re.compile(r"bps::.*bn_act")),
    ("fused_opt", re.compile(r"bps::")),
    ("bn", re.compile(r"batch_norm|batchnorm|bn_fw|bn_bw|cudnn::bn|nhwc_batch_norm|welford", re.I)),
    ("relu", re.compile(r"threshold|clamp_min|clamp_scalar|relu", re.I)),
    ("add", re.compile(r"AddFunctor|add_kernel|CUDAFunctor_add|\badd\b", re.I)),
    ("conv", re.compile(r"conv|gemm|xmma|cutlass|wgrad|dgrad|fprop|implicit|nchwToNhwc|nhwcToNchw|cudnn|cublas|"
                        r"sm90_|sm80_|nvjet", re.I)),
]


def category(name):
    for cat, rx in CATEGORIES:
        if rx.search(name):
            return cat
    return "other"


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="resnet50")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--seq-len", type=int, default=128)
    ap.add_argument("--steps", type=int, default=5, help="profiled eager steps")
    ap.add_argument("--graph-steps", type=int, default=50, help="timed graph replays")
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "step_breakdown"))
    ap.add_argument("--top", type=int, default=25, help="kernels listed per run")
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from torch.profiler import ProfilerActivity, profile

    import bench
    import byteps_b200.torch as bps
    from byteps_b200.torch.graph import GraphedStep

    if not torch.cuda.is_available():
        raise SystemExit("step_breakdown.py needs a GPU")
    os.makedirs(args.out_dir, exist_ok=True)
    torch.cuda.set_device(0)
    device = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = False
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    bps.init()
    torch.manual_seed(0)
    model, _, sx, sy, _ = bench.build(args, torch, bps, device)
    base = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.0)
    opt = bps.DistributedOptimizer(base, named_parameters=model.named_parameters(), fused_update=True)
    bps.broadcast_parameters(model.state_dict(), root_rank=0)

    def train_step():
        opt.zero_grad()
        loss = F.cross_entropy(model(sx).float(), sy)
        loss.backward()
        opt.step()
        return loss

    # graphed step time (what bench.py reports), profiler off
    stepper = GraphedStep(train_step, warmup=3, pre_replay=opt.refresh_hparams, device=device)
    for _ in range(10):
        stepper()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.graph_steps):
        stepper()
    e1.record()
    torch.cuda.synchronize()
    graph_ms = e0.elapsed_time(e1) / args.graph_steps
    info = gpu_info()

    # eager steps under the profiler (a separate run: tracing slows the host, not the kernels)
    for _ in range(3):
        train_step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            train_step()
        torch.cuda.synchronize()
    trace = os.path.join(args.out_dir, "trace.json")
    prof.export_chrome_trace(trace)

    per_kernel = collections.defaultdict(lambda: [0.0, 0])
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        per_kernel[ev.name][0] += ev.time_range.elapsed_us() / 1e3
        per_kernel[ev.name][1] += 1
    cats = collections.OrderedDict((c, 0.0) for c in ["conv", "bn", "relu", "add", "fused_opt", "bn_act", "other"])
    for name, (ms, _) in per_kernel.items():
        cats[category(name)] += ms / args.steps
    total = sum(cats.values())
    rows = sorted(((ms / args.steps, n // args.steps, category(k), k) for k, (ms, n) in per_kernel.items()),
                  reverse=True)
    with open(os.path.join(args.out_dir, "kernels.txt"), "w") as f:
        for ms, n, cat, k in rows:
            f.write("%9.3f ms  %4d  %-9s %s\n" % (ms, n, cat, k))

    print("GPU: %s" % info)
    print("%s %s batch %d: graphed step %.3f ms; eager kernel time %.3f ms/step (%d profiled steps)"
          % (args.model, args.dtype, args.batch_size, graph_ms, total, args.steps))
    print("%-10s %9s %7s %7s" % ("category", "ms/step", "%kern", "%graph"))
    for c, ms in cats.items():
        print("%-10s %9.3f %6.1f%% %6.1f%%" % (c, ms, 100 * ms / total, 100 * ms / graph_ms))
    print("top kernels per step (all in %s):" % os.path.join(args.out_dir, "kernels.txt"))
    for ms, n, cat, k in rows[:args.top]:
        print("  %8.3f ms %4d  %-9s %s" % (ms, n, cat, k[:140]))
    out = {"gpu": info, "model": args.model, "dtype": args.dtype, "batch": args.batch_size,
           "graph_ms_per_step": graph_ms, "kernel_ms_per_step": total, "categories_ms": cats, "trace": trace}
    with open(os.path.join(args.out_dir, "breakdown.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))
    bps.shutdown()


if __name__ == "__main__":
    main()
