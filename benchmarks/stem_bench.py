#!/usr/bin/env python
"""ResNet's 7x7 stem convolution (3 -> 64 channels, stride 2, padding 3) at the bench shape: a 64 x 3 x 224 x 224
bf16 image and weight, both channels_last, the input not requiring grad.

Two arms run the same calls:

    stock    F.conv2d (cuDNN, cudnn.benchmark off, as in bench.py)
    kernel   ops/stem_conv.py's StemConv2d (kernels/stem_conv.cu)

and each times two passes:

    fwd        y = conv(x)
    fwd+wgrad  y = conv(x); dW = torch.autograd.grad(y, w, dy)   (no dgrad: the image needs no gradient)

Each pass is captured in one CUDA graph of --iters calls that cycle through --copies copies of x and dy, so no call
finds its input in the 50 MB L2 from the call before; the graph is replayed --reps times between CUDA events and the
median replay is reported per call.  Bytes and FLOPs are the least the algorithm needs, computed from the shapes:

    fwd    read x, write y              FLOPs 2 * N*OH*OW * 64 * 147
    wgrad  read dy and x, write dW      FLOPs 2 * N*OH*OW * 64 * 147

and the floor of a pass is the larger of bytes / 3.35 TB/s and FLOPs / 989 TFLOP/s (H100 SXM data sheet, dense
bf16, 700 W); the share of the floor names which of the two bounds it.  Each arm then runs once more under
torch.profiler and lists the kernels it launched per fwd+wgrad call with their time.  The GPU name, power limit and
SM clock are read in the same run.

    python benchmarks/stem_bench.py [--batch 64] [--size 224] [--dtype bf16] [--arms stock,kernel] [--json out.json]
"""
import argparse
import collections
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


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp16"])
    ap.add_argument("--arms", default="stock,kernel")
    ap.add_argument("--iters", type=int, default=20, help="calls per graph")
    ap.add_argument("--reps", type=int, default=10, help="timed graph replays")
    ap.add_argument("--copies", type=int, default=4, help="copies of x and dy the calls cycle through")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from torch.profiler import ProfilerActivity, profile

    from byteps_b200.ops.stem_conv import StemConv2d

    if not torch.cuda.is_available():
        raise SystemExit("stem_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cudnn.benchmark = False
    dt = torch.bfloat16 if args.dtype == "bf16" else torch.float16
    e = 2
    n, h = args.batch, args.size
    oh = (h - 1) // 2 + 1
    p = n * oh * oh
    flops = 2.0 * p * 64 * 147
    bytes_x, bytes_y, bytes_w = n * 3 * h * h * e, p * 64 * e, 64 * 147 * e
    least = {"fwd": bytes_x + bytes_y, "wgrad": bytes_y + bytes_x + bytes_w}

    torch.manual_seed(0)
    stock = torch.nn.Conv2d(3, 64, 7, 2, 3, bias=False)
    kern = StemConv2d(3, 64, 7, 2, 3, bias=False)
    kern.load_state_dict(stock.state_dict())
    mods = {}
    for name, m in (("stock", stock), ("kernel", kern)):
        mods[name] = m.to(dev).to(dt).to(memory_format=torch.channels_last)
    g = torch.Generator(device=dev).manual_seed(1)
    xs = [torch.rand(n, 3, h, h, device=dev, generator=g).to(dt).contiguous(memory_format=torch.channels_last)
          for _ in range(args.copies)]
    dys = [torch.randn(n, 64, oh, oh, device=dev, generator=g).to(dt).contiguous(memory_format=torch.channels_last)
           for _ in range(args.copies)]

    def fwd(m, i):
        return m(xs[i % args.copies])

    def fwd_wgrad(m, i):
        y = m(xs[i % args.copies])
        return torch.autograd.grad(y, m.weight, dys[i % args.copies])[0]

    def timed(fn, m):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for i in range(3):
                fn(m, i)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for i in range(args.iters):
                fn(m, i)
        graph.replay()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            graph.replay()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b) / args.iters)
        del graph
        return statistics.median(ms), max(ms) - min(ms)

    def kernels(fn, m):
        for i in range(3):
            fn(m, i)
        torch.cuda.synchronize()
        calls = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(calls):
                fn(m, i)
            torch.cuda.synchronize()
        per = collections.defaultdict(lambda: [0.0, 0])
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                per[ev.name][0] += ev.time_range.elapsed_us() / calls
                per[ev.name][1] += 1
        return sorted(((us, cnt / calls, k) for k, (us, cnt) in per.items()), reverse=True)

    def floor_us(b):
        tb, tf = b / (PEAK_GBS * 1e3), flops / (PEAK_TFLOPS * 1e6)
        return max(tb, tf), "bytes" if tb >= tf else "FLOPs"

    info = gpu_info()
    print("GPU (name, power limit, SM clock, max SM clock): %s" % info)
    print("stem conv %d x 3 x %d x %d %s -> %d x 64 x %d x %d, channels_last; %.2f GFLOP per pass"
          % (n, h, h, args.dtype, n, oh, oh, flops / 1e9))
    rows = []
    print("%-7s %-10s %9s %9s %8s %9s %10s %7s" % ("arm", "pass", "us", "spread", "GB/s", "TFLOP/s", "floor us",
                                                  "%floor"))
    for arm in [a for a in args.arms.split(",") if a]:
        m = mods[arm]
        t_f, s_f = timed(fwd, m)
        t_fw, s_fw = timed(fwd_wgrad, m)
        t_w = t_fw - t_f
        for pas, ms, spread, b, fl in (("fwd", t_f, s_f, least["fwd"], flops),
                                       ("wgrad", t_w, None, least["wgrad"], flops),
                                       ("fwd+wgrad", t_fw, s_fw, least["fwd"] + least["wgrad"], 2 * flops)):
            us = ms * 1e3
            fl_us, bound = floor_us(b) if pas != "fwd+wgrad" else (floor_us(least["fwd"])[0]
                                                                   + floor_us(least["wgrad"])[0], "bytes")
            row = {"arm": arm, "pass": pas, "us": us, "spread_us": None if spread is None else spread * 1e3,
                   "gbs": b / (us * 1e3), "tflops": fl / (us * 1e6), "floor_us": fl_us, "bound": bound,
                   "pct_floor": 100 * fl_us / us}
            rows.append(row)
            print("%-7s %-10s %9.1f %9s %8.0f %9.1f %10.1f %6.1f%% (%s)"
                  % (arm, pas, us, "-" if spread is None else "%.1f" % (spread * 1e3), row["gbs"], row["tflops"],
                     fl_us, row["pct_floor"], bound))
    kern_rows = {}
    for arm in [a for a in args.arms.split(",") if a]:
        ks = kernels(fwd_wgrad, mods[arm])
        kern_rows[arm] = [{"us": us, "launches": c, "name": k} for us, c, k in ks]
        print("%s arm, kernels per fwd+wgrad call (profiler, eager):" % arm)
        for us, c, k in ks:
            print("  %9.1f us %5.1f  %s" % (us, c, k[:150]))
        print("  %9.1f us total" % sum(us for us, _, _ in ks))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "rows": rows, "kernels": kern_rows}, f, indent=1)


if __name__ == "__main__":
    main()
