#!/usr/bin/env python
"""Fused batch norm + residual add + ReLU kernels (kernels/bn_act.cu) against the stock torch sequence, at the
12 distinct ResNet-50 batch-norm shapes (C, H, W) and batch 64, bf16 activations with fp32 parameters (the
bench.py configuration), NHWC.

Each shape runs the variants the model uses: BN + ReLU everywhere; BN + residual + ReLU (bn3) and plain BN
(downsample) on the four expanded shapes.  Times are CUDA events over --iters launches after a warm-up.  Bytes
are the least each fused pass must move, computed from the shape (e = element bytes, N = elements, mask N / 8):

    fwd_stats   read x                                   N e
    fwd_apply   read x [, residual]; write y [, mask]     N e (2 [+1]) [+ N / 8]
    bwd_reduce  read dy, x [, mask]                       2 N e [+ N / 8]
    bwd_apply   read dy, x [, mask]; write dx [, dres]    N e (3 [+1]) [+ N / 8]

The stock rows time F.batch_norm [+ add] [+ relu] and its autograd backward; their GB/s use the fused passes'
bytes, i.e. they are the rate at which the stock sequence delivers the same work.  Share of peak is against the
H100 SXM data-sheet 3.35 TB/s; the GPU name and power limit are printed with the table.

    python benchmarks/bn_act_bench.py [--batch 64] [--iters 50] [--json out.json]
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
SHAPES = [(64, 112, 112), (64, 56, 56), (256, 56, 56), (128, 56, 56), (128, 28, 28), (512, 28, 28),
          (256, 28, 28), (256, 14, 14), (1024, 14, 14), (512, 14, 14), (512, 7, 7), (2048, 7, 7)]
EXPANDED = {(256, 56, 56), (512, 28, 28), (1024, 14, 14), (2048, 7, 7)}


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
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F

    from byteps_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("bn_act_bench.py needs a GPU")
    cu = _native.cuda()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    s = torch.cuda.current_stream().cuda_stream
    dt, code, e = torch.bfloat16, 1, 2

    def timed(fn):
        for _ in range(3):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.iters

    info = gpu_info()
    rows = []
    print("GPU: %s; batch %d, bf16 activations, fp32 parameters, NHWC" % (info, args.batch))
    print("%-14s %-9s %-11s %9s %9s %8s %6s" % ("C x H x W", "variant", "pass", "MB", "us", "GB/s", "%peak"))
    for (c, h, w) in SHAPES:
        variants = ["relu"] + (["relu_res", "none"] if (c, h, w) in EXPANDED else [])
        n, m = args.batch * c * h * w, args.batch * h * w
        for var in variants:
            relu, res = var != "none", var == "relu_res"
            g = torch.Generator(device=dev).manual_seed(0)
            x = torch.randn(args.batch, c, h, w, device=dev, generator=g).to(dt).contiguous(
                memory_format=torch.channels_last)
            r = torch.randn_like(x) if res else None
            dy = torch.randn_like(x)
            wt, bs = torch.ones(c, device=dev), torch.zeros(c, device=dev)
            rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
            mean, inv, dw, db = (torch.empty(c, device=dev) for _ in range(4))
            nws, nctr = cu.bn_act_workspace(m, c)
            ws = torch.empty(nws, device=dev)
            ctr = torch.zeros(nctr, dtype=torch.int32, device=dev)
            y, dx = torch.empty_like(x), torch.empty_like(x)
            dres = torch.empty_like(x) if res else None
            mask = torch.empty(m, c // 8, dtype=torch.uint8, device=dev) if relu else None
            mp, rp, dp = (mask.data_ptr() if relu else 0), (r.data_ptr() if res else 0), (dres.data_ptr() if res else 0)
            mb = n // 8 if relu else 0
            passes = [
                ("fwd_stats", n * e, lambda: cu.bn_act_fwd_stats(x.data_ptr(), code, m, c, 1e-5, 0.1, rm.data_ptr(),
                                                                 rv.data_ptr(), mean.data_ptr(), inv.data_ptr(),
                                                                 ws.data_ptr(), ctr.data_ptr(), s)),
                ("fwd_apply", n * e * (3 if res else 2) + mb,
                 lambda: cu.bn_act_fwd_apply(x.data_ptr(), rp, code, m, c, mean.data_ptr(), inv.data_ptr(),
                                             wt.data_ptr(), bs.data_ptr(), relu, y.data_ptr(), mp, s)),
                ("bwd_reduce", 2 * n * e + mb,
                 lambda: cu.bn_act_bwd_reduce(dy.data_ptr(), x.data_ptr(), mp, code, m, c, mean.data_ptr(),
                                              inv.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr(),
                                              ctr.data_ptr(), s)),
                ("bwd_apply", n * e * (4 if res else 3) + mb,
                 lambda: cu.bn_act_bwd_apply(dy.data_ptr(), x.data_ptr(), mp, code, m, c, mean.data_ptr(),
                                             inv.data_ptr(), wt.data_ptr(), dw.data_ptr(), db.data_ptr(),
                                             dx.data_ptr(), dp, s)),
            ]
            tot = {"fwd": [0.0, 0], "bwd": [0.0, 0]}
            for name, nbytes, fn in passes:
                ms = timed(fn)
                side = tot[name[:3]]
                side[0] += ms
                side[1] += nbytes
                rows.append(dict(shape=[c, h, w], variant=var, impl="fused", kind=name, bytes=nbytes, us=ms * 1e3))

            # stock sequence on the same tensors
            xs = x.detach().requires_grad_(True)
            rs = r.detach().requires_grad_(True) if res else None
            ws_, bs_ = wt.clone().requires_grad_(True), bs.clone().requires_grad_(True)

            def stock_fwd():
                t = F.batch_norm(xs, rm, rv, ws_, bs_, True, 0.1, 1e-5)
                if res:
                    t = t + rs
                return F.relu(t, inplace=True) if relu else t

            def stock_both():
                t = stock_fwd()
                torch.autograd.grad(t, [xs, ws_, bs_] + ([rs] if res else []), dy)

            with torch.no_grad():
                ms_f = timed(stock_fwd)
            ms_b = timed(stock_both) - timed(stock_fwd)
            rows.append(dict(shape=[c, h, w], variant=var, impl="stock", kind="fwd", bytes=tot["fwd"][1],
                             us=ms_f * 1e3))
            rows.append(dict(shape=[c, h, w], variant=var, impl="stock", kind="bwd", bytes=tot["bwd"][1],
                             us=ms_b * 1e3))
            for side in ("fwd", "bwd"):
                rows.append(dict(shape=[c, h, w], variant=var, impl="fused", kind=side, bytes=tot[side][1],
                                 us=tot[side][0] * 1e3))
            for row in rows[-(len(passes) + 4):]:
                gbs = row["bytes"] / (row["us"] * 1e3)
                row["gbs"], row["peak_share"] = gbs, gbs / PEAK_GBS
                print("%-14s %-9s %-11s %9.1f %9.1f %8.0f %5.0f%%" % (
                    "%dx%dx%d" % (c, h, w), var, row["impl"] + ":" + row["kind"], row["bytes"] / 1e6, row["us"], gbs,
                    100 * row["peak_share"]))
    f_tot = sum(r_["us"] for r_ in rows if r_["impl"] == "fused" and r_["kind"] in ("fwd", "bwd"))
    s_tot = sum(r_["us"] for r_ in rows if r_["impl"] == "stock")
    print("sum over the variants above: fused %.0f us, stock %.0f us" % (f_tot, s_tot))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "batch": args.batch, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
