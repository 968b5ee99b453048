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

    single:fwd  read x once [, residual]; write y [, mask]  N e (2 [+1]) [+ N / 8]   (fwd_stats + fwd_apply in one launch)
    single:bwd  read dy, x [, mask] once; write dx [, dres]  N e (3 [+1]) [+ N / 8]   (bwd_reduce + bwd_apply)

The fused:fwd / fused:bwd rows sum the two-pass kernels; the single rows are the single-launch kernels the module
takes where their plan allows it.  On the expanded shapes the junction rows time bn3's backward at a ResNet block
junction, where the output has two consumers: junction:add+bwd is torch's add of the two gradients followed by the
single-launch backward (what autograd did before the kernel took both), junction:bwd2 the single-launch backward
reading both gradients.  Their bytes are what the launches move (the add: 3 N e; the plans' bytes_moved), and the
table ends with the saving per ResNet-50 step over its 15 junctions.  Those rows also print the bytes the launch actually moves (the plan's
bytes_moved: the rows a block does not hold are read twice) with the share of peak over them, and the plan's held
rows per chunk and ring depth.  Every timed launch moves to the next of enough copies of the tensors that the
launches of a row touch more than --rotate-mb together, so no pass finds its input in the 50 MB L2 from the launch
before.  The stock rows time F.batch_norm [+ add] [+ relu] and its autograd backward; their GB/s use the fused passes'
bytes, i.e. they are the rate at which the stock sequence delivers the same work.  Share of peak is against the
H100 SXM data-sheet 3.35 TB/s; the GPU name and power limit are printed with the table.

The stem rows (64 x 112 x 112, ReLU) compare what the stem ran before the pooled kernels with them.  chain:fwd is
the single-launch forward then torch's max pool with indices (as autograd runs it); chain:bwd is torch's add of the
two pooled gradients (the junction before layer1), torch's max-pool backward and the single-launch backward.
pooled:fwd / pooled:bwd are bn_act_fwd_pool / bn_act_bwd_pool with both gradients.  They report the bytes the
launches move (the plans' bytes_moved; torch's passes: their tensors once, int64 indices) and the least bytes, P
pooled rows, M rows, C channels:

    least fwd   read x; write the pooled output and 4-bit codes        M C e + P C (e + 1/2)
    least bwd   read both pooled gradients, the codes and x; write dx  2 M C e + P C (2 e + 1/2)

with the share of 3.35 TB/s over the least bytes.

    python benchmarks/bn_act_bench.py [--batch 64] [--iters 50] [--rotate-mb 200] [--stem-only] [--json out.json]
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
# ResNet-50's block junctions per expanded shape: identity and downsample skip paths of the block that follows
JUNCTIONS = {(256, 56, 56): 3, (512, 28, 28): 4, (1024, 14, 14): 6, (2048, 7, 7): 2}


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
    ap.add_argument("--rotate-mb", type=float, default=200.0, help="bytes the tensor copies of a row span together")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    ap.add_argument("--stem-only", action="store_true", help="only the stem rows (batch norm, ReLU and max pool)")
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

    def timed(fn, k):
        """fn(i) on tensor copy i % k"""
        for i in range(max(3, k)):
            fn(i % k)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(args.iters):
            fn(i % k)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.iters

    info = gpu_info()
    rows = []
    print("GPU: %s; batch %d, bf16 activations, fp32 parameters, NHWC" % (info, args.batch))
    print("%-14s %-9s %-11s %9s %9s %8s %6s %9s %7s" % ("C x H x W", "variant", "pass", "MB", "us", "GB/s", "%peak",
                                                       "moved MB", "%peak"))
    for (c, h, w) in ([] if args.stem_only else SHAPES):
        variants = ["relu"] + (["relu_res", "none"] if (c, h, w) in EXPANDED else [])
        n, m = args.batch * c * h * w, args.batch * h * w
        for var in variants:
            relu, res = var != "none", var == "relu_res"
            g = torch.Generator(device=dev).manual_seed(0)
            mb = n // 8 if relu else 0
            k = max(1, int(-(-args.rotate_mb * 1e6 // (n * e * (7 if res else 3) + 2 * mb))))

            def copies():
                x = torch.randn(args.batch, c, h, w, device=dev, generator=g).to(dt).contiguous(
                    memory_format=torch.channels_last)
                return dict(x=x, r=torch.randn_like(x) if res else None, dy=torch.randn_like(x),
                            y=torch.empty_like(x), dx=torch.empty_like(x),
                            dres=torch.empty_like(x) if res else None,
                            dy2=torch.randn_like(x) if res else None, dsum=torch.empty_like(x) if res else None,
                            mask=torch.empty(m, c // 8, dtype=torch.uint8, device=dev) if relu else None)

            first = len(rows)
            T = [copies() for _ in range(k)]
            P = [{key: (0 if t is None else t.data_ptr()) for key, t in tk.items()} for tk in T]
            wt, bs = torch.ones(c, device=dev), torch.zeros(c, device=dev)
            rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
            mean, inv, dw, db = (torch.empty(c, device=dev) for _ in range(4))
            nws, nctr = cu.bn_act_workspace(m, c)
            ws = torch.empty(nws, device=dev)
            ctr = torch.zeros(nctr, dtype=torch.int32, device=dev)
            passes = [
                ("fwd_stats", n * e, lambda i: cu.bn_act_fwd_stats(P[i]["x"], code, m, c, 1e-5, 0.1, rm.data_ptr(),
                                                                   rv.data_ptr(), mean.data_ptr(), inv.data_ptr(),
                                                                   ws.data_ptr(), ctr.data_ptr(), s)),
                ("fwd_apply", n * e * (3 if res else 2) + mb,
                 lambda i: cu.bn_act_fwd_apply(P[i]["x"], P[i]["r"], code, m, c, mean.data_ptr(), inv.data_ptr(),
                                               wt.data_ptr(), bs.data_ptr(), relu, P[i]["y"], P[i]["mask"], s)),
                ("bwd_reduce", 2 * n * e + mb,
                 lambda i: cu.bn_act_bwd_reduce(P[i]["dy"], P[i]["x"], P[i]["mask"], code, m, c, mean.data_ptr(),
                                                inv.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr(),
                                                ctr.data_ptr(), s)),
                ("bwd_apply", n * e * (4 if res else 3) + mb,
                 lambda i: cu.bn_act_bwd_apply(P[i]["dy"], P[i]["x"], P[i]["mask"], code, m, c, mean.data_ptr(),
                                               inv.data_ptr(), wt.data_ptr(), dw.data_ptr(), db.data_ptr(),
                                               P[i]["dx"], P[i]["dres"], s)),
            ]
            tot = {"fwd": [0.0, 0], "bwd": [0.0, 0]}
            for name, nbytes, fn in passes:
                ms = timed(fn, k)
                side = tot[name[:3]]
                side[0] += ms
                side[1] += nbytes
                rows.append(dict(shape=[c, h, w], variant=var, impl="fused", kind=name, bytes=nbytes, us=ms * 1e3))

            # the single-launch kernels; their counters are left non-zero, so each launch gets a zeroed set
            fplan = cu.bn_act_plan(0, code, m, c, relu=relu, residual=res)
            bplan = cu.bn_act_plan(1, code, m, c, relu=relu, residual=res)
            single = []
            if fplan is not None and bplan is not None:
                nctr1 = max(fplan["counters"], bplan["counters"])
                ws1 = torch.empty(max(fplan["ws_floats"], bplan["ws_floats"]), device=dev)
                ctrs = torch.zeros(args.iters + max(3, k), nctr1, dtype=torch.int32, device=dev)
                launch = [0]

                def zeroed():
                    launch[0] += 1
                    return ctrs[launch[0] - 1].data_ptr()

                single = [
                    ("fwd", n * e * (3 if res else 2) + mb,
                     lambda i: cu.bn_act_fwd(P[i]["x"], P[i]["r"], code, m, c, 1e-5, 0.1, rm.data_ptr(), rv.data_ptr(),
                                             mean.data_ptr(), inv.data_ptr(), wt.data_ptr(), bs.data_ptr(), relu,
                                             P[i]["y"], P[i]["mask"], ws1.data_ptr(), zeroed(), s)),
                    ("bwd", n * e * (4 if res else 3) + mb,
                     lambda i: cu.bn_act_bwd(P[i]["dy"], P[i]["x"], P[i]["mask"], code, m, c, mean.data_ptr(),
                                             inv.data_ptr(), wt.data_ptr(), dw.data_ptr(), db.data_ptr(), P[i]["dx"],
                                             P[i]["dres"], ws1.data_ptr(), zeroed(), s)),
                ]
                for name, nbytes, fn in single:
                    launch[0] = 0
                    ctrs.zero_()
                    ms = timed(fn, k)
                    plan = fplan if name == "fwd" else bplan
                    rows.append(dict(shape=[c, h, w], variant=var, impl="single", kind=name, bytes=nbytes,
                                     us=ms * 1e3, held_rows=plan["held_rows"], rows_per_chunk=plan["rows_per_chunk"],
                                     ring_depth=plan["ring_depth"], bytes_moved=plan["bytes_moved"]))

                if res:
                    jplan = cu.bn_act_plan(1, code, m, c, relu=relu, residual=True, dy2=True)

                    def bwd(i, dy, dy2=0):
                        cu.bn_act_bwd(dy, P[i]["x"], P[i]["mask"], code, m, c, mean.data_ptr(), inv.data_ptr(),
                                      wt.data_ptr(), dw.data_ptr(), db.data_ptr(), P[i]["dx"], P[i]["dres"],
                                      ws1.data_ptr(), zeroed(), s, -1, dy2)

                    def add_bwd(i):
                        torch.add(T[i]["dy"], T[i]["dy2"], out=T[i]["dsum"])
                        bwd(i, P[i]["dsum"])

                    for name, plan, fn in (("add+bwd", bplan, add_bwd),
                                           ("bwd2", jplan, lambda i: bwd(i, P[i]["dy"], P[i]["dy2"]))):
                        launch[0] = 0
                        ctrs.zero_()
                        ms = timed(fn, k)
                        moved = plan["bytes_moved"] + (3 * n * e if name == "add+bwd" else 0)
                        rows.append(dict(shape=[c, h, w], variant=var, impl="junction", kind=name, bytes=moved,
                                         us=ms * 1e3, held_rows=plan["held_rows"],
                                         rows_per_chunk=plan["rows_per_chunk"], ring_depth=plan["ring_depth"],
                                         bytes_moved=moved))

            # stock sequence on the same tensors
            XS = [t["x"].detach().requires_grad_(True) for t in T]
            RS = [t["r"].detach().requires_grad_(True) if res else None for t in T]
            ws_, bs_ = wt.clone().requires_grad_(True), bs.clone().requires_grad_(True)

            def stock_fwd(i):
                t = F.batch_norm(XS[i], rm, rv, ws_, bs_, True, 0.1, 1e-5)
                if res:
                    t = t + RS[i]
                return F.relu(t, inplace=True) if relu else t

            def stock_both(i):
                t = stock_fwd(i)
                torch.autograd.grad(t, [XS[i], ws_, bs_] + ([RS[i]] if res else []), T[i]["dy"])

            with torch.no_grad():
                ms_f = timed(stock_fwd, k)
            ms_b = timed(stock_both, k) - timed(stock_fwd, k)
            rows.append(dict(shape=[c, h, w], variant=var, impl="stock", kind="fwd", bytes=tot["fwd"][1],
                             us=ms_f * 1e3))
            rows.append(dict(shape=[c, h, w], variant=var, impl="stock", kind="bwd", bytes=tot["bwd"][1],
                             us=ms_b * 1e3))
            for side in ("fwd", "bwd"):
                rows.append(dict(shape=[c, h, w], variant=var, impl="fused", kind=side, bytes=tot[side][1],
                                 us=tot[side][0] * 1e3))
            for row in rows[first:]:
                gbs = row["bytes"] / (row["us"] * 1e3)
                row["gbs"], row["peak_share"] = gbs, gbs / PEAK_GBS
                extra = ""
                if row["impl"] in ("single", "junction"):
                    row["moved_share"] = row["bytes_moved"] / (row["us"] * 1e3) / PEAK_GBS
                    extra = " %9.1f %6.0f%%  held %d/%d ring %d" % (
                        row["bytes_moved"] / 1e6, 100 * row["moved_share"], row["held_rows"], row["rows_per_chunk"],
                        row["ring_depth"])
                print("%-14s %-9s %-11s %9.1f %9.1f %8.0f %5.0f%%%s" % (
                    "%dx%dx%d" % (c, h, w), var, row["impl"] + ":" + row["kind"], row["bytes"] / 1e6, row["us"], gbs,
                    100 * row["peak_share"], extra))
            del T, P, XS, RS
    rows += stem_rows(args, torch, cu, dev, s, timed)
    f_tot = sum(r_["us"] for r_ in rows if r_["impl"] == "fused" and r_["kind"] in ("fwd", "bwd"))
    g_tot = sum(r_["us"] for r_ in rows if r_["impl"] == "single")
    s_tot = sum(r_["us"] for r_ in rows if r_["impl"] == "stock")
    print("sum over the variants above: two-pass %.0f us, single-launch %.0f us, stock %.0f us" % (f_tot, g_tot, s_tot))
    junction = {(tuple(r_["shape"]), r_["kind"]): r_["us"] for r_ in rows if r_["impl"] == "junction"}
    if junction:
        saved = sum(cnt * (junction[(shp, "add+bwd")] - junction[(shp, "bwd2")]) for shp, cnt in JUNCTIONS.items()
                    if (shp, "bwd2") in junction)
        print("ResNet-50 junctions (%s): add+bwd -> bwd2 saves %.0f us per step" % (
            ", ".join("%dx%dx%d: %d" % (shp + (cnt,)) for shp, cnt in JUNCTIONS.items()), saved))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "batch": args.batch, "rows": rows}, fh, indent=1)


def stem_rows(args, torch, cu, dev, s, timed):
    """The stem's batch norm, ReLU, max pool and pooled junction: the stock chain against the pooled kernels."""
    c, h, w, e, code = 64, 112, 112, 2, 1
    oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    m, p = args.batch * h * w, args.batch * oh * ow
    g = torch.Generator(device=dev).manual_seed(0)
    nhwc = dict(memory_format=torch.channels_last)
    k = max(1, int(-(-args.rotate_mb * 1e6 // (m * c * e * 3 + p * c * e * 2))))

    def copies():
        x = torch.randn(args.batch, c, h, w, device=dev, generator=g).to(torch.bfloat16).contiguous(**nhwc)
        g1 = torch.randn(args.batch, c, oh, ow, device=dev, generator=g).to(torch.bfloat16).contiguous(**nhwc)
        return dict(x=x, y=torch.empty_like(x), dx=torch.empty_like(x), g1=g1, g2=torch.randn_like(g1),
                    pooled=torch.empty_like(g1), mask=torch.empty(m, c // 8, dtype=torch.uint8, device=dev),
                    code=torch.empty(p, c // 8, dtype=torch.int32, device=dev))

    T = [copies() for _ in range(k)]
    wt, bs = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
    mean, inv, dw, db = (torch.empty(c, device=dev) for _ in range(4))
    fplan, bplan = cu.bn_act_plan(0, code, m, c, relu=True), cu.bn_act_plan(1, code, m, c, relu=True)
    pf = cu.bn_act_plan(0, code, m, c, relu=True, pool_h=h, pool_w=w)
    pb = cu.bn_act_plan(1, code, m, c, relu=True, dy2=True, pool_h=h, pool_w=w)
    if None in (fplan, bplan, pf, pb):
        print("stem: a single-launch plan is refused on this device; no stem rows")
        return []
    ws = torch.empty(max(pl["ws_floats"] for pl in (fplan, bplan, pf, pb)), device=dev)
    ctrs = torch.zeros(2 * (args.iters + max(3, k)), max(pl["counters"] for pl in (fplan, bplan, pf, pb)),
                       dtype=torch.int32, device=dev)
    launch = [0]

    def zeroed():
        launch[0] += 1
        return ctrs[launch[0] - 1].data_ptr()

    def fwd(i):
        t = T[i]
        cu.bn_act_fwd(t["x"].data_ptr(), 0, code, m, c, 1e-5, 0.1, rm.data_ptr(), rv.data_ptr(), mean.data_ptr(),
                      inv.data_ptr(), wt.data_ptr(), bs.data_ptr(), True, t["y"].data_ptr(), t["mask"].data_ptr(),
                      ws.data_ptr(), zeroed(), s)

    def chain_fwd(i):
        fwd(i)
        T[i]["pool"] = torch.ops.aten.max_pool2d_with_indices(T[i]["y"], [3, 3], [2, 2], [1, 1])

    def chain_bwd(i):
        t = T[i]
        gsum = torch.add(t["g1"], t["g2"])
        dy = torch.ops.aten.max_pool2d_with_indices_backward(gsum, t["y"], [3, 3], [2, 2], [1, 1], [1, 1], False,
                                                              t["pool"][1])
        cu.bn_act_bwd(dy.data_ptr(), t["x"].data_ptr(), t["mask"].data_ptr(), code, m, c, mean.data_ptr(),
                      inv.data_ptr(), wt.data_ptr(), dw.data_ptr(), db.data_ptr(), t["dx"].data_ptr(), 0,
                      ws.data_ptr(), zeroed(), s)

    def pooled_fwd(i):
        t = T[i]
        cu.bn_act_fwd_pool(t["x"].data_ptr(), code, args.batch, h, w, c, 1e-5, 0.1, rm.data_ptr(), rv.data_ptr(),
                           mean.data_ptr(), inv.data_ptr(), wt.data_ptr(), bs.data_ptr(), t["pooled"].data_ptr(),
                           t["code"].data_ptr(), ws.data_ptr(), zeroed(), s)

    def pooled_bwd(i):
        t = T[i]
        cu.bn_act_bwd_pool(t["g1"].data_ptr(), t["g2"].data_ptr(), t["code"].data_ptr(), t["x"].data_ptr(), code,
                           args.batch, h, w, c, mean.data_ptr(), inv.data_ptr(), wt.data_ptr(), dw.data_ptr(),
                           db.data_ptr(), t["dx"].data_ptr(), ws.data_ptr(), zeroed(), s)

    def run(fn):
        launch[0] = 0
        ctrs.zero_()
        return timed(fn, k)

    for i in range(k):   # the chain's indices and the pooled codes the backward rows read
        chain_fwd(i)
        pooled_fwd(i)
    torch.cuda.synchronize()
    least_f, least_b = m * c * e + p * c * (e + 0.5), 2 * m * c * e + p * c * (2 * e + 0.5)
    pool_f = m * c * e + p * c * (e + 8)                     # torch's max pool: read y; write the output, indices
    pool_b = p * c * (e + 8) + m * c * e + 3 * p * c * e      # its backward and the add of the two gradients
    out = []
    for impl, kind, fn, moved, least in (
            ("chain", "fwd", chain_fwd, fplan["bytes_moved"] + pool_f, least_f),
            ("chain", "bwd", chain_bwd, bplan["bytes_moved"] + pool_b, least_b),
            ("pooled", "fwd", pooled_fwd, pf["bytes_moved"], least_f),
            ("pooled", "bwd", pooled_bwd, pb["bytes_moved"], least_b)):
        us = run(fn) * 1e3
        out.append(dict(shape=[c, h, w], variant="relu_pool", impl=impl, kind=kind, us=us, bytes=least,
                        bytes_moved=moved, gbs=least / (us * 1e3), peak_share=least / (us * 1e3) / PEAK_GBS))
    print("stem %dx%dx%d, batch %d: ReLU, max pool 3 / 2 / 1 and the pooled junction (least MB: forward %.1f, "
          "backward %.1f)" % (c, h, w, args.batch, least_f / 1e6, least_b / 1e6))
    print("%-12s %9s %9s %9s %7s" % ("pass", "us", "moved MB", "least MB", "%peak"))
    for r_ in out:
        print("%-12s %9.1f %9.1f %9.1f %6.0f%%" % (r_["impl"] + ":" + r_["kind"], r_["us"], r_["bytes_moved"] / 1e6,
                                                  r_["bytes"] / 1e6, 100 * r_["peak_share"]))
    us = {(r_["impl"], r_["kind"]): r_["us"] for r_ in out}
    print("stem: chain -> pooled saves %.0f us per step" % (
        us[("chain", "fwd")] + us[("chain", "bwd")] - us[("pooled", "fwd")] - us[("pooled", "bwd")]))
    return out


if __name__ == "__main__":
    main()
