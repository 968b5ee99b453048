#!/usr/bin/env python
"""Single-GPU roofline check of our memory-bound kernels (also the ncu target).

world=1 variants of the fused kernels stream HBM only, so achieved bytes/time is
compared with the measured copy bandwidth in MEASURED_PEAKS.json.
"""
import argparse
import json
import os
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=512, help="gradient window size in MB (bf16)")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    ap.add_argument("--sweep-blocks", default="", help="comma list: also time the fused Adam kernels at these grid sizes")
    args = ap.parse_args()
    from byteps_b200 import _native
    from byteps_b200.comm.symm import VirtualCluster

    cu = _native.cuda()
    torch.cuda.set_device(0)
    n = args.mb * (1 << 20) // 2 // 8 * 8
    es = 2
    goff, poff = 0, (n * es + 255) // 256 * 256
    vc = VirtualCluster(1, "cuda:0", poff + n * es + 4096)
    view, arena = vc.views[0], vc.arenas[0]
    arena[goff:goff + n * es].view(torch.bfloat16).normal_()
    arena[poff:poff + n * es].view(torch.bfloat16).normal_()
    master = torch.randn(n, device="cuda")
    mom = torch.zeros(n, device="cuda")
    m2 = torch.zeros(n, device="cuda")
    hp = torch.zeros(64, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:  # noqa: BLE001
        pass
    hbm = peaks.get("hbm_gbs", 6650.0)
    fl = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []

    def timed(fn, bytes_moved, name):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        tot = 0.0
        for _ in range(args.iters):
            cu.l2_flush(fl.data_ptr(), fl.numel(), 1, s)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            tot += e0.elapsed_time(e1)
        ms = tot / args.iters
        gbs = bytes_moved / ms / 1e6
        rows.append({"kernel": name, "ms": ms, "algorithmic_bytes": bytes_moved, "gbs": gbs,
                     "frac_of_measured_hbm": gbs / hbm})
        print("%-34s %8.3f ms  %8.1f GB/s  %.2f of measured HBM copy (%.0f GB/s)" % (name, ms, gbs, gbs / hbm, hbm))

    blob = struct.pack("<9f3if3i", 0.01, 1e-4, 0.9, 0.0, 0.9, 0.999, 1e-8, 0.1, 0.001, 0, 0, 0, 1.0, 0, 0, 0)
    cu.write_blob(hp.data_ptr(), blob, s)
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    blocks = sms * 2
    # fused SGD+momentum: read g(2) + w(4) + m(4), write w(4) + m(4) + p(2) = 20 B/elem
    timed(lambda: cu.pushpull_fused_opt(view, 1, 1, 1, cu.OPT_SGD, 0, 0, goff, poff, n, 1.0, master.data_ptr(),
                                        mom.data_ptr(), 0, hp.data_ptr(), blocks, 512, 0, False, s),
          n * 20, "fused_opt_sgd_momentum_bf16")
    # fused Adam: read g(2)+w(4)+m(4)+v(4), write w(4)+m(4)+v(4)+p(2) = 28 B/elem
    timed(lambda: cu.pushpull_fused_opt(view, 1, 1, 1, cu.OPT_ADAM, 0, 0, goff, poff, n, 1.0, master.data_ptr(),
                                        mom.data_ptr(), m2.data_ptr(), hp.data_ptr(), blocks, 512, 0, False, s),
          n * 28, "fused_opt_adam_bf16")
    # same two optimizers with the state streamed through shared memory by bulk copies (TMA variant)
    timed(lambda: cu.pushpull_fused_opt_tma(view, 1, cu.OPT_SGD, goff, poff, n, 1.0, master.data_ptr(), mom.data_ptr(),
                                            0, hp.data_ptr(), blocks, 6, False, 0, s),
          n * 20, "fused_opt_tma_sgd_momentum_bf16")
    timed(lambda: cu.pushpull_fused_opt_tma(view, 1, cu.OPT_ADAM, goff, poff, n, 1.0, master.data_ptr(),
                                            mom.data_ptr(), m2.data_ptr(), hp.data_ptr(), blocks, 4, False, 0, s),
          n * 28, "fused_opt_tma_adam_bf16")
    for nb in [int(x) for x in args.sweep_blocks.split(",") if x]:
        timed(lambda: cu.pushpull_fused_opt_tma(view, 1, cu.OPT_ADAM, goff, poff, n, 1.0, master.data_ptr(),
                                                mom.data_ptr(), m2.data_ptr(), hp.data_ptr(), nb, 4, False, 0, s),
              n * 28, "fused_opt_tma_adam_bf16[blocks=%d,stages=4]" % nb)
        if nb <= sms:
            timed(lambda: cu.pushpull_fused_opt_tma(view, 1, cu.OPT_ADAM, goff, poff, n, 1.0, master.data_ptr(),
                                                    mom.data_ptr(), m2.data_ptr(), hp.data_ptr(), nb, 8, False, 0, s),
                  n * 28, "fused_opt_tma_adam_bf16[blocks=%d,stages=8]" % nb)
        timed(lambda: cu.pushpull_fused_opt(view, 1, 1, 1, cu.OPT_ADAM, 0, 0, goff, poff, n, 1.0, master.data_ptr(),
                                            mom.data_ptr(), m2.data_ptr(), hp.data_ptr(), nb, 512, 0, False, s),
              n * 28, "fused_opt_adam_bf16[blocks=%d]" % nb)
    # in-place scale (world 1): read 2 + write 2
    timed(lambda: cu.pushpull_inplace(view, 1, goff, n, 0.5, blocks, 512, 0, False, s), n * 4, "inplace_world1_bf16")
    # torch reference points
    a = arena[goff:goff + n * es].view(torch.bfloat16)
    b = arena[poff:poff + n * es].view(torch.bfloat16)
    timed(lambda: b.copy_(a), n * 4, "torch_copy_bf16")
    p32 = torch.nn.Parameter(master.clone())
    p32.grad = torch.randn_like(master)
    opt = torch.optim.SGD([p32], lr=0.01, momentum=0.9, weight_decay=1e-4, foreach=True)
    opt.step()
    timed(lambda: opt.step(), n * 20, "torch_sgd_momentum_fp32(20B/elem)")
    if args.out:
        json.dump({"hbm_gbs_measured": hbm, "rows": rows}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
