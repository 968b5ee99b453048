"""Fused optimizer exchange kernels against torch.optim in float64 (shared by test_gpu_kernels.py, which runs the
register and TMA-streamed kernels, and test_gpu_ring.py, which runs the descriptor-ring kernel).

`check_fused_optimizer` runs N virtual ranks on one GPU (`VirtualCluster`), as the other kernel tests do.
"""
import struct

import torch

DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}


def _cu():
    from byteps_b200 import _native

    return _native.cuda()


def _code(dt):
    from byteps_b200.comm.symm import wire_code

    return wire_code(dt)


def _hp(lr=0.1, wd=0.0, mom=0.0, damp=0.0, b1=0.9, b2=0.999, eps=1e-8, t=1, nesterov=0, adamw=0, first=1, gs=1.0):
    return struct.pack("<9f3if3i", lr, wd, mom, damp, b1, b2, eps, 1 - b1 ** t, 1 - b2 ** t, nesterov, adamw, first,
                       gs, 0, 0, 0)


# engine -> (gradient dtype, wire dtype) pairs: what parallel/bucket.py launches it with.  The parameter dtype is the
# gradient dtype.  "lsu" is the register kernel on gradients in the arena; "pack" is the same kernel with a segment
# table: it gathers the user gradients, casts them to the wire dtype into a staging window and reduces from there
# (every wire cast takes this path); "tma" streams the optimizer state through shared memory; "ring" is the
# descriptor-ring kernel with RING_SGD / RING_ADAM descriptors.
_SAME = [("f32", "f32"), ("bf16", "bf16"), ("f16", "f16")]
ENGINE_DTYPES = {"lsu": _SAME, "pack": [("f32", "bf16"), ("f32", "f16")], "tma": _SAME, "ring": _SAME}
# The optimizers, by the names the test ids use.  "sgd" keeps momentum 0.9 and weight decay 0.01 and adds dampening.
FUSED_OPTS = {
    "sgd_plain": (torch.optim.SGD, dict(lr=0.1)),
    "sgd": (torch.optim.SGD, dict(lr=0.1, momentum=0.9, dampening=0.1, weight_decay=0.01)),
    "sgd_nesterov": (torch.optim.SGD, dict(lr=0.1, momentum=0.9, nesterov=True, weight_decay=0.01)),
    "adam": (torch.optim.Adam, dict(lr=0.01, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.01)),
    "adamw": (torch.optim.AdamW, dict(lr=0.01, weight_decay=0.01)),
}


def fused_cases(dtypes):
    """(world, (grad, wire), optimizer) cases for one engine: every optimizer at worlds 1 and 3, the cases the earlier
    fp32-tolerance tests ran at world 4 (f32/bf16 with sgd, sgd_nesterov, adam, adamw), and world 8 (ranks 3..7 own an
    empty shard of the 8*3 bucket) with plain SGD, momentum SGD and Adam."""
    out = [(w, d, o) for w in (1, 3) for d in dtypes for o in FUSED_OPTS]
    out += [(4, d, o) for d in dtypes if d[0] == d[1] and d[0] in ("f32", "bf16")
            for o in ("sgd", "sgd_nesterov", "adam", "adamw")]
    out += [(8, d, o) for d in dtypes for o in ("sgd_plain", "sgd", "adam")]
    return out


def dt_id(d):
    return d[0] if d[0] == d[1] else "%s_%s" % d


# Buckets as lists of user-tensor lengths, each tensor starting 8-element aligned inside the bucket:
# 8*3 elements (ranks 3..7 of 8 own an empty shard), 8*5003 (several tiles per CTA, ragged tail), 8*41.
_FUSED_BUCKETS = [[5, 11], [16003, 24013], [200, 128]]
_U = 2.0 ** -24          # unit roundoff of fp32
_CANARY = 0xFF           # all-ones bytes are a NaN in fp32, bf16 and fp16


def _bits(x):
    return x.view(torch.int32 if x.element_size() == 4 else torch.int16)


def _guarded(n, init=None):
    """fp32 buffer of max(n, 8) elements plus 256 canary bytes (all canary when init is None: a buffer the
    optimizer has no use for).  Returns (buffer, number of leading elements the kernel may write)."""
    buf = torch.full((max(n, 8) + 64,), -1, dtype=torch.int32, device="cuda").view(torch.float32)
    if init is None:
        return buf, 0
    buf[:n] = init
    return buf, n


def _opt_blob(kind, adamw, g, t, grad_scale):
    """The 64-byte hyper-parameter block of step t, from a torch param group (as BucketedGradSync.refresh_hparams)."""
    if kind == "sgd":
        return _hp(lr=g["lr"], wd=g["weight_decay"], mom=g["momentum"], damp=g["dampening"],
                   nesterov=int(g["nesterov"]), first=int(t == 1), gs=grad_scale)
    b1, b2 = g["betas"]
    return _hp(lr=g["lr"], wd=g["weight_decay"], b1=b1, b2=b2, eps=g["eps"], t=t, adamw=int(adamw),
               first=int(t == 1), gs=grad_scale)


def _advance_bounds(kind, adamw, g, t, e, grad, w_prev, w_new, st):
    """Advance the elementwise bounds on |fp32 kernel - float64 reference| by step t.

    Each fp32 operation rounds to within u*|result|, and |result| <= the sum of the magnitudes of its terms.  `e`
    carries those magnitudes ("*mag": the value with every term taken positive, so cancellation cannot hide a
    rounding) and the bounds on each state's error.  The summed gradient itself is exact (see _fused_grad), so
    its error is the rounding of scale * grad_scale and of the product with it.  Errors of the master feed back
    through the weight decay."""
    lr, wd = g["lr"], g["weight_decay"]
    decay_in_grad = kind == "sgd" or not adamw
    gmag = grad.abs() + (wd * w_prev.abs() if decay_in_grad else 0.0)
    eg = 4 * _U * gmag + (wd * e["w"] if decay_in_grad else 0.0)
    extra = 0.0
    if kind == "sgd":
        mu, damp = g["momentum"], g["dampening"]
        if mu:
            e["bmag"] = gmag if t == 1 else mu * e["bmag"] + (1 - damp) * gmag
            e["b"] = eg + 4 * _U * e["bmag"] if t == 1 else mu * e["b"] + (1 - damp) * eg + 4 * _U * e["bmag"]
            if g["nesterov"]:
                dmag, ed = gmag + mu * e["bmag"], eg + mu * e["b"]
            else:
                dmag, ed = e["bmag"], e["b"]
        else:
            dmag, ed = gmag, eg
        step = lr * dmag
        eu = lr * ed
    else:
        b1, b2 = g["betas"]
        c1, c2 = 1 - b1 ** t, 1 - b2 ** t
        # the kernel forms 1 - beta from the fp32 beta: off by up to u * beta, i.e. ~1000 ulp of 1 - 0.999
        e["mmag"] = b1 * e["mmag"] + (1 - b1) * gmag
        e["m"] = b1 * e["m"] + (1 - b1) * eg + 4 * _U * e["mmag"] + _U * b1 * gmag
        e["vmag"] = b2 * e["vmag"] + (1 - b2) * gmag * gmag
        e["v"] = b2 * e["v"] + (1 - b2) * (2 * gmag * eg + eg * eg) + 5 * _U * e["vmag"] + _U * b2 * gmag * gmag
        sv = (st["exp_avg_sq"] / c2).sqrt()
        den = sv + g["eps"]
        step = lr * (st["exp_avg"] / c1).abs() / den
        # sqrt of a perturbed v (first order, or sqrt(dv) near v = 0), plus sqrt.approx (<= 2 ulp)
        esqrt = torch.minimum(e["v"] / c2 / (2 * sv).clamp_min(1e-300), (e["v"] / c2).sqrt()) + 4 * _U * sv
        # m error through the division; the denominator error; 1/c1, 1/c2, lr*m and __fdividef (<= 2 ulp)
        eu = lr / c1 * e["m"] / den + step * ((esqrt + _U * den) / den + 8 * _U)
        if adamw:
            extra = 3 * _U * w_prev.abs()          # w *= fl(1 - lr*wd)
    e["w"] = e["w"] + eu + extra + 4 * _U * (w_new.abs() + step)


def _fused_grad(n, loss_scale):
    """A gradient in fp32 whose values are multiples of 2^-10 * loss_scale below 8 * loss_scale.  Any of these rounded
    to bf16/fp16 is still such a multiple, so sums over up to 8 ranks are exact in fp32 and the only differences to
    the float64 reference are the optimizer's own roundings."""
    return (torch.randn(n, device="cuda") * 1024).round().clamp(-8191, 8191) * (loss_scale / 1024)


def check_fused_optimizer(world, eng, gname, wname, opt):
    """Fused exchange + SGD/Adam(W) step, 4 steps on 3 buckets, against torch.optim on float64 parameters fed
    sum_r g_r.to(wire) * scale * grad_scale.  Exact: replicas bit-identical, every parameter window equals the
    concatenated fp32 master shards rounded to the parameter dtype, the staging window holds the user gradients
    rounded to the wire dtype, and no byte outside the windows and shards the kernel owns changes (gradients,
    canaries around every window, after every master/state shard, unused state buffers).  Within fp32 rounding
    bounds: masters, momentum and Adam moments.  lr changes before step 3, the loss scale between steps."""
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops.ring import RingEntry, RingTable

    cu = _cu()
    gdt, wdt = DT[gname], DT[wname]
    ges, wes = torch.empty((), dtype=gdt).element_size(), torch.empty((), dtype=wdt).element_size()
    cls, kw = FUSED_OPTS[opt]
    kind = "sgd" if cls is torch.optim.SGD else "adam"
    adamw = cls is torch.optim.AdamW
    scale, blocks = 1.0 / world, 3
    seg_starts = [[sum((s + 7) // 8 * 8 for s in segs[:j]) for j in range(len(segs))] for segs in _FUSED_BUCKETS]
    sizes = [sum((s + 7) // 8 * 8 for s in segs) for segs in _FUSED_BUCKETS]

    # arena layout (the same on every rank): 256-byte aligned windows with >= 256 canary bytes between them
    end = 256

    def window(nbytes):
        nonlocal end
        start = end
        end = (start + nbytes + 255) // 256 * 256 + 256
        return start

    goffs = [window(n * wes) for n in sizes]      # gradients in the arena; "pack": the staging window
    poffs = [window(n * ges) for n in sizes]
    vc = VirtualCluster(world, "cuda:0", end)
    written = torch.zeros(vc.arenas[0].numel(), dtype=torch.bool, device="cuda")
    for i, n in enumerate(sizes):
        written[poffs[i]:poffs[i] + n * ges] = True
        if eng == "pack":
            written[goffs[i]:goffs[i] + n * wes] = True

    torch.manual_seed(5)
    w0 = [torch.randn(n, device="cuda").to(gdt) for n in sizes]
    ref_w = [torch.nn.Parameter(w.double()) for w in w0]
    ref_opt = cls(ref_w, **kw)
    grp = ref_opt.param_groups[0]
    uses_mom = kind == "adam" or grp["momentum"] != 0
    shard = [[cu.shard_units(n // 8, world, r) for n in sizes] for r in range(world)]
    lens = [[(e - b) * 8 for b, e in shard[r]] for r in range(world)]
    bufs = []       # [rank][bucket] -> [(master), (state0), (state1)] as (buffer, written prefix)
    for r in range(world):
        vc.arenas[r].fill_(_CANARY)
        bufs.append([])
        for i, n in enumerate(sizes):
            b, e = shard[r][i]
            bufs[r].append([_guarded(lens[r][i], w0[i][b * 8:e * 8].float()),
                            _guarded(lens[r][i], 0.0) if uses_mom else _guarded(lens[r][i]),
                            _guarded(lens[r][i], 0.0) if kind == "adam" else _guarded(lens[r][i])])
            vc.arenas[r][poffs[i]:poffs[i] + n * ges].view(gdt).copy_(w0[i])
    hp_dev = torch.zeros(64, dtype=torch.uint8, device="cuda")
    code = cu.OPT_SGD if kind == "sgd" else cu.OPT_ADAM
    if eng == "ring":
        rkind = cu.RING_SGD if kind == "sgd" else cu.RING_ADAM
        tables = [RingTable([RingEntry(grad_off=goffs[i], param_off=poffs[i], numel=n, wire=_code(wdt), slot=i,
                                       kind=rkind, scale=scale, master=bufs[r][i][0][0].data_ptr(),
                                       state0=bufs[r][i][1][0].data_ptr(), state1=bufs[r][i][2][0].data_ptr(),
                                       hp=hp_dev.data_ptr()) for i, n in enumerate(sizes)], "cuda:0")
                  for r in range(world)]
    zeros = lambda: [torch.zeros(n, dtype=torch.float64, device="cuda") for n in sizes]  # noqa: E731
    bounds = [{k: z for k, z in zip(("w", "b", "bmag", "m", "mmag", "v", "vmag"), zs)}
              for zs in zip(*[zeros() for _ in range(7)])]

    for t in range(1, 5):
        if t == 3:
            grp["lr"] *= 0.5
        loss_scale = 128.0 if t % 2 == 0 else 1.0
        grads = [[_fused_grad(n, loss_scale).to(gdt) for n in sizes] for _ in range(world)]
        if eng == "pack":
            # user tensors: the bucket's segments, separate allocations; the second one of each bucket starts one
            # element past a 16-byte boundary (element-wise gather)
            users, seg_tabs = [], []
            for r in range(world):
                users.append([])
                seg_tabs.append([])
                for i, segs in enumerate(_FUSED_BUCKETS):
                    gapless = torch.zeros(sizes[i], dtype=gdt, device="cuda")
                    rows = []
                    for j, (s, st0) in enumerate(zip(segs, seg_starts[i])):
                        base = torch.empty(s + j, dtype=gdt, device="cuda")
                        base[j:].copy_(grads[r][i][st0:st0 + s])
                        gapless[st0:st0 + s] = grads[r][i][st0:st0 + s]
                        users[r].append((base, base.clone()))
                        ptr = base[j:].data_ptr()
                        rows.append([ptr, ptr, st0, s])
                    grads[r][i] = gapless
                    seg_tabs[r].append(torch.tensor(rows, dtype=torch.int64, device="cuda"))
        else:
            for r in range(world):
                for i, n in enumerate(sizes):
                    vc.arenas[r][goffs[i]:goffs[i] + n * wes].view(wdt).copy_(grads[r][i])
        cu.write_blob(hp_dev.data_ptr(), _opt_blob(kind, adamw, grp, t, 1.0 / loss_scale),
                      torch.cuda.current_stream().cuda_stream)
        snap = [a.clone() for a in vc.arenas]
        stages = 2 if t % 2 else 8        # TMA state ring: shallowest and deepest

        def launch(r, view, arena, s):
            if eng == "ring":
                tables[r].launch(view, blocks, s)
                return
            for i, n in enumerate(sizes):
                m, s0, s1 = (x[0].data_ptr() for x in bufs[r][i])
                if eng == "tma":
                    cu.pushpull_fused_opt_tma(view, _code(wdt), code, goffs[i], poffs[i], n, scale, m, s0, s1,
                                              hp_dev.data_ptr(), blocks, stages, False, 0, s)
                else:
                    segs, nsegs = ((seg_tabs[r][i].data_ptr(), len(_FUSED_BUCKETS[i])) if eng == "pack" else (0, 0))
                    cu.pushpull_fused_opt(view, _code(gdt), _code(wdt), _code(gdt), code, segs, nsegs, goffs[i],
                                          poffs[i], n, scale, m, s0, s1, hp_dev.data_ptr(), blocks, 256, 0, False, s)

        vc.run(launch)
        torch.cuda.synchronize()

        w_prev = [p.detach().clone() for p in ref_w]
        for i, p in enumerate(ref_w):
            p.grad = torch.stack([grads[r][i].to(wdt).double() for r in range(world)]).sum(0) * scale / loss_scale
        ref_opt.step()
        for i, p in enumerate(ref_w):
            _advance_bounds(kind, adamw, grp, t, bounds[i], p.grad, w_prev[i], p.detach(), ref_opt.state[p])

        for r in range(world):
            changed = (vc.arenas[r] != snap[r]) & ~written
            assert not changed.any(), ("bytes outside the parameter/staging windows changed", r,
                                       changed.nonzero()[:8].flatten().tolist())
            for i in range(len(sizes)):
                for which, (buf, used) in zip(("master", "state0", "state1"), bufs[r][i]):
                    assert bool((buf[used:].view(torch.int32) == -1).all()), (which, "canary overwritten", r, i)
            if eng == "pack":
                for base, keep in users[r]:
                    assert torch.equal(_bits(base), _bits(keep)), "user gradients must only be read"
                for i, n in enumerate(sizes):
                    stage = vc.arenas[r][goffs[i]:goffs[i] + n * wes].view(wdt)
                    assert torch.equal(_bits(stage), _bits(grads[r][i].to(wdt))), ("staging window", r, i)
        for i, n in enumerate(sizes):
            win = [vc.arenas[r][poffs[i]:poffs[i] + n * ges].view(gdt) for r in range(world)]
            for r in range(1, world):
                assert torch.equal(_bits(win[r]), _bits(win[0])), ("replicas must be bit-identical", t, r, i)
            cat = lambda k: torch.cat([bufs[r][i][k][0][:lens[r][i]] for r in range(world)])  # noqa: E731
            master = cat(0)
            assert torch.equal(_bits(win[0]), _bits(master.to(gdt))), ("window != round(master)", t, i)
            # fp32 rounding bounds (see _advance_bounds), with a factor 2 for the first-order terms
            checks = [("master", master, ref_w[i].detach(), bounds[i]["w"])]
            st = ref_opt.state[ref_w[i]]
            if kind == "sgd" and uses_mom:
                checks.append(("momentum", cat(1), st["momentum_buffer"], bounds[i]["b"]))
            if kind == "adam":
                checks += [("exp_avg", cat(1), st["exp_avg"], bounds[i]["m"]),
                           ("exp_avg_sq", cat(2), st["exp_avg_sq"], bounds[i]["v"])]
            for name, got, want, bound in checks:
                err = (got.double() - want).abs()
                bad = err > 2 * bound
                assert not bad.any(), (name, t, i, int(bad.sum()), err.max().item(), (err / bound).max().item())
