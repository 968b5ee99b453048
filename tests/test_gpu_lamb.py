"""LAMB in the fused exchange on one H100: the three kernels of pushpull_lamb.cu on virtual ranks (`VirtualCluster`)
against a float64 reference, and DistributedOptimizer(Lamb(...), fused_update=True) through the public API.

The kernel checks are exact where the design makes them exact (replicas and runs bit for bit, parameter windows
equal to the rounded masters, nothing outside the kernels' windows and shards written, a skipped step writes nothing)
and within a rounding bound derived below where fp32 arithmetic enters (masters and moments)."""
import struct

import pytest
import torch
from _fused_opt import _CANARY, _FUSED_BUCKETS, DT, _bits, _code, _cu, _fused_grad, _guarded, dt_id
from _lamb import _advance

pytestmark = pytest.mark.gpu

PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("f16", "f16"), ("f32", "bf16"), ("f32", "f16")]
WORLDS = (1, 2, 3, 5, 8)
_G = torch.Generator().manual_seed(11)
# Buckets as lists of parameter lengths (each parameter starts 8-element aligned):
#   fused     the fused Adam test's buckets; at world 8 ranks 3..7 own an empty shard of the first one
#   odd200    one bucket of 200 parameters of odd lengths 1..777 (a warp's 32 units cross many parameters)
#   straddle  one parameter that crosses every shard boundary, between two small ones
LAYOUTS = {
    "fused": _FUSED_BUCKETS,
    "odd200": [(torch.randint(0, 389, (200,), generator=_G) * 2 + 1).tolist()],
    "straddle": [[13, 40001, 7]],
}
# per bucket (weight_decay, adapt); the last bucket of a layout takes the adapt=False group
_GROUPS = [(0.01, 1), (0.0, 1), (0.0, 0)]
_KW = dict(lr=0.01, betas=(0.9, 0.99), eps=1e-6)


def _pad8(n):
    return (n + 7) // 8 * 8


def _hp(lr, wd, b1, b2, eps, t, gs, adapt, skip=0):
    """OptHParams of one LAMB step (as BucketedGradSync.refresh_hparams packs it)."""
    return struct.pack("<9f3if3i", lr, wd, 0.0, 0.0, b1, b2, eps, 1 - b1 ** t, 1 - b2 ** t, 0, 0, int(t == 1), gs,
                       skip, adapt, 0)


def _group_of(bi, nb):
    return _GROUPS[2] if bi == nb - 1 and nb > 1 else _GROUPS[bi % 2]


def _run_lamb(world, gname, wname, layout, skip_last=True, check=True):
    """4 steps of the LAMB sequence on virtual ranks (plus a skipped fifth); returns every rank's final state."""
    from byteps_b200.comm.symm import VirtualCluster

    from byteps_b200.torch import Lamb

    cu = _cu()
    gdt, wdt = DT[gname], DT[wname]
    ges, wes = torch.empty((), dtype=gdt).element_size(), torch.empty((), dtype=wdt).element_size()
    buckets = LAYOUTS[layout]
    nb = len(buckets)
    starts = [[sum(_pad8(s) for s in segs[:j]) for j in range(len(segs))] for segs in buckets]
    sizes = [sum(_pad8(s) for s in segs) for segs in buckets]
    scale, blocks = 1.0 / world, 3
    pack = gdt != wdt

    end = 256

    def window(nbytes):
        nonlocal end
        start = end
        end = (start + nbytes + 255) // 256 * 256 + 256
        return start

    goffs = [window(n * wes) for n in sizes]       # gradients in the arena, or the staging window of a wire cast
    poffs = [window(n * ges) for n in sizes]
    loffs = [window(cu.lamb_window_bytes(len(segs), world)) for segs in buckets]
    vc = VirtualCluster(world, "cuda:0", end)
    written = torch.zeros(vc.arenas[0].numel(), dtype=torch.bool, device="cuda")
    for i, n in enumerate(sizes):
        written[poffs[i]:poffs[i] + n * ges] = True
        written[loffs[i]:loffs[i] + cu.lamb_window_bytes(len(buckets[i]), world)] = True
        if pack:
            written[goffs[i]:goffs[i] + n * wes] = True

    torch.manual_seed(7)
    w0 = [torch.randn(n, device="cuda").to(gdt) for n in sizes]
    zero_param = layout == "odd200"
    if zero_param:
        w0[0][starts[0][3]:starts[0][3] + buckets[0][3]] = 0          # all-zero parameter: phi = 1
    # Padding starts at zero, as in the bucket layer.  Its gradients are not zero here: the padding's master then
    # moves, and a norm that counted it would be off.  The comparisons skip it.
    real = [torch.zeros(n, dtype=torch.bool, device="cuda") for n in sizes]
    for i, segs in enumerate(buckets):
        for st, s in zip(starts[i], segs):
            w0[i][st + s:st + _pad8(s)] = 0
            real[i][st:st + s] = True
    ref_params = [[torch.nn.Parameter(w0[i][st:st + s].double()) for st, s in zip(starts[i], segs)]
                  for i, segs in enumerate(buckets)]
    ref = Lamb([dict(params=ps, weight_decay=_group_of(i, nb)[0], adapt=bool(_group_of(i, nb)[1]))
                for i, ps in enumerate(ref_params)], **_KW)
    b1, b2 = _KW["betas"]
    tables = [torch.tensor([[st, s] for st, s in zip(starts[i], segs)], dtype=torch.int64, device="cuda")
              for i, segs in enumerate(buckets)]
    nmax = max(len(segs) for segs in buckets)
    shard = [[cu.shard_units(n // 8, world, r) for n in sizes] for r in range(world)]
    lens = [[(e - b) * 8 for b, e in shard[r]] for r in range(world)]
    smax = max(max(x) for x in lens)
    scratch = [torch.zeros(cu.lamb_scratch_bytes(smax, nmax) // 8, dtype=torch.float64, device="cuda")
               for _ in range(world)]
    phis = [torch.ones(nmax, dtype=torch.float32, device="cuda") for _ in range(world)]
    bufs = []
    for r in range(world):
        vc.arenas[r].fill_(_CANARY)
        bufs.append([])
        for i, n in enumerate(sizes):
            b, e = shard[r][i]
            bufs[r].append([_guarded(lens[r][i], w0[i][b * 8:e * 8].float()), _guarded(lens[r][i], 0.0),
                            _guarded(lens[r][i], 0.0)])
            vc.arenas[r][poffs[i]:poffs[i] + n * ges].view(gdt).copy_(w0[i])
    hp_dev = torch.zeros((nb, 64), dtype=torch.uint8, device="cuda")
    zeros = lambda: [torch.zeros(n, dtype=torch.float64, device="cuda") for n in sizes]  # noqa: E731
    bounds = [{k: z for k, z in zip(("w", "m", "mmag", "v", "vmag"), zs)} for zs in zip(*[zeros() for _ in range(5)])]
    steps = 5 if skip_last else 4
    for t in range(1, steps + 1):
        skip = int(t == 5)
        if t == 3:
            for g in ref.param_groups:
                g["lr"] *= 0.5
        lr = ref.param_groups[0]["lr"]
        loss_scale = 128.0 if t % 2 == 0 else 1.0
        grads = [[_fused_grad(n, loss_scale).to(gdt) for n in sizes] for _ in range(world)]
        if zero_param:
            for r in range(world):                                   # a parameter whose gradient is zero
                grads[r][0][starts[0][5]:starts[0][5] + buckets[0][5]] = 0
        users = []
        for r in range(world):
            if pack:
                users.append([g.clone() for g in grads[r]])
            else:
                for i, n in enumerate(sizes):
                    vc.arenas[r][goffs[i]:goffs[i] + n * wes].view(wdt).copy_(grads[r][i])
        segtabs = [[torch.tensor([[u.data_ptr(), u.data_ptr(), 0, u.numel()]], dtype=torch.int64, device="cuda")
                    for u in users[r]] for r in range(world)] if pack else None
        blob = b"".join(_hp(lr, _group_of(i, nb)[0], b1, b2, _KW["eps"], t - skip, 1.0 / loss_scale,
                            _group_of(i, nb)[1], skip) for i in range(nb))
        cu.write_blob(hp_dev.data_ptr(), blob, torch.cuda.current_stream().cuda_stream)
        snap = [a.clone() for a in vc.arenas]
        state_snap = [[[x[0].clone() for x in bb] for bb in bufs[r]] for r in range(world)]

        def launch(r, view, arena, s):
            for i, n in enumerate(sizes):
                m, s0, s1 = (x[0].data_ptr() for x in bufs[r][i])
                hp = hp_dev[i].data_ptr()
                segs, nsegs = (segtabs[r][i].data_ptr(), 1) if pack else (0, 0)
                np_ = len(buckets[i])
                cu.lamb_moments(view, _code(gdt), _code(wdt), segs, nsegs, goffs[i], n, scale, m, s0, s1,
                                tables[i].data_ptr(), np_, scratch[r].data_ptr(), hp, blocks, 512, 0, False, s)
                cu.lamb_norms(view, _code(wdt), n, tables[i].data_ptr(), np_, scratch[r].data_ptr(), loffs[i],
                              phis[r].data_ptr(), hp, min(np_, 32), 0, s)
                cu.lamb_apply(view, _code(gdt), _code(wdt), poffs[i], n, m, s0, s1, tables[i].data_ptr(), np_,
                              phis[r].data_ptr(), hp, blocks, 512, 0, False, s)

        vc.run(launch)
        torch.cuda.synchronize()
        if skip:
            for r in range(world):
                for i in range(nb):
                    for which, (buf, _), old in zip(("master", "m", "v"), bufs[r][i], state_snap[r][i]):
                        assert torch.equal(_bits(buf), _bits(old)), ("skipped step wrote", which, r, i)
                for i, n in enumerate(sizes):
                    win = slice(poffs[i], poffs[i] + n * ges)
                    assert torch.equal(vc.arenas[r][win], snap[r][win]), ("skipped step wrote parameters", r, i)
            break
        if not check:
            continue
        for i, ps in enumerate(ref_params):
            for p, st, s in zip(ps, starts[i], buckets[i]):
                p.grad = (torch.stack([grads[r][i][st:st + s].to(wdt).double() for r in range(world)]).sum(0)
                          * scale / loss_scale)
        w_prev = [torch.cat([torch.cat([p.detach(), p.new_zeros(_pad8(p.numel()) - p.numel())]) for p in ps])
                  for ps in ref_params]
        w_norm = [[p.detach().norm() for p in ps] for ps in ref_params]
        ref.step()
        for i, ps in enumerate(ref_params):
            wd, adapt = _group_of(i, nb)
            pad = lambda x, n: torch.cat([x, x.new_zeros(_pad8(n) - n)])  # noqa: E731
            g = torch.cat([pad(p.grad, p.numel()) for p in ps])
            st_ = {k: torch.cat([pad(ref.state[p][k], p.numel()) for p in ps]) for k in ("exp_avg", "exp_avg_sq")}
            c1, c2 = 1 - b1 ** t, 1 - b2 ** t
            u_ref = (st_["exp_avg"] / c1) / ((st_["exp_avg_sq"] / c2).sqrt() + _KW["eps"]) + wd * w_prev[i]
            slices = [(s0, s0 + _pad8(p.numel())) for s0, p in zip(starts[i], ps)]
            _advance(bounds[i], g, w_prev[i], st_, lr, wd, b1, b2, _KW["eps"], t, adapt, w_norm[i], u_ref, slices)
        for r in range(world):
            changed = (vc.arenas[r] != snap[r]) & ~written
            assert not changed.any(), ("bytes outside the kernels' windows changed", r,
                                       changed.nonzero()[:8].flatten().tolist())
            for i in range(nb):
                for which, (buf, used) in zip(("master", "m", "v"), bufs[r][i]):
                    assert bool((buf[used:].view(torch.int32) == -1).all()), (which, "canary overwritten", r, i)
        for i, n in enumerate(sizes):
            win = [vc.arenas[r][poffs[i]:poffs[i] + n * ges].view(gdt) for r in range(world)]
            for r in range(1, world):
                assert torch.equal(_bits(win[r]), _bits(win[0])), ("replicas must be bit-identical", t, r, i)
            cat = lambda k: torch.cat([bufs[r][i][k][0][:lens[r][i]] for r in range(world)])  # noqa: E731
            master = cat(0)
            assert torch.equal(_bits(win[0]), _bits(master.to(gdt))), ("window != round(master)", t, i)
            want_w = torch.cat([torch.cat([p.detach(), p.new_zeros(_pad8(p.numel()) - p.numel())])
                                for p in ref_params[i]])
            want = {k: torch.cat([torch.cat([ref.state[p][k], p.new_zeros(_pad8(p.numel()) - p.numel())])
                                  for p in ref_params[i]]) for k in ("exp_avg", "exp_avg_sq")}
            for name, got, ref_v, bound in (("master", master, want_w, bounds[i]["w"]),
                                            ("exp_avg", cat(1), want["exp_avg"], bounds[i]["m"]),
                                            ("exp_avg_sq", cat(2), want["exp_avg_sq"], bounds[i]["v"])):
                err = (got.double() - ref_v).abs()
                bad = (err > 2 * bound) & real[i]
                assert not bad.any(), (name, t, i, int(bad.sum()), err.max().item(),
                                       (err / bound.clamp_min(1e-300)).max().item())
    return [[[x[0].clone() for x in bb] for bb in bufs[r]] for r in range(world)]


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("dtypes", PAIRS, ids=dt_id)
@pytest.mark.parametrize("world", WORLDS)
def test_lamb_kernels_virtual(world, dtypes, layout):
    """Four steps and a skipped fifth against the float64 Lamb, bounds derived in _advance."""
    _run_lamb(world, *dtypes, layout)


@pytest.mark.parametrize("dtypes", [("bf16", "bf16"), ("f32", "f16")], ids=dt_id)
def test_lamb_kernels_reproducible(dtypes):
    """Two runs of the same steps leave the same bits in every rank's master and moments."""
    a = _run_lamb(5, *dtypes, "odd200", skip_last=False, check=False)
    b = _run_lamb(5, *dtypes, "odd200", skip_last=False, check=False)
    for r, (ra, rb) in enumerate(zip(a, b)):
        for i, (ba, bb) in enumerate(zip(ra, rb)):
            for k, (x, y) in enumerate(zip(ba, bb)):
                assert torch.equal(_bits(x), _bits(y)), ("run-to-run bits differ", r, i, k)
