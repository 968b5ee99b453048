"""LARS in the fused exchange on one H100: the three kernels of pushpull_lars.cu on virtual ranks (`VirtualCluster`)
against the float64 Lars, on the layouts and (gradient, wire) pairs of test_gpu_lamb.py.

Exact where the design makes it exact: replicas and repeated runs bit for bit, parameter windows equal to the rounded
masters, nothing outside the kernels' windows and shards written, padding excluded from the norms (its gradients
are not zero here), and a skipped step writes no state, no window slot and no parameter.  Masters and momentum agree
with float64 within the bound of _lars.advance, which includes phi's relative error."""
import struct

import pytest
import torch
from _fused_opt import _CANARY, _bits, _code, _cu, _fused_grad, _guarded, DT, dt_id
from _lars import advance
from test_gpu_lamb import LAYOUTS, PAIRS, WORLDS

pytestmark = pytest.mark.gpu

# per bucket (weight_decay, adapt); the last bucket of a layout takes the adapt=False group
_GROUPS = [(0.01, 1), (0.0, 1), (0.0, 0)]
_KW = dict(lr=0.1, momentum=0.9, trust_coefficient=0.02, eps=1e-6)


def _pad8(n):
    return (n + 7) // 8 * 8


def _hp(lr, wd, mom, eps, gs, adapt, eta, skip=0):
    """OptHParams of one LARS step (as BucketedGradSync.refresh_hparams packs it)."""
    return struct.pack("<9f3if2if", lr, wd, mom, 0.0, 0.0, 0.0, eps, 1.0, 1.0, 0, 0, 0, gs, skip, adapt, eta)


def _group_of(bi, nb):
    return _GROUPS[2] if bi == nb - 1 and nb > 1 else _GROUPS[bi % 2]


def _run_lars(world, gname, wname, layout, skip_last=True, check=True):
    """4 steps of the LARS sequence on virtual ranks (plus a skipped fifth); returns every rank's final state."""
    from byteps_b200.comm.symm import VirtualCluster

    from byteps_b200.torch import Lars

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
    special = layout == "odd200"
    if special:
        w0[0][starts[0][3]:starts[0][3] + buckets[0][3]] = 0          # all-zero parameter: phi = 1 at first
    real = [torch.zeros(n, dtype=torch.bool, device="cuda") for n in sizes]
    for i, segs in enumerate(buckets):
        for st, s in zip(starts[i], segs):
            w0[i][st + s:st + _pad8(s)] = 0
            real[i][st:st + s] = True
    ref_params = [[torch.nn.Parameter(w0[i][st:st + s].double()) for st, s in zip(starts[i], segs)]
                  for i, segs in enumerate(buckets)]
    ref = Lars([dict(params=ps, weight_decay=_group_of(i, nb)[0], adapt=bool(_group_of(i, nb)[1]))
                for i, ps in enumerate(ref_params)], **_KW)
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
            bufs[r].append([_guarded(lens[r][i], w0[i][b * 8:e * 8].float()), _guarded(lens[r][i], 0.0)])
            vc.arenas[r][poffs[i]:poffs[i] + n * ges].view(gdt).copy_(w0[i])
    hp_dev = torch.zeros((nb, 64), dtype=torch.uint8, device="cuda")
    bounds = [{k: torch.zeros(n, dtype=torch.float64, device="cuda") for k in ("w", "v", "vmag")} for n in sizes]
    steps = 5 if skip_last else 4
    for t in range(1, steps + 1):
        skip = int(t == 5)
        if t == 3:
            for g in ref.param_groups:
                g["lr"] *= 0.5
        lr = ref.param_groups[0]["lr"]
        loss_scale = 128.0 if t % 2 == 0 else 1.0
        grads = [[_fused_grad(n, loss_scale).to(gdt) for n in sizes] for _ in range(world)]
        if special:
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
        blob = b"".join(_hp(lr, _group_of(i, nb)[0], _KW["momentum"], _KW["eps"], 1.0 / loss_scale,
                            _group_of(i, nb)[1], _KW["trust_coefficient"], skip) for i in range(nb))
        cu.write_blob(hp_dev.data_ptr(), blob, torch.cuda.current_stream().cuda_stream)
        snap = [a.clone() for a in vc.arenas]
        state_snap = [[[x[0].clone() for x in bb] for bb in bufs[r]] for r in range(world)]

        def launch(r, view, arena, s):
            for i, n in enumerate(sizes):
                m, v = (x[0].data_ptr() for x in bufs[r][i])
                hp = hp_dev[i].data_ptr()
                segs, nsegs = (segtabs[r][i].data_ptr(), 1) if pack else (0, 0)
                np_ = len(buckets[i])
                cu.lars_norms_partial(view, _code(gdt), _code(wdt), segs, nsegs, goffs[i], n, scale, m,
                                      tables[i].data_ptr(), np_, scratch[r].data_ptr(), hp, blocks, 512, 0, False, s)
                cu.lars_norms(view, _code(wdt), n, tables[i].data_ptr(), np_, scratch[r].data_ptr(), loffs[i],
                              phis[r].data_ptr(), hp, min(np_, 32), 0, s)
                cu.lars_apply(view, _code(gdt), _code(wdt), goffs[i], poffs[i], n, scale, m, v,
                              tables[i].data_ptr(), np_, phis[r].data_ptr(), hp, blocks, 512, 0, False, s)

        vc.run(launch)
        torch.cuda.synchronize()
        if skip:
            for r in range(world):
                for i in range(nb):
                    for which, (buf, _), old in zip(("master", "v"), bufs[r][i], state_snap[r][i]):
                        assert torch.equal(_bits(buf), _bits(old)), ("skipped step wrote", which, r, i)
                for i, n in enumerate(sizes):
                    for win in (slice(poffs[i], poffs[i] + n * ges),
                                slice(loffs[i], loffs[i] + cu.lamb_window_bytes(len(buckets[i]), world))):
                        assert torch.equal(vc.arenas[r][win], snap[r][win]), ("skipped step wrote the arena", r, i)
            break
        if not check:
            continue
        for i, ps in enumerate(ref_params):
            for p, st, s in zip(ps, starts[i], buckets[i]):
                p.grad = (torch.stack([grads[r][i][st:st + s].to(wdt).double() for r in range(world)]).sum(0)
                          * scale / loss_scale)
        pad = lambda x, n: torch.cat([x, x.new_zeros(_pad8(n) - n)])  # noqa: E731
        w_prev = [torch.cat([pad(p.detach(), p.numel()) for p in ps]) for ps in ref_params]
        ref.step()
        for i, ps in enumerate(ref_params):
            wd, adapt = _group_of(i, nb)
            g = torch.cat([pad(p.grad, p.numel()) for p in ps])
            slices = [(s0, s0 + p.numel(), s0 + _pad8(p.numel())) for s0, p in zip(starts[i], ps)]
            advance(bounds[i], g, w_prev[i], lr, _KW["momentum"], wd, _KW["trust_coefficient"], _KW["eps"], adapt,
                    slices)
        for r in range(world):
            changed = (vc.arenas[r] != snap[r]) & ~written
            assert not changed.any(), ("bytes outside the kernels' windows changed", r,
                                       changed.nonzero()[:8].flatten().tolist())
            for i in range(nb):
                for which, (buf, used) in zip(("master", "v"), bufs[r][i]):
                    assert bool((buf[used:].view(torch.int32) == -1).all()), (which, "canary overwritten", r, i)
        for i, n in enumerate(sizes):
            win = [vc.arenas[r][poffs[i]:poffs[i] + n * ges].view(gdt) for r in range(world)]
            for r in range(1, world):
                assert torch.equal(_bits(win[r]), _bits(win[0])), ("replicas must be bit-identical", t, r, i)
            cat = lambda k: torch.cat([bufs[r][i][k][0][:lens[r][i]] for r in range(world)])  # noqa: E731
            master = cat(0)
            assert torch.equal(_bits(win[0]), _bits(master.to(gdt))), ("window != round(master)", t, i)
            want_w = torch.cat([pad(p.detach(), p.numel()) for p in ref_params[i]])
            want_v = torch.cat([pad(ref.state[p]["momentum_buffer"], p.numel()) for p in ref_params[i]])
            for name, got, ref_v, bound in (("master", master, want_w, bounds[i]["w"]),
                                            ("momentum", cat(1), want_v, bounds[i]["v"])):
                err = (got.double() - ref_v).abs()
                bad = (err > 2 * bound) & real[i]
                assert not bad.any(), (name, t, i, int(bad.sum()), err.max().item(),
                                       (err / bound.clamp_min(1e-300)).max().item())
    return [[[x[0].clone() for x in bb] for bb in bufs[r]] for r in range(world)]


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("dtypes", PAIRS, ids=dt_id)
@pytest.mark.parametrize("world", WORLDS)
def test_lars_kernels_virtual(world, dtypes, layout):
    """Four steps and a skipped fifth against the float64 Lars, bounds derived in _lars.advance."""
    _run_lars(world, *dtypes, layout)


@pytest.mark.parametrize("dtypes", [("bf16", "bf16"), ("f32", "f16")], ids=dt_id)
def test_lars_kernels_reproducible(dtypes):
    """Two runs of the same steps leave the same bits in every rank's master and momentum."""
    a = _run_lars(5, *dtypes, "odd200", skip_last=False, check=False)
    b = _run_lars(5, *dtypes, "odd200", skip_last=False, check=False)
    for r, (ra, rb) in enumerate(zip(a, b)):
        for i, (ba, bb) in enumerate(zip(ra, rb)):
            for k, (x, y) in enumerate(zip(ba, bb)):
                assert torch.equal(_bits(x), _bits(y)), ("run-to-run bits differ", r, i, k)
