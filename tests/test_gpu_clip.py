"""Global gradient-norm clipping in the fused exchange on one H100: the two kernels of grad_clip.cu on virtual ranks
(`VirtualCluster`), on the layouts, worlds and (gradient, wire) pairs of test_gpu_lamb.py.

Per step every rank runs clip_norm_partial over each bucket, then clip_norm_update.  Checked: the norm N against a
float64 sum within a bound derived from the rounding order; padding (whose gradients are not zero here) counts in
no norm; N and every group's new grad_scale are bit-identical on every rank and across runs; grad_scale is
multiplied by the coefficient exactly once; nothing but the staging window, the clipping window, the scratch rows
and the grad_scale fields is written; a step marked skipped still meets every barrier and yields its norm."""
import struct

import pytest
import torch
from _fused_opt import _CANARY, _U, _bits, _code, _cu, _fused_grad, DT, dt_id
from test_gpu_lamb import LAYOUTS, PAIRS, WORLDS

pytestmark = pytest.mark.gpu

_GS_OFF = 48          # byte offset of OptHParams::grad_scale


def _pad8(n):
    return (n + 7) // 8 * 8


def _hp(gs, skip=0):
    """An OptHParams block with grad_scale gs (the other fields play no part in clipping)."""
    return struct.pack("<9f3if2if", 0.1, 0.01, 0.9, 0.0, 0.9, 0.999, 1e-8, 0.1, 0.001, 0, 0, 1, gs, skip, 1, 0.001)


def _run_clip(world, gname, wname, layout, ratios=(0.5, 2.0, 0.25), skip_step=None, blocks=3):
    """One step per entry of `ratios`, max_norm = ratio * N of the float64 reference (ratio >= 1: no clipping).
    Returns [(N per rank, grad_scale fields per rank)] per step, as raw bits."""
    from byteps_b200.comm.symm import VirtualCluster

    cu = _cu()
    gdt, wdt = DT[gname], DT[wname]
    wes = torch.empty((), dtype=wdt).element_size()
    buckets = LAYOUTS[layout]
    nb = len(buckets)
    starts = [[sum(_pad8(s) for s in segs[:j]) for j in range(len(segs))] for segs in buckets]
    sizes = [sum(_pad8(s) for s in segs) for segs in buckets]
    scale = 1.0 / world
    pack = gdt != wdt
    end = 256

    def window(nbytes):
        nonlocal end
        start = end
        end = (start + nbytes + 255) // 256 * 256 + 256
        return start

    if pack:
        stage = window(max(sizes) * wes)      # one staging window shared by all buckets, as in the arena
        goffs = [stage] * nb
    else:
        goffs = [window(n * wes) for n in sizes]
    clip_off = window(cu.CLIP_WINDOW_BYTES)
    vc = VirtualCluster(world, "cuda:0", end)
    written = torch.zeros(vc.arenas[0].numel(), dtype=torch.bool, device="cuda")
    written[clip_off:clip_off + cu.CLIP_WINDOW_BYTES] = True
    if pack:
        written[stage:stage + max(sizes) * wes] = True
    real = [torch.zeros(n, dtype=torch.bool, device="cuda") for n in sizes]
    for i, segs in enumerate(buckets):
        for st, s in zip(starts[i], segs):
            real[i][st:st + s] = True
    tables = [torch.tensor([[st, s] for st, s in zip(starts[i], segs)], dtype=torch.int64, device="cuda")
              for i, segs in enumerate(buckets)]
    # one scratch row per bucket, wider than the grid: the entries no CTA writes stay zero
    row = blocks + 2
    scratch = [torch.zeros((nb, row), dtype=torch.float64, device="cuda") for _ in range(world)]
    norms = [torch.full((2,), -1, dtype=torch.int32, device="cuda").view(torch.float32) for _ in range(world)]
    hps = [torch.zeros((nb, 64), dtype=torch.uint8, device="cuda") for _ in range(world)]
    for r in range(world):
        vc.arenas[r].fill_(_CANARY)
    torch.manual_seed(11)
    out = []
    for t, ratio in enumerate(ratios):
        loss_scale = 128.0 if t % 2 else 1.0
        skip = int(t == skip_step)
        # the padding of every parameter holds gradients too: they must count in no norm
        grads = [[_fused_grad(n, loss_scale).to(gdt) for n in sizes] for _ in range(world)]
        users = []
        for r in range(world):
            if pack:
                users.append([g.clone() for g in grads[r]])
            else:
                for i, n in enumerate(sizes):
                    vc.arenas[r][goffs[i]:goffs[i] + n * wes].view(wdt).copy_(grads[r][i])
        segtabs = [[torch.tensor([[u.data_ptr(), u.data_ptr(), 0, u.numel()]], dtype=torch.int64, device="cuda")
                    for u in users[r]] for r in range(world)] if pack else None
        # the float64 reference: sum over ranks of the wire values (exact), times scale / loss_scale, squared over
        # the parameters' elements
        ref_sq = 0.0
        for i in range(nb):
            g = torch.stack([grads[r][i].to(wdt).double() for r in range(world)]).sum(0) * scale / loss_scale
            ref_sq += float((g[real[i]] ** 2).sum())
        ref_n = ref_sq ** 0.5
        max_norm = ratio * ref_n
        gs = 1.0 / loss_scale
        blob = b"".join(_hp(gs, skip) for _ in range(nb))
        for r in range(world):
            cu.write_blob(hps[r].data_ptr(), blob, torch.cuda.current_stream().cuda_stream)
        snap = [a.clone() for a in vc.arenas]
        hp_snap = [h.clone() for h in hps]

        def launch(r, view, arena, s):
            for i, n in enumerate(sizes):
                segs, nsegs = (segtabs[r][i].data_ptr(), 1) if pack else (0, 0)
                cu.clip_norm_partial(view, _code(gdt), _code(wdt), segs, nsegs, goffs[i], n, scale,
                                     tables[i].data_ptr(), len(buckets[i]), scratch[r][i].data_ptr(),
                                     hps[r][i].data_ptr(), blocks, 512, 0, False, s)
            cu.clip_norm_update(view, 0, clip_off, scratch[r].data_ptr(), nb, row, max_norm, norms[r].data_ptr(),
                                hps[r].data_ptr(), nb, s)

        vc.run(launch)
        torch.cuda.synchronize()

        # N: fp32 g = fl(g_sum * fl(scale * gs)) squares to within (1 + u)^4 of the exact square; the float64 sum of
        # n terms adds at most n * 2^-53 relative; sqrt halves the relative error and the rounding to fp32 adds u
        n_terms = sum(int(x.sum()) for x in real)
        bound = (2 * _U + n_terms * 2.0 ** -53 + _U) * 1.01 * ref_n
        got = [float(norms[r][0]) for r in range(world)]
        assert abs(got[0] - ref_n) <= bound, (t, got[0], ref_n, bound)
        coef_ref = min(1.0, max_norm / (ref_n + 1e-6))
        for r in range(world):
            assert torch.equal(_bits(norms[r][:1]), _bits(norms[0][:1])), ("N differs between replicas", t, r)
            assert bool((norms[r][1:].view(torch.int32) == -1).all()), ("canary after N overwritten", t, r)
            assert torch.equal(hps[r], hps[0]), ("grad_scale differs between replicas", t, r)
            changed = (vc.arenas[r] != snap[r]) & ~written
            assert not changed.any(), ("bytes outside the staging and clipping windows changed", t, r,
                                       changed.nonzero()[:8].flatten().tolist())
            assert int((scratch[r][:, blocks:] != 0).sum()) == 0, ("scratch beyond the grid written", t, r)
            other = torch.ones(64, dtype=torch.bool, device="cuda")
            other[_GS_OFF:_GS_OFF + 4] = False
            assert torch.equal(hps[r][:, other], hp_snap[r][:, other]), ("a field besides grad_scale changed", t, r)
            if pack:
                for u, g in zip(users[r], grads[r]):
                    assert torch.equal(_bits(u), _bits(g)), "user gradients must only be read"
        new_gs = hps[0][:, _GS_OFF:_GS_OFF + 4].contiguous().view(torch.float32).double()
        # gs is a power of two: fl(gs * coef) = gs * coef exactly, so new_gs / gs is the coefficient the kernel used,
        # once (twice would give about coef^2)
        coef = new_gs / gs
        assert bool((coef == coef[0]).all()), coef
        if ratio >= 1.0:
            assert bool((coef == 1.0).all()), ("no clipping must leave grad_scale bit-identical", t, coef)
        else:
            c = float(coef[0])
            assert abs(c - coef_ref) <= (bound / ref_n + 2 * _U) * coef_ref * 1.01, (t, c, coef_ref)
        out.append(([int(_bits(norms[r][:1])[0]) for r in range(world)], [h.clone() for h in hps]))
    return out


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("dtypes", PAIRS, ids=dt_id)
@pytest.mark.parametrize("world", WORLDS)
def test_clip_kernels_virtual(world, dtypes, layout):
    """Three steps (clipped, not clipped, clipped) against the float64 norm."""
    _run_clip(world, *dtypes, layout)


@pytest.mark.parametrize("dtypes", [("bf16", "bf16"), ("f32", "f16")], ids=dt_id)
def test_clip_kernels_reproducible(dtypes):
    """Two runs of the same steps give the same N and grad_scale bits on every rank."""
    a = _run_clip(5, *dtypes, "odd200")
    b = _run_clip(5, *dtypes, "odd200")
    for t, ((na, ha), (nb_, hb)) in enumerate(zip(a, b)):
        assert na == nb_, ("run-to-run N differs", t)
        for r, (x, y) in enumerate(zip(ha, hb)):
            assert torch.equal(x, y), ("run-to-run grad_scale differs", t, r)


@pytest.mark.parametrize("world", [2, 8])
def test_skipped_step_meets_every_barrier(world):
    """A step whose OptHParams::skip is set (dynamic loss scaling found an overflow) still reduces, meets every
    barrier and yields its norm; the steps after it pair their barriers as before."""
    a = _run_clip(world, "bf16", "bf16", "fused", skip_step=1)
    b = _run_clip(world, "bf16", "bf16", "fused")
    for t, ((na, _), (nb_, _)) in enumerate(zip(a, b)):
        assert na == nb_, ("a skipped step changed N", t)


def test_grid_wider_than_a_small_bucket():
    """More CTAs than tiles (most CTAs of the 24-element bucket own nothing) and an empty shard at world 8."""
    _run_clip(8, "f32", "f32", "fused", blocks=16)
