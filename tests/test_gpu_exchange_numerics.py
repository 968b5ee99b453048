"""Every gradient-exchange kernel against a float64 sum with one rounding to the wire dtype.

For one output element, with wire-dtype inputs a_1..a_P (one per rank; for the packed kernel each user value
first rounded to the wire dtype) and the fp32 scale s passed to the kernel:

    e = s * sum(a_p)            (float64)
    A = |s| * sum |a_p|
    |out - e| <= u_W |e| + m_W + c P 2^-24 A

u_W is half an ulp relative to |e| and m_W half the smallest subnormal of the wire dtype; the last term covers
the P - 1 fp32 additions and the fp32 scaling.  c = 1 for the CUDA-core kernels and 2 for the wgmma kernel,
whose fp32 accumulation inside the tensor core is not documented.  Where e overflows the output dtype the result
must be an inf of the same sign; where an input is inf or NaN it must be non-finite.  For the packed kernel the
result is rounded once more, to the user dtype.

The bound is half an ulp wide, so it tells a kernel that sums in fp32 and rounds once to nearest from one that
sums in the wire dtype, truncates, or rounds the sum before it scales it: `test_bound_rejects_wrong_models`
checks that on the CPU.  Every GPU case also asserts that the replicas are bitwise identical and that no byte
outside the exchanged windows changed (4 KiB bands around and between the windows, on every rank).

Multi-rank kernels run on virtual ranks of one GPU (`VirtualCluster`): every CTA of every rank must be resident
at once, so world * blocks stays <= 64, and nothing is launched for the first time while a rank's kernel spins.
"""
import math
import types

import pytest
import torch

from _bounds import BF16, DT, F16, F32, HALF_MIN_SUB, UNIT, stored
LOSS_SCALE_SUM_LIMIT = 3.38e38       # kLossScaleSumLimit, csrc/kernels/loss_scale.cuh
GUARD = 4096
WORLDS = [1, 2, 3, 5, 8]
# (world, poison): every world with finite inputs, and inf / NaN inputs at worlds 3 and 8
CASES = [(w, False) for w in WORLDS] + [(3, True), (8, True)]
CASE_IDS = ["w%d%s" % (w, "-nonfinite" if p else "") for w, p in CASES]
# 16-byte units per CTA tile: LSU kernels (in-place, reduce-scatter / all-gather, packed, ring) run 512 threads
# x 2 units, the TMA kernel 256 units; the wgmma kernel's tile is 8192 elements
TILE_UNITS = {"lsu": 1024, "tma": 256, "ring": 1024, "rsag": 1024, "packed": 1024}
UMMA_TILE = 8192


def _cu():
    from byteps_b200 import _native

    return _native.cuda()


def _code(dt):
    from byteps_b200.comm.symm import wire_code

    return wire_code(dt)


def pad8(n):
    return (n + 7) // 8 * 8


def bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def scales(world):
    return [1.0 / world, 1.0] if world > 1 else [1.0]


def report(engine, what, ratio):
    print("exchange-numerics: %-6s %-28s max err/bound = %.4f" % (engine, what, ratio))


# ------------------------------------------------------------------------------------------------ reference
def _inf_threshold(dt):
    """Smallest magnitude that rounds to inf in dt: the largest finite value plus half its ulp."""
    fmax = torch.finfo(dt).max
    return fmax + UNIT[dt] * 2.0 ** (math.frexp(fmax)[1] - 1)


def reference(ins, scale):
    """e = scale * sum(a_p) and A = |scale| * sum |a_p| in float64, with the scale rounded to fp32 as the kernels
    receive it."""
    s = float(torch.tensor(scale, dtype=F32))
    e = torch.zeros(ins[0].shape, dtype=torch.float64, device=ins[0].device)
    a = torch.zeros_like(e)
    for x in ins:
        d = x.double()
        e += d
        a += d.abs()
    return e * s, a * abs(s)


def violations(out, e, a, world, c, wire, user=None):
    """Boolean mask of the elements of `out` that break the rule in the module docstring, and the largest
    |out - e| / bound over the elements with a finite, representable reference."""
    user = user or wire
    o = out.double()
    fin = torch.isfinite(e)
    ovf = fin & (e.abs() >= min(_inf_threshold(wire), _inf_threshold(user)))
    ok = fin & ~ovf
    b = UNIT[wire] * e.abs() + HALF_MIN_SUB[wire] + c * world * 2.0 ** -24 * a
    if user != wire:
        b = stored(e.abs(), b, user)
    err = (o - e).abs()
    bad = ok & ~(err <= b)
    bad |= ovf & (o != e.sign() * math.inf)
    bad |= ~fin & torch.isfinite(o)
    ratio = (err[ok] / b[ok]).max().item() if ok.any() else 0.0
    return bad, ratio


def check_bound(out, e, a, world, c, wire, user=None, what=""):
    bad, ratio = violations(out, e, a, world, c, wire, user)
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: %d elements out of bound, first at %d: got %r, want %r (A = %r)" % (
            what, int(bad.sum()), i, out[i].item(), e[i].item(), a[i].item()))
    return ratio


# ------------------------------------------------------------------------------------------------ inputs
def sum_limit_value(world, dt):
    """Largest dt value not above kLossScaleSumLimit / world (divided in fp32, as the overflow check does)."""
    lim = torch.tensor(LOSS_SCALE_SUM_LIMIT, dtype=F32) / world
    v = lim.to(dt).reshape(1)
    if v.float().item() > lim.item():
        bits(v).sub_(1)
    return v.item()


def make_inputs(world, n, dt, seed, device="cuda", poison=False):
    """One tensor per rank: normals spread over many binades, and from 64 elements on, at fixed positions:
    [0:4) zeros, [4:16) a_1 = -a_0, [16:32) subnormals, [32:40) +-60000 (fp16) or +-the largest value whose
    world-fold sum stays below kLossScaleSumLimit (bf16, fp32), and with `poison` +inf on rank 0 and -inf on
    rank 1 at 48, NaN on the last rank at 49."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    lo, hi = (-10, 6) if dt == F16 else (-30, 30)
    ins = []
    for _ in range(world):
        x = torch.randn(n, generator=g, device=device)
        x *= torch.exp2(torch.randint(lo, hi + 1, (n,), generator=g, device=device).float())
        ins.append(x.to(dt))
    if n >= 64:
        kmax, emin = {F16: (1023, -24), BF16: (127, -133), F32: (1 << 22, -149)}[dt]
        big = 60000.0 if dt == F16 else sum_limit_value(world, dt)
        for x in ins:
            x[0:2] = 0.0
            x[2:4] = -0.0
            k = torch.randint(-kmax, kmax + 1, (16,), generator=g, device=device).double()
            x[16:32] = (k * 2.0 ** emin).to(dt)
            x[32:36] = big
            x[36:40] = -big
        if world >= 2:
            ins[1][4:16] = -ins[0][4:16]
        if poison:
            assert world >= 2
            ins[0][48] = math.inf
            ins[1][48] = -math.inf
            ins[world - 1][49] = math.nan
    return ins


def check_specials(out, n, dt, scale, world):
    """The value classes of make_inputs that carry a claim of their own."""
    if n < 64:
        return
    o = out[32:40].double()
    if dt == F16:
        if world >= 2 and scale == 1.0:      # 60000 summed over ranks overflows fp16
            assert (o[:4] == math.inf).all() and (o[4:] == -math.inf).all(), o
        else:                                # averaged it is 60000 again
            assert (o[:4] == 60000.0).all() and (o[4:] == -60000.0).all(), o
    else:                                    # loss_scale.cuh: no sum of checked values overflows
        assert torch.isfinite(o).all(), o


def window_sizes(engine, world, dt):
    """8 elements (one group: at world 8 seven ranks own empty shards), 8 world - 8, an odd number of groups with
    a ragged tail, the engine's tile -8 / +8 elements per shard, and about 2^20 elements.  The ring and wgmma
    kernels take multiples of 8."""
    tile = UMMA_TILE if engine == "umma" else TILE_UNITS[engine] * (16 // dt.itemsize)
    sizes = [8, 8 * world - 8, 8 * 77 - 3, world * (tile - 8), world * (tile + 8), (1 << 20) + 8 * 13 + 5]
    if engine in ("umma", "ring"):
        sizes = [pad8(n) for n in sizes]
    return [n for n in sizes if n > 0]


def layout(sizes, es, misalign):
    """Window offsets with a 4 KiB band before, between and after the windows.  Every second window starts
    `misalign` bytes past a 256-byte boundary."""
    offs, off = [], GUARD
    for i, n in enumerate(sizes):
        off += misalign if i % 2 else 0
        offs.append(off)
        off = (off + pad8(n) * es + GUARD + 255) // 256 * 256
    return offs, off


def sentinel(nbytes, seed):
    """Random bytes that are finite in every wire dtype (top exponent bit of each 16-bit word clear): the wgmma
    kernel reads, but does not write, up to 63 elements past a shard whose last 64-element row is ragged, and a
    non-finite value there would reach the results through 0 x inf."""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    b = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=g)
    b[1::2] &= 0xBF
    return b


def check_unchanged(buf, snap, allowed, what):
    """Bytes of `buf` outside the [lo, hi) ranges of `allowed` equal `snap`."""
    mask = torch.zeros(buf.numel(), dtype=torch.bool, device=buf.device)
    for lo, hi in allowed:
        mask[lo:hi] = True
    changed = (buf != snap) & ~mask
    if changed.any():
        raise AssertionError("%s: byte %d outside the exchanged windows changed" % (what, int(changed.nonzero()[0])))


def same_replicas(outs, what):
    for r, o in enumerate(outs[1:], 1):
        assert torch.equal(bits(o), bits(outs[0])), "%s: rank %d differs from rank 0" % (what, r)


# ------------------------------------------------------------------------------------------------ CPU self-test
def _truncate(x32, dt):
    """Round toward zero from fp32 to a 16-bit dtype."""
    r = x32.to(dt)
    bits(r)[r.float().abs() > x32.abs()] -= 1
    return r


@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_bound_rejects_wrong_models(dt):
    """On seeded world-3 inputs averaged with scale 1/3, the bound accepts the fp32 model on every element and
    rejects each of three wrong ones on some element."""
    wire, world = DT[dt], 3
    ins = make_inputs(world, 1 << 16, wire, seed=5, device="cpu")
    s = torch.tensor(1.0 / world, dtype=F32)
    acc = torch.zeros(ins[0].shape, dtype=F32)
    for x in ins:
        acc += x.float()
    acc_w = ins[0].clone()
    for x in ins[1:]:
        acc_w = acc_w + x                        # rounded to the wire dtype after every addition
    models = {
        "sum in the wire dtype": (acc_w.float() * s).to(wire),
        "truncated": _truncate(acc * s, wire),
        "rounded twice": (acc.to(wire).float() * s).to(wire),
    }
    e, a = reference(ins, s.item())
    right = (acc * s).to(wire)
    check_bound(right, e, a, world, 1, wire, what="fp32 model")
    for name, out in models.items():
        bad, _ = violations(out, e, a, world, 1, wire)
        assert bad.any(), "the bound accepts the model '%s'" % name


# ------------------------------------------------------------------------------------------------ in-place engines
def _fill(vc, end, windows, dt, seed):
    """Sentinel bytes over [0, end) of every arena, the inputs in their windows; returns the snapshots."""
    snaps = []
    for r in range(vc.world):
        arena = vc.arenas[r]
        arena[:end].copy_(sentinel(end, seed * 16 + r))
        for off, x in windows:
            arena[off:off + x[r].numel() * dt.itemsize].view(dt).copy_(x[r])
        snaps.append(arena[:end].clone())
    torch.cuda.synchronize()
    return snaps


def _window(vc, r, off, n, dt):
    return vc.arenas[r][off:off + n * dt.itemsize].view(dt)


def _run_inplace(engine, world, dt, poison, launch_all, c, misalign=48, seed=0):
    """Exchange every window of window_sizes(engine) in place with scale 1/world and 1, and check them.
    launch_all(vc, offs, sizes, scale) issues the exchanges."""
    from byteps_b200.comm.symm import VirtualCluster

    es = dt.itemsize
    sizes = window_sizes(engine, world, dt)
    offs, end = layout(sizes, es, misalign)
    vc = VirtualCluster(world, "cuda:0", end)
    ins = [make_inputs(world, n, dt, seed=seed * 100 + i, poison=poison) for i, n in enumerate(sizes)]
    worst = 0.0
    for scale in scales(world):
        snaps = _fill(vc, end, list(zip(offs, ins)), dt, seed)
        launch_all(vc, offs, sizes, scale)
        torch.cuda.synchronize()
        # kernels round the window up to whole groups of 8 elements
        allowed = [(o, o + pad8(n) * es) for o, n in zip(offs, sizes)]
        for r in range(world):
            check_unchanged(vc.arenas[r][:end], snaps[r], allowed, "rank %d" % r)
        for i, (off, n, x) in enumerate(zip(offs, sizes, ins)):
            what = "%s %s world %d window %d (n=%d) scale %g" % (engine, dt, world, i, n, scale)
            outs = [_window(vc, r, off, n, dt) for r in range(world)]
            same_replicas(outs, what)
            e, a = reference(x, scale)
            if engine == "umma" and poison and n >= 64:
                # an inf in the B operand meets the identity's zeros: 0 x inf = NaN in its column of the
                # 64-row half tile.  Only the poisoned elements are asserted.
                nf = ~torch.isfinite(outs[0])
                assert nf[48] and nf[49], what
                print("exchange-numerics: umma   %s: %d non-finite outputs from 2 poisoned elements" % (
                    what, int(nf.sum())))
                continue
            worst = max(worst, check_bound(outs[0], e, a, world, c, dt, what=what))
            check_specials(outs[0], n, dt, scale, world)
    report(engine, "%s world %d%s" % (dt, world, " nonfinite" if poison else ""), worst)


def _per_window(launch):
    def launch_all(vc, offs, sizes, scale):
        for off, n in zip(offs, sizes):
            torch.cuda.synchronize()
            vc.run(lambda r, view, arena, s: launch(view, off, n, scale, s))
    return launch_all


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", [1, 3])
@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("world,poison", CASES, ids=CASE_IDS)
def test_lsu_inplace(world, poison, dt, blocks):
    cu, d = _cu(), DT[dt]
    _run_inplace("lsu", world, d, poison, _per_window(
        lambda view, off, n, scale, s: cu.pushpull_inplace(view, _code(d), off, n, scale, blocks, 512, 0, False, s)),
        c=1, seed=1)


@pytest.mark.gpu
@pytest.mark.parametrize("stages", [1, 4])
@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("world,poison", CASES, ids=CASE_IDS)
def test_tma_inplace(world, poison, dt, stages):
    cu, d = _cu(), DT[dt]
    _run_inplace("tma", world, d, poison, _per_window(
        lambda view, off, n, scale, s: cu.pushpull_inplace_tma(view, _code(d), off, n, scale, 3, stages, 0, s)),
        c=1, seed=2)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("world,poison", CASES, ids=CASE_IDS)
def test_wgmma_inplace(world, poison, dt):
    cu, d = _cu(), DT[dt]

    def launch(view, off, n, scale, s):
        maps = cu.make_umma_maps(view, _code(d), off, n)
        cu.pushpull_inplace_umma(view, maps, _code(d), off, n, scale, 2, 0, s)

    _run_inplace("umma", world, d, poison, _per_window(launch), c=2, misalign=128, seed=3)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("world,poison", CASES, ids=CASE_IDS)
def test_ring_allreduce(world, poison, dt):
    """Every window is one RING_ALLREDUCE descriptor of a single ring launch."""
    from byteps_b200.ops.ring import RingEntry, RingTable

    d = DT[dt]

    def launch_all(vc, offs, sizes, scale):
        entries = [RingEntry(grad_off=o, numel=n, wire=_code(d), slot=i, scale=scale)
                   for i, (o, n) in enumerate(zip(offs, sizes))]
        tables = [RingTable(entries, "cuda:0") for _ in range(vc.world)]
        torch.cuda.synchronize()
        vc.run(lambda r, view, arena, s: tables[r].launch(view, 2, s))

    _run_inplace("ring", world, d, poison, launch_all, c=1, seed=4)


# ------------------------------------------------------------------------------------------------ split phases
@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("world,poison", CASES, ids=CASE_IDS)
def test_reduce_scatter_then_all_gather(world, poison, dt):
    """The reduce-scatter leaves this rank's shard (`ops.pushpull.shard_elems`) holding the sum and the rest of
    its window holding its own input; the all-gather then writes the wire rounding of scale x owner's value into
    every replica.  Even windows go through the bindings, odd ones through the `ops.pushpull` wrappers."""
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops import pushpull as pp

    cu, d = _cu(), DT[dt]
    es = d.itemsize
    sizes = window_sizes("rsag", world, d)
    offs, end = layout(sizes, es, 48)
    vc = VirtualCluster(world, "cuda:0", end)
    ctxs = [types.SimpleNamespace(cu=cu, view=vc.views[r], world=world, rank=r, nvls=False,
                                  device=torch.device("cuda:0")) for r in range(world)]
    ins = [make_inputs(world, n, d, seed=500 + i, poison=poison) for i, n in enumerate(sizes)]
    shards = [[pp.shard_elems(ctxs[r], n) for r in range(world)] for n in sizes]
    for n, sh in zip(sizes, shards):      # the shards tile the window in rank order
        assert sh[0][0] == 0 and sh[-1][1] == n and all(sh[r][1] == sh[r + 1][0] for r in range(world - 1)), sh

    def launch(phase, scale):
        for i, (off, n) in enumerate(zip(offs, sizes)):
            torch.cuda.synchronize()
            if phase == "rs" and i % 2 == 0:
                vc.run(lambda r, v, a, s: cu.reduce_scatter(v, _code(d), off, n, 3, 512, 0, False, s))
            elif phase == "rs":
                vc.run(lambda r, v, a, s: pp.reduce_scatter(ctxs[r], off, n, d, stream=torch.cuda.ExternalStream(s),
                                                            blocks=3))
            elif i % 2 == 0:
                vc.run(lambda r, v, a, s: cu.all_gather(v, _code(d), off, n, scale, 3, 512, 0, False, s))
            else:
                vc.run(lambda r, v, a, s: pp.all_gather(ctxs[r], off, n, d, scale, stream=torch.cuda.ExternalStream(s),
                                                        blocks=3))
        torch.cuda.synchronize()

    worst_rs = worst_ag = 0.0
    for scale in scales(world):
        snaps = _fill(vc, end, list(zip(offs, ins)), d, 5)
        launch("rs", 1.0)
        for r in range(world):
            # the shard ending at n also covers the padding up to the next group of 8
            allowed = [(o + sh[r][0] * es, o + (pad8(n) if sh[r][1] == n else sh[r][1]) * es)
                       for o, n, sh in zip(offs, sizes, shards)]
            check_unchanged(vc.arenas[r][:end], snaps[r], allowed, "reduce-scatter rank %d" % r)
        owner = []
        for i, (off, n, x, sh) in enumerate(zip(offs, sizes, ins, shards)):
            e, a = reference(x, 1.0)
            parts = []
            for r in range(world):
                b0, b1 = sh[r]
                got = _window(vc, r, off, n, d)[b0:b1]
                what = "reduce-scatter %s world %d window %d rank %d" % (dt, world, i, r)
                worst_rs = max(worst_rs, check_bound(got, e[b0:b1], a[b0:b1], world, 1, d, what=what))
                parts.append(got.clone())
            owner.append(torch.cat(parts))
        snaps = [vc.arenas[r][:end].clone() for r in range(world)]
        launch("ag", scale)
        allowed = [(o, o + pad8(n) * es) for o, n in zip(offs, sizes)]
        for r in range(world):
            check_unchanged(vc.arenas[r][:end], snaps[r], allowed, "all-gather rank %d" % r)
        for i, (off, n, own) in enumerate(zip(offs, sizes, owner)):
            what = "all-gather %s world %d window %d scale %g" % (dt, world, i, scale)
            outs = [_window(vc, r, off, n, d) for r in range(world)]
            same_replicas(outs, what)
            e, a = reference([own], scale)
            worst_ag = max(worst_ag, check_bound(outs[0], e, a, 1, 1, d, what=what))
    report("rs", "%s world %d%s" % (d, world, " nonfinite" if poison else ""), worst_rs)
    report("ag", "%s world %d%s" % (d, world, " nonfinite" if poison else ""), worst_ag)


# ------------------------------------------------------------------------------------------------ packed
PACKED_PAIRS = [("f32", "f32"), ("f32", "bf16"), ("f32", "f16"), ("bf16", "bf16"), ("f16", "f16"), ("bf16", "f32"),
                ("f16", "f32")]


def _run_packed(world, user, wire, one_shot, poison, scale_list=None):
    """One packed launch over user tensors of window_sizes lengths.  Segment i starts i % 8 elements past a
    16-byte boundary; every third segment is exchanged in place (dst == src).  Returns, per scale, rank 0's
    outputs."""
    from byteps_b200.comm.symm import VirtualCluster

    cu = _cu()
    ud, wd = DT[user], DT[wire]
    gen = wd if wd.itemsize <= ud.itemsize else ud        # values exact in both dtypes
    ues, wes = ud.itemsize, wd.itemsize
    sizes = [5] + window_sizes("packed", world, wd)
    ins = [[x.to(ud) for x in make_inputs(world, n, gen, seed=900 + i, poison=poison)] for i, n in enumerate(sizes)]
    src, dst, cur = [], [], GUARD
    for i, n in enumerate(sizes):
        cur = (cur + 255) // 256 * 256 + (i % 8) * ues
        src.append(cur)
        cur += n * ues + GUARD
        if i % 3 == 2:
            dst.append(src[-1])
        else:
            cur = (cur + 255) // 256 * 256 + (i % 8) * ues
            dst.append(cur)
            cur += n * ues + GUARD
    uend = cur
    starts = [sum(pad8(m) for m in sizes[:i]) for i in range(len(sizes))]
    total = sum(pad8(n) for n in sizes)
    stage_off = GUARD + 48
    end = stage_off + total * wes + GUARD
    vc = VirtualCluster(world, "cuda:0", end)
    ubufs = [torch.empty(uend, dtype=torch.uint8, device="cuda") for _ in range(world)]
    tables = [torch.tensor([[ubufs[r].data_ptr() + so, ubufs[r].data_ptr() + do, st, n]
                            for so, do, st, n in zip(src, dst, starts, sizes)], dtype=torch.int64, device="cuda")
              for r in range(world)]
    results = {}
    worst = 0.0
    for scale in scale_list or scales(world):
        snaps, usnaps = [], []
        for r in range(world):
            vc.arenas[r][:end].copy_(sentinel(end, 70 + r))
            ubufs[r].copy_(sentinel(uend, 80 + r))
            for so, n, x in zip(src, sizes, ins):
                ubufs[r][so:so + n * ues].view(ud).copy_(x[r])
            snaps.append(vc.arenas[r][:end].clone())
            usnaps.append(ubufs[r].clone())
        torch.cuda.synchronize()
        vc.run(lambda r, view, arena, s: cu.pushpull_packed(view, _code(ud), _code(wd), tables[r].data_ptr(),
                                                            len(sizes), stage_off, total, scale, 2, 512, 0, False,
                                                            one_shot, True, s))
        torch.cuda.synchronize()
        for r in range(world):
            check_unchanged(vc.arenas[r][:end], snaps[r], [(stage_off, stage_off + total * wes)], "staging rank %d" % r)
            check_unchanged(ubufs[r], usnaps[r], [(do, do + n * ues) for do, n in zip(dst, sizes)],
                            "user tensors rank %d" % r)
        outs0 = []
        for i, (do, n, x) in enumerate(zip(dst, sizes, ins)):
            what = "packed %s->%s world %d one_shot %d segment %d (n=%d) scale %g" % (
                user, wire, world, one_shot, i, n, scale)
            outs = [ubufs[r][do:do + n * ues].view(ud) for r in range(world)]
            same_replicas(outs, what)
            e, a = reference([v.to(wd) for v in x], scale)
            worst = max(worst, check_bound(outs[0], e, a, world, 1, wd, ud, what=what))
            check_specials(outs[0], n, gen, scale, world)
            outs0.append(outs[0].clone())
        results[scale] = outs0
    report("packed", "%s->%s world %d one_shot %d%s" % (user, wire, world, one_shot, " nonfinite" if poison else ""),
           worst)
    return results


@pytest.mark.gpu
@pytest.mark.parametrize("one_shot", [False, True])
@pytest.mark.parametrize("user,wire", PACKED_PAIRS)
@pytest.mark.parametrize("world,poison", CASES, ids=CASE_IDS)
def test_packed(world, poison, user, wire, one_shot):
    _run_packed(world, user, wire, one_shot, poison)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 5])
def test_packed_one_shot_matches_two_shot(world):
    """The engine picks one-shot for small tensors and two-shot for large ones; both must give the same bits,
    which at world > 2 needs the same peer order in the fp32 sum."""
    for scale in scales(world):
        one = _run_packed(world, "f32", "f32", True, False, [scale])[scale]
        two = _run_packed(world, "f32", "f32", False, False, [scale])[scale]
        for i, (x, y) in enumerate(zip(one, two)):
            diff = int((bits(x) != bits(y)).sum())
            assert diff == 0, "segment %d: %d of %d elements differ at scale %g" % (i, diff, x.numel(), scale)


# ------------------------------------------------------------------------------------------------ > 2^31 elements
@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["lsu", "ring"])
def test_exchange_above_2_31_elements(engine):
    """World 2, bf16, 2^31 + 2^16 + 8 elements (4 GiB per arena); inputs regenerated and checked in chunks."""
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops.ring import RingEntry, RingTable

    cu = _cu()
    world, d, es, scale = 2, BF16, 2, 0.5
    n = (1 << 31) + (1 << 16) + 8
    off = GUARD + 48
    end = off + n * es + GUARD
    chunk = 1 << 26
    vc = VirtualCluster(world, "cuda:0", end)

    def chunks():
        for c, lo in enumerate(range(0, n, chunk)):
            hi = min(n, lo + chunk)
            yield lo, hi, make_inputs(world, hi - lo, d, seed=3000 + c)

    bands = [(0, off), (off + n * es, end)]
    snaps = []
    for r in range(world):
        for lo, hi in bands:
            vc.arenas[r][lo:hi].copy_(sentinel(hi - lo, 90 + r))
        snaps.append([vc.arenas[r][lo:hi].clone() for lo, hi in bands])
    for lo, hi, xs in chunks():
        for r in range(world):
            _window(vc, r, off, n, d)[lo:hi].copy_(xs[r])
    if engine == "ring":
        tables = [RingTable([RingEntry(grad_off=off, numel=n, wire=_code(d), slot=0, scale=scale)], "cuda:0")
                  for _ in range(world)]
    torch.cuda.synchronize()
    if engine == "lsu":
        vc.run(lambda r, view, arena, s: cu.pushpull_inplace(view, _code(d), off, n, scale, 32, 512, 0, False, s))
    else:
        vc.run(lambda r, view, arena, s: tables[r].launch(view, 16, s))
    torch.cuda.synchronize()
    for r in range(world):
        for (lo, hi), snap in zip(bands, snaps[r]):
            assert torch.equal(vc.arenas[r][lo:hi], snap), "rank %d: bytes [%d, %d) changed" % (r, lo, hi)
    worst = 0.0
    for lo, hi, xs in chunks():
        outs = [_window(vc, r, off, n, d)[lo:hi] for r in range(world)]
        what = "%s > 2^31 elements, chunk at %d" % (engine, lo)
        same_replicas(outs, what)
        e, a = reference(xs, scale)
        worst = max(worst, check_bound(outs[0], e, a, world, 1, d, what=what))
    report(engine, "bf16 world 2, %d elements" % n, worst)
