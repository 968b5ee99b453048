"""Dynamic loss scaling of the fused optimizer (kernels/loss_scale.cu, BucketedGradSync, DistributedOptimizer).

- The overflow check and the cross-rank agreement + scaler update, on VirtualCluster worlds 1, 2, 3 and 8.
- A skipped step on the register, TMA and ring engines leaves every byte of the optimizer's memory as it was, and
  the next applied step matches torch.optim whose step count did not advance.
- The scale trajectory equals torch.amp.GradScaler's for the same overflow sequence.
- The public API at world 1 against torch.optim + torch.amp.GradScaler on fp32 masters, eager and in a CUDA graph;
  checkpoints; two processes; the argument checks (CPU).
"""
import math
import os
import struct
import subprocess
import sys
import textwrap

import pytest
import torch

from _fused_opt import (_CANARY, DT, FUSED_OPTS, _advance_bounds, _bits, _code, _cu, _fused_grad, _guarded,
                        _opt_blob)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_STATE_FMT = "<2df5i"      # LossScaleState
_ENTRY_FMT = "<2Q4i"       # LossScaleCheckEntry
_SKIP_OFF = 52             # OptHParams::skip


def _state_blob(scale, growth=2.0, backoff=0.5, interval=2000, tracker=0, skipped=0):
    return struct.pack(_STATE_FMT, growth, backoff, scale, interval, tracker, skipped, 0, 0)


def _f32(x):
    return struct.unpack("<f", struct.pack("<f", x))[0]


def _ulp_diff(a, b):
    ia, ib = (struct.unpack("<i", struct.pack("<f", v))[0] for v in (a, b))
    return abs(ia - ib)


# ---------------------------------------------------------------------------------------------------------------
# 1. check + agreement kernels

# (gradient, wire) pairs the bucket layer launches
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("f16", "f16"), ("f32", "bf16"), ("f32", "f16")]
# two buckets: 8*40 elements with no padding, 8*37 holding 293 elements and 3 padding zeros
_LENS, _NUMEL = [320, 293], [320, 296]


def _trips(value, grad, wire, world):
    """Does `value`, stored as a `grad` gradient, count as an overflow at `world` ranks with S >= 1?"""
    if value in ("inf", "nan"):
        return True
    if value == "flt_max":                 # inf in bf16 and fp16; above the sum limit 3.38e38 / world in fp32
        return True
    if value == "big":                     # 2e38: inf in fp16; two of them overflow an fp32 (or bf16) sum
        return grad == "f16" or wire == "f16" or world > 1
    if value == 65520.0:                   # rounds to inf in fp16 only
        return grad == "f16" or wire == "f16"
    return False


def _value(v):
    return {"inf": float("inf"), "nan": float("nan"), "flt_max": 3.4028234663852886e38, "big": 2e38}.get(v, v)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("pair", PAIRS, ids=["%s_%s" % p if p[0] != p[1] else p[0] for p in PAIRS])
def test_check_and_agreement(world, pair):
    """One value at a time at one place on one rank (every rank in turn at worlds 2 and 3, rank 5 at world 8):
    every rank must reach the same decision and bit-identical scaler state, step counts and hyper-parameters."""
    from byteps_b200.comm.symm import VirtualCluster

    cu = _cu()
    gname, wname = pair
    gdt = DT[gname]
    es = torch.empty((), dtype=gdt).element_size()
    win = 0
    offs = [256, 256 + (_NUMEL[0] * es + 255) // 256 * 256]
    vc = VirtualCluster(world, "cuda:0", offs[1] + 4096)
    table = torch.frombuffer(bytearray(b"".join(
        struct.pack(_ENTRY_FMT, o, n, _code(gdt), _code(DT[wname]), 0, 0) for o, n in zip(offs, _NUMEL))),
        dtype=torch.uint8).cuda()
    maxvec = max(n * es // 16 for n in _NUMEL)
    ng = 2
    betas = torch.tensor([[0.9, 0.999], [0.8, 0.99]], dtype=torch.float64, device="cuda")
    states = [torch.zeros(40, dtype=torch.uint8, device="cuda") for _ in range(world)]
    steps = [torch.tensor([0, 6], dtype=torch.int32, device="cuda") for _ in range(world)]
    hps = [torch.zeros((ng, 64), dtype=torch.uint8, device="cuda") for _ in range(world)]
    for r in range(world):
        vc.arenas[r].zero_()
        states[r].copy_(torch.frombuffer(bytearray(_state_blob(1024.0, interval=3, tracker=2)), dtype=torch.uint8))

    values = ["inf", "nan", 65520.0, 65519.99, "flt_max", "big"]
    places = [(0, 0), (0, _LENS[0] - 1), (1, _LENS[1] - 1), (1, 0)]   # first, last, next to the padding
    ranks = {1: [0], 2: [0, 1], 3: [0, 1, 2], 8: [5]}[world]
    cases = [(None, None, None)] + [(v, p, r) for v in values for p in places for r in ranks]
    torch.manual_seed(0)
    grads = [[(torch.randn(n, device="cuda") * 100).to(gdt) for n in _LENS] for _ in range(world)]
    for value, place, who in cases:
        for r in range(world):
            for i, o in enumerate(offs):
                g = grads[r][i].clone()
                if who == r and place[0] == i:
                    g[place[1]] = _value(value)
                vc.arenas[r][o:o + _LENS[i] * es].view(gdt).copy_(g)
        before = [(states[r].clone(), steps[r].clone()) for r in range(world)]
        old = struct.unpack(_STATE_FMT, before[0][0].cpu().numpy().tobytes())

        def launch(r, view, arena, s):
            cu.loss_scale_check(view, table.data_ptr(), 2, maxvec, states[r].data_ptr(), s)
            cu.loss_scale_update(view, 0, win, states[r].data_ptr(), steps[r].data_ptr(), betas.data_ptr(),
                                 hps[r].data_ptr(), ng, True, s)

        vc.run(launch)
        torch.cuda.synchronize()
        found = value is not None and _trips(value, gname, wname, world)
        for r in range(1, world):
            assert torch.equal(states[r], states[0]), (value, place, who, r)
            assert torch.equal(steps[r], steps[0]), (value, place, who, r)
            assert torch.equal(hps[r], hps[0]), (value, place, who, r)
        growth, backoff, scale, interval, tracker, skipped, fl, _ = struct.unpack(
            _STATE_FMT, states[0].cpu().numpy().tobytes())
        assert fl == 0, "the local flag must be consumed"
        o_scale, o_tracker, o_skipped = old[2], old[4], old[5]
        if found:
            assert (scale, tracker, skipped) == (o_scale / 2, 0, o_skipped + 1), (value, place, who)
        else:
            grow = o_tracker + 1 == interval
            assert (scale, tracker, skipped) == (o_scale * 2 if grow else o_scale, 0 if grow else o_tracker + 1,
                                                 o_skipped), (value, place, who)
        st_prev = before[0][1].tolist()
        assert steps[0].tolist() == (st_prev if found else [s + 1 for s in st_prev]), (value, place, who)
        for gi in range(ng):
            h = struct.unpack("<9f3if3i", hps[0][gi].cpu().numpy().tobytes())
            t = st_prev[gi] + 1
            assert h[12] == _f32(1.0 / o_scale) and h[13] == int(found) and h[11] == int(t == 1), (h, value)
            b1, b2 = betas[gi].tolist()
            assert _ulp_diff(h[7], _f32(1 - b1 ** t)) <= 1 and _ulp_diff(h[8], _f32(1 - b2 ** t)) <= 1, (h, t)
        # keep the scale in a range where both branches stay exact
        if scale < 1 or scale > 2 ** 20:
            for r in range(world):
                states[r].copy_(torch.frombuffer(bytearray(_state_blob(1024.0, interval=3, tracker=tracker,
                                                                       skipped=skipped)), dtype=torch.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("eng", ["lsu", "ring"])
def test_fp16_sum_past_fp16_range_is_applied_exactly(eng):
    """8 ranks each send 10000 in one fp16 element: every local value is finite on the wire, their sum (80000) is
    not representable in fp16.  The peer-load path (the only one the bucket layer uses for an fp16 wire in this
    mode) sums in fp32, so the step is not skipped and the master moves by exactly lr * 80000 / 8 / S."""
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops.ring import RingEntry, RingTable

    cu = _cu()
    world, n, lr, S = 8, 8 * 64, 0.5, 1024.0
    goff, poff = 256, 256 + 2048
    vc = VirtualCluster(world, "cuda:0", poff + 2048 + 256)
    table = torch.frombuffer(bytearray(struct.pack(_ENTRY_FMT, goff, n, 2, 2, 0, 0)), dtype=torch.uint8).cuda()
    states = [torch.frombuffer(bytearray(_state_blob(S)), dtype=torch.uint8).cuda() for _ in range(world)]
    steps = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(world)]
    hps = [torch.frombuffer(bytearray(_opt_blob("sgd", False, dict(lr=lr, weight_decay=0.0, momentum=0.0,
                                                                     dampening=0.0, nesterov=False), 1, 1.0)),
                            dtype=torch.uint8).cuda() for _ in range(world)]
    w0 = torch.zeros(n, dtype=torch.float16, device="cuda")
    masters, moms = [], []
    for r in range(world):
        vc.arenas[r].zero_()
        g = torch.zeros(n, dtype=torch.float16, device="cuda")
        g[77] = 10000.0
        vc.arenas[r][goff:goff + 2 * n].view(torch.float16).copy_(g)
        b, e = cu.shard_units(n // 8, world, r)
        masters.append(torch.zeros(max((e - b) * 8, 8), device="cuda"))
        moms.append(torch.zeros(max((e - b) * 8, 8), device="cuda"))
    if eng == "ring":
        tables = [RingTable([RingEntry(grad_off=goff, param_off=poff, numel=n, wire=2, slot=0, kind=cu.RING_SGD,
                                       scale=1.0 / world, master=masters[r].data_ptr(), state0=moms[r].data_ptr(),
                                       hp=hps[r].data_ptr())], "cuda:0") for r in range(world)]

    def agree(r, view, arena, s):
        cu.loss_scale_check(view, table.data_ptr(), 1, n // 8, states[r].data_ptr(), s)
        cu.loss_scale_update(view, 0, 0, states[r].data_ptr(), steps[r].data_ptr(), 0, hps[r].data_ptr(), 1, False,
                             s)

    def exchange(r, view, arena, s):
        if eng == "ring":
            tables[r].launch(view, 2, s)
        else:
            cu.pushpull_fused_opt(view, 2, 2, 2, cu.OPT_SGD, 0, 0, goff, poff, n, 1.0 / world, masters[r].data_ptr(),
                                  moms[r].data_ptr(), 0, hps[r].data_ptr(), 2, 256, 0, False, s)

    # One launch kind per pass over the virtual ranks, as in the other kernel tests: the ranks share one process, so
    # a kernel loaded lazily by rank 0 while rank 0's agreement kernel waits for ranks not yet launched would wait
    # for that kernel.  (Processes of a real job each load their own modules.)
    cu.loss_scale_load_kernels()
    vc.run(agree)
    vc.run(exchange)
    torch.cuda.synchronize()
    assert all(steps[r].item() == 1 for r in range(world)), "the step must not be skipped"
    want = w0.float().clone()
    want[77] = -lr * (8 * 10000.0) / world / S
    full = torch.cat([masters[r][:(lambda b, e: (e - b) * 8)(*cu.shard_units(n // 8, world, r))] for r in range(world)])
    assert torch.equal(full, want), (full[77].item(), want[77].item())
    for r in range(world):
        assert torch.equal(vc.arenas[r][poff:poff + 2 * n].view(torch.float16), want.half())


# ---------------------------------------------------------------------------------------------------------------
# 2. a skipped step on every engine

SKIP_ENGINES = ["lsu", "tma", "ring"]
SKIP_OPTS = ["sgd", "sgd_nesterov", "adam", "adamw"]


@pytest.mark.gpu
@pytest.mark.parametrize("opt", SKIP_OPTS)
@pytest.mark.parametrize("eng", SKIP_ENGINES)
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_skipped_step_leaves_state_untouched(eng, opt, dt):
    """World 3, two buckets.  Step 1 applies, step 2 is skipped with inf/NaN gradients in the windows: every
    parameter window, master and state shard keeps its bytes, canaries included.  Step 3 applies and matches
    float64 torch.optim after 2 steps (its step count did not advance) within _fused_opt.py's bounds."""
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops.ring import RingEntry, RingTable

    cu = _cu()
    world, blocks = 3, 3
    gdt = DT[dt]
    es = torch.empty((), dtype=gdt).element_size()
    cls, kw = FUSED_OPTS[opt]
    kind = "sgd" if cls is torch.optim.SGD else "adam"
    adamw = cls is torch.optim.AdamW
    scale = 1.0 / world
    sizes = [8 * 5003, 8 * 41]
    end = 256

    def window(nbytes):
        nonlocal end
        start = end
        end = (start + nbytes + 255) // 256 * 256 + 256
        return start

    goffs = [window(n * es) for n in sizes]
    poffs = [window(n * es) for n in sizes]
    vc = VirtualCluster(world, "cuda:0", end)
    torch.manual_seed(7)
    w0 = [torch.randn(n, device="cuda").to(gdt) for n in sizes]
    ref_w = [torch.nn.Parameter(w.double()) for w in w0]
    ref_opt = cls(ref_w, **kw)
    grp = ref_opt.param_groups[0]
    uses_mom = kind == "adam" or grp["momentum"] != 0
    shard = [[cu.shard_units(n // 8, world, r) for n in sizes] for r in range(world)]
    lens = [[(e - b) * 8 for b, e in shard[r]] for r in range(world)]
    bufs = []
    for r in range(world):
        vc.arenas[r].fill_(_CANARY)
        bufs.append([])
        for i, n in enumerate(sizes):
            b, e = shard[r][i]
            bufs[r].append([_guarded(lens[r][i], w0[i][b * 8:e * 8].float()),
                            _guarded(lens[r][i], 0.0) if uses_mom else _guarded(lens[r][i]),
                            _guarded(lens[r][i], 0.0) if kind == "adam" else _guarded(lens[r][i])])
            vc.arenas[r][poffs[i]:poffs[i] + n * es].view(gdt).copy_(w0[i])
    hp_dev = torch.zeros(64, dtype=torch.uint8, device="cuda")
    code = cu.OPT_SGD if kind == "sgd" else cu.OPT_ADAM
    if eng == "ring":
        rkind = cu.RING_SGD if kind == "sgd" else cu.RING_ADAM
        tables = [RingTable([RingEntry(grad_off=goffs[i], param_off=poffs[i], numel=n, wire=_code(gdt), slot=i,
                                       kind=rkind, scale=scale, master=bufs[r][i][0][0].data_ptr(),
                                       state0=bufs[r][i][1][0].data_ptr(), state1=bufs[r][i][2][0].data_ptr(),
                                       hp=hp_dev.data_ptr()) for i, n in enumerate(sizes)], "cuda:0")
                  for r in range(world)]

    def launch(r, view, arena, s):
        if eng == "ring":
            tables[r].launch(view, blocks, s)
            return
        for i, n in enumerate(sizes):
            m, s0, s1 = (x[0].data_ptr() for x in bufs[r][i])
            if eng == "tma":
                cu.pushpull_fused_opt_tma(view, _code(gdt), code, goffs[i], poffs[i], n, scale, m, s0, s1,
                                          hp_dev.data_ptr(), blocks, 4, False, 0, s)
            else:
                cu.pushpull_fused_opt(view, _code(gdt), _code(gdt), _code(gdt), code, 0, 0, goffs[i], poffs[i], n,
                                      scale, m, s0, s1, hp_dev.data_ptr(), blocks, 256, 0, False, s)

    zeros = lambda: [torch.zeros(n, dtype=torch.float64, device="cuda") for n in sizes]  # noqa: E731
    bounds = [{k: z for k, z in zip(("w", "b", "bmag", "m", "mmag", "v", "vmag"), zs)}
              for zs in zip(*[zeros() for _ in range(7)])]
    t = 0
    for step in range(1, 4):
        skip = step == 2
        loss_scale = 256.0
        grads = [[_fused_grad(n, loss_scale).to(gdt) for n in sizes] for _ in range(world)]
        if skip:
            grads[1][0][0] = float("inf")
            grads[2][1][-1] = float("nan")
            grads[0][0][5] = -float("inf")
        for r in range(world):
            for i, n in enumerate(sizes):
                vc.arenas[r][goffs[i]:goffs[i] + n * es].view(gdt).copy_(grads[r][i])
        blob = bytearray(_opt_blob(kind, adamw, grp, t + 1, 1.0 / loss_scale))
        blob[_SKIP_OFF:_SKIP_OFF + 4] = struct.pack("<i", int(skip))
        cu.write_blob(hp_dev.data_ptr(), bytes(blob), torch.cuda.current_stream().cuda_stream)
        snap = [a.clone() for a in vc.arenas]
        snap_bufs = [[[x[0].clone() for x in b] for b in bufs[r]] for r in range(world)]
        vc.run(launch)
        torch.cuda.synchronize()
        for r in range(world):
            changed = vc.arenas[r] != snap[r]
            for i, n in enumerate(sizes):
                changed[poffs[i]:poffs[i] + n * es] &= skip     # an applied step rewrites the parameter windows
            assert not changed.any(), ("bytes changed", step, r, changed.nonzero()[:8].flatten().tolist())
            for i in range(len(sizes)):
                for which, (buf, used), old in zip(("master", "state0", "state1"), bufs[r][i], snap_bufs[r][i]):
                    assert bool((buf[used:].view(torch.int32) == -1).all()), (which, "canary", r, i)
                    if skip:
                        assert torch.equal(buf.view(torch.int32), old.view(torch.int32)), (which, "changed", r, i)
        if skip:
            continue
        t += 1
        w_prev = [p.detach().clone() for p in ref_w]
        for i, p in enumerate(ref_w):
            p.grad = torch.stack([grads[r][i].double() for r in range(world)]).sum(0) * scale / loss_scale
        ref_opt.step()
        for i, p in enumerate(ref_w):
            _advance_bounds(kind, adamw, grp, t, bounds[i], p.grad, w_prev[i], p.detach(), ref_opt.state[p])
        for i, n in enumerate(sizes):
            wins = [vc.arenas[r][poffs[i]:poffs[i] + n * es].view(gdt) for r in range(world)]
            for r in range(1, world):
                assert torch.equal(_bits(wins[r]), _bits(wins[0])), ("replicas", step, r, i)
            cat = lambda k: torch.cat([bufs[r][i][k][0][:lens[r][i]] for r in range(world)])  # noqa: E731
            master = cat(0)
            assert torch.equal(_bits(wins[0]), _bits(master.to(gdt))), ("window != round(master)", step, i)
            checks = [("master", master, ref_w[i].detach(), bounds[i]["w"])]
            st = ref_opt.state[ref_w[i]]
            if kind == "sgd":
                checks.append(("momentum", cat(1), st["momentum_buffer"], bounds[i]["b"]))
            else:
                checks += [("exp_avg", cat(1), st["exp_avg"], bounds[i]["m"]),
                           ("exp_avg_sq", cat(2), st["exp_avg_sq"], bounds[i]["v"])]
            for name, got, want, bound in checks:
                err = (got.double() - want).abs()
                bad = err > 2 * bound
                assert not bad.any(), (name, step, i, int(bad.sum()), err.max().item())


# ---------------------------------------------------------------------------------------------------------------
# 3. the scale trajectory against torch.amp.GradScaler

@pytest.mark.gpu
def test_scale_trajectory_matches_grad_scaler():
    """60 steps, growth_interval 3, world 2, overflows at chosen steps (on one rank only, alternating): the device
    scale, growth tracker and skipped count equal a GradScaler fed the same found_inf sequence, exactly."""
    from byteps_b200.comm.symm import VirtualCluster

    cu = _cu()
    world, n = 2, 64
    vc = VirtualCluster(world, "cuda:0", 4096)
    table = torch.frombuffer(bytearray(struct.pack(_ENTRY_FMT, 256, n, 0, 0, 0, 0)), dtype=torch.uint8).cuda()
    states = [torch.frombuffer(bytearray(_state_blob(2.0 ** 16, interval=3)), dtype=torch.uint8).cuda()
              for _ in range(world)]
    steps = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(world)]
    hps = [torch.zeros((1, 64), dtype=torch.uint8, device="cuda") for _ in range(world)]
    overflow = {0, 1, 2, 7, 8, 15, 16, 17, 18, 30, 31, 45, 50, 59}

    p = torch.nn.Parameter(torch.zeros(4, device="cuda"))
    sgd = torch.optim.SGD([p], lr=0.0)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 16, growth_factor=2.0, backoff_factor=0.5,
                                  growth_interval=3)
    for i in range(60):
        bad = i in overflow
        for r in range(world):
            vc.arenas[r][256:256 + 4 * n].view(torch.float32).fill_(1.0)
        if bad:
            vc.arenas[i % world][256:260].view(torch.float32).fill_(float("inf"))

        def launch(r, view, arena, s):
            cu.loss_scale_check(view, table.data_ptr(), 1, n // 4, states[r].data_ptr(), s)
            cu.loss_scale_update(view, 0, 0, states[r].data_ptr(), steps[r].data_ptr(), 0, hps[r].data_ptr(), 1,
                                 False, s)

        vc.run(launch)
        scaler.scale(torch.ones((), device="cuda"))
        p.grad = torch.full((4,), float("inf") if bad else 1.0, device="cuda")
        scaler.step(sgd)
        scaler.update()
        torch.cuda.synchronize()
        assert torch.equal(states[0], states[1])
        _, _, scale, _, tracker, skipped, _, _ = struct.unpack(_STATE_FMT, states[0].cpu().numpy().tobytes())
        want = scaler.state_dict()
        assert (scale, tracker) == (want["scale"], want["_growth_tracker"]), (i, scale, tracker, want)
        assert skipped == sum(1 for j in overflow if j <= i)
        assert steps[0].item() == i + 1 - skipped


# ---------------------------------------------------------------------------------------------------------------
# 4-5. the public API at world 1 (a process per case)

def _run(body: str, timeout=300):
    code = "import sys; sys.path.insert(0, %r)\n" % ROOT + textwrap.dedent(body)
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "DMLC_ROLE", "DMLC_NUM_WORKER", "DMLC_NUM_SERVER"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout


_API_PRELUDE = """
import copy, io, os, torch
import byteps_b200.torch as bps
from byteps_b200.torch.graph import GraphedStep
torch.backends.cuda.matmul.allow_tf32 = False
dev = "cuda"

def make(dt, seed=1):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.Tanh(), torch.nn.Linear(64, 8)).to(dev).to(dt)

def inner(kind, params):
    if kind == "sgd":
        return torch.optim.SGD(params, lr=0.05, momentum=0.9, weight_decay=1e-3)
    return torch.optim.AdamW(params, lr=1e-3, weight_decay=1e-2)

def data(dt):
    torch.manual_seed(11)
    return torch.randn(16, 32, device=dev).to(dt), torch.randint(0, 8, (16,), device=dev)

class Reference:
    # fp32 masters stepped by torch.optim under torch.amp.GradScaler; the model keeps the run's dtype
    def __init__(self, kind, model, scaler_kw, wire):
        self.model, self.wire = model, wire
        self.masters = [p.detach().float().clone().requires_grad_() for p in model.parameters()]
        self.opt = inner(kind, self.masters)
        self.scaler = torch.amp.GradScaler("cuda", **scaler_kw)
        self.skipped = 0

    def step(self, x, y):
        for p in self.model.parameters():
            p.grad = None
        loss = torch.nn.functional.cross_entropy(self.model(x).float(), y)
        self.scaler.scale(loss).backward()
        for p, m in zip(self.model.parameters(), self.masters):
            g = p.grad if self.wire is None else p.grad.to(self.wire)
            m.grad = g.float()
        s0 = self.scaler.get_scale()
        self.scaler.step(self.opt)
        self.scaler.update()
        self.skipped += int(self.scaler.get_scale() < s0)
        with torch.no_grad():
            for p, m in zip(self.model.parameters(), self.masters):
                p.copy_(m)

def stepper(model, opt, x, y):
    def step():
        opt.zero_grad()
        loss = torch.nn.functional.cross_entropy(model(x).float(), y)
        opt.scale_loss(loss).backward()
        opt.step()
        return loss
    return step
"""

API_CASES = [("float16", "sgd", "none"), ("float16", "adamw", "none"), ("float32", "sgd", "fp16"),
             ("float32", "adamw", "fp16")]


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("case", API_CASES, ids=["-".join(c) for c in API_CASES])
def test_public_api_matches_grad_scaler(case, graph):
    """init_scale 2**24 overflows the first steps; growth_interval 4 grows the scale until it overflows again.  In
    graph mode an overflow is injected on a replay by writing inf into the static input."""
    dtn, kind, comp = case
    out = _run(_API_PRELUDE + textwrap.dedent("""
    DTN, KIND, COMP, GRAPH = %r, %r, %r, %r
    bps.init()
    dt = getattr(torch, DTN)
    wire = torch.float16 if COMP == "fp16" else None
    cfg = {"init_scale": 2.0 ** 24, "growth_interval": 4}
    kw = {"init_scale": 2.0 ** 24, "growth_interval": 4}
    x, y = data(dt)
    ours, ref_model = make(dt), make(dt)
    opt = bps.DistributedOptimizer(inner(KIND, ours.parameters()), named_parameters=ours.named_parameters(),
                                   compression=getattr(bps.Compression, COMP), fused_update=True,
                                   dynamic_loss_scale=cfg)
    ref = Reference(KIND, ref_model, kw, wire)
    step = stepper(ours, opt, x, y)
    inject = {9, 17}
    if GRAPH:
        g = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams)
        for _ in range(2):
            ref.step(x, y)
        for i in range(2, 24):
            if i in inject:
                x[0, 0] = float("inf")
            g()
            ref.step(x, y)
            if i in inject:
                x[0, 0] = 1.0
    else:
        for i in range(24):
            if i in inject:
                x[0, 0] = float("inf")
            step()
            ref.step(x, y)
            if i in inject:
                x[0, 0] = 1.0
    torch.cuda.synchronize()
    assert opt.skipped_steps == ref.skipped and ref.skipped >= 3, (opt.skipped_steps, ref.skipped)
    assert opt.loss_scale == ref.scaler.get_scale(), (opt.loss_scale, ref.scaler.get_scale())
    # the two runs' updates differ in the last fp32 bits, so a 16-bit value near a rounding boundary can land one
    # ulp apart: a parameter ulp for an fp16 model, a wire ulp of the gradient (times lr) on the fp16 wire
    tol = 2e-3 if dt == torch.float16 else 2e-4
    for (n, a), b in zip(ours.named_parameters(), ref_model.parameters()):
        assert torch.isfinite(a).all(), n
        err = (a.float() - b.float()).abs().max().item()
        assert err <= tol, (n, err)
    print("OK", opt.skipped_steps, opt.loss_scale)
    bps.shutdown()
    """ % (dtn, kind, comp, graph)))
    assert "OK" in out


@pytest.mark.gpu
def test_accumulated_gradients_are_checked_at_the_step():
    """backward_passes_per_step=2: an inf in the first of the two micro-batches skips the step (the check runs on
    the accumulated gradients), and the run matches GradScaler over the same accumulated gradients."""
    out = _run(_API_PRELUDE + textwrap.dedent("""
    bps.init()
    dt = torch.float16
    x, y = data(dt)
    x[0, 0] = 1.0
    ours, ref_model = make(dt), make(dt)
    opt = bps.DistributedOptimizer(inner("sgd", ours.parameters()), named_parameters=ours.named_parameters(),
                                   fused_update=True, backward_passes_per_step=2,
                                   dynamic_loss_scale={"init_scale": 2.0 ** 20, "growth_interval": 3})
    ref = Reference("sgd", ref_model, {"init_scale": 2.0 ** 20, "growth_interval": 3}, None)
    for i in range(12):
        opt.zero_grad()
        for p in ref_model.parameters():
            p.grad = None
        for micro in range(2):
            xm = x.clone()
            if i == 7 and micro == 0:
                xm[0, 0] = float("inf")
            opt.scale_loss(torch.nn.functional.cross_entropy(ours(xm).float(), y)).backward()
            ref.scaler.scale(torch.nn.functional.cross_entropy(ref_model(xm).float(), y)).backward()
        opt.step()
        for p, m in zip(ref_model.parameters(), ref.masters):
            m.grad = p.grad.float()
        s0 = ref.scaler.get_scale()
        ref.scaler.step(ref.opt)
        ref.scaler.update()
        ref.skipped += int(ref.scaler.get_scale() < s0)
        with torch.no_grad():
            for p, m in zip(ref_model.parameters(), ref.masters):
                p.copy_(m)
    torch.cuda.synchronize()
    assert opt.skipped_steps == ref.skipped and ref.skipped >= 2, (opt.skipped_steps, ref.skipped)
    assert opt.loss_scale == ref.scaler.get_scale()
    for (n, a), b in zip(ours.named_parameters(), ref_model.parameters()):
        err = (a.float() - b.float()).abs().max().item()
        assert err <= 2e-3, (n, err)
    print("OK", opt.skipped_steps)
    bps.shutdown()
    """))
    assert "OK" in out


@pytest.mark.gpu
def test_checkpoint_after_a_skipped_step():
    """fp16 AdamW.  Run A takes 10 steps; run B takes 4 (the 4th skipped), saves, and a fresh model and optimizer
    load and take 6 more: parameters and scaler equal A's bit for bit.  The scaler entry loads into
    torch.amp.GradScaler, the Adam state into torch.optim.AdamW with the applied-step count, and a checkpoint without
    the entry leaves the scaler at its initial values."""
    out = _run(_API_PRELUDE + textwrap.dedent("""
    bps.init()
    dt = torch.float16
    cfg = {"init_scale": 2.0 ** 15, "growth_interval": 2}
    x, y = data(dt)
    x[0, 0] = 1.0
    def run(model):
        return bps.DistributedOptimizer(inner("adamw", model.parameters()), named_parameters=model.named_parameters(),
                                        fused_update=True, dynamic_loss_scale=cfg)
    def save(obj):
        b = io.BytesIO(); torch.save(obj, b); b.seek(0)
        return torch.load(b, weights_only=False)
    ma = make(dt); oa = run(ma)
    for i in range(10):
        if i == 3:
            x[0, 0] = float("inf")
        stepper(ma, oa, x, y)()
        x[0, 0] = 1.0
    mb = make(dt); ob = run(mb)
    for i in range(4):
        if i == 3:
            x[0, 0] = float("inf")
        stepper(mb, ob, x, y)()
    x[0, 0] = 1.0
    assert ob.skipped_steps >= 1
    ckpt = save({"model": mb.state_dict(), "optimizer": ob.state_dict()})
    sd = ckpt["optimizer"]
    applied = 4 - ob.skipped_steps
    assert sorted(sd["loss_scaler"]) == ["_growth_tracker", "backoff_factor", "growth_factor", "growth_interval",
                                         "scale"], sd["loss_scaler"]
    gs = torch.amp.GradScaler("cuda")
    gs.load_state_dict(sd["loss_scaler"])
    assert gs.get_scale() == ob.loss_scale and gs.get_growth_interval() == 2
    assert all(float(e["step"]) == applied for e in sd["state"].values()), (applied, sd["state"][0]["step"])
    tm = [torch.nn.Parameter(p.detach().float().clone()) for p in mb.parameters()]
    ta = torch.optim.AdamW(tm, lr=1e-3, weight_decay=1e-2)
    ta.load_state_dict({"state": sd["state"], "param_groups": sd["param_groups"]})
    assert float(ta.state[tm[0]]["step"]) == applied
    mc = make(dt, seed=2); oc = run(mc)
    mc.load_state_dict(ckpt["model"])
    oc.load_state_dict(sd)
    assert oc.loss_scale == ob.loss_scale
    for _ in range(6):
        stepper(mc, oc, x, y)()
    torch.cuda.synchronize()
    for (n, a), c in zip(ma.named_parameters(), mc.parameters()):
        assert torch.equal(a, c), (n, (a.float() - c.float()).abs().max().item())
    assert oa.loss_scale == oc.loss_scale
    assert oa.state_dict()["loss_scaler"] == oc.state_dict()["loss_scaler"]
    md = make(dt, seed=3); od = run(md)
    for _ in range(3):
        stepper(md, od, x, y)()
    nols = dict(sd); del nols["loss_scaler"]
    od.load_state_dict(nols)
    assert od.loss_scale == cfg["init_scale"] and od.state_dict()["loss_scaler"]["_growth_tracker"] == 0
    print("OK")
    bps.shutdown()
    """))
    assert "OK" in out


# ---------------------------------------------------------------------------------------------------------------
# 6. two processes

def _two_ranks(rank, world):
    import byteps_b200.torch as bps

    torch.cuda.set_device(rank)
    bps.init()
    torch.manual_seed(1)
    model = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.Tanh(), torch.nn.Linear(64, 8)).cuda().half()
    opt = bps.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9),
                                   named_parameters=model.named_parameters(), fused_update=True,
                                   dynamic_loss_scale={"init_scale": 1024.0})
    bps.broadcast_parameters(model.state_dict(), root_rank=0)
    torch.manual_seed(10 + rank)
    x, y = torch.randn(16, 32, device="cuda").half(), torch.randint(0, 8, (16,), device="cuda")
    for i in range(6):
        if i == 3 and rank == 1:
            x[0, 0] = float("inf")
        before = [p.detach().clone() for p in model.parameters()]
        opt.zero_grad()
        opt.scale_loss(torch.nn.functional.cross_entropy(model(x).float(), y)).backward()
        opt.step()
        torch.cuda.synchronize()
        if i == 3:
            x[0, 0] = 1.0
            assert all(torch.equal(a, b) for a, b in zip(before, model.parameters())), "rank %d did not skip" % rank
    assert opt.skipped_steps == 1 and opt.loss_scale == 512.0, (opt.skipped_steps, opt.loss_scale)
    flat = torch.cat([p.detach().float().flatten() for p in model.parameters()])
    both = bps.push_pull(flat.clone(), average=False, name="replica_check")
    assert torch.equal(both, 2 * flat), "replicas differ"
    bps.shutdown()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_processes_skip_together():
    from _mp import run_workers

    run_workers(_two_ranks, world=2, timeout=300)


# ---------------------------------------------------------------------------------------------------------------
# 7. argument checks (CPU)

@pytest.mark.parametrize("option,fused", [
    ({"init_scales": 2.0}, True),
    ({"init_scale": float("inf")}, True),
    ({"init_scale": float("nan")}, True),
    ({"init_scale": 0.0}, True),
    ({"init_scale": -1.0}, True),
    ({"init_scale": 1e39}, True),          # not finite as the float32 the device holds
    ({"init_scale": 1e-50}, True),         # 0 as a float32
    ({"init_scale": 1e-45}, True),         # a float32 whose reciprocal is not finite
    ({"growth_factor": 1.0}, True),
    ({"growth_factor": 0.5}, True),
    ({"backoff_factor": 0.0}, True),
    ({"backoff_factor": 1.0}, True),
    ({"backoff_factor": 1.5}, True),
    ({"growth_interval": 0}, True),
    ({"growth_interval": 2.5}, True),
    (True, False),
], ids=lambda v: str(v))
def test_invalid_options_raise(option, fused):
    import byteps_b200.torch as bps

    p = torch.nn.Parameter(torch.zeros(4))
    with pytest.raises(ValueError):
        bps.DistributedOptimizer(torch.optim.SGD([p], lr=0.1), fused_update=fused, dynamic_loss_scale=option)


def test_option_needs_the_symmetric_memory_path():
    """CPU parameters never take the fused symmetric-memory path: the option is refused, not ignored."""
    import byteps_b200.torch as bps

    bps.init()
    try:
        p = torch.nn.Parameter(torch.zeros(4))
        with pytest.raises(ValueError, match="symmetric-memory"):
            bps.DistributedOptimizer(torch.optim.SGD([p], lr=0.1), fused_update=True, dynamic_loss_scale=True)
    finally:
        bps.shutdown()


def test_defaults_are_grad_scalers():
    from byteps_b200.torch import _loss_scale_config

    s = torch.amp.GradScaler("cpu") if hasattr(torch.amp, "GradScaler") else None
    cfg = _loss_scale_config(True)
    assert cfg == {"init_scale": 65536.0, "growth_factor": 2.0, "backoff_factor": 0.5, "growth_interval": 2000}
    if s is not None:
        assert (s._init_scale, s._growth_factor, s._backoff_factor, s._growth_interval) == tuple(cfg.values())
    assert _loss_scale_config(False) is None
    assert _loss_scale_config({"growth_interval": 3})["growth_interval"] == 3
    assert math.isclose(_loss_scale_config({"backoff_factor": 0.25})["backoff_factor"], 0.25)


@pytest.mark.parametrize("entry", [
    {"scale": 0.0}, {"scale": float("inf")}, {"scale": 1e-50}, {"growth_interval": 0}, {"backoff_factor": 1.0},
    {"growth_factor": 1.0}, {"_growth_tracker": -1}, {"_growth_tracker": 2000}, {"_growth_tracker": 1.5},
    {"scale": None},
], ids=lambda v: str(v))
def test_loaded_scaler_entries_are_checked(entry):
    from byteps_b200.torch import _checked_scaler_entry

    good = {"scale": 1024.0, "growth_factor": 2.0, "backoff_factor": 0.5, "growth_interval": 2000,
            "_growth_tracker": 7}
    assert _checked_scaler_entry(good) == (1024.0, 2.0, 0.5, 2000, 7)
    bad = dict(good, **entry)
    if entry == {"scale": None}:
        del bad["scale"]
    with pytest.raises(ValueError):
        _checked_scaler_entry(bad)


def test_fp16_wire_keeps_off_the_in_switch_reduction():
    """With dynamic loss scaling an fp16 wire is summed by peer loads in fp32, never by multimem.ld_reduce, which
    returns the sum in fp16; other wires, and every wire without the option, keep NVLS when it is available."""
    from types import SimpleNamespace

    from byteps_b200.parallel.bucket import BucketedGradSync

    def nvls(scaler, wire, available=True):
        fake = SimpleNamespace(ctx=SimpleNamespace(nvls=available), loss_scaler=scaler)
        return BucketedGradSync._nvls_for(fake, wire)

    on = {"init_scale": 1.0}
    assert not nvls(on, torch.float16)
    assert nvls(on, torch.bfloat16) and nvls(on, torch.float32)
    assert nvls(None, torch.float16) and nvls(None, torch.bfloat16)
    assert not nvls(None, torch.float16, available=False)
