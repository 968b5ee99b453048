"""Checkpoints of the fused optimizer (``DistributedOptimizer(..., fused_update=True)``).

Its state lives in the exchange's sharded fp32 buffers.  ``state_dict()`` gathers it into torch.optim's format
(plus ``master_param`` for 16-bit parameters) and ``load_state_dict()`` puts a full state back into each rank's
shard.  The CPU tests check the one function that maps a bucket's flat shard layout to per-parameter tensors.
The GPU tests check that a save / restore in the middle of a run continues bit for bit, that checkpoints move
between the fused optimizer and torch.optim, that ``broadcast_optimizer_state`` restores a root-only load, and
(two GPUs) that checkpoints move between world sizes.  Each single-GPU case is its own process so
init()/shutdown() state never leaks between tests.
"""
import os
import subprocess
import sys
import textwrap

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------- layout (CPU)
def _param(shape, channels_last=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(shape, generator=g)
    return t.contiguous(memory_format=torch.channels_last) if channels_last else t


LAYOUTS = {
    # channels_last conv weights, ragged sizes (padding inside the bucket), a 1-element bias
    "mixed": [((64, 3, 7, 7), True), ((13,), False), ((5, 3), False), ((1,), False), ((16, 8, 3, 3), True),
              ((7, 1, 1, 5), True), ((203,), False)],
    # one 8-element unit: at world > 1 every rank but the first owns an empty shard
    "tiny": [((5,), False)],
    # a few units: at world 8 the trailing ranks own empty shards
    "small": [((2, 3, 2, 2), True), ((9,), False)],
}


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_bucket_state_layout_roundtrip(layout, world):
    from byteps_b200.parallel.bucket import _pad8, _strided_view, copy_bucket_state, shard_bounds

    params = [_param(s, cl, seed=i) for i, (s, cl) in enumerate(LAYOUTS[layout])]
    starts, numel = [], 0
    for p in params:
        starts.append(numel)
        numel += _pad8(p.numel())
    # the bucket as the exchange lays it out (through the same views the parameters become)
    bucket = torch.zeros(numel)
    for p, st in zip(params, starts):
        _strided_view(bucket, p, st).copy_(p)
    shards = []
    for r in range(world):
        s0, s1 = shard_bounds(numel, world, r)
        shard = torch.full((max(s1 - s0, 8),), float("nan"))      # the exchange allocates at least 8
        copy_bucket_state(shard, (s0, s1), starts, params, to_shard=True)
        assert torch.equal(shard[:s1 - s0], bucket[s0:s1]), r
        assert not shard[s1 - s0:].any(), "the tail of an over-allocated shard must be zero"
        shards.append((s0, s1, shard))
    # the shards tile the bucket, padding included, and the padding is zero
    assert shards[0][0] == 0 and shards[-1][1] == numel
    assert all(a[1] == b[0] for a, b in zip(shards, shards[1:]))
    flat = torch.cat([sh[:s1 - s0] for s0, s1, sh in shards])
    assert torch.equal(flat.view(torch.int32), bucket.view(torch.int32))
    covered = torch.zeros(numel, dtype=torch.bool)
    for p, st in zip(params, starts):
        covered[st:st + p.numel()] = True
    assert not flat[~covered].any()
    # gather every shard back into tensors with the parameters' shapes and strides
    outs = [torch.full_like(p, float("nan"), memory_format=torch.preserve_format) for p in params]
    for s0, s1, sh in shards:
        copy_bucket_state(sh, (s0, s1), starts, outs, to_shard=False)
    for p, o in zip(params, outs):
        assert o.shape == p.shape and o.stride() == p.stride()
        assert torch.equal(o.view(torch.int32), p.view(torch.int32))


def test_bucket_state_layout_logical_indices():
    """A channels_last weight sits in the bucket in NHWC order; the gathered tensor holds each value at its
    logical (n, c, h, w) index, whatever strides the receiving tensor has."""
    from byteps_b200.parallel.bucket import _pad8, _strided_view, copy_bucket_state

    p = torch.arange(2 * 3 * 2 * 2, dtype=torch.float32).view(2, 3, 2, 2).contiguous(memory_format=torch.channels_last)
    bucket = torch.zeros(_pad8(p.numel()))
    _strided_view(bucket, p, 0).copy_(p)
    assert torch.equal(bucket[:p.numel()], p.permute(0, 2, 3, 1).reshape(-1))
    out = torch.empty_like(p, memory_format=torch.preserve_format)
    copy_bucket_state(bucket, (0, bucket.numel()), [0], [out], to_shard=False)
    assert torch.equal(out, p) and out.stride() == p.stride()


def test_shard_bounds_match_the_exchange():
    """The per-rank shard of the fused optimizer: 8-element units, ceil-divided, trailing ranks empty."""
    from byteps_b200.parallel.bucket import shard_bounds

    assert [shard_bounds(24, 8, r) for r in range(8)] == [(0, 8), (8, 16), (16, 24)] + [(24, 24)] * 5
    assert [shard_bounds(40, 3, r) for r in range(3)] == [(0, 16), (16, 32), (32, 40)]
    assert shard_bounds(48, 1, 0) == (0, 48)


class _TwoRankEngine:
    """Stands in for the engine of one of two ranks: records what export_state pushes and, given the other
    rank's record, adds it the way the host all-reduce does."""

    def __init__(self, peer=None):
        self.peer, self.seen = peer, {}

    def push_pull_async(self, t, out, average, name):
        assert t.dtype == torch.int32 and not t.is_cuda and out is t and not average
        self.seen[name] = t.clone()
        if self.peer is not None:
            t.add_(self.peer[name])
        return 0

    def synchronize(self, h):
        pass


def test_export_state_sums_bit_patterns_exactly():
    """At world > 1 export_state sums the ranks' zero-padded shards as int32 bit patterns on the host, so every
    value comes back bit for bit (a negative zero and a NaN payload included) whatever float wire the device
    exchange would use."""
    from byteps_b200.parallel.bucket import Bucket, BucketedGradSync, _pad8, copy_bucket_state, shard_bounds

    params = [_param((8, 4, 3, 3), True, seed=1), _param((13,), seed=2), _param((5,), seed=3)]
    vals = [_param(tuple(p.shape), p.dim() == 4, seed=10 + i) for i, p in enumerate(params)]
    vals[1][0] = -0.0
    vals[1][1] = torch.tensor(0x7FC12345, dtype=torch.int32).view(torch.float32)

    def sync(rank, engine):
        s = object.__new__(BucketedGradSync)
        s.world, s.rank, s.fused, s.engine = 2, rank, "sgd", engine
        b = Bucket(0, 0, torch.float32)
        for p in params:
            b.params.append(p)
            b.starts.append(b.numel)
            b.numel += _pad8(p.numel())
        s0, s1 = shard_bounds(b.numel, 2, rank)
        b.master, b.state0 = torch.zeros(max(s1 - s0, 8)), torch.zeros(max(s1 - s0, 8))
        copy_bucket_state(b.master, (s0, s1), b.starts, params, to_shard=True)
        copy_bucket_state(b.state0, (s0, s1), b.starts, vals, to_shard=True)
        s.buckets = [b]
        return s

    e1 = _TwoRankEngine()
    sync(1, e1).export_state()
    out = sync(0, _TwoRankEngine(peer=e1.seen)).export_state()
    for p, v in zip(params, vals):
        for key, want in (("master", p), ("state0", v)):
            got = out[p][key]
            assert got.shape == p.shape and got.stride() == p.stride()
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), key


# ---------------------------------------------------------------------------------------------- GPU, world 1
def _run(body: str, timeout=400, env=None, prelude=True):
    code = "import sys; sys.path.insert(0, %r)\n" % ROOT + (PRELUDE if prelude else "") + textwrap.dedent(body)
    e = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "DMLC_ROLE", "DMLC_NUM_WORKER", "DMLC_NUM_SERVER",
              "BYTEPS_FUSED_ENGINE"):
        e.pop(k, None)
    e.update(env or {})
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, env=e)
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout


# a conv layer and ragged linear layers; optimizers as the fused kernels support them.  The conv weight stays
# contiguous: a channels_last parameter's arena view is placed from the start of the arena, not of its bucket
# window (_strided_view ignores the window's storage offset), so fused training of such a parameter does not
# follow torch.optim yet.  The CPU tests cover the channels_last layout of the checkpoint itself.
PRELUDE = """
import io, os
import torch
import torch.nn.functional as F
import byteps_b200.torch as bps
from byteps_b200.torch.graph import GraphedStep

def make(dt, seed=1):
    torch.manual_seed(seed)
    m = torch.nn.Sequential(torch.nn.Conv2d(4, 8, 3, padding=1), torch.nn.ReLU(), torch.nn.Flatten(),
                            torch.nn.Linear(288, 13), torch.nn.Tanh(), torch.nn.Linear(13, 5))
    return m.cuda().to(dt)

def mk(kind, params):
    if kind == "sgd_nesterov":
        return torch.optim.SGD(params, lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-3)
    if kind == "adam":
        return torch.optim.Adam(params, lr=1e-2, weight_decay=1e-2)
    return torch.optim.AdamW(params, lr=1e-2, weight_decay=1e-2)

def fused(kind, m, comp="none"):
    return bps.DistributedOptimizer(mk(kind, m.parameters()), named_parameters=m.named_parameters(),
                                    compression=getattr(bps.Compression, comp), fused_update=True)

def data(dt, n=16, seed=7):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, 4, 6, 6, device="cuda", generator=g).to(dt)
    return x, torch.randint(0, 5, (n,), device="cuda", generator=g)

def stepper(m, o, x, y):
    def step():
        o.zero_grad()
        loss = F.cross_entropy(m(x).float(), y)
        loss.backward()
        o.step()
        return loss
    return step

def roundtrip(obj):
    buf = io.BytesIO()
    torch.save(obj, buf)
    buf.seek(0)
    return torch.load(buf)

def same_state(a, b):
    assert a["param_groups"] == b["param_groups"]
    assert sorted(a["state"]) == sorted(b["state"])
    for i in a["state"]:
        assert sorted(a["state"][i]) == sorted(b["state"][i]), (i, sorted(a["state"][i]), sorted(b["state"][i]))
        for k, v in a["state"][i].items():
            assert torch.equal(v, b["state"][i][k]), (i, k)
"""

# (model dtype, fused engine, wire): TMA is the world-1 default; lsu is the register kernel; an fp32 model on a
# bf16 wire goes through the register kernel's pack path
RESUME_CONFIGS = [("float32", "tma", "none"), ("bfloat16", "tma", "none"), ("float32", "lsu", "none"),
                  ("bfloat16", "lsu", "none"), ("float32", "auto", "bf16")]


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("optim", ["sgd_nesterov", "adam", "adamw"])
def test_resume_is_bit_identical(optim, graph):
    """Run A takes 6 steps.  Run B takes 3, saves model + optimizer through torch.save, builds a fresh model and
    optimizer, loads and takes 3 more.  Final parameters and exported state equal A's exactly.  In graph mode B's
    continuation replays a CUDA graph captured before the load (its warm-up step runs on the fresh weights)."""
    out = _run("""
    KIND, GRAPH, CONFIGS = %r, %r, %r
    bps.init()
    for dtn, engine, comp in CONFIGS:
        os.environ["BYTEPS_FUSED_ENGINE"] = engine
        dt = getattr(torch, dtn)
        x, y = data(dt)
        ma = make(dt); oa = fused(KIND, ma, comp)
        for _ in range(6):
            stepper(ma, oa, x, y)()
        sda = oa.state_dict()
        mb = make(dt); ob = fused(KIND, mb, comp)
        for _ in range(3):
            stepper(mb, ob, x, y)()
        ckpt = roundtrip({"model": mb.state_dict(), "optimizer": ob.state_dict()})
        mc = make(dt, seed=2); oc = fused(KIND, mc, comp)
        g = GraphedStep(stepper(mc, oc, x, y), warmup=1, pre_replay=oc.refresh_hparams) if GRAPH else None
        mc.load_state_dict(ckpt["model"])
        oc.load_state_dict(ckpt["optimizer"])
        for _ in range(3):
            g() if GRAPH else stepper(mc, oc, x, y)()
        torch.cuda.synchronize()
        for (n, a), c in zip(ma.named_parameters(), mc.parameters()):
            assert torch.equal(a, c), (dtn, engine, comp, n, (a.float() - c.float()).abs().max().item())
        sdc = oc.state_dict()
        same_state(sda, sdc)
        want = {"sgd_nesterov": ["momentum_buffer"], "adam": ["exp_avg", "exp_avg_sq", "step"]}.get(
            KIND, ["exp_avg", "exp_avg_sq", "step"])
        if dt != torch.float32:
            want = sorted(want + ["master_param"])
        assert all(sorted(e) == want for e in sdc["state"].values()), sdc["state"][0].keys()
        assert len(sdc["state"]) == len(list(mc.parameters()))
        print("config ok", dtn, engine, comp)
    print("OK")
    bps.shutdown()
    """ % (optim, graph, RESUME_CONFIGS))
    assert out.count("config ok") == len(RESUME_CONFIGS) and "OK" in out


@pytest.mark.gpu
@pytest.mark.parametrize("optim", ["sgd_nesterov", "adam", "adamw"])
def test_interchange_with_torch_optim(optim):
    """fp32 model.  A fused state_dict() has torch's keys, shapes, strides and dtypes after the same steps, loads
    into torch.optim and agrees with torch's own state.  A torch.optim checkpoint loaded into the fused optimizer
    gives the next update torch gives: SGD's momentum continues, Adam's bias correction continues at t + 1."""
    out = _run("""
    KIND = %r
    bps.init()
    dt = torch.float32
    x, y = data(dt)
    ref, ours = make(dt), make(dt)
    ropt, oopt = mk(KIND, ref.parameters()), fused(KIND, ours)
    for _ in range(3):
        stepper(ref, ropt, x, y)()
        stepper(ours, oopt, x, y)()
    torch.cuda.synchronize()
    sdr, sdo = ropt.state_dict(), roundtrip(oopt.state_dict())
    assert sdr["param_groups"] == sdo["param_groups"]
    assert sorted(sdr["state"]) == sorted(sdo["state"])
    for i, ent in sdr["state"].items():
        assert list(ent) == list(sdo["state"][i]), (list(ent), list(sdo["state"][i]))
        for k, v in ent.items():
            o = sdo["state"][i][k]
            assert o.dtype == v.dtype and o.shape == v.shape, (k, o.dtype, v.dtype, o.shape, v.shape)
            if v.dim():
                assert o.stride() == v.stride(), (k, o.stride(), v.stride())
                # the two runs' weights differ in the last fp32 bits after step 1 (test_gpu_api's bound is 2e-5)
                err = (o - v.cpu()).abs().max().item()
                assert err <= 1e-4 * v.abs().max().item() + 1e-9, (i, k, err, v.abs().max().item())
            else:
                assert torch.equal(o, v.cpu()), (k, o, v)
    # the fused checkpoint drives a plain torch.optim optimizer
    m2 = make(dt); m2.load_state_dict(ours.state_dict())
    o2 = mk(KIND, m2.parameters())
    o2.load_state_dict(sdo)
    stepper(m2, o2, x, y)()
    stepper(ref, ropt, x, y)()
    for a, b in zip(ref.parameters(), m2.parameters()):
        assert (a - b).abs().max().item() < 2e-5
    # and a torch.optim checkpoint drives the fused optimizer: one more step on both sides from equal weights
    m3 = make(dt); m3.load_state_dict(ref.state_dict())
    o3 = fused(KIND, m3)
    o3.load_state_dict(roundtrip(ropt.state_dict()))
    w0 = [p.detach().clone() for p in ref.parameters()]
    stepper(ref, ropt, x, y)()
    stepper(m3, o3, x, y)()
    torch.cuda.synchronize()
    for a, b, w in zip(ref.parameters(), m3.parameters(), w0):
        upd = (a - w).abs().max().item()
        err = (a - b).abs().max().item()
        assert err < 2e-5 and err < 1e-2 * upd, (err, upd)
    # a restart (t = 1, first momentum step) would move these weights by a different amount
    print("OK")
    bps.shutdown()
    """ % optim)
    assert "OK" in out


@pytest.mark.gpu
def test_broadcast_restores_loaded_state_and_options():
    """bf16 model, Adam.  load_state_dict, then the documented broadcast_parameters -> broadcast_optimizer_state:
    broadcast_parameters re-derives the masters from the bf16 weights, broadcast_optimizer_state puts the loaded
    fp32 masters back, applies the saved options (a changed lr) and drops the full copies."""
    out = _run("""
    bps.init()
    dt = torch.bfloat16
    x, y = data(dt)
    # before its first step a 16-bit Adam has no entries (torch.optim.Adam creates its state only for a parameter
    # without any), and torch.optim.Adam can load that and step
    m0 = make(dt); o0 = fused("adam", m0)
    sd0 = roundtrip(o0.state_dict())
    assert sd0["state"] == {}, sd0["state"]
    mt = make(dt); t0 = mk("adam", mt.parameters())
    t0.load_state_dict(sd0)
    stepper(mt, t0, x, y)()
    ma = make(dt); oa = fused("adam", ma)
    for _ in range(3):
        stepper(ma, oa, x, y)()
    ckpt = roundtrip({"model": ma.state_dict(), "optimizer": oa.state_dict()})
    ckpt["optimizer"]["param_groups"][0]["lr"] = 3e-3
    want = oa.state_dict()
    want["param_groups"][0]["lr"] = 3e-3
    for grp in oa.param_groups:
        grp["lr"] = 3e-3
    oa.grad_sync.refresh_hparams()                     # eager step() publishes the next step's options at its end
    for _ in range(2):
        stepper(ma, oa, x, y)()
    torch.cuda.synchronize()
    # broadcast_parameters re-derives the masters of every live fused optimizer: record A before any broadcast
    want_w = [p.detach().clone() for p in ma.parameters()]
    want_after = oa.state_dict()
    mb = make(dt, seed=2); base = mk("adam", mb.parameters()); ob = bps.DistributedOptimizer(
        base, named_parameters=mb.named_parameters(), fused_update=True)
    mb.load_state_dict(ckpt["model"])
    ob.load_state_dict(ckpt["optimizer"])
    assert ob.state, "the loaded full state waits for broadcast_optimizer_state"
    assert base.param_groups[0]["lr"] == 3e-3 and ob.grad_sync.param_groups[0]["lr"] == 3e-3
    bps.broadcast_parameters(mb.state_dict(), root_rank=0)
    bps.broadcast_optimizer_state(ob, root_rank=0)
    assert not ob.state
    assert ob.param_groups[0]["lr"] == 3e-3 and base.param_groups[0]["lr"] == 3e-3
    got = ob.state_dict()
    same_state(want, got)
    # masters really differ from the bf16 weights, so re-deriving them would have been visible
    assert any(not torch.equal(e["master_param"], p.detach().float().cpu())
               for e, p in zip(got["state"].values(), mb.parameters()))
    for _ in range(2):
        stepper(mb, ob, x, y)()
    torch.cuda.synchronize()
    for a, b in zip(want_w, mb.parameters()):
        assert torch.equal(a, b)
    same_state(want_after, ob.state_dict())
    # a broadcast with nothing loaded keeps the live moments, steps and the root's options; like every
    # broadcast_parameters call, the pickled options' exchange re-derives the masters from the bf16 weights
    ob.param_groups[0]["lr"] = 1e-3
    bps.broadcast_optimizer_state(ob, root_rank=0)
    want_after["param_groups"][0]["lr"] = 1e-3
    for e, p in zip(want_after["state"].values(), mb.parameters()):
        e["master_param"] = p.detach().float().cpu()
    same_state(want_after, ob.state_dict())
    # a load no broadcast consumes is dropped by the next step: a later broadcast offers the live state
    ob.load_state_dict(ob.state_dict())
    assert ob.state
    stepper(mb, ob, x, y)()
    assert not ob.state
    # Adam step counts must agree within a param group
    bad = ob.state_dict()
    bad["state"][0]["step"] = torch.tensor(9.0)
    try:
        ob.load_state_dict(bad)
        raise SystemExit("mismatched Adam steps were accepted")
    except ValueError:
        pass
    print("OK")
    bps.shutdown()
    """)
    assert "OK" in out


# ---------------------------------------------------------------------------------------------- two GPUs
def _two_gpu_checkpoints(rank, world, ckpt_dir):
    """Save at world 2 and restore at world 2 (rank 0 loads, then the broadcasts): the continuation is bit
    identical.  Load the world-1 checkpoint at world 2: every rank's exported state equals it."""
    import torch.nn.functional as F

    import byteps_b200.torch as bps

    torch.cuda.set_device(rank)
    bps.init()
    dt = torch.bfloat16

    def make():
        torch.manual_seed(1)
        m = torch.nn.Sequential(torch.nn.Conv2d(4, 8, 3, padding=1), torch.nn.ReLU(), torch.nn.Flatten(),
                                torch.nn.Linear(288, 13), torch.nn.Tanh(), torch.nn.Linear(13, 5))
        return m.cuda().to(dt)

    def opt(m):
        return bps.DistributedOptimizer(torch.optim.Adam(m.parameters(), lr=1e-2, weight_decay=1e-2),
                                        named_parameters=m.named_parameters(), fused_update=True)

    torch.manual_seed(7)
    x = torch.randn(world * 8, 4, 6, 6, device="cuda").to(dt)
    y = torch.randint(0, 5, (world * 8,), device="cuda")
    x, y = x[rank * 8:(rank + 1) * 8], y[rank * 8:(rank + 1) * 8]

    def step(m, o):
        o.zero_grad()
        F.cross_entropy(m(x).float(), y).backward()
        o.step()

    def equal_state(a, b):
        assert sorted(a["state"]) == sorted(b["state"])
        for i, ent in a["state"].items():
            for k, v in ent.items():
                assert torch.equal(v, b["state"][i][k]), (i, k)

    ma = make()
    oa = opt(ma)
    bps.broadcast_parameters(ma.state_dict(), root_rank=0)
    for _ in range(6):
        step(ma, oa)
    sda = oa.state_dict()                                  # collective
    mb = make()
    ob = opt(mb)
    bps.broadcast_parameters(mb.state_dict(), root_rank=0)
    for _ in range(3):
        step(mb, ob)
    sdb = ob.state_dict()                                  # every rank calls it, rank 0 saves
    path = os.path.join(ckpt_dir, "w2.pt")
    if rank == 0:
        torch.save({"model": mb.state_dict(), "optimizer": sdb}, path)
    mc = make()
    oc = opt(mc)
    if rank == 0:
        ck = torch.load(path)
        mc.load_state_dict(ck["model"])
        oc.load_state_dict(ck["optimizer"])
    bps.broadcast_parameters(mc.state_dict(), root_rank=0)
    bps.broadcast_optimizer_state(oc, root_rank=0)
    equal_state(sdb, oc.state_dict())
    for _ in range(3):
        step(mc, oc)
    torch.cuda.synchronize()
    for a, c in zip(ma.parameters(), mc.parameters()):
        assert torch.equal(a, c)
    equal_state(sda, oc.state_dict())
    # the world-1 checkpoint
    ck1 = torch.load(os.path.join(ckpt_dir, "w1.pt"))
    md = make()
    od = opt(md)
    if rank == 0:
        md.load_state_dict(ck1["model"])
        od.load_state_dict(ck1["optimizer"])
    bps.broadcast_parameters(md.state_dict(), root_rank=0)
    bps.broadcast_optimizer_state(od, root_rank=0)
    equal_state(ck1["optimizer"], od.state_dict())
    step(md, od)
    bps.shutdown()


W1_BODY = """
    import torch, torch.nn.functional as F
    import byteps_b200.torch as bps
    bps.init()
    DIR, LOAD = %r, %r
    dt = torch.bfloat16
    def make():
        torch.manual_seed(1)
        m = torch.nn.Sequential(torch.nn.Conv2d(4, 8, 3, padding=1), torch.nn.ReLU(), torch.nn.Flatten(),
                                torch.nn.Linear(288, 13), torch.nn.Tanh(), torch.nn.Linear(13, 5))
        return m.cuda().to(dt)
    m = make()
    o = bps.DistributedOptimizer(torch.optim.Adam(m.parameters(), lr=1e-2, weight_decay=1e-2),
                                 named_parameters=m.named_parameters(), fused_update=True)
    torch.manual_seed(7)
    x = torch.randn(8, 4, 6, 6, device="cuda").to(dt)
    y = torch.randint(0, 5, (8,), device="cuda")
    if LOAD:
        ck = torch.load(DIR + "/w2.pt")
        m.load_state_dict(ck["model"])
        o.load_state_dict(ck["optimizer"])
        got = o.state_dict()
        for i, ent in ck["optimizer"]["state"].items():
            for k, v in ent.items():
                assert torch.equal(v, got["state"][i][k]), (i, k)
    for _ in range(2):
        o.zero_grad()
        F.cross_entropy(m(x).float(), y).backward()
        o.step()
    if not LOAD:
        torch.save({"model": m.state_dict(), "optimizer": o.state_dict()}, DIR + "/w1.pt")
    print("OK")
    bps.shutdown()
"""


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("wire", ["", "bf16", "fp16"], ids=["fp32_wire", "bf16_wire", "fp16_wire"])
def test_checkpoint_across_world_sizes(tmp_path, wire):
    """BYTEPS_WIRE_DTYPE casts float32 push_pulls on the device; the exported state must not go through it: the
    checks are bit-exact under every wire setting."""
    from _mp import run_workers

    env = {"BYTEPS_WIRE_DTYPE": wire}
    assert "OK" in _run(W1_BODY % (str(tmp_path), False), prelude=False, env=env)
    run_workers(_two_gpu_checkpoints, world=2, args=(str(tmp_path),), env=env, timeout=400)
    assert "OK" in _run(W1_BODY % (str(tmp_path), True), prelude=False, env=env)
