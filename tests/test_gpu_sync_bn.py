"""Synchronised batch norm (ops/bn_act.py::SyncBatchNormAct2d, kernels/bn_act.cu::bn_sync_kernel).

GPU tests run N virtual ranks on one device (comm/symm.py::VirtualCluster) and compare with a float64 batch norm
over the concatenated batch.  The bounds are those of test_gpu_bn_act.py with the global row count N: the
cross-rank merge adds at most W - 1 Chan steps (or W - 1 additions) to chains that C_ACC already covers.

The virtual ranks' sync kernels wait for each other on one GPU, so the tests are written so that they cannot
hang: every rank's work is enqueued on its own stream; between one rank's first sync launch and its peers' there
are only kernel launches (buffers are allocated first, nothing reads a value back or synchronises); every kernel
the ranks launch is loaded before (the context loads the batch-norm kernels, a local warm-up run loads torch's);
and every rank runs the same launch sequence, so no barrier waits for something that never comes.
"""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from byteps_b200.models import resnet18, resnet50
from byteps_b200.ops.bn_act import BatchNormAct2d, SyncBatchNormAct2d, SyncBatchNormContext, convert_sync_batchnorm
from test_gpu_bn_act import ACTS, C_ACC, DTYPES, RESNET50_BN_SHAPES, TINY, U32, UNIT, _dt_id


# ---------------------------------------------------------------------------------------------- CPU
def _plain_model():
    return nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.BatchNorm2d(16), nn.ReLU(),
                         nn.Conv2d(16, 8, 1), nn.BatchNorm2d(8, momentum=None))


MODELS = [("resnet18", resnet18), ("resnet50", resnet50), ("plain", _plain_model)]


def _randomise_stats(model, seed=0):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.copy_(torch.randn(m.num_features, generator=g))
                m.bias.copy_(torch.randn(m.num_features, generator=g))
                m.running_mean.copy_(torch.randn(m.num_features, generator=g))
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
    return model


@pytest.mark.parametrize("name,ctor", MODELS, ids=[m[0] for m in MODELS])
def test_convert_reuses_parameters_and_buffers(name, ctor):
    torch.manual_seed(0)
    model = _randomise_stats(ctor())
    before = dict(model.named_modules())
    params = [(n, p) for n, p in model.named_parameters()]
    buffers = [(n, b) for n, b in model.named_buffers()]
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    out = convert_sync_batchnorm(model, None)
    assert out is model
    for n, m in out.named_modules():
        if isinstance(before[n], nn.BatchNorm2d):
            assert type(m) is SyncBatchNormAct2d, n
            assert m.act == getattr(before[n], "act", None), n
            assert (m.eps, m.momentum, m.num_features) == (before[n].eps, before[n].momentum, before[n].num_features)
        else:
            assert not isinstance(m, nn.BatchNorm2d) or m is before[n], n
    assert [(n, id(p)) for n, p in out.named_parameters()] == [(n, id(p)) for n, p in params]
    assert [(n, id(b)) for n, b in out.named_buffers()] == [(n, id(b)) for n, b in buffers]
    new_sd = out.state_dict()
    assert list(new_sd) == list(sd)
    for k, v in new_sd.items():
        assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize("name,ctor", MODELS, ids=[m[0] for m in MODELS])
def test_converted_eval_forward_is_unchanged(name, ctor):
    torch.manual_seed(0)
    model = _randomise_stats(ctor())
    twin = copy.deepcopy(model)
    convert_sync_batchnorm(model, None)
    x = torch.randn(2, 3, 64, 64)
    with torch.no_grad():
        assert torch.equal(model.eval()(x), twin.eval()(x))


class _StubContext:
    world, rank, cmax = 2, 0, 2048


def test_unfusable_training_input_raises_at_world_2():
    bn = SyncBatchNormAct2d(16, act="relu", sync=_StubContext())
    with pytest.raises(ValueError, match="not a CUDA tensor"):
        bn.train()(torch.randn(2, 16, 4, 4))
    # eval mode is the stock path, without communication
    assert bn.eval()(torch.randn(2, 16, 4, 4)).shape == (2, 16, 4, 4)


def test_public_convert_rejects_other_backends(monkeypatch):
    import byteps_b200.torch as bps

    class _Engine:
        backend, size = "gloo", 2

    monkeypatch.setattr(bps, "_engine", lambda: _Engine())
    with pytest.raises(ValueError, match="symmetric-memory backend"):
        bps.convert_sync_batchnorm(resnet18())


def test_public_convert_at_world_1(monkeypatch):
    import byteps_b200.torch as bps

    class _Engine:
        backend, size = "local", 1

    monkeypatch.setattr(bps, "_engine", lambda: _Engine())
    model = bps.convert_sync_batchnorm(resnet18())
    bns = [m for m in model.modules() if isinstance(m, nn.BatchNorm2d)]
    assert bns and all(type(m) is SyncBatchNormAct2d and m.sync is None for m in bns)


# ---------------------------------------------------------------------------------------------- GPU: kernels
def _cluster(world, cmax):
    from byteps_b200.comm.symm import VirtualCluster

    vc = VirtualCluster(world, "cuda", max(1 << 20, SyncBatchNormContext.window_bytes(world, cmax)))
    return vc, [SyncBatchNormContext.from_virtual(vc, r, cmax) for r in range(world)]


def _rows(world, hw):
    """Unequal per-rank row counts; the last rank holds a single row."""
    return [hw * (1 + r % 2) for r in range(world - 1)] + [1]


class _RankBufs:
    """Every buffer one rank's forward + backward needs, allocated before any launch."""

    def __init__(self, m, c, dtype, act, residual, g):
        dev = "cuda"
        f32 = dict(dtype=torch.float32, device=dev)
        scale = torch.rand(c, device=dev, generator=g, dtype=torch.float64) * 2 + 0.5
        loc = torch.randn(c, device=dev, generator=g, dtype=torch.float64)
        self.m, self.c, self.dtype, self.relu = m, c, dtype, act == "relu"
        self.x = (torch.randn(m, c, device=dev, generator=g, dtype=torch.float64) * scale + loc).to(dtype)
        self.r = torch.randn(m, c, device=dev, generator=g, dtype=torch.float64).to(dtype) if residual else None
        self.dy = torch.randn(m, c, device=dev, generator=g, dtype=torch.float64).to(dtype)
        self.local = torch.empty(2, c, **f32)
        self.mean, self.invstd, self.total = torch.empty(c, **f32), torch.empty(c, **f32), torch.empty(1, **f32)
        self.y = torch.empty_like(self.x)
        self.mask = torch.empty(m, c // 8, dtype=torch.uint8, device=dev) if self.relu else None
        self.dw, self.db, self.sums = torch.empty(c, **f32), torch.empty(c, **f32), torch.empty(2, c, **f32)
        self.dx = torch.empty_like(self.x)
        self.dres = torch.empty_like(self.x) if residual else None
        import byteps_b200._native as nat

        nws, nctr = nat.cuda().bn_act_workspace(m, c)
        self.ws = torch.empty(nws, **f32)
        self.ctr = torch.zeros(nctr, dtype=torch.int32, device=dev)


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _launch_fwd(cu, ctx, b, w, bias, rm, rv, s, eps=1e-5, mom=0.1):
    code = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[b.dtype]
    cu.bn_act_fwd_stats_local(b.x.data_ptr(), code, b.m, b.c, b.local[0].data_ptr(), b.local[1].data_ptr(),
                              b.ws.data_ptr(), b.ctr.data_ptr(), s)
    cu.bn_sync_stats(ctx.view, ctx.channel, 0, ctx.cmax, b.c, b.local[0].data_ptr(), b.local[1].data_ptr(),
                     float(b.m), eps, mom, rm.data_ptr(), rv.data_ptr(), b.mean.data_ptr(), b.invstd.data_ptr(),
                     b.total.data_ptr(), s)
    cu.bn_act_fwd_apply(b.x.data_ptr(), _ptr(b.r), code, b.m, b.c, b.mean.data_ptr(), b.invstd.data_ptr(),
                        w.data_ptr(), bias.data_ptr(), b.relu, b.y.data_ptr(), _ptr(b.mask), s)


def _launch_bwd(cu, ctx, b, w, s):
    code = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[b.dtype]
    cu.bn_act_bwd_reduce(b.dy.data_ptr(), b.x.data_ptr(), _ptr(b.mask), code, b.m, b.c, b.mean.data_ptr(),
                         b.invstd.data_ptr(), b.dw.data_ptr(), b.db.data_ptr(), b.ws.data_ptr(), b.ctr.data_ptr(), s)
    cu.bn_sync_grad(ctx.view, ctx.channel, 0, ctx.cmax, b.c, b.db.data_ptr(), b.dw.data_ptr(), b.sums[0].data_ptr(),
                    b.sums[1].data_ptr(), s)
    cu.bn_act_bwd_apply(b.dy.data_ptr(), b.x.data_ptr(), _ptr(b.mask), code, b.m, b.c, b.mean.data_ptr(),
                        b.invstd.data_ptr(), w.data_ptr(), b.sums[1].data_ptr(), b.sums[0].data_ptr(), b.dx.data_ptr(),
                        _ptr(b.dres), s, b.total.data_ptr())


def _check_against_float64(bufs, w, bias, rms, rvs, rm0, rv0, act, eps=1e-5, mom=0.1):
    dtype = bufs[0].dtype
    ut = UNIT[dtype]
    n_tot = sum(b.m for b in bufs)
    xd = torch.cat([b.x.double() for b in bufs])
    wd, bd = w.double(), bias.double()
    mu = xd.mean(0)
    var = xd.var(0, unbiased=False)
    inv = 1.0 / torch.sqrt(var + eps)
    shift = mu.abs() * inv + 1.0

    # statistics: bit-identical on every rank, within the float64 bounds
    for r, b in enumerate(bufs):
        for name, a, ref in (("mean", b.mean, bufs[0].mean), ("invstd", b.invstd, bufs[0].invstd),
                             ("running_mean", rms[r], rms[0]), ("running_var", rvs[r], rvs[0])):
            assert torch.equal(a, ref), "%s differs between rank %d and rank 0" % (name, r)
        assert b.total.item() == n_tot
    assert torch.all((bufs[0].mean.double() - mu).abs() <= C_ACC * U32 * (mu.abs() + var.sqrt()))
    assert torch.all((bufs[0].invstd.double() - inv).abs() <= C_ACC * U32 * inv * shift)
    rm_ref = (1 - mom) * rm0.double() + mom * mu
    rv_ref = (1 - mom) * rv0.double() + mom * var * n_tot / (n_tot - 1)
    assert torch.all((rms[0].double() - rm_ref).abs() <= C_ACC * U32 * (rm0.double().abs() + mu.abs() + var.sqrt()))
    assert torch.all((rvs[0].double() - rv_ref).abs() <= C_ACC * U32 * (rv0.double().abs() + var * shift))

    gs, xhats = [], []
    for b in bufs:
        xhat = (b.x.double() - mu) * inv
        z = xhat * wd + bd + (b.r.double() if b.r is not None else 0.0)
        y_ref = torch.relu(z) if act == "relu" else z
        mag = (xhat.abs() * shift + shift) * wd.abs() + bd.abs() + (b.r.double().abs() if b.r is not None else 0.0)
        tol_y = C_ACC * U32 * mag + ut * (y_ref.abs() + C_ACC * U32 * mag) + TINY[dtype]
        err = (b.y.double() - y_ref).abs()
        assert (err <= tol_y).all(), "y: worst excess %g" % (err - tol_y).max().item()
        g = b.dy.double() * ((b.y > 0).double() if act == "relu" else 1.0)
        if b.r is not None:
            assert torch.equal(b.dres, g.to(dtype)), "d(residual) must be dy * mask exactly"
        # this rank's dweight / dbias are its local sums
        db_ref, dw_ref = g.sum(0), (g * xhat).sum(0)
        sg, sgx = g.abs().sum(0), (g * xhat).abs().sum(0)
        assert torch.all((b.db.double() - db_ref).abs() <= C_ACC * U32 * sg), "local dbias"
        assert torch.all((b.dw.double() - dw_ref).abs() <= C_ACC * U32 * (sgx + shift * sg + dw_ref.abs())), "dweight"
        gs.append(g)
        xhats.append(xhat)

    g_all, xhat_all = torch.cat(gs), torch.cat(xhats)
    DB, DW = g_all.sum(0), (g_all * xhat_all).sum(0)
    SG, SGX = g_all.abs().sum(0), (g_all * xhat_all).abs().sum(0)
    a = wd * inv
    for b, g, xhat in zip(bufs, gs, xhats):
        assert torch.equal(b.sums, bufs[0].sums), "global sums differ between ranks"
        dx_ref = a * (g - DB / n_tot - xhat * DW / n_tot)
        mag_dx = a.abs() * (g.abs() + (xhat.abs() * shift + shift) * ((SGX + shift * SG + DW.abs()) / n_tot)
                            + SG / n_tot)
        tol_dx = C_ACC * U32 * mag_dx * (1 + ut) * 2 + ut * dx_ref.abs() + TINY[dtype]
        err = (b.dx.double() - dx_ref).abs()
        assert (err <= tol_dx).all(), "dx: worst excess %g" % (err - tol_dx).max().item()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sync_kernels_resnet50_shapes(world, dtype):
    import byteps_b200._native as nat

    cu = nat.cuda()
    vc, ctxs = _cluster(world, 2048)
    for i, (c, h, w_) in enumerate(RESNET50_BN_SHAPES):
        _, act, residual = ACTS[i % len(ACTS)]
        g = torch.Generator(device="cuda").manual_seed(1000 * world + i)
        bufs = [_RankBufs(m, c, dtype, act, residual, g) for m in _rows(world, h * w_)]
        w = torch.randn(c, device="cuda", generator=g)
        bias = torch.randn(c, device="cuda", generator=g) * 0.5
        rm0, rv0 = torch.randn(c, device="cuda", generator=g), torch.rand(c, device="cuda", generator=g) + 0.5
        rms, rvs = [rm0.clone() for _ in range(world)], [rv0.clone() for _ in range(world)]
        vc.run(lambda r, view, arena, s: _launch_fwd(cu, ctxs[r], bufs[r], w, bias, rms[r], rvs[r], s))
        vc.run(lambda r, view, arena, s: _launch_bwd(cu, ctxs[r], bufs[r], w, s))
        torch.cuda.synchronize()
        _check_against_float64(bufs, w, bias, rms, rvs, rm0, rv0, act)


@pytest.mark.gpu
def test_sync_kernels_graph_replay_equals_eager():
    """One CUDA graph per virtual rank, each replayed twice on its rank's stream: bit-identical to eager.  The
    window parity comes from device memory, so replays keep alternating slots correctly."""
    import byteps_b200._native as nat

    cu = nat.cuda()
    world, c = 3, 256
    vc, ctxs = _cluster(world, c)
    g = torch.Generator(device="cuda").manual_seed(7)
    bufs = [_RankBufs(m, c, torch.bfloat16, "relu", True, g) for m in (196, 392, 1)]
    w = torch.randn(c, device="cuda", generator=g)
    bias = torch.randn(c, device="cuda", generator=g)
    rm0, rv0 = torch.randn(c, device="cuda", generator=g), torch.rand(c, device="cuda", generator=g) + 0.5
    rms, rvs = [torch.empty_like(rm0) for _ in range(world)], [torch.empty_like(rv0) for _ in range(world)]

    def step(r):
        with torch.cuda.stream(vc.streams[r]):
            s = vc.streams[r].cuda_stream
            rms[r].copy_(rm0)
            rvs[r].copy_(rv0)
            _launch_fwd(cu, ctxs[r], bufs[r], w, bias, rms[r], rvs[r], s)
            _launch_bwd(cu, ctxs[r], bufs[r], w, s)

    def outputs():
        return [[t.clone() for t in (b.mean, b.invstd, b.y, b.mask, b.dx, b.dres, b.dw, b.db, rms[r], rvs[r])]
                for r, b in enumerate(bufs)]

    for r in range(world):         # load the copy kernels before the first multi-rank launch
        rms[r].copy_(rm0)
        rvs[r].copy_(rv0)
    torch.cuda.synchronize()
    vc.run(lambda r, view, arena, s: step(r))
    torch.cuda.synchronize()
    eager = outputs()
    for b in bufs:
        for t in (b.y, b.dx, b.dres):
            t.zero_()

    graphs = []
    for r in range(world):   # capturing runs nothing, so ranks can be captured one after the other
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=vc.streams[r]):
            step(r)
        graphs.append(gr)
    torch.cuda.synchronize()
    for _ in range(2):
        cur = torch.cuda.current_stream()
        for s in vc.streams:
            s.wait_stream(cur)
        for r in range(world):
            with torch.cuda.stream(vc.streams[r]):
                graphs[r].replay()
        for s in vc.streams:
            cur.wait_stream(s)
        torch.cuda.synchronize()
        for r, (a, e) in enumerate(zip(outputs(), eager)):
            for i, (x, y) in enumerate(zip(a, e)):
                assert torch.equal(x, y), "rank %d output %d" % (r, i)


# ---------------------------------------------------------------------------------------------- GPU: module
class _Chain(nn.Module):
    """Three synchronised batch norms of different C (so slots and parities are reused), with ReLU and a
    residual, joined by channel concatenation and slicing (no library kernels that keep per-stream handles)."""

    def __init__(self, sync):
        super().__init__()
        self.a = SyncBatchNormAct2d(32, act="relu", sync=sync)
        self.b = SyncBatchNormAct2d(64, act="relu", sync=sync)
        self.c = SyncBatchNormAct2d(16, sync=sync)

    def forward(self, x, res):
        t = self.a(x)
        t = torch.cat([t, t * 0.5 - 1.0], 1).contiguous(memory_format=torch.channels_last)
        t = self.b(t, res)
        return self.c(t[:, 8:24].contiguous(memory_format=torch.channels_last))


def _reference_chain(chain, x, res):
    """The same chain in float64 autograd over the concatenated batch."""
    def bn(m, t):
        return F.batch_norm(t, None, None, m.weight.double(), m.bias.double(), True, 0.0, m.eps)

    t = F.relu(bn(chain.a, x))
    t = torch.cat([t, t * 0.5 - 1.0], 1)
    t = F.relu(bn(chain.b, t) + res)
    return bn(chain.c, t[:, 8:24])


@pytest.mark.gpu
def test_sync_module_chain_matches_float64_concatenated_batch():
    world = 3
    vc, ctxs = _cluster(world, 64)
    torch.manual_seed(0)
    base = _Chain(None).cuda()
    with torch.no_grad():
        for name, p in base.named_parameters():
            p.copy_(torch.randn_like(p) * 0.5 + (1.0 if name.endswith("weight") else 0.0))
    chains = [copy.deepcopy(base) for _ in range(world)]
    ns = [2, 1, 3]
    nhwc = lambda t: t.contiguous(memory_format=torch.channels_last)  # noqa: E731
    xs = [nhwc(torch.randn(n, 32, 5, 4, device="cuda") * 2 + 1) for n in ns]
    rs = [nhwc(torch.randn(n, 64, 5, 4, device="cuda")) for n in ns]
    dys = [nhwc(torch.randn(n, 16, 5, 4, device="cuda")) for n in ns]

    # warm-up on every rank's stream with local statistics: loads every torch kernel the synchronised run uses
    state = copy.deepcopy(base.state_dict())
    for r in range(world):
        with torch.cuda.stream(vc.streams[r]):
            xg = xs[r].clone().requires_grad_(True)
            chains[r](xg, rs[r]).backward(dys[r])
    torch.cuda.synchronize()
    for r, ch in enumerate(chains):
        ch.load_state_dict(state)
        ch.zero_grad(set_to_none=True)
        for m in ch.modules():
            if isinstance(m, SyncBatchNormAct2d):
                m.sync = ctxs[r]

    xg = [x.clone().requires_grad_(True) for x in xs]
    ys = [None] * world
    cur = torch.cuda.current_stream()
    for s in vc.streams:
        s.wait_stream(cur)
    for r in range(world):
        with torch.cuda.stream(vc.streams[r]):
            ys[r] = chains[r](xg[r], rs[r])
    for r in range(world):
        with torch.cuda.stream(vc.streams[r]):
            ys[r].backward(dys[r])
    for s in vc.streams:
        cur.wait_stream(s)
    torch.cuda.synchronize()

    ref = copy.deepcopy(base).double()
    xd = torch.cat(xs).double().requires_grad_(True)
    yd = _reference_chain(ref, xd, torch.cat(rs).double())
    yd.backward(torch.cat(dys).double())
    close = dict(rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(torch.cat(ys).double(), yd, **close)
    torch.testing.assert_close(torch.cat([x.grad for x in xg]).double(), xd.grad, **close)
    for name, p in ref.named_parameters():
        summed = sum(dict(ch.named_parameters())[name].grad.double() for ch in chains)
        torch.testing.assert_close(summed, p.grad, **close, msg=lambda m: "%s: %s" % (name, m))
    for name, buf in chains[0].named_buffers():
        for ch in chains[1:]:
            assert torch.equal(dict(ch.named_buffers())[name], buf), name
    # running statistics follow the global batch (unbiased variance)
    with torch.no_grad():
        x_all = torch.cat(xs).double()
        mu, var = x_all.mean((0, 2, 3)), x_all.var((0, 2, 3), unbiased=True)
        torch.testing.assert_close(chains[0].a.running_mean.double(), 0.9 * state["a.running_mean"].double() + 0.1 * mu,
                                   rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(chains[0].a.running_var.double(), 0.9 * state["a.running_var"].double() + 0.1 * var,
                                   rtol=1e-5, atol=1e-5)


@pytest.mark.gpu
def test_sync_module_rejects_unfusable_cuda_inputs_and_foreign_streams():
    vc, ctxs = _cluster(2, 64)
    bn = SyncBatchNormAct2d(24, sync=ctxs[0]).cuda().train()
    with pytest.raises(ValueError, match="channels_last"):
        bn(torch.randn(2, 24, 4, 4, device="cuda"))
    bn12 = SyncBatchNormAct2d(12, sync=ctxs[0]).cuda().train()
    with pytest.raises(ValueError, match="multiple of 8"):
        bn12(torch.randn(2, 12, 4, 4, device="cuda").contiguous(memory_format=torch.channels_last))
    x = torch.randn(2, 24, 4, 4, device="cuda").contiguous(memory_format=torch.channels_last)
    with pytest.raises(RuntimeError, match="one stream"):
        bn(x)   # the current stream is not rank 0's stream; raises before any launch


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_sync_module_world1_is_bn_act(dtype):
    from byteps_b200.comm.symm import VirtualCluster

    torch.manual_seed(0)
    vc = VirtualCluster(1, "cuda", 1 << 20)
    ref = BatchNormAct2d(64, act="relu").cuda()
    with torch.no_grad():
        ref.weight.copy_(torch.randn(64))
        ref.bias.copy_(torch.randn(64))
    g = torch.Generator("cuda").manual_seed(1)
    x0 = torch.randn(4, 64, 7, 7, device="cuda", generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
    r = torch.randn(4, 64, 7, 7, device="cuda", generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
    outs = []
    for sync in (None, SyncBatchNormContext.from_virtual(vc, 0, 64)):
        bn = copy.deepcopy(ref)
        if sync is not None:
            bn = convert_sync_batchnorm(bn, sync)
            assert type(bn) is SyncBatchNormAct2d
        x = x0.clone().requires_grad_(True)
        y = bn(x, r)
        y.backward(torch.ones_like(y))
        outs.append([y, x.grad, bn.weight.grad, bn.bias.grad, bn.running_mean, bn.running_var])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------- two GPUs
def _train_resnet18(rank, world):
    import byteps_b200.torch as bps
    from byteps_b200.ops.bn_act import SyncBatchNormAct2d as Sync

    torch.cuda.set_device(rank)
    bps.init()
    torch.manual_seed(0)
    base = resnet18(num_classes=10).cuda().to(memory_format=torch.channels_last)
    ref = copy.deepcopy(base)
    model = bps.convert_sync_batchnorm(base)
    assert all(type(m) is Sync for m in model.modules() if isinstance(m, nn.BatchNorm2d))
    opt = bps.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9),
                                   named_parameters=model.named_parameters(), fused_update=True)
    ref_opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9)
    g = torch.Generator(device="cuda").manual_seed(1)
    per = 4
    for _ in range(3):
        x = torch.randn(world * per, 3, 32, 32, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (world * per,), device="cuda", generator=g)
        opt.zero_grad()
        loss = F.cross_entropy(model(x[rank * per:(rank + 1) * per]), y[rank * per:(rank + 1) * per])
        loss.backward()
        opt.step()
        ref_opt.zero_grad()
        ref_loss = F.cross_entropy(ref(x), y)
        ref_loss.backward()
        ref_opt.step()
    torch.cuda.synchronize()
    losses = bps.push_pull(loss.detach().reshape(1), average=True, name="syncbn.loss")
    torch.testing.assert_close(losses.item(), ref_loss.item(), rtol=2e-3, atol=2e-3)
    for (n, p), (_, q) in zip(model.named_parameters(), ref.named_parameters()):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=2e-3, atol=2e-3, msg=lambda m: "%s: %s" % (n, m))
    for n, b in model.named_buffers():
        if b.is_floating_point():
            gathered = bps.push_pull(b.detach().clone(), average=False, name="syncbn." + n)
            assert torch.equal(gathered, b * world), "running statistic %s differs between ranks" % n
    bps.shutdown()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_process_resnet18_matches_concatenated_batch():
    from _mp import run_workers

    run_workers(_train_resnet18, world=2, timeout=600)
