"""Numerics of the sm_90a push-pull kernels against plain PyTorch fp32 references, and of the fused
optimizer kernels against torch.optim in float64.

Multi-peer behaviour is exercised on ONE GPU with `VirtualCluster`: N virtual
ranks, N concurrent kernels on N streams, same flag protocol and peer-pointer
arithmetic as the real multi-process setup.
"""
import pytest
import torch
from _fused_opt import ENGINE_DTYPES, check_fused_optimizer, dt_id, fused_cases

pytestmark = pytest.mark.gpu

DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}


def _cu():
    from byteps_b200 import _native

    return _native.cuda()


def _code(dt):
    from byteps_b200.comm.symm import wire_code

    return wire_code(dt)


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
def test_inplace_pushpull_virtual(world, dt):
    from byteps_b200.comm.symm import VirtualCluster

    cu = _cu()
    dtype = DT[dt]
    n = 8 * 1031 * 3 + 8      # not a multiple of the tile; multiple of 8
    vc = VirtualCluster(world, "cuda:0", 1 << 22)
    torch.manual_seed(0)
    inputs = [torch.randn(n, device="cuda").to(dtype) for _ in range(world)]
    off = 256
    es = inputs[0].element_size()
    for r in range(world):
        vc.arenas[r][off:off + n * es].view(dtype).copy_(inputs[r])
    ref = torch.stack([x.float() for x in inputs]).sum(0) / world
    for blocks in (1, 3):
        for r in range(world):   # restore inputs between runs
            vc.arenas[r][off:off + n * es].view(dtype).copy_(inputs[r])
        vc.run(lambda r, view, arena, s: cu.pushpull_inplace(view, _code(dtype), off, n, 1.0 / world, blocks, 256, 0,
                                                              False, s))
        torch.cuda.synchronize()
        outs = [vc.arenas[r][off:off + n * es].view(dtype).float() for r in range(world)]
        for o in outs[1:]:
            assert torch.equal(o, outs[0]), "ranks must hold bit-identical results"
        tol = 1e-6 if dtype == torch.float32 else (1e-2 if dtype == torch.bfloat16 else 2e-3)
        assert torch.allclose(outs[0], ref, atol=tol * max(1.0, ref.abs().max().item()), rtol=tol)


@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
def test_inplace_pushpull_tma_virtual(world, dt):
    """TMA (cp.async.bulk + mbarrier ring) variant must agree bit for bit with the LSU kernel."""
    from byteps_b200.comm.symm import VirtualCluster

    cu = _cu()
    dtype = DT[dt]
    n = 8 * 4099 * 5          # several tiles per CTA, ragged tail
    es = torch.empty((), dtype=dtype).element_size()
    vc = VirtualCluster(world, "cuda:0", 1 << 22)
    torch.manual_seed(7)
    inputs = [torch.randn(n, device="cuda").to(dtype) for _ in range(world)]
    results = []
    for use_tma in (False, True):
        for r in range(world):
            vc.arenas[r][256:256 + n * es].view(dtype).copy_(inputs[r])
        if use_tma:
            for stages in (1, 3):
                for r in range(world):
                    vc.arenas[r][256:256 + n * es].view(dtype).copy_(inputs[r])
                vc.run(lambda r, view, arena, s: cu.pushpull_inplace_tma(view, _code(dtype), 256, n, 1.0 / world, 3,
                                                                         stages, 0, s))
                torch.cuda.synchronize()
                results.append(vc.arenas[0][256:256 + n * es].view(dtype).clone())
                for r in range(1, world):
                    assert torch.equal(vc.arenas[r][256:256 + n * es].view(dtype), results[-1])
        else:
            vc.run(lambda r, view, arena, s: cu.pushpull_inplace(view, _code(dtype), 256, n, 1.0 / world, 3, 256, 0,
                                                                 False, s))
            torch.cuda.synchronize()
            results.append(vc.arenas[0][256:256 + n * es].view(dtype).clone())
    ref = torch.stack([x.float() for x in inputs]).sum(0) / world
    tol = 1e-6 if dtype == torch.float32 else (1e-2 if dtype == torch.bfloat16 else 2e-3)
    for res in results:
        assert torch.allclose(res.float(), ref, atol=tol * max(1.0, ref.abs().max().item()), rtol=tol)
    if world <= 2:      # same summation order only when the peer rotation coincides
        assert torch.equal(results[0], results[1])


@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_inplace_pushpull_umma_virtual(world, dt):
    """wgmma variant: the peer sum computed by the tensor core as [I|I|...|I] x [X_0;...;X_{P-1}]
    with TMA-fed operands and a register accumulator must match the fp32 reference."""
    from byteps_b200.comm.symm import VirtualCluster

    cu = _cu()
    dtype = DT[dt]
    n = 8192 * 5 * world + 64 * 3 + 8        # several tiles per shard, ragged rows and a ragged tail
    es = 2
    vc = VirtualCluster(world, "cuda:0", 1 << 23)
    torch.manual_seed(11)
    inputs = [torch.randn(n, device="cuda").to(dtype) for _ in range(world)]
    off = 1024
    for r in range(world):
        vc.arenas[r][off:off + n * es].view(dtype).copy_(inputs[r])
    maps = [cu.make_umma_maps(vc.views[r], _code(dtype), off, n) for r in range(world)]
    vc.run(lambda r, view, arena, s: cu.pushpull_inplace_umma(view, maps[r], _code(dtype), off, n, 1.0 / world, 2, 0, s))
    torch.cuda.synchronize()
    ref = torch.stack([x.float() for x in inputs]).sum(0) / world
    outs = [vc.arenas[r][off:off + n * es].view(dtype).float() for r in range(world)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    tol = 1e-2 if dtype == torch.bfloat16 else 2e-3
    assert torch.allclose(outs[0], ref, atol=tol * max(1.0, ref.abs().max().item()), rtol=tol), \
        (outs[0] - ref).abs().max()


@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("one_shot", [False, True])
@pytest.mark.parametrize("user,wire", [("f32", "f32"), ("f32", "bf16"), ("bf16", "bf16"), ("f16", "f16"),
                                       ("f32", "f16")])
def test_packed_pushpull_virtual(world, one_shot, user, wire):
    from byteps_b200.comm.symm import VirtualCluster

    cu = _cu()
    ud, wd = DT[user], DT[wire]
    sizes = [5, 8, 1000, 4097, 33, 70000]     # odd sizes: partial units, padding between segments
    vc = VirtualCluster(world, "cuda:0", 1 << 22)
    torch.manual_seed(1)
    ins = [[torch.randn(s, device="cuda").to(ud) for s in sizes] for _ in range(world)]
    outs = [[torch.full((s,), 7.0, device="cuda", dtype=ud) for s in sizes] for _ in range(world)]
    tables, total = [], 0
    for r in range(world):
        rows, start = [], 0
        for a, b in zip(ins[r], outs[r]):
            rows.append([a.data_ptr(), b.data_ptr(), start, a.numel()])
            start += (a.numel() + 7) // 8 * 8
        total = start
        tables.append(torch.tensor(rows, dtype=torch.int64, device="cuda"))
    vc.run(lambda r, view, arena, s: cu.pushpull_packed(view, _code(ud), _code(wd), tables[r].data_ptr(), len(sizes),
                                                        512, total, 1.0, 2, 256, 0, False, one_shot, True, s))
    torch.cuda.synchronize()
    for i, s in enumerate(sizes):
        # reference: inputs rounded to the wire dtype, summed in fp32, rounded to wire then to user dtype
        ref = torch.stack([ins[r][i].to(wd).float() for r in range(world)]).sum(0).to(wd).to(ud)
        for r in range(world):
            got = outs[r][i]
            assert torch.equal(got, outs[0][i])
            tol = 1e-6 if wd == torch.float32 else (2e-2 if wd == torch.bfloat16 else 4e-3)
            assert torch.allclose(got.float(), ref.float(), atol=tol * max(1.0, ref.float().abs().max().item()),
                                  rtol=tol), (i, s)
        # inputs untouched
    for r in range(world):
        for a in ins[r]:
            assert torch.isfinite(a.float()).all()


_FUSED_CASES = [(w, eng, d, o) for eng in ("lsu", "pack", "tma") for w, d, o in fused_cases(ENGINE_DTYPES[eng])]


@pytest.mark.parametrize("world,engine,dtypes,opt", _FUSED_CASES,
                         ids=["%s-%s-%s-%d" % (e, dt_id(d), o, w) for w, e, d, o in _FUSED_CASES])
def test_fused_optimizer_virtual(world, engine, dtypes, opt):
    """Register (LSU) kernel with gradients in the arena or packed from user tensors through a wire cast, and the
    TMA-streamed kernel: against torch.optim in float64 (see _fused_opt.check_fused_optimizer)."""
    check_fused_optimizer(world, engine, dtypes[0], dtypes[1], opt)


def test_reduce_scatter_then_all_gather_virtual():
    from byteps_b200.comm.symm import VirtualCluster

    cu = _cu()
    world, n = 4, 8 * 999
    vc = VirtualCluster(world, "cuda:0", 1 << 20)
    ins = [torch.randn(n, device="cuda") for _ in range(world)]
    for r in range(world):
        vc.arenas[r][:n * 4].view(torch.float32).copy_(ins[r])
    vc.run(lambda r, v, a, s: cu.reduce_scatter(v, 0, 0, n, 2, 256, 0, False, s))
    torch.cuda.synchronize()
    tot = torch.stack(ins).sum(0)
    for r in range(world):
        b, e = cu.shard_units(n // 8, world, r)
        got = vc.arenas[r][:n * 4].view(torch.float32)[b * 8:e * 8]
        assert torch.allclose(got, tot[b * 8:e * 8], atol=1e-5)
    vc.run(lambda r, v, a, s: cu.all_gather(v, 0, 0, n, 0.5, 2, 256, 0, False, s))
    torch.cuda.synchronize()
    for r in range(world):
        assert torch.allclose(vc.arenas[r][:n * 4].view(torch.float32), tot * 0.5, atol=1e-5)


def test_engine_pushpull_single_gpu_and_optimizer():
    """Public API on one GPU: generic push_pull + fused DistributedOptimizer vs torch SGD."""
    import byteps_b200.torch as bps

    bps.init()
    t = torch.randn(12345, device="cuda")
    assert torch.equal(bps.push_pull(t, name="a"), t)
    torch.manual_seed(3)
    model = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 10)).cuda()
    ref = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 10)).cuda()
    ref.load_state_dict(model.state_dict())
    opt = bps.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4),
                                   named_parameters=model.named_parameters(), fused_update=True)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    for i in range(5):
        x = torch.randn(16, 32, device="cuda")
        y = torch.randint(0, 10, (16,), device="cuda")
        opt.zero_grad()
        torch.nn.functional.cross_entropy(model(x), y).backward()
        opt.step()
        ropt.zero_grad()
        torch.nn.functional.cross_entropy(ref(x), y).backward()
        ropt.step()
    torch.cuda.synchronize()
    for a, b in zip(model.parameters(), ref.parameters()):
        assert torch.allclose(a, b, atol=1e-5), (a - b).abs().max()
    bps.shutdown()


def test_graphed_step_matches_eager():
    import byteps_b200.torch as bps
    from byteps_b200.torch.graph import GraphedStep

    bps.init()
    torch.manual_seed(4)
    mk = lambda: torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.Tanh(), torch.nn.Linear(32, 4)).cuda()  # noqa: E731
    m1, m2 = mk(), mk()
    m2.load_state_dict(m1.state_dict())
    o1 = bps.DistributedOptimizer(torch.optim.Adam(m1.parameters(), lr=1e-2), named_parameters=m1.named_parameters(),
                                  fused_update=True)
    o2 = torch.optim.Adam(m2.parameters(), lr=1e-2)
    x = torch.randn(8, 16, device="cuda")
    y = torch.randn(8, 4, device="cuda")

    def step():
        o1.zero_grad()
        loss = torch.nn.functional.mse_loss(m1(x), y)
        loss.backward()
        o1.step()
        return loss

    g = GraphedStep(step, warmup=2, pre_replay=o1.refresh_hparams)   # 2 eager + 1 capture (not executed)
    for _ in range(3):
        g()
    for _ in range(5):     # 2 warm-up + 3 replays
        o2.zero_grad()
        torch.nn.functional.mse_loss(m2(x), y).backward()
        o2.step()
    torch.cuda.synchronize()
    for a, b in zip(m1.parameters(), m2.parameters()):
        assert torch.allclose(a, b, atol=2e-5), (a - b).abs().max()
    bps.shutdown()
