"""Real multi-process / multi-GPU runs of the symmetric-memory path (>= 2 GPUs)."""
import pytest
import torch

from _mp import run_workers

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _pushpull(rank, world):
    import byteps_b200.torch as bps
    from byteps_b200.common import engine

    torch.cuda.set_device(rank)
    bps.init()
    assert engine().backend == "symm"
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        for n in (7, 4096, 1_000_003, 8_000_000):
            x = (torch.arange(n, device="cuda") % 13).to(dt) * (rank + 1)
            x0 = x.clone()
            y = bps.push_pull(x, average=False, name="t%s_%d" % (str(dt)[6:], n))
            tot = sum(r + 1 for r in range(world))
            ref = ((torch.arange(n, device="cuda") % 13).float() * tot).to(dt)
            assert torch.equal(x, x0)
            assert torch.allclose(y.float(), ref.float(), rtol=1e-2 if dt != torch.float32 else 1e-6), (dt, n)
    # unnamed tensors (auto-named per call) go through the same native adapter
    launches0 = engine()._native.launches
    for dt in (torch.float32, torch.bfloat16):
        for n in (4096, 8_000_000):
            x = (torch.arange(n, device="cuda") % 13).to(dt) * (rank + 1)
            x0 = x.clone()
            y = bps.synchronize(bps.push_pull_async(x, average=False))
            tot = sum(r + 1 for r in range(world))
            ref = ((torch.arange(n, device="cuda") % 13).float() * tot).to(dt)
            assert torch.equal(x, x0)
            assert torch.allclose(y.float(), ref.float(), rtol=1e-2 if dt != torch.float32 else 1e-6), (dt, n)
    assert engine()._native.launches > launches0 and engine().outstanding() == 0
    with pytest.raises(ValueError):           # the kernels write input-dtype elements through the output pointer
        engine().push_pull_async(x, torch.empty(n, device="cuda", dtype=torch.float16), False, "mismatch")
    # many small tensors issued back to back, synchronised at the end (priority order inside the flush)
    ts = [torch.full((1000 + i,), float(rank), device="cuda") for i in range(20)]
    hs = [bps.push_pull_async_inplace(t, average=True, name="many%d" % i, priority=-i) for i, t in enumerate(ts)]
    for h, t in zip(hs, ts):
        out = bps.synchronize(h)
        assert torch.allclose(out, torch.full_like(out, sum(range(world)) / world))
    # integer / CPU tensors fall back to the torch.distributed transport
    z = torch.ones(10, dtype=torch.int64, device="cuda") * (rank + 1)
    assert bps.push_pull(z, average=False, name="ints").tolist() == [sum(r + 1 for r in range(world))] * 10
    c = torch.ones(10) * (rank + 1)
    assert bps.push_pull(c, average=True, name="cpu").tolist() == [sum(r + 1 for r in range(world)) / world] * 10
    bps.shutdown()


def test_pushpull_two_gpus():
    run_workers(_pushpull, world=2, timeout=300)


def _optimizer(rank, world, fused, graph):
    import byteps_b200.torch as bps
    from byteps_b200.torch.graph import GraphedStep

    torch.cuda.set_device(rank)
    bps.init()
    torch.manual_seed(100 + rank)
    mk = lambda: torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 16)).cuda()  # noqa: E731
    model = mk()
    opt = bps.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9),
                                   named_parameters=model.named_parameters(), fused_update=fused)
    bps.broadcast_parameters(model.state_dict(), root_rank=0)
    if not fused:
        bps.broadcast_optimizer_state(opt, root_rank=0)
    ref = mk()
    ref.load_state_dict(model.state_dict())
    ropt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9)
    torch.manual_seed(7)
    steps = 5
    xs = torch.randn(steps, world * 8, 64, device="cuda")
    ys = torch.randn(steps, world * 8, 16, device="cuda")
    sx = torch.empty(8, 64, device="cuda")
    sy = torch.empty(8, 16, device="cuda")

    def step():
        opt.zero_grad()
        loss = torch.nn.functional.mse_loss(model(sx), sy)
        loss.backward()
        opt.step()
        return loss

    runner = None
    for i in range(steps):
        sx.copy_(xs[i, rank * 8:(rank + 1) * 8])
        sy.copy_(ys[i, rank * 8:(rank + 1) * 8])
        if graph and i == 2:
            runner = GraphedStep(step, warmup=1, pre_replay=opt.refresh_hparams)   # consumes this batch eagerly
        elif runner is not None:
            runner()
        else:
            step()
        ropt.zero_grad()
        torch.nn.functional.mse_loss(ref(xs[i]), ys[i]).backward()
        ropt.step()
    torch.cuda.synchronize()
    for a, b in zip(model.parameters(), ref.parameters()):
        assert torch.allclose(a, b, atol=1e-4), (a - b).abs().max()
    bps.shutdown()


@pytest.mark.parametrize("fused,graph", [(False, False), (True, False), (True, True)])
def test_distributed_optimizer_two_gpus(fused, graph):
    run_workers(_optimizer, world=2, args=(fused, graph), timeout=300)


def _ddp_and_cross_barrier(rank, world):
    import byteps_b200.torch as bps
    from byteps_b200.torch.cross_barrier import CrossBarrier
    from byteps_b200.torch.half_optimizer import HalfPrecisionDistributedOptimizer
    from byteps_b200.torch.parallel import DistributedDataParallel as DDP

    torch.cuda.set_device(rank)
    bps.init()
    mk = lambda: torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 8)).cuda()  # noqa: E731
    torch.manual_seed(5)
    xs = torch.randn(4, world * 4, 32, device="cuda")
    ys = torch.randn(4, world * 4, 8, device="cuda")
    # ---- DDP + plain optimizer == full-batch training
    torch.manual_seed(100 + rank)
    model = DDP(mk(), device_ids=[rank])           # broadcasts rank 0's weights
    ref = mk()
    ref.load_state_dict(model.module.state_dict())
    opt, ropt = torch.optim.SGD(model.parameters(), lr=0.1), torch.optim.SGD(ref.parameters(), lr=0.1)
    for i in range(3):
        opt.zero_grad(set_to_none=False)
        torch.nn.functional.mse_loss(model(xs[i, rank * 4:(rank + 1) * 4]), ys[i, rank * 4:(rank + 1) * 4]).backward()
        opt.step()
        ropt.zero_grad()
        torch.nn.functional.mse_loss(ref(xs[i]), ys[i]).backward()
        ropt.step()
    for a, b in zip(model.module.parameters(), ref.parameters()):
        assert torch.allclose(a, b, atol=1e-5), (a - b).abs().max()
    # no_sync accumulates locally, the next backward synchronises the sum of both
    opt.zero_grad(set_to_none=False)
    with model.no_sync():
        model(xs[3, rank * 4:(rank + 1) * 4]).sum().backward()
    g_local = [p.grad.clone() for p in model.module.parameters()]
    model(xs[3, rank * 4:(rank + 1) * 4]).sum().backward()
    torch.cuda.synchronize()
    # ---- CrossBarrier (fused per-bucket updates, no global barrier) == torch SGD on the full batch
    m2, r2 = mk(), mk()
    o2 = CrossBarrier(m2, torch.optim.SGD(m2.parameters(), lr=0.05, momentum=0.9), m2.named_parameters(), num_steps=4)
    bps.broadcast_parameters(m2.state_dict(), root_rank=0)
    r2.load_state_dict(m2.state_dict())
    ro2 = torch.optim.SGD(r2.parameters(), lr=0.05, momentum=0.9)
    for i in range(4):
        o2.zero_grad()
        torch.nn.functional.mse_loss(m2(xs[i, rank * 4:(rank + 1) * 4]), ys[i, rank * 4:(rank + 1) * 4]).backward()
        o2.step()
        ro2.zero_grad()
        torch.nn.functional.mse_loss(r2(xs[i]), ys[i]).backward()
        ro2.step()
    torch.cuda.synchronize()
    for a, b in zip(m2.parameters(), r2.parameters()):
        assert torch.allclose(a, b, atol=1e-4), (a - b).abs().max()
    # ---- half-precision optimizer: bf16 weights follow an fp32-master reference
    m3 = mk().to(torch.bfloat16)
    o3 = HalfPrecisionDistributedOptimizer(torch.optim.SGD(m3.parameters(), lr=0.05), m3.named_parameters(),
                                           loss_scale=128.0)
    bps.broadcast_parameters(m3.state_dict(), root_rank=0)
    r3 = mk()
    r3.load_state_dict({k: v.float() for k, v in m3.state_dict().items()})
    ro3 = torch.optim.SGD(r3.parameters(), lr=0.05)
    for i in range(3):
        o3.zero_grad()
        xb, yb = xs[i, rank * 4:(rank + 1) * 4].bfloat16(), ys[i, rank * 4:(rank + 1) * 4].bfloat16()
        o3.backward(torch.nn.functional.mse_loss(m3(xb), yb))
        o3.step()
        ro3.zero_grad()
        torch.nn.functional.mse_loss(r3(xs[i]), ys[i]).backward()
        ro3.step()
    torch.cuda.synchronize()
    for a, b in zip(m3.parameters(), r3.parameters()):
        assert torch.allclose(a.float(), b, atol=3e-2), (a.float() - b).abs().max()
    assert len(o3.master_params()) > 0
    bps.shutdown()


def test_ddp_cross_barrier_half_optimizer_two_gpus():
    run_workers(_ddp_and_cross_barrier, world=2, timeout=300)


def _cross_barrier_overlap(rank, world):
    """The point of CrossBarrier: in the canonical loop `zero_grad(); forward; backward; step()` the forward of
    step i+1 starts while the exchange of step i is still running.  Device stamps (globaltimer) prove it: the
    compute stream reaches the start of forward i+1 (stamp 2) BEFORE the communication stream finishes step i's
    last bucket (stamp 1).  Round 1's zero_grad() waited for every bucket and put the barrier back."""
    import byteps_b200.torch as bps
    from byteps_b200.torch.cross_barrier import CrossBarrier

    torch.cuda.set_device(rank)
    bps.init()
    torch.manual_seed(1)
    # a small head (needed first by the next forward) on top of a big body: ~800 MB of gradients per step, i.e.
    # milliseconds of exchange behind a backward pass of a few hundred microseconds
    mk = lambda: torch.nn.Sequential(torch.nn.Linear(64, 8192), *[torch.nn.Linear(8192, 8192) for _ in range(3)],  # noqa: E731
                                     torch.nn.Linear(8192, 8)).cuda()
    model, ref = mk(), mk()
    opt = CrossBarrier(model, torch.optim.SGD(model.parameters(), lr=0.01), model.named_parameters(), num_steps=5)
    bps.broadcast_parameters(model.state_dict(), root_rank=0)
    ref.load_state_dict(model.state_dict())
    ropt = torch.optim.SGD(ref.parameters(), lr=0.01)
    gs = opt.grad_sync
    cu, view = gs.ctx.cu, gs.ctx.view
    model.register_forward_pre_hook(
        lambda m, inp: cu.ring_stamp(view, 2, torch.cuda.current_stream().cuda_stream))
    torch.manual_seed(2)
    xs = torch.randn(5, world * 4, 64, device="cuda")
    overlapped, seen = 0, []
    for i in range(5):
        opt.zero_grad()
        model(xs[i, rank * 4:(rank + 1) * 4]).square().mean().backward()
        opt.step()
        if 1 <= i < 4:          # steps without a global wait: look at the NEXT forward against THIS exchange
            opt.zero_grad()
            model(xs[i, :4])                      # a forward only: its start is stamped (2)
            torch.cuda.synchronize()
            _, st = cu.ring_trace(view, [])
            overlapped += int(st[2] < st[1])
            seen.append((st[1] - st[2]) / 1e3)     # us the exchange was still running after the next forward began
        ropt.zero_grad()
        ref(xs[i]).square().mean().backward()
        ropt.step()
    torch.cuda.synchronize()
    for a, b in zip(model.parameters(), ref.parameters()):
        assert torch.allclose(a, b, atol=1e-5), (a - b).abs().max()
    assert overlapped >= 2, "forward of step i+1 never started before step i's exchange finished: %s" % (seen,)
    bps.shutdown()


def test_cross_barrier_overlaps_next_forward_with_exchange():
    run_workers(_cross_barrier_overlap, world=2, timeout=300)


def _timeline(rank, world, trace_dir):
    import json
    import os

    os.environ.update({"BYTEPS_TRACE_ON": "1", "BYTEPS_TRACE_START_STEP": "1", "BYTEPS_TRACE_END_STEP": "3",
                       "BYTEPS_TRACE_DIR": trace_dir})
    import byteps_b200.torch as bps

    torch.cuda.set_device(rank)
    bps.init()
    m = torch.nn.Linear(256, 256).cuda()
    opt = bps.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters())
    for _ in range(4):
        opt.zero_grad()
        m(torch.randn(8, 256, device="cuda")).sum().backward()
        opt.step()
    torch.cuda.synchronize()
    bps.shutdown()
    path = os.path.join(trace_dir, str(rank), "comm.json")
    ev = json.load(open(path))["traceEvents"]
    assert len(ev) >= 2 and all(e["ph"] == "X" and e["dur"] >= 1 for e in ev)
    assert any(e["name"].endswith(".PUSHPULL") for e in ev)


def test_device_timed_timeline(tmp_path):
    run_workers(_timeline, world=2, args=(str(tmp_path),), timeout=240)


def _compressed(rank, world):
    """Per-tensor lossy compression through the public API on the NVLink path: GPU compressors,
    payloads exchanged through symmetric memory, two-stage (worker then "server") contract."""
    import byteps_b200.torch as bps
    from byteps_b200.common import engine

    torch.cuda.set_device(rank)
    bps.init()
    assert engine().backend == "symm"
    n = 100_000
    # top-k (k = 64 per rank, disjoint supports): both stages keep exactly the world*64 entries if k2 >= that
    bps.declare("c.topk", compressor_type="topk", compressor_k=64 * world)
    x = torch.zeros(n, device="cuda")
    x[rank * 64:(rank + 1) * 64] = 1.0 + rank
    y = bps.push_pull(x, average=False, name="c.topk")
    ref = torch.zeros(n, device="cuda")
    for r in range(world):
        ref[r * 64:(r + 1) * 64] = 1.0 + r
    assert torch.equal(y, ref), (y - ref).abs().max()
    # onebit with scaling: sign and mean magnitude survive both stages
    bps.declare("c.onebit", compressor_type="onebit", compressor_onebit_scaling="true")
    g = torch.full((n,), 0.5 * (rank + 1), device="cuda")
    out = bps.push_pull(g, average=True, name="c.onebit")
    want = sum(0.5 * (r + 1) for r in range(world)) / world
    assert torch.allclose(out, torch.full_like(out, want), rtol=1e-5), out[:4]
    # replicas stay bit-identical under random-k + error feedback + momentum over several steps
    bps.declare("c.rk", compressor_type="randomk", compressor_k=0.05, ef_type="vanilla",
                momentum_type="nesterov", momentum_mu=0.9, seed=11)
    torch.manual_seed(rank)
    acc = None
    for step in range(4):
        bps.set_learning_rate(0.1 / (step + 1))
        gg = torch.randn(n, device="cuda")
        acc = bps.push_pull(gg, average=True, name="c.rk")
    gathered = [torch.empty_like(acc) for _ in range(world)]
    torch.distributed.all_gather(gathered, acc)
    assert all(torch.equal(gathered[0], t) for t in gathered)
    assert torch.isfinite(acc).all() and acc.abs().sum() > 0
    # small tensors (< BYTEPS_MIN_COMPRESS_BYTES) skip compression: exact sum
    bps.declare("c.small", compressor_type="topk", compressor_k=1)
    s = torch.arange(100, device="cuda", dtype=torch.float32) * (rank + 1)
    assert torch.equal(bps.push_pull(s, average=False, name="c.small"),
                       torch.arange(100, device="cuda", dtype=torch.float32) * sum(r + 1 for r in range(world)))
    # DistributedOptimizer(compression_params=...): per-tensor path, replicas identical after steps
    torch.manual_seed(5)
    model = torch.nn.Linear(512, 256).cuda()
    opt = bps.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9),
                                   named_parameters=model.named_parameters(),
                                   compression_params={"compressor": "topk", "k": 0.01, "ef": "vanilla"})
    bps.broadcast_parameters(model.state_dict(), root_rank=0)
    torch.manual_seed(50 + rank)
    for _ in range(3):
        opt.zero_grad()
        model(torch.randn(8, 512, device="cuda")).square().mean().backward()
        opt.step()
    w = model.weight.detach().clone()
    ws = [torch.empty_like(w) for _ in range(world)]
    torch.distributed.all_gather(ws, w)
    assert all(torch.equal(ws[0], t) for t in ws)
    bps.shutdown()


def test_compressed_pushpull_two_gpus():
    run_workers(_compressed, world=2, timeout=300)
