"""Descriptor-ring exchange kernel (csrc/kernels/pushpull_ring.cu) on one GPU with virtual ranks:
numerics against fp32 PyTorch references, bit-identical replicas, producer marks, CUDA-graph
replays, and the scheduling contract of the reference's BytePSScheduledQueue
(/root/reference/byteps/common/scheduled_queue.cc:82-163): priority desc, key asc, byte credits.
Fused-optimizer descriptors are checked against torch.optim in float64 (tests/_fused_opt.py).
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


def _layout(sizes, es):
    offs, off = [], 256
    for n in sizes:
        offs.append(off)
        off = (off + n * es + 255) // 256 * 256
    return offs, off


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("self_mark", [True, False])
def test_ring_allreduce_virtual(world, dt, self_mark):
    """Several buckets of odd sizes in one launch; replicas bit-identical; two launches back to
    back reuse the same slots (generation counters)."""
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops.ring import RingEntry, RingTable

    cu = _cu()
    dtype = DT[dt]
    es = torch.empty((), dtype=dtype).element_size()
    sizes = [8 * 1031, 8, 8 * 40007, 8 * 513, 8 * 3]
    offs, end = _layout(sizes, es)
    vc = VirtualCluster(world, "cuda:0", max(end, 1 << 20))
    entries = [RingEntry(grad_off=o, numel=n, wire=_code(dtype), slot=3 + 2 * i, scale=1.0 / world)
               for i, (o, n) in enumerate(zip(offs, sizes))]
    tables = [RingTable(entries, "cuda:0") for _ in range(world)]
    for it in range(2):
        torch.manual_seed(it)
        ins = [[torch.randn(n, device="cuda").to(dtype) for n in sizes] for _ in range(world)]
        for r in range(world):
            for o, n, x in zip(offs, sizes, ins[r]):
                vc.arenas[r][o:o + n * es].view(dtype).copy_(x)
        torch.cuda.synchronize()

        def run(r, view, arena, s):
            if not self_mark:
                # producers mark in a different order on different ranks, some after the launch
                order = list(range(len(sizes)))
                order = order[r % len(order):] + order[:r % len(order)]
                cu.ring_mark(view, [entries[i].slot for i in order[:2]], s)
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.ExternalStream(s))     # BEFORE the launch: the marks must not wait for it
                tables[r].launch(view, 2, s, self_mark=False)
                cu.ring_mark(view, [entries[i].slot for i in order[2:]], side.cuda_stream)
                run.keep.append(side)
            else:
                tables[r].launch(view, 2, s)
        run.keep = []
        vc.run(run)
        torch.cuda.synchronize()
        for i, (o, n) in enumerate(zip(offs, sizes)):
            ref = torch.stack([ins[r][i].float() for r in range(world)]).sum(0) / world
            outs = [vc.arenas[r][o:o + n * es].view(dtype) for r in range(world)]
            for x in outs[1:]:
                assert torch.equal(x, outs[0]), "replicas must be bit-identical"
            tol = 1e-6 if dtype == torch.float32 else (1e-2 if dtype == torch.bfloat16 else 2e-3)
            assert torch.allclose(outs[0].float(), ref, atol=tol * max(1.0, ref.abs().max().item()), rtol=tol), (it, i)


_RING_FUSED_CASES = fused_cases(ENGINE_DTYPES["ring"])


@pytest.mark.parametrize("world,dtypes,opt", _RING_FUSED_CASES,
                         ids=["%s-%s-%d" % (dt_id(d), o, w) for w, d, o in _RING_FUSED_CASES])
def test_ring_fused_optimizer_virtual(world, dtypes, opt):
    """RING_SGD / RING_ADAM descriptors: three buckets in one table, against torch.optim in float64."""
    check_fused_optimizer(world, "ring", dtypes[0], dtypes[1], opt)


def _sched_order(credit_bytes, sched=True, world=4):
    """Bucket A (big, low priority) is ready before the launch; B, C (low priority) and H (high
    priority) become ready, in that order, while A is being exchanged.  Returns the order in which
    the ring processed them (from the device-side trace) and the results."""
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops.ring import RingEntry, RingTable

    cu = _cu()
    dtype = torch.float32
    big, small = 8 * 8_000_000, 8 * 2048          # 256 MB (hundreds of microseconds) and 64 KB
    sizes = [big, small, small, small]
    prios = [0, 0, 0, 10]
    names = "ABCH"
    offs, end = _layout(sizes, 4)
    vc = VirtualCluster(world, "cuda:0", end)
    entries = [RingEntry(grad_off=o, numel=n, wire=_code(dtype), slot=i, priority=p, scale=1.0)
               for i, (o, n, p) in enumerate(zip(offs, sizes, prios))]
    tables = [RingTable(entries, "cuda:0") for _ in range(world)]
    for r in range(world):
        for o, n in zip(offs, sizes):
            vc.arenas[r][o:o + n * 4].view(dtype).fill_(float(r + 1))
    # every kernel used below must be loaded BEFORE a ring kernel starts spinning: CUDA loads modules
    # lazily and a first-time load can wait for running kernels (a documented lazy-loading deadlock)
    torch.cuda._sleep(10)
    torch.cuda.synchronize()
    sides = [torch.cuda.Stream() for _ in range(world)]

    def run(r, view, arena, s):
        cu.ring_mark(view, [0], s)                                    # A is ready
        sides[r].wait_stream(torch.cuda.ExternalStream(s))
        tables[r].launch(view, 2, s, self_mark=False, sched=sched, credit_bytes=credit_bytes)
        with torch.cuda.stream(sides[r]):
            for slot in (1, 2, 3):                                    # B, C, then H - one mark kernel each,
                torch.cuda._sleep(20000)                              # ~10 us apart
                cu.ring_mark(view, [slot], sides[r].cuda_stream)

    vc.run(run)
    torch.cuda.synchronize()
    trace, _ = cu.ring_trace(vc.views[0], [0, 1, 2, 3])
    order = "".join(names[i] for i in sorted(range(4), key=lambda i: trace[i][0]))
    tot = float(sum(range(1, world + 1)))
    for r in range(world):
        for o, n in zip(offs, sizes):
            assert torch.all(vc.arenas[r][o:o + n * 4].view(dtype) == tot)
    return order, trace


def test_ring_priority_overtakes_queued_low_priority():
    """scheduled_queue.cc:82-102: with a credit window of one partition the late high-priority
    bucket H goes out before the low-priority B and C that were queued ahead of it."""
    order, trace = _sched_order(credit_bytes=1)
    assert order == "AHBC", order
    # device timestamps agree: H started before B and C
    assert trace[3][1] <= trace[1][1] and trace[3][1] <= trace[2][1]


def test_ring_unlimited_credit_and_static_order_are_fifo():
    """BYTEPS_SCHEDULING_CREDIT has a measurable effect: with an unlimited window the root hands
    out B and C as they arrive (before H exists); without scheduling the table order is used."""
    order, _ = _sched_order(credit_bytes=0)
    assert order[0] == "A" and order.index("B") < order.index("H"), order
    order, _ = _sched_order(credit_bytes=0, sched=False)
    assert order == "ABCH", order


def test_ring_under_cuda_graph_replay():
    """Marks + ring launch captured once and replayed: generations live in device memory."""
    from byteps_b200.comm.symm import VirtualCluster
    from byteps_b200.ops.ring import RingEntry, RingTable

    cu = _cu()
    world, dtype, n = 2, torch.bfloat16, 8 * 4099
    vc = VirtualCluster(world, "cuda:0", 1 << 20)
    entries = [RingEntry(grad_off=256, numel=n, wire=_code(dtype), slot=0, scale=1.0),
               RingEntry(grad_off=256 + 2 * n + 256, numel=n, wire=_code(dtype), slot=1, scale=1.0)]
    tables = [RingTable(entries, "cuda:0") for _ in range(world)]
    src = [torch.zeros(2, n, device="cuda", dtype=dtype) for _ in range(world)]

    def step():
        def run(r, view, arena, s):
            with torch.cuda.stream(torch.cuda.ExternalStream(s)):
                for i, e in enumerate(entries):
                    arena[e.grad_off:e.grad_off + 2 * n].view(dtype).copy_(src[r][i])
            cu.ring_mark(view, [0, 1], s)
            tables[r].launch(view, 2, s, self_mark=False)
        vc.run(run)

    step()                    # eager once (also warms the allocator)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for it in range(3):
        for r in range(world):
            src[r].fill_(float(it + r + 1))
        g.replay()
        torch.cuda.synchronize()
        want = float(sum(it + r + 1 for r in range(world)))
        for r in range(world):
            for e in entries:
                assert torch.all(vc.arenas[r][e.grad_off:e.grad_off + 2 * n].view(dtype).float() == want), (it, r)
