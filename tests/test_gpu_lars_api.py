"""DistributedOptimizer(Lars(...), fused_update=True) on one H100 (and two, when there are two): against a float64
Lars within the rounding bounds of _lars.advance, with gradient accumulation and dynamic loss scaling, a CUDA-graph
replay against eager, checkpoints through the plain Lars, a graphed ResNet-18 against the plain Lars on fp32 masters,
and the launch count.  The gradients come from loss = sum_i (p_i * G_i).sum(), so each step hands the optimizer
exactly G whatever the weights are.  Each single-GPU case is its own process so init()/shutdown() state never leaks
between tests."""
import os
import subprocess
import sys
import textwrap

import pytest
import torch

from _mp import run_workers

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))


def _run(body, timeout=300):
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n" % (ROOT, TESTS)
            + "import io, torch\nimport byteps_b200.torch as bps\nfrom _lars import *\n" + textwrap.dedent(body))
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "DMLC_ROLE", "DMLC_NUM_WORKER", "DMLC_NUM_SERVER",
              "BYTEPS_FUSED_ENGINE"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout


def test_fused_lars_matches_float64_reference():
    """fp32 and bf16 parameters (fp32 masters), five steps with the lr halved before the third; fp32 also on a bf16
    wire, whose gradients are exact in bf16 here."""
    out = _run("""
    bps.init()
    for dt, comp in ((torch.float32, "none"), (torch.bfloat16, "none"), (torch.float32, "bf16")):
        ps = make_params(dt)
        ref = Reference(ps)
        opt = bps.DistributedOptimizer(bps.Lars(groups(ps), **KW), named_parameters=[("p%d" % i, p) for i, p in
                                       enumerate(ps)], compression=getattr(bps.Compression, comp), fused_update=True)
        for t in range(1, 6):
            if t == 3:
                for g in opt.param_groups:
                    g["lr"] *= 0.5
                opt.grad_sync.refresh_hparams()    # eager: the kernels read the step's lr from the device block
                ref.set_lr(opt.param_groups[0]["lr"])
            gs = grads(t, torch.bfloat16 if comp == "bf16" else dt)
            opt.zero_grad()
            backward(ps, [g.to(dt) for g in gs])
            opt.step()
            ref.step(gs)
            torch.cuda.synchronize()
            ref.check(opt, ps, (str(dt), comp, t))
        print("config ok", dt, comp)
    print("OK")
    bps.shutdown()
    """)
    assert out.count("config ok") == 3 and "OK" in out


def test_backward_passes_per_step_and_dynamic_loss_scale():
    """Two backward passes per step sum their gradients before the update.  With dynamic_loss_scale on fp16
    parameters an inf in one step's gradients skips that step on the device: masters, momentum and parameters keep
    their bits, the step is not counted, and the following steps continue the reference that never saw it."""
    out = _run("""
    bps.init()
    ps = make_params(torch.float32)
    ref = Reference(ps)
    opt = fused_lars(ps, backward_passes_per_step=2)
    for t in range(1, 4):
        a, b = grads(t, torch.float32, seed=1), grads(t, torch.float32, seed=2)
        opt.zero_grad()
        backward(ps, a)
        backward(ps, b)
        opt.step()
        ref.step([x + y for x, y in zip(a, b)])
    torch.cuda.synchronize()
    ref.check(opt, ps, "accumulated")

    ps = make_params(torch.float16, seed=3)
    ref = Reference(ps)
    opt = fused_lars(ps, dynamic_loss_scale=dict(init_scale=256.0))
    for t in range(1, 6):
        gs = [g.to(torch.float16) for g in grads(t, torch.float32)]
        if t == 3:
            gs[2][17] = float("inf")
            before = opt.grad_sync.export_state()
            params = [p.detach().clone() for p in ps]
        opt.zero_grad()
        backward(ps, gs, opt)
        opt.step()
        torch.cuda.synchronize()
        if t == 3:
            after = opt.grad_sync.export_state()
            for p, q in zip(ps, params):
                assert torch.equal(p.view(torch.int16), q.view(torch.int16))
                for k in ("master", "state0"):
                    assert torch.equal(after[p][k].view(torch.int32), before[p][k].view(torch.int32)), k
        else:
            ref.step(gs)
            ref.check(opt, ps, ("scaled", t))
    assert opt.skipped_steps == 1 and opt.grad_sync.applied_steps() == [4, 4]
    print("OK")
    bps.shutdown()
    """)
    assert "OK" in out


def test_graphed_step_equals_eager_and_launch_count():
    """bf16 parameters: a CUDA-graph replay of the step leaves the bits eager steps leave, lr schedule included.
    An eager step launches three LARS kernels per bucket, the two stamps and the hyper-parameter write;
    launches_per_step() and the engine's count agree with the profiler."""
    out = _run("""
    from byteps_b200.common import engine
    from byteps_b200.torch.graph import GraphedStep

    def run(graph):
        ps = make_params(torch.bfloat16)
        opt = fused_lars(ps)
        static = [torch.zeros_like(p) for p in ps]

        def step():
            opt.zero_grad()
            backward(ps, static)
            opt.step()

        for s, g in zip(static, grads(1, torch.bfloat16)):
            s.copy_(g)
        if graph:
            runner = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams)   # two eager steps on these
        else:
            step()
            step()
        for t in range(3, 7):
            for s, g in zip(static, grads(t, torch.bfloat16)):
                s.copy_(g)
            if t == 4:
                for grp in opt.param_groups:
                    grp["lr"] *= 0.5
                if not graph:
                    opt.grad_sync.refresh_hparams()   # a replay's pre_replay publishes it
            runner() if graph else step()
        torch.cuda.synchronize()
        return ps, opt

    bps.init()
    pe, oe = run(False)
    pg, og = run(True)
    se, sg = oe.grad_sync.export_state(), og.grad_sync.export_state()
    for a, b in zip(pe, pg):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
        for k in ("master", "state0"):
            assert torch.equal(se[a][k].view(torch.int32), sg[b][k].view(torch.int32)), k

    n0 = engine().launches
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        oe.zero_grad()
        backward(pe, grads(9, torch.bfloat16))
        oe.step()
        torch.cuda.synchronize()
    n1 = engine().launches
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ours = [n for n in names if "lars_" in n or "ring_stamp" in n]
    blobs = [n for n in names if "write_blob" in n]
    nb = len(oe.grad_sync.buckets)
    assert len([n for n in ours if "lars_" in n]) == 3 * nb, ours
    assert oe.grad_sync.launches_per_step() == len(ours), (oe.grad_sync.launches_per_step(), ours)
    assert len(blobs) == 1 and n1 - n0 == len(ours) + 1, (n1 - n0, ours, blobs)
    print("OK")
    bps.shutdown()
    """)
    assert "OK" in out


def test_checkpoint_through_the_plain_lars():
    """Run A takes 6 steps.  Run B takes 3, its state_dict() goes through torch.save into the plain Lars, whose own
    state_dict() goes into a fresh fused optimizer that takes 3 more: the final parameters and state equal A's bit
    for bit.  The fused checkpoint has the plain Lars's key, momentum_buffer."""
    out = _run("""
    def roundtrip(obj):
        buf = io.BytesIO()
        torch.save(obj, buf)
        buf.seek(0)
        return torch.load(buf)

    def steps(ps, opt, ts):
        for t in ts:
            opt.zero_grad()
            backward(ps, grads(t, torch.float32))
            opt.step()

    bps.init()
    pa = make_params(torch.float32)
    oa = fused_lars(pa)
    steps(pa, oa, range(1, 7))
    pb = make_params(torch.float32)
    ob = fused_lars(pb)
    steps(pb, ob, range(1, 4))
    sd = roundtrip(ob.state_dict())
    assert all(sorted(e) == ["momentum_buffer"] for e in sd["state"].values()), sd["state"][0].keys()
    plain_ps = [torch.nn.Parameter(p.detach().clone()) for p in pb]
    plain = bps.Lars(groups(plain_ps), **KW)
    plain.load_state_dict(sd)
    pc = make_params(torch.float32, seed=9)
    with torch.no_grad():
        for p, q in zip(pc, pb):
            p.copy_(q)
    oc = fused_lars(pc)
    oc.load_state_dict(roundtrip(plain.state_dict()))
    steps(pc, oc, range(4, 7))
    torch.cuda.synchronize()
    sa, sc = oa.grad_sync.export_state(), oc.grad_sync.export_state()
    for a, c in zip(pa, pc):
        assert torch.equal(a.view(torch.int32), c.view(torch.int32))
        for k in ("master", "state0"):
            assert torch.equal(sa[a][k].view(torch.int32), sc[c][k].view(torch.int32)), k
    print("OK")
    bps.shutdown()
    """)
    assert "OK" in out


def test_resnet18_graphed_against_plain_lars(tmp_path):
    """A contiguous-format ResNet-18 in fp32, one CUDA graph per step, with fused LARS (batch-norm parameters and
    biases in an adapt=False, weight_decay=0 group); and the same run eager with the plain Lars.  The two optimizers
    round differently and the network turns last-bit differences of the weights into different gradients (the
    adapt=False group takes SGD-sized steps of lr), so the losses agree within 1% and each tensor's difference between
    the runs stays below a tenth of how far training moved it."""
    code = """
    import torch.nn.functional as F
    from byteps_b200.models import get_model
    from byteps_b200.torch.graph import GraphedStep
    FUSED = %r
    bps.init()
    torch.manual_seed(0)
    model = get_model("resnet18").cuda().train()
    init = {n: p.detach().float().cpu() for n, p in model.named_parameters()}

    def lars_groups(ps):
        return [dict(params=[p for p in ps if p.dim() > 1], weight_decay=5e-5),
                dict(params=[p for p in ps if p.dim() <= 1], weight_decay=0.0, adapt=False)]

    opt = bps.Lars(lars_groups(list(model.parameters())), lr=0.05, momentum=0.9)
    if FUSED:
        opt = bps.DistributedOptimizer(opt, named_parameters=model.named_parameters(), fused_update=True)
    g = torch.Generator().manual_seed(1)
    x = torch.rand(16, 3, 64, 64, generator=g).cuda()
    y = torch.randint(0, 1000, (16,), generator=g).cuda()

    def step():
        opt.zero_grad()
        loss = F.cross_entropy(model(x), y)
        loss.backward()
        opt.step()
        return loss

    stepper = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams) if FUSED else step
    if not FUSED:
        for _ in range(2):   # the graph's eager warm-up steps
            step()
    losses = [stepper().detach().float().item() for _ in range(4)]
    torch.save({"losses": losses, "init": init,
                "params": {n: p.detach().float().cpu() for n, p in model.named_parameters()}}, %r)
    print("OK")
    bps.shutdown()
    """
    runs = {}
    for fused in (True, False):
        path = str(tmp_path / ("fused.pt" if fused else "plain.pt"))
        assert "OK" in _run(code % (fused, path))
        runs[fused] = torch.load(path)
    a, b = runs[True], runs[False]
    for x, y in zip(a["losses"], b["losses"]):
        assert abs(x - y) <= 1e-2 * abs(y), (a["losses"], b["losses"])
    for n, x in a["params"].items():
        y, w0 = b["params"][n], b["init"][n]
        assert torch.equal(a["init"][n], w0), n
        assert (x - y).norm() <= 0.1 * (y - w0).norm(), (n, (x - y).norm().item(), (y - w0).norm().item())


def _two_ranks(rank, world):
    import byteps_b200.torch as bps
    from _lars import Reference, backward, fused_lars, grads, make_params

    torch.cuda.set_device(rank)
    bps.init()
    for dt in (torch.float32, torch.bfloat16):
        ps = make_params(dt)
        ref = Reference(ps)
        opt = fused_lars(ps)
        for t in range(1, 5):
            mine = grads(t, dt, seed=rank + 1)
            opt.zero_grad()
            backward(ps, mine)
            opt.step()
            every = [grads(t, dt, seed=r + 1) for r in range(world)]
            ref.step([sum(g[i].double() for g in every) / world for i in range(len(ps))])
            torch.cuda.synchronize()
            ref.check(opt, ps, (rank, str(dt), t))
    bps.shutdown()


@pytest.mark.multigpu
def test_two_processes_against_float64_reference():
    """Two ranks, each with its own gradients: the fused LARS follows the float64 Lars on their average (the partial
    norms of every parameter cross the ranks)."""
    run_workers(_two_ranks, world=2, timeout=300)
