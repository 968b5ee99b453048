"""DistributedOptimizer(..., fused_update=True, max_grad_norm=...) on one H100 (and two, when there are two): every
fused kind against a float64 "average, clip, step" (_clip.Reference); a max_grad_norm above the norm leaves every
bit as without it; gradient accumulation and an unused parameter; dynamic loss scaling with an injected overflow; a
CUDA-graph replay against eager; the launch count; and a graphed bert_tiny FP8 run against the plain Lamb with
clip_grad_norm_.  Each single-GPU case is its own process so init()/shutdown() state never leaks between tests."""
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
            + "import io, math, torch\nimport byteps_b200.torch as bps\nfrom _clip import *\n" + textwrap.dedent(body))
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "DMLC_ROLE", "DMLC_NUM_WORKER", "DMLC_NUM_SERVER",
              "BYTEPS_FUSED_ENGINE"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout


def test_every_fused_kind_against_float64_reference():
    """SGD with momentum, Adam, AdamW, Lamb and Lars; fp32 and bf16 parameters, and fp32 on a bf16 wire; five steps
    whose gradients change scale, so some clip hard, one not at all."""
    out = _run("""
    bps.init()
    for kind in KINDS:
        for dt, comp in ((torch.float32, "none"), (torch.bfloat16, "none"), (torch.float32, "bf16")):
            ps = make_params(dt)
            ref = Reference(kind, ps)
            opt = fused(kind, ps, compression=getattr(bps.Compression, comp), max_grad_norm=MAX_NORM)
            for t in range(1, 6):
                gs = grads(t, dt)
                opt.zero_grad()
                backward(ps, gs)
                opt.step()
                ref.step(gs)
                torch.cuda.synchronize()
                ref.check(opt, ps, (kind, str(dt), comp, t))
            assert min(ref.norms) < MAX_NORM < max(ref.norms), ref.norms
            print("config ok", kind, dt, comp)
    print("OK")
    bps.shutdown()
    """, timeout=600)
    assert out.count("config ok") == 15 and "OK" in out


def test_norm_below_max_grad_norm_changes_no_bit():
    """With max_grad_norm above every step's norm the coefficient is exactly 1: parameters, optimizer state and the
    checkpoint are bit-identical to the same run without the option, for every fused kind."""
    out = _run("""
    bps.init()
    for kind in KINDS:
        runs = []
        for clip in (None, 1e6):
            ps = make_params(torch.bfloat16)
            opt = fused(kind, ps, max_grad_norm=clip)
            for t in range(1, 5):
                opt.zero_grad()
                backward(ps, grads(t, torch.bfloat16))
                opt.step()
            torch.cuda.synchronize()
            runs.append((ps, opt.grad_sync.export_state(), opt.state_dict()))
        (pa, sa, da), (pb, sb, db) = runs
        for a, b in zip(pa, pb):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), kind
            for k in sa[a]:
                assert torch.equal(sa[a][k].view(torch.int32), sb[b][k].view(torch.int32)), (kind, k)
        assert da["state"].keys() == db["state"].keys()
        for i in da["state"]:
            for k, v in da["state"][i].items():
                assert torch.equal(v, db["state"][i][k]), (kind, i, k)
        print("kind ok", kind)
    print("OK")
    bps.shutdown()
    """)
    assert out.count("kind ok") == 5 and "OK" in out


def test_accumulation_unused_parameter_and_consecutive_steps():
    """backward_passes_per_step=2 sums two passes before the norm; a parameter the loss never reaches contributes a
    zero gradient; the coefficient of one step never carries into the next (grad_scale is rewritten every step)."""
    out = _run("""
    bps.init()
    for kind in ("sgd", "adamw"):
        ps = make_params(torch.float32)
        ref = Reference(kind, ps)
        opt = fused(kind, ps, backward_passes_per_step=2, max_grad_norm=MAX_NORM)
        for t in range(1, 6):
            a, b = grads(t, torch.float32, seed=1), grads(t, torch.float32, seed=2)
            a[4].zero_()
            b[4].zero_()
            opt.zero_grad()
            used = [i for i in range(len(ps)) if i != 4]
            backward([ps[i] for i in used], [a[i] for i in used])
            backward([ps[i] for i in used], [b[i] for i in used])
            opt.step()
            ref.step([x + y for x, y in zip(a, b)])
            torch.cuda.synchronize()
            ref.check(opt, ps, (kind, t))
        print("kind ok", kind)
    print("OK")
    bps.shutdown()
    """)
    assert out.count("kind ok") == 2 and "OK" in out


def test_dynamic_loss_scale_with_an_overflow():
    """fp16 parameters with dynamic_loss_scale: an inf in step 3 skips the step on the device (parameters and state
    keep their bits), grad_norm holds the non-finite norm, and the later steps clip the unscaled gradients as the
    reference that never saw step 3 does."""
    out = _run("""
    bps.init()
    for kind in ("sgd", "adam", "lamb"):
        ps = make_params(torch.float16, seed=3)
        ref = Reference(kind, ps)
        opt = fused(kind, ps, dynamic_loss_scale=dict(init_scale=256.0), max_grad_norm=MAX_NORM)
        for t in range(1, 7):
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
                assert not math.isfinite(opt.grad_norm.item()), opt.grad_norm
                after = opt.grad_sync.export_state()
                for p, q in zip(ps, params):
                    assert torch.equal(p.view(torch.int16), q.view(torch.int16))
                    for k in before[p]:
                        assert torch.equal(after[p][k].view(torch.int32), before[p][k].view(torch.int32)), k
            else:
                ref.step(gs)
                ref.check(opt, ps, (kind, t))
        assert opt.skipped_steps == 1
        print("kind ok", kind)
    print("OK")
    bps.shutdown()
    """)
    assert out.count("kind ok") == 3 and "OK" in out


def test_graphed_step_equals_eager_and_launch_count():
    """bf16 parameters: CUDA-graph replays of a clipped step leave the bits eager steps leave, grad_norm included,
    over several replays whose gradients change scale (a grad_scale that compounded over replays would show).  An
    eager step launches one clip_norm_partial per bucket and one clip_norm_update; launches_per_step() and the
    engine's count agree with the profiler."""
    out = _run("""
    from byteps_b200.common import engine
    from byteps_b200.torch.graph import GraphedStep

    def run(kind, graph):
        ps = make_params(torch.bfloat16)
        opt = fused(kind, ps, max_grad_norm=MAX_NORM)
        static = [torch.zeros_like(p) for p in ps]

        def step():
            opt.zero_grad()
            backward(ps, static)
            opt.step()

        for s, g in zip(static, grads(1, torch.bfloat16)):
            s.copy_(g)
        if graph:
            runner = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams)
        else:
            step()
            step()
        norms = []
        for t in range(2, 8):
            for s, g in zip(static, grads(t, torch.bfloat16)):
                s.copy_(g)
            runner() if graph else step()
            norms.append(opt.grad_norm.clone())
        torch.cuda.synchronize()
        return ps, opt, norms

    bps.init()
    for kind in ("adamw", "lars"):
        pe, oe, ne = run(kind, False)
        pg, og, ng = run(kind, True)
        se, sg = oe.grad_sync.export_state(), og.grad_sync.export_state()
        for a, b in zip(pe, pg):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), kind
            for k in se[a]:
                assert torch.equal(se[a][k].view(torch.int32), sg[b][k].view(torch.int32)), (kind, k)
        assert all(torch.equal(x, y) for x, y in zip(ne, ng)), (kind, ne, ng)
        assert min(x.item() for x in ne) < MAX_NORM < max(x.item() for x in ne), ne
        print("kind ok", kind)

    n0 = engine().launches
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        oe.zero_grad()
        backward(pe, grads(9, torch.bfloat16))
        oe.step()
        torch.cuda.synchronize()
    n1 = engine().launches
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ours = [n for n in names if "lars_" in n or "clip_norm" in n or "ring_stamp" in n]
    blobs = [n for n in names if "write_blob" in n]
    nb = len(oe.grad_sync.buckets)
    assert len([n for n in ours if "clip_norm_partial" in n]) == nb, ours
    assert len([n for n in ours if "clip_norm_update" in n]) == 1, ours
    assert oe.grad_sync.launches_per_step() == len(ours), (oe.grad_sync.launches_per_step(), ours)
    assert len(blobs) == 1 and n1 - n0 == len(ours) + 1, (n1 - n0, ours, blobs)
    print("OK")
    bps.shutdown()
    """)
    assert out.count("kind ok") == 2 and "OK" in out


def test_bert_tiny_fp8_graphed_against_plain_lamb_with_clipping(tmp_path):
    """bert_tiny with fp8_linear in bf16, one CUDA graph per step, fused LAMB with max_grad_norm=1.0; and the same run
    eager with the plain Lamb on fp32 masters after clip_grad_norm_(..., 1.0).  As in test_gpu_lamb_api.py, the FP8
    GEMMs turn last-bit differences into different gradients, so the losses agree within 1% and each tensor's
    difference between the runs stays below a tenth of how far training moved it.  The first step's norms agree."""
    code = """
    from byteps_b200.models import bert_tiny
    from byteps_b200.torch.graph import GraphedStep
    FUSED = %r
    bps.init()
    torch.manual_seed(0)
    model = bert_tiny(fp8_linear=True, fused_loss=True, fused_norm=True, dropout=0.0).cuda().to(torch.bfloat16).train()
    init = {n: p.detach().float().cpu() for n, p in model.named_parameters()}

    def lamb_groups(ps):
        return [dict(params=[p for p in ps if p.dim() > 1], weight_decay=0.01),
                dict(params=[p for p in ps if p.dim() <= 1], weight_decay=0.0, adapt=False)]

    if FUSED:
        opt = bps.DistributedOptimizer(bps.Lamb(lamb_groups(list(model.parameters())), lr=1e-3),
                                       named_parameters=model.named_parameters(), fused_update=True,
                                       max_grad_norm=1.0)
    else:
        masters = [torch.nn.Parameter(p.detach().float()) for p in model.parameters()]
        opt = bps.Lamb(lamb_groups(masters), lr=1e-3)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 30522, (4, 64), generator=g).cuda()
    labels = torch.randint(0, 30522, (4, 64), generator=g)
    labels[torch.rand(4, 64, generator=g) > 0.15] = -100
    labels = labels.cuda()
    norms = []

    def step():
        model.zero_grad() if not FUSED else opt.zero_grad()
        loss = model(ids, mlm_labels=labels)
        loss.backward()
        if FUSED:
            opt.step()
            norms.append(opt.grad_norm.clone())
        else:
            with torch.no_grad():
                for m, p in zip(masters, model.parameters()):
                    m.grad = p.grad.float() if p.grad is not None else torch.zeros_like(m)
            norms.append(torch.nn.utils.clip_grad_norm_([m for grp in opt.param_groups for m in grp["params"]], 1.0))
            with torch.no_grad():
                opt.step()
                for m, p in zip(masters, model.parameters()):
                    p.copy_(m)
        return loss

    stepper = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams) if FUSED else step
    if not FUSED:
        for _ in range(2):
            step()
    losses = [stepper().detach().float().item() for _ in range(4)]
    torch.save({"losses": losses, "init": init, "norms": [float(n) for n in norms],
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
    assert abs(a["norms"][0] - b["norms"][0]) <= 1e-4 * b["norms"][0], (a["norms"], b["norms"])
    for x, y in zip(a["losses"], b["losses"]):
        assert abs(x - y) <= 1e-2 * abs(y), (a["losses"], b["losses"])
    for n, x in a["params"].items():
        y, w0 = b["params"][n], b["init"][n]
        assert torch.equal(a["init"][n], w0), n
        assert (x - y).norm() <= 0.1 * (y - w0).norm(), (n, (x - y).norm().item(), (y - w0).norm().item())


def _two_ranks(rank, world):
    import byteps_b200.torch as bps
    from _clip import MAX_NORM, Reference, backward, fused, grads, make_params

    torch.cuda.set_device(rank)
    bps.init()
    for kind in ("sgd", "lamb"):
        for dt in (torch.float32, torch.bfloat16):
            ps = make_params(dt)
            ref = Reference(kind, ps)
            opt = fused(kind, ps, max_grad_norm=MAX_NORM)
            for t in range(1, 5):
                mine = grads(t, dt, seed=rank + 1)
                opt.zero_grad()
                backward(ps, mine)
                opt.step()
                every = [grads(t, dt, seed=r + 1) for r in range(world)]
                ref.step([sum(g[i].double() for g in every) / world for i in range(len(ps))])
                torch.cuda.synchronize()
                ref.check(opt, ps, (rank, kind, str(dt), t))
    bps.shutdown()


@pytest.mark.multigpu
def test_two_processes_against_float64_reference():
    """Two ranks, each with its own gradients: the norm is that of their average, and both ranks clip by it."""
    run_workers(_two_ranks, world=2, timeout=300)
