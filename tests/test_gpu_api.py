"""Single-GPU runs of the public API on the CUDA path (world = 1): the fused
optimizer kernels against torch.optim in fp32, whole-step graph capture, the
generic push_pull kernels, and the driver's smoke().  Each case is its own
process so init()/shutdown() state never leaks between tests.
"""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(body: str, timeout=240):
    code = "import sys; sys.path.insert(0, %r)\n" % ROOT + textwrap.dedent(body)
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "DMLC_ROLE", "DMLC_NUM_WORKER", "DMLC_NUM_SERVER"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout


@pytest.mark.parametrize("optim,compression",
                         [pytest.param(o, "none", id=o) for o in ("sgd", "sgd_momentum_nesterov", "adam", "adamw")]
                         + [pytest.param(o, c, id="%s-%s" % (o, c))
                            for c in ("bf16", "fp16") for o in ("sgd_momentum_nesterov", "adam")])
def test_fused_optimizer_matches_torch(optim, compression):
    """fp32 model; with a compressed wire the fused kernel first casts the gradients to bf16/fp16, so the
    reference's gradients are rounded the same way before its step."""
    out = _run("""
        import copy, torch
        import byteps_b200.torch as bps
        torch.manual_seed(0)
        bps.init()
        dev = "cuda"
        def make():
            torch.manual_seed(1)
            return torch.nn.Sequential(torch.nn.Linear(64, 96), torch.nn.Tanh(), torch.nn.Linear(96, 10)).to(dev)
        def mk(params):
            kind = %r
            if kind == "sgd":
                return torch.optim.SGD(params, lr=0.1, weight_decay=1e-3)
            if kind == "sgd_momentum_nesterov":
                return torch.optim.SGD(params, lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-3)
            if kind == "adam":
                return torch.optim.Adam(params, lr=1e-2, weight_decay=1e-2)
            return torch.optim.AdamW(params, lr=1e-2, weight_decay=1e-2)
        comp = %r
        wire = {"none": None, "bf16": torch.bfloat16, "fp16": torch.float16}[comp]
        ref, ours = make(), make()
        ropt = mk(ref.parameters())
        oopt = bps.DistributedOptimizer(mk(ours.parameters()), named_parameters=ours.named_parameters(),
                                        compression=getattr(bps.Compression, comp), fused_update=True)
        x = torch.randn(32, 64, device=dev); y = torch.randint(0, 10, (32,), device=dev)
        for step in range(6):
            for m, o in ((ref, ropt), (ours, oopt)):
                o.zero_grad()
                torch.nn.functional.cross_entropy(m(x), y).backward()
                if o is ropt and wire is not None:
                    for p in ref.parameters():
                        p.grad.copy_(p.grad.to(wire))
                o.step()
        torch.cuda.synchronize()
        # After the first step the two models' gradients differ in the last fp32 bits, so with a 16-bit wire an
        # element near a rounding boundary can land one wire ulp apart in the two runs (about lr * 2^-8 * |g|
        # per step, carried on by momentum).
        tol = 2e-5 if wire is None else 2e-4
        for a, b in zip(ref.parameters(), ours.parameters()):
            err = (a - b).abs().max().item()
            assert err < tol, err
        eng = __import__("byteps_b200.common", fromlist=["engine"]).engine()
        assert eng.launches > 0
        print("OK", eng.launches)
        bps.shutdown()
    """ % (optim, compression))
    assert "OK" in out


def test_graphed_step_with_lr_schedule():
    out = _run("""
        import torch
        import byteps_b200.torch as bps
        from byteps_b200.torch.graph import GraphedStep
        bps.init()
        dev = "cuda"
        def make():
            torch.manual_seed(3)
            return torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 4)).to(dev)
        ref, ours = make(), make()
        ropt = torch.optim.SGD(ref.parameters(), lr=0.2, momentum=0.9)
        base = torch.optim.SGD(ours.parameters(), lr=0.2, momentum=0.9)
        oopt = bps.DistributedOptimizer(base, named_parameters=ours.named_parameters(), fused_update=True)
        x = torch.randn(16, 32, device=dev); y = torch.randint(0, 4, (16,), device=dev)
        def step():
            oopt.zero_grad()
            loss = torch.nn.functional.cross_entropy(ours(x), y)
            loss.backward()
            oopt.step()
            return loss
        g = GraphedStep(step, warmup=2, pre_replay=oopt.refresh_hparams)   # 2 eager + 1 captured (not run) steps
        n_eager = 2
        for _ in range(n_eager):
            ropt.zero_grad(); torch.nn.functional.cross_entropy(ref(x), y).backward(); ropt.step()
        for i in range(5):
            lr = 0.2 * (0.5 ** i)
            for grp in base.param_groups: grp["lr"] = lr
            for grp in ropt.param_groups: grp["lr"] = lr
            g()
            ropt.zero_grad(); torch.nn.functional.cross_entropy(ref(x), y).backward(); ropt.step()
        torch.cuda.synchronize()
        for a, b in zip(ref.parameters(), ours.parameters()):
            err = (a - b).abs().max().item()
            assert err < 5e-5, err
        print("OK")
        bps.shutdown()
    """)
    assert "OK" in out


def test_push_pull_family_world1():
    out = _run("""
        import torch
        import byteps_b200.torch as bps
        bps.init()
        for dt in (torch.float32, torch.bfloat16, torch.float16):
            t = torch.randn(100003, device="cuda").to(dt)
            keep = t.clone()
            o = bps.push_pull(t, average=True, name="w1.%s" % dt)
            assert torch.equal(o, keep)
            h = bps.push_pull_async_inplace(t, average=False, name="w1i.%s" % dt)
            while not bps.poll(h):
                pass
            bps.synchronize(h)
            assert torch.equal(t, keep)
        # same contract as the reference: non-contiguous tensors are rejected
        m = torch.randn(64, 48, device="cuda").t()
        try:
            bps.push_pull(m, name="nc")
            raise SystemExit("non-contiguous tensor was accepted")
        except ValueError:
            pass
        print("OK")
        bps.shutdown()
    """)
    assert "OK" in out


def test_smoke_entry():
    out = _run("""
        import __graft_entry__ as g
        g.smoke()
    """, timeout=400)
    assert "smoke ok" in out
