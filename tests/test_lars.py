"""The plain LARS optimizer (byteps_b200.torch.Lars) on the CPU: the update rule against the float64 transcription of
_lars.py (the trust ratio's phi = 1 cases included), argument checks, the fused kind and checkpoint keys the exchange
relies on, two gloo processes against one, and the ResNet-50 example with --optimizer lars."""
import pytest
import torch

from _lars import transcribed
from _mp import run_workers
from test_examples import _torchrun


@pytest.mark.parametrize("wd", [0.0, 5e-4])
def test_step_matches_float64_transcription(wd):
    """Two groups (the second with adapt=False), five steps with the lr changing, an all-zero parameter (phi = 1 while
    its weights are zero) and a parameter whose gradient is always zero (phi = 1)."""
    from byteps_b200.torch import Lars

    gen = torch.Generator().manual_seed(3)
    shapes = [[(7, 5), (13,), (4,)], [(6,), (3, 2)]]
    params = [[torch.nn.Parameter(torch.randn(s, generator=gen, dtype=torch.float64)) for s in g] for g in shapes]
    with torch.no_grad():
        params[0][2].zero_()                               # all-zero parameter
    groups = [dict(lr=0.2, momentum=0.9, weight_decay=wd, trust_coefficient=0.01, eps=1e-9, adapt=True),
              dict(lr=0.05, momentum=0.8, weight_decay=wd, trust_coefficient=0.001, eps=0.0, adapt=False)]
    start = [[p.detach().flatten().tolist() for p in g] for g in params]
    opt = Lars([dict(params=ps, **grp) for ps, grp in zip(params, groups)])
    lrs = [1.0, 1.0, 0.5, 0.5, 0.25]
    grads = []
    for s in lrs:
        step_grads = []
        for gi, ps in enumerate(params):
            gs = []
            for pi, p in enumerate(ps):
                g = torch.randn(p.shape, generator=gen, dtype=torch.float64)
                if gi == 0 and pi == 1:
                    g.zero_()                              # a parameter whose gradient is zero
                p.grad = g
                gs.append(g.flatten().tolist())
            step_grads.append(gs)
        grads.append(step_grads)
        for grp, base in zip(opt.param_groups, groups):
            grp["lr"] = base["lr"] * s
        opt.step()
    want = transcribed(start, grads, groups, lrs)
    for gi, ps in enumerate(params):
        for pi, p in enumerate(ps):
            got = p.detach().flatten()
            exp = torch.tensor(want[gi][pi], dtype=torch.float64)
            assert torch.allclose(got, exp, rtol=1e-12, atol=1e-14), (gi, pi, (got - exp).abs().max().item())
            assert sorted(opt.state[p]) == ["momentum_buffer"]
    assert not torch.equal(params[0][2].detach(), torch.zeros(4, dtype=torch.float64))


def test_phi_is_one_without_adapt_or_a_norm():
    """adapt=False, w = 0 and g = 0 each give phi = 1: the first step is v = lr * (g + wd * w)."""
    from byteps_b200.torch import Lars

    g = torch.tensor([0.5, -1.0, 2.0], dtype=torch.float64)
    for w0, grad, adapt in ((torch.tensor([1.0, 2.0, -2.0]), g, False), (torch.zeros(3), g, True),
                            (torch.tensor([1.0, 2.0, -2.0]), torch.zeros(3), True)):
        p = torch.nn.Parameter(w0.double())
        opt = Lars([p], lr=0.1, momentum=0.9, weight_decay=0.01, trust_coefficient=0.001, adapt=adapt)
        p.grad = grad.double().clone()
        opt.step()
        v = 0.1 * (grad.double() + 0.01 * w0.double())
        assert torch.allclose(opt.state[p]["momentum_buffer"], v, rtol=1e-15, atol=0), adapt
        assert torch.allclose(p.detach(), w0.double() - v, rtol=1e-15, atol=0), adapt


@pytest.mark.parametrize("kw, msg", [(dict(lr=-1.0), "learning rate"), (dict(momentum=-0.1), "momentum"),
                                     (dict(weight_decay=-0.1), "weight_decay"),
                                     (dict(trust_coefficient=0.0), "trust_coefficient"),
                                     (dict(eps=-1e-6), "epsilon")])
def test_argument_errors(kw, msg):
    from byteps_b200.torch import Lars

    with pytest.raises(ValueError, match=msg):
        Lars([torch.nn.Parameter(torch.zeros(3))], **kw)


def test_sparse_gradients_are_rejected():
    from byteps_b200.torch import Lars

    emb = torch.nn.Embedding(10, 4, sparse=True)
    emb(torch.tensor([1, 2])).sum().backward()
    with pytest.raises(RuntimeError, match="sparse"):
        Lars(emb.parameters()).step()


def test_fused_kind_and_state_keys():
    from byteps_b200.torch import Lars, _DistributedOptimizer, _fused_kind

    class MyLars(Lars):
        pass

    assert _fused_kind(Lars, [{}]) == "lars"
    assert _fused_kind(MyLars, [{}]) == "lars"
    assert _DistributedOptimizer._FUSED_KEYS["lars"] == ("momentum_buffer",)
    p = torch.nn.Parameter(torch.randn(5))
    lars = Lars([p], momentum=0.0)
    p.grad = torch.ones(5)
    lars.step()
    assert sorted(lars.state_dict()["state"][0]) == ["momentum_buffer"]


def test_step_does_not_sync_with_the_host(monkeypatch):
    """phi is formed with torch.where: no .item() / bool() of a tensor inside step()."""
    from byteps_b200.torch import Lars

    p = torch.nn.Parameter(torch.randn(6))
    opt = Lars([p], weight_decay=1e-4)
    p.grad = torch.randn(6)

    def refuse(*a, **k):
        raise AssertionError("host sync in Lars.step")

    monkeypatch.setattr(torch.Tensor, "item", refuse)
    monkeypatch.setattr(torch.Tensor, "__bool__", refuse)
    opt.step()


def _two_process_lars(rank, world):
    import byteps_b200.torch as bps

    bps.init()
    torch.manual_seed(1234 + rank)   # different init per rank: broadcast must fix it
    mk = lambda: torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 4))  # noqa: E731
    model = mk()
    groups = lambda m: [dict(params=[m[0].weight, m[2].weight], weight_decay=1e-4),  # noqa: E731
                        dict(params=[m[0].bias, m[2].bias], weight_decay=0.0, adapt=False)]
    opt = bps.DistributedOptimizer(bps.Lars(groups(model), lr=0.5, trust_coefficient=0.02),
                                   named_parameters=model.named_parameters())
    bps.broadcast_parameters(model.state_dict(), root_rank=0)
    ref = mk()
    ref.load_state_dict(model.state_dict())
    ref_opt = bps.Lars(groups(ref), lr=0.5, trust_coefficient=0.02)
    torch.manual_seed(99)
    for _ in range(4):
        x, y = torch.randn(world * 4, 8), torch.randn(world * 4, 4)
        opt.zero_grad()
        torch.nn.functional.mse_loss(model(x[rank * 4:(rank + 1) * 4]), y[rank * 4:(rank + 1) * 4]).backward()
        opt.step()
        ref_opt.zero_grad()
        torch.nn.functional.mse_loss(ref(x), y).backward()    # the full batch: the average of the ranks' gradients
        ref_opt.step()
    for a, b in zip(model.parameters(), ref.parameters()):
        assert torch.allclose(a, b, atol=1e-5), (a - b).abs().max()
    bps.shutdown()


def test_two_gloo_processes_match_one():
    run_workers(_two_process_lars, world=2)


def test_resnet_example_with_lars(tmp_path):
    out = _torchrun("train_imagenet_resnet50_byteps.py", "--no-cuda", "--model", "resnet18", "--image-size", "32",
                    "--batch-size", "2", "--steps-per-epoch", "2", "--epochs", "1", "--optimizer", "lars",
                    "--checkpoint-format", str(tmp_path / "ckpt-{epoch}.pt"))
    assert "epoch 1" in out
