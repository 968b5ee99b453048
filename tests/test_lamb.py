"""The plain LAMB optimizer (byteps_b200.torch.Lamb) on the CPU: the update rule against a float64 transcription,
argument checks, the fused kind and checkpoint keys the exchange relies on, two gloo processes against one, and the
BERT example with --optimizer lamb."""
import pytest
import torch

from _mp import run_workers
from test_examples import _torchrun


def _transcribed(ws, grads, groups, lrs):
    """The rule in float64, written out element by element from its definition: per step t and parameter,
    m, v, u = m^ / (sqrt(v^) + eps) + wd * w, phi = ||w|| / ||u|| (1 if not adapt or a norm is 0), w -= lr*phi*u."""
    import math

    ws = [[list(map(float, w.flatten().tolist())) for w in g_ws] for g_ws in ws]
    ms = [[[0.0] * len(w) for w in g_ws] for g_ws in ws]
    vs = [[[0.0] * len(w) for w in g_ws] for g_ws in ws]
    for t, lr_scale in enumerate(lrs, start=1):
        for gi, grp in enumerate(groups):
            b1, b2 = grp["betas"]
            lr, eps, wd, adapt = grp["lr"] * lr_scale, grp["eps"], grp["weight_decay"], grp["adapt"]
            for pi, w in enumerate(ws[gi]):
                g = grads[t - 1][gi][pi]
                m, v = ms[gi][pi], vs[gi][pi]
                u = []
                for k in range(len(w)):
                    m[k] = b1 * m[k] + (1 - b1) * g[k]
                    v[k] = b2 * v[k] + (1 - b2) * g[k] * g[k]
                    u.append((m[k] / (1 - b1 ** t)) / (math.sqrt(v[k] / (1 - b2 ** t)) + eps) + wd * w[k])
                wn = math.sqrt(sum(x * x for x in w))
                un = math.sqrt(sum(x * x for x in u))
                phi = wn / un if adapt and wn > 0 and un > 0 else 1.0
                for k in range(len(w)):
                    w[k] -= lr * phi * u[k]
    return ws


@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_step_matches_float64_transcription(wd):
    """Two groups (the second with adapt=False), five steps with the lr changing, an all-zero parameter (phi = 1) and
    a parameter whose gradient is always zero."""
    from byteps_b200.torch import Lamb

    gen = torch.Generator().manual_seed(3)
    shapes = [[(7, 5), (13,), (4,)], [(6,), (3, 2)]]
    params = [[torch.nn.Parameter(torch.randn(s, generator=gen, dtype=torch.float64)) for s in g] for g in shapes]
    with torch.no_grad():
        params[0][2].zero_()                               # all-zero parameter
    groups = [dict(lr=0.02, betas=(0.9, 0.99), eps=1e-6, weight_decay=wd, adapt=True),
              dict(lr=0.05, betas=(0.8, 0.999), eps=1e-8, weight_decay=wd, adapt=False)]
    start = [[p.detach().clone() for p in g] for g in params]
    opt = Lamb([dict(params=ps, **{k: v for k, v in grp.items()}) for ps, grp in zip(params, groups)])
    lrs = [1.0, 1.0, 0.5, 0.5, 0.25]
    grads = []
    for t, s in enumerate(lrs):
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
    want = _transcribed(start, grads, groups, lrs)
    for gi, ps in enumerate(params):
        for pi, p in enumerate(ps):
            got = p.detach().flatten()
            exp = torch.tensor(want[gi][pi], dtype=torch.float64)
            assert torch.allclose(got, exp, rtol=1e-12, atol=1e-14), (gi, pi, (got - exp).abs().max().item())
            assert int(opt.state[p]["step"].item()) == len(lrs)
    assert not torch.equal(params[0][2].detach(), torch.zeros(4, dtype=torch.float64))


@pytest.mark.parametrize("kw, msg", [(dict(lr=-1.0), "learning rate"), (dict(eps=-1e-6), "epsilon"),
                                     (dict(betas=(1.0, 0.999)), "beta parameter at index 0"),
                                     (dict(betas=(0.9, -0.1)), "beta parameter at index 1"),
                                     (dict(weight_decay=-0.1), "weight_decay")])
def test_argument_errors(kw, msg):
    from byteps_b200.torch import Lamb

    with pytest.raises(ValueError, match=msg):
        Lamb([torch.nn.Parameter(torch.zeros(3))], **kw)


def test_sparse_gradients_are_rejected():
    from byteps_b200.torch import Lamb

    emb = torch.nn.Embedding(10, 4, sparse=True)
    emb(torch.tensor([1, 2])).sum().backward()
    with pytest.raises(RuntimeError, match="sparse"):
        Lamb(emb.parameters()).step()


def test_fused_kind_and_state_keys():
    from byteps_b200.torch import Lamb, _fused_kind

    class MyLamb(Lamb):
        pass

    p = torch.nn.Parameter(torch.randn(5))
    assert _fused_kind(Lamb, [{}]) == "lamb"
    assert _fused_kind(MyLamb, [{}]) == "lamb"
    lamb, adam = Lamb([p]), torch.optim.Adam([torch.nn.Parameter(p.detach().clone())])
    for o in (lamb, adam):
        o.param_groups[0]["params"][0].grad = torch.ones(5)
        o.step()
    a, b = lamb.state_dict()["state"][0], adam.state_dict()["state"][0]
    assert sorted(a) == sorted(b) == ["exp_avg", "exp_avg_sq", "step"]
    assert a["step"].dtype == b["step"].dtype and a["step"].shape == b["step"].shape


def _two_process_lamb(rank, world):
    import byteps_b200.torch as bps

    bps.init()
    torch.manual_seed(1234 + rank)   # different init per rank: broadcast must fix it
    mk = lambda: torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 4))  # noqa: E731
    model = mk()
    groups = lambda m: [dict(params=[m[0].weight, m[2].weight], weight_decay=0.01),  # noqa: E731
                        dict(params=[m[0].bias, m[2].bias], weight_decay=0.0, adapt=False)]
    opt = bps.DistributedOptimizer(bps.Lamb(groups(model), lr=0.01), named_parameters=model.named_parameters())
    bps.broadcast_parameters(model.state_dict(), root_rank=0)
    ref = mk()
    ref.load_state_dict(model.state_dict())
    ref_opt = bps.Lamb(groups(ref), lr=0.01)
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
    run_workers(_two_process_lamb, world=2)


def test_bert_example_with_lamb():
    out = _torchrun("train_bert_byteps.py", "--no-cuda", "--model", "bert_tiny", "--batch-size", "2", "--seq-len", "16",
                    "--steps", "2", "--warmup-steps", "1", "--optimizer", "lamb")
    assert "tokens/sec" in out
