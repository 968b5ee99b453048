"""Global gradient-norm clipping (DistributedOptimizer's max_grad_norm) on the paths that do not fuse the update,
on the CPU: bit for bit what synchronize() + clip_grad_norm_ + step() of torch gives, in one process and over gloo
at two; the argument checks; and grad_norm."""
import math

import pytest
import torch

from _mp import run_workers


def _clip_against_hand_written(rank, world):
    """Model A: DistributedOptimizer(..., max_grad_norm=0.3).  Model B, same weights: the recipe written out,
    synchronize(); clip_grad_norm_(); with skip_synchronize(): step().  Both see the same per-rank batches, and one
    of B's steps has a norm below max_grad_norm (no clipping)."""
    import byteps_b200.torch as bps

    bps.init()
    torch.manual_seed(5)
    mk = lambda: torch.nn.Sequential(torch.nn.Linear(6, 12), torch.nn.Tanh(), torch.nn.Linear(12, 3))  # noqa: E731
    a, b = mk(), mk()
    b.load_state_dict(a.state_dict())
    groups = lambda m: [dict(params=[m[0].weight, m[2].weight]),  # noqa: E731
                        dict(params=[m[0].bias, m[2].bias], weight_decay=0.0)]
    oa = bps.DistributedOptimizer(torch.optim.SGD(groups(a), lr=0.1, momentum=0.9, weight_decay=1e-3),
                                  named_parameters=[("a." + n, p) for n, p in a.named_parameters()],
                                  max_grad_norm=0.3)
    ob = bps.DistributedOptimizer(torch.optim.SGD(groups(b), lr=0.1, momentum=0.9, weight_decay=1e-3),
                                  named_parameters=[("b." + n, p) for n, p in b.named_parameters()])
    with pytest.raises(RuntimeError, match="max_grad_norm"):
        ob.grad_norm
    assert float(oa.grad_norm) == 0.0
    torch.manual_seed(17)
    clipped = 0
    for step in range(5):
        x, y = torch.randn(world * 4, 6), torch.randn(world * 4, 3) * 3.0
        k = 1e-3 if step == 2 else 1.0       # a step whose norm stays below max_grad_norm
        mine = slice(rank * 4, (rank + 1) * 4)
        for m, o in ((a, oa), (b, ob)):
            o.zero_grad()
            (k * torch.nn.functional.mse_loss(m(x[mine]), y[mine])).backward()
        oa.step()
        ob.synchronize()
        # in param-group order, as the optimizer passes them: the order of the per-tensor norms rounds the total
        norm = torch.nn.utils.clip_grad_norm_([p for g in ob.param_groups for p in g["params"]], 0.3)
        with ob.skip_synchronize():
            ob.step()
        assert oa.grad_norm.dtype == torch.float32 and oa.grad_norm.dim() == 0
        assert torch.equal(oa.grad_norm, norm), (step, oa.grad_norm, norm)
        clipped += int(norm.item() > 0.3)
        for p, q in zip(a.parameters(), b.parameters()):
            assert torch.equal(p, q), (step, (p - q).abs().max())
    assert 0 < clipped < 5
    bps.shutdown()


def test_unfused_clip_matches_hand_written_one_process():
    run_workers(_clip_against_hand_written, world=1)


def test_unfused_clip_matches_hand_written_two_gloo_processes():
    run_workers(_clip_against_hand_written, world=2)


@pytest.mark.parametrize("bad", [0.0, -1.0, math.inf, math.nan, True, "1.0x", [1.0], object()])
def test_max_grad_norm_must_be_finite_and_positive(bad):
    from byteps_b200.torch import _checked_max_grad_norm

    with pytest.raises(ValueError, match="max_grad_norm"):
        _checked_max_grad_norm(bad)


def test_max_grad_norm_accepts_numbers():
    from byteps_b200.torch import _checked_max_grad_norm

    assert _checked_max_grad_norm(None) is None
    assert _checked_max_grad_norm(1) == 1.0 and isinstance(_checked_max_grad_norm(1), float)
    assert _checked_max_grad_norm("0.5") == 0.5
    assert _checked_max_grad_norm(torch.tensor(2.0)) == 2.0


def _bad_argument_in_constructor(rank, world):
    import byteps_b200.torch as bps

    bps.init()
    p = torch.nn.Parameter(torch.zeros(3))
    with pytest.raises(ValueError, match="max_grad_norm"):
        bps.DistributedOptimizer(torch.optim.SGD([p], lr=0.1), named_parameters=[("p", p)], max_grad_norm=-2.0)
    bps.shutdown()


def test_constructor_rejects_a_bad_max_grad_norm():
    run_workers(_bad_argument_in_constructor, world=1)


def test_bucket_layer_needs_the_fused_update():
    from byteps_b200.parallel.bucket import BucketedGradSync

    class Eng:
        size, rank = 1, 0

    p = torch.nn.Parameter(torch.zeros(3))
    with pytest.raises(ValueError, match="max_grad_norm"):
        BucketedGradSync(Eng(), [dict(params=[p])], fused=None, max_grad_norm=1.0)


def test_bert_example_with_max_grad_norm():
    from test_examples import _torchrun

    out = _torchrun("train_bert_byteps.py", "--no-cuda", "--model", "bert_tiny", "--batch-size", "2", "--seq-len", "16",
                    "--steps", "2", "--warmup-steps", "1", "--max-grad-norm", "1.0")
    assert "tokens/sec" in out
