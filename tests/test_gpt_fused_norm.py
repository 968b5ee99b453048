"""GPT-2-style decoder with fused_norm (models/gpt.py) and DropoutAddLayerNorm's return_sum (ops/ln.py) on the CPU,
where every junction takes the stock dropout / add / layer_norm composition: the flag keeps the stock parameters
and state_dict, and the model computes the stock loss and gradients bit for bit, dropout included, padded and
packed, alone and with the other flags."""
import pytest
import torch
import torch.nn.functional as F

from byteps_b200.models import gpt_tiny
from byteps_b200.ops.ln import DropoutAddLayerNorm, dropout_add_layer_norm

OTHER = dict(fused_attention=True, fused_loss=True, fp8_linear=True)


def test_fused_norm_keeps_parameters_and_state_dict():
    torch.manual_seed(0)
    stock = gpt_tiny()
    fused = gpt_tiny(fused_norm=True)
    norms = [m for blk in fused.blocks for m in (blk.ln1, blk.ln2)] + [fused.ln_f]
    assert all(type(m) is DropoutAddLayerNorm and m.p == 0.1 and m.eps == 1e-5 for m in norms)
    assert all(type(m) is not DropoutAddLayerNorm for m in stock.modules())
    assert [(n, p.shape) for n, p in fused.named_parameters()] == [(n, p.shape) for n, p in stock.named_parameters()]
    ours, theirs = fused.state_dict(), stock.state_dict()
    assert list(ours) == list(theirs)
    assert all(ours[k].shape == theirs[k].shape and ours[k].dtype == theirs[k].dtype for k in ours)
    sd = {k: v + 1 for k, v in theirs.items()}
    fused.load_state_dict(sd, strict=True)
    for k, v in fused.state_dict().items():
        assert torch.equal(v, sd[k]), k
    stock.load_state_dict(fused.state_dict(), strict=True)


def test_fused_norm_block_has_no_stock_forward():
    blk = gpt_tiny(fused_norm=True).blocks[0]
    with pytest.raises(RuntimeError, match="fused_forward"):
        blk(torch.zeros(1, 4, 128))


@pytest.mark.parametrize("flags", ["norm", "all"])
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
def test_fused_norm_on_cpu_is_stock(packed, flags):
    """dropout 0.1, seeded: loss, logits and every gradient bit-identical to the stock model, in training and eval"""
    torch.manual_seed(0)
    stock = gpt_tiny(dropout=0.1)
    fused = gpt_tiny(dropout=0.1, fused_norm=True, **(OTHER if flags == "all" else {}))
    fused.load_state_dict(stock.state_dict())
    ids = torch.randint(0, 50257, (2, 24))
    labels = ids.clone()
    labels[1, 17:] = -100
    kw = {}
    if packed:
        kw = dict(cu_seqlens=torch.tensor([1, 9, 9, 30, 44], dtype=torch.int32), max_seqlen=24)
    for training in (True, False):
        stock.train(training)
        fused.train(training)
        torch.manual_seed(2)
        a = stock(ids, labels, **kw)
        a.backward()
        torch.manual_seed(2)
        c = fused(ids, labels, **kw)
        c.backward()
        assert torch.equal(a, c), training
        for (n, p), (_, q) in zip(stock.named_parameters(), fused.named_parameters()):
            assert torch.equal(p.grad, q.grad), (n, training)
            p.grad = q.grad = None
        torch.manual_seed(3)
        a = stock(ids, **kw)
        torch.manual_seed(3)
        assert torch.equal(a, fused(ids, **kw)), training


def test_dropout_is_drawn():
    """the fused model's junction dropouts are live in training: two draws differ, the same seed repeats"""
    torch.manual_seed(0)
    m = gpt_tiny(dropout=0.1, fused_norm=True).train()
    ids = torch.randint(0, 50257, (2, 16))
    torch.manual_seed(1)
    a = m(ids, ids)
    b = m(ids, ids)
    torch.manual_seed(1)
    assert torch.equal(m(ids, ids), a) and not torch.equal(a, b)


# ------------------------------------------------------------------------------------- the op's return_sum on CPU
@pytest.mark.parametrize("residual", [False, True], ids=["no_residual", "residual"])
@pytest.mark.parametrize("p", [0.0, 0.25])
def test_return_sum_cpu_is_stock(residual, p):
    torch.manual_seed(0)
    mod = DropoutAddLayerNorm(64, eps=1e-6, p=p)
    with torch.no_grad():
        mod.weight.normal_()
        mod.bias.normal_()
    y = torch.randn(5, 7, 64, requires_grad=True)
    r = torch.randn(5, 7, 64, requires_grad=True) if residual else None
    inputs = [y, mod.weight, mod.bias] + ([r] if residual else [])
    for training in (True, False):
        mod.train(training)
        torch.manual_seed(1)
        out, z = mod(y, r, return_sum=True)
        torch.manual_seed(1)
        z_ref = F.dropout(y, p, training)
        if residual:
            z_ref = r + z_ref
        ref = F.layer_norm(z_ref, (64,), mod.weight, mod.bias, 1e-6)
        assert torch.equal(out, ref) and torch.equal(z, z_ref), training
        # both outputs carry gradient, and the residual stream's reaches y and residual
        dz = torch.randn_like(z)
        ga = torch.autograd.grad((out * out).sum() + (z * dz).sum(), inputs)
        gb = torch.autograd.grad((ref * ref).sum() + (z_ref * dz).sum(), inputs)
        for a, b in zip(ga, gb):
            assert torch.equal(a, b), training


def test_return_sum_and_mask_order():
    y = torch.randn(3, 16)
    w, b = torch.ones(16), torch.zeros(16)
    res = dropout_add_layer_norm(y, y, w, b, 0.0, 1e-5, True, return_mask=True, return_sum=True)
    assert len(res) == 3 and res[2] is None and torch.equal(res[1], y + y)
    out, z = dropout_add_layer_norm(y, None, w, b, 0.0, 1e-5, True, return_sum=True)
    assert z is y and torch.equal(out, F.layer_norm(y, (16,), w, b, 1e-5))
    assert isinstance(dropout_add_layer_norm(y, None, w, b, 0.0, 1e-5, True), torch.Tensor)
