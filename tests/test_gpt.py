"""GPT-2-style decoder (models/gpt.py) on the CPU: the fused flags keep the stock parameters and, on the CPU, the
stock computation bit for bit; a packed stream equals its sequences run one at a time; the loss is next-token cross
entropy with targets that never cross a sequence boundary."""
import pytest
import torch
import torch.nn.functional as F

from byteps_b200.models import GptLMHeadModel, get_model, gpt2_medium, gpt2_small, gpt_tiny
from byteps_b200.models.bert import num_params

FLAGS = dict(fused_attention=True, fused_loss=True, fp8_linear=True)


def test_flags_keep_parameters_and_state_dict():
    torch.manual_seed(0)
    stock = gpt_tiny()
    fused = gpt_tiny(**FLAGS)
    assert [n for n, _ in fused.named_parameters()] == [n for n, _ in stock.named_parameters()]
    ours, theirs = fused.state_dict(), stock.state_dict()
    assert list(ours) == list(theirs)
    assert all(ours[k].shape == theirs[k].shape and ours[k].dtype == theirs[k].dtype for k in ours)
    fused.load_state_dict(theirs, strict=True)
    stock.load_state_dict(fused.state_dict(), strict=True)


def test_sizes_and_factories():
    assert 124e6 < num_params(gpt2_small()) < 125e6
    assert 350e6 < num_params(gpt2_medium()) < 356e6
    m = get_model("gpt_tiny")
    assert isinstance(m, GptLMHeadModel) and m.config.vocab_size % 64 == 0
    assert m.wte.weight is not None and "lm_head" not in dict(m.named_parameters())   # tied head


@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
def test_flags_on_cpu_are_stock(packed):
    torch.manual_seed(0)
    stock = gpt_tiny()
    fused = gpt_tiny(**FLAGS)
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
            assert torch.equal(p.grad, q.grad), n
            p.grad = q.grad = None
        torch.manual_seed(2)
        a = stock(ids, **kw)
        torch.manual_seed(2)
        assert torch.equal(a, fused(ids, **kw))


def _tiny64():
    torch.manual_seed(0)
    return gpt_tiny(dropout=0.0).double()


def test_loss_is_next_token_cross_entropy():
    m = _tiny64()
    ids = torch.randint(0, 50257, (3, 20))
    labels = ids.clone()
    labels[2, 11:] = -100
    logits = m(ids)
    terms = []
    for b in range(3):
        for t in range(19):
            y = int(labels[b, t + 1])
            if y != -100:
                terms.append(-torch.log_softmax(logits[b, t], -1)[y])
    ref = torch.stack(terms).mean()
    loss = m(ids, labels)
    assert abs(loss.item() - ref.item()) <= 1e-12 * abs(ref.item())


def test_packed_stream_equals_sequences_one_at_a_time():
    """float64: the loss within fp64 rounding, gradients within 1e-10"""
    m = _tiny64()
    b, s = 2, 30
    cu = [2, 13, 13, 40, 41, 57]     # an empty and a one-token sequence, tokens outside before and after
    ids = torch.randint(0, 50257, (b, s), generator=torch.Generator().manual_seed(1))
    flat = ids.view(-1)
    loss = m(ids, ids, cu_seqlens=torch.tensor(cu, dtype=torch.int32), max_seqlen=s)
    loss.backward()
    packed = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad()
    total, count = 0.0, 0
    for a, c in zip(cu[:-1], cu[1:]):
        if c - a < 2:
            continue     # no target inside a sequence of fewer than 2 tokens
        part = m(flat[None, a:c], flat[None, a:c])
        (part * (c - a - 1)).backward()
        total += part.item() * (c - a - 1)
        count += c - a - 1
    ref = total / count
    assert abs(loss.item() - ref) <= 1e-13 * abs(ref)
    for n, p in m.named_parameters():
        g = p.grad / count
        assert (packed[n] - g).abs().max().item() <= 1e-10 * max(g.abs().max().item(), 1e-30), n


def test_boundary_targets_are_ignored():
    """Changing the label of a token that starts a sequence, or lies outside every sequence, changes nothing; the
    label of a token inside a sequence does."""
    m = _tiny64()
    ids = torch.randint(0, 50257, (1, 24), generator=torch.Generator().manual_seed(3))
    cu = torch.tensor([2, 10, 20], dtype=torch.int32)
    base = m(ids, ids, cu_seqlens=cu)
    for t, moves in ((0, False), (1, False), (2, False), (10, False), (20, False), (23, False), (5, True),
                     (15, True)):
        lab = ids.clone()
        lab[0, t] = (lab[0, t] + 1) % 50257
        assert torch.equal(m(ids, lab, cu_seqlens=cu), base) != moves, t
    # equal to a padded batch of the two sequences with -100 past their ends
    pad = torch.full((2, 10), 0, dtype=ids.dtype)
    lab = torch.full((2, 10), -100, dtype=ids.dtype)
    pad[0, :8], pad[1] = ids[0, 2:10], ids[0, 10:20]
    lab[0, :8], lab[1] = ids[0, 2:10], ids[0, 10:20]
    padded = m(pad, lab)
    assert abs(padded.item() - base.item()) <= 1e-13 * abs(base.item())


def test_returns_logits_without_labels():
    m = gpt_tiny()
    out = m(torch.randint(0, 100, (2, 7)))
    assert out.shape == (2, 7, 50304) and out.is_contiguous()
