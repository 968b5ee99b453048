"""Gradient sums at ResNet's block junctions inside the batch-norm backward (ops/bn_act.py, kernels/bn_act.cu).

A block's output feeds the next block's conv1 and its skip path.  ``BatchNormAct2d(..., pair=True)`` returns the
output and an alias of it, so autograd hands the last batch norm of a block the two gradients separately, and the
single-launch backward with a residual sums them as it reads them.  The sum rounds as torch's ``add`` does (fp32,
one rounding to the activation dtype), so every result must be bit-identical to the same backward fed the gradient
torch summed.  Every other path sums the two in torch first.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from byteps_b200.models import resnet18, resnet50
from byteps_b200.ops import bn_act as bn_mod
from byteps_b200.ops.bn_act import BatchNormAct2d

CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
DTYPES = [torch.bfloat16, torch.float16, torch.float32]
# the four expanded ResNet-50 shapes at batch 64, and small odd ones: C = 8, row counts that are no multiple of a
# block's row step, a partial channel group
SHAPES = [(64, 256, 56, 56), (64, 512, 28, 28), (64, 1024, 14, 14), (64, 2048, 7, 7),
          (3, 8, 5, 7), (2, 40, 9, 7), (1, 24, 37, 3)]
CAPS = ["full", "part", "none"]


def _dt_id(d):
    return str(d).replace("torch.", "")


def _shape_id(s):
    return "x".join(map(str, s))


def _chained(model, x):
    """ResNet forward with every block called on one tensor: autograd sums the junction gradients."""
    t = model.maxpool(model.bn1(model.conv1(x)))
    for layer in (model.layer1, model.layer2, model.layer3, model.layer4):
        for b in layer:
            t = b(t)
    return model.fc(torch.flatten(model.avgpool(t), 1))


def _param_grads(model, fwd, x, y):
    for p in model.parameters():
        p.grad = None
    F.cross_entropy(fwd(x).float(), y).backward()
    return [p.grad.clone() for p in model.parameters()]


# ----------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("ctor", [resnet18, resnet50], ids=["resnet18", "resnet50"])
def test_resnet_cpu_pair_grads_match_chained_blocks(ctor):
    torch.manual_seed(0)
    model = ctor()
    twin = copy.deepcopy(model)
    model.train()
    twin.train()
    x = torch.randn(2, 3, 64, 64)
    y = torch.randint(0, 1000, (2,))
    got = _param_grads(model, model, x, y)
    want = _param_grads(twin, lambda t: _chained(twin, t), x, y)
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), "parameter %d" % i


def test_stock_path_returns_the_alias():
    bn = BatchNormAct2d(8, act="relu").train()
    x = torch.randn(2, 8, 3, 3, requires_grad=True)
    r = torch.randn(2, 8, 3, 3)
    y, alias = bn(x, r, pair=True)
    assert alias is y
    (y * 2 + alias * 3).sum().backward()
    g = x.grad.clone()
    x.grad = None
    bn(x, r).mul(5).sum().backward()
    assert torch.equal(x.grad, g)


# ----------------------------------------------------------------------------------------------------------- GPU
def _make(shape, dtype, seed=0):
    n, c, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    nhwc = lambda t: t.to(dtype).contiguous(memory_format=torch.channels_last)  # noqa: E731
    x = nhwc(torch.randn(n, c, h, w, device="cuda", generator=g) * 1.5 + 0.3)
    r, g1, g2 = (nhwc(torch.randn(n, c, h, w, device="cuda", generator=g)) for _ in range(3))
    bn = BatchNormAct2d(c, act="relu").cuda().train()
    with torch.no_grad():
        bn.weight.copy_(torch.randn(c, device="cuda", generator=g))
        bn.bias.copy_(torch.randn(c, device="cuda", generator=g) * 0.5)
    return bn, x, r, g1, g2


def _backward(bn, state, x, r, grads, pair):
    """dx, dres, dweight, dbias of one step from `state`; grads = (g_main, g_skip or None) with pair, else (g,)."""
    bn.load_state_dict(state)
    bn.weight.grad = bn.bias.grad = None
    xg, rg = x.detach().clone().requires_grad_(True), r.detach().clone().requires_grad_(True)
    if pair:
        y, alias = bn(xg, rg, pair=True)
        outs, gs = ([y, alias], list(grads)) if grads[1] is not None else ([y], [grads[0]])
    else:
        outs, gs = [bn(xg, rg)], [grads[0]]
    assert type(outs[0].grad_fn).__name__ == "_BatchNormActFnBackward", "fused path not taken"
    torch.autograd.backward(outs, gs)
    return dict(dx=xg.grad, dres=rg.grad, dw=bn.weight.grad.clone(), db=bn.bias.grad.clone())


@pytest.fixture
def summed_in_kernel(monkeypatch):
    """Records, per backward with two gradients, whether the kernel summed them."""
    seen = []
    real = bn_mod._sum_in_kernel

    def spy(dy, dy2, x):
        seen.append(real(dy, dy2, x))
        return seen[-1]

    monkeypatch.setattr(bn_mod, "_sum_in_kernel", spy)
    yield seen
    bn_mod.RESIDENT_CAP = None


def _set_cap(mode, shape, dtype):
    n, c, h, w = shape
    bn_mod.RESIDENT_CAP = None
    full = bn_mod._native.cuda().bn_act_plan(1, CODES[dtype], n * h * w, c, -1, True, True, True)
    assert full is not None and full["ring_depth"] > 0
    bn_mod.RESIDENT_CAP = {"full": None, "part": full["held_bytes"] // 2, "none": 0}[mode]
    p = bn_mod._native.cuda().bn_act_plan(1, CODES[dtype], n * h * w, c, bn_mod._cap(), True, True, True)
    if mode == "part":
        assert 0 <= p["held_rows"] < full["held_rows"]
    elif mode == "none":
        assert p["held_rows"] == 0


def _assert_same(got, want):
    for k, v in want.items():
        assert torch.equal(got[k], v), k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", CAPS)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
def test_two_gradients_match_torch_sum(shape, dtype, mode, summed_in_kernel):
    bn, x, r, g1, g2 = _make(shape, dtype)
    state = copy.deepcopy(bn.state_dict())
    _set_cap(mode, shape, dtype)
    want = _backward(bn, state, x, r, (g1 + g2,), pair=False)
    got = _backward(bn, state, x, r, (g1, g2), pair=True)
    assert summed_in_kernel == [True]
    _assert_same(got, want)
    # the alias unused: dy2 absent
    _assert_same(_backward(bn, state, x, r, (g1, None), pair=True), _backward(bn, state, x, r, (g1,), pair=False))
    assert summed_in_kernel == [True]


def _misaligned(t):
    """A channels_last copy of t whose data starts one element past a 16-byte boundary."""
    n, c, h, w = t.shape
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    v.copy_(t)
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["nchw", "misaligned"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("shape", [(3, 8, 5, 7), (2, 40, 9, 7), (64, 512, 28, 28)], ids=_shape_id)
def test_second_gradient_fallbacks(shape, dtype, case, summed_in_kernel):
    bn, x, r, g1, g2 = _make(shape, dtype, seed=1)
    state = copy.deepcopy(bn.state_dict())
    odd = g2.contiguous() if case == "nchw" else _misaligned(g2)
    assert torch.equal(odd, g2) and (case != "misaligned" or odd.data_ptr() % 16 != 0)
    want = _backward(bn, state, x, r, (g1 + g2,), pair=False)
    got = _backward(bn, state, x, r, (g1, odd), pair=True)
    assert summed_in_kernel == [False]
    _assert_same(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_second_gradient_of_another_dtype_is_summed_in_torch(dtype):
    """Autograd casts a gradient to its output's dtype before backward; a direct caller may not, so the kernel only
    reads a second gradient of the activation dtype."""
    _, x, _, g1, g2 = _make((2, 40, 9, 7), dtype)
    other = torch.float32 if dtype != torch.float32 else torch.bfloat16
    assert bn_mod._sum_in_kernel(g1, g2, x)
    assert not bn_mod._sum_in_kernel(g1, g2.to(other), x)
    assert not bn_mod._sum_in_kernel(g1.to(other), g2, x)


@pytest.mark.gpu
def test_resnet50_bf16_junctions_bitwise(monkeypatch):
    """ResNet-50 bf16 at batch 64: parameter gradients of model(x) equal, bit for bit, those of the chain of blocks
    called on one tensor; a CUDA-graph replay of the step equals eager; 15 junctions are summed in the kernel and the
    last block's unused alias reaches backward as None."""
    from byteps_b200.torch.graph import GraphedStep

    prev = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        torch.manual_seed(0)
        model = resnet50().cuda().to(memory_format=torch.channels_last).to(torch.bfloat16)
        for mod in model.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.float()
        model.train()
        x = torch.rand(64, 3, 224, 224, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 1000, (64,), device="cuda")
        state = copy.deepcopy(model.state_dict())

        calls = []
        real = bn_mod._BatchNormActFn.backward

        def spy(ctx, *grads):
            if len(grads) == 2:
                calls.append((grads[0] is not None, grads[1] is not None))
            return real(ctx, *grads)

        monkeypatch.setattr(bn_mod._BatchNormActFn, "backward", staticmethod(spy))
        want = _param_grads(model, lambda t: _chained(model, t), x, y)
        assert calls == []
        model.load_state_dict(state)
        got = _param_grads(model, model, x, y)
        assert sorted(calls) == [(True, False)] + [(True, True)] * 15
        for i, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a, b), "parameter %d" % i

        def step():
            for p in model.parameters():
                p.grad = None
            F.cross_entropy(model(x).float(), y).backward()

        g = GraphedStep(step, warmup=2)
        model.load_state_dict(state)
        g()
        torch.cuda.synchronize()
        for i, (p, b) in enumerate(zip(model.parameters(), want)):
            assert torch.equal(p.grad, b), "graph replay, parameter %d" % i
    finally:
        torch.backends.cudnn.deterministic = prev
