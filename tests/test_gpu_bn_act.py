"""Fused batch norm + residual add + ReLU (ops/bn_act.py, kernels/bn_act.cu).

GPU tests compare the fused kernels with a float64 reference.  The bounds follow the kernels' rounding steps:

* every fp32 quantity the kernels form (mean, M2, sums over rows, the affine maps) is a chain of at most a few
  hundred roundings (a thread's rows, the chunk merges, two fixed trees), so its absolute error is below
  C_ACC * u32 times the sum of the magnitudes that enter it (u32 = 2^-24, C_ACC = 256);
* the mean's error enters every centred value x - mean, so those magnitudes include |mean| * invstd;
* the output is then rounded once to its dtype: half an ulp, u_t * |value| with u_t = 2^-8 (bf16), 2^-11 (fp16),
  2^-24 (fp32), or half the subnormal spacing near 0.

d(residual) = dy * mask is exact.  The reference backward uses the kernel's own ReLU mask (y > 0), so an element
whose pre-activation is within rounding of 0 cannot flip the comparison; the forward bound covers such elements.

CPU tests (no marker) check that the models keep the stock BatchNorm2d state_dict and compute the stock
composition on the path every non-CUDA input takes.
"""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from byteps_b200.models import resnet18, resnet50
from byteps_b200.models.resnet import BasicBlock, Bottleneck
from byteps_b200.ops.bn_act import BatchNormAct2d

U32 = 2.0 ** -24
C_ACC = 256
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
# half the spacing of the subnormals: the absolute rounding error near 0
TINY = {torch.bfloat16: 2.0 ** -134, torch.float16: 2.0 ** -25, torch.float32: 2.0 ** -150}

# the 12 distinct (C, H, W) of ResNet-50's batch norms at 224x224
RESNET50_BN_SHAPES = [(64, 112, 112), (64, 56, 56), (256, 56, 56), (128, 56, 56), (128, 28, 28), (512, 28, 28),
                      (256, 28, 28), (256, 14, 14), (1024, 14, 14), (512, 14, 14), (512, 7, 7), (2048, 7, 7)]
ACTS = [("none", None, False), ("relu", "relu", False), ("relu_res", "relu", True)]
DTYPES = [torch.bfloat16, torch.float16, torch.float32]


def _dt_id(d):
    return str(d).replace("torch.", "")


def _nhwc(t):
    return t.contiguous(memory_format=torch.channels_last)


def _make(n, c, h, w, dtype, act, residual, mean_shift=0.0, zero_gamma=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    scale = torch.rand(c, device=dev, generator=g, dtype=torch.float64) * 2 + 0.5
    loc = torch.randn(c, device=dev, generator=g, dtype=torch.float64) + mean_shift * scale
    x = _nhwc((torch.randn(n, c, h, w, device=dev, generator=g, dtype=torch.float64) * scale.view(1, -1, 1, 1)
               + loc.view(1, -1, 1, 1)).to(dtype))
    r = _nhwc(torch.randn(n, c, h, w, device=dev, generator=g, dtype=torch.float64).to(dtype)) if residual else None
    dy = _nhwc(torch.randn(n, c, h, w, device=dev, generator=g, dtype=torch.float64).to(dtype))
    bn = BatchNormAct2d(c, act=act).to(dev)
    with torch.no_grad():
        bn.weight.copy_(torch.randn(c, device=dev, generator=g))
        bn.bias.copy_(torch.randn(c, device=dev, generator=g) * 0.5)
        if zero_gamma:
            bn.weight[c // 2] = 0.0
        bn.running_mean.copy_(torch.randn(c, device=dev, generator=g))
        bn.running_var.copy_(torch.rand(c, device=dev, generator=g) + 0.5)
    bn.train()
    return bn, x, r, dy


def _run(bn, x, r, dy):
    xg = x.detach().clone().requires_grad_(True)
    rg = r.detach().clone().requires_grad_(True) if r is not None else None
    y = bn(xg, rg)
    assert type(y.grad_fn).__name__ == "_BatchNormActFnBackward", "fused path not taken"
    _, _, mean, invstd, _ = y.grad_fn.saved_tensors
    y.backward(dy)
    return dict(y=y.detach(), dx=xg.grad, dres=None if r is None else rg.grad, dw=bn.weight.grad.clone(),
                db=bn.bias.grad.clone(), mean=mean.clone(), invstd=invstd.clone())


def _check_bn_act(n, c, h, w, dtype, act, residual, **kw):
    bn, x, r, dy = _make(n, c, h, w, dtype, act, residual, **kw)
    rm0, rv0 = bn.running_mean.clone().double(), bn.running_var.clone().double()
    out = _run(bn, x, r, dy)
    ut = UNIT[dtype]
    m = n * h * w
    dims = (0, 2, 3)
    v = lambda t: t.view(1, -1, 1, 1)  # noqa: E731

    # ---- forward reference
    xd = x.double()
    wd, bd = bn.weight.detach().double(), bn.bias.detach().double()
    mu = xd.mean(dims)
    var = xd.var(dims, unbiased=False)
    inv = 1.0 / torch.sqrt(var + bn.eps)
    xhat = (xd - v(mu)) * v(inv)
    z = xhat * v(wd) + v(bd)
    if r is not None:
        z = z + r.double()
    y_ref = torch.relu(z) if act == "relu" else z
    shift = (mu.abs() * inv + 1.0)                         # |mean| / std + 1: how the mean's error is amplified
    mag = (xhat.abs() * v(shift) + v(shift)) * v(wd.abs()) + v(bd.abs())
    if r is not None:
        mag = mag + r.double().abs()
    tol_y = C_ACC * U32 * mag + ut * (y_ref.abs() + C_ACC * U32 * mag) + TINY[dtype]
    err_y = (out["y"].double() - y_ref).abs()
    assert (err_y <= tol_y).all(), "y: worst excess %g" % (err_y - tol_y).max().item()

    # saved statistics, running statistics, num_batches_tracked
    assert torch.all((out["mean"].double() - mu).abs() <= C_ACC * U32 * (mu.abs() + var.sqrt()))
    assert torch.all((out["invstd"].double() - inv).abs() <= C_ACC * U32 * inv * shift)
    mom = bn.momentum
    rm_ref = (1 - mom) * rm0 + mom * mu
    rv_ref = (1 - mom) * rv0 + mom * var * m / (m - 1)
    assert torch.all((bn.running_mean.double() - rm_ref).abs() <= C_ACC * U32 * (rm0.abs() + mu.abs() + var.sqrt()))
    assert torch.all((bn.running_var.double() - rv_ref).abs() <= C_ACC * U32 * (rv0.abs() + var * shift))
    assert int(bn.num_batches_tracked) == 1

    # ---- backward reference, with the kernel's mask
    gd = dy.double()
    if act == "relu":
        gd = gd * (out["y"] > 0).double()
    if r is not None:
        assert torch.equal(out["dres"], gd.to(dtype)), "d(residual) must be dy * mask exactly"
    db_ref = gd.sum(dims)
    dw_ref = (gd * xhat).sum(dims)
    sg = gd.abs().sum(dims)
    sgx = (gd * xhat).abs().sum(dims)
    tol_db = C_ACC * U32 * sg
    tol_dw = C_ACC * U32 * (sgx + shift * sg + dw_ref.abs())
    assert torch.all((out["db"].double() - db_ref).abs() <= tol_db), "dbias"
    assert torch.all((out["dw"].double() - dw_ref).abs() <= tol_dw), "dweight"
    a = wd * inv
    dx_ref = v(a) * (gd - v(db_ref / m) - xhat * v(dw_ref / m))
    mag_dx = v(a.abs()) * (gd.abs() + (xhat.abs() * v(shift) + v(shift)) * v((sgx + shift * sg + dw_ref.abs()) / m)
                           + v(sg / m))
    tol_dx = C_ACC * U32 * mag_dx * (1 + ut) + ut * dx_ref.abs() + TINY[dtype]
    err_dx = (out["dx"].double() - dx_ref).abs()
    assert (err_dx <= tol_dx).all(), "dx: worst excess %g" % (err_dx - tol_dx).max().item()
    return bn, x, r, dy, out


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("act_id,act,residual", ACTS, ids=[a[0] for a in ACTS])
@pytest.mark.parametrize("chw", RESNET50_BN_SHAPES, ids=lambda s: "%dx%dx%d" % s)
def test_bn_act_resnet50_shapes(chw, act_id, act, residual, dtype):
    c, h, w = chw
    _check_bn_act(2, c, h, w, dtype, act, residual)


@pytest.mark.gpu
@pytest.mark.parametrize("act_id,act,residual", ACTS, ids=[a[0] for a in ACTS])
def test_bn_act_stem_batch64(act_id, act, residual):
    """The 64x64x112x112 stem at batch 64: M = 802 816 rows, the largest reduction of the model."""
    _check_bn_act(64, 64, 112, 112, torch.bfloat16, act, residual)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("case,shape,kw", [
    ("c8", (4, 8, 9, 9), {}),                               # one 8-channel unit per row
    ("odd_rows", (3, 24, 5, 7), {}),                        # M = 105: no block divides it; C = 24: partial group
    ("c40_odd_rows", (1, 40, 37, 3), {}),
    ("mean_100_std", (2, 64, 28, 28), dict(mean_shift=100.0)),
    ("zero_gamma", (2, 128, 14, 14), dict(zero_gamma=True)),
], ids=lambda p: p if isinstance(p, str) else None)
def test_bn_act_edge_cases(case, shape, kw, dtype):
    for act_id, act, residual in ACTS:
        _check_bn_act(*shape, dtype, act, residual, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_bn_act_deterministic_and_graphed(dtype):
    from byteps_b200.torch.graph import GraphedStep

    bn, x, r, dy = _make(8, 256, 28, 28, dtype, "relu", True, seed=3)
    state = copy.deepcopy(bn.state_dict())
    a = _run(bn, x, r, dy)
    bn.load_state_dict(state)
    bn.weight.grad = None
    bn.bias.grad = None
    b = _run(bn, x, r, dy)
    for k in a:
        assert torch.equal(a[k], b[k]), k

    # the same step captured in a CUDA graph and replayed equals eager, bit for bit
    xs, rs = x.detach().clone().requires_grad_(True), r.detach().clone().requires_grad_(True)
    outs = {}

    def step():
        xs.grad = None
        rs.grad = None
        bn.weight.grad = None
        bn.bias.grad = None
        y = bn(xs, rs)
        y.backward(dy)
        outs.update(y=y.detach(), dx=xs.grad, dres=rs.grad, dw=bn.weight.grad, db=bn.bias.grad)
        return y

    g = GraphedStep(step, warmup=2)
    bn.load_state_dict(state)
    g()
    torch.cuda.synchronize()
    for k in ("y", "dx", "dres", "dw", "db"):
        assert torch.equal(outs[k], a[k]), k
    assert torch.equal(bn.running_mean, b_running_mean(state, bn, x, r, dy)), "running_mean"


def b_running_mean(state, bn, x, r, dy):
    """running_mean after one eager step from `state`."""
    ref = copy.deepcopy(bn)
    ref.load_state_dict(state)
    _run(ref, x, r, dy)
    return ref.running_mean


# ---------------------------------------------------------------------------------------------- model level
def _stock_bn_forward(model):
    """Route every BatchNormAct2d of `model` through the stock F.batch_norm / add / relu composition."""
    for mod in model.modules():
        if isinstance(mod, BatchNormAct2d):
            mod._fusable = lambda *a, **k: False
    return model


@pytest.mark.gpu
def test_resnet50_bf16_step_matches_stock():
    """One bf16 training step of ResNet-50 at batch 4, fused against the stock composition with the same weights.
    Both are compared with the stock model in fp32: the fused step's loss and every parameter's gradient must be
    as close to it as bf16 allows - within twice the stock bf16 step's error, or 2 % relative L2, whichever is
    larger (the fused kernels round once where the stock passes round two or three times)."""
    torch.manual_seed(0)
    base = resnet50().cuda().to(memory_format=torch.channels_last)
    x = torch.rand(4, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (4,), device="cuda")

    def grads(model, dtype):
        model = model.to(dtype)
        for mod in model.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.float()
        model.train()
        loss = F.cross_entropy(model(x.to(dtype)).float(), y)
        loss.backward()
        return loss.item(), [p.grad.double() for p in model.parameters()]

    l_ref, g_ref = grads(_stock_bn_forward(copy.deepcopy(base)), torch.float32)
    l_stock, g_stock = grads(_stock_bn_forward(copy.deepcopy(base)), torch.bfloat16)
    l_fused, g_fused = grads(copy.deepcopy(base), torch.bfloat16)
    assert abs(l_fused - l_ref) <= max(2 * abs(l_stock - l_ref), 1e-2 * abs(l_ref)), (l_fused, l_stock, l_ref)
    for i, (gf, gs, gr) in enumerate(zip(g_fused, g_stock, g_ref)):
        nr = gr.norm().item() + 1e-30
        ef, es = (gf - gr).norm().item() / nr, (gs - gr).norm().item() / nr
        assert ef <= max(2 * es, 0.02), "parameter %d: fused %.3g stock %.3g" % (i, ef, es)


def _stock_copy(model):
    """The same model with every BatchNormAct2d replaced by a plain nn.BatchNorm2d."""
    model = copy.deepcopy(model)
    for parent in list(model.modules()):
        for name, child in list(parent.named_children()):
            if isinstance(child, BatchNormAct2d):
                setattr(parent, name, nn.BatchNorm2d(child.num_features, child.eps, child.momentum))
    return model


def _stock_forward(model, x):
    """The ResNet forward as composed before the fused module: BN, then separate (in-place) ReLU and add."""
    bn = lambda m, t: nn.BatchNorm2d.forward(m, t)  # noqa: E731

    def seq(s, t):
        return bn(s[1], s[0](t))

    def block(b, t):
        idt = t if b.downsample is None else seq(b.downsample, t)
        out = F.relu(bn(b.bn1, b.conv1(t)), inplace=True)
        if isinstance(b, Bottleneck):
            out = F.relu(bn(b.bn2, b.conv2(out)), inplace=True)
            out = bn(b.bn3, b.conv3(out))
        else:
            out = bn(b.bn2, b.conv2(out))
        return F.relu(out + idt, inplace=True)

    t = model.maxpool(F.relu(bn(model.bn1, model.conv1(x)), inplace=True))
    for layer in (model.layer1, model.layer2, model.layer3, model.layer4):
        for b in layer:
            assert isinstance(b, (BasicBlock, Bottleneck))
            t = block(b, t)
    return model.fc(torch.flatten(model.avgpool(t), 1))


@pytest.mark.parametrize("ctor", [resnet18, resnet50], ids=["resnet18", "resnet50"])
def test_resnet_state_dict_is_stock(ctor):
    torch.manual_seed(0)
    model = ctor()
    stock = _stock_copy(model)
    ours, theirs = model.state_dict(), stock.state_dict()
    assert list(ours) == list(theirs)
    assert all(ours[k].shape == theirs[k].shape and ours[k].dtype == theirs[k].dtype for k in ours)
    assert [n for n, _ in model.named_parameters()] == [n for n, _ in stock.named_parameters()]
    # a stock state_dict (perturbed so that every entry differs) loads strictly
    sd = {k: (v + 1 if v.is_floating_point() else v + 3) for k, v in theirs.items()}
    model.load_state_dict(sd, strict=True)
    for k, v in model.state_dict().items():
        assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize("ctor", [resnet18, resnet50], ids=["resnet18", "resnet50"])
def test_resnet_cpu_forward_is_stock(ctor):
    torch.manual_seed(0)
    model = ctor()
    twin = copy.deepcopy(model)
    x = torch.randn(2, 3, 64, 64)
    model.train()
    twin.train()
    y = model(x)
    y_ref = _stock_forward(twin, x)
    assert torch.equal(y, y_ref)
    for (k, a), (_, b) in zip(model.state_dict().items(), twin.state_dict().items()):
        assert torch.equal(a, b), k       # running statistics and num_batches_tracked too
    model.eval()
    twin.eval()
    with torch.no_grad():
        assert torch.equal(model(x), _stock_forward(twin, x))
