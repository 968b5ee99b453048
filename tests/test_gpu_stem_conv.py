"""ResNet's stem convolution kernels (ops/stem_conv.py, kernels/stem_conv.cu).

Forward and weight gradient are checked against a float64 convolution with bounds from the rounding order, and
against cuDNN's own error on the same reference; the fallbacks are checked bit for bit against F.conv2d.  The ResNet-50
test trains the model with the kernels and with stock nn.Conv2d from the same seed and checks that the two runs track
each other: they are not bit-identical, since the convolution rounds in a different order.
"""
import json
import os
import re
import subprocess

import pytest
import torch
import torch.nn.functional as F

from _bounds import BF16, stored
from byteps_b200.ops.stem_conv import StemConv2d
from test_gpu_attn import _run_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUSED = "_StemConvFnBackward"
U24 = 2.0 ** -24
# N x H x W: the bench shape, odd and small images, 1 x 1 outputs, and output rows longer than one 128-pixel segment
SHAPES = [(64, 224, 224), (1, 7, 9), (1, 9, 7), (1, 223, 225), (1, 225, 223), (2, 1, 2), (1, 2, 1), (3, 300, 263)]


def _sid(s):
    return "x".join(map(str, s))


def _module(w_cl, seed=0, dtype=torch.bfloat16):
    torch.manual_seed(seed)
    m = StemConv2d(3, 64, 7, 2, 3, bias=False).cuda().to(dtype)
    if w_cl:
        m = m.to(memory_format=torch.channels_last)
    return m


def _image(n, h, w, seed=1, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, 3, h, w, device="cuda", generator=g).to(dtype).contiguous(memory_format=torch.channels_last)


def _grad_out(x, seed=2):
    n, _, h, w = x.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, 64, (h - 1) // 2 + 1, (w - 1) // 2 + 1, device="cuda", generator=g).to(x.dtype).contiguous(
        memory_format=torch.channels_last)


def _run(m, x, dy):
    """(y, dW) through the kernels; y is returned detached, so no autograd graph outlives the call"""
    y = m(x)
    assert type(y.grad_fn).__name__ == FUSED
    dw, = torch.autograd.grad(y, m.weight, dy)
    return y.detach(), dw


def _equal_bits(a, b):
    return a.shape == b.shape and a.stride() == b.stride() and torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---------------------------------------------------------------------------------------------- numerics
@pytest.mark.gpu
@pytest.mark.parametrize("w_cl", [True, False], ids=["wcl", "wcontig"])
@pytest.mark.parametrize("shape", SHAPES, ids=_sid)
def test_matches_float64(shape, w_cl):
    """y: fp32 accumulation of 147 products, rounded once to bf16.  dW: fp32 sums over the CTA's pixels then over the
    partials (depth at most N OH OW + partials), rounded once.  Each also within 2x cuDNN's error."""
    from byteps_b200 import _native

    m = _module(w_cl)
    x = _image(*shape)
    dy = _grad_out(x)
    y, dw = _run(m, x, dy)
    assert y.is_contiguous(memory_format=torch.channels_last) and dw.stride() == m.weight.stride()
    assert torch.isfinite(y).all() and torch.isfinite(dw).all()

    w64, x64, dy64 = m.weight.double(), x.double(), dy.double()
    ref_y = F.conv2d(x64, w64, stride=2, padding=3)
    abs_y = F.conv2d(x64.abs(), w64.abs(), stride=2, padding=3)
    ref_dw = torch.nn.grad.conv2d_weight(x64, w64.shape, dy64, stride=2, padding=3)
    abs_dw = torch.nn.grad.conv2d_weight(x64.abs(), w64.shape, dy64.abs(), stride=2, padding=3)
    n, _, h, w = x.shape
    depth = n * ((h - 1) // 2 + 1) * ((w - 1) // 2 + 1) + _native.cuda().stem_conv_wgrad_partials(n, h, w)
    err_y, err_dw = (y.double() - ref_y).abs(), (dw.double() - ref_dw).abs()
    assert (err_y <= stored(ref_y.abs(), 147 * U24 * abs_y, BF16)).all(), err_y.max()
    assert (err_dw <= stored(ref_dw.abs(), depth * U24 * abs_dw, BF16)).all(), err_dw.max()

    cy = F.conv2d(x, m.weight, stride=2, padding=3)
    cdw, = torch.autograd.grad(cy, m.weight, dy)
    tiny = 2.0 ** -133
    assert err_y.max() <= 2 * (cy.double() - ref_y).abs().max() + tiny
    assert err_dw.max() <= 2 * (cdw.double() - ref_dw).abs().max() + tiny


@pytest.mark.gpu
def test_misaligned_image_takes_the_kernels():
    """x is read with 2-byte loads, so a view at an odd element offset runs the kernels and gives the same bits."""
    m = _module(True)
    x = _image(2, 31, 29)
    dy = _grad_out(x)
    base = torch.empty(x.numel() + 1, dtype=x.dtype, device="cuda")
    xm = base[1:].view(2, 31, 29, 3).permute(0, 3, 1, 2)
    xm.copy_(x)
    assert xm.is_contiguous(memory_format=torch.channels_last) and xm.data_ptr() % 4 == 2
    ya, dwa = _run(m, x, dy)
    yb, dwb = _run(m, xm, dy)
    assert _equal_bits(ya, yb) and _equal_bits(dwa, dwb)


# ---------------------------------------------------------------------------------------------- determinism, graphs
@pytest.mark.gpu
def test_deterministic_and_graph_replay_equals_eager():
    m = _module(True)
    x = _image(64, 224, 224)
    dy = _grad_out(x)
    runs = [_run(m, x, dy) for _ in range(2)]
    assert _equal_bits(runs[0][0], runs[1][0]) and _equal_bits(runs[0][1], runs[1][1])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _run(m, x, dy)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y, dw = _run(m, x, dy)
    graph.replay()
    torch.cuda.synchronize()
    assert _equal_bits(y, runs[0][0]) and _equal_bits(dw, runs[0][1])


@pytest.mark.gpu
@pytest.mark.parametrize("w_cl", [True, False], ids=["wcl", "wcontig"])
@pytest.mark.parametrize("shape", [(2, 37, 41), (1, 300, 263)], ids=_sid)
def test_buffers_keep_their_bands(shape, w_cl):
    """y, dW and the workspace sit inside canary and NaN bands; y and dW are written in full on NaN-filled memory."""
    from byteps_b200 import _native

    cu = _native.cuda()
    m = _module(w_cl)
    x = _image(*shape)
    dy = _grad_out(x)
    ref_y, ref_dw = _run(m, x, dy)
    n, _, h, w = x.shape
    pad = 256
    st = torch.cuda.current_stream().cuda_stream
    for band in (1234.0, float("nan")):
        y_b = torch.full((ref_y.numel() + 2 * pad,), band, dtype=x.dtype, device="cuda")
        dw_b = torch.full((ref_dw.numel() + 2 * pad,), band, dtype=x.dtype, device="cuda")
        parts = cu.stem_conv_wgrad_partials(n, h, w)
        ws_b = torch.full((parts * 64 * 147 + 2 * pad,), band, dtype=torch.float32, device="cuda")
        y, dw = y_b[pad:pad + ref_y.numel()], dw_b[pad:pad + ref_dw.numel()]
        y.fill_(float("nan"))
        dw.fill_(float("nan"))
        cu.stem_conv_fwd(x.data_ptr(), m.weight.data_ptr(), w_cl, y.data_ptr(), 1, n, h, w, st)
        cu.stem_conv_wgrad(x.data_ptr(), dy.data_ptr(), ws_b[pad:].data_ptr(), parts, dw.data_ptr(), w_cl, 1, n, h,
                           w, st)
        torch.cuda.synchronize()
        for b in (y_b[:pad], y_b[pad + y.numel():], dw_b[:pad], dw_b[pad + dw.numel():], ws_b[:pad],
                  ws_b[pad + parts * 64 * 147:]):
            assert (b == band).all() if band == band else b.isnan().all()
        assert torch.equal(y.view(torch.int16), ref_y.permute(0, 2, 3, 1).reshape(-1).view(torch.int16))
        assert torch.equal(dw.view(torch.int16), ref_dw.permute(*((0, 2, 3, 1) if w_cl else (0, 1, 2, 3)))
                           .reshape(-1).view(torch.int16))


_LAUNCHES = """
import json
import torch
from torch.profiler import ProfilerActivity, profile
from byteps_b200.ops.stem_conv import StemConv2d

def launches(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

m = StemConv2d(3, 64, 7, 2, 3, bias=False).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
x = torch.randn(8, 3, 224, 224, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
dy = torch.randn(8, 64, 112, 112, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
torch.autograd.grad(m(x), m.weight, dy)
out = {}
fwd = launches(lambda: out.setdefault("y", m(x)))
bwd = launches(lambda: torch.autograd.grad(out["y"], m.weight, dy))
print(json.dumps({"fwd": fwd, "bwd": bwd}))
"""


@pytest.mark.gpu
def test_launch_count():
    """One launch forward, two for the weight gradient, and no other kernel, memset or copy."""
    names = json.loads(_run_py(_LAUNCHES).strip().splitlines()[-1])
    fwd, bwd = names["fwd"], names["bwd"]
    assert len(fwd) == 1 and "stem_conv_fwd_kernel" in fwd[0], fwd
    assert len(bwd) == 2 and "stem_conv_wgrad_kernel" in bwd[0] and "stem_conv_wgrad_reduce_kernel" in bwd[1], bwd


# ---------------------------------------------------------------------------------------------- fallbacks, arguments
FALLBACKS = ["fp32", "fp16", "nchw", "x_requires_grad", "kernel5", "stride1", "padding2", "bias", "out32",
             "w_strided"]


def _fallback(case, device):
    """(StemConv2d, nn.Conv2d with the same weights, x) for an input or module the kernels do not cover"""
    dt = {"fp32": torch.float32, "fp16": torch.float16}.get(case, torch.bfloat16)
    kw = dict(in_channels=3, out_channels=64, kernel_size=7, stride=2, padding=3, bias=False)
    kw.update({"kernel5": dict(kernel_size=5, padding=2), "stride1": dict(stride=1), "padding2": dict(padding=2),
               "bias": dict(bias=True), "out32": dict(out_channels=32)}.get(case, {}))
    torch.manual_seed(0)
    a = StemConv2d(**kw).to(device).to(dt)
    b = torch.nn.Conv2d(**kw).to(device).to(dt)
    b.load_state_dict(a.state_dict())
    if case != "nchw":
        a, b = a.to(memory_format=torch.channels_last), b.to(memory_format=torch.channels_last)
    if case == "w_strided":
        big = torch.randn(64, 3, 7, 14, device=device).to(dt)
        wv = big[..., ::2]
        a.weight, b.weight = torch.nn.Parameter(wv), torch.nn.Parameter(wv.clone())
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 33, 30, generator=g).to(dt).to(device)
    if case != "nchw":
        x = x.contiguous(memory_format=torch.channels_last)
    return a, b, x


def _check_fallback(case, device):
    a, b, x = _fallback(case, device)
    xa, xb = x.clone(), x.clone()
    if case == "x_requires_grad":
        xa.requires_grad_(True)
        xb.requires_grad_(True)
    ya, yb = a(xa), b(xb)
    assert type(ya.grad_fn).__name__ != FUSED
    assert torch.equal(ya, yb) and ya.stride() == yb.stride()
    dy = torch.randn(ya.shape, generator=torch.Generator().manual_seed(2)).to(ya.dtype).to(device)
    ya.backward(dy)
    yb.backward(dy)
    assert torch.equal(a.weight.grad, b.weight.grad) and a.weight.grad.stride() == b.weight.grad.stride()
    if case == "x_requires_grad":
        assert torch.equal(xa.grad, xb.grad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FALLBACKS)
def test_fallbacks_are_stock_cuda(case):
    _check_fallback(case, "cuda")


@pytest.mark.parametrize("case", ["bf16", "fp32", "nchw"])
def test_fallbacks_are_stock_cpu(case):
    _check_fallback(case, "cpu")


def test_same_parameters_and_init_as_conv2d():
    torch.manual_seed(3)
    a = StemConv2d(3, 64, 7, 2, 3, bias=False)
    torch.manual_seed(3)
    b = torch.nn.Conv2d(3, 64, 7, 2, 3, bias=False)
    assert isinstance(a, torch.nn.Conv2d)
    assert list(a.state_dict()) == list(b.state_dict()) and torch.equal(a.weight, b.weight)


@pytest.mark.gpu
def test_binding_rejects_bad_arguments():
    from byteps_b200 import _native

    cu = _native.cuda()
    buf = torch.zeros(1 << 20, dtype=torch.float32, device="cuda")
    b = buf.data_ptr()
    parts = cu.stem_conv_wgrad_partials(1, 16, 16)
    fwd = dict(x=b, w=b, y=b, dtype=1, N=1, H=16, W=16)
    for bad in [dict(dtype=0), dict(dtype=2), dict(N=0), dict(H=0), dict(W=-1), dict(H=2 ** 31), dict(x=0),
                dict(x=b + 1), dict(w=0), dict(w=b + 1), dict(y=0), dict(y=b + 8)]:
        a = dict(fwd, **bad)
        with pytest.raises(ValueError):
            cu.stem_conv_fwd(a["x"], a["w"], True, a["y"], a["dtype"], a["N"], a["H"], a["W"], 0)
    wg = dict(x=b, dy=b, ws=b, parts=parts, dw=b, dtype=1, N=1, H=16, W=16)
    for bad in [dict(dtype=0), dict(N=0), dict(W=0), dict(x=b + 1), dict(dy=b + 2), dict(ws=0), dict(ws=b + 4),
                dict(dw=0), dict(dw=b + 1), dict(parts=0), dict(parts=parts + 1)]:
        a = dict(wg, **bad)
        with pytest.raises(ValueError):
            cu.stem_conv_wgrad(a["x"], a["dy"], a["ws"], a["parts"], a["dw"], True, a["dtype"], a["N"], a["H"],
                               a["W"], 0)


# ---------------------------------------------------------------------------------------------- build
def test_stem_kernels_compile_without_spills(tmp_path):
    from byteps_b200 import _build

    nvcc = _build._nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "byteps_b200", "csrc", "kernels", "stem_conv.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + _build.ARCH_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                                         str(tmp_path / "stem_conv.o")],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    found = 0
    for block in r.stderr.split("Compiling entry function '")[1:]:
        if not re.match(r"_ZN\S*stem_conv_(fwd|wgrad|wgrad_reduce)_kernel", block):
            continue
        found += 1
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block[:400]
    assert found == 3, found


# ---------------------------------------------------------------------------------------------- ResNet-50
_RESNET_STEPS = """
import json
import torch
import torch.nn.functional as F
import byteps_b200.torch as bps
from byteps_b200.models import resnet50
from byteps_b200.torch.graph import GraphedStep
STOCK, STEPS = %r, %r
bps.init()
torch.manual_seed(0)
model = resnet50()
if STOCK:
    conv = torch.nn.Conv2d(3, 64, 7, 2, 3, bias=False)
    conv.load_state_dict(model.conv1.state_dict())
    model.conv1 = conv
model = model.cuda().to(memory_format=torch.channels_last).to(torch.bfloat16)
for m in model.modules():
    if isinstance(m, torch.nn.BatchNorm2d):
        m.float()
opt = bps.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.02, momentum=0.9),
                               named_parameters=model.named_parameters(), fused_update=True)
g = torch.Generator().manual_seed(1)
x = torch.rand(16, 3, 224, 224, generator=g).to(torch.bfloat16).cuda().contiguous(memory_format=torch.channels_last)
y = torch.randint(0, 1000, (16,), generator=g).cuda()
losses = []

def step():
    opt.zero_grad()
    loss = F.cross_entropy(model(x).float(), y)
    loss.backward()
    opt.step()
    return loss

stepper = GraphedStep(step, warmup=3, pre_replay=opt.refresh_hparams, device=torch.device("cuda", 0))
for _ in range(STEPS):
    losses.append(float(stepper()))
sample = {n: p.detach().float().flatten()[:256].tolist() for n, p in model.named_parameters()
          if n in ("conv1.weight", "layer1.0.conv1.weight", "fc.bias")}
print(json.dumps({"losses": losses, "sample": sample, "conv1": [type(model.conv1).__name__]}))
bps.shutdown()
"""


@pytest.mark.gpu
def test_resnet50_tracks_stock_conv():
    """60 graphed bf16 steps on one batch: the losses stay within 5 % of each other (plus 0.02) and sampled
    parameters within 5 % of their norm.  The two runs are not bit-identical: the stem rounds in another order."""
    steps = 60
    runs = [json.loads(_run_py(_RESNET_STEPS % (stock, steps)).strip().splitlines()[-1]) for stock in (False, True)]
    kern, stock = runs
    assert kern["conv1"] == ["StemConv2d"] and stock["conv1"] == ["Conv2d"]
    la, lb = torch.tensor(kern["losses"]), torch.tensor(stock["losses"])
    assert la.numel() == steps and torch.isfinite(la).all() and la[-1] < la[0]
    assert ((la - lb).abs() <= 0.05 * lb.abs() + 0.02).all(), (la - lb).abs().max()
    for name, va in kern["sample"].items():
        a, b = torch.tensor(va), torch.tensor(stock["sample"][name])
        assert (a - b).norm() <= 0.05 * b.norm() + 1e-6, (name, (a - b).norm(), b.norm())
