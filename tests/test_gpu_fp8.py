"""FP8 linear layers with delayed scaling (ops/fp8.py, kernels/fp8.cu).

GPU tests:

* casts are compared bit for bit with ``clamp(x.float() * s, -fmax, fmax).to(fp8)`` (torch's own cast turns values
  above fmax into NaN, hence the clamp), and the recorded amax, the next scale and the per-call inverse scale with the
  same fp32 expressions computed by torch;
* a scripted sequence of calls follows a Python model of the delayed-scaling rule, including the wrap of the
  16-entry history, saturation, and inf / NaN calls that must poison that call's outputs and leave the state alone;
* ``Fp8Linear`` is compared with float64 products of the dequantised FP8 operands (rebuilt with the reference cast).
  The bound is half a unit of the output dtype on |ref| plus (K 2^-24 + 2^-11) sum |a||b|: K fp32 additions, and the
  Hopper tensor cores add each k-block of FP8 products at reduced precision before the fp32 accumulation;
* determinism, CUDA-graph replay, and bert_tiny with ``fp8_linear=True`` graphed, with the fused norm and loss and
  a dynamic loss scale, and trained next to the bf16 model on a learnable task.

CPU tests check that every non-CUDA input is exactly ``F.linear``, that the model's parameters and state_dict do not
change, and that ``model.to(dtype)`` leaves the scaling state alone.
"""
import copy
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from byteps_b200.models import bert_tiny
from byteps_b200.ops import fp8
from byteps_b200.ops.fp8 import DY, E4M3, E5M2, FP8_DTYPES, FP8_MAX, W, X, Fp8Linear

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUSED = "_Fp8LinearFnBackward"
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
MIN_SUB = {E4M3: 2.0 ** -9, E5M2: 2.0 ** -16}
LAYOUTS = {"rows": fp8.ROWS, "cols": fp8.COLS, "both": fp8.BOTH}


def _dt_id(d):
    return str(d).replace("torch.", "")


def _f32(v):
    return torch.tensor(v, dtype=torch.float32)


def ref_cast(x, s, fmt):
    fmax = FP8_MAX[fmt]
    return torch.clamp(x.float() * s, -fmax, fmax).to(FP8_DTYPES[fmt])


def _bits(t):
    return t.view(torch.uint8)


def _fresh_state(scale):
    st = torch.zeros(fp8.STATE_WORDS, dtype=torch.int32, device="cuda")
    st.view(torch.float32)[fp8.HISTORY] = scale
    return st


def _values(m, k, dtype, fmt, s, seed):
    """normal values with zeros, values that saturate at scale s and values near the FP8 subnormals"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(m, k, device="cuda", generator=g) * 2
    sel = torch.randint(0, 8, (m, k), device="cuda", generator=g)
    x = torch.where(sel == 0, torch.zeros_like(x), x)
    x = torch.where(sel == 1, x * (FP8_MAX[fmt] / s), x)                 # well past the saturation point
    x = torch.where(sel == 2, x * (4 * MIN_SUB[fmt] / s), x)             # lands on FP8 subnormals
    return x.to(dtype)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=_dt_id)
@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("m,k", [(16, 16), (48, 208), (1008, 272), (8192, 4096), (2064, 3072)])
def test_cast_is_bit_exact(m, k, fmt, dtype, layout):
    fmax = FP8_MAX[fmt]
    s = _f32(fmax / 3.0)
    x = _values(m, k, dtype, fmt, s.item(), seed=m + k + fmt)
    st = _fresh_state(s)
    rows, cols, inv, db = fp8.cast(x, st, fmt, LAYOUTS[layout])
    ref = ref_cast(x, s, fmt)
    assert (rows is None) == (layout == "cols") and (cols is None) == (layout == "rows") and db is None
    if rows is not None:
        assert torch.equal(_bits(rows), _bits(ref))
    if cols is not None:
        assert torch.equal(_bits(cols), _bits(ref.t().contiguous()))
    amax = x.float().abs().max().cpu()
    assert torch.equal(inv.cpu(), _f32(1.0) / s)
    hist = st.view(torch.float32)[: fp8.HISTORY].cpu()
    assert torch.equal(hist[0], amax) and not hist[1:].any()
    assert st[fp8.HISTORY + 1].item() == 1
    assert torch.equal(st.view(torch.float32)[fp8.HISTORY].cpu(), _f32(fmax) / torch.maximum(amax, _f32(1e-12)))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=_dt_id)
@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=["e4m3", "e5m2"])
def test_seed_and_zero_tensor(fmt, dtype):
    """fp8_amax seeds the history and the scale from the tensor; an all-zero tensor needs no special case"""
    fmax = FP8_MAX[fmt]
    x = (torch.randn(96, 160, device="cuda") * 5).to(dtype)
    st = _fresh_state(0.0)
    fp8.seed(x, st, fmt)
    amax = x.float().abs().max().cpu()
    s = _f32(fmax) / torch.maximum(amax, _f32(1e-12))
    assert torch.equal(st.view(torch.float32)[0].cpu(), amax) and st[fp8.HISTORY + 1].item() == 0
    assert torch.equal(st.view(torch.float32)[fp8.HISTORY].cpu(), s)
    z = torch.zeros(32, 64, dtype=dtype, device="cuda")
    fp8.seed(z, st, fmt)
    s0 = _f32(fmax) / _f32(1e-12)
    assert torch.equal(st.view(torch.float32)[fp8.HISTORY].cpu(), s0)
    rows, _, inv, _ = fp8.cast(z, st, fmt, fp8.ROWS)
    assert not _bits(rows).any() and torch.equal(inv.cpu(), _f32(1.0) / s0)


@pytest.mark.gpu
def test_cast_more_than_2_31_elements():
    m, k = 2 ** 31 // 4096 + 16, 4096
    assert m * k > 2 ** 31
    s = _f32(448.0 / 3.0)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(m, k, device="cuda", generator=g, dtype=torch.bfloat16)
    st = _fresh_state(s)
    rows, cols, inv, _ = fp8.cast(x, st, E4M3, fp8.BOTH)
    for r0 in list(range(0, m, 65536)) + [m - 4096]:
        r1 = min(m, r0 + 4096)
        ref = _bits(ref_cast(x[r0:r1], s, E4M3))
        assert torch.equal(_bits(rows[r0:r1]), ref), r0
        assert torch.equal(_bits(cols[:, r0:r1]), ref.t()), r0
    del rows, cols
    assert torch.equal(st.view(torch.float32)[0].cpu(), x.abs().max().float().cpu())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=_dt_id)
@pytest.mark.parametrize("m,n", [(16, 16), (8192, 1024), (8192, 4096), (2000 // 16 * 16, 3072)])
def test_bias_gradient(m, n, dtype):
    g = torch.Generator(device="cuda").manual_seed(n)
    dy = (torch.randn(m, n, device="cuda", generator=g) + 0.25).to(dtype)
    outs = []
    for _ in range(2):
        st = _fresh_state(57344.0 / 4)
        outs.append(fp8.cast(dy, st, E5M2, fp8.BOTH, dtype)[3])
    assert torch.equal(outs[0], outs[1]), "bias gradient must be bitwise identical run to run"
    ref = dy.double().sum(0)
    tol = m * 2.0 ** -24 * dy.double().abs().sum(0) + UNIT[dtype] * ref.abs()
    assert ((outs[0].double() - ref).abs() <= tol).all()


class _StateModel:
    """Python model of the delayed-scaling rule of one tensor, in float32."""

    def __init__(self, fmax):
        self.fmax, self.hist, self.count, self.scale = np.float32(fmax), [np.float32(0)] * 16, 0, None

    def _next(self):
        return np.float32(self.fmax / np.maximum(np.float32(max(self.hist)), np.float32(1e-12)))

    def seed(self, a):
        ok = np.isfinite(a)
        self.hist = [np.float32(a if ok else 0)] + [np.float32(0)] * 15
        self.count = 0
        self.scale = np.float32(self.fmax / np.maximum(np.float32(a), np.float32(1e-12))) if ok else np.float32("nan")

    def call(self, a):
        s = self.scale
        if not np.isfinite(a):
            return s, np.float32("nan")
        inv = np.float32(np.float32(1) / s)
        self.hist[self.count % 16] = np.float32(a)
        self.count += 1
        self.scale = self._next()
        return s, inv


def _with_amax(shape, a, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(*shape, device="cuda", generator=g) * 2 - 1
    x = (x * 0.9 * (a if math.isfinite(a) else 1.0)).to(torch.bfloat16)
    x.view(-1)[7] = a
    return x


def _dq_matmul(a8, inv_a, b8, inv_b):
    """float64 a8 @ b8^T dequantised, and sum |a||b| of the same product"""
    ad, bd = a8.double() * inv_a.double(), b8.double() * inv_b.double()
    return ad @ bd.t(), ad.abs() @ bd.abs().t()


def _check_gemm(out, ref, absprod, k, dtype):
    tol = UNIT[dtype] * ref.abs() + (k * 2.0 ** -24 + 2.0 ** -11) * absprod + 2.0 ** -120
    err = (out.double() - ref).abs()
    assert (err <= tol).all(), "worst excess %g" % (err - tol).max().item()


@pytest.mark.gpu
def test_delayed_scaling_sequence():
    """x amaxes: a seeded first call, 18 more (the history wraps), growth that saturates, inf, NaN, then finite
    calls.  Each call's inverse scales, the state and y / dx / dW follow the model."""
    torch.manual_seed(0)
    m, k, n = 32, 64, 48
    lin = Fp8Linear(k, n).cuda().to(torch.bfloat16)
    amaxes = [1.0, 2.0, 0.5, 3.0] + [0.25 * (i + 1) for i in range(15)] + [40.0, float("inf"), float("nan"), 1.5, 0.75]
    dy_inf_at = 22              # an inf in dy on this call (x finite)
    mx, mw, mdy = _StateModel(448.0), _StateModel(448.0), _StateModel(57344.0)
    g = torch.Generator(device="cuda").manual_seed(5)
    dy0 = (torch.rand(m, n, device="cuda", generator=g) - 0.5).to(torch.bfloat16)
    w_a = lin.weight.detach().float().abs().max().item()
    dy_a = dy0.float().abs().max().item()
    for i, a in enumerate(amaxes):
        x = _with_amax((m, k), a, seed=i).requires_grad_(True)
        dy = dy0.clone()
        if i == dy_inf_at:
            dy[3, 4] = float("inf")
        if i == 0:
            mx.seed(np.float32(a)), mw.seed(np.float32(w_a))
        sx, ix = mx.call(np.float32(a))
        sw, iw = mw.call(np.float32(w_a))
        y = lin(x)
        assert type(y.grad_fn).__name__ == FUSED
        xt8, wt8, inv_x, inv_w = y.grad_fn.saved_tensors
        assert np.array_equal(inv_x.cpu().numpy(), ix, equal_nan=True), (i, inv_x.item(), ix)
        assert np.array_equal(inv_w.cpu().numpy(), iw, equal_nan=True), i
        if i == 0:
            mdy.seed(np.float32(dy_a))
        sdy, idy = mdy.call(np.float32(float("inf") if i == dy_inf_at else dy_a))
        y.backward(dy)
        st = lin.scaling_state(x.device)
        for row, mod in ((X, mx), (W, mw), (DY, mdy)):
            assert np.array_equal(st.history(row).cpu().numpy(), np.array(mod.hist, dtype=np.float32)), (i, row)
            assert st.count(row).item() == mod.count, (i, row)
            assert np.array_equal(st.scale(row).cpu().numpy(), mod.scale, equal_nan=True), (i, row)
        finite_x, finite_dy = math.isfinite(a), i != dy_inf_at
        assert bool(y.isfinite().all()) == finite_x, i
        assert bool(x.grad.isfinite().all()) == finite_dy, i
        assert bool(lin.weight.grad.isfinite().all()) == (finite_x and finite_dy), i
        if finite_x and finite_dy:
            x8 = ref_cast(x.detach(), _f32(sx), E4M3)
            w8 = ref_cast(lin.weight.detach(), _f32(sw), E4M3)
            ref, ab = _dq_matmul(x8, inv_x, w8, inv_w)
            ref = ref + lin.bias.detach().double()
            _check_gemm(y.detach(), ref, ab, k, torch.bfloat16)
            if a == 40.0:
                assert (x8.float().abs() == 448).sum() > 1, "growth past the history's amax saturates"
        lin.weight.grad = lin.bias.grad = None


def _linear_case(shape, n, bias, dtype, seed):
    torch.manual_seed(seed)
    k = shape[-1]
    lin = Fp8Linear(k, n, bias=bias).cuda().to(dtype)
    if bias:
        nn.init.normal_(lin.bias, std=0.5)
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(*shape, device="cuda", generator=g).to(dtype).requires_grad_(True)
    dy = torch.randn(*shape[:-1], n, device="cuda", generator=g).to(dtype)
    return lin, x, dy


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=_dt_id)
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("shape,n", [((8192, 1024), 3072), ((8192, 1024), 1024), ((8192, 1024), 4096),
                                     ((8192, 4096), 1024), ((16, 16), 16), ((3, 48, 80), 32), ((2, 8, 16), 64)])
def test_fp8_linear_matches_float64(shape, n, bias, dtype):
    lin, x, dy = _linear_case(shape, n, bias, dtype, seed=n + len(shape))
    k = shape[-1]
    y = lin(x)
    assert type(y.grad_fn).__name__ == FUSED and y.shape == (*shape[:-1], n) and y.dtype == dtype
    xt8, wt8, inv_x, inv_w = y.grad_fn.saved_tensors
    y.backward(dy)
    st = lin.scaling_state(x.device)
    x2, dy2 = x.detach().reshape(-1, k), dy.reshape(-1, n)
    # first call: every scale is seeded from the tensor itself
    sx, sw, sdy = (_f32(fmax) / torch.maximum(t.float().abs().max().cpu(), _f32(1e-12))
                   for t, fmax in ((x2, 448.0), (lin.weight.detach(), 448.0), (dy2, 57344.0)))
    assert torch.equal(inv_x.cpu(), 1 / sx) and torch.equal(inv_w.cpu(), 1 / sw)
    x8, w8, dy8 = ref_cast(x2, sx, E4M3), ref_cast(lin.weight.detach(), sw, E4M3), ref_cast(dy2, sdy, E5M2)
    assert torch.equal(_bits(xt8), _bits(x8.t().contiguous())) and torch.equal(_bits(wt8), _bits(w8.t().contiguous()))
    inv_dy = 1 / sdy
    ref, ab = _dq_matmul(x8, inv_x, w8, inv_w)
    if bias:
        ref = ref + lin.bias.detach().double()
    _check_gemm(y.detach().reshape(-1, n), ref, ab, k, dtype)
    ref, ab = _dq_matmul(dy8, inv_dy, w8.t(), inv_w)
    _check_gemm(x.grad.reshape(-1, k), ref, ab, n, dtype)
    ref, ab = _dq_matmul(dy8.t(), inv_dy, x8.t(), inv_x)
    _check_gemm(lin.weight.grad, ref, ab, x2.shape[0], dtype)
    if bias:
        rb = dy2.double().sum(0)
        tol = x2.shape[0] * 2.0 ** -24 * dy2.double().abs().sum(0) + UNIT[dtype] * rb.abs()
        assert ((lin.bias.grad.double() - rb).abs() <= tol).all()
    else:
        assert lin.bias is None
    assert st.count(X).item() == 1 and st.count(DY).item() == 1
    # sanity against the bf16 / fp16 nn.Linear: relative L2 error within 12 %
    ref_lin = nn.Linear(k, n, bias=bias).cuda().to(dtype)
    ref_lin.load_state_dict(lin.state_dict())
    xr = x.detach().clone().requires_grad_(True)
    yr = ref_lin(xr)
    yr.backward(dy)
    for a, b in ((y, yr), (x.grad, xr.grad), (lin.weight.grad, ref_lin.weight.grad)):
        a, b = a.detach().double(), b.detach().double()
        assert (a - b).norm() <= 0.12 * b.norm(), (a - b).norm().item() / b.norm().item()


@pytest.mark.gpu
def test_fp8_linear_deterministic_and_graph_replay():
    from byteps_b200.torch.graph import GraphedStep

    lin, x, dy = _linear_case((4, 256, 1024), 3072, True, torch.bfloat16, seed=1)
    lin2 = copy.deepcopy(lin)

    def run(layer):
        layer.weight.grad = layer.bias.grad = None
        x.grad = None
        y = layer(x)
        y.backward(dy)
        return y.detach().clone(), x.grad.clone(), layer.weight.grad.clone(), layer.bias.grad.clone()

    eager = [run(lin) for _ in range(4)]
    again = [run(lin2) for _ in range(4)]
    for a, b in zip(eager, again):
        assert all(torch.equal(u, v) for u, v in zip(a, b)), "run-to-run"
    # the same calls on a fresh copy, the fourth replayed from a graph captured after three eager calls
    lin3 = copy.deepcopy(lin2)
    lin3._fp8 = None
    xg = x.detach().clone().requires_grad_(True)

    def step():
        y = lin3(xg)
        y.backward(dy)
        return y

    for i in range(2):
        assert torch.equal(step(), eager[i][0]), i
        xg.grad = lin3.weight.grad = lin3.bias.grad = None
    for t in (xg, lin3.weight, lin3.bias):
        t.grad = torch.zeros_like(t)
    g = GraphedStep(step, warmup=1)
    for t in (xg, lin3.weight, lin3.bias):
        t.grad.zero_()
    y = g()
    torch.cuda.synchronize()
    assert torch.equal(y, eager[3][0]) and torch.equal(xg.grad, eager[3][1])
    assert torch.equal(lin3.weight.grad, eager[3][2]) and torch.equal(lin3.bias.grad, eager[3][3])


def _run_py(body: str, timeout=900):
    code = "import sys; sys.path.insert(0, %r)\n" % ROOT + textwrap.dedent(body)
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "DMLC_ROLE", "DMLC_NUM_WORKER", "DMLC_NUM_SERVER"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout


_BERT_STEPS = """
import torch
import byteps_b200.torch as bps
from byteps_b200.models import bert_tiny
from byteps_b200.torch.graph import GraphedStep
GRAPH, FUSED, SCALE, INJECT, OUT = %r, %r, %r, %r, %r
bps.init()
torch.manual_seed(0)
model = bert_tiny(fp8_linear=True, fused_loss=FUSED, fused_norm=FUSED, dropout=0.0).cuda().to(torch.bfloat16).train()
opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=0.01),
                               named_parameters=model.named_parameters(), fused_update=True,
                               dynamic_loss_scale={"init_scale": SCALE} if SCALE else False)
g = torch.Generator().manual_seed(1)
ids = torch.randint(0, 30522, (4, 64), generator=g).cuda()
labels = torch.randint(0, 30522, (4, 64), generator=g)
labels[torch.rand(4, 64, generator=g) > 0.15] = -100
labels = labels.cuda()
poison = torch.ones((), device="cuda")

def step():
    opt.zero_grad()
    loss = model(ids, mlm_labels=labels)
    (opt.scale_loss(loss * poison) if SCALE else loss).backward()
    opt.step()
    return loss

stepper = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams) if GRAPH else step
if not GRAPH:
    for _ in range(2):   # the graph's eager warm-up steps
        step()
losses = []
for i in range(4):
    poison.fill_(float("inf") if i == INJECT else 1.0)
    losses.append(stepper().detach().float().clone())
torch.cuda.synchronize()
torch.save({"losses": [l.item() for l in losses], "skipped": opt.skipped_steps if SCALE else 0,
            "params": {n: p.detach().float().cpu() for n, p in model.named_parameters()}}, OUT)
print("OK")
bps.shutdown()
"""


def _close(e, g):
    for a, b in zip(e["losses"], g["losses"]):
        assert abs(a - b) <= 1e-2 * abs(a), (e["losses"], g["losses"])
    for n, a in e["params"].items():
        b = g["params"][n]
        assert ((a - b).abs() <= 2.0 ** -6 * a.abs() + 1e-4).all(), n


@pytest.mark.gpu
def test_bert_tiny_fp8_graphed_step_matches_eager(tmp_path):
    runs = {}
    for graph in (False, True):
        out = str(tmp_path / ("graph.pt" if graph else "eager.pt"))
        assert "OK" in _run_py(_BERT_STEPS % (graph, False, 0.0, -1, out))
        runs[graph] = torch.load(out)
    _close(runs[False], runs[True])


@pytest.mark.gpu
def test_bert_tiny_fp8_with_fused_norm_loss_and_dynamic_loss_scale(tmp_path):
    """fp8_linear with fused_norm, fused_loss and a dynamic loss scale, graphed: without an overflow no step is
    skipped and the run follows the unscaled eager one; an inf injected into one step's loss is skipped (every
    parameter stays finite and the later steps train on)."""
    scaled, plain, hit = str(tmp_path / "scaled.pt"), str(tmp_path / "plain.pt"), str(tmp_path / "hit.pt")
    assert "OK" in _run_py(_BERT_STEPS % (True, True, 1024.0, -1, scaled))
    assert "OK" in _run_py(_BERT_STEPS % (False, True, 0.0, -1, plain))
    assert "OK" in _run_py(_BERT_STEPS % (True, True, 1024.0, 1, hit))
    s, p, h = torch.load(scaled), torch.load(plain), torch.load(hit)
    assert all(math.isfinite(v) for v in s["losses"]) and s["skipped"] == 0, s["losses"]
    _close(p, s)
    assert h["skipped"] == 1, h["skipped"]
    assert all(bool(t.isfinite().all()) for t in h["params"].values())
    assert all(math.isfinite(v) for v in h["losses"])


_CONVERGE = """
import torch
import byteps_b200.torch as bps
from byteps_b200.models import bert_tiny
bps.init()
torch.manual_seed(0)
base = bert_tiny(dropout=0.0)
res = {}
for fp8_linear in (False, True):
    model = bert_tiny(dropout=0.0, fp8_linear=fp8_linear)
    model.load_state_dict(base.state_dict())
    model = model.cuda().to(torch.bfloat16).train()
    opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=2e-3, weight_decay=0.01),
                                   named_parameters=model.named_parameters(), fused_update=True)
    g = torch.Generator().manual_seed(1)
    losses = []
    for i in range(300):
        ids = torch.randint(0, 512, (8, 64), generator=g)
        labels = ids.clone()
        labels[torch.rand(8, 64, generator=g) > 0.3] = -100
        opt.zero_grad()
        loss = model(ids.cuda(), mlm_labels=labels.cuda())
        loss.backward()
        opt.step()
        losses.append(loss.item())
    res[fp8_linear] = sum(losses[-20:]) / 20
print("RESULT %r %r" % (res[False], res[True]))
bps.shutdown()
"""


@pytest.mark.gpu
def test_bert_tiny_fp8_converges_like_bf16():
    """300 AdamW steps of a copy task (labels = input ids over 512 tokens), seeded, from the same weights: both
    models get the mean loss of the last 20 steps below 1.0, and fp8 ends within 0.25 of bf16."""
    out = _run_py(_CONVERGE)
    line = [l for l in out.splitlines() if l.startswith("RESULT")][0]
    bf16, f8 = (float(v) for v in line.split()[1:])
    assert bf16 < 1.0 and f8 < 1.0, (bf16, f8)
    assert abs(f8 - bf16) <= 0.25, (bf16, f8)


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=_dt_id)
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("shape", [(32, 64), (2, 16, 64), (5, 64)])
def test_cpu_fallback_is_f_linear(shape, bias, dtype):
    torch.manual_seed(0)
    lin = Fp8Linear(64, 48, bias=bias).to(dtype)
    x = torch.randn(*shape).to(dtype).requires_grad_(True)
    y = lin(x)
    assert type(y.grad_fn).__name__ != FUSED
    ref = F.linear(x, lin.weight, lin.bias)
    assert torch.equal(y, ref)
    gy = torch.randn_like(y)
    params = [x, lin.weight] + ([lin.bias] if bias else [])
    ga = torch.autograd.grad(y, params, gy)
    gb = torch.autograd.grad(ref, params, gy)
    assert all(torch.equal(a, b) for a, b in zip(ga, gb))
    assert lin._fp8 is None, "no scaling state off the fast path"


def test_bert_fp8_linear_keeps_the_stock_parameters_and_state_dict():
    torch.manual_seed(0)
    stock = bert_tiny()
    ours = bert_tiny(fp8_linear=True)
    assert ours.config.fp8_linear and not stock.config.fp8_linear
    layer = ours.layers[0]
    assert all(isinstance(getattr(layer, n), Fp8Linear) for n in ("qkv", "proj", "fc1", "fc2"))
    assert not any(isinstance(m, Fp8Linear) for m in (ours.pooler, ours.mlm_dense, ours.nsp))
    assert [(n, p.shape) for n, p in ours.named_parameters()] == [(n, p.shape) for n, p in stock.named_parameters()]
    a, b = ours.state_dict(), stock.state_dict()
    assert list(a) == list(b) and all(a[k].shape == b[k].shape and a[k].dtype == b[k].dtype for k in a)
    ours.load_state_dict(b, strict=True)
    stock2 = bert_tiny()
    stock2.load_state_dict(ours.state_dict(), strict=True)
    ids = torch.randint(0, 30522, (2, 16))
    labels = torch.randint(0, 30522, (2, 16))
    for training in (True, False):
        stock.train(training)
        ours.train(training)
        torch.manual_seed(2)
        l1 = stock(ids, mlm_labels=labels)
        torch.manual_seed(2)
        l2 = ours(ids, mlm_labels=labels)
        assert torch.equal(l1, l2), training


def test_model_to_dtype_leaves_the_scaling_state_alone():
    model = bert_tiny(fp8_linear=True)
    layers = [m for m in model.modules() if isinstance(m, Fp8Linear)]
    states = []
    for i, m in enumerate(layers):
        st = m.scaling_state("cpu")
        st.buf.view(torch.float32)[:, :fp8.HISTORY + 1] = 1.0 + i + torch.arange(3 * (fp8.HISTORY + 1)).view(3, -1)
        st.buf[:, fp8.HISTORY + 1] = 7
        st.seeded = [True, True]
        states.append((st, st.buf.clone()))
    model.to(torch.bfloat16)
    model.half()
    model.float()
    for m, (st, before) in zip(layers, states):
        assert m._fp8 is st and m.scaling_state("cpu") is st and st.seeded == [True, True]
        assert st.buf.dtype == torch.int32 and torch.equal(st.buf, before)
    assert not any("fp8" in k for k in model.state_dict())
