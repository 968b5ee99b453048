"""Fused dropout + residual add + LayerNorm (ops/ln.py, kernels/ln.cu).

GPU tests compare the fused kernels with a float64 reference.  The bounds follow the kernels' rounding steps:

* z = residual + dropout(y) is formed in fp32 and rounded once to the activation dtype (half an ulp, u_t * |z|
  with u_t = 2^-8 (bf16), 2^-11 (fp16), 2^-24 (fp32), or half the subnormal spacing near 0);
* the rest is checked against the reference formed from the kernel's own z: every fp32 quantity the kernels form
  (row sums, mean, variance, the dgamma / dbeta sums over rows) is a chain of at most a few hundred roundings, so
  its absolute error is below C_ACC * u32 times the sum of the magnitudes that enter it (u32 = 2^-24,
  C_ACC = 256); the mean's error enters every centred value z - mean, so those magnitudes include |mean| * rstd;
* the outputs are then rounded once to their dtype.

With dropout the reference uses the kernel's keep mask (``return_mask=True``); the mask itself is checked for its
kept fraction, its dependence on the seed only, and fresh bits on every call and every graph replay.

CPU tests (no marker) check that the module keeps nn.LayerNorm's state_dict, that BERT with ``fused_norm=True``
keeps the stock model's parameters and state_dict, and that both compute the stock composition on the path every
non-CUDA input takes.
"""
import copy
import os
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from byteps_b200.models import bert_tiny
from byteps_b200.ops.ln import DropoutAddLayerNorm, dropout_add_layer_norm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32 = 2.0 ** -24
C_ACC = 256
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
TINY = {torch.bfloat16: 2.0 ** -134, torch.float16: 2.0 ** -25, torch.float32: 2.0 ** -150}
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
EPS = 1e-5


def _dt_id(d):
    return str(d).replace("torch.", "")


def _stock(y, residual, weight, bias, p, eps, training):
    """The composition models/bert.py runs at each junction."""
    z = F.dropout(y, p, training)
    if residual is not None:
        z = residual + z
    return F.layer_norm(z, (y.shape[-1],), weight, bias, eps)


def _unpack(mask, shape):
    bits = (mask.unsqueeze(-1) >> torch.arange(8, device=mask.device, dtype=torch.uint8)) & 1
    return bits.reshape(shape).bool()


def _make(m, h, dtype, wdtype, residual, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    loc = torch.randn(m, 1, device=dev, generator=g, dtype=torch.float64)
    y = (torch.randn(m, h, device=dev, generator=g, dtype=torch.float64) * 2 + loc).to(dtype)
    r = torch.randn(m, h, device=dev, generator=g, dtype=torch.float64).to(dtype) if residual else None
    dout = torch.randn(m, h, device=dev, generator=g, dtype=torch.float64).to(dtype)
    w = (torch.randn(h, device=dev, generator=g, dtype=torch.float64)).to(wdtype)
    b = (torch.randn(h, device=dev, generator=g, dtype=torch.float64) * 0.5).to(wdtype)
    return y, r, dout, w, b


def _run(y, r, dout, w, b, p):
    yg = y.detach().clone().requires_grad_(True)
    rg = r.detach().clone().requires_grad_(True) if r is not None else None
    wg, bg = w.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
    out, mask = dropout_add_layer_norm(yg, rg, wg, bg, p, EPS, True, return_mask=True)
    assert type(out.grad_fn).__name__ == "_DropoutAddLayerNormFnBackward", "fused path not taken"
    z = out.grad_fn.saved_tensors[0]
    out.backward(dout)
    return dict(out=out.detach(), z=z.detach().clone(), mask=mask, dy=yg.grad, dres=None if r is None else rg.grad,
                dw=wg.grad, db=bg.grad)


def _check(m, h, dtype, wdtype, residual, p=0.0, seed=0):
    y, r, dout, w, b = _make(m, h, dtype, wdtype, residual, seed)
    res = _run(y, r, dout, w, b, p)
    ut, uw = UNIT[dtype], UNIT[wdtype]
    scale = 1.0 / (1.0 - p)

    # ---- z = residual + dropout(y), with the kernel's mask
    keep = torch.ones_like(y, dtype=torch.bool) if p == 0 else _unpack(res["mask"], y.shape)
    if p == 0:
        assert res["mask"] is None
    yk = torch.where(keep, y.double() * scale, torch.zeros((), dtype=torch.float64, device=y.device))
    z_ref = yk + (r.double() if r is not None else 0.0)
    mag_z = yk.abs() + (r.double().abs() if r is not None else 0.0)
    err_z = (res["z"].double() - z_ref).abs()
    assert (err_z <= 4 * U32 * mag_z + ut * z_ref.abs() + TINY[dtype]).all(), "z"

    # ---- forward, from the kernel's z
    zd = res["z"].double()
    mu = zd.mean(-1, keepdim=True)
    var = zd.var(-1, unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + EPS)
    xhat = (zd - mu) * rstd
    wd, bd = w.double(), b.double()
    out_ref = xhat * wd + bd
    shift = mu.abs() * rstd + 1.0
    mag = (xhat.abs() + shift) * wd.abs() + bd.abs()
    tol = C_ACC * U32 * mag + ut * (out_ref.abs() + C_ACC * U32 * mag) + TINY[dtype]
    err = (res["out"].double() - out_ref).abs()
    assert (err <= tol).all(), "out: worst excess %g" % (err - tol).max().item()

    # ---- backward
    gd = dout.double()
    g = gd * wd
    ma, mb = g.mean(-1, keepdim=True), (g * xhat).mean(-1, keepdim=True)
    dz_ref = rstd * (g - ma - xhat * mb)
    big_a = g.abs().mean(-1, keepdim=True)
    big_b = (g.abs() * (xhat.abs() + shift)).mean(-1, keepdim=True)
    mag_dz = rstd * (g.abs() + big_a + (xhat.abs() + shift) * big_b)
    tol_dz = C_ACC * U32 * mag_dz + ut * (dz_ref.abs() + C_ACC * U32 * mag_dz) + TINY[dtype]
    if r is not None:
        err = (res["dres"].double() - dz_ref).abs()
        assert (err <= tol_dz).all(), "dres: worst excess %g" % (err - tol_dz).max().item()
    dy_ref = torch.where(keep, dz_ref * scale, torch.zeros((), dtype=torch.float64, device=y.device))
    err = (res["dy"].double() - dy_ref).abs()
    assert (err <= tol_dz * scale).all(), "dy: worst excess %g" % (err - tol_dz * scale).max().item()
    assert not res["dy"][~keep].any(), "dropped elements must get no gradient"

    dw_ref, db_ref = (gd * xhat).sum(0), gd.sum(0)
    tol_dw = C_ACC * U32 * (gd.abs() * (xhat.abs() + shift)).sum(0)
    tol_db = C_ACC * U32 * gd.abs().sum(0)
    tol_dw = tol_dw + uw * (dw_ref.abs() + tol_dw) + TINY[wdtype]
    tol_db = tol_db + uw * (db_ref.abs() + tol_db) + TINY[wdtype]
    assert res["dw"].dtype == wdtype and res["db"].dtype == wdtype
    assert ((res["dw"].double() - dw_ref).abs() <= tol_dw).all(), "dgamma"
    assert ((res["db"].double() - db_ref).abs() <= tol_db).all(), "dbeta"
    return res


WDTYPES = [(dt, wdt) for dt in DTYPES for wdt in ([torch.float32] if dt == torch.float32 else [torch.float32, dt])]


# ---------------------------------------------------------------------------------------------------- GPU, p = 0
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,wdtype", WDTYPES, ids=["%s-w%s" % (_dt_id(a), _dt_id(b)) for a, b in WDTYPES])
@pytest.mark.parametrize("h", [8, 128, 768, 1024, 2048])
@pytest.mark.parametrize("m", [1, 7, 8192 + 3])
def test_ln_matches_float64(m, h, dtype, wdtype):
    for residual in (False, True):
        _check(m, h, dtype, wdtype, residual)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["h12", "h4096", "noncontiguous"])
def test_ln_unsupported_inputs_take_the_stock_path(case):
    torch.manual_seed(0)
    h = {"h12": 12, "h4096": 4096, "noncontiguous": 64}[case]
    y = torch.randn(33, h, device="cuda", dtype=torch.bfloat16)
    r = torch.randn(33, h, device="cuda", dtype=torch.bfloat16)
    if case == "noncontiguous":
        y = torch.randn(h, 33, device="cuda", dtype=torch.bfloat16).t()
        assert not y.is_contiguous()
    mod = DropoutAddLayerNorm(h, eps=EPS, p=0.1).cuda().to(torch.bfloat16)
    with torch.no_grad():
        mod.weight.normal_()
        mod.bias.normal_()
    yg, rg = y.detach().clone().requires_grad_(True), r.detach().clone().requires_grad_(True)
    out = mod(yg, rg)
    assert type(out.grad_fn).__name__ != "_DropoutAddLayerNormFnBackward"
    torch.manual_seed(1)
    out = mod(yg, rg)
    torch.manual_seed(1)
    ref = _stock(y, r, mod.weight, mod.bias, 0.1, EPS, True)
    assert torch.equal(out, ref)


# ---------------------------------------------------------------------------------------------------- GPU, p > 0
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,wdtype", WDTYPES, ids=["%s-w%s" % (_dt_id(a), _dt_id(b)) for a, b in WDTYPES])
@pytest.mark.parametrize("h", [128, 768, 1024])
def test_ln_dropout_matches_float64_with_its_mask(h, dtype, wdtype):
    for residual in (False, True):
        _check(515, h, dtype, wdtype, residual, p=0.1, seed=1)
    _check(64, h, dtype, wdtype, True, p=0.5, seed=2)


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_ln_dropout_mask_statistics_and_seeding(p):
    m, h = 8192, 1024
    y = torch.randn(m, h, device="cuda", dtype=torch.bfloat16)
    r = torch.randn_like(y)
    w = torch.ones(h, device="cuda", dtype=torch.bfloat16)
    b = torch.zeros_like(w)

    def mask(rows=m):
        return dropout_add_layer_norm(y[:rows], r[:rows], w, b, p, EPS, True, return_mask=True)[1]

    torch.manual_seed(7)
    a = mask()
    n = m * h
    kept = _unpack(a, (m, h)).sum().item()
    sd = (n * p * (1 - p)) ** 0.5
    assert abs(kept - n * (1 - p)) <= 5 * sd, (kept, n * (1 - p), sd)
    b2 = mask()
    assert not torch.equal(a, b2), "two calls drew the same mask"
    torch.manual_seed(7)
    assert torch.equal(mask(), a), "re-seeding did not reproduce the mask"
    # the bits depend on the element index only, not on the launch geometry
    torch.manual_seed(7)
    assert torch.equal(mask(37), a[:37])


@pytest.mark.gpu
def test_ln_eval_mode_has_no_dropout():
    torch.manual_seed(0)
    mod = DropoutAddLayerNorm(768, eps=EPS, p=0.5).cuda().to(torch.bfloat16).eval()
    y = torch.randn(100, 768, device="cuda", dtype=torch.bfloat16)
    r = torch.randn_like(y)
    out = mod(y, r)
    assert type(out.grad_fn).__name__ == "_DropoutAddLayerNormFnBackward"
    ref, mask = dropout_add_layer_norm(y, r, mod.weight, mod.bias, 0.0, EPS, True, return_mask=True)
    assert mask is None
    assert torch.equal(out, ref)


# ---------------------------------------------------------------------------------------------- determinism, graphs
@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_ln_deterministic(p):
    y, r, dout, w, b = _make(8192 + 3, 1024, torch.bfloat16, torch.bfloat16, True, seed=5)
    torch.manual_seed(3)
    a = _run(y, r, dout, w, b, p)
    torch.manual_seed(3)
    c = _run(y, r, dout, w, b, p)
    for k in a:
        assert (a[k] is None and c[k] is None) or torch.equal(a[k], c[k]), k


@pytest.mark.gpu
def test_ln_graph_replays_draw_new_masks():
    from byteps_b200.torch.graph import GraphedStep

    y, r, dout, w, b = _make(256, 768, torch.bfloat16, torch.bfloat16, True, seed=6)
    yg, rg = y.clone().requires_grad_(True), r.clone().requires_grad_(True)
    wg, bg = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    seen = torch.zeros(256, 96, dtype=torch.uint8, device="cuda")

    def step():
        out, mask = dropout_add_layer_norm(yg, rg, wg, bg, 0.1, EPS, True, return_mask=True)
        seen.copy_(mask)
        out.backward(dout)
        return out

    g = GraphedStep(step, warmup=2)
    masks = []
    for _ in range(3):
        g()
        torch.cuda.synchronize()
        masks.append(seen.clone())
    assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2])


def _run_py(body: str, timeout=600):
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
GRAPH, DROPOUT, OUT = %r, %r, %r
bps.init()
torch.manual_seed(0)
model = bert_tiny(fused_norm=True, dropout=DROPOUT).cuda().to(torch.bfloat16).train()
opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=0.01),
                               named_parameters=model.named_parameters(), fused_update=True)
g = torch.Generator().manual_seed(1)
ids = torch.randint(0, 30522, (4, 64), generator=g).cuda()
labels = torch.randint(0, 30522, (4, 64), generator=g).cuda()

def step():
    opt.zero_grad()
    loss = model(ids, mlm_labels=labels)
    loss.backward()
    opt.step()
    return loss

if GRAPH:
    stepper = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams)
else:
    stepper = step
    for _ in range(2):   # the graph's eager warm-up steps
        step()
losses = [stepper().detach().float().clone() for _ in range(4)]
torch.cuda.synchronize()
torch.save({"losses": [l.item() for l in losses],
            "params": {n: p.detach().float().cpu() for n, p in model.named_parameters()}}, OUT)
print("OK")
bps.shutdown()
"""


@pytest.mark.gpu
def test_bert_tiny_fused_norm_graphed_step_matches_eager(tmp_path):
    """A captured step of bert_tiny(fused_norm=True) in bf16 with the fused AdamW update replays and, with dropout
    0, gives the eager run's losses and parameters (two warm-up steps, then the graph's first replays)."""
    runs = {}
    for graph in (False, True):
        out = str(tmp_path / ("graph.pt" if graph else "eager.pt"))
        assert "OK" in _run_py(_BERT_STEPS % (graph, 0.0, out))
        runs[graph] = torch.load(out)
    e, g = runs[False], runs[True]
    for a, b in zip(e["losses"], g["losses"]):
        assert abs(a - b) <= 1e-2 * abs(a), (e["losses"], g["losses"])
    for n, a in e["params"].items():
        b = g["params"][n]
        assert ((a - b).abs() <= 2.0 ** -6 * a.abs() + 1e-4).all(), n


@pytest.mark.gpu
def test_bert_tiny_fused_norm_graphed_step_with_dropout(tmp_path):
    out = str(tmp_path / "drop.pt")
    assert "OK" in _run_py(_BERT_STEPS % (True, 0.1, out))
    res = torch.load(out)
    assert all(torch.isfinite(torch.tensor(res["losses"])))


@pytest.mark.gpu
def test_bert_tiny_fused_norm_matches_stock_bf16():
    """One bf16 forward + backward of bert_tiny at dropout 0, fused junctions against stock ones with the same
    weights.  Both are compared with the stock model in fp32: the fused loss and every parameter's gradient must be
    as close to it as bf16 allows - within twice the stock bf16 error, or 2 % relative L2, whichever is larger."""
    torch.manual_seed(0)
    stock = bert_tiny(dropout=0.0).cuda()
    fused = bert_tiny(dropout=0.0, fused_norm=True).cuda()
    fused.load_state_dict(stock.state_dict())
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 30522, (8, 128), generator=g).cuda()
    labels = torch.randint(0, 30522, (8, 128), generator=g).cuda()

    def grads(model, dtype):
        model = copy.deepcopy(model).to(dtype).train()
        loss = model(ids, mlm_labels=labels)
        loss.backward()
        # the pooler and NSP head get no gradient from the MLM loss alone
        return loss.item(), [None if p.grad is None else p.grad.double() for p in model.parameters()]

    l_ref, g_ref = grads(stock, torch.float32)
    l_stock, g_stock = grads(stock, torch.bfloat16)
    l_fused, g_fused = grads(fused, torch.bfloat16)
    assert abs(l_fused - l_ref) <= max(2 * abs(l_stock - l_ref), 1e-2 * abs(l_ref)), (l_fused, l_stock, l_ref)
    for (n, _), gf, gs, gr in zip(stock.named_parameters(), g_fused, g_stock, g_ref):
        assert (gf is None) == (gr is None), n
        if gr is None:
            continue
        nr = gr.norm().item() + 1e-30
        ef, es = (gf - gr).norm().item() / nr, (gs - gr).norm().item() / nr
        assert ef <= max(2 * es, 0.02), "%s: fused %.3g stock %.3g" % (n, ef, es)


# ---------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("residual", [False, True], ids=["no_residual", "residual"])
def test_module_cpu_is_stock(residual):
    torch.manual_seed(0)
    mod = DropoutAddLayerNorm(64, eps=1e-12, p=0.25)
    with torch.no_grad():
        mod.weight.normal_()
        mod.bias.normal_()
    y = torch.randn(5, 7, 64, requires_grad=True)
    r = torch.randn(5, 7, 64, requires_grad=True) if residual else None
    for training in (True, False):
        mod.train(training)
        torch.manual_seed(1)
        out = mod(y, r)
        torch.manual_seed(1)
        ref = _stock(y, r, mod.weight, mod.bias, 0.25, 1e-12, training)
        assert torch.equal(out, ref), training
        ga = torch.autograd.grad(out.sum(), [y, mod.weight, mod.bias] + ([r] if residual else []))
        gb = torch.autograd.grad(ref.sum(), [y, mod.weight, mod.bias] + ([r] if residual else []))
        for a, b in zip(ga, gb):
            assert torch.equal(a, b), training


def test_module_state_dict_is_layernorm():
    mod, ln = DropoutAddLayerNorm(96, eps=1e-6, p=0.1), nn.LayerNorm(96, eps=1e-6)
    assert isinstance(mod, nn.LayerNorm) and mod.p == 0.1 and mod.eps == 1e-6
    assert list(mod.state_dict()) == list(ln.state_dict())
    assert [n for n, _ in mod.named_parameters()] == [n for n, _ in ln.named_parameters()]
    sd = {k: v + 1 for k, v in ln.state_dict().items()}
    mod.load_state_dict(sd, strict=True)
    for k, v in mod.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_bert_fused_norm_keeps_the_stock_parameters():
    torch.manual_seed(0)
    stock = bert_tiny()
    fused = bert_tiny(fused_norm=True)
    assert all(isinstance(layer.norm1, DropoutAddLayerNorm) and isinstance(layer.norm2, DropoutAddLayerNorm)
               and layer.norm1.p == 0.1 for layer in fused.layers)
    assert type(fused.embeddings.norm) is nn.LayerNorm and type(fused.mlm_norm) is nn.LayerNorm
    assert all(type(m) is not DropoutAddLayerNorm for m in stock.modules())
    assert [n for n, _ in fused.named_parameters()] == [n for n, _ in stock.named_parameters()]
    ours, theirs = fused.state_dict(), stock.state_dict()
    assert list(ours) == list(theirs)
    assert all(ours[k].shape == theirs[k].shape and ours[k].dtype == theirs[k].dtype for k in ours)
    sd = {k: (v + 1 if v.is_floating_point() else v) for k, v in theirs.items()}
    fused.load_state_dict(sd, strict=True)
    for k, v in fused.state_dict().items():
        assert torch.equal(v, sd[k]), k
    stock.load_state_dict(fused.state_dict(), strict=True)


def test_bert_fused_norm_cpu_is_stock():
    torch.manual_seed(0)
    stock = bert_tiny()
    fused = bert_tiny(fused_norm=True)
    fused.load_state_dict(stock.state_dict())
    ids = torch.randint(0, 30522, (2, 16))
    labels = torch.randint(0, 30522, (2, 16))
    for training in (True, False):
        stock.train(training)
        fused.train(training)
        torch.manual_seed(2)
        a = stock(ids, mlm_labels=labels)
        torch.manual_seed(2)
        b = fused(ids, mlm_labels=labels)
        assert torch.equal(a, b), training
