"""DropoutAddLayerNorm's pre-LN form (ops/ln.py ``return_sum=True``, kernels/ln.cu with dsum): the residual sum
z = residual + dropout(y) as a second, differentiable output, whose own gradient dsum the backward kernel adds to
the LayerNorm's before it forms d(residual) and dy.

* against float64, with the bounds of test_gpu_ln.py plus the two roundings of s = round(round(dz) + dsum);
* bit for bit: z and out are what the single-output call computes and saves; with dsum, dres and dy are today's
  d(residual), then torch's add of dsum in the activation dtype, then torch's dropout backward s * keep * scale;
  without dsum every result equals the single-output call's;
* repeats, graph replays, launch counts, the stock fallbacks (z included) and the binding's alignment check.
"""
import json

import pytest
import torch
import torch.nn.functional as F

from byteps_b200 import _native
from byteps_b200.ops.ln import DropoutAddLayerNorm, dropout_add_layer_norm
from test_gpu_ln import C_ACC, EPS, TINY, U32, UNIT, WDTYPES, _check, _dt_id, _make, _run_py, _unpack

_CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
WIDS = ["%s-w%s" % (_dt_id(a), _dt_id(b)) for a, b in WDTYPES]


def _dsum(y, seed):
    g = torch.Generator(device="cuda").manual_seed(1000 + seed)
    return torch.randn(y.shape, device="cuda", generator=g, dtype=torch.float64).to(y.dtype)


def _run_sum(y, r, dout, dsum, w, b, p):
    """return_sum=True, backward with dout into out and dsum (or nothing) into z"""
    yg = y.detach().clone().requires_grad_(True)
    rg = r.detach().clone().requires_grad_(True) if r is not None else None
    wg, bg = w.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
    out, z, mask = dropout_add_layer_norm(yg, rg, wg, bg, p, EPS, True, return_mask=True, return_sum=True)
    assert type(out.grad_fn).__name__ == "_DropoutAddLayerNormFnBackward", "fused path not taken"
    outs, grads = [out], [dout]
    if dsum is not None:
        outs.append(z)
        grads.append(dsum)
    inputs = [yg, wg, bg] + ([rg] if r is not None else [])
    g = torch.autograd.grad(outs, inputs, grads)
    return dict(out=out.detach(), z=z.detach().clone(), mask=mask, dy=g[0], dw=g[1], db=g[2],
                dres=g[3] if r is not None else None)


def _check_sum(m, h, dtype, wdtype, residual, p, seed):
    """float64 reference with dsum: z and out as test_gpu_ln._check, then s = dz + dsum, dres = s and
    dy = s * keep * scale"""
    y, r, dout, w, b = _make(m, h, dtype, wdtype, residual, seed)
    dsum = _dsum(y, seed)
    res = _run_sum(y, r, dout, dsum, w, b, p)
    ut, uw = UNIT[dtype], UNIT[wdtype]
    scale = 1.0 / (1.0 - p)
    keep = torch.ones_like(y, dtype=torch.bool) if p == 0 else _unpack(res["mask"], y.shape)
    zero = torch.zeros((), dtype=torch.float64, device=y.device)
    yk = torch.where(keep, y.double() * scale, zero)
    z_ref = yk + (r.double() if r is not None else 0.0)
    mag_z = yk.abs() + (r.double().abs() if r is not None else 0.0)
    assert ((res["z"].double() - z_ref).abs() <= 4 * U32 * mag_z + ut * z_ref.abs() + TINY[dtype]).all(), "z"

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

    gd = dout.double()
    g = gd * wd
    ma, mb = g.mean(-1, keepdim=True), (g * xhat).mean(-1, keepdim=True)
    dz_ref = rstd * (g - ma - xhat * mb)
    big_a = g.abs().mean(-1, keepdim=True)
    big_b = (g.abs() * (xhat.abs() + shift)).mean(-1, keepdim=True)
    acc = C_ACC * U32 * rstd * (g.abs() + big_a + (xhat.abs() + shift) * big_b)
    s_ref = dz_ref + dsum.double()
    # dz in fp32 (acc), rounded to the dtype, dsum added in fp32 and the sum rounded once more
    tol_s = (acc + ut * (dz_ref.abs() + acc)) * (1 + 2 * ut) + (ut + U32) * s_ref.abs() + 2 * TINY[dtype]
    if r is not None:
        err = (res["dres"].double() - s_ref).abs()
        assert (err <= tol_s).all(), "dres: worst excess %g" % (err - tol_s).max().item()
    dy_ref = torch.where(keep, s_ref * scale, zero)
    tol_dy = tol_s * scale * (1 + 2 * ut) + (ut + U32) * dy_ref.abs() + TINY[dtype]
    err = (res["dy"].double() - dy_ref).abs()
    assert (err <= tol_dy).all(), "dy: worst excess %g" % (err - tol_dy).max().item()
    assert not res["dy"][~keep].any(), "dropped elements must get no gradient"

    dw_ref, db_ref = (gd * xhat).sum(0), gd.sum(0)
    tol_dw = C_ACC * U32 * (gd.abs() * (xhat.abs() + shift)).sum(0)
    tol_db = C_ACC * U32 * gd.abs().sum(0)
    tol_dw = tol_dw + uw * (dw_ref.abs() + tol_dw) + TINY[wdtype]
    tol_db = tol_db + uw * (db_ref.abs() + tol_db) + TINY[wdtype]
    assert ((res["dw"].double() - dw_ref).abs() <= tol_dw).all(), "dgamma"
    assert ((res["db"].double() - db_ref).abs() <= tol_db).all(), "dbeta"


def _check_no_dsum(m, h, dtype, wdtype, residual, p, seed):
    """float64 reference of test_gpu_ln._check through return_sum=True with nothing reaching z"""
    y, r, dout, w, b = _make(m, h, dtype, wdtype, residual, seed)
    torch.manual_seed(seed)
    single = _check(m, h, dtype, wdtype, residual, p, seed)
    torch.manual_seed(seed)
    res = _run_sum(y, r, dout, None, w, b, p)
    for k in ("out", "mask", "dy", "dres", "dw", "db"):
        assert (single[k] is None and res[k] is None) or torch.equal(single[k], res[k]), k
    assert torch.equal(res["z"], single["z"])


# ------------------------------------------------------------------------------------------------- float64
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,wdtype", WDTYPES, ids=WIDS)
@pytest.mark.parametrize("h", [8, 128, 768, 1024, 2048])
@pytest.mark.parametrize("m", [1, 7, 8192 + 3])
def test_prenorm_matches_float64(m, h, dtype, wdtype):
    for residual in (False, True):
        for p in (0.0, 0.1):
            seed = 3 * residual + (p > 0)
            torch.manual_seed(seed)
            _check_sum(m, h, dtype, wdtype, residual, p, seed)
            _check_no_dsum(m, h, dtype, wdtype, residual, p, seed)


# --------------------------------------------------------------------------------------------------- bit-exact
def _today_dz(single_out, dout):
    """today's d(residual) = dz of the single-output call's saved tensors, through the binding with a dres pointer"""
    z, w, mean, rstd, mask = single_out.grad_fn.saved_tensors
    cu = _native.cuda()
    m, h = z.numel() // z.shape[-1], z.shape[-1]
    dres = torch.empty_like(z)
    dw, db = torch.empty_like(w), torch.empty_like(w)
    nws, nctr = cu.ln_workspace(m, h)
    ws = torch.empty(nws, dtype=torch.float32, device="cuda")
    ctr = torch.zeros(nctr, dtype=torch.int32, device="cuda")
    cu.ln_bwd(dout.data_ptr(), z.data_ptr(), 0 if mask is None else mask.data_ptr(), _CODES[z.dtype],
              _CODES[w.dtype], m, h, 1.0, mean.data_ptr(), rstd.data_ptr(), w.data_ptr(), dres.data_ptr(), 0,
              dw.data_ptr(), db.data_ptr(), ws.data_ptr(), ctr.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return dres


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,wdtype", WDTYPES, ids=WIDS)
@pytest.mark.parametrize("h", [128, 768, 1024])
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("residual", [False, True], ids=["no_residual", "residual"])
def test_prenorm_bit_exact_against_autograd_composition(residual, p, h, dtype, wdtype):
    m = 1031
    y, r, dout, w, b = _make(m, h, dtype, wdtype, residual, seed=11)
    dsum = _dsum(y, 11)
    yg = y.clone().requires_grad_(True)
    rg = r.clone().requires_grad_(True) if residual else None
    wg, bg = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    torch.manual_seed(4)
    single, mask = dropout_add_layer_norm(yg, rg, wg, bg, p, EPS, True, return_mask=True)
    inputs = [yg, wg, bg] + ([rg] if residual else [])
    today = torch.autograd.grad(single, inputs, dout, retain_graph=True)
    dz = _today_dz(single, dout)
    if residual:
        assert torch.equal(dz, today[3])
    torch.manual_seed(4)
    res = _run_sum(y, r, dout, dsum, w, b, p)

    # forward: out and z are the single-output call's output and saved z
    assert torch.equal(res["out"], single.detach())
    assert torch.equal(res["z"], single.grad_fn.saved_tensors[0])
    assert (mask is None and res["mask"] is None) or torch.equal(res["mask"], mask)
    # backward: today's dz, torch's add of dsum, then torch's dropout backward
    s = dz + dsum
    keep = torch.ones_like(y, dtype=torch.bool) if mask is None else _unpack(mask, y.shape)
    scale = torch.tensor(1.0 / (1.0 - p), dtype=torch.float32, device="cuda")
    dy = (s.float() * keep * scale).to(dtype)
    assert torch.equal(res["dy"], dy)
    if residual:
        assert torch.equal(res["dres"], s)
    # dgamma and dbeta do not depend on dsum
    assert torch.equal(res["dw"], today[1]) and torch.equal(res["db"], today[2])


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_prenorm_gradient_of_z_alone(p):
    """nothing reaches out: d(residual) is dsum itself, dy = dsum * keep * scale and dgamma = dbeta = 0"""
    y, r, _, w, b = _make(515, 768, torch.bfloat16, torch.bfloat16, True, seed=12)
    dsum = _dsum(y, 12)
    yg, rg = y.clone().requires_grad_(True), r.clone().requires_grad_(True)
    wg, bg = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    out, z, mask = dropout_add_layer_norm(yg, rg, wg, bg, p, EPS, True, return_mask=True, return_sum=True)
    dy, dres, dw, db = torch.autograd.grad(z, [yg, rg, wg, bg], dsum)
    keep = torch.ones_like(y, dtype=torch.bool) if mask is None else _unpack(mask, y.shape)
    assert torch.equal(dres, dsum)
    assert torch.equal(dy, (dsum.float() * keep * torch.tensor(1.0 / (1.0 - p), device="cuda")).to(y.dtype))
    assert not dw.any() and not db.any()


@pytest.mark.gpu
def test_prenorm_z_is_written_without_grad_and_in_eval():
    torch.manual_seed(0)
    mod = DropoutAddLayerNorm(768, eps=EPS, p=0.1).cuda().to(torch.bfloat16)
    y = torch.randn(100, 768, device="cuda", dtype=torch.bfloat16)
    r = torch.randn_like(y)
    for training in (True, False):
        mod.train(training)
        with torch.no_grad():
            torch.manual_seed(5)
            out, z, mask = dropout_add_layer_norm(y, r, mod.weight, mod.bias, mod.p, EPS, training,
                                                  return_mask=True, return_sum=True)
        assert (mask is None) == (not training)
        keep = torch.ones_like(y, dtype=torch.bool) if mask is None else _unpack(mask, y.shape)
        scale = torch.tensor(1.0 / (1.0 - 0.1) if training else 1.0, device="cuda")
        ref = (r.float() + torch.where(keep, y.float() * scale, torch.zeros((), device="cuda"))).to(y.dtype)
        assert torch.equal(z, ref), training
        torch.manual_seed(5)
        assert torch.equal(out, mod(y, r)), training
    # nothing added or dropped: z is y, and a backward through it still adds dsum
    mod.eval()
    yg = y.clone().requires_grad_(True)
    out, z = mod(yg, return_sum=True)
    assert torch.equal(z, y)
    dsum, dout = torch.randn_like(y), torch.randn_like(y)
    (dy,) = torch.autograd.grad([out, z], [yg], [dout, dsum])
    (dy_ln,) = torch.autograd.grad(mod(yg), [yg], dout)
    assert torch.equal(dy, dy_ln + dsum)


# -------------------------------------------------------------------------------------- repeats and graphs
@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_prenorm_deterministic(p):
    y, r, dout, w, b = _make(8192 + 3, 1024, torch.bfloat16, torch.bfloat16, True, seed=5)
    dsum = _dsum(y, 5)
    torch.manual_seed(3)
    a = _run_sum(y, r, dout, dsum, w, b, p)
    torch.manual_seed(3)
    c = _run_sum(y, r, dout, dsum, w, b, p)
    for k in a:
        assert (a[k] is None and c[k] is None) or torch.equal(a[k], c[k]), k


@pytest.mark.gpu
def test_prenorm_graph_replay_equals_eager_and_draws_new_masks():
    from byteps_b200.torch.graph import GraphedStep

    y, r, dout, w, b = _make(256, 768, torch.bfloat16, torch.bfloat16, True, seed=6)
    dsum = _dsum(y, 6)
    leaves = [t.clone().requires_grad_(True) for t in (y, r, w, b)]
    seen = {0.0: [torch.zeros(256, 768, dtype=torch.bfloat16, device="cuda") for _ in range(5)],
            0.1: [torch.zeros(256, 96, dtype=torch.uint8, device="cuda")]}

    def step(p):
        out, z, mask = dropout_add_layer_norm(leaves[0], leaves[1], leaves[2], leaves[3], p, EPS, True,
                                              return_mask=True, return_sum=True)
        grads = torch.autograd.grad([out, z], leaves, [dout, dsum])
        if p == 0.0:
            for dst, src in zip(seen[0.0], [out, z, grads[0], grads[1], grads[2].expand(256, 768)]):
                dst.copy_(src)
        else:
            seen[0.1][0].copy_(mask)

    g = GraphedStep(lambda: step(0.0), warmup=2)
    # capturing runs nothing: the buffers hold the last eager warm-up step's results
    eager = [t.clone() for t in seen[0.0]]
    for _ in range(2):
        g()
        torch.cuda.synchronize()
        for a, c in zip(eager, seen[0.0]):
            assert torch.equal(a, c)
    g = GraphedStep(lambda: step(0.1), warmup=2)
    masks = []
    for _ in range(3):
        g()
        torch.cuda.synchronize()
        masks.append(seen[0.1][0].clone())
    assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2])


_LAUNCHES = """
import json
import torch
from torch.profiler import ProfilerActivity, profile
from byteps_b200.ops.ln import dropout_add_layer_norm

def launches(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

res = {}
for p in (0.0, 0.1):
    y = torch.randn(4096, 768, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    r = torch.randn_like(y, requires_grad=True)
    w = torch.ones(768, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    b = torch.zeros_like(w, requires_grad=True)
    dout, dsum = torch.randn_like(y), torch.randn_like(y)
    run = lambda: dropout_add_layer_norm(y, r, w, b, p, 1e-5, True, return_sum=True)
    torch.autograd.grad(run(), [y, r, w, b], [dout, dsum])
    o = {}
    fwd = launches(lambda: o.setdefault("o", run()))
    bwd = launches(lambda: torch.autograd.grad(o["o"], [y, r, w, b], [dout, dsum]))
    res[str(p)] = {"fwd": fwd, "bwd": bwd}
print(json.dumps(res))
"""


@pytest.mark.gpu
def test_prenorm_launch_count():
    """one LayerNorm launch each way (forward also draws the dropout seed; backward zeroes its counters)"""
    res = json.loads(_run_py(_LAUNCHES).strip().splitlines()[-1])
    for p, names in res.items():
        fwd, bwd = names["fwd"], names["bwd"]
        assert sum("ln_fwd_kernel" in n for n in fwd) == 1 and len(fwd) == (1 if p == "0.0" else 2), (p, fwd)
        assert sum("ln_bwd_kernel" in n for n in bwd) == 1 and len(bwd) <= 2, (p, bwd)
        assert all("ln_bwd_kernel" in n or "emset" in n or "Fill" in n for n in bwd), (p, bwd)


# ----------------------------------------------------------------------------------------------- fallbacks
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["h12", "h4096", "noncontiguous", "float64", "p1"])
@pytest.mark.parametrize("residual", [False, True], ids=["no_residual", "residual"])
def test_prenorm_unsupported_inputs_take_the_stock_path(case, residual):
    torch.manual_seed(0)
    h = {"h12": 12, "h4096": 4096}.get(case, 64)
    dtype = torch.float64 if case == "float64" else torch.bfloat16
    p = 1.0 if case == "p1" else 0.1
    y = torch.randn(33, h, device="cuda", dtype=dtype)
    r = torch.randn(33, h, device="cuda", dtype=dtype) if residual else None
    if case == "noncontiguous":
        y = torch.randn(h, 33, device="cuda", dtype=dtype).t()
    mod = DropoutAddLayerNorm(h, eps=EPS, p=p).cuda().to(dtype)
    with torch.no_grad():
        mod.weight.normal_()
        mod.bias.normal_()
    leaves = [y.detach().clone().requires_grad_(True), mod.weight] + (
        [r.detach().clone().requires_grad_(True)] if residual else [])
    torch.manual_seed(1)
    out, z = mod(leaves[0], leaves[2] if residual else None, return_sum=True)
    assert type(out.grad_fn).__name__ != "_DropoutAddLayerNormFnBackward"
    torch.manual_seed(1)
    z_ref = F.dropout(leaves[0], p, True)
    if residual:
        z_ref = leaves[2] + z_ref
    ref = F.layer_norm(z_ref, (h,), mod.weight, mod.bias, EPS)
    assert torch.equal(out, ref) and torch.equal(z, z_ref)
    dout, dsum = torch.randn_like(out), torch.randn_like(out)
    ga = torch.autograd.grad([out, z], leaves, [dout, dsum])
    gb = torch.autograd.grad([ref, z_ref], leaves, [dout, dsum])
    for a, c in zip(ga, gb):
        assert torch.equal(a, c)


# ------------------------------------------------------------------------------------------------- binding
@pytest.mark.gpu
def test_binding_rejects_misaligned_dsum():
    cu = _native.cuda()
    m, h = 64, 128
    f = dict(device="cuda")
    z, dres = torch.randn(m, h, dtype=torch.bfloat16, **f), torch.empty(m, h, dtype=torch.bfloat16, **f)
    dout = torch.zeros_like(z)   # dz = 0, so dres is dsum itself
    dsum = torch.randn(m * h + 8, dtype=torch.bfloat16, **f)
    w = torch.ones(h, dtype=torch.bfloat16, **f)
    dw, db = torch.empty_like(w), torch.empty_like(w)
    mean, rstd = torch.zeros(m, **f), torch.ones(m, **f)
    nws, nctr = cu.ln_workspace(m, h)
    ws = torch.empty(nws, **f)
    ctr = torch.zeros(nctr, dtype=torch.int32, **f)
    stream = torch.cuda.current_stream().cuda_stream
    args = (dout.data_ptr(), z.data_ptr(), 0, 1, 1, m, h, 1.0, mean.data_ptr(), rstd.data_ptr(), w.data_ptr(),
            dres.data_ptr(), 0, dw.data_ptr(), db.data_ptr(), ws.data_ptr(), ctr.data_ptr(), stream)
    with pytest.raises(RuntimeError, match="ln_bwd"):
        cu.ln_bwd(*args, dsum=dsum.data_ptr() + 2)
    cu.ln_bwd(*args, dsum=dsum.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(dres, dsum[: m * h].view(m, h))
