"""Fused softmax cross-entropy (ops/xent.py, kernels/xent.cu).

GPU tests compare the fused kernels with a float64 reference built from the same low-precision logits x.  The bounds
follow the kernels' rounding steps (u32 = 2^-24, C_ACC = 256 as in test_gpu_ln.py):

* each term exp(x_k - m) of a row's sum s is formed from a rounded difference, a rounded product with log2(e) and
  ex2, so its relative error is below a few u32 plus 2 u32 |x_k - m|; the terms are added in chains of at most a
  few hundred roundings, and the running maximum rescales partial sums with errors of the same kind.  So s is off
  by at most C_ACC u32 A, with A = sum (1 + |x_k - m|) exp(x_k - m), and lse = m + log(s) by
  C_ACC u32 A / s + 4 u32 |lse| (the log and the final add); the loss lse - x[t] adds one more rounding;
* the reduced loss adds the rows' errors plus C_ACC u32 times the sum of |loss|; the mean divides once more;
* dlogits = g (exp(x - lse) - [j == t]): exp(x - lse) inherits lse's error as a relative error and adds
  C_ACC u32 (1 + |x - lse|) of its own; the subtraction and the product with g round once each, and the result is
  rounded once to the logits dtype (half an ulp: u_t = 2^-8 bf16, 2^-11 fp16, 2^-24 fp32, or half the subnormal
  spacing near 0).

CPU tests (no marker) check that the op is exactly the stock F.cross_entropy(logits.float(), ...) on the path every
non-CUDA input takes, and that BERT with ``fused_loss=True`` keeps the stock model's parameters, state_dict and loss.
"""
import copy
import math
import os
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn.functional as F

from byteps_b200.models import bert_tiny
from byteps_b200.ops.xent import softmax_cross_entropy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32 = 2.0 ** -24
C_ACC = 256
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
TINY = {torch.bfloat16: 2.0 ** -134, torch.float16: 2.0 ** -25, torch.float32: 2.0 ** -150}
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
IGNORE = -100
FUSED = "_SoftmaxCrossEntropyFnBackward"


def _dt_id(d):
    return str(d).replace("torch.", "")


def _make(m, v, dtype, ignore="some", scale=3.0, offset=0.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    loc = torch.randn(m, 1, device="cuda", generator=g, dtype=torch.float64) * offset
    x = (torch.randn(m, v, device="cuda", generator=g, dtype=torch.float64) * scale + loc).to(dtype)
    t = torch.randint(0, v, (m,), device="cuda", generator=g)
    if ignore == "some":
        t[torch.arange(m, device="cuda") % 7 == 3] = IGNORE
    elif ignore == "all":
        t.fill_(IGNORE)
    return x, t


def _run(x, t, reduction, grad=None):
    xg = x.detach().clone().requires_grad_(True)
    loss = softmax_cross_entropy(xg, t, ignore_index=IGNORE, reduction=reduction)
    assert type(loss.grad_fn).__name__ == FUSED, "fused path not taken"
    assert loss.dtype == torch.float32
    if grad is None:
        grad = torch.ones_like(loss)
    loss.backward(grad)
    assert xg.grad.dtype == x.dtype
    return loss.detach(), xg.grad


def _reference(x, t):
    """float64 per-row lse, loss (0 where ignored), the valid mask and the lse error bound"""
    xd = x.double()
    valid = t != IGNORE
    m = xd.max(1, keepdim=True).values
    e = torch.exp(xd - m)
    s = e.sum(1)
    a = ((1 + (xd - m).abs()) * e).sum(1)
    lse = m.squeeze(1) + torch.log(s)
    tc = torch.where(valid, t, torch.zeros_like(t))
    xt = xd.gather(1, tc.unsqueeze(1)).squeeze(1)
    loss = torch.where(valid, lse - xt, torch.zeros_like(lse))
    tol_lse = C_ACC * U32 * a / s + 4 * U32 * lse.abs()
    tol_loss = torch.where(valid, tol_lse + 2 * U32 * loss.abs(), torch.zeros_like(lse))
    return dict(lse=lse, loss=loss, valid=valid, tol_lse=tol_lse, tol_loss=tol_loss)


def _check_dlogits(dx, x, t, ref, g_row):
    """g_row: float64 [M] gradient scale of each row"""
    xd = x.double()
    valid = ref["valid"]
    p = torch.exp(xd - ref["lse"].unsqueeze(1))
    hot = torch.zeros_like(p)
    rows = valid.nonzero().squeeze(1)
    hot[rows, t[rows]] = 1.0
    g = g_row.unsqueeze(1)
    d_ref = g * (p - hot)
    d_ref[~valid] = 0.0
    err_p = p * (1.01 * ref["tol_lse"].unsqueeze(1) + C_ACC * U32 * (1 + (xd - ref["lse"].unsqueeze(1)).abs()))
    tol = g.abs() * (err_p + C_ACC * U32 * (p - hot).abs())
    ut = UNIT[x.dtype]
    tol = tol + ut * (d_ref.abs() + tol) + TINY[x.dtype]
    err = (dx.double() - d_ref).abs()
    assert (err <= tol).all(), "dlogits: worst excess %g" % (err - tol).max().item()
    assert not dx[~valid].any(), "ignored rows must get zero gradient"


def _check(x, t):
    m = x.shape[0]
    ref = _reference(x, t)
    count = int(ref["valid"].sum().item())
    tot = ref["loss"].sum().item()
    tol_tot = ref["tol_loss"].sum().item() + C_ACC * U32 * ref["loss"].abs().sum().item()

    # none: per-row losses, with a per-row gradient
    gen = torch.Generator(device="cuda").manual_seed(11)
    grad_rows = torch.randn(m, device="cuda", generator=gen)
    loss, dx = _run(x, t, "none", grad_rows)
    assert loss.shape == (m,)
    err = (loss.double() - ref["loss"]).abs()
    assert (err <= ref["tol_loss"]).all(), "loss rows: worst excess %g" % (err - ref["tol_loss"]).max().item()
    assert not loss[~ref["valid"]].any(), "ignored rows have loss 0"
    _check_dlogits(dx, x, t, ref, grad_rows.double())

    # sum
    loss, dx = _run(x, t, "sum", torch.tensor(0.75, device="cuda"))
    assert loss.shape == ()
    assert abs(loss.item() - tot) <= tol_tot, (loss.item(), tot, tol_tot)
    _check_dlogits(dx, x, t, ref, torch.full((m,), 0.75, dtype=torch.float64, device="cuda"))

    # mean
    loss, dx = _run(x, t, "mean", torch.tensor(1.5, device="cuda"))
    if count == 0:
        assert math.isnan(loss.item()), "mean over no rows is NaN"
        assert not dx.any()
        return
    mean = tot / count
    assert abs(loss.item() - mean) <= tol_tot / count + 2 * U32 * abs(mean), (loss.item(), mean)
    _check_dlogits(dx, x, t, ref, torch.full((m,), 1.5 / count, dtype=torch.float64, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("v", [1, 7, 1000, 30522, 65539])
@pytest.mark.parametrize("m", [1, 37, 8192])
def test_xent_matches_float64(m, v, dtype):
    if v == 65539 and m == 8192:
        m = 4099      # keeps the float64 reference's temporaries small
    x, t = _make(m, v, dtype)
    _check(x, t)


@pytest.mark.gpu
@pytest.mark.parametrize("ignore", ["none", "some", "all"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_xent_ignored_rows(ignore, dtype):
    x, t = _make(257, 1000, dtype, ignore=ignore, seed=3)
    _check(x, t)
    if ignore == "all":
        stock = F.cross_entropy(x.float(), t, ignore_index=IGNORE)
        assert math.isnan(stock.item())


@pytest.mark.gpu
def test_xent_large_offsets_fp32():
    """rows centred around +-1e4: the row max, not a fixed reference, keeps the exponentials in range"""
    x, t = _make(64, 30522, torch.float32, offset=1e4, seed=4)
    assert x.abs().max().item() > 5e3
    _check(x, t)


@pytest.mark.gpu
def test_xent_unsupported_inputs_take_the_stock_path():
    x, t = _make(33, 100, torch.bfloat16, seed=5)
    cases = {
        "noncontiguous": (x.t().contiguous().t(), t),
        "1d": (x[0], t[0]),
        "float64": (x.double(), t),
        "misaligned base": (torch.cat([x.view(-1)[:1], x.view(-1)])[1:].view(33, 100), t),
        "empty": (x[:0], t[:0]),
    }
    for name, (xi, ti) in cases.items():
        xg = xi.detach().requires_grad_(True)
        out = softmax_cross_entropy(xg, ti, ignore_index=IGNORE)
        assert type(out.grad_fn).__name__ != FUSED, name
        ref = F.cross_entropy(xg.float(), ti, ignore_index=IGNORE)
        assert torch.equal(out, ref) or (out.isnan().all() and ref.isnan().all()), name


@pytest.mark.gpu
def test_xent_target_out_of_range_is_nan():
    """A target outside [0, V) is never read: its row's loss and gradient are NaN, the others are unaffected."""
    x, t = _make(50, 1000, torch.bfloat16, seed=6)
    bad = torch.tensor([4, 17, 31], device="cuda")
    t[bad] = torch.tensor([-1, 1000, 1 << 40], device="cuda")
    good = torch.ones(50, dtype=torch.bool, device="cuda")
    good[bad] = False
    for reduction in ("mean", "sum"):
        loss, dx = _run(x, t, reduction)
        assert math.isnan(loss.item()), reduction
        assert dx[bad].isnan().all() and not dx[good].isnan().any()
    loss, dx = _run(x, t, "none")
    assert loss[bad].isnan().all() and loss[good].isfinite().all()
    tg = t.clone()
    tg[bad] = IGNORE
    ref = _reference(x, tg)
    err = (loss[good].double() - ref["loss"][good]).abs()
    assert (err <= ref["tol_loss"][good]).all()


@pytest.mark.gpu
def test_xent_grad_output_scale_is_read_on_the_device():
    """A power-of-two loss scale enters through grad_output and scales dlogits exactly (fp32 logits)."""
    x, t = _make(300, 1000, torch.float32, seed=7)
    _, d1 = _run(x, t, "mean", torch.tensor(1.0, device="cuda"))
    _, d2 = _run(x, t, "mean", torch.tensor(1024.0, device="cuda"))
    assert torch.equal(d2, d1 * 1024)


@pytest.mark.gpu
def test_xent_deterministic():
    x, t = _make(8192, 30522, torch.bfloat16, seed=8)
    a = [_run(x, t, "mean") for _ in range(2)]
    assert torch.equal(a[0][0], a[1][0]) and torch.equal(a[0][1], a[1][1])
    b = [_run(x, t, "none", torch.ones(8192, device="cuda")) for _ in range(2)]
    assert torch.equal(b[0][0], b[1][0]) and torch.equal(b[0][1], b[1][1])


@pytest.mark.gpu
def test_xent_graph_replay_matches_eager():
    """Nothing is read back to the host, so forward and backward capture into a CUDA graph and replay bit-exactly."""
    from byteps_b200.torch.graph import GraphedStep

    x, t = _make(1024, 30522, torch.bfloat16, seed=9)
    loss_e, d_e = _run(x, t, "mean")
    xg = x.clone().requires_grad_(True)

    def step():
        loss = softmax_cross_entropy(xg, t)
        loss.backward()
        return loss

    g = GraphedStep(step, warmup=2)
    for _ in range(3):
        xg.grad.zero_()
        out = g()
        torch.cuda.synchronize()
        assert torch.equal(out, loss_e) and torch.equal(xg.grad, d_e)


@pytest.mark.gpu
def test_xent_more_than_2_31_elements():
    """70 400 x 30 522 bf16 logits (2.15e9 elements): rows past element 2^31 checked against float64."""
    m, v = 70400, 30522
    assert m * v > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(10)
    x = torch.randn(m, v, device="cuda", generator=g, dtype=torch.bfloat16) * 3
    t = torch.randint(0, v, (m,), device="cuda", generator=g)
    xg = x.requires_grad_(True)
    loss = softmax_cross_entropy(xg, t, reduction="sum")
    assert type(loss.grad_fn).__name__ == FUSED
    lse_k = loss.grad_fn.saved_tensors[1]
    loss.backward()
    dx = xg.grad
    rows = torch.tensor([0, 1, 2 ** 31 // v - 1, 2 ** 31 // v, 2 ** 31 // v + 1, m - 2, m - 1], device="cuda")
    xs, ts = x.detach()[rows], t[rows]
    ref = _reference(xs, ts)
    err = (lse_k[rows].double() - ref["lse"]).abs()
    assert (err <= ref["tol_lse"]).all(), err
    _check_dlogits(dx[rows], xs, ts, ref, torch.ones(len(rows), dtype=torch.float64, device="cuda"))
    # the reduced loss over every row, float64 in chunks
    tot, tol = 0.0, 0.0
    for r0 in range(0, m, 4096):
        rc = _reference(x.detach()[r0:r0 + 4096], t[r0:r0 + 4096])
        tot += rc["loss"].sum().item()
        tol += rc["tol_loss"].sum().item() + C_ACC * U32 * rc["loss"].abs().sum().item()
    assert abs(loss.item() - tot) <= tol, (loss.item(), tot, tol)


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
GRAPH, FUSED_LOSS, FUSED_NORM, SCALE, OUT = %r, %r, %r, %r, %r
bps.init()
torch.manual_seed(0)
model = bert_tiny(fused_loss=FUSED_LOSS, fused_norm=FUSED_NORM, dropout=0.0).cuda().to(torch.bfloat16).train()
opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=0.01),
                               named_parameters=model.named_parameters(), fused_update=True,
                               dynamic_loss_scale={"init_scale": SCALE} if SCALE else False)
g = torch.Generator().manual_seed(1)
ids = torch.randint(0, 30522, (4, 64), generator=g).cuda()
labels = torch.randint(0, 30522, (4, 64), generator=g)
labels[torch.rand(4, 64, generator=g) > 0.15] = -100     # MLM masking: most positions carry no label
labels = labels.cuda()

def step():
    opt.zero_grad()
    loss = model(ids, mlm_labels=labels)
    (opt.scale_loss(loss) if SCALE else loss).backward()
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
def test_bert_tiny_fused_loss_graphed_step_matches_eager(tmp_path):
    """A captured step of bert_tiny(fused_loss=True) in bf16 with the fused AdamW update replays and gives the eager
    run's losses and parameters (two warm-up steps, then the graph's first replays)."""
    runs = {}
    for graph in (False, True):
        out = str(tmp_path / ("graph.pt" if graph else "eager.pt"))
        assert "OK" in _run_py(_BERT_STEPS % (graph, True, False, 0.0, out))
        runs[graph] = torch.load(out)
    _close(runs[False], runs[True])


@pytest.mark.gpu
def test_bert_tiny_fused_loss_with_fused_norm_and_dynamic_loss_scale(tmp_path):
    """fused_loss together with fused_norm and a dynamic loss scale of 2^12, graphed: the scale reaches the loss
    kernel through grad_output, no step is skipped, and losses and parameters follow the unscaled eager run."""
    scaled, plain = str(tmp_path / "scaled.pt"), str(tmp_path / "plain.pt")
    assert "OK" in _run_py(_BERT_STEPS % (True, True, True, 4096.0, scaled))
    assert "OK" in _run_py(_BERT_STEPS % (False, True, True, 0.0, plain))
    s, p = torch.load(scaled), torch.load(plain)
    assert all(math.isfinite(v) for v in s["losses"]) and s["skipped"] == 0, s["losses"]
    _close(p, s)


@pytest.mark.gpu
def test_bert_tiny_fused_loss_matches_stock_bf16():
    """One bf16 forward + backward of bert_tiny at dropout 0, fused loss against the stock loss with the same
    weights.  Both are compared with the stock model in fp32: the fused loss and every parameter's gradient must be
    as close to it as bf16 allows - within twice the stock bf16 error, or 2 % relative L2, whichever is larger."""
    torch.manual_seed(0)
    stock = bert_tiny(dropout=0.0).cuda()
    fused = bert_tiny(dropout=0.0, fused_loss=True).cuda()
    fused.load_state_dict(stock.state_dict())
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 30522, (8, 128), generator=g).cuda()
    labels = torch.randint(0, 30522, (8, 128), generator=g)
    labels[torch.rand(8, 128, generator=g) > 0.15] = -100
    labels = labels.cuda()

    def grads(model, dtype):
        model = copy.deepcopy(model).to(dtype).train()
        loss = model(ids, mlm_labels=labels)
        loss.backward()
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


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=_dt_id)
@pytest.mark.parametrize("reduction", ["mean", "sum", "none"])
def test_xent_cpu_is_stock(reduction, dtype):
    torch.manual_seed(0)
    x = (torch.randn(40, 77) * 3).to(dtype).requires_grad_(True)
    t = torch.randint(0, 77, (40,))
    t[::5] = IGNORE
    out = softmax_cross_entropy(x, t, reduction=reduction)
    ref = F.cross_entropy(x.float(), t, ignore_index=IGNORE, reduction=reduction)
    assert out.dtype == torch.float32 and torch.equal(out, ref)
    gr = torch.randn_like(ref)
    ga, = torch.autograd.grad(out, x, gr)
    gb, = torch.autograd.grad(ref, x, gr)
    assert ga.dtype == dtype and torch.equal(ga, gb)


def test_xent_rejects_unknown_reduction():
    with pytest.raises(ValueError):
        softmax_cross_entropy(torch.randn(3, 4), torch.zeros(3, dtype=torch.int64), reduction="avg")


def test_bert_fused_loss_keeps_the_stock_parameters_and_loss():
    torch.manual_seed(0)
    stock = bert_tiny()
    fused = bert_tiny(fused_loss=True)
    assert fused.config.fused_loss and not stock.config.fused_loss
    assert [n for n, _ in fused.named_parameters()] == [n for n, _ in stock.named_parameters()]
    ours, theirs = fused.state_dict(), stock.state_dict()
    assert list(ours) == list(theirs)
    assert all(ours[k].shape == theirs[k].shape and ours[k].dtype == theirs[k].dtype for k in ours)
    fused.load_state_dict(theirs, strict=True)
    ids = torch.randint(0, 30522, (2, 16))
    labels = torch.randint(0, 30522, (2, 16))
    labels[0, :5] = -100
    nsp = torch.tensor([0, 1])
    for training in (True, False):
        stock.train(training)
        fused.train(training)
        torch.manual_seed(2)
        a = stock(ids, mlm_labels=labels, nsp_labels=nsp)
        torch.manual_seed(2)
        b = fused(ids, mlm_labels=labels, nsp_labels=nsp)
        assert torch.equal(a, b), training
