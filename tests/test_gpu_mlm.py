"""The labelled-row gather of the masked-LM head (ops/mlm.py, kernels/mlm_gather.cu) and BERT's
max_predictions_per_seq head built on it.

GPU tests compare the kernels bit for bit with the stock expression (ops.mlm._stock): the gather and the scatter copy
bits, so rows, row labels, the dropped count and dx must be identical.  CPU tests check the argument rules, the stock
expression's fallbacks and bert_tiny in float64 against the dense head.
"""
import os
import re
import subprocess

import pytest
import torch

import byteps_b200.ops.mlm as mlm
from byteps_b200.models import bert_tiny
from byteps_b200.ops.mlm import _stock, gather_labelled
from test_gpu_attn import _run_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
FUSED = "_GatherLabelledFnBackward"


def _dt_id(d):
    return str(d).replace("torch.", "")


def _labels(t, share, device="cuda", ignore=-100, seed=0):
    """int64 labels [t]: none, one token, about 15 % or all labelled; some labels lie outside any vocabulary"""
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(-5, 40000, (t,), generator=g)
    lab[lab == ignore] = ignore + 1
    if share == "none":
        lab[:] = ignore
    elif share == "one":
        lab[:] = ignore
        lab[t // 2] = 7
    elif share == "p15":
        lab[torch.rand(t, generator=g) >= 0.15] = ignore
    return lab.to(device)


def _capacities(n, t):
    """below, equal to and above the labelled count n, 1 and past t"""
    return sorted({max(1, n - 3), max(1, n), n + 3, 1, t + 5})


def _both(x, lab, c, ignore=-100):
    """(kernel rows, row_labels, dropped, dx) and the same from the stock expression, with one random drows"""
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    ra, la, da = gather_labelled(xa, lab, c, ignore)
    assert type(ra.grad_fn).__name__ == FUSED, "kernel path not taken"
    rb, lb, db = _stock(xb, lab, c, ignore)
    g = torch.randn(ra.shape, device=x.device, generator=torch.Generator(device=x.device).manual_seed(c)).to(x.dtype)
    ra.backward(g)
    rb.backward(g)
    return (ra, la, da, xa.grad), (rb, lb, db, xb.grad)


def _equal_bits(a, b):
    """same shape, dtype and bits (so NaN payloads and -0.0 count too)"""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.is_floating_point():
        ints = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
        a, b = a.contiguous().view(ints), b.contiguous().view(ints)
    return torch.equal(a, b)


# ---------------------------------------------------------------------------------------------- against stock
@pytest.mark.gpu
@pytest.mark.parametrize("t", [1, 7, 8192, 65539], ids=lambda v: "T%d" % v)
@pytest.mark.parametrize("h", [8, 64, 768, 1024, 1000], ids=lambda v: "H%d" % v)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_matches_stock_expression(dtype, h, t):
    x = torch.randn(t, h, device="cuda", generator=torch.Generator(device="cuda").manual_seed(t + h)).to(dtype)
    for share in ("none", "one", "p15", "all"):
        lab = _labels(t, share, seed=h)
        n = int((lab != -100).sum())
        for c in _capacities(n, t):
            got, ref = _both(x, lab, c)
            for name, a, b in zip(("rows", "row_labels", "dropped", "dx"), got, ref):
                assert _equal_bits(a, b), (share, c, name)
            assert int(got[2]) == max(0, n - c)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_custom_ignore_index_and_leading_shape(dtype):
    b, s, h = 5, 37, 64
    x = torch.randn(b, s, h, device="cuda").to(dtype)
    lab = torch.randint(0, 4, (b, s), device="cuda")   # ignore_index 0; labels -100 count as labelled
    lab[1, 3] = -100
    n = int((lab != 0).sum())
    for c in _capacities(n, b * s):
        got, ref = _both(x, lab, c, ignore=0)
        for a, r in zip(got, ref):
            assert _equal_bits(a, r), c
        assert got[3].shape == (b, s, h)
        assert bool((got[1][n:] == 0).all())


@pytest.mark.gpu
def test_offsets_past_2_to_31_elements():
    """T H just above 2^31: the last rows sit past element 2^31, in both the gather and the scatter."""
    h, dtype = 1024, torch.bfloat16
    t = 2 ** 31 // h + 3
    x = torch.empty(t, h, dtype=dtype, device="cuda")
    x[:16].normal_()
    x[-16:].normal_()
    lab = torch.full((t,), -100, dtype=torch.int64, device="cuda")
    picked = torch.tensor([0, 5, t - 9, t - 2, t - 1], device="cuda")
    lab[picked] = torch.arange(5, device="cuda")
    xr = x.requires_grad_(True)
    rows, row_labels, dropped = gather_labelled(xr, lab, 6)
    assert torch.equal(rows[:5], x.detach()[picked]) and (rows[5] == 0).all()
    assert row_labels.tolist() == [0, 1, 2, 3, 4, -100] and int(dropped) == 0
    g = torch.randn(6, h, device="cuda").to(dtype)
    rows.backward(g)
    dx = xr.grad
    assert torch.equal(dx[picked], g[:5])
    assert int(dx.count_nonzero()) == int(g[:5].count_nonzero())
    del dx, xr, x


# ---------------------------------------------------------------------------------------------- memory
@pytest.mark.gpu
def test_dx_exact_on_nan_filled_memory():
    t, h, dtype = 8192, 1024, torch.bfloat16
    x = torch.randn(t, h, device="cuda").to(dtype).requires_grad_(True)
    lab = _labels(t, "p15")
    rows, _, _ = gather_labelled(x, lab, 2000)
    g = torch.randn_like(rows)
    torch.cuda.synchronize()
    junk = torch.full((t, h), float("nan"), dtype=dtype, device="cuda")
    del junk   # dx reuses this NaN-filled block
    rows.backward(g)
    assert torch.isfinite(x.grad).all()
    xs = x.detach().clone().requires_grad_(True)
    rs, _, _ = _stock(xs, lab, 2000, -100)
    rs.backward(g)
    assert _equal_bits(x.grad, xs.grad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["under", "over"])
def test_buffers_keep_their_bands(case):
    """Every buffer the binding writes sits inside a canary band (and x, labels, drows inside NaN / junk bands)."""
    from byteps_b200 import _native

    cu = _native.cuda()
    t, h, pad = 3000, 64, 64
    c = 1000 if case == "under" else 100
    dt = torch.bfloat16
    canary = 1234.0
    x_b = torch.full((t + 2 * pad, h), float("nan"), dtype=dt, device="cuda")
    x = x_b[pad:pad + t]
    x.copy_(torch.randn(t, h, device="cuda").to(dt))
    lab_b = torch.full((t + 2 * pad,), 3, dtype=torch.int64, device="cuda")
    lab = lab_b[pad:pad + t]
    lab.copy_(_labels(t, "p15"))
    rows_b = torch.full((c + 2 * pad, h), canary, dtype=dt, device="cuda")
    rl_b = torch.full((c + 2 * pad,), 777, dtype=torch.int64, device="cuda")
    slot_b = torch.full((t + 2 * pad,), 777, dtype=torch.int32, device="cuda")
    src_b = torch.full((c + 2 * pad,), 777, dtype=torch.int32, device="cuda")
    drop_b = torch.full((2 * pad + 1,), 777, dtype=torch.int64, device="cuda")
    dx_b = torch.full((t + 2 * pad, h), canary, dtype=dt, device="cuda")
    drows_b = torch.full((c + 2 * pad, h), float("nan"), dtype=dt, device="cuda")
    drows = drows_b[pad:pad + c]
    drows.copy_(torch.randn(c, h, device="cuda").to(dt))
    rows, rl, slot, src = rows_b[pad:pad + c], rl_b[pad:pad + c], slot_b[pad:pad + t], src_b[pad:pad + c]
    dropped, dx = drop_b[pad], dx_b[pad:pad + t]
    st = torch.cuda.current_stream().cuda_stream
    cu.mlm_gather_fwd(x.data_ptr(), lab.data_ptr(), 1, t, h, c, -100, rows.data_ptr(), rl.data_ptr(), slot.data_ptr(),
                      src.data_ptr(), dropped.data_ptr(), st)
    cu.mlm_scatter_bwd(drows.data_ptr(), slot.data_ptr(), 1, t, h, c, dx.data_ptr(), st)
    torch.cuda.synchronize()
    for band in (rows_b[:pad], rows_b[pad + c:], dx_b[:pad], dx_b[pad + t:]):
        assert (band == canary).all()
    for band in (rl_b[:pad], rl_b[pad + c:], slot_b[:pad], slot_b[pad + t:], src_b[:pad], src_b[pad + c:],
                 drop_b[:pad], drop_b[pad + 1:]):
        assert (band == 777).all()
    r, l_, d = _stock(x, lab, c, -100)
    assert _equal_bits(rows, r) and torch.equal(rl, l_) and int(dropped) == int(d)
    xs = x.clone().requires_grad_(True)
    _stock(xs, lab, c, -100)[0].backward(drows)
    assert _equal_bits(dx, xs.grad)


# ---------------------------------------------------------------------------------------------- determinism, graphs
@pytest.mark.gpu
def test_deterministic_and_graph_replays_follow_labels():
    t, h, c, dtype = 8192, 1024, 1400, torch.bfloat16
    x = torch.randn(t, h, device="cuda").to(dtype)
    g = torch.randn(c, h, device="cuda").to(dtype)
    lab_a, lab_b = _labels(t, "p15", seed=1), _labels(t, "all", seed=2)

    def eager(lab):
        xr = x.clone().requires_grad_(True)
        rows, rl, d = gather_labelled(xr, lab, c)
        rows.backward(g)
        return rows.detach(), rl, d, xr.grad

    runs = [eager(lab_a) for _ in range(2)]
    for a, b in zip(*runs):
        assert _equal_bits(a, b)
    ref_b = eager(lab_b)
    assert int(ref_b[2]) == t - c

    lab = lab_a.clone()
    xr = x.clone().requires_grad_(True)
    acc = torch.zeros((), dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            xr.grad = None
            gather_labelled(xr, lab, c)[0].backward(g)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    xr.grad = None
    with torch.cuda.graph(graph):
        rows, rl, d = gather_labelled(xr, lab, c)
        acc.add_(d)
        rows.backward(g)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip((rows, rl, d, xr.grad), runs[0]):
        assert _equal_bits(a.detach(), b)
    assert int(acc) == 0
    lab.copy_(lab_b)   # new positions, refreshed in place
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip((rows, rl, d, xr.grad), ref_b):
        assert _equal_bits(a.detach(), b)
    assert int(acc) == 2 * (t - c)


_LAUNCHES = """
import json
import torch
from torch.profiler import ProfilerActivity, profile
from byteps_b200.ops.mlm import gather_labelled

def launches(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

x = torch.randn(4096, 1024, device="cuda").to(torch.bfloat16).requires_grad_(True)
lab = torch.where(torch.rand(4096, device="cuda") < 0.15, 7, -100)
g = torch.randn(700, 1024, device="cuda").to(torch.bfloat16)
gather_labelled(x, lab, 700)[0].backward(g)
x.grad = None
out = {}
fwd = launches(lambda: out.setdefault("rows", gather_labelled(x, lab, 700)[0]))
bwd = launches(lambda: out["rows"].backward(g))
print(json.dumps({"fwd": fwd, "bwd": bwd}))
"""


@pytest.mark.gpu
def test_launch_count():
    """Two launches forward and one backward, and no memset or fill.  The profiler runs in a process of its own, as
    the other launch counts of the suite do: in the shared test process, earlier profiler sessions can leave it
    recording no CUDA activity at all."""
    import json

    names = json.loads(_run_py(_LAUNCHES).strip().splitlines()[-1])
    fwd, bwd = names["fwd"], names["bwd"]
    assert [n for n in fwd if "mlm_scan_kernel" in n] and [n for n in fwd if "mlm_copy_rows_kernel" in n], fwd
    assert len(fwd) == 2 and len(bwd) == 1 and "mlm_copy_rows_kernel" in bwd[0], (fwd, bwd)


# ---------------------------------------------------------------------------------------------- fallbacks, arguments
def _fallback_case(case, device):
    """(x, labels); for "noncontig" x is the [T, 2H] base of the strided view the op takes"""
    t, h, dtype = 300, 64, torch.bfloat16
    if case == "fp64":
        dtype = torch.float64
    elif case == "h12":
        h = 12     # 24 bytes per bf16 row
    elif case == "h3f32":
        h, dtype = 3, torch.float32
    elif case == "noncontig":
        h *= 2
    x = torch.randn(t, h, generator=torch.Generator().manual_seed(0)).to(dtype).to(device)
    return x, _labels(t, "p15", device=device)


FALLBACKS = ["fp64", "h12", "h3f32", "noncontig"]


def _check_fallback(case, device):
    x, lab = _fallback_case(case, device)
    view = (lambda v: v[:, ::2]) if case == "noncontig" else (lambda v: v)
    n = int((lab != -100).sum())
    for c in (n - 5, n + 5):
        xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        ra, la, da = gather_labelled(view(xa), lab, c)
        assert type(ra.grad_fn).__name__ != FUSED
        rb, lb, db = _stock(view(xb), lab, c, -100)
        assert torch.equal(ra, rb) and torch.equal(la, lb) and torch.equal(da, db)
        assert int(da) == max(0, n - c)
        g = torch.randn_like(ra)
        ra.backward(g)
        rb.backward(g)
        assert torch.equal(xa.grad, xb.grad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FALLBACKS)
def test_fallbacks_are_stock_cuda(case):
    _check_fallback(case, "cuda")


@pytest.mark.parametrize("case", FALLBACKS + ["bf16"])
def test_fallbacks_are_stock_cpu(case):
    _check_fallback(case, "cpu")


def test_stock_expression_selects_in_token_order():
    x = torch.arange(12.0).view(6, 2)
    lab = torch.tensor([-100, 4, -100, 9, 9, -1])
    rows, rl, d = gather_labelled(x, lab, 5)
    assert rows.tolist() == [[2, 3], [6, 7], [8, 9], [10, 11], [0, 0]]
    assert rl.tolist() == [4, 9, 9, -1, -100] and int(d) == 0
    rows, rl, d = gather_labelled(x, lab, 2)
    assert rows.tolist() == [[2, 3], [6, 7]] and rl.tolist() == [4, 9] and int(d) == 2


def test_bad_arguments_raise():
    x = torch.zeros(4, 6, 16)
    lab = torch.zeros(4, 6, dtype=torch.int64)
    for args in [(x, lab.view(24), 4), (x, lab[:, :5], 4), (x, lab.int(), 4), (x, lab.float(), 4), (x, lab, 0),
                 (x, lab, -3), (x, lab, 2.0), (x, lab, True), (torch.zeros(()), torch.zeros((), dtype=torch.int64), 1)]:
        with pytest.raises(ValueError):
            gather_labelled(*args)


@pytest.mark.gpu
def test_binding_rejects_bad_arguments():
    from byteps_b200 import _native

    cu = _native.cuda()
    buf = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")
    i64 = torch.zeros(1 << 12, dtype=torch.int64, device="cuda")
    b, l = buf.data_ptr(), i64.data_ptr()
    ok = dict(x=b, labels=l, dtype=1, T=8, H=64, C=4, rows=b, row_labels=l, slot=l, src=l, dropped=l)
    cases = [dict(dtype=3), dict(dtype=-1), dict(T=0), dict(T=2 ** 31), dict(H=0), dict(H=12), dict(dtype=0, H=2),
             dict(C=0), dict(C=2 ** 31), dict(x=0), dict(x=b + 8), dict(rows=b + 4), dict(labels=l + 4),
             dict(row_labels=0), dict(dropped=l + 2), dict(slot=l + 2), dict(src=0)]
    for bad in cases:
        a = dict(ok, **bad)
        with pytest.raises(ValueError):
            cu.mlm_gather_fwd(a["x"], a["labels"], a["dtype"], a["T"], a["H"], a["C"], -100, a["rows"],
                              a["row_labels"], a["slot"], a["src"], a["dropped"], 0)
    bwd = dict(drows=b, slot=l, dtype=1, T=8, H=64, C=4, dx=b)
    for bad in [dict(dtype=5), dict(T=0), dict(H=4), dict(C=0), dict(drows=b + 8), dict(dx=0), dict(slot=l + 1)]:
        a = dict(bwd, **bad)
        with pytest.raises(ValueError):
            cu.mlm_scatter_bwd(a["drows"], a["slot"], a["dtype"], a["T"], a["H"], a["C"], a["dx"], 0)


# ---------------------------------------------------------------------------------------------- build
def test_mlm_kernels_compile_without_spills(tmp_path):
    from byteps_b200 import _build

    nvcc = _build._nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "byteps_b200", "csrc", "kernels", "mlm_gather.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + _build.ARCH_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                                         str(tmp_path / "mlm_gather.o")],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    found = 0
    for block in r.stderr.split("Compiling entry function '")[1:]:
        if not re.match(r"_ZN\S*mlm_(scan|copy_rows)_kernel", block):
            continue
        found += 1
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block[:400]
    assert found == 2, found


# ---------------------------------------------------------------------------------------------- model, CPU
def _pair(k, **kw):
    """a dense bert_tiny in float64 and the same weights with max_predictions_per_seq = k"""
    torch.manual_seed(0)
    dense = bert_tiny(dropout=0.0, **kw).double()
    sparse = bert_tiny(dropout=0.0, max_predictions_per_seq=k, **kw).double()
    sparse.load_state_dict(dense.state_dict())
    assert list(sparse.state_dict()) == list(dense.state_dict())
    return dense, sparse


def _batch(b, s, share=0.15, seed=1):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 1000, (b, s), generator=g)
    labels = torch.where(torch.rand(b, s, generator=g) < share, torch.randint(0, 30522, (b, s), generator=g),
                         torch.full((b, s), -100))
    nsp = torch.randint(0, 2, (b,), generator=g)
    return ids, labels, nsp


def _loss_grads(model, ids, labels, nsp, **kw):
    model.zero_grad()
    loss = model(ids, mlm_labels=labels, nsp_labels=nsp, **kw)
    loss.backward()
    return loss.detach(), {n: p.grad.clone() for n, p in model.named_parameters()}


def _close(a, b, rel=1e-10):
    return (a - b).abs().max().item() <= rel * max(b.abs().max().item(), 1e-300)


def _close_loss(a, b):
    """the model takes both losses in fp32 (F.cross_entropy of logits.float()), summing the dense head's 8x more rows
    in another order: equal within a few fp32 units"""
    return (a - b).abs().item() <= 4 * 2.0 ** -24 * b.abs().item()


@pytest.mark.parametrize("fused_loss", [False, True], ids=["stock_loss", "fused_loss"])
def test_bert_sparse_head_matches_dense_cpu(fused_loss):
    b, s = 4, 32
    dense, sparse = _pair(10, fused_loss=fused_loss)
    ids, labels, nsp = _batch(b, s)
    assert int((labels != -100).sum()) <= b * 10
    ld, gd = _loss_grads(dense, ids, labels, nsp)
    ls, gs = _loss_grads(sparse, ids, labels, nsp)
    assert _close_loss(ls, ld)
    for n in gd:
        assert _close(gs[n], gd[n]), n
    assert int(sparse.mlm_dropped_targets) == 0
    assert "mlm_dropped_targets" not in sparse.state_dict()


def test_bert_sparse_head_overflow_cpu():
    b, s, k = 3, 24, 2
    dense, sparse = _pair(k)
    ids, labels, nsp = _batch(b, s, share=0.3)
    flat = labels.view(-1)
    pos = (flat != -100).nonzero().squeeze(1)
    assert pos.numel() > b * k
    kept = flat.clone()
    kept[pos[b * k:]] = -100
    ld, gd = _loss_grads(dense, ids, kept.view(b, s), nsp)
    ls, gs = _loss_grads(sparse, ids, labels, nsp)
    assert _close_loss(ls, ld)
    for n in gd:
        assert _close(gs[n], gd[n]), n
    over = pos.numel() - b * k
    assert int(sparse.mlm_dropped_targets) == over
    sparse(ids, mlm_labels=labels)
    assert int(sparse.mlm_dropped_targets) == 2 * over


def test_bert_sparse_head_all_ignored_and_no_labels_cpu():
    b, s = 2, 16
    dense, sparse = _pair(4)
    ids, _, _ = _batch(b, s)
    none = torch.full((b, s), -100)
    assert torch.isnan(dense(ids, mlm_labels=none)) and torch.isnan(sparse(ids, mlm_labels=none))
    ld, nd = dense(ids)
    ls, ns = sparse(ids)
    assert torch.equal(ld, ls) and torch.equal(nd, ns)
    assert ls.shape == (b, s, 30522)


def test_bert_sparse_head_packed_cpu():
    b, s = 3, 24
    dense, sparse = _pair(6)
    ids, labels, _ = _batch(b, s, share=0.2, seed=4)
    cu = torch.tensor([2, 20, 31, 31, 60, 70], dtype=torch.int32)   # tokens outside every sequence at both ends
    nsp = torch.tensor([0, 1, -100, 1, 0])
    ld, gd = _loss_grads(dense, ids, labels, nsp, cu_seqlens=cu, max_seqlen=s + 6)
    ls, gs = _loss_grads(sparse, ids, labels, nsp, cu_seqlens=cu, max_seqlen=s + 6)
    assert _close_loss(ls, ld)
    for n in gd:
        assert _close(gs[n], gd[n]), n
    assert int(sparse.mlm_dropped_targets) == 0


# ---------------------------------------------------------------------------------------------- model, GPU
_BERT_GRAPHED = """
import torch
import byteps_b200.ops.mlm as mlm
from byteps_b200.models import bert_tiny
PACKED, OPTS, OUT = %r, %r, %r
torch.manual_seed(0)
model = bert_tiny(dropout=0.0, max_predictions_per_seq=24, **OPTS).cuda().to(torch.bfloat16).train()
g = torch.Generator().manual_seed(1)
b, s = 8, 128
ids = torch.randint(0, 1000, (b, s), generator=g).cuda()
lengths = torch.randint(16, 129, (b,), generator=g)
attend = torch.arange(s)[None, :] < lengths[:, None]
labels = torch.where(attend & (torch.rand(b, s, generator=g) < 0.15), torch.randint(0, 30522, (b, s), generator=g),
                     torch.full((b, s), -100)).cuda()
mask = attend.view(b, 1, 1, s).cuda()
cu = [0]
for n in lengths.tolist():
    cu += [cu[-1] + n, cu[-1] + s]
cu = torch.tensor(cu, dtype=torch.int32).cuda()

def fwd_bwd():
    model.zero_grad(set_to_none=False)
    if PACKED:
        loss = model(ids, cu_seqlens=cu, max_seqlen=s, mlm_labels=labels)
    else:
        loss = model(ids, mask=mask, mlm_labels=labels)
    loss.backward()
    return loss

for p in model.parameters():
    p.grad = torch.zeros_like(p)
side = torch.cuda.Stream()
side.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(side):
    for _ in range(2):
        fwd_bwd()
torch.cuda.current_stream().wait_stream(side)
graph = torch.cuda.CUDAGraph()
with torch.cuda.graph(graph):
    loss = fwd_bwd()
model.mlm_dropped_targets.zero_()
# the graph and the eager step below start from the same FP8 scaling state
fp8 = [m._fp8.buf for m in model.modules() if getattr(m, "_fp8", None) is not None]
saved = [b.clone() for b in fp8]
graph.replay()
torch.cuda.synchronize()
got = (loss.detach().clone(), {n: p.grad.clone() for n, p in model.named_parameters()})
for b, v in zip(fp8, saved):
    b.copy_(v)
fused = mlm._fusable
mlm._fusable = lambda *a: False
ref_loss = fwd_bwd().detach()
ref = {n: p.grad.clone() for n, p in model.named_parameters()}
mlm._fusable = fused
assert torch.equal(got[0], ref_loss), (got[0], ref_loss)
for n in ref:
    assert torch.equal(got[1][n], ref[n]), n
assert int(model.mlm_dropped_targets) == 0
print("OK")
"""


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
@pytest.mark.parametrize("opts", ["alone", "fused_loss", "all"])
def test_bert_tiny_graphed_equals_eager_stock_gather(tmp_path, packed, opts):
    """bert_tiny in bf16, forward and backward captured in one CUDA graph, gives the loss and parameter gradients of
    the same model run eagerly with the stock gather expression, bit for bit (the head's GEMMs have the same
    shapes on both sides).  Attention is the fused kernel throughout: its backward is deterministic, where SDPA's
    memory-efficient and flash backwards are not."""
    kw = {"alone": {}, "fused_loss": dict(fused_loss=True),
          "all": dict(fused_loss=True, fused_norm=True, fp8_linear=True)}[opts]
    kw = dict(kw, fused_attention=True)
    assert "OK" in _run_py(_BERT_GRAPHED % (packed, kw, str(tmp_path / "o.pt")))


_BERT_TRACK = """
import torch
import byteps_b200.torch as bps
from byteps_b200.models import bert_tiny
from byteps_b200.torch.graph import GraphedStep
K, PACKED, STEPS, OUT = %r, %r, %r, %r
bps.init()
torch.manual_seed(0)
model = bert_tiny(dropout=0.0, max_predictions_per_seq=K, fused_loss=True, fused_norm=True, fused_attention=True,
                  fp8_linear=True).cuda().to(torch.bfloat16).train()
opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=0.01),
                               named_parameters=model.named_parameters(), fused_update=True)
g = torch.Generator().manual_seed(1)
b, s = 8, 128
ids = torch.randint(0, 1000, (b, s), generator=g).cuda()
labels = torch.where(torch.rand(b, s, generator=g) < 0.15, torch.randint(0, 1000, (b, s), generator=g),
                     torch.full((b, s), -100)).cuda()
cu = torch.tensor([0, 300, 301, 700, 1024], dtype=torch.int32).cuda()

def step():
    opt.zero_grad()
    if PACKED:
        loss = model(ids, cu_seqlens=cu, max_seqlen=512, mlm_labels=labels)
    else:
        loss = model(ids, mlm_labels=labels)
    loss.backward()
    opt.step()
    return loss

stepper = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams)
losses = [stepper().detach().float().item() for _ in range(STEPS)]
torch.save({"losses": losses, "dropped": int(model.mlm_dropped_targets)}, OUT)
print("OK")
bps.shutdown()
"""


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
def test_bert_tiny_graphed_sparse_head_tracks_dense(tmp_path, packed):
    """300 graphed bf16 steps with every fused option and fused AdamW: the sparse head's losses track the dense
    head's, which sees the same labels."""
    runs = {}
    for k in (0, 40):
        out = str(tmp_path / ("%d.pt" % k))
        assert "OK" in _run_py(_BERT_TRACK % (k, packed, 300, out))
        runs[k] = torch.load(out)
    assert runs[40]["dropped"] == 0
    d, sp = torch.tensor(runs[0]["losses"]), torch.tensor(runs[40]["losses"])
    assert torch.isfinite(sp).all()
    assert ((d - sp).abs() <= 0.05 * d.abs() + 0.05).all(), (runs[0]["losses"][::30], runs[40]["losses"][::30])
    assert sp[-20:].mean() < 0.5 * sp[:5].mean()


def test_bert_example_with_max_predictions_per_seq(monkeypatch):
    """The example's CPU run (--no-cuda, two processes over gloo) with the sparse head.  The processes see no GPU, so
    on a machine with one they do not both claim it through NCCL."""
    from test_examples import _torchrun

    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", "")
    out = _torchrun("train_bert_byteps.py", "--no-cuda", "--model", "bert_tiny", "--batch-size", "2", "--seq-len", "16",
                    "--steps", "2", "--warmup-steps", "1", "--max-predictions-per-seq", "4")
    assert "tokens/sec" in out
