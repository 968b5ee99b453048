"""Fused self-attention (ops/attn.py, kernels/attn.cu).

GPU tests compare the fused kernels with a float64 reference that applies the same mask and the same dropout bits
(generated here by a NumPy Philox4x32-10 of the documented indexing, which a separate test checks bit for bit against
the bits the kernel applied).  The bounds follow the kernels' rounding steps, with u the unit roundoff of the
activation dtype: the probabilities are rounded once before P V, dS once before dS K and dS^T Q, delta is formed from
the rounded output, and every output is rounded once; the fp32 sums and exp2 add errors far below u.  So each result
is within 4 u of the sum of the magnitudes that enter it, plus 2 u of itself.  At p = 0 the fused error must also be
at most twice that of torch's SDPA on the same inputs.

CPU tests (no marker) check that BERT with ``fused_attention=True`` keeps the stock model's parameters and
state_dict, and that every input the kernels do not take runs the stock expression.
"""
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from byteps_b200.models import bert_tiny
from byteps_b200.ops.attn import _stock, self_attention

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
TINY = {torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24}
DTYPES = [torch.bfloat16, torch.float16]


def _dt_id(d):
    return str(d).replace("torch.", "")


# ---------------------------------------------------------------------------------------------- NumPy Philox
_M32 = np.uint64(0xFFFFFFFF)


def _philox(c0, c1, c2, c3, k0, k1):
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return c0, c1, c2, c3


def _keep_bits(seed, offset, shape, p):
    """keep mask of the attention matrix [B, H, S, S]: element i kept when word i % 4 of Philox with counter
    (i / 4, offset) and key seed is below (1 - p) 2^32."""
    n = int(np.prod(shape))
    g = np.arange((n + 3) // 4, dtype=np.uint64)
    sd, of = np.uint64(seed), np.uint64(offset)
    full = lambda v: np.full_like(g, v)   # noqa: E731
    r = _philox(g & _M32, g >> np.uint64(32), full(of & _M32), full(of >> np.uint64(32)), np.uint64(sd & _M32),
                np.uint64(sd >> np.uint64(32)))
    words = np.stack(r, -1).reshape(-1)[:n]
    keep = min(int(round((1.0 - p) * 2.0 ** 32)), 2 ** 32 - 1)
    return torch.from_numpy(words < np.uint64(keep)).reshape(shape)


def _drawn_seed(rng_seed):
    """the (seed, offset) pair a fused call draws first after torch.manual_seed(rng_seed)"""
    torch.manual_seed(rng_seed)
    s = torch.randint(0, 2 ** 62, (2,), dtype=torch.int64, device="cuda").tolist()
    return s[0], s[1]


# ---------------------------------------------------------------------------------------------- reference
def _reference(qkv, h, mask, keep, p, dout):
    """float64 output, d(qkv) and magnitude bounds of softmax(Q K^T / 8 + mask) -> dropout(keep) -> @ V."""
    b, s, e3 = qkv.shape
    d = e3 // (3 * h)
    x = qkv.detach().double().requires_grad_(True)
    q, k, v = x.view(b, s, 3, h, d).permute(2, 0, 3, 1, 4)
    sc = q @ k.transpose(-1, -2) / d ** 0.5
    if mask is not None:
        am = mask.double() if mask.dtype != torch.bool else torch.where(mask, 0.0, float("-inf")).double()
        sc = sc + am
    m = sc.detach().amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    ex = torch.exp(sc - m)
    den = ex.sum(-1, keepdim=True)
    pr = ex / torch.where(den > 0, den, torch.ones_like(den))
    scale = 1.0 / (1.0 - p)
    pd = pr * keep.double() * scale if keep is not None else pr
    o = pd @ v
    out = o.transpose(1, 2).reshape(b, s, e3 // 3)
    out.backward(dout.double())
    with torch.no_grad():
        do = dout.double().view(b, s, h, d).transpose(1, 2)
        pa, ka, qa, va, doa = pr.abs(), k.abs(), q.abs(), v.abs(), do.abs()
        pda = pd.abs()
        mag_o = pda @ va
        mag_dv = pda.transpose(-1, -2) @ doa
        dp_mag = (doa @ va.transpose(-1, -2)) * (keep.double() * scale if keep is not None else 1.0)
        delta_mag = (doa * mag_o).sum(-1, keepdim=True)
        ds_mag = pa * (dp_mag + delta_mag)
        mag_dq = ds_mag @ ka / d ** 0.5
        mag_dk = ds_mag.transpose(-1, -2) @ qa / d ** 0.5
        mags = torch.stack([mag_dq, mag_dk, mag_dv]).permute(1, 3, 0, 2, 4).reshape(b, s, e3)
        return out.detach(), x.grad, mag_o.transpose(1, 2).reshape(b, s, e3 // 3), mags


def _lengths(b, s, g):
    """key-padding lengths: 1 for batch 0, all masked for batch 1, random for the rest"""
    ln = torch.randint(1, s + 1, (b,), generator=g)
    ln[0] = 1
    if b > 1:
        ln[1] = 0
    return ln


def _make_mask(kind, b, s, dtype, g):
    if kind == "none":
        return None
    attend = torch.arange(s)[None, :] < _lengths(b, s, g)[:, None]
    if kind == "bool":
        return attend.view(b, 1, 1, s).cuda()
    add = torch.randint(-4, 5, (b, s), generator=g).double() * 0.25
    add = torch.where(attend, add, torch.full_like(add, float("-inf")))
    return add.view(b, 1, 1, s).to(dtype).cuda()


def _make(b, s, h, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = (torch.randn(b, s, 3 * h * 64, device="cuda", generator=g, dtype=torch.float64) * 1.5).to(dtype)
    dout = torch.randn(b, s, h * 64, device="cuda", generator=g, dtype=torch.float64).to(dtype)
    return qkv, dout


def _fused(qkv, h, mask, p, dout, rng_seed=1234):
    x = qkv.detach().clone().requires_grad_(True)
    torch.manual_seed(rng_seed)
    out = self_attention(x, h, mask, p, True)
    assert type(out.grad_fn).__name__ == "_SelfAttentionFnBackward", "fused path not taken"
    out.backward(dout)
    return out.detach(), x.grad


def _stock_run(qkv, h, mask, dout):
    x = qkv.detach().clone().requires_grad_(True)
    out = _stock(x, h, mask, 0.0)
    out.backward(dout)
    return out.detach(), x.grad


SHAPES = [(3, 1, 2), (3, 17, 2), (3, 64, 2), (3, 100, 2), (64, 128, 16), (3, 384, 2), (2, 512, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1], ids=["p0", "p01"])
@pytest.mark.parametrize("mask_kind", ["none", "bool", "add"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda t: "x".join(map(str, t)))
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_matches_float64(dtype, shape, mask_kind, p):
    b, s, h = shape
    g = torch.Generator().manual_seed(b * 1000 + s)
    qkv, dout = _make(b, s, h, dtype, seed=s)
    mask = _make_mask(mask_kind, b, s, dtype, g)
    keep = None
    if p > 0:
        keep = _keep_bits(*_drawn_seed(1234), (b, h, s, s), p).cuda()
    out, dqkv = _fused(qkv, h, mask, p, dout)
    out_ref, dqkv_ref, mag_o, mags = _reference(qkv, h, mask, keep, p, dout)
    u = UNIT[dtype]
    err_o = (out.double() - out_ref).abs()
    tol_o = 4 * u * mag_o + 2 * u * out_ref.abs() + TINY[dtype]
    assert (err_o <= tol_o).all(), "out: worst excess %g" % (err_o - tol_o).max().item()
    err_d = (dqkv.double() - dqkv_ref).abs()
    tol_d = 4 * u * mags + 2 * u * dqkv_ref.abs() + TINY[dtype]
    assert (err_d <= tol_d).all(), "dqkv: worst excess %g" % (err_d - tol_d).max().item()
    if mask is not None:
        # masked keys: exactly zero dK and dV; fully masked rows (batch 1): zero output and dQ
        attend = (mask if mask.dtype == torch.bool else torch.isfinite(mask)).view(b, s).cpu()
        e = h * 64
        for bi in range(b):
            dead = ~attend[bi]
            assert (dqkv[bi, dead.cuda(), e:] == 0).all()
        if b > 1:
            assert (out[1] == 0).all() and (dqkv[1, :, :e] == 0).all()
    if p == 0:
        so, sd = _stock_run(qkv, h, mask, dout)
        live = torch.ones(b, dtype=torch.bool, device="cuda")
        if mask is not None:
            live[1] = False   # fully masked: compared with zeros above
        es_o = (so.double() - out_ref)[live].abs().max().item()
        es_d = (sd.double() - dqkv_ref)[live].abs().max().item()
        ef_o = err_o[live].max().item()
        ef_d = err_d[live].max().item()
        floor_o = u * out_ref.abs().max().item()
        floor_d = u * dqkv_ref.abs().max().item()
        assert ef_o <= max(2 * es_o, floor_o), (ef_o, es_o)
        assert ef_d <= max(2 * es_d, floor_d), (ef_d, es_d)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["bool", "add"])
def test_fully_masked_rows_are_zero_like_sdpa(kind):
    """A batch element whose keys are all masked gives zero output and zero d(qkv), as torch's SDPA does on the CPU
    and, with an additive mask, on CUDA.  (On CUDA with a bool mask the stock expression does not give zeros.)"""
    b, s, h = 2, 100, 2
    qkv, dout = _make(b, s, h, torch.bfloat16)
    attend = torch.ones(b, s, dtype=torch.bool)
    attend[0] = False
    mask = attend if kind == "bool" else torch.where(attend, 0.0, float("-inf"))
    mask = mask.view(b, 1, 1, s)
    if kind == "add":
        mask = mask.to(torch.bfloat16)
    runs = [_fused(qkv, h, mask.cuda(), 0.0, dout), _stock_run(qkv.cpu(), h, mask, dout.cpu())]
    if kind == "add":
        runs.append(_stock_run(qkv, h, mask.cuda(), dout))
    for out, dq in runs:
        assert (out[0] == 0).all() and (dq[0] == 0).all()
        assert torch.isfinite(out).all() and torch.isfinite(dq).all()


@pytest.mark.gpu
def test_fp32_and_bf16_additive_masks_agree():
    b, s, h = 3, 100, 2
    qkv, dout = _make(b, s, h, torch.bfloat16)
    g = torch.Generator().manual_seed(5)
    m16 = _make_mask("add", b, s, torch.bfloat16, g)
    a = _fused(qkv, h, m16, 0.0, dout)
    c = _fused(qkv, h, m16.float(), 0.0, dout)
    c1 = _fused(qkv, h, m16[:1].float(), 0.0, dout)
    a1 = _fused(qkv, h, m16[:1].expand(b, 1, 1, s), 0.0, dout)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
    assert torch.equal(c1[0], a1[0]) and torch.equal(c1[1], a1[1])


# ---------------------------------------------------------------------------------------------- dropout
def _extract_bits(b, s, h, p, rng_seed, dtype=torch.bfloat16):
    """Keep bits of the whole attention matrix read from the output: Q = K = 0 makes P uniform, and V one-hot on the
    keys of a 64-key window makes O[q, j] nonzero exactly when (q, key w0 + j) is kept.  One call per window, each
    after torch.manual_seed(rng_seed), so all use the same (seed, offset)."""
    e = h * 64
    bits = torch.zeros(b, h, s, s, dtype=torch.bool)
    for w0 in range(0, s, 64):
        qkv = torch.zeros(b, s, 3, h, 64, dtype=dtype, device="cuda")
        n = min(64, s - w0)
        idx = torch.arange(n, device="cuda")
        qkv[:, w0 + idx, 2, :, idx] = 1.0
        torch.manual_seed(rng_seed)
        out = self_attention(qkv.view(b, s, 3 * e), h, None, p, True).view(b, s, h, 64)
        bits[..., w0:w0 + n] = (out[..., :n] != 0).permute(0, 2, 1, 3).cpu()
    return bits


@pytest.mark.gpu
@pytest.mark.parametrize("s", [17, 100, 128], ids=lambda v: "S%d" % v)
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout_bits_are_philox(s, p):
    b, h = 2, 3
    bits = _extract_bits(b, s, h, p, rng_seed=77)
    ref = _keep_bits(*_drawn_seed(77), (b, h, s, s), p)
    assert torch.equal(bits, ref)
    n = bits.numel()
    frac = bits.double().mean().item()
    sigma = (p * (1 - p) / n) ** 0.5
    assert abs(frac - (1 - p)) <= 5 * sigma, (frac, 1 - p, sigma)


@pytest.mark.gpu
def test_backward_uses_the_forward_mask():
    """dV of the one-hot read-out against the float64 reference built from the bits the forward applied."""
    b, s, h, p = 2, 100, 2, 0.1
    bits = _extract_bits(b, s, h, p, rng_seed=9)
    e = h * 64
    qkv = torch.zeros(b, s, 3, h, 64, dtype=torch.bfloat16, device="cuda")
    qkv[:, :, 2] = torch.randn(b, s, h, 64, device="cuda").to(torch.bfloat16)
    dout = torch.randn(b, s, e, device="cuda").to(torch.bfloat16)
    x = qkv.view(b, s, 3 * e).clone().requires_grad_(True)
    torch.manual_seed(9)
    out = self_attention(x, h, None, p, True)
    out.backward(dout)
    pd = bits.double().cuda() / (1 - p) / s                      # [b, h, q, k]
    do = dout.double().view(b, s, h, 64).transpose(1, 2)          # [b, h, q, d]
    dv_ref = (pd.transpose(-1, -2) @ do).transpose(1, 2)          # [b, k, h, d]
    dv = x.grad.view(b, s, 3, h, 64)[:, :, 2].double()
    mag = (pd.transpose(-1, -2) @ do.abs()).transpose(1, 2)
    u = UNIT[torch.bfloat16]
    assert ((dv - dv_ref).abs() <= 4 * u * mag + 2 * u * dv_ref.abs()).all()
    o_ref = (pd @ qkv[:, :, 2].double().transpose(1, 2)).transpose(1, 2).reshape(b, s, e)
    assert ((out.double() - o_ref).abs() <= 4 * u * (pd @ qkv[:, :, 2].double().abs().transpose(1, 2)).transpose(1, 2).reshape(b, s, e) + 2 * u * o_ref.abs()).all()


@pytest.mark.gpu
def test_dropout_follows_the_generator():
    b, s, h = 2, 100, 2
    qkv, _ = _make(b, s, h, torch.bfloat16)
    torch.manual_seed(3)
    a = self_attention(qkv, h, None, 0.1, True)
    c = self_attention(qkv, h, None, 0.1, True)
    torch.manual_seed(3)
    a2 = self_attention(qkv, h, None, 0.1, True)
    assert torch.equal(a, a2) and not torch.equal(a, c)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["p0", "eval"])
def test_no_draw_without_dropout(case):
    qkv, dout = _make(2, 64, 2, torch.bfloat16)
    x = qkv.clone().requires_grad_(True)
    before = torch.cuda.get_rng_state()
    out = self_attention(x, 2, None, 0.0 if case == "p0" else 0.1, case == "p0")
    out.backward(dout)
    torch.cuda.synchronize()
    assert type(out.grad_fn).__name__ == "_SelfAttentionFnBackward"
    assert torch.equal(before, torch.cuda.get_rng_state())


@pytest.mark.gpu
def test_deterministic_and_graph_replays_match_eager():
    b, s, h, p = 4, 200, 4, 0.1
    qkv, dout = _make(b, s, h, torch.bfloat16)
    mask = _make_mask("bool", b, s, torch.bfloat16, torch.Generator().manual_seed(0))
    runs = [_fused(qkv, h, mask, p, dout, rng_seed=11) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])

    x = qkv.clone().requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            x.grad = None
            self_attention(x, h, mask, p, True).backward(dout)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    x.grad = None
    with torch.cuda.graph(graph):
        out = self_attention(x, h, mask, p, True)
        out.backward(dout)
    torch.manual_seed(11)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, runs[0][0]) and torch.equal(x.grad, runs[0][1])
    first = out.clone()
    graph.replay()
    torch.cuda.synchronize()
    assert not torch.equal(out, first)


# ---------------------------------------------------------------------------------------------- fallbacks
def _fallback_case(case, device):
    b, s, h, d, dtype = 2, 40, 2, 64, torch.bfloat16
    mask = None
    if case == "fp32":
        dtype = torch.float32
    elif case in ("d32", "d128"):
        d = int(case[1:])
    elif case == "s513":
        s = 513
    g = torch.Generator().manual_seed(0)
    qkv = (torch.randn(b, s, 3 * h * d, generator=g)).to(dtype).to(device)
    if case == "square_mask":
        mask = (torch.rand(b, 1, s, s, generator=g) > 0.3).to(device)
    elif case == "grad_mask":
        mask = torch.zeros(b, 1, 1, s, dtype=dtype, device=device).requires_grad_(True)
    elif case == "noncontig":
        qkv = torch.randn(b, s, 2 * 3 * h * d, generator=g).to(dtype).to(device)
    return qkv, h, mask


FALLBACKS = ["fp32", "d32", "d128", "s513", "square_mask", "grad_mask", "noncontig"]


def _check_fallback(case, device):
    qkv, h, mask = _fallback_case(case, device)
    x1, x2 = qkv.clone().requires_grad_(True), qkv.clone().requires_grad_(True)
    view = (lambda t: t[..., ::2]) if case == "noncontig" else (lambda t: t)
    assert not view(x1).is_contiguous() or case != "noncontig"
    a = self_attention(view(x1), h, mask, 0.0, True)
    assert type(a.grad_fn).__name__ != "_SelfAttentionFnBackward"
    ref = _stock(view(x2), h, mask, 0.0)
    assert torch.equal(a, ref)
    g = torch.randn_like(a)
    a.backward(g)
    ref.backward(g)
    if device == "cpu":
        assert torch.equal(x1.grad, x2.grad)
    else:   # the flash and efficient SDPA backwards sum dQ with atomics, so two stock runs may differ in the last bit
        assert (x1.grad - x2.grad).abs().max() <= 2.0 ** -7 * x2.grad.abs().max()


@pytest.mark.gpu
@pytest.mark.parametrize("case", FALLBACKS)
def test_fallbacks_are_stock_cuda(case):
    _check_fallback(case, "cuda")


@pytest.mark.parametrize("case", FALLBACKS + ["bf16"])
def test_fallbacks_are_stock_cpu(case):
    _check_fallback(case, "cpu")


@pytest.mark.gpu
def test_misaligned_view_matches_aligned_copy():
    b, s, h = 2, 100, 2
    qkv, dout = _make(b, s, h, torch.bfloat16)
    flat = torch.empty(qkv.numel() + 1, dtype=qkv.dtype, device="cuda")
    view = flat[1:].view_as(qkv)
    view.copy_(qkv)
    assert view.data_ptr() % 16 != 0
    a = _fused(view, h, None, 0.1, dout, rng_seed=5)
    c = _fused(qkv, h, None, 0.1, dout, rng_seed=5)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


def test_bad_arguments_raise():
    with pytest.raises(ValueError):
        self_attention(torch.zeros(2, 3, 10), 2)
    with pytest.raises(ValueError):
        self_attention(torch.zeros(2, 3, 384), 2, p=1.5)


@pytest.mark.gpu
def test_binding_rejects_bad_arguments():
    from byteps_b200 import _native

    cu = _native.cuda()
    buf = torch.zeros(1 << 20, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(1 << 16, device="cuda")
    for dtype, d, s in [(0, 64, 8), (1, 32, 8), (1, 64, 0), (1, 64, 513)]:
        with pytest.raises(ValueError):
            cu.attn_fwd(buf.data_ptr(), dtype, 1, s, 1, d, 0, 0, 0, 0, 0, 1.0, buf.data_ptr(), lse.data_ptr(), 0)


# ---------------------------------------------------------------------------------------------- build
def test_attention_kernels_compile_without_spills(tmp_path):
    from byteps_b200 import _build

    nvcc = _build._nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "byteps_b200", "csrc", "kernels", "attn.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + _build.ARCH_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                                         str(tmp_path / "attn.o")],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    found = 0
    for block in r.stderr.split("Compiling entry function '")[1:]:
        if not re.match(r"_ZN\S*attn_(fwd|bwd_dq|bwd_dkv)_kernel", block):
            continue
        found += 1
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block[:400]
    assert found == 12, found


# ---------------------------------------------------------------------------------------------- model
def test_bert_fused_attention_keeps_the_stock_parameters():
    torch.manual_seed(0)
    stock = bert_tiny()
    fused = bert_tiny(fused_attention=True)
    assert all(layer.fused_attention for layer in fused.layers)
    assert [n for n, _ in fused.named_parameters()] == [n for n, _ in stock.named_parameters()]
    ours, theirs = fused.state_dict(), stock.state_dict()
    assert list(ours) == list(theirs)
    assert all(ours[k].shape == theirs[k].shape and ours[k].dtype == theirs[k].dtype for k in ours)
    fused.load_state_dict(theirs, strict=True)
    stock.load_state_dict(fused.state_dict(), strict=True)


def test_bert_fused_attention_cpu_is_stock():
    torch.manual_seed(0)
    stock = bert_tiny()
    fused = bert_tiny(fused_attention=True)
    fused.load_state_dict(stock.state_dict())
    ids = torch.randint(0, 30522, (2, 16))
    labels = torch.randint(0, 30522, (2, 16))
    mask = torch.ones(2, 1, 1, 16, dtype=torch.bool)
    mask[1, ..., 9:] = False
    for training in (True, False):
        stock.train(training)
        fused.train(training)
        torch.manual_seed(2)
        a = stock(ids, mask=mask, mlm_labels=labels)
        torch.manual_seed(2)
        c = fused(ids, mask=mask, mlm_labels=labels)
        assert torch.equal(a, c), training


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
FUSED, ALL, DROPOUT, STEPS, OUT = %r, %r, %r, %r, %r
bps.init()
torch.manual_seed(0)
kw = dict(fp8_linear=True, fused_norm=True, fused_loss=True) if ALL else {}
model = bert_tiny(fused_attention=FUSED, dropout=DROPOUT, **kw).cuda().to(torch.bfloat16).train()
opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=0.01),
                               named_parameters=model.named_parameters(), fused_update=True)
g = torch.Generator().manual_seed(1)
ids = torch.randint(0, 1000, (8, 128), generator=g).cuda()
labels = torch.randint(0, 1000, (8, 128), generator=g).cuda()
lengths = torch.randint(16, 129, (8,), generator=g)
mask = (torch.arange(128)[None, :] < lengths[:, None]).view(8, 1, 1, 128).cuda()

def step():
    opt.zero_grad()
    loss = model(ids, mask=mask, mlm_labels=labels)
    loss.backward()
    opt.step()
    return loss

stepper = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams)
losses = [stepper().detach().float().item() for _ in range(STEPS)]
torch.save({"losses": losses, "params": {n: p.detach().float().cpu() for n, p in model.named_parameters()}}, OUT)
print("OK")
bps.shutdown()
"""


def _bert_runs(tmp_path, all_fused, dropout, steps):
    runs = {}
    for fused in (False, True):
        out = str(tmp_path / ("%d.pt" % fused))
        assert "OK" in _run_py(_BERT_STEPS % (fused, all_fused, dropout, steps, out))
        runs[fused] = torch.load(out)
    return runs[False], runs[True]


@pytest.mark.gpu
@pytest.mark.parametrize("all_fused", [False, True], ids=["alone", "fp8_norm_loss"])
def test_bert_tiny_graphed_steps_track_stock(tmp_path, all_fused):
    """bert_tiny in bf16 with a key-padding mask, dropout 0, fused AdamW and one CUDA graph per step: with
    fused_attention the losses and parameters track the stock model's within bf16 rounding."""
    s, f = _bert_runs(tmp_path, all_fused, 0.0, 6)
    for a, b in zip(s["losses"], f["losses"]):
        assert abs(a - b) <= 1e-2 * abs(a), (s["losses"], f["losses"])
    assert all(torch.isfinite(p).all() for p in f["params"].values())


@pytest.mark.gpu
def test_bert_tiny_dropout_loss_curve_tracks_stock(tmp_path):
    """300 graphed steps at dropout 0.1: the fused model's loss curve stays next to the stock one (means of the
    last 50 steps within 2 %)."""
    s, f = _bert_runs(tmp_path, True, 0.1, 300)
    ls, lf = np.array(s["losses"]), np.array(f["losses"])
    assert np.isfinite(lf).all()
    assert lf[-50:].mean() < lf[:10].mean() * 0.9
    assert abs(lf[-50:].mean() - ls[-50:].mean()) <= 0.02 * ls[-50:].mean(), (ls[-50:].mean(), lf[-50:].mean())
