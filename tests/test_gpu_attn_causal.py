"""Causal self-attention (ops/attn.py with causal=True, kernels/attn_causal.cu), padded and packed.

GPU tests compare the causal kernels with the float64 reference of test_gpu_attn.py given the causal mask combined
with any key-padding mask, under the same rounding-order bounds (4 u of the magnitudes that enter a result plus 2 u of
itself; for fp16 also the absolute error of P and dS rounded below its normal range, 2^-24 per term) and, at p = 0,
at most twice the error of torch's SDPA with the causal mask.  Dropout references use the NumPy
Philox of test_gpu_attn.py and test_gpu_attn_varlen.py: the causal kernels keep the documented numbering.

Bit-exact properties follow from the tile walk: the last query row visits every key tile the bidirectional kernel
visits, in the same order, so it equals that kernel's row bit for bit; a query row never reads a later token, so a
prefix of the sequence gives the same rows, and changing later tokens changes no earlier row.

CPU tests check the stock causal expressions, the fallbacks and the argument rules.
"""
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from byteps_b200.ops.attn import _stock, _stock_varlen, self_attention
from test_gpu_attn import TINY, UNIT, _drawn_seed, _keep_bits, _make, _make_mask, _reference, _run_py
from test_gpu_attn_varlen import LEAD, LENGTHS, TAIL, _cu, _keep_rows, _outside, _sequences

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16]
PADDED, PACKED = "_SelfAttentionFnBackward", "_VarlenAttentionFnBackward"


def _dt_id(d):
    return str(d).replace("torch.", "")


def _tril(s, device="cuda"):
    return torch.ones(s, s, dtype=torch.bool, device=device).tril()


def _with_causal(mask, s, device="cuda"):
    """the key-padding mask (or None) combined with k <= q, as a [B or 1, 1, S, S] mask of the reference"""
    c = _tril(s, device)
    if mask is None:
        return c.view(1, 1, s, s)
    if mask.dtype == torch.bool:
        return mask & c
    return torch.where(c, mask.double(), float("-inf"))


def _subnormal_slack(qkv, dout, h, allowed, dtype):
    """(out, d(qkv)) slack for fp16, whose P and dS roundings below 2^-14 lose relative precision: each adds at most
    2^-24 (with the dropout scale) absolutely, summed over the allowed terms of each product.  Zero for bf16, whose
    exponent range is fp32's."""
    b, s, e3 = qkv.shape
    if dtype != torch.float16:
        return 0.0, 0.0
    q, k, v = qkv.double().abs().view(b, s, 3, h, 64).permute(2, 0, 3, 1, 4)
    do = dout.double().abs().view(b, s, h, 64).transpose(1, 2)
    a = allowed.double()
    at = a.transpose(-1, -2)
    sl_o = a @ v
    mags = torch.stack([a @ k / 8, at @ q / 8, at @ do]).permute(1, 3, 0, 2, 4).reshape(b, s, e3)
    return 2.0 ** -24 * sl_o.transpose(1, 2).reshape(b, s, e3 // 3), 2.0 ** -24 * mags


def _excess(err, tol, ref):
    i = torch.argmax(err - tol)
    return "worst excess %g at |ref| %g, tol %g" % ((err - tol).flatten()[i], ref.abs().flatten()[i], tol.flatten()[i])


def _fused(qkv, h, mask, p, dout, rng_seed=1234, **kw):
    x = qkv.detach().clone().requires_grad_(True)
    torch.manual_seed(rng_seed)
    out = self_attention(x, h, mask, p, True, causal=True, **kw)
    assert type(out.grad_fn).__name__ == (PACKED if "cu_seqlens" in kw else PADDED), "fused path not taken"
    lse = out.grad_fn.saved_tensors[2].clone()
    out.backward(dout)
    return out.detach(), x.grad, lse


def _bidirectional(qkv, h, mask, p, dout, rng_seed=1234):
    x = qkv.detach().clone().requires_grad_(True)
    torch.manual_seed(rng_seed)
    out = self_attention(x, h, mask, p, True)
    lse = out.grad_fn.saved_tensors[2].clone()
    out.backward(dout)
    return out.detach(), x.grad, lse


def _causal_key_mask(kind, b, s, dtype, g):
    """test_gpu_attn's key-padding masks (batch 1 all masked), plus batch 2 with key 0 masked, so its row 0 has no
    allowed key while its later rows have some"""
    mask = _make_mask(kind, b, s, dtype, g)
    if mask is not None and b > 2 and s > 1:
        mask = mask.clone()
        mask[2, ..., 0] = False if kind == "bool" else float("-inf")
        mask[2, ..., 1:] = True if kind == "bool" else mask[2, ..., 1:].nan_to_num(neginf=0.0)
    return mask


# ---------------------------------------------------------------------------------------------- float64
SHAPES = [(3, 1, 2), (3, 17, 2), (3, 63, 2), (3, 64, 2), (3, 65, 16), (3, 100, 2), (4, 128, 16), (3, 384, 2),
          (3, 512, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1], ids=["p0", "p01"])
@pytest.mark.parametrize("mask_kind", ["none", "bool", "add"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda t: "x".join(map(str, t)))
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_matches_float64(dtype, shape, mask_kind, p):
    b, s, h = shape
    g = torch.Generator().manual_seed(b * 1000 + s)
    qkv, dout = _make(b, s, h, dtype, seed=s)
    mask = _causal_key_mask(mask_kind, b, s, dtype, g)
    keep = _keep_bits(*_drawn_seed(1234), (b, h, s, s), p).cuda() if p > 0 else None
    out, dqkv, lse = _fused(qkv, h, mask, p, dout)
    full = _with_causal(mask, s)
    out_ref, dqkv_ref, mag_o, mags = _reference(qkv, h, full, keep, p, dout)
    allowed = full.expand(b, 1, s, s)
    allowed = allowed if allowed.dtype == torch.bool else torch.isfinite(allowed)
    sl_o, sl_d = _subnormal_slack(qkv, dout, h, allowed, dtype)
    allowed = allowed[:, 0]
    u = UNIT[dtype]
    err_o = (out.double() - out_ref).abs()
    tol_o = 4 * u * mag_o + 2 * u * out_ref.abs() + TINY[dtype] + sl_o
    assert (err_o <= tol_o).all(), "out: " + _excess(err_o, tol_o, out_ref)
    err_d = (dqkv.double() - dqkv_ref).abs()
    tol_d = 4 * u * mags + 2 * u * dqkv_ref.abs() + TINY[dtype] + sl_d
    assert (err_d <= tol_d).all(), "dqkv: " + _excess(err_d, tol_d, dqkv_ref)
    dead = ~allowed.any(-1)                                       # [b, s] rows with no allowed key
    e = h * 64
    assert (out[dead] == 0).all() and (dqkv[dead][:, :e] == 0).all()
    assert (lse.permute(0, 2, 1)[dead] == float("inf")).all() and torch.isfinite(lse.permute(0, 2, 1)[~dead]).all()
    if mask is not None and b > 2 and s > 1:
        assert dead[2, 0] and not dead[2, 1:].any()
    if p == 0:
        live = ~dead.any(-1)                                      # batches SDPA can run without an empty row
        x = qkv[live].clone().requires_grad_(True)
        so = _stock(x, h, None if mask is None else mask[live] if mask.shape[0] > 1 else mask, 0.0, causal=True)
        so.backward(dout[live])
        es_o = (so.double() - out_ref[live]).abs().max().item()
        es_d = (x.grad.double() - dqkv_ref[live]).abs().max().item()
        assert err_o[live].max().item() <= max(2 * es_o, u * out_ref.abs().max().item()), es_o
        assert err_d[live].max().item() <= max(2 * es_d, u * dqkv_ref.abs().max().item()), es_d


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1], ids=["p0", "p01"])
@pytest.mark.parametrize("h", [2, 16], ids=lambda v: "H%d" % v)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_packed_matches_float64(dtype, h, p):
    """empty sequences, cu[0] > 0, a tail outside every sequence, lengths around the tile edges up to 512"""
    cu = _cu(LEAD, LENGTHS)
    t = cu[-1] + TAIL
    g = torch.Generator(device="cuda").manual_seed(h)
    qkv = (torch.randn(t, 3 * h * 64, device="cuda", generator=g, dtype=torch.float64) * 1.5).to(dtype)
    dout = torch.randn(t, h * 64, device="cuda", generator=g, dtype=torch.float64).to(dtype)
    cu_d = torch.tensor(cu, dtype=torch.int32, device="cuda")
    out, dqkv, _ = _fused(qkv, h, None, p, dout, cu_seqlens=cu_d, max_seqlen=512)
    seed = _drawn_seed(1234) if p > 0 else None
    u = UNIT[dtype]
    for a, n in _sequences(cu):
        keep = _keep_rows(*seed, h, t, a, n, p)[None].cuda() if p > 0 else None
        q1, d1 = qkv[None, a:a + n], dout[None, a:a + n]
        out_ref, dqkv_ref, mag_o, mags = _reference(q1, h, _with_causal(None, n), keep, p, d1)
        sl_o, sl_d = _subnormal_slack(q1, d1, h, _with_causal(None, n), dtype)
        err_o = (out[None, a:a + n].double() - out_ref).abs()
        tol_o = 4 * u * mag_o + 2 * u * out_ref.abs() + TINY[dtype] + sl_o
        assert (err_o <= tol_o).all(), (n, "out: " + _excess(err_o, tol_o, out_ref))
        err_d = (dqkv[None, a:a + n].double() - dqkv_ref).abs()
        tol_d = 4 * u * mags + 2 * u * dqkv_ref.abs() + TINY[dtype] + sl_d
        assert (err_d <= tol_d).all(), (n, "dqkv: " + _excess(err_d, tol_d, dqkv_ref))
        if p == 0:
            x = q1.clone().requires_grad_(True)
            so = _stock(x, h, None, 0.0, causal=True)
            so.backward(d1)
            es_o = (so.double() - out_ref).abs().max().item()
            es_d = (x.grad.double() - dqkv_ref).abs().max().item()
            assert err_o.max().item() <= max(2 * es_o, u * out_ref.abs().max().item()), (n, es_o)
            assert err_d.max().item() <= max(2 * es_d, u * dqkv_ref.abs().max().item()), (n, es_d)
    dead = _outside(cu, t).cuda()
    assert (out[dead] == 0).all() and (dqkv[dead] == 0).all()


# ---------------------------------------------------------------------------------------------- bit-exact properties
@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1], ids=["p0", "p01"])
@pytest.mark.parametrize("mask_kind", ["none", "bool"])
@pytest.mark.parametrize("s", [100, 128, 512], ids=lambda v: "S%d" % v)
def test_last_row_equals_bidirectional(s, mask_kind, p):
    b, h = 3, 2
    qkv, dout = _make(b, s, h, torch.bfloat16, seed=s)
    mask = _make_mask(mask_kind, b, s, torch.bfloat16, torch.Generator().manual_seed(s))
    co, cd, cl = _fused(qkv, h, mask, p, dout, rng_seed=5)
    bo, bd, bl = _bidirectional(qkv, h, mask, p, dout, rng_seed=5)
    e = h * 64
    assert torch.equal(co[:, -1], bo[:, -1])
    assert torch.equal(cl[..., -1], bl[..., -1])
    assert torch.equal(cd[:, -1, :e], bd[:, -1, :e])
    assert not torch.equal(co, bo)


@pytest.mark.gpu
@pytest.mark.parametrize("s,lens", [(200, (1, 77, 128, 199)), (512, (64, 300, 511))], ids=["S200", "S512"])
def test_prefix_equals_shorter_call(s, lens):
    """At p = 0 a call on the first L tokens gives rows < L of the full call, and so do its d(qkv) rows when the full
    call's dout rows >= L are zero; padded and packed."""
    b, h = 2, 2
    qkv, dout = _make(b, s, h, torch.bfloat16, seed=1)
    for n in lens:
        d_full = dout.clone()
        d_full[:, n:] = 0
        fo, fd, _ = _fused(qkv, h, None, 0.0, d_full)
        so, sd, _ = _fused(qkv[:, :n].contiguous(), h, None, 0.0, dout[:, :n].contiguous())
        assert torch.equal(fo[:, :n], so) and torch.equal(fd[:, :n], sd), n
        cu = torch.tensor([0, n], dtype=torch.int32, device="cuda")
        po, pd, _ = _fused(qkv[0], h, None, 0.0, d_full[0], cu_seqlens=cu, max_seqlen=s)
        assert torch.equal(po[:n], so[0]) and torch.equal(pd[:n], sd[0]), n


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1], ids=["p0", "p01"])
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
def test_later_tokens_do_not_reach_earlier_rows(packed, p):
    b, s, h = 2, 300, 2
    qkv, dout = _make(b, s, h, torch.bfloat16, seed=2)
    kw = {}
    if packed:
        qkv, dout = qkv.view(b * s, -1), dout.view(b * s, -1)
        kw = dict(cu_seqlens=torch.tensor([0, s, 2 * s], dtype=torch.int32, device="cuda"), max_seqlen=s)
    base = _fused(qkv, h, None, p, dout, rng_seed=3, **kw)
    e = h * 64
    for j in (1, 64, 65, 200, 299):
        q2, d2 = qkv.clone().view(-1, s, 3 * e), dout.clone().view(-1, s, e)
        q2[:, j:] = (q2[:, j:].float() * -0.5 + 0.25).to(q2.dtype)
        d2[:, j:] = (d2[:, j:].float() * 3.0 - 1.0).to(d2.dtype)
        o, d, _ = _fused(q2.view_as(qkv), h, None, p, d2.view_as(dout), rng_seed=3, **kw)
        o, d, bo, bd = o.view(-1, s, e), d.view(-1, s, 3 * e), base[0].view(-1, s, e), base[1].view(-1, s, 3 * e)
        assert torch.equal(o[:, :j], bo[:, :j]) and torch.equal(d[:, :j, :e], bd[:, :j, :e]), j
        assert not torch.equal(o[:, j:], bo[:, j:])


@pytest.mark.gpu
@pytest.mark.parametrize("s", [200, 512], ids=lambda v: "S%d" % v)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_padded_batch_as_stream_equals_padded_kernel(dtype, s):
    b, h = 4, 2
    lengths = torch.randint(1, s + 1, (b,), generator=torch.Generator().manual_seed(s))
    lengths[0], lengths[1] = s, 1
    attend = torch.arange(s)[None, :] < lengths[:, None]
    qkv, dout = _make(b, s, h, dtype, seed=3)
    dout = dout * attend[..., None].cuda().to(dtype)
    out, dq, _ = _fused(qkv, h, attend.view(b, 1, 1, s).cuda(), 0.0, dout)
    cu = [0]
    for n in lengths.tolist():
        cu += [cu[-1] + n, cu[-1] + s]
    cu_d = torch.tensor(cu, dtype=torch.int32, device="cuda")
    po, pd, _ = _fused(qkv.view(b * s, -1), h, None, 0.0, dout.view(b * s, -1), cu_seqlens=cu_d, max_seqlen=512)
    real = attend.reshape(-1).cuda()
    assert torch.equal(po[real], out.view(b * s, -1)[real])
    assert torch.equal(pd[real], dq.view(b * s, -1)[real])


# ---------------------------------------------------------------------------------------------- dropout
def _extract_bits(b, s, h, p, rng_seed, packed):
    """Keep bits [B, H, S, S] of the lower triangle read from the output: Q = K = 0 makes P uniform over the keys
    k <= q, and V one-hot on the keys of a 64-key window makes O[q, j] nonzero exactly when (q, key w0 + j) is
    allowed and kept."""
    e = h * 64
    bits = torch.zeros(b, h, s, s, dtype=torch.bool)
    cu = torch.tensor([s * i for i in range(b + 1)], dtype=torch.int32, device="cuda")
    for w0 in range(0, s, 64):
        qkv = torch.zeros(b, s, 3, h, 64, dtype=torch.bfloat16, device="cuda")
        n = min(64, s - w0)
        idx = torch.arange(n, device="cuda")
        qkv[:, w0 + idx, 2, :, idx] = 1.0
        torch.manual_seed(rng_seed)
        if packed:
            out = self_attention(qkv.view(b * s, 3 * e), h, p=p, cu_seqlens=cu, max_seqlen=s, causal=True)
        else:
            out = self_attention(qkv.view(b, s, 3 * e), h, None, p, True, causal=True)
        bits[..., w0:w0 + n] = (out.view(b, s, h, 64)[..., :n] != 0).permute(0, 2, 1, 3).cpu()
    return bits


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout_bits_are_philox(p, packed):
    b, s, h = 2, 100, 3
    bits = _extract_bits(b, s, h, p, 77, packed)
    seed = _drawn_seed(77)
    if packed:
        ref = torch.stack([_keep_rows(*seed, h, b * s, i * s, s, p) for i in range(b)])
    else:
        ref = _keep_bits(*seed, (b, h, s, s), p)
    low = _tril(s, "cpu")
    assert torch.equal(bits, ref & low)
    n = int(low.sum()) * b * h
    frac = int(bits.sum()) / n
    sigma = (p * (1 - p) / n) ** 0.5
    assert abs(frac - (1 - p)) <= 5 * sigma, (frac, 1 - p)


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
@pytest.mark.parametrize("case", ["p0", "eval"])
def test_no_draw_without_dropout(case, packed):
    qkv, dout = _make(2, 150, 2, torch.bfloat16)
    kw = dict(causal=True)
    if packed:
        qkv, dout = qkv.view(300, -1), dout.view(300, -1)
        kw.update(cu_seqlens=torch.tensor([0, 100, 300], dtype=torch.int32, device="cuda"), max_seqlen=200)
    x = qkv.clone().requires_grad_(True)
    before = torch.cuda.get_rng_state()
    out = self_attention(x, 2, None, 0.0 if case == "p0" else 0.1, case == "p0", **kw)
    out.backward(dout)
    torch.cuda.synchronize()
    assert type(out.grad_fn).__name__ == (PACKED if packed else PADDED)
    assert torch.equal(before, torch.cuda.get_rng_state())


# ---------------------------------------------------------------------------------------------- memory, repeatability
def _banded(rows, cols, fill, pad, dt):
    buf = torch.full((rows + 2 * pad, cols), fill, dtype=dt, device="cuda")
    return buf, buf[pad:pad + rows]


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1], ids=["p0", "p01"])
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
def test_buffers_keep_their_bands_and_every_row_is_written(packed, p):
    """qkv and dout inside NaN bands, out / dqkv / lse / delta NaN-filled inside canary bands: the bands stay as they
    were, and no output element is left NaN (every row was written)."""
    from byteps_b200 import _native

    cu = _native.cuda()
    h, pad, canary, dt = 2, 37, 1234.0, torch.bfloat16
    e = h * 64
    if packed:
        cl = _cu(LEAD, LENGTHS)
        t = cl[-1] + TAIL
        b, s = 1, t
    else:
        b, s = 3, 300
        t = b * s
    qkv, dout = _make(1, t, h, dt, seed=4)
    qb, q = _banded(t, 3 * e, float("nan"), pad, dt)
    db, d = _banded(t, e, float("nan"), pad, dt)
    q.copy_(qkv[0])
    d.copy_(dout[0])
    ob, o = _banded(t, e, canary, pad, dt)
    gb, g = _banded(t, 3 * e, canary, pad, dt)
    lb, lse = _banded(h * t, 1, canary, pad, torch.float32)
    xb, delta = _banded(h * t, 1, canary, pad, torch.float32)
    for inner in (o, g, lse, delta):
        inner.fill_(float("nan"))
    seed = torch.tensor([7, 9], dtype=torch.int64, device="cuda") if p else None
    sp = 0 if seed is None else seed.data_ptr()
    keep, scale = (0, 1.0) if seed is None else (int(0.9 * 2 ** 32), 1 / 0.9)
    st = torch.cuda.current_stream().cuda_stream
    if packed:
        cu_d = torch.tensor(cl, dtype=torch.int32, device="cuda")
        n = len(cl) - 1
        cu.attn_varlen_fwd(q.data_ptr(), 1, t, n, h, 64, 512, cu_d.data_ptr(), sp, keep, scale, o.data_ptr(),
                           lse.data_ptr(), st, causal=True)
        cu.attn_varlen_bwd(q.data_ptr(), o.data_ptr(), d.data_ptr(), lse.data_ptr(), 1, t, n, h, 64, 512,
                           cu_d.data_ptr(), sp, keep, scale, delta.data_ptr(), g.data_ptr(), st, causal=True)
    else:
        cu.attn_fwd(q.data_ptr(), 1, b, s, h, 64, 0, 0, 0, sp, keep, scale, o.data_ptr(), lse.data_ptr(), st,
                    causal=True)
        cu.attn_bwd(q.data_ptr(), o.data_ptr(), d.data_ptr(), lse.data_ptr(), 1, b, s, h, 64, 0, 0, 0, sp, keep,
                    scale, delta.data_ptr(), g.data_ptr(), st, causal=True)
    torch.cuda.synchronize()
    for buf, inner_rows in ((ob, t), (gb, t), (lb, h * t), (xb, h * t)):
        assert (buf[:pad] == canary).all() and (buf[pad + inner_rows:] == canary).all()
    assert not torch.isnan(o).any() and not torch.isnan(g).any() and not torch.isnan(lse).any()
    if packed:
        dead = _outside(cl, t).cuda()
        assert (o[dead] == 0).all() and (g[dead] == 0).all()
        assert not torch.isnan(delta.view(h, t)[:, ~dead]).any()
    else:
        assert not torch.isnan(delta).any()


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
def test_deterministic_and_graph_replays_match_eager(packed):
    h, p = 4, 0.1
    if packed:
        t = 720
        qkv, dout = _make(1, t, h, torch.bfloat16)
        qkv, dout = qkv[0], dout[0]
        ca = torch.tensor(_cu(0, [200, 0, 150, 350, 0]), dtype=torch.int32, device="cuda")
        cb = torch.tensor(_cu(3, [50, 450, 0, 100, 90]), dtype=torch.int32, device="cuda")
        cu = ca.clone()
        mask, kw, kw_b = None, dict(cu_seqlens=cu, max_seqlen=512), dict(cu_seqlens=cb, max_seqlen=512)
    else:
        b, s = 4, 200
        qkv, dout = _make(b, s, h, torch.bfloat16)
        mask = _make_mask("bool", b, s, torch.bfloat16, torch.Generator().manual_seed(0))
        kw = {}
    runs = [_fused(qkv, h, mask, p, dout, rng_seed=11, **kw) for _ in range(2)]
    assert all(torch.equal(a, c) for a, c in zip(runs[0], runs[1]))
    if packed:
        ref_b = _fused(qkv, h, mask, p, dout, rng_seed=11, **kw_b)

    x = qkv.clone().requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            x.grad = None
            self_attention(x, h, mask, p, True, causal=True, **kw).backward(dout)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    x.grad = None
    with torch.cuda.graph(graph):
        out = self_attention(x, h, mask, p, True, causal=True, **kw)
        out.backward(dout)
    torch.manual_seed(11)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, runs[0][0]) and torch.equal(x.grad, runs[0][1])
    first = out.clone()
    graph.replay()
    torch.cuda.synchronize()
    assert not torch.equal(out, first)
    if packed:
        cu.copy_(cb)   # new offsets, same capacity, refreshed in place
        torch.manual_seed(11)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ref_b[0]) and torch.equal(x.grad, ref_b[1])


_LAUNCHES = """
import json
import torch
from torch.profiler import ProfilerActivity, profile
from byteps_b200.ops.attn import self_attention

def launches(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

res = {}
for packed in (False, True):
    qkv = torch.randn(4, 256, 3 * 128, device="cuda").to(torch.bfloat16)
    kw = dict(causal=True)
    if packed:
        qkv = qkv.view(1024, -1)
        kw.update(cu_seqlens=torch.tensor([0, 300, 1024], dtype=torch.int32, device="cuda"), max_seqlen=512)
    qkv.requires_grad_(True)
    dout = torch.randn(*qkv.shape[:-1], 128, device="cuda").to(torch.bfloat16)
    self_attention(qkv, 2, None, 0.0, True, **kw).backward(dout)
    out = {}
    fwd = launches(lambda: out.setdefault("o", self_attention(qkv, 2, None, 0.0, True, **kw)))
    bwd = launches(lambda: torch.autograd.grad(out["o"], qkv, dout))
    res["packed" if packed else "padded"] = {"fwd": fwd, "bwd": bwd}
print(json.dumps(res))
"""


@pytest.mark.gpu
def test_launch_count():
    """One launch forward and two backward, padded and packed, in a process of its own as the suite's other launch
    counts are."""
    res = json.loads(_run_py(_LAUNCHES).strip().splitlines()[-1])
    for form, names in res.items():
        fwd, bwd = names["fwd"], names["bwd"]
        assert len(fwd) == 1 and "fwd_kernel" in fwd[0], (form, fwd)
        assert len(bwd) == 2 and "bwd_dq_kernel" in bwd[0] and "bwd_dkv_kernel" in bwd[1], (form, bwd)


# ---------------------------------------------------------------------------------------------- fallbacks
def _fallback_case(case, device):
    b, s, h, d, dtype = 2, 40, 2, 64, torch.bfloat16
    if case == "fp32":
        dtype = torch.float32
    elif case in ("d32", "d128"):
        d = int(case[1:])
    elif case == "s513":
        s = 513
    g = torch.Generator().manual_seed(0)
    width = 2 if case == "noncontig" else 1
    qkv = torch.randn(b, s, width * 3 * h * d, generator=g).to(dtype).to(device)
    return qkv, h


FALLBACKS = ["fp32", "d32", "d128", "s513", "noncontig"]


def _check_fallback(case, device, form):
    qkv, h = _fallback_case(case, device)
    b, s = qkv.shape[:2]
    x1, x2 = qkv.clone().requires_grad_(True), qkv.clone().requires_grad_(True)
    view = (lambda t: t[..., ::2]) if case == "noncontig" else (lambda t: t)
    if form == "packed":
        cu = torch.tensor([3, 20, 20, 55], dtype=torch.int32, device=device)
        a = self_attention(view(x1), h, p=0.0, cu_seqlens=cu, max_seqlen=s, causal=True)
        ref = _stock_varlen(view(x2), h, cu, s, 0.0, causal=True)
    else:
        mask = None
        if form == "mask":
            mask = (torch.arange(s, device=device) < s - 5).view(1, 1, 1, s).expand(b, 1, 1, s)
        a = self_attention(view(x1), h, mask, 0.0, True, causal=True)
        ref = _stock(view(x2), h, mask, 0.0, causal=True)
    assert type(a.grad_fn).__name__ not in (PADDED, PACKED)
    assert torch.equal(a, ref)
    g = torch.randn_like(a)
    a.backward(g)
    ref.backward(g)
    if device == "cpu":
        assert torch.equal(x1.grad, x2.grad)
    else:   # the flash and efficient SDPA backwards sum dQ with atomics, so two stock runs may differ in the last bit
        assert (x1.grad - x2.grad).abs().max() <= 2.0 ** -7 * x2.grad.abs().max()


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["padded", "mask", "packed"])
@pytest.mark.parametrize("case", FALLBACKS)
def test_fallbacks_are_stock_cuda(case, form):
    _check_fallback(case, "cuda", form)


@pytest.mark.parametrize("form", ["padded", "mask", "packed"])
@pytest.mark.parametrize("case", FALLBACKS + ["bf16"])
def test_fallbacks_are_stock_cpu(case, form):
    _check_fallback(case, "cpu", form)


@pytest.mark.parametrize("kind", ["bool", "add"])
def test_stock_causal_expression_cpu(kind):
    """The stock expressions equal an explicit float64 softmax with the causal mask, on top of a key-padding mask,
    and the packed one equals the sequences run one at a time."""
    b, s, h = 2, 30, 2
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(b, s, 3 * h * 64, generator=g, dtype=torch.float64)
    attend = torch.arange(s)[None, :] < torch.tensor([s, 11])[:, None]
    attend[0, 0] = False   # row 0 of batch 0 has no allowed key: SDPA's result there is not compared
    mask = attend.view(b, 1, 1, s)
    if kind == "add":
        mask = torch.where(mask, torch.rand(b, 1, 1, s, generator=g, dtype=torch.float64), float("-inf"))
    out = _stock(qkv, h, mask, 0.0, causal=True)
    q, k, v = qkv.view(b, s, 3, h, 64).permute(2, 0, 3, 1, 4)
    sc = q @ k.transpose(-1, -2) / 8
    sc = sc + (mask.double() if kind == "add" else torch.where(mask, 0.0, float("-inf")))
    sc = sc.masked_fill(~_tril(s, "cpu"), float("-inf"))
    ref = (torch.softmax(sc, -1) @ v).transpose(1, 2).reshape(b, s, -1)
    live = torch.ones(b, s, dtype=torch.bool)
    live[0, 0] = False
    assert torch.allclose(out[live], ref[live], rtol=1e-12, atol=1e-12)
    assert torch.equal(_stock(qkv, h, None, 0.0, causal=True),
                       torch.nn.functional.scaled_dot_product_attention(
                           *qkv.view(b, s, 3, h, 64).permute(2, 0, 3, 1, 4), is_causal=True).transpose(1, 2)
                       .reshape(b, s, -1))
    flat = qkv.reshape(b * s, -1)
    cu = torch.tensor([2, 12, 12, 40, 55], dtype=torch.int32)
    packed = _stock_varlen(flat, h, cu, 60, 0.0, causal=True)
    for a, c in ((2, 12), (12, 40), (40, 55)):
        one = _stock(flat[None, a:c], h, None, 0.0, causal=True)[0]
        assert torch.allclose(packed[a:c], one, rtol=1e-12, atol=1e-12)
    outside = torch.ones(b * s, dtype=torch.bool)
    outside[2:55] = False
    assert (packed[outside] == 0).all()


def test_bad_arguments_raise():
    with pytest.raises(ValueError):
        self_attention(torch.zeros(2, 3, 10), 2, causal=True)
    with pytest.raises(ValueError):
        self_attention(torch.zeros(2, 3, 384), 2, p=1.5, causal=True)
    with pytest.raises(ValueError):
        self_attention(torch.zeros(2, 3, 384), 2, torch.ones(2, 1, 1, 3, dtype=torch.bool), causal=True,
                       cu_seqlens=torch.tensor([0, 6], dtype=torch.int32))


def _native_cuda_or_skip():
    from byteps_b200 import _native

    try:
        return _native.cuda()
    except Exception as exc:   # noqa: BLE001 - the extension is not built on this machine
        pytest.skip("CUDA extension unavailable: %s" % exc)


def test_binding_rejects_bad_arguments():
    """The checks run before any launch, so this needs the built extension but no GPU; the good call shape with
    causal=True is rejected only for the argument under test."""
    cu = _native_cuda_or_skip()
    ptr, seed = 1 << 20, 0
    for dtype, d, s in [(0, 64, 8), (1, 32, 8), (1, 64, 0), (1, 64, 513)]:
        with pytest.raises(ValueError):
            cu.attn_fwd(ptr, dtype, 1, s, 1, d, 0, 0, 0, seed, 0, 1.0, ptr, ptr, 0, causal=True)
        with pytest.raises(ValueError):
            cu.attn_bwd(ptr, ptr, ptr, ptr, dtype, 1, s, 1, d, 0, 0, 0, seed, 0, 1.0, ptr, ptr, 0, causal=True)
    for t, n, ms, cup in [(0, 1, 64, ptr), (8, 0, 64, ptr), (8, 1, 513, ptr), (8, 1, 64, 0), (8, 1, 64, ptr + 2)]:
        with pytest.raises(ValueError):
            cu.attn_varlen_fwd(ptr, 1, t, n, 1, 64, ms, cup, seed, 0, 1.0, ptr, ptr, 0, causal=True)
        with pytest.raises(ValueError):
            cu.attn_varlen_bwd(ptr, ptr, ptr, ptr, 1, t, n, 1, 64, ms, cup, seed, 0, 1.0, ptr, ptr, 0, causal=True)
    with pytest.raises(TypeError):   # causal is keyword-only
        cu.attn_fwd(ptr, 1, 1, 8, 1, 64, 0, 0, 0, seed, 0, 1.0, ptr, ptr, 0, True)


# ---------------------------------------------------------------------------------------------- build
def _compile(tmp_path, name):
    from byteps_b200 import _build

    nvcc = _build._nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "byteps_b200", "csrc", "kernels", name)
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + _build.ARCH_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                                         str(tmp_path / "k.o")],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    return nvcc, r.stderr


def test_causal_kernels_compile_without_spills(tmp_path):
    _, log = _compile(tmp_path, "attn_causal.cu")
    found = {"padded": 0, "varlen": 0}
    for block in log.split("Compiling entry function '")[1:]:
        m = re.match(r"_ZN\S*attn_(varlen_)?(fwd|bwd_dq|bwd_dkv)_kernel", block)
        if not m:
            continue
        found["varlen" if m.group(1) else "padded"] += 1
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block[:400]
    assert found == {"padded": 12, "varlen": 12}, found


@pytest.mark.parametrize("name", ["attn.cu", "attn_varlen.cu"])
def test_bidirectional_units_hold_no_causal_kernel(tmp_path, name):
    """The causal instantiations stay in their own translation unit: attn.cu and attn_varlen.cu compile to exactly
    the 12 bidirectional kernels each, every one with the causal flag false."""
    nvcc, log = _compile(tmp_path, name)
    names = [b.split("'")[0] for b in log.split("Compiling entry function '")[1:]]
    attn = [n for n in names if re.search(r"attn_\w*kernel", n)]
    assert len(attn) == 12, attn
    # the template arguments <bool BF, bool DROP, bool CAUSAL> mangle as Lb0E / Lb1E; CAUSAL is the last
    assert all(n.endswith("Lb0EEEvNS_8AttnArgsE") or n.endswith("Lb0EEEvNS_9AttnVArgsE") for n in attn), attn
