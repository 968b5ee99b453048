"""Fused self-attention over packed variable-length sequences (ops/attn.py with cu_seqlens, kernels/attn_varlen.cu).

GPU tests compare the kernels with a float64 reference run sequence by sequence, with the error bound of
test_gpu_attn.py (4 u of the magnitudes that enter a result plus 2 u of itself) and, at p = 0, at most twice the error
of torch's SDPA on the same sequence.  Dropout references use a NumPy Philox of the documented numbering
i = (h T + t) 512 + (u - cu[n]); a separate test checks that numbering bit for bit against the bits the kernel
applied, so the float64 comparison at p = 0.1 also shows that the backward applies the forward's bits.

A padded batch written as a stream (each row's padding run a sequence of its own) must give the padded kernel's
results exactly: the padded kernel's extra key and query tiles add exact zeros.

CPU tests check the argument rules, the stock block-diagonal expression against per-sequence SDPA, and BERT on a
packed stream against the key-padding-mask model.
"""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from byteps_b200.models import bert_tiny
from byteps_b200.ops.attn import _stock, _stock_varlen, self_attention
from test_gpu_attn import TINY, UNIT, _drawn_seed, _philox, _reference, _run_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16]
FUSED = "_VarlenAttentionFnBackward"


def _dt_id(d):
    return str(d).replace("torch.", "")


def _cu(lead, lengths):
    """cu_seqlens starting at `lead` for the given lengths"""
    return [lead] + list(lead + np.cumsum(lengths))


# lengths 1 .. 512 around the tile edges, zero-length sequences in the middle and at the end, cu[0] > 0 and a tail
# of tokens outside every sequence
LEAD, LENGTHS, TAIL = 5, [1, 63, 64, 65, 0, 128, 200, 511, 512, 0], 7


def _keep_rows(seed, offset, h_count, t_count, row0, length, p):
    """keep bits [H, L, L] of the sequence of tokens row0 .. row0 + L - 1 in a stream of t_count tokens"""
    rows = (np.arange(h_count, dtype=np.uint64)[:, None] * np.uint64(t_count)
            + np.uint64(row0) + np.arange(length, dtype=np.uint64)[None, :]) * np.uint64(512)
    nblk = (length + 3) // 4
    g = (rows[..., None] // np.uint64(4) + np.arange(nblk, dtype=np.uint64)).reshape(-1)
    m32 = np.uint64(0xFFFFFFFF)
    sd, of = np.uint64(seed), np.uint64(offset)
    full = lambda v: np.full_like(g, v)   # noqa: E731
    r = _philox(g & m32, g >> np.uint64(32), full(of & m32), full(of >> np.uint64(32)), np.uint64(sd & m32),
                np.uint64(sd >> np.uint64(32)))
    words = np.stack(r, -1).reshape(h_count, length, 4 * nblk)[..., :length]
    keep = min(int(round((1.0 - p) * 2.0 ** 32)), 2 ** 32 - 1)
    return torch.from_numpy(words < np.uint64(keep))


def _make(t, h, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = (torch.randn(t, 3 * h * 64, device="cuda", generator=g, dtype=torch.float64) * 1.5).to(dtype)
    dout = torch.randn(t, h * 64, device="cuda", generator=g, dtype=torch.float64).to(dtype)
    return qkv, dout


def _fused(qkv, h, cu, p, dout, max_seqlen=512, rng_seed=1234):
    x = qkv.detach().clone().requires_grad_(True)
    torch.manual_seed(rng_seed)
    out = self_attention(x, h, p=p, cu_seqlens=cu, max_seqlen=max_seqlen)
    assert type(out.grad_fn).__name__ == FUSED, "fused path not taken"
    out.backward(dout)
    return out.detach(), x.grad


def _sequences(cu):
    return [(a, b - a) for a, b in zip(cu[:-1], cu[1:]) if b > a]


def _outside(cu, t):
    inside = torch.zeros(t, dtype=torch.bool)
    for a, n in _sequences(cu):
        inside[a:a + n] = True
    return ~inside


# ---------------------------------------------------------------------------------------------- float64
@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.1], ids=["p0", "p01"])
@pytest.mark.parametrize("h", [2, 16], ids=lambda v: "H%d" % v)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_matches_float64(dtype, h, p):
    cu = _cu(LEAD, LENGTHS)
    t = cu[-1] + TAIL
    qkv, dout = _make(t, h, dtype, seed=h)
    cu_d = torch.tensor(cu, dtype=torch.int32, device="cuda")
    out, dqkv = _fused(qkv, h, cu_d, p, dout)
    seed = _drawn_seed(1234) if p > 0 else None
    u = UNIT[dtype]
    e = h * 64
    for a, n in _sequences(cu):
        keep = _keep_rows(*seed, h, t, a, n, p)[None].cuda() if p > 0 else None
        q1, d1 = qkv[None, a:a + n], dout[None, a:a + n]
        out_ref, dqkv_ref, mag_o, mags = _reference(q1, h, None, keep, p, d1)
        err_o = (out[None, a:a + n].double() - out_ref).abs()
        assert (err_o <= 4 * u * mag_o + 2 * u * out_ref.abs() + TINY[dtype]).all(), (n, "out")
        err_d = (dqkv[None, a:a + n].double() - dqkv_ref).abs()
        assert (err_d <= 4 * u * mags + 2 * u * dqkv_ref.abs() + TINY[dtype]).all(), (n, "dqkv")
        if p == 0:
            x = q1.clone().requires_grad_(True)
            so = _stock(x, h, None, 0.0)
            so.backward(d1)
            es_o = (so.double() - out_ref).abs().max().item()
            es_d = (x.grad.double() - dqkv_ref).abs().max().item()
            assert err_o.max().item() <= max(2 * es_o, u * out_ref.abs().max().item()), (n, es_o)
            assert err_d.max().item() <= max(2 * es_d, u * dqkv_ref.abs().max().item()), (n, es_d)
    dead = _outside(cu, t).cuda()
    assert (out[dead] == 0).all() and (dqkv[dead] == 0).all()
    assert out.shape == (t, e) and dqkv.shape == (t, 3 * e)


# ---------------------------------------------------------------------------------------------- padded kernel
@pytest.mark.gpu
@pytest.mark.parametrize("s", [200, 512], ids=lambda v: "S%d" % v)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_padded_batch_as_stream_equals_padded_kernel(dtype, s):
    b, h = 4, 2
    lengths = torch.randint(1, s + 1, (b,), generator=torch.Generator().manual_seed(s))
    lengths[0] = s   # a padding run of length zero
    lengths[1] = 1
    attend = torch.arange(s)[None, :] < lengths[:, None]
    g = torch.Generator(device="cuda").manual_seed(3)
    qkv = (torch.randn(b, s, 3 * h * 64, device="cuda", generator=g) * 1.5).to(dtype)
    dout = torch.randn(b, s, h * 64, device="cuda", generator=g).to(dtype) * attend[..., None].cuda().to(dtype)
    x = qkv.clone().requires_grad_(True)
    out = self_attention(x, h, attend.view(b, 1, 1, s).cuda(), 0.0, True)
    assert type(out.grad_fn).__name__ == "_SelfAttentionFnBackward"
    out.backward(dout)
    cu = [0]
    for n in lengths.tolist():
        cu += [cu[-1] + n, cu[-1] + s]
    cu_d = torch.tensor(cu, dtype=torch.int32, device="cuda")
    po, pd = _fused(qkv.view(b * s, -1), h, cu_d, 0.0, dout.view(b * s, -1))
    real = attend.reshape(-1).cuda()
    assert torch.equal(po[real], out.detach().view(b * s, -1)[real])
    assert torch.equal(pd[real], x.grad.view(b * s, -1)[real])


# ---------------------------------------------------------------------------------------------- dropout
def _extract_bits(h, cu, t, p, rng_seed):
    """Keep bits [H, t, key offset] read from the output: Q = K = 0 makes P uniform over each sequence's keys, and V
    one-hot on the keys of a 64-key window of every sequence makes O[t, j] nonzero exactly when (t, key w0 + j of
    its sequence) is kept.  One call per window, each after torch.manual_seed(rng_seed)."""
    e = h * 64
    seqs = _sequences(cu)
    longest = max(n for _, n in seqs)
    bits = torch.zeros(h, t, longest, dtype=torch.bool)
    for w0 in range(0, longest, 64):
        qkv = torch.zeros(t, 3, h, 64, dtype=torch.bfloat16, device="cuda")
        for a, n in seqs:
            k = torch.arange(min(64, max(n - w0, 0)), device="cuda")
            qkv[a + w0 + k, 2, :, k] = 1.0
        torch.manual_seed(rng_seed)
        out = self_attention(qkv.view(t, 3 * e), h, p=p, cu_seqlens=torch.tensor(cu, dtype=torch.int32,
                                                                                  device="cuda"))
        w = min(64, longest - w0)
        bits[..., w0:w0 + w] = (out.view(t, h, 64)[..., :w] != 0).permute(1, 0, 2).cpu()
    return bits


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout_bits_are_philox(p):
    h = 3
    cu = _cu(3, [17, 100, 128, 0, 70])
    t = cu[-1] + 2
    bits = _extract_bits(h, cu, t, p, rng_seed=77)
    seed = _drawn_seed(77)
    kept, total = 0, 0
    for a, n in _sequences(cu):
        ref = _keep_rows(*seed, h, t, a, n, p)
        got = bits[:, a:a + n, :n]
        assert torch.equal(got, ref), n
        kept += int(got.sum())
        total += got.numel()
    assert not bits[:, _outside(cu, t)].any()
    sigma = (p * (1 - p) / total) ** 0.5
    assert abs(kept / total - (1 - p)) <= 5 * sigma, (kept / total, 1 - p)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["p0", "eval"])
def test_no_draw_without_dropout(case):
    qkv, dout = _make(300, 2, torch.bfloat16)
    cu = torch.tensor([0, 100, 300], dtype=torch.int32, device="cuda")
    x = qkv.clone().requires_grad_(True)
    before = torch.cuda.get_rng_state()
    out = self_attention(x, 2, None, 0.0 if case == "p0" else 0.1, case == "p0", cu_seqlens=cu, max_seqlen=200)
    out.backward(dout)
    torch.cuda.synchronize()
    assert type(out.grad_fn).__name__ == FUSED
    assert torch.equal(before, torch.cuda.get_rng_state())


# ---------------------------------------------------------------------------------------------- bounds
@pytest.mark.gpu
def test_outside_tokens_are_zero_on_nan_filled_memory():
    h, dtype = 2, torch.bfloat16
    cu = _cu(LEAD, LENGTHS)
    t = cu[-1] + TAIL
    qkv, dout = _make(t, h, dtype)
    cu_d = torch.tensor(cu, dtype=torch.int32, device="cuda")
    x = qkv.clone().requires_grad_(True)
    torch.cuda.synchronize()
    junk = [torch.full((t, n), float("nan"), dtype=dtype, device="cuda") for n in (h * 64, 3 * h * 64)]
    del junk   # the output allocations below reuse these NaN-filled blocks
    out = self_attention(x, h, cu_seqlens=cu_d, max_seqlen=512)
    out.backward(dout)
    dead = _outside(cu, t).cuda()
    assert dead.sum() == LEAD + TAIL
    assert (out[dead] == 0).all() and (x.grad[dead] == 0).all()
    assert torch.isfinite(out).all() and torch.isfinite(x.grad).all()


def _banded_call(cu_list, t, h, max_seqlen, pad=37, seed=None):
    """Runs both kernels through the binding with qkv, out, dout, dqkv, lse and delta inside larger buffers whose
    bands hold NaN (inputs) or a canary (outputs).  Returns (out, dqkv, lse, bands intact)."""
    from byteps_b200 import _native

    cu = _native.cuda()
    e = h * 64
    dt = torch.bfloat16
    canary = 1234.0
    qkv_b = torch.full((t + 2 * pad, 3 * e), float("nan"), dtype=dt, device="cuda")
    dout_b = torch.full((t + 2 * pad, e), float("nan"), dtype=dt, device="cuda")
    qkv, dout = _make(t, h, dt, seed=5)
    qkv_b[pad:pad + t] = qkv
    dout_b[pad:pad + t] = dout
    out_b = torch.full((t + 2 * pad, e), canary, dtype=dt, device="cuda")
    dqkv_b = torch.full((t + 2 * pad, 3 * e), canary, dtype=dt, device="cuda")
    lse_b = torch.full((h * t + 2 * pad * 4,), canary, device="cuda")
    delta_b = torch.full((h * t + 2 * pad * 4,), canary, device="cuda")
    cu_d = torch.tensor(cu_list, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    sp = 0 if seed is None else seed.data_ptr()
    keep, scale = (0, 1.0) if seed is None else (int(0.9 * 2 ** 32), 1 / 0.9)
    o, dq = out_b[pad:pad + t], dqkv_b[pad:pad + t]
    l, d = lse_b[pad * 4:pad * 4 + h * t], delta_b[pad * 4:pad * 4 + h * t]
    cu.attn_varlen_fwd(qkv_b[pad:pad + t].data_ptr(), 1, t, len(cu_list) - 1, h, 64, max_seqlen, cu_d.data_ptr(), sp,
                       keep, scale, o.data_ptr(), l.data_ptr(), st)
    cu.attn_varlen_bwd(qkv_b[pad:pad + t].data_ptr(), o.data_ptr(), dout_b[pad:pad + t].data_ptr(), l.data_ptr(), 1,
                       t, len(cu_list) - 1, h, 64, max_seqlen, cu_d.data_ptr(), sp, keep, scale, d.data_ptr(),
                       dq.data_ptr(), st)
    torch.cuda.synchronize()
    intact = all((band == canary).all().item() for band in (
        out_b[:pad], out_b[pad + t:], dqkv_b[:pad], dqkv_b[pad + t:], lse_b[:pad * 4], lse_b[pad * 4 + h * t:],
        delta_b[:pad * 4], delta_b[pad * 4 + h * t:]))
    return o.clone(), dq.clone(), l.clone().view(h, t), intact


@pytest.mark.gpu
@pytest.mark.parametrize("dropout", [False, True], ids=["p0", "p01"])
def test_buffers_keep_their_bands(dropout):
    cu = _cu(LEAD, LENGTHS)
    t = cu[-1] + TAIL
    seed = torch.tensor([7, 9], dtype=torch.int64, device="cuda") if dropout else None
    o, dq, lse, intact = _banded_call(cu, t, 2, 512, seed=seed)
    assert intact
    assert torch.isfinite(o).all() and torch.isfinite(dq).all()
    dead = _outside(cu, t).cuda()
    assert (o[dead] == 0).all() and (dq[dead] == 0).all() and (lse[:, dead] == float("inf")).all()


@pytest.mark.gpu
@pytest.mark.parametrize("cu", [
    [-40, 10, 100000, 300],                 # offsets before 0 and past T
    [0, 200, 50, 300, 2 ** 31 - 1],         # out of order, the last far past T
    [300, 0],                               # decreasing
    [-2 ** 31, 2 ** 31 - 1],                # the widest span an int32 pair can give
], ids=["range", "order", "decreasing", "extremes"])
def test_bad_offsets_stay_in_bounds(cu):
    """For offsets outside [0, T] or out of order the results are unspecified, but nothing outside the buffers is
    read or written: the NaN bands of the inputs and the canary bands of the outputs stay as they were."""
    _, _, _, intact = _banded_call(cu, 300, 2, 512)
    assert intact


@pytest.mark.gpu
def test_sequence_longer_than_max_seqlen_is_nan():
    h = 2
    cu = _cu(0, [100, 300, 50])
    t = cu[-1] + 4
    qkv, dout = _make(t, h, torch.bfloat16)
    cu_d = torch.tensor(cu, dtype=torch.int32, device="cuda")
    short = _fused(qkv, h, cu_d, 0.0, dout, max_seqlen=256)
    full = _fused(qkv, h, cu_d, 0.0, dout, max_seqlen=512)
    bad = torch.zeros(t, dtype=torch.bool, device="cuda")
    bad[100:400] = True
    for a, c in zip(short, full):
        assert torch.isnan(a[bad]).all()
        assert torch.equal(a[~bad], c[~bad])
        assert torch.isfinite(c).all()


# ---------------------------------------------------------------------------------------------- determinism, graphs
@pytest.mark.gpu
def test_deterministic_and_graph_replays_match_eager():
    h, p = 4, 0.1
    cu_a, cu_b = _cu(0, [200, 0, 150, 350, 0]), _cu(3, [50, 450, 0, 100, 90])
    t = 720
    qkv, dout = _make(t, h, torch.bfloat16)
    ca = torch.tensor(cu_a, dtype=torch.int32, device="cuda")
    cb = torch.tensor(cu_b, dtype=torch.int32, device="cuda")
    runs = [_fused(qkv, h, ca, p, dout, rng_seed=11) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    ref_b = _fused(qkv, h, cb, p, dout, rng_seed=11)

    cu = ca.clone()
    x = qkv.clone().requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            x.grad = None
            self_attention(x, h, p=p, cu_seqlens=cu, max_seqlen=512).backward(dout)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    x.grad = None
    with torch.cuda.graph(graph):
        out = self_attention(x, h, p=p, cu_seqlens=cu, max_seqlen=512)
        out.backward(dout)
    torch.manual_seed(11)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, runs[0][0]) and torch.equal(x.grad, runs[0][1])
    first = out.clone()
    graph.replay()
    torch.cuda.synchronize()
    assert not torch.equal(out, first)
    cu.copy_(cb)   # new offsets, same capacity, refreshed in place
    torch.manual_seed(11)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref_b[0]) and torch.equal(x.grad, ref_b[1])


# ---------------------------------------------------------------------------------------------- fallbacks
def _fallback_case(case, device):
    t, h, d, dtype, max_seqlen = 90, 2, 64, torch.bfloat16, 64
    lengths = [30, 0, 40, 15]
    if case == "fp32":
        dtype = torch.float32
    elif case in ("d32", "d128"):
        d = int(case[1:])
    elif case == "s513":
        t, lengths, max_seqlen = 560, [513, 40], 513
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(t, 3 * h * d, generator=g).to(dtype).to(device)
    if case == "noncontig":
        qkv = torch.randn(t, 2 * 3 * h * d, generator=g).to(dtype).to(device)
    cu = torch.tensor(_cu(2, lengths), dtype=torch.int32, device=device)
    return qkv, h, cu, max_seqlen


FALLBACKS = ["fp32", "d32", "d128", "s513", "noncontig"]


def _check_fallback(case, device):
    qkv, h, cu, max_seqlen = _fallback_case(case, device)
    x1, x2 = qkv.clone().requires_grad_(True), qkv.clone().requires_grad_(True)
    view = (lambda v: v[..., ::2]) if case == "noncontig" else (lambda v: v)
    a = self_attention(view(x1), h, cu_seqlens=cu, max_seqlen=max_seqlen)
    assert type(a.grad_fn).__name__ != FUSED
    ref = _stock_varlen(view(x2), h, cu, max_seqlen, 0.0)
    assert torch.equal(a, ref)
    g = torch.randn_like(a)
    a.backward(g)
    ref.backward(g)
    if device == "cpu":
        assert torch.equal(x1.grad, x2.grad)
    else:
        assert (x1.grad - x2.grad).abs().max() <= 2.0 ** -7 * x2.grad.abs().max()
    # against SDPA run on each sequence alone, and zeros outside every sequence
    xs = view(qkv)
    tol = 1e-5 if xs.dtype == torch.float32 else 2.0 ** -7
    cu_l = cu.tolist()
    for s0, n in _sequences(cu_l):
        one = _stock(xs[None, s0:s0 + n], h, None, 0.0)[0]
        assert (a[s0:s0 + n].float() - one.float()).abs().max() <= tol * (1 + one.float().abs().max()), (case, n)
    dead = _outside(cu_l, xs.shape[0]).to(device)
    assert (a[dead] == 0).all() and (x1.grad[dead] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("case", FALLBACKS)
def test_fallbacks_are_stock_cuda(case):
    _check_fallback(case, "cuda")


@pytest.mark.parametrize("case", FALLBACKS + ["bf16"])
def test_fallbacks_are_stock_cpu(case):
    _check_fallback(case, "cpu")


def test_stock_expression_marks_long_sequences_nan():
    qkv = torch.randn(50, 3 * 2 * 16)
    cu = torch.tensor([0, 10, 40, 50], dtype=torch.int32)
    out = self_attention(qkv, 2, cu_seqlens=cu, max_seqlen=20)
    assert torch.isnan(out[10:40]).all() and torch.isfinite(out[:10]).all() and torch.isfinite(out[40:]).all()


@pytest.mark.gpu
def test_misaligned_view_matches_aligned_copy():
    qkv, dout = _make(300, 2, torch.bfloat16)
    cu = torch.tensor([0, 100, 300], dtype=torch.int32, device="cuda")
    flat = torch.empty(qkv.numel() + 1, dtype=qkv.dtype, device="cuda")
    view = flat[1:].view_as(qkv)
    view.copy_(qkv)
    assert view.data_ptr() % 16 != 0
    a = _fused(view, 2, cu, 0.1, dout, max_seqlen=200, rng_seed=5)
    c = _fused(qkv, 2, cu, 0.1, dout, max_seqlen=200, rng_seed=5)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


def test_bad_arguments_raise():
    qkv = torch.zeros(8, 384)
    cu = torch.tensor([0, 8], dtype=torch.int32)
    bad = [
        dict(mask=torch.ones(1, 1, 1, 8, dtype=torch.bool), cu_seqlens=cu),
        dict(cu_seqlens=cu.long()),
        dict(cu_seqlens=cu.view(1, 2)),
        dict(cu_seqlens=cu[:1]),
        dict(cu_seqlens=[0, 8]),
        dict(cu_seqlens=cu.to("meta")),
        dict(cu_seqlens=cu, max_seqlen=0),
        dict(cu_seqlens=cu, max_seqlen=8.0),
        dict(max_seqlen=8),
    ]
    for kw in bad:
        mask = kw.pop("mask", None)
        with pytest.raises(ValueError):
            self_attention(qkv, 2, mask, **kw)
    with pytest.raises(ValueError):
        self_attention(torch.zeros(8, 10), 2, cu_seqlens=cu)


@pytest.mark.gpu
def test_binding_rejects_bad_arguments():
    from byteps_b200 import _native

    cu = _native.cuda()
    buf = torch.zeros(1 << 20, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(1 << 16, device="cuda")
    offs = torch.tensor([0, 8, 8], dtype=torch.int32, device="cuda")
    b, l, c = buf.data_ptr(), lse.data_ptr(), offs.data_ptr()
    ok = dict(qkv=b, dtype=1, T=8, N=2, H=1, D=64, max_seqlen=8, cu_seqlens=c, out=b, lse=l)
    cases = [dict(dtype=0), dict(D=32), dict(max_seqlen=0), dict(max_seqlen=513), dict(N=0), dict(N=65536),
             dict(H=0), dict(H=65536), dict(T=0), dict(qkv=0), dict(qkv=b + 2), dict(out=b + 8), dict(lse=0),
             dict(lse=l + 2), dict(cu_seqlens=0), dict(cu_seqlens=c + 2)]
    for bad in cases:
        a = dict(ok, **bad)
        with pytest.raises(ValueError):
            cu.attn_varlen_fwd(a["qkv"], a["dtype"], a["T"], a["N"], a["H"], a["D"], a["max_seqlen"],
                               a["cu_seqlens"], 0, 0, 1.0, a["out"], a["lse"], 0)
        with pytest.raises(ValueError):
            cu.attn_varlen_bwd(a["qkv"], a["out"], b, a["lse"], a["dtype"], a["T"], a["N"], a["H"], a["D"],
                               a["max_seqlen"], a["cu_seqlens"], 0, 0, 1.0, l, b, 0)
    with pytest.raises(ValueError):   # misaligned dout, delta, dqkv
        cu.attn_varlen_bwd(b, b, b + 2, l, 1, 8, 2, 1, 64, 8, c, 0, 0, 1.0, l, b, 0)
    with pytest.raises(ValueError):
        cu.attn_varlen_bwd(b, b, b, l, 1, 8, 2, 1, 64, 8, c, 0, 0, 1.0, l + 1, b, 0)
    with pytest.raises(ValueError):
        cu.attn_varlen_bwd(b, b, b, l, 1, 8, 2, 1, 64, 8, c, 0, 0, 1.0, l, b + 4, 0)


# ---------------------------------------------------------------------------------------------- build
def test_varlen_kernels_compile_without_spills(tmp_path):
    from byteps_b200 import _build

    nvcc = _build._nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "byteps_b200", "csrc", "kernels", "attn_varlen.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + _build.ARCH_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                                         str(tmp_path / "attn_varlen.o")],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    found = 0
    for block in r.stderr.split("Compiling entry function '")[1:]:
        assert not re.match(r"_ZN\S*attn_(fwd|bwd_dq|bwd_dkv)_kernel", block), block[:200]
        if not re.match(r"_ZN\S*attn_varlen_(fwd|bwd_dq|bwd_dkv)_kernel", block):
            continue
        found += 1
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block[:400]
    assert found == 12, found


# ---------------------------------------------------------------------------------------------- model
def _padded_as_stream(lengths, s):
    cu = [0]
    for n in lengths:
        cu += [cu[-1] + n, cu[-1] + s]
    return torch.tensor(cu, dtype=torch.int32)


def test_bert_packed_stream_matches_key_padding_mask_cpu():
    """bert_tiny in fp32 on the CPU (stock attention): a padded batch written as a stream, each row's padding run a
    sequence of its own, gives the key-padding-mask model's real-token logits, loss and gradients."""
    b, s = 3, 24
    lengths = [24, 9, 17]
    torch.manual_seed(0)
    model = bert_tiny(dropout=0.0)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 1000, (b, s), generator=g)
    type_ids = torch.randint(0, 2, (b, s), generator=g)
    attend = torch.arange(s)[None, :] < torch.tensor(lengths)[:, None]
    labels = torch.where(attend, torch.randint(0, 1000, (b, s), generator=g), torch.full((b, s), -100))
    nsp = torch.randint(0, 2, (b,), generator=g)
    cu = _padded_as_stream(lengths, s)
    nsp_packed = torch.full((2 * b,), -100)
    nsp_packed[0::2] = nsp

    def run(**kw):
        model.zero_grad()
        logits, nsp_logits = model(ids, type_ids, **{k: v for k, v in kw.items() if k not in ("labels", "nsp")})
        loss = model(ids, type_ids, mlm_labels=kw["labels"], nsp_labels=kw["nsp"],
                     **{k: v for k, v in kw.items() if k not in ("labels", "nsp")})
        loss.backward()
        return logits, nsp_logits, loss.detach(), {n: p.grad.clone() for n, p in model.named_parameters()}

    la, na, loss_a, ga = run(mask=attend.view(b, 1, 1, s), labels=labels, nsp=nsp)
    lp, np_, loss_p, gp = run(cu_seqlens=cu, labels=labels, nsp=nsp_packed)
    assert np_.shape == (2 * b, 2)
    torch.testing.assert_close(lp[attend], la[attend], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(np_[0::2], na, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(loss_p, loss_a, rtol=1e-5, atol=1e-6)
    for n in ga:
        torch.testing.assert_close(gp[n], ga[n], rtol=1e-4, atol=1e-6, msg=n)


def test_bert_packed_positions_and_labels_stay_in_range_cpu():
    """Offsets that put tokens outside every sequence, or a sequence past max_position, never index outside the
    position table; tokens outside every sequence take no MLM loss."""
    model = bert_tiny(dropout=0.0, max_position=16)
    ids = torch.randint(0, 1000, (2, 20))
    labels = torch.randint(0, 1000, (2, 20))
    cu = torch.tensor([4, 30, 30, 36], dtype=torch.int32)   # 4 leading and 4 trailing tokens outside
    loss = model(ids, cu_seqlens=cu, max_seqlen=40, mlm_labels=labels)
    assert torch.isfinite(loss)
    keep = labels.clone().view(-1)
    keep[:4] = -100
    keep[36:] = -100
    ref = model(ids, cu_seqlens=cu, max_seqlen=40, mlm_labels=keep.view(2, 20))
    assert torch.equal(loss, ref)
    with pytest.raises(ValueError):
        model(ids, mask=torch.ones(2, 1, 1, 20, dtype=torch.bool), cu_seqlens=cu)


_BERT_PACKED = """
import torch
import byteps_b200.torch as bps
from byteps_b200.models import bert_tiny
from byteps_b200.torch.graph import GraphedStep
PACKED, ALL, STEPS, OUT = %r, %r, %r, %r
bps.init()
torch.manual_seed(0)
kw = dict(fp8_linear=True, fused_norm=True, fused_loss=True) if ALL else {}
model = bert_tiny(fused_attention=True, dropout=0.0, **kw).cuda().to(torch.bfloat16).train()
opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=0.01),
                               named_parameters=model.named_parameters(), fused_update=True)
g = torch.Generator().manual_seed(1)
b, s = 8, 128
ids = torch.randint(0, 1000, (b, s), generator=g).cuda()
labels = torch.randint(0, 1000, (b, s), generator=g)
lengths = torch.randint(16, 129, (b,), generator=g)
attend = torch.arange(s)[None, :] < lengths[:, None]
labels = torch.where(attend, labels, torch.full_like(labels, -100)).cuda()
mask = attend.view(b, 1, 1, s).cuda()
cu = [0]
for n in lengths.tolist():
    cu += [cu[-1] + n, cu[-1] + s]
cu = torch.tensor(cu, dtype=torch.int32).cuda()

calls = [0]

def step():
    opt.zero_grad()
    # the second eager warm-up step reports any host synchronisation of the packed forward and backward as an error
    check = PACKED and calls[0] == 1
    calls[0] += 1
    if check:
        torch.cuda.set_sync_debug_mode("error")
    if PACKED:
        loss = model(ids, cu_seqlens=cu, max_seqlen=s, mlm_labels=labels)
    else:
        loss = model(ids, mask=mask, mlm_labels=labels)
    loss.backward()
    if check:
        torch.cuda.set_sync_debug_mode(0)
    opt.step()
    return loss

stepper = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams)
losses = [stepper().detach().float().item() for _ in range(STEPS)]
torch.save({"losses": losses, "params": {n: p.detach().float().cpu() for n, p in model.named_parameters()}}, OUT)
print("OK")
bps.shutdown()
"""


@pytest.mark.gpu
@pytest.mark.parametrize("all_fused", [False, True], ids=["alone", "fp8_norm_loss"])
def test_bert_tiny_graphed_packed_steps_track_padded(tmp_path, all_fused):
    """bert_tiny in bf16 with fused attention, fused AdamW and one CUDA graph per step: the packed stream (padding
    runs as their own sequences) tracks the key-padding-mask model within 1 %, and its forward and backward run
    without a host synchronisation."""
    runs = {}
    for packed in (False, True):
        out = str(tmp_path / ("%d.pt" % packed))
        assert "OK" in _run_py(_BERT_PACKED % (packed, all_fused, 6, out))
        runs[packed] = torch.load(out)
    for a, c in zip(runs[False]["losses"], runs[True]["losses"]):
        assert abs(a - c) <= 1e-2 * abs(a), (runs[False]["losses"], runs[True]["losses"])
    assert all(torch.isfinite(p).all() for p in runs[True]["params"].values())
