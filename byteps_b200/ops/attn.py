"""Self-attention of the BERT encoder fused into sm_90a kernels (kernels/attn.cu), reading Q, K and V in place from
the qkv projection's output.

``self_attention(qkv, num_heads, mask, p, training)`` takes the [B, S, 3E] output of the qkv projection (per row: Q,
K and V, each H heads of D) and returns the [B, S, E] context ``softmax(Q K^T / sqrt(D) + mask) -> dropout(p) -> @ V``
with its heads side by side, the layout the output projection reads.  On CUDA, for a contiguous bf16 / fp16 qkv with
D = 64, 1 <= S <= 512 and a mask that is None or a key-padding mask of shape [B, 1, 1, S] or [1, 1, 1, S] (bool, True
attends, or an additive float mask that needs no gradient), forward is one launch that writes the context and an fp32
log-sum-exp per query row, and backward is two launches that write d(qkv) as one [B, S, 3E] tensor.  Every other input
runs the stock view / permute / ``F.scaled_dot_product_attention`` / reshape expression, which computes the same
function.  A qkv whose data does not start on a 16-byte boundary is copied to one that does first.

A query row whose keys are all masked gives a zero context and zero gradients, as SDPA does.  Dropout bits come from
Philox4x32-10 keyed by a (seed, offset) pair drawn on the device from torch's CUDA generator on every call (nothing is
drawn at p = 0 or in eval mode), so ``torch.manual_seed`` reproduces them and each replay of a captured CUDA graph
draws new ones; element ((b H + h) S + q) S + k of the attention matrix is kept when word i % 4 of the Philox block
with counter (i / 4, offset) is below (1 - p) 2^32, and the backward regenerates the bits.  Both directions are
deterministic: no atomics, results bit-identical from run to run.

Packed sequences: with ``cu_seqlens`` (device int32 [N + 1]) the rows of ``qkv`` flattened to [T, 3E] are one stream
of tokens in which sequence n is tokens [cu[n], cu[n + 1]), and attention stays inside each sequence.  ``max_seqlen``
bounds every length (default T); it fixes the kernels' grid, so a step with a fixed T and a fixed number of sequence
slots (pad cu_seqlens by repeating its last value) captures into one CUDA graph and cu_seqlens can be refreshed in
place between replays.  Nothing reads cu_seqlens on the host.  Tokens outside every sequence (before cu[0] or from
cu[N] on) get a zero context and zero gradients.  On CUDA, for a contiguous bf16 / fp16 qkv with D = 64 and
max_seqlen <= 512, three kernels of kernels/attn_varlen.cu run; a sequence longer than max_seqlen then gets NaN in
its context and gradient rows.  Every other input runs SDPA over the whole stream with a block-diagonal additive mask
built on the device.  Dropout element (h, t, u) of sequence n, for query token t and key token u, has index
i = (h T + t) 512 + (u - cu[n]) in the same Philox scheme.

Causal attention: with ``causal=True`` query q attends to key k only when k <= q (in the packed form, positions within
the sequence), on top of any key-padding mask.  The kernels then visit only the key tiles on or below the diagonal
(kernels/attn_causal.cu), about half the work at S = 512; the fast-path conditions and the dropout numbering are the
ones above, so a kept element is one the bidirectional call with the same seed keeps.  Every other input runs the
stock expression with the causal mask: SDPA with ``is_causal=True`` without a mask, an explicit combined mask with one
(SDPA takes only one of the two), and for packed streams the block-diagonal mask intersected with t >= u.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from .. import _native
from .ln import _aligned, _keep_threshold, _ptr

# activation dtype -> kernel dtype code (WireDType of kernels/pushpull.cuh)
_CODES = {torch.bfloat16: 1, torch.float16: 2}
# mask dtype -> AttnMaskKind of kernels/attn.cuh
_MASK_KINDS = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2, torch.bool: 3}
_HEAD_DIM = 64
_MAX_SEQ = 512


def _causal_mask(mask, s, device):
    """``mask`` combined with the causal mask k <= q, as one bool or additive mask broadcast to [..., S, S]"""
    allowed = torch.ones(s, s, dtype=torch.bool, device=device).tril_()
    if mask.dtype == torch.bool:
        return mask & allowed
    return torch.where(allowed, mask, torch.full((), float("-inf"), dtype=mask.dtype, device=device))


def _stock(qkv, num_heads, mask, p, causal=False):
    """The expression models/bert.py runs without fused attention, with the causal mask when ``causal``."""
    b, s, e3 = qkv.shape
    e = e3 // 3
    q, k, v = qkv.view(b, s, 3, num_heads, e // num_heads).permute(2, 0, 3, 1, 4)
    if causal and mask is not None:
        a = F.scaled_dot_product_attention(q, k, v, attn_mask=_causal_mask(mask, s, qkv.device), dropout_p=p)
    elif causal:
        a = F.scaled_dot_product_attention(q, k, v, dropout_p=p, is_causal=True)
    else:
        a = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=p)
    return a.transpose(1, 2).reshape(b, s, e)


class _SelfAttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, mask, num_heads, p, causal):
        cu = _native.cuda()
        qkv = _aligned(qkv)
        b, s, e3 = qkv.shape
        e = e3 // 3
        out = torch.empty(b, s, e, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(b, num_heads, s, dtype=torch.float32, device=qkv.device)
        seed = None
        if p > 0.0:
            # (seed, offset) from torch's generator: graph-safe, so every replay of a captured step gets new bits
            seed = torch.randint(0, 2 ** 62, (2,), dtype=torch.int64, device=qkv.device)
        kind, bstride = (_MASK_KINDS[mask.dtype], s if mask.shape[0] > 1 else 0) if mask is not None else (0, 0)
        ctx.args = (_CODES[qkv.dtype], b, s, num_heads, _HEAD_DIM, kind, bstride,
                    _keep_threshold(p) if p > 0.0 else 0, 1.0 / (1.0 - p))
        code, _, _, _, _, _, _, keep, scale = ctx.args
        cu.attn_fwd(qkv.data_ptr(), code, b, s, num_heads, _HEAD_DIM, _ptr(mask), kind, bstride, _ptr(seed), keep,
                    scale, out.data_ptr(), lse.data_ptr(), torch.cuda.current_stream(qkv.device).cuda_stream,
                    causal=causal)
        ctx.causal = causal
        ctx.save_for_backward(qkv, out, lse, mask, seed)
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, out, lse, mask, seed = ctx.saved_tensors
        cu = _native.cuda()
        code, b, s, h, d, kind, bstride, keep, scale = ctx.args
        dout = _aligned(dout.to(qkv.dtype).contiguous())
        delta = torch.empty(b, h, s, dtype=torch.float32, device=qkv.device)
        dqkv = torch.empty_like(qkv)
        cu.attn_bwd(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), code, b, s, h, d, _ptr(mask),
                    kind, bstride, _ptr(seed), keep, scale, delta.data_ptr(), dqkv.data_ptr(),
                    torch.cuda.current_stream(qkv.device).cuda_stream, causal=ctx.causal)
        return dqkv, None, None, None, None


def _key_padding(mask, b, s, device):
    """mask as a contiguous [B or 1, S] tensor when it is a key-padding mask the kernels take, else None."""
    if mask is None:
        return None
    if (mask.dtype not in _MASK_KINDS or mask.requires_grad or mask.device != device or mask.dim() != 4
            or mask.shape[0] not in (1, b) or tuple(mask.shape[1:]) != (1, 1, s)):
        return None
    return mask.reshape(mask.shape[0], s).contiguous()


def _packed_tokens(cu_seqlens, t):
    """(index of the sequence of each token, whether it lies inside one) for a [T] arange, on the device"""
    n = cu_seqlens.numel() - 1
    seq = torch.searchsorted(cu_seqlens, t.to(cu_seqlens.dtype), right=True) - 1
    inside = (seq >= 0) & (seq < n)
    return seq.clamp(0, n - 1), inside


def _stock_varlen(qkv, num_heads, cu_seqlens, max_seqlen, p, causal=False):
    """SDPA over the whole stream with a block-diagonal additive mask, the expression the packed kernels compute; with
    ``causal`` the mask also requires key token <= query token.

    A token outside every sequence attends to itself only, so no row of the mask is all -inf (which SDPA turns into
    NaN on some backends), and its context is zeroed.  A sequence longer than max_seqlen gets NaN rows, as the
    kernels give."""
    shape, e3 = qkv.shape, qkv.shape[-1]
    x = qkv.reshape(-1, e3)
    t_all = x.shape[0]
    t = torch.arange(t_all, device=qkv.device)
    seq, inside = _packed_tokens(cu_seqlens, t)
    allowed = (seq[:, None] == seq[None, :]) & inside[:, None] & inside[None, :]
    if causal:
        allowed &= t[:, None] >= t[None, :]
    allowed |= torch.eye(t_all, dtype=torch.bool, device=qkv.device)
    mask = torch.zeros(t_all, t_all, dtype=qkv.dtype, device=qkv.device).masked_fill_(~allowed, float("-inf"))
    out = _stock(x.unsqueeze(0), num_heads, mask, p)[0]
    out = torch.where(inside[:, None], out, torch.zeros((), dtype=out.dtype, device=out.device))
    too_long = (cu_seqlens[1:] - cu_seqlens[:-1]) > max_seqlen
    out = out + torch.where(too_long[seq] & inside, float("nan"), 0.0).to(out.dtype)[:, None]
    return out.view(*shape[:-1], e3 // 3)


class _VarlenAttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, cu_seqlens, num_heads, max_seqlen, p, causal):
        cu = _native.cuda()
        qkv = _aligned(qkv)
        e3 = qkv.shape[-1]
        t = qkv.numel() // e3
        out = torch.empty(*qkv.shape[:-1], e3 // 3, dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty(num_heads, t, dtype=torch.float32, device=qkv.device)
        seed = None
        if p > 0.0:
            seed = torch.randint(0, 2 ** 62, (2,), dtype=torch.int64, device=qkv.device)
        ctx.args = (_CODES[qkv.dtype], t, cu_seqlens.numel() - 1, num_heads, _HEAD_DIM, max_seqlen,
                    _keep_threshold(p) if p > 0.0 else 0, 1.0 / (1.0 - p))
        code, _, n, _, _, _, keep, scale = ctx.args
        cu.attn_varlen_fwd(qkv.data_ptr(), code, t, n, num_heads, _HEAD_DIM, max_seqlen, cu_seqlens.data_ptr(),
                           _ptr(seed), keep, scale, out.data_ptr(), lse.data_ptr(),
                           torch.cuda.current_stream(qkv.device).cuda_stream, causal=causal)
        ctx.causal = causal
        ctx.save_for_backward(qkv, out, lse, cu_seqlens, seed)
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, out, lse, cu_seqlens, seed = ctx.saved_tensors
        cu = _native.cuda()
        code, t, n, h, d, max_seqlen, keep, scale = ctx.args
        dout = _aligned(dout.to(qkv.dtype).contiguous())
        delta = torch.empty(h, t, dtype=torch.float32, device=qkv.device)
        dqkv = torch.empty_like(qkv)
        cu.attn_varlen_bwd(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), code, t, n, h, d,
                           max_seqlen, cu_seqlens.data_ptr(), _ptr(seed), keep, scale, delta.data_ptr(),
                           dqkv.data_ptr(), torch.cuda.current_stream(qkv.device).cuda_stream, causal=ctx.causal)
        return dqkv, None, None, None, None, None


def _varlen(qkv, num_heads, mask, p, cu_seqlens, max_seqlen, causal):
    if mask is not None:
        raise ValueError("mask and cu_seqlens cannot be used together")
    if (not isinstance(cu_seqlens, torch.Tensor) or cu_seqlens.dim() != 1 or cu_seqlens.dtype != torch.int32
            or cu_seqlens.device != qkv.device or cu_seqlens.numel() < 2):
        raise ValueError("cu_seqlens must be a 1-D int32 tensor of at least 2 offsets on qkv's device")
    if qkv.dim() < 2 or qkv.shape[-1] % (3 * num_heads) != 0:
        raise ValueError("qkv must be [..., 3 * num_heads * D], got %s with %d heads" % (tuple(qkv.shape), num_heads))
    e3 = qkv.shape[-1]
    t = qkv.numel() // e3 if e3 else 0
    if max_seqlen is None:
        max_seqlen = t
    if isinstance(max_seqlen, bool) or not isinstance(max_seqlen, int) or max_seqlen < 1:
        raise ValueError("max_seqlen must be an int >= 1, got %r" % (max_seqlen,))
    n = cu_seqlens.numel() - 1
    fusable = (qkv.is_cuda and qkv.dtype in _CODES and e3 // (3 * num_heads) == _HEAD_DIM and t >= 1
               and max_seqlen <= _MAX_SEQ and n <= 65535 and num_heads <= 65535 and qkv.is_contiguous() and p < 1.0)
    if not fusable:
        return _stock_varlen(qkv, num_heads, cu_seqlens, max_seqlen, p, causal)
    return _VarlenAttentionFn.apply(qkv, cu_seqlens.contiguous(), num_heads, max_seqlen, p, causal)


def self_attention(qkv: torch.Tensor, num_heads: int, mask: Optional[torch.Tensor] = None, p: float = 0.0,
                   training: bool = True, *, cu_seqlens: Optional[torch.Tensor] = None,
                   max_seqlen: Optional[int] = None, causal: bool = False) -> torch.Tensor:
    """The [B, S, E] context of multi-head self-attention over ``qkv`` = [B, S, 3E] (Q, K, V of ``num_heads`` heads
    each), with the additive or boolean ``mask`` of ``F.scaled_dot_product_attention`` and dropout ``p`` on the
    attention probabilities when ``training``.

    With ``cu_seqlens`` the rows of ``qkv`` are one packed stream of sequences (see the module docstring), ``mask``
    must be None, and the result has ``qkv``'s shape with E columns.  With ``causal`` query q attends to key k only
    when k <= q (positions within the sequence for a packed stream), on top of ``mask``."""
    if not 0.0 <= p <= 1.0:
        raise ValueError("dropout probability has to be between 0 and 1, but got %r" % (p,))
    p = float(p) if training else 0.0
    if cu_seqlens is not None:
        return _varlen(qkv, num_heads, mask, p, cu_seqlens, max_seqlen, bool(causal))
    if max_seqlen is not None:
        raise ValueError("max_seqlen is only taken together with cu_seqlens")
    if qkv.dim() != 3 or qkv.shape[-1] % (3 * num_heads) != 0:
        raise ValueError("qkv must be [B, S, 3 * num_heads * D], got %s with %d heads" % (tuple(qkv.shape), num_heads))
    b, s, e3 = qkv.shape
    fusable = (qkv.is_cuda and qkv.dtype in _CODES and e3 // (3 * num_heads) == _HEAD_DIM and 1 <= s <= _MAX_SEQ
               and b >= 1 and qkv.is_contiguous() and p < 1.0)
    if fusable:
        kp = _key_padding(mask, b, s, qkv.device)
        if mask is None or kp is not None:
            return _SelfAttentionFn.apply(qkv, kp, num_heads, p, bool(causal))
    return _stock(qkv, num_heads, mask, p, bool(causal))
