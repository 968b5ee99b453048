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


def _stock(qkv, num_heads, mask, p):
    """The expression models/bert.py runs without fused attention."""
    b, s, e3 = qkv.shape
    e = e3 // 3
    q, k, v = qkv.view(b, s, 3, num_heads, e // num_heads).permute(2, 0, 3, 1, 4)
    a = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=p)
    return a.transpose(1, 2).reshape(b, s, e)


class _SelfAttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, mask, num_heads, p):
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
                    scale, out.data_ptr(), lse.data_ptr(), torch.cuda.current_stream(qkv.device).cuda_stream)
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
                    torch.cuda.current_stream(qkv.device).cuda_stream)
        return dqkv, None, None, None


def _key_padding(mask, b, s, device):
    """mask as a contiguous [B or 1, S] tensor when it is a key-padding mask the kernels take, else None."""
    if mask is None:
        return None
    if (mask.dtype not in _MASK_KINDS or mask.requires_grad or mask.device != device or mask.dim() != 4
            or mask.shape[0] not in (1, b) or tuple(mask.shape[1:]) != (1, 1, s)):
        return None
    return mask.reshape(mask.shape[0], s).contiguous()


def self_attention(qkv: torch.Tensor, num_heads: int, mask: Optional[torch.Tensor] = None, p: float = 0.0,
                   training: bool = True) -> torch.Tensor:
    """The [B, S, E] context of multi-head self-attention over ``qkv`` = [B, S, 3E] (Q, K, V of ``num_heads`` heads
    each), with the additive or boolean ``mask`` of ``F.scaled_dot_product_attention`` and dropout ``p`` on the
    attention probabilities when ``training``."""
    if not 0.0 <= p <= 1.0:
        raise ValueError("dropout probability has to be between 0 and 1, but got %r" % (p,))
    p = float(p) if training else 0.0
    if qkv.dim() != 3 or qkv.shape[-1] % (3 * num_heads) != 0:
        raise ValueError("qkv must be [B, S, 3 * num_heads * D], got %s with %d heads" % (tuple(qkv.shape), num_heads))
    b, s, e3 = qkv.shape
    fusable = (qkv.is_cuda and qkv.dtype in _CODES and e3 // (3 * num_heads) == _HEAD_DIM and 1 <= s <= _MAX_SEQ
               and b >= 1 and qkv.is_contiguous() and p < 1.0)
    if fusable:
        kp = _key_padding(mask, b, s, qkv.device)
        if mask is None or kp is not None:
            return _SelfAttentionFn.apply(qkv, kp, num_heads, p)
    return _stock(qkv, num_heads, mask, p)
