"""Dropout, residual add and LayerNorm of the BERT encoder fused into one sm_90a kernel per direction (kernels/ln.cu).

``dropout_add_layer_norm(y, residual, weight, bias, p, eps, training)`` computes
``layer_norm(residual + dropout(y, p if training else 0))`` over the last dimension, and ``DropoutAddLayerNorm`` is
an ``nn.LayerNorm`` (same parameters and state_dict keys, plus a dropout probability ``p``) whose
``forward(y, residual=None)`` does the same.  On CUDA, contiguous fp32 / bf16 / fp16 rows of a width H that is a
multiple of 8 and at most 2048, with affine parameters in fp32 or the activation dtype, forward is one launch that
writes the output, z = residual + dropout(y), the per-row mean and rstd and a 1-bit keep mask, and backward is one
launch that writes d(residual), dy, dgamma and dbeta; torch runs dropout, the add and layer_norm as separate passes
each way.  Every other input takes the stock ``F.dropout`` / add / ``F.layer_norm`` composition, which computes the
same function.

Dropout bits come from Philox4x32-10 keyed by a (seed, offset) pair drawn on the device from torch's CUDA generator
on every call, so ``torch.manual_seed`` reproduces them and each replay of a captured CUDA graph draws new ones.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _native

# activation / parameter dtype -> kernel dtype code (WireDType of kernels/pushpull.cuh)
_CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
_UNIT = 8        # elements per mask byte; H must be a multiple of it
_MAX_H = 2048    # widest row a thread group holds in registers (kLnMaxH)


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def _keep_threshold(p: float) -> int:
    return min(int(round((1.0 - p) * 2.0 ** 32)), 2 ** 32 - 1)


class _DropoutAddLayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, residual, weight, bias, p, eps, grad):
        cu = _native.cuda()
        h = y.shape[-1]
        m = y.numel() // h
        code, wcode = _CODES[y.dtype], _CODES[weight.dtype]
        stream = torch.cuda.current_stream(y.device).cuda_stream
        f32 = dict(dtype=torch.float32, device=y.device)
        mean, rstd = torch.empty(m, **f32), torch.empty(m, **f32)
        out = torch.empty_like(y)
        drop = p > 0.0
        mask = seed = None
        if drop:
            mask = torch.empty(y.shape[:-1] + (h // _UNIT,), dtype=torch.uint8, device=y.device)
            # (seed, offset) from torch's generator: graph-safe, so every replay of a captured step gets new bits
            seed = torch.randint(0, 2 ** 62, (2,), dtype=torch.int64, device=y.device)
        # z is y when nothing is added or dropped, and only a backward reads it
        z = torch.empty_like(y) if grad and (drop or residual is not None) else None
        cu.ln_fwd(y.data_ptr(), _ptr(residual), code, wcode, m, h, float(eps), weight.data_ptr(), bias.data_ptr(),
                  _ptr(seed), _keep_threshold(p) if drop else 0, 1.0 / (1.0 - p), _ptr(z), out.data_ptr(),
                  mean.data_ptr(), rstd.data_ptr(), _ptr(mask), stream)
        ctx.save_for_backward(y if z is None else z, weight, mean, rstd, mask)
        ctx.p = p
        ctx.has_residual = residual is not None
        if mask is not None:
            ctx.mark_non_differentiable(mask)
        return out, mask

    @staticmethod
    def backward(ctx, dout, _dmask):
        z, weight, mean, rstd, mask = ctx.saved_tensors
        cu = _native.cuda()
        h = z.shape[-1]
        m = z.numel() // h
        code, wcode = _CODES[z.dtype], _CODES[weight.dtype]
        dout = dout.to(z.dtype).contiguous()
        stream = torch.cuda.current_stream(z.device).cuda_stream
        dweight, dbias = torch.empty_like(weight), torch.empty_like(weight)
        dres = torch.empty_like(z) if ctx.has_residual else None
        # without dropout dy is d(residual) itself: one tensor serves both
        dy = torch.empty_like(z) if (mask is not None or dres is None) else None
        nws, nctr = cu.ln_workspace(m, h)
        ws = torch.empty(nws, dtype=torch.float32, device=z.device)
        ctr = torch.zeros(nctr, dtype=torch.int32, device=z.device)
        cu.ln_bwd(dout.data_ptr(), z.data_ptr(), _ptr(mask), code, wcode, m, h, 1.0 / (1.0 - ctx.p), mean.data_ptr(),
                  rstd.data_ptr(), weight.data_ptr(), _ptr(dres), _ptr(dy), dweight.data_ptr(), dbias.data_ptr(),
                  ws.data_ptr(), ctr.data_ptr(), stream)
        if dy is None:
            dy = dres
        return dy, dres, dweight, dbias, None, None, None


def _fusable(y, residual, weight, bias, normalized_shape) -> bool:
    h = y.shape[-1] if y.dim() > 0 else 0
    return (y.is_cuda and y.dtype in _CODES and tuple(normalized_shape) == (h,) and h % _UNIT == 0
            and _UNIT <= h <= _MAX_H and y.numel() > 0 and y.is_contiguous()
            and weight is not None and bias is not None and weight.dtype in (torch.float32, y.dtype)
            and bias.dtype == weight.dtype and weight.shape == (h,) and bias.shape == (h,)
            and weight.is_contiguous() and bias.is_contiguous() and weight.device == y.device
            and bias.device == y.device
            and (residual is None or (residual.shape == y.shape and residual.dtype == y.dtype
                                      and residual.is_contiguous() and residual.device == y.device)))


def dropout_add_layer_norm(y: torch.Tensor, residual: Optional[torch.Tensor], weight: Optional[torch.Tensor],
                           bias: Optional[torch.Tensor], p: float, eps: float, training: bool,
                           return_mask: bool = False, normalized_shape: Optional[Sequence[int]] = None):
    """``layer_norm(residual + dropout(y, p if training else 0))`` over ``normalized_shape`` (default: the last
    dimension); ``residual`` may be None.

    With ``return_mask`` the result is ``(out, mask)``: the keep mask of the fused kernels, one uint8 per 8
    elements of a row (bit k = element 8j + k), shaped ``y.shape[:-1] + (H // 8,)``; None when no dropout was
    applied or the input took the stock composition."""
    if not 0.0 <= p <= 1.0:
        raise ValueError("dropout probability has to be between 0 and 1, but got %r" % (p,))
    p = float(p) if training else 0.0
    if normalized_shape is None:
        normalized_shape = tuple(weight.shape) if weight is not None else (y.shape[-1],)
    if p < 1.0 and _fusable(y, residual, weight, bias, normalized_shape):
        grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (y, residual, weight, bias))
        out, mask = _DropoutAddLayerNormFn.apply(y, residual, weight, bias, p, float(eps), grad)
    else:
        z = F.dropout(y, p, training) if p > 0.0 else y
        if residual is not None:
            z = residual + z
        out, mask = F.layer_norm(z, tuple(normalized_shape), weight, bias, eps), None
    return (out, mask) if return_mask else out


class DropoutAddLayerNorm(nn.LayerNorm):
    """``nn.LayerNorm`` applied to ``residual + dropout(y, p)``: ``forward(y, residual=None)``.  Dropout is active in
    training mode only, as ``nn.Dropout``."""

    def __init__(self, normalized_shape, eps=1e-5, elementwise_affine=True, bias=True, p=0.0, device=None,
                 dtype=None):
        super().__init__(normalized_shape, eps, elementwise_affine, bias, device, dtype)
        if not 0.0 <= p <= 1.0:
            raise ValueError("dropout probability has to be between 0 and 1, but got %r" % (p,))
        self.p = p

    def extra_repr(self):
        return super().extra_repr() + ", p=%g" % self.p

    def forward(self, y, residual=None):
        return dropout_add_layer_norm(y, residual, self.weight, self.bias, self.p, self.eps, self.training,
                                      normalized_shape=self.normalized_shape)
