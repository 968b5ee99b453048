"""Softmax cross-entropy over [M, V] logits in one sm_90a kernel per direction (kernels/xent.cu).

``softmax_cross_entropy(logits, target, ignore_index=-100, reduction="mean")`` computes
``F.cross_entropy(logits.float(), target, ignore_index=ignore_index, reduction=reduction)``: the result is fp32
whatever the logits dtype, and the gradient flows to the logits in their own dtype.  On CUDA, for contiguous 2-D
fp32 / bf16 / fp16 logits with a 16-byte aligned base and contiguous int64 targets, forward reads each row once and
writes the per-row log-sum-exp and loss, the count of rows not ignored and the reduced loss; backward reads each row
once and writes dlogits = g * (softmax - onehot).  Eager torch instead casts the logits to fp32, writes and keeps an
fp32 log-softmax, and runs three more full-size passes backward.  Every other input takes the stock expression above.

Nothing is read back to the host: the count and the gradient scale stay on the device, so the op captures into a
CUDA graph.  A target outside [0, V) that is not ``ignore_index`` gives a NaN loss (and NaN gradients in its row)
instead of torch's device-side assert.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .. import _native

# logits dtype -> kernel dtype code (WireDType of kernels/pushpull.cuh)
_CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
_MODES = {"none": 0, "sum": 1, "mean": 2}     # XentMode of kernels/xent.cuh


class _SoftmaxCrossEntropyFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, ignore_index, mode):
        cu = _native.cuda()
        m, v = logits.shape
        dev = logits.device
        stream = torch.cuda.current_stream(dev).cuda_stream
        f32 = dict(dtype=torch.float32, device=dev)
        lse, loss_rows, out = torch.empty(m, **f32), torch.empty(m, **f32), torch.empty((), **f32)
        count = torch.empty((), dtype=torch.int64, device=dev)
        nws, nctr = cu.xent_workspace(m)
        ws = torch.empty(nws, **f32)
        ctr = torch.zeros(nctr, dtype=torch.int32, device=dev)
        cu.xent_fwd(logits.data_ptr(), target.data_ptr(), _CODES[logits.dtype], m, v, ignore_index,
                    mode == _MODES["mean"], lse.data_ptr(), loss_rows.data_ptr(), out.data_ptr(), count.data_ptr(),
                    ws.data_ptr(), ctr.data_ptr(), stream)
        ctx.save_for_backward(logits, lse, target, count)
        ctx.ignore_index, ctx.mode = ignore_index, mode
        return loss_rows if mode == _MODES["none"] else out

    @staticmethod
    def backward(ctx, grad):
        logits, lse, target, count = ctx.saved_tensors
        cu = _native.cuda()
        m, v = logits.shape
        grad = grad.float().contiguous()
        dlogits = torch.empty_like(logits, memory_format=torch.contiguous_format)
        cu.xent_bwd(logits.data_ptr(), target.data_ptr(), _CODES[logits.dtype], m, v, ctx.ignore_index,
                    lse.data_ptr(), grad.data_ptr(), ctx.mode, count.data_ptr(), dlogits.data_ptr(),
                    torch.cuda.current_stream(logits.device).cuda_stream)
        return dlogits, None, None, None


def _fusable(logits: torch.Tensor, target: torch.Tensor) -> bool:
    return (logits.is_cuda and logits.dtype in _CODES and logits.dim() == 2 and logits.numel() > 0
            and logits.is_contiguous() and logits.data_ptr() % 16 == 0
            and target.dtype == torch.int64 and target.dim() == 1 and target.shape[0] == logits.shape[0]
            and target.is_contiguous() and target.device == logits.device)


def softmax_cross_entropy(logits: torch.Tensor, target: torch.Tensor, ignore_index: int = -100,
                          reduction: str = "mean") -> torch.Tensor:
    """``F.cross_entropy(logits.float(), target, ignore_index=ignore_index, reduction=reduction)`` for logits
    ``[M, V]`` and class-index targets ``[M]``; one fused kernel per direction where the input allows it."""
    if reduction not in _MODES:
        raise ValueError("%r is not a valid value for reduction" % (reduction,))
    if _fusable(logits, target):
        return _SoftmaxCrossEntropyFn.apply(logits, target, int(ignore_index), _MODES[reduction])
    return F.cross_entropy(logits.float(), target, ignore_index=ignore_index, reduction=reduction)
