"""Training-mode batch norm fused with the residual add and ReLU that follow it (kernels/bn_act.cu).

``BatchNormAct2d`` is an ``nn.BatchNorm2d`` (same parameters, buffers and state_dict keys) whose
``forward(x, residual=None)`` computes ``act(batch_norm(x) [+ residual])``.  On a CUDA, NHWC-contiguous
(channels_last) input in training mode it runs two sm_90a kernels forward (statistics, then apply + 1-bit ReLU
mask) and two backward (reduce, then apply), instead of torch's separate batch-norm, add, ReLU and
threshold-backward passes.  Every other input - CPU, eval mode, NCHW, C not a multiple of 8 - takes the stock
``F.batch_norm`` / add / ``relu`` composition, which computes the same function.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _native

# activation dtype -> kernel dtype code (WireDType of kernels/pushpull.cuh)
_CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
_UNIT = 8   # channels per thread and per mask byte


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def _nhwc(t: torch.Tensor) -> bool:
    return t.is_contiguous(memory_format=torch.channels_last)


class _BatchNormActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, bias, running_mean, running_var, momentum, eps, relu):
        cu = _native.cuda()
        n, c, h, w = x.shape
        m = n * h * w
        code = _CODES[x.dtype]
        stream = torch.cuda.current_stream(x.device).cuda_stream
        f32 = dict(dtype=torch.float32, device=x.device)
        mean, invstd = torch.empty(c, **f32), torch.empty(c, **f32)
        nws, nctr = cu.bn_act_workspace(m, c)
        ws = torch.empty(nws, **f32)
        ctr = torch.zeros(nctr, dtype=torch.int32, device=x.device)
        cu.bn_act_fwd_stats(x.data_ptr(), code, m, c, float(eps), float(momentum), _ptr(running_mean),
                            _ptr(running_var), mean.data_ptr(), invstd.data_ptr(), ws.data_ptr(), ctr.data_ptr(), stream)
        y = torch.empty_like(x)
        mask = torch.empty((m, c // _UNIT), dtype=torch.uint8, device=x.device) if relu else None
        cu.bn_act_fwd_apply(x.data_ptr(), _ptr(residual), code, m, c, mean.data_ptr(), invstd.data_ptr(),
                            weight.data_ptr(), bias.data_ptr(), bool(relu), y.data_ptr(), _ptr(mask), stream)
        ctx.save_for_backward(x, weight, mean, invstd, mask)
        ctx.has_residual = residual is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, invstd, mask = ctx.saved_tensors
        cu = _native.cuda()
        n, c, h, w = x.shape
        m = n * h * w
        code = _CODES[x.dtype]
        dy = dy.to(x.dtype).contiguous(memory_format=torch.channels_last)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        f32 = dict(dtype=torch.float32, device=x.device)
        dweight, dbias = torch.empty(c, **f32), torch.empty(c, **f32)
        nws, nctr = cu.bn_act_workspace(m, c)
        ws = torch.empty(nws, **f32)
        ctr = torch.zeros(nctr, dtype=torch.int32, device=x.device)
        cu.bn_act_bwd_reduce(dy.data_ptr(), x.data_ptr(), _ptr(mask), code, m, c, mean.data_ptr(), invstd.data_ptr(),
                             dweight.data_ptr(), dbias.data_ptr(), ws.data_ptr(), ctr.data_ptr(), stream)
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if ctx.has_residual else None
        cu.bn_act_bwd_apply(dy.data_ptr(), x.data_ptr(), _ptr(mask), code, m, c, mean.data_ptr(), invstd.data_ptr(),
                            weight.data_ptr(), dweight.data_ptr(), dbias.data_ptr(), dx.data_ptr(), _ptr(dres), stream)
        return dx, dres, dweight, dbias, None, None, None, None, None


class BatchNormAct2d(nn.BatchNorm2d):
    """``nn.BatchNorm2d`` followed by an optional residual add and activation (``act``: None or "relu")."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True, act=None,
                 device=None, dtype=None):
        super().__init__(num_features, eps, momentum, affine, track_running_stats, device, dtype)
        if act not in (None, "relu"):
            raise ValueError("BatchNormAct2d: act must be None or 'relu', got %r" % (act,))
        self.act = act

    def extra_repr(self):
        return super().extra_repr() + ", act=%s" % self.act

    def _fusable(self, x, residual, batch_stats):
        return (batch_stats and self.affine and x.is_cuda and x.dtype in _CODES and x.dim() == 4
                and self.weight.dtype == torch.float32 and x.size(1) % _UNIT == 0 and _nhwc(x)
                and x.numel() > x.size(1)
                and (residual is None or (residual.shape == x.shape and residual.dtype == x.dtype and _nhwc(residual))))

    def forward(self, x, residual=None):
        # statistics bookkeeping exactly as nn.BatchNorm2d.forward
        self._check_input_dim(x)
        factor = 0.0 if self.momentum is None else self.momentum
        if self.training and self.track_running_stats and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
            factor = 1.0 / float(self.num_batches_tracked) if self.momentum is None else self.momentum
        batch_stats = self.training or (self.running_mean is None and self.running_var is None)
        track = not self.training or self.track_running_stats
        running_mean = self.running_mean if track else None
        running_var = self.running_var if track else None
        if self._fusable(x, residual, batch_stats):
            return _BatchNormActFn.apply(x, residual, self.weight, self.bias, running_mean, running_var, factor,
                                         self.eps, self.act == "relu")
        y = F.batch_norm(x, running_mean, running_var, self.weight, self.bias, batch_stats, factor, self.eps)
        if residual is not None:
            y = y + residual
        if self.act == "relu":
            y = F.relu(y, inplace=True)
        return y
