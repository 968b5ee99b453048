"""The labelled rows of a token stream gathered into fixed slots, for a masked-LM head that runs on them only
(kernels/mlm_gather.cu).

``gather_labelled(x, labels, capacity, ignore_index=-100)`` takes ``x`` [..., H] and int64 ``labels`` of shape
``x.shape[:-1]``, read as one stream of T tokens in row-major order.  It returns ``(rows, row_labels, dropped)``:
``rows`` [C, H] holds the rows of the tokens whose label is not ``ignore_index``, in token order, and
``row_labels`` [C] their labels, for C = ``capacity``.  Slots past the labelled count hold exact zeros and
``ignore_index``.  Labels outside any vocabulary still count as labelled.  The gradient flows back to ``x``: each
kept token gets its slot's gradient and every other token zero.

On CUDA, for contiguous fp32 / bf16 / fp16 ``x`` whose row is a multiple of 16 bytes, forward is two launches: one CTA
scans the labels and writes each token's slot, and a grid copies the rows.  Backward is one launch that writes every
element of dx, with no memset and no atomics.  The copies move bits exactly, so results are identical from run to
run.  Nothing is read back to the host and no launch depends on the labelled count, so the op captures into a CUDA
graph, and refreshing ``labels`` in place between replays selects the new positions.  A tensor whose data does not
start on a 16-byte boundary is copied to one that does first.  Every other input runs the stock expression
(``_stock``): ``x`` padded with one zero row and indexed with
``torch.nonzero_static(labels != ignore_index, size=C, fill_value=T)``.

On overflow, when more than C tokens are labelled, the first C in token order are kept.  ``dropped`` is a 0-dim int64
device tensor holding the count of labelled tokens past C (0 when none is dropped).
"""
from __future__ import annotations

import torch

from .. import _native
from .ln import _aligned

# x dtype -> kernel dtype code (WireDType of kernels/pushpull.cuh)
_CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


class _GatherLabelledFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, labels, capacity, ignore_index):
        cu = _native.cuda()
        x = _aligned(x)
        t, h = labels.numel(), x.shape[-1]
        dev = x.device
        rows = torch.empty(capacity, h, dtype=x.dtype, device=dev)
        row_labels = torch.empty(capacity, dtype=torch.int64, device=dev)
        slot = torch.empty(t, dtype=torch.int32, device=dev)
        src = torch.empty(capacity, dtype=torch.int32, device=dev)
        dropped = torch.empty((), dtype=torch.int64, device=dev)
        cu.mlm_gather_fwd(x.data_ptr(), labels.data_ptr(), _CODES[x.dtype], t, h, capacity, ignore_index,
                          rows.data_ptr(), row_labels.data_ptr(), slot.data_ptr(), src.data_ptr(), dropped.data_ptr(),
                          torch.cuda.current_stream(dev).cuda_stream)
        ctx.save_for_backward(slot)
        ctx.shape = x.shape
        ctx.mark_non_differentiable(row_labels, dropped)
        ctx.set_materialize_grads(False)   # no zero-filled gradients for the integer outputs
        return rows, row_labels, dropped

    @staticmethod
    def backward(ctx, drows, _dlabels, _ddropped):
        if drows is None:
            return None, None, None, None
        (slot,) = ctx.saved_tensors
        cu = _native.cuda()
        capacity, h = drows.shape
        drows = _aligned(drows.contiguous())
        dx = torch.empty(ctx.shape, dtype=drows.dtype, device=drows.device)
        cu.mlm_scatter_bwd(drows.data_ptr(), slot.data_ptr(), _CODES[drows.dtype], slot.numel(), h, capacity,
                           dx.data_ptr(), torch.cuda.current_stream(drows.device).cuda_stream)
        return dx, None, None, None


def _stock(x: torch.Tensor, labels: torch.Tensor, capacity: int, ignore_index: int):
    """The expression the kernels compute, in stock torch ops (no host synchronisation on CUDA either)."""
    h = x.shape[-1]
    flat, lab = x.reshape(-1, h), labels.reshape(-1)
    t = lab.numel()
    keep = lab != ignore_index
    idx = torch.nonzero_static(keep, size=capacity, fill_value=t).squeeze(1)
    rows = torch.cat([flat, flat.new_zeros(1, h)])[idx]
    row_labels = torch.cat([lab, lab.new_full((1,), ignore_index)])[idx]
    dropped = (keep.sum() - capacity).clamp_min(0)
    return rows, row_labels, dropped


def _fusable(x: torch.Tensor, labels: torch.Tensor) -> bool:
    return (x.is_cuda and x.dtype in _CODES and x.dim() >= 1 and x.numel() > 0 and x.is_contiguous()
            and (x.shape[-1] * x.element_size()) % 16 == 0 and labels.is_contiguous()
            and labels.device == x.device and labels.numel() < 2 ** 31)


def gather_labelled(x: torch.Tensor, labels: torch.Tensor, capacity: int, ignore_index: int = -100):
    """``(rows [C, H], row_labels [C], dropped)``: the rows of ``x`` [..., H] whose label is not ``ignore_index``, the
    first C = ``capacity`` in token order, with their labels; empty slots hold zeros and ``ignore_index``, and
    ``dropped`` (0-dim int64) counts the labelled tokens past C."""
    if x.dim() < 1 or tuple(labels.shape) != tuple(x.shape[:-1]):
        raise ValueError("labels must have shape x.shape[:-1] = %s, got %s" % (tuple(x.shape[:-1]),
                                                                              tuple(labels.shape)))
    if labels.dtype != torch.int64:
        raise ValueError("labels must be int64, got %s" % labels.dtype)
    if isinstance(capacity, bool) or not isinstance(capacity, int) or capacity < 1:
        raise ValueError("capacity must be an int >= 1, got %r" % (capacity,))
    if _fusable(x, labels):
        return _GatherLabelledFn.apply(x, labels, capacity, int(ignore_index))
    return _stock(x, labels, capacity, int(ignore_index))
