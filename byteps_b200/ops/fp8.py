"""Linear layers in FP8 with delayed scaling: sm_90a cast kernels (kernels/fp8.cu) around cuBLASLt FP8 GEMMs.

``Fp8Linear`` is an ``nn.Linear`` (same parameters and state_dict keys) whose forward, for a CUDA input on sm_90
with x and weight both bf16 or both fp16, a bias absent or in that dtype, the last dimension K, the out_features N
and the flattened rows M all multiples of 16 and contiguous 16-byte aligned rows, runs

* forward:  x -> E4M3 rows (+ E4M3 x^T when the weight needs a gradient), W -> E4M3 rows (+ W^T when x needs one),
  each in one pass; ``y = _scaled_mm(x8, W8.t(), inv_x, inv_w, bias)``; only x^T, W^T (FP8) and the two inverse
  scales are saved;
* backward: dy -> E5M2 rows and dy^T in one pass that also writes the bias gradient (fp32 column sums);
  ``dx = _scaled_mm(dy8, WT8.t(), inv_dy, inv_w)``, ``dW = _scaled_mm(dyT8, xT8.t(), inv_dy, inv_x)``.

Every GEMM accumulates without fast accumulation.  Every other input runs ``F.linear`` itself.

Scaling (one fixed recipe): x, W and dy each keep an amax history of 16 floats, the next scale and a count in device
memory, written only by the kernels, so a step captures into a CUDA graph and the host never reads the state.  The
scale is ``s = fmax / max(max(history), 1e-12)`` (fmax 448 for E4M3, 57344 for E5M2).  The first forward and the
first backward of a module seed x / W and dy from the tensors themselves (an extra read-only pass); every later call
casts with the current s and then records its own amax.  Each cast writes the inverse scale it applied to a fresh
tensor that the GEMMs read, so a module called twice before its backward still uses the right scales.  A tensor with
an inf or NaN gets a NaN inverse scale - its GEMM outputs are non-finite, which a loss-scale check sees - and leaves
the state unchanged; finite values beyond fmax / s saturate.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _native

# input dtype -> kernel dtype code (WireDType of kernels/pushpull.cuh)
_CODES = {torch.bfloat16: 1, torch.float16: 2}
E4M3, E5M2 = 0, 1                  # Fp8Format of kernels/fp8.cuh
ROWS, COLS, BOTH = 1, 2, 3         # Fp8Layout
FP8_DTYPES = {E4M3: torch.float8_e4m3fn, E5M2: torch.float8_e5m2}
FP8_MAX = {E4M3: 448.0, E5M2: 57344.0}
HISTORY = 16
STATE_WORDS = HISTORY + 2          # Fp8State: hist[16], scale, count
X, W, DY = 0, 1, 2                 # rows of a ScalingState


class ScalingState:
    """Delayed-scaling state of one ``Fp8Linear``: ``buf`` is int32 [3, 18] on the device, one Fp8State per tensor
    (x, W, dy): ``buf.view(torch.float32)[i, :16]`` the amax history, ``[i, 16]`` the scale and ``buf[i, 17]`` the
    count of recorded amaxes.  It is int32 and not a buffer of the module, so ``.to(dtype)`` and the state_dict never
    see it.  ``seeded`` holds the host-side first-call flags of forward and backward."""

    def __init__(self, device):
        self.buf = torch.zeros(3, STATE_WORDS, dtype=torch.int32, device=device)
        self.seeded = [False, False]

    def row(self, i: int) -> torch.Tensor:
        return self.buf[i]

    def history(self, i: int) -> torch.Tensor:
        return self.buf.view(torch.float32)[i, :HISTORY]

    def scale(self, i: int) -> torch.Tensor:
        return self.buf.view(torch.float32)[i, HISTORY]

    def count(self, i: int) -> torch.Tensor:
        return self.buf[i, HISTORY + 1]


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def seed(x: torch.Tensor, state: torch.Tensor, fmt: int) -> None:
    """Seed one Fp8State (an int32 [18] row) from max |x| of a contiguous 2-D bf16 / fp16 tensor."""
    cu = _native.cuda()
    m, k = x.shape
    nws, nctr = cu.fp8_amax_workspace(m, k, _CODES[x.dtype])
    ws = torch.empty(nws, dtype=torch.float32, device=x.device)
    ctr = torch.zeros(nctr, dtype=torch.int32, device=x.device)
    cu.fp8_amax(x.data_ptr(), _CODES[x.dtype], m, k, fmt, state.data_ptr(), ws.data_ptr(), ctr.data_ptr(),
                _stream(x))


def cast(x: torch.Tensor, state: torch.Tensor, fmt: int, layout: int, dbias_dtype: Optional[torch.dtype] = None):
    """FP8 copies of a contiguous 2-D bf16 / fp16 tensor [M, K] at the state's current scale, then the state's
    update.  Returns (rows [M, K] or None, transposed [K, M] or None, the inverse scale applied (fp32, 0-d), the
    column sums of x in ``dbias_dtype`` or None)."""
    cu = _native.cuda()
    m, k = x.shape
    dev = x.device
    f8 = FP8_DTYPES[fmt]
    rows = torch.empty(m, k, dtype=f8, device=dev) if layout & ROWS else None
    cols = torch.empty(k, m, dtype=f8, device=dev) if layout & COLS else None
    inv = torch.empty((), dtype=torch.float32, device=dev)
    dbias = torch.empty(k, dtype=dbias_dtype, device=dev) if dbias_dtype is not None else None
    nws, nctr = cu.fp8_cast_workspace(m, k, _CODES[x.dtype], fmt, layout, dbias is not None)
    ws = torch.empty(nws, dtype=torch.float32, device=dev)
    ctr = torch.zeros(nctr, dtype=torch.int32, device=dev)
    cu.fp8_cast(x.data_ptr(), _CODES[x.dtype], m, k, fmt, layout, state.data_ptr(),
                0 if rows is None else rows.data_ptr(), 0 if cols is None else cols.data_ptr(), inv.data_ptr(),
                0 if dbias is None else dbias.data_ptr(), ws.data_ptr(), ctr.data_ptr(), _stream(x))
    return rows, cols, inv, dbias


def _gemm(a, b, scale_a, scale_b, out_dtype, bias=None):
    return torch._scaled_mm(a, b, scale_a, scale_b, bias=bias, out_dtype=out_dtype, use_fast_accum=False)


class _Fp8LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, st):
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        k = x.shape[-1]
        x2 = x.view(-1, k)
        if not st.seeded[0]:
            seed(x2, st.row(X), E4M3)
            seed(weight, st.row(W), E4M3)
            st.seeded[0] = True
        x8, xt8, inv_x, _ = cast(x2, st.row(X), E4M3, ROWS | (COLS if need_dw else 0))
        w8, wt8, inv_w, _ = cast(weight, st.row(W), E4M3, ROWS | (COLS if need_dx else 0))
        y = _gemm(x8, w8.t(), inv_x, inv_w, x.dtype, bias)
        ctx.save_for_backward(xt8, wt8, inv_x, inv_w)
        ctx.st, ctx.x_shape, ctx.dtypes = st, x.shape, (x.dtype, weight.dtype, None if bias is None else bias.dtype)
        return y.view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        xt8, wt8, inv_x, inv_w = ctx.saved_tensors
        need_dx, need_dw, need_db = ctx.needs_input_grad[:3]
        x_dtype, w_dtype, b_dtype = ctx.dtypes
        st = ctx.st
        dy2 = dy.to(x_dtype).reshape(-1, dy.shape[-1]).contiguous()
        if dy2.data_ptr() % 16:
            dy2 = dy2.clone()
        if not st.seeded[1]:
            seed(dy2, st.row(DY), E5M2)
            st.seeded[1] = True
        layout = (ROWS if need_dx else 0) | (COLS if need_dw else 0)
        dy8, dyt8, inv_dy, db = cast(dy2, st.row(DY), E5M2, layout or ROWS, b_dtype if need_db else None)
        dx = dw = None
        if need_dx:
            dx = _gemm(dy8, wt8.t(), inv_dy, inv_w, x_dtype).view(ctx.x_shape)
        if need_dw:
            dw = _gemm(dyt8, xt8.t(), inv_dy, inv_x, w_dtype)
        return dx, dw, db, None


_SM90 = {}


def _sm90(device: torch.device) -> bool:
    i = device.index if device.index is not None else torch.cuda.current_device()
    if i not in _SM90:
        _SM90[i] = torch.cuda.get_device_capability(i) == (9, 0)
    return _SM90[i]


def _fusable(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> bool:
    if not (x.is_cuda and x.dtype in _CODES and weight.dtype == x.dtype and x.dim() >= 1 and weight.dim() == 2):
        return False
    n, k = weight.shape
    m = x.numel() // k if k else 0
    return (x.shape[-1] == k and m > 0 and m % 16 == 0 and k % 16 == 0 and n % 16 == 0
            and x.is_contiguous() and weight.is_contiguous() and x.data_ptr() % 16 == 0
            and weight.data_ptr() % 16 == 0 and weight.device == x.device
            and (bias is None or (bias.dtype == x.dtype and bias.shape == (n,) and bias.device == x.device
                                  and bias.is_contiguous()))
            and _sm90(x.device))


class Fp8Linear(nn.Linear):
    """``nn.Linear`` whose matrix products run in FP8 with delayed scaling where the input allows it (see the
    module docstring); same parameters and state_dict as ``nn.Linear``."""

    def __init__(self, in_features, out_features, bias=True, device=None, dtype=None):
        super().__init__(in_features, out_features, bias, device, dtype)
        self._fp8 = None

    def scaling_state(self, device) -> ScalingState:
        """The delayed-scaling state on ``device``, allocated (and to be seeded again) when the module has none
        there yet."""
        device = torch.device(device)
        if self._fp8 is None or self._fp8.buf.device != device:
            self._fp8 = ScalingState(device)
        return self._fp8

    def forward(self, x):
        if _fusable(x, self.weight, self.bias):
            return _Fp8LinearFn.apply(x, self.weight, self.bias, self.scaling_state(x.device))
        return F.linear(x, self.weight, self.bias)
