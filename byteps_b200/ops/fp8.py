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

``fp8_gelu_mlp(x, fc1, fc2)`` is ``fc2(F.gelu(fc1(x)))`` for two ``Fp8Linear`` with the GELU inside the casts next
to it: forward, fc1's output z is cast to E4M3 for fc2 as gelu(z) (``ACT_GELU``), so h = gelu(z) is never written in
bf16 / fp16; backward, fc2's dx is cast to E5M2 for fc1 as gelu_backward(dh, z) (``ACT_DGELU``), with fc1's bias
gradient, so dz is never written either.  The kernels round the activation to the input dtype before anything else,
so every output, gradient and scaling state equals the composition's bit for bit; only the kernels that run change.

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
ACT_NONE, ACT_GELU, ACT_DGELU = 0, 1, 2   # Fp8Act
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


def cast(x: torch.Tensor, state: torch.Tensor, fmt: int, layout: int, dbias_dtype: Optional[torch.dtype] = None,
         *, act: int = ACT_NONE, aux: Optional[torch.Tensor] = None, counters: Optional[torch.Tensor] = None):
    """FP8 copies of a contiguous 2-D bf16 / fp16 tensor [M, K] at the state's current scale, then the state's
    update.  Returns (rows [M, K] or None, transposed [K, M] or None, the inverse scale applied (fp32, 0-d), the
    column sums of x in ``dbias_dtype`` or None).

    ``act`` casts a function of x in its place, rounded to x's dtype first: ``ACT_GELU`` gelu(x) (no ``dbias_dtype``)
    and ``ACT_DGELU`` ``torch.ops.aten.gelu_backward(x, aux)``, ``aux`` a tensor like x.  ``counters``, if given, is
    a zeroed int32 tensor of at least the counters the launch needs (``counters_for``), so that several casts can
    share one zero fill."""
    cu = _native.cuda()
    m, k = x.shape
    if aux is not None and (aux.shape != x.shape or aux.dtype != x.dtype or aux.device != x.device
                            or not aux.is_contiguous()):
        raise ValueError("fp8 cast: aux must be a contiguous tensor of x's shape, dtype and device")
    dev = x.device
    f8 = FP8_DTYPES[fmt]
    rows = torch.empty(m, k, dtype=f8, device=dev) if layout & ROWS else None
    cols = torch.empty(k, m, dtype=f8, device=dev) if layout & COLS else None
    inv = torch.empty((), dtype=torch.float32, device=dev)
    dbias = torch.empty(k, dtype=dbias_dtype, device=dev) if dbias_dtype is not None else None
    nws, nctr = cu.fp8_cast_workspace(m, k, _CODES[x.dtype], fmt, layout, dbias is not None, act)
    ws = torch.empty(nws, dtype=torch.float32, device=dev)
    if counters is None:
        ctr = torch.zeros(nctr, dtype=torch.int32, device=dev)
    elif counters.numel() < nctr or counters.dtype != torch.int32:
        raise ValueError("fp8 cast: counters needs %d int32 words" % nctr)
    else:
        ctr = counters
    cu.fp8_cast(x.data_ptr(), _CODES[x.dtype], m, k, fmt, layout, state.data_ptr(),
                0 if rows is None else rows.data_ptr(), 0 if cols is None else cols.data_ptr(), inv.data_ptr(),
                0 if dbias is None else dbias.data_ptr(), ws.data_ptr(), ctr.data_ptr(), _stream(x), act,
                0 if aux is None else aux.data_ptr())
    return rows, cols, inv, dbias


def counters_for(m: int, k: int, dtype: torch.dtype, fmt: int, layout: int, dbias: bool = False,
                 act: int = ACT_NONE) -> int:
    """The zeroed int32 counters one ``cast`` of an [m, k] ``dtype`` tensor needs."""
    return _native.cuda().fp8_cast_workspace(m, k, _CODES[dtype], fmt, layout, dbias, act)[1]


def _zeroed_counters(device, *sizes):
    """Zeroed counters for several casts, filled in one launch: one view per size."""
    return torch.zeros(sum(sizes), dtype=torch.int32, device=device).split(list(sizes))


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
    if not (x.is_cuda and x.dtype in _CODES and x.dim() >= 1 and weight.dim() == 2):
        return False
    k = weight.shape[1]
    m = x.numel() // k if k else 0
    return (x.shape[-1] == k and m > 0 and m % 16 == 0 and x.is_contiguous() and x.data_ptr() % 16 == 0
            and _weight_fusable(weight, bias, x.dtype, x.device) and _sm90(x.device))


def _weight_fusable(weight: torch.Tensor, bias: Optional[torch.Tensor], dtype: torch.dtype,
                    device: torch.device) -> bool:
    """The weight and bias half of ``_fusable``, for an input of ``dtype`` on ``device``."""
    if not (weight.dtype == dtype and weight.dim() == 2):
        return False
    n, k = weight.shape
    return (k % 16 == 0 and n % 16 == 0 and weight.is_contiguous() and weight.data_ptr() % 16 == 0
            and weight.device == device
            and (bias is None or (bias.dtype == dtype and bias.shape == (n,) and bias.device == device
                                  and bias.is_contiguous())))


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


class _Fp8GeluMlpFn(torch.autograd.Function):
    """fc2(gelu(fc1(x))) for two Fp8Linear: each step is the one ``_Fp8LinearFn`` takes for that layer, with the
    GELU and its gradient inside the casts of fc2's input and fc1's output gradient."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, st1, st2, need_h):
        need_dx, need_dw1, _, need_dw2 = ctx.needs_input_grad[:4]
        k = x.shape[-1]
        x2 = x.view(-1, k)
        if not st1.seeded[0]:
            seed(x2, st1.row(X), E4M3)
            seed(w1, st1.row(W), E4M3)
            st1.seeded[0] = True
        x8, xt8, inv_x, _ = cast(x2, st1.row(X), E4M3, ROWS | (COLS if need_dw1 else 0))
        w18, w1t8, inv_w1, _ = cast(w1, st1.row(W), E4M3, ROWS | (COLS if need_dx else 0))
        z = _gemm(x8, w18.t(), inv_x, inv_w1, x.dtype, b1)
        if not st2.seeded[0]:
            seed(F.gelu(z), st2.row(X), E4M3)
            seed(w2, st2.row(W), E4M3)
            st2.seeded[0] = True
        m, i = z.shape
        h_layout, w2_layout = ROWS | (COLS if need_dw2 else 0), ROWS | (COLS if need_h else 0)
        ch, cw = _zeroed_counters(x.device, counters_for(m, i, x.dtype, E4M3, h_layout, act=ACT_GELU),
                                  counters_for(w2.shape[0], i, x.dtype, E4M3, w2_layout))
        h8, ht8, inv_h, _ = cast(z, st2.row(X), E4M3, h_layout, act=ACT_GELU, counters=ch)
        w28, w2t8, inv_w2, _ = cast(w2, st2.row(W), E4M3, w2_layout, counters=cw)
        y = _gemm(h8, w28.t(), inv_h, inv_w2, x.dtype, b2)
        ctx.save_for_backward(xt8, w1t8, z if need_h else None, ht8, w2t8, inv_x, inv_w1, inv_h, inv_w2)
        ctx.st, ctx.need_h, ctx.x_shape, ctx.i = (st1, st2), need_h, x.shape, i
        ctx.dtypes = (x.dtype, w1.dtype, None if b1 is None else b1.dtype, w2.dtype, None if b2 is None else b2.dtype)
        return y.view(*x.shape[:-1], w2.shape[0])

    @staticmethod
    def backward(ctx, dy):
        xt8, w1t8, z, ht8, w2t8, inv_x, inv_w1, inv_h, inv_w2 = ctx.saved_tensors
        need_dx, need_dw1, need_db1, need_dw2, need_db2 = ctx.needs_input_grad[:5]
        dtype, w1_dtype, b1_dtype, w2_dtype, b2_dtype = ctx.dtypes
        st1, st2 = ctx.st
        need_h = ctx.need_h
        dy2 = dy.to(dtype).reshape(-1, dy.shape[-1]).contiguous()
        if dy2.data_ptr() % 16:
            dy2 = dy2.clone()
        if not st2.seeded[1]:
            seed(dy2, st2.row(DY), E5M2)
            st2.seeded[1] = True
        m, n = dy2.shape
        i = ctx.i
        dy_layout = (ROWS if need_h else 0) | (COLS if need_dw2 else 0) or ROWS
        dz_layout = (ROWS if need_dx else 0) | (COLS if need_dw1 else 0) or ROWS
        sizes = [counters_for(m, n, dtype, E5M2, dy_layout, need_db2)]
        if need_h:
            sizes.append(counters_for(m, i, dtype, E5M2, dz_layout, need_db1, ACT_DGELU))
        ctr = _zeroed_counters(dy2.device, *sizes)
        dy8, dyt8, inv_dy, db2 = cast(dy2, st2.row(DY), E5M2, dy_layout, b2_dtype if need_db2 else None,
                                      counters=ctr[0])
        dx = dw1 = db1 = dw2 = None
        if need_dw2:
            dw2 = _gemm(dyt8, ht8.t(), inv_dy, inv_h, w2_dtype)
        if need_h:
            dh = _gemm(dy8, w2t8.t(), inv_dy, inv_w2, dtype)
            z2 = z.view(-1, i)
            if not st1.seeded[1]:
                seed(torch.ops.aten.gelu_backward(dh, z2), st1.row(DY), E5M2)
                st1.seeded[1] = True
            dz8, dzt8, inv_dz, db1 = cast(dh, st1.row(DY), E5M2, dz_layout, b1_dtype if need_db1 else None,
                                          act=ACT_DGELU, aux=z2, counters=ctr[1])
            if need_dx:
                dx = _gemm(dz8, w1t8.t(), inv_dz, inv_w1, dtype).view(ctx.x_shape)
            if need_dw1:
                dw1 = _gemm(dzt8, xt8.t(), inv_dz, inv_x, w1_dtype)
        return dx, dw1, db1, dw2, db2, None, None, None


def fp8_gelu_mlp(x: torch.Tensor, fc1: nn.Module, fc2: nn.Module) -> torch.Tensor:
    """``fc2(F.gelu(fc1(x)))`` with the GELU and its gradient fused into the FP8 casts when both layers are
    ``Fp8Linear`` and both would take their FP8 path (x for fc1, an [M, fc1.out_features] tensor of x's dtype for
    fc2); bit for bit the composition's outputs, gradients and scaling states.  Anything else is the composition."""
    if (isinstance(fc1, Fp8Linear) and isinstance(fc2, Fp8Linear) and _fusable(x, fc1.weight, fc1.bias)
            and fc2.weight.dim() == 2 and fc2.weight.shape[1] == fc1.weight.shape[0]
            and _weight_fusable(fc2.weight, fc2.bias, x.dtype, x.device)):
        w1, b1, w2, b2 = fc1.weight, fc1.bias, fc2.weight, fc2.bias
        need_h = torch.is_grad_enabled() and (x.requires_grad or w1.requires_grad
                                               or (b1 is not None and b1.requires_grad))
        return _Fp8GeluMlpFn.apply(x, w1, b1, w2, b2, fc1.scaling_state(x.device), fc2.scaling_state(x.device),
                                   need_h)
    return fc2(F.gelu(fc1(x)))
