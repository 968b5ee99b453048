"""Training-mode batch norm fused with the residual add and ReLU that follow it (kernels/bn_act.cu).

``BatchNormAct2d`` is an ``nn.BatchNorm2d`` (same parameters, buffers and state_dict keys) whose
``forward(x, residual=None)`` computes ``act(batch_norm(x) [+ residual])``.  On a CUDA, NHWC-contiguous
(channels_last) input in training mode it runs one sm_90a kernel forward (statistics, grid barrier, apply + 1-bit
ReLU mask) and one backward (reduce, grid barrier, apply), or two each (the same phases as separate launches) where
the device cannot run the single-launch kernels at that shape, instead of torch's separate batch-norm, add, ReLU
and threshold-backward passes.  Every other input - CPU, eval mode, NCHW, C not a multiple of 8 - takes the stock
``F.batch_norm`` / add / ``relu`` composition, which computes the same function.  A channels_last view whose data
does not start on a 16-byte boundary (x, the residual or a gradient) is copied to one that does before the kernels
read it.

``forward(x, residual, pair=True)`` returns ``(y, alias of y)`` for an output with two consumers (a ResNet block's
output feeds the next block's conv1 and its skip path).  Autograd then hands backward the two gradients separately,
and the single-launch backward sums them as it reads them instead of a separate ``add`` pass over the tensor.

``forward(x, pool=nn.MaxPool2d(3, 2, 1), pair=True)`` returns ``pool`` of the output (and an alias of it): ResNet's
stem.  With ReLU on a fusable input the pooled kernels compute it in one launch per direction, without storing y, its
mask or the pool's indices; otherwise it is ``pool`` of the unpooled path.
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


#: Bytes of rows a block of the single-launch kernels may hold in shared memory; None: as many as fit.  Only tests
#: change it, to reach the fully held, partly held and fully streamed (0) cases at small shapes.
RESIDENT_CAP: Optional[int] = None


def _cap() -> int:
    return -1 if RESIDENT_CAP is None else int(RESIDENT_CAP)


def _sum_in_kernel(dy, dy2, x) -> bool:
    """Whether the kernel can read the second gradient beside dy: same dtype as x and dy (so that summing in the
    kernel rounds as torch's add would), shape of x, channels_last and 16-byte aligned."""
    return (dy2.dtype == x.dtype and dy.dtype == x.dtype and dy2.shape == x.shape and _nhwc(dy2)
            and dy2.data_ptr() % 16 == 0)


def _aligned(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """t, or a channels_last copy of it when its data does not start on the 16-byte boundary the kernels' vector
    loads need (a view at an odd element offset)."""
    return t if t is None or t.data_ptr() % 16 == 0 else t.clone(memory_format=torch.channels_last)


def _workspace(nws, nctr, device):
    return (torch.empty(nws, dtype=torch.float32, device=device),
            torch.zeros(nctr, dtype=torch.int32, device=device))


class _BatchNormActFn(torch.autograd.Function):
    """Each direction is one single-launch kernel where the device can run it at the input's shape
    (``bn_act_plan``), and the two-pass kernels otherwise.  With ``pair`` the output is ``(y, y.view_as(y))`` and
    backward receives the gradients of the two separately (None for an alias nobody used); the single-launch
    backward with a residual sums them in the kernel, every other path sums them in torch first."""

    @staticmethod
    def forward(ctx, x, residual, weight, bias, running_mean, running_var, momentum, eps, relu, pair=False):
        cu = _native.cuda()
        x, residual = _aligned(x), _aligned(residual)
        n, c, h, w = x.shape
        m = n * h * w
        code = _CODES[x.dtype]
        stream = torch.cuda.current_stream(x.device).cuda_stream
        f32 = dict(dtype=torch.float32, device=x.device)
        mean, invstd = torch.empty(c, **f32), torch.empty(c, **f32)
        y = torch.empty_like(x)
        mask = torch.empty((m, c // _UNIT), dtype=torch.uint8, device=x.device) if relu else None
        plan = cu.bn_act_plan(0, code, m, c, _cap())
        if plan is not None:
            ws, ctr = _workspace(plan["ws_floats"], plan["counters"], x.device)
            cu.bn_act_fwd(x.data_ptr(), _ptr(residual), code, m, c, float(eps), float(momentum), _ptr(running_mean),
                          _ptr(running_var), mean.data_ptr(), invstd.data_ptr(), weight.data_ptr(), bias.data_ptr(),
                          bool(relu), y.data_ptr(), _ptr(mask), ws.data_ptr(), ctr.data_ptr(), stream, _cap())
        else:
            ws, ctr = _workspace(*cu.bn_act_workspace(m, c), x.device)
            cu.bn_act_fwd_stats(x.data_ptr(), code, m, c, float(eps), float(momentum), _ptr(running_mean),
                                _ptr(running_var), mean.data_ptr(), invstd.data_ptr(), ws.data_ptr(), ctr.data_ptr(),
                                stream)
            cu.bn_act_fwd_apply(x.data_ptr(), _ptr(residual), code, m, c, mean.data_ptr(), invstd.data_ptr(),
                                weight.data_ptr(), bias.data_ptr(), bool(relu), y.data_ptr(), _ptr(mask), stream)
        ctx.save_for_backward(x, weight, mean, invstd, mask)
        ctx.has_residual = residual is not None
        ctx.single_launch_fwd = plan is not None
        if pair:
            ctx.set_materialize_grads(False)
            return y, y.view_as(y)
        return y

    @staticmethod
    def backward(ctx, dy, dy2=None):
        x, weight, mean, invstd, mask = ctx.saved_tensors
        cu = _native.cuda()
        n, c, h, w = x.shape
        m = n * h * w
        code = _CODES[x.dtype]
        if dy is None:
            dy, dy2 = dy2, None
        stream = torch.cuda.current_stream(x.device).cuda_stream
        f32 = dict(dtype=torch.float32, device=x.device)
        dweight, dbias = torch.empty(c, **f32), torch.empty(c, **f32)
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if ctx.has_residual else None
        plan = cu.bn_act_plan(1, code, m, c, _cap(), residual=ctx.has_residual)
        if dy2 is not None and not (plan is not None and ctx.has_residual and _sum_in_kernel(dy, dy2, x)):
            dy, dy2 = dy + dy2, None
        dy = _aligned(dy.to(x.dtype).contiguous(memory_format=torch.channels_last))
        if plan is not None:
            ws, ctr = _workspace(plan["ws_floats"], plan["counters"], x.device)
            cu.bn_act_bwd(dy.data_ptr(), x.data_ptr(), _ptr(mask), code, m, c, mean.data_ptr(), invstd.data_ptr(),
                          weight.data_ptr(), dweight.data_ptr(), dbias.data_ptr(), dx.data_ptr(), _ptr(dres),
                          ws.data_ptr(), ctr.data_ptr(), stream, _cap(), _ptr(dy2))
        else:
            ws, ctr = _workspace(*cu.bn_act_workspace(m, c), x.device)
            cu.bn_act_bwd_reduce(dy.data_ptr(), x.data_ptr(), _ptr(mask), code, m, c, mean.data_ptr(),
                                 invstd.data_ptr(), dweight.data_ptr(), dbias.data_ptr(), ws.data_ptr(), ctr.data_ptr(),
                                 stream)
            cu.bn_act_bwd_apply(dy.data_ptr(), x.data_ptr(), _ptr(mask), code, m, c, mean.data_ptr(),
                                invstd.data_ptr(), weight.data_ptr(), dweight.data_ptr(), dbias.data_ptr(),
                                dx.data_ptr(), _ptr(dres), stream)
        return dx, dres, dweight, dbias, None, None, None, None, None, None


def _stem_pool(pool) -> bool:
    """Whether ``pool`` is the max pool the pooled kernels implement: kernel 3, stride 2, padding 1, dilation 1, no
    ceil mode, no indices returned (ResNet's stem)."""
    two = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)  # noqa: E731
    return (isinstance(pool, nn.MaxPool2d) and two(pool.kernel_size) == (3, 3) and two(pool.stride) == (2, 2)
            and two(pool.padding) == (1, 1) and two(pool.dilation) == (1, 1) and not pool.ceil_mode
            and not pool.return_indices)


def _pool_planned(x) -> bool:
    """Whether the pooled forward and backward can both run at x's shape on its device."""
    cu = _native.cuda()
    n, c, h, w = x.shape
    code, m = _CODES[x.dtype], n * h * w
    return all(cu.bn_act_plan(d, code, m, c, _cap(), relu=True, pool_h=h, pool_w=w) is not None for d in (0, 1))


def _pooled_grad(g, x):
    """A pooled gradient as the kernel reads it: x's dtype, channels_last, 16-byte aligned."""
    return _aligned(g.to(x.dtype).contiguous(memory_format=torch.channels_last))


class _BatchNormActPoolFn(torch.autograd.Function):
    """Batch norm, ReLU and the stem's max pool (``_stem_pool``) as one single-launch kernel per direction.

    Forward writes the pooled output and a 4-bit window code per channel instead of y and its ReLU mask.  With
    ``pair`` the output is ``(p, p.view_as(p))`` and backward receives the two pooled gradients separately (None for
    an alias nobody used); the kernel sums them as torch's add would while it forms the max-pool and ReLU backward,
    so the gradient at y is never stored.  The caller checks both plans (``_pool_planned``) first."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, momentum, eps, pair):
        cu = _native.cuda()
        x = _aligned(x)
        n, c, h, w = x.shape
        code = _CODES[x.dtype]
        stream = torch.cuda.current_stream(x.device).cuda_stream
        f32 = dict(dtype=torch.float32, device=x.device)
        mean, invstd = torch.empty(c, **f32), torch.empty(c, **f32)
        oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        p = torch.empty((n, c, oh, ow), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        codes = torch.empty((n * oh * ow, c // _UNIT), dtype=torch.int32, device=x.device)
        plan = cu.bn_act_plan(0, code, n * h * w, c, _cap(), relu=True, pool_h=h, pool_w=w)
        ws, ctr = _workspace(plan["ws_floats"], plan["counters"], x.device)
        cu.bn_act_fwd_pool(x.data_ptr(), code, n, h, w, c, float(eps), float(momentum), _ptr(running_mean),
                           _ptr(running_var), mean.data_ptr(), invstd.data_ptr(), weight.data_ptr(), bias.data_ptr(),
                           p.data_ptr(), codes.data_ptr(), ws.data_ptr(), ctr.data_ptr(), stream, _cap())
        ctx.save_for_backward(x, weight, mean, invstd, codes)
        if pair:
            ctx.set_materialize_grads(False)
            return p, p.view_as(p)
        return p

    @staticmethod
    def backward(ctx, g1, g2=None):
        x, weight, mean, invstd, codes = ctx.saved_tensors
        cu = _native.cuda()
        n, c, h, w = x.shape
        code = _CODES[x.dtype]
        if g1 is None:
            g1, g2 = g2, None
        g1 = _pooled_grad(g1, x)
        g2 = None if g2 is None else _pooled_grad(g2, x)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        f32 = dict(dtype=torch.float32, device=x.device)
        dweight, dbias = torch.empty(c, **f32), torch.empty(c, **f32)
        dx = torch.empty_like(x)
        plan = cu.bn_act_plan(1, code, n * h * w, c, _cap(), relu=True, pool_h=h, pool_w=w)
        if plan is None:
            raise RuntimeError("bn_act_bwd_pool cannot run at %s on this device" % (tuple(x.shape),))
        ws, ctr = _workspace(plan["ws_floats"], plan["counters"], x.device)
        cu.bn_act_bwd_pool(g1.data_ptr(), _ptr(g2), codes.data_ptr(), x.data_ptr(), code, n, h, w, c,
                           mean.data_ptr(), invstd.data_ptr(), weight.data_ptr(), dweight.data_ptr(),
                           dbias.data_ptr(), dx.data_ptr(), ws.data_ptr(), ctr.data_ptr(), stream, _cap())
        return dx, dweight, dbias, None, None, None, None, None


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

    def _fused(self, x, residual, running_mean, running_var, factor, pair=False):
        return _BatchNormActFn.apply(x, residual, self.weight, self.bias, running_mean, running_var, factor, self.eps,
                                     self.act == "relu", pair)

    def _poolable(self, x, pool):
        """Whether ``pool(relu(batch_norm(x)))`` can take the pooled single-launch kernels (``_fusable`` checked)."""
        return self.act == "relu" and _stem_pool(pool) and _pool_planned(x)

    def forward(self, x, residual=None, pair=False, pool=None):
        """``act(batch_norm(x) [+ residual])``, then ``pool`` of it when one is given; with ``pair``, ``(out, alias
        of out)`` for two consumers of the output (see the module docstring).  Neither tensor of the pair may be
        modified in place."""
        if pool is not None:
            return self._forward_pooled(x, residual, pair, pool)
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
            return self._fused(x, residual, running_mean, running_var, factor, pair)
        y = F.batch_norm(x, running_mean, running_var, self.weight, self.bias, batch_stats, factor, self.eps)
        if residual is not None:
            y = y + residual
        if self.act == "relu":
            y = F.relu(y, inplace=True)
        return (y, y) if pair else y

    def _forward_pooled(self, x, residual, pair, pool):
        """``pool`` of the output: the pooled kernels for the stem's ReLU and max pool on a fusable input without a
        residual, ``pool`` of the unpooled path otherwise."""
        self._check_input_dim(x)
        batch_stats = self.training or (self.running_mean is None and self.running_var is None)
        if residual is None and self._fusable(x, None, batch_stats) and self._poolable(x, pool):
            factor = 0.0 if self.momentum is None else self.momentum
            if self.training and self.track_running_stats and self.num_batches_tracked is not None:
                self.num_batches_tracked.add_(1)
                factor = 1.0 / float(self.num_batches_tracked) if self.momentum is None else self.momentum
            track = not self.training or self.track_running_stats
            return _BatchNormActPoolFn.apply(x, self.weight, self.bias, self.running_mean if track else None,
                                             self.running_var if track else None, factor, self.eps, pair)
        p = pool(self.forward(x, residual))
        return (p, p) if pair else p


# ---------------------------------------------------------------------------------------------------------------
# Synchronised batch norm: statistics and gradient sums over the union of all ranks' batches
# (torch.nn.SyncBatchNorm semantics), exchanged through a peer-mapped window by two small kernels.

class SyncBatchNormContext:
    """Cross-rank state shared by every synchronised batch norm of a model on one rank.

    It owns (or borrows, for a :class:`~byteps_b200.comm.symm.VirtualCluster` rank) a peer-mapped window of
    ``[parity][source rank][count vectors + 2 * cmax]`` floats and the barrier generations of its own signal pad,
    separate from the exchange's arena, so the sync kernels never interfere with the exchange kernels running on
    the communication stream.  The sync kernels of every layer meet the peers in the same order on every rank, so
    all calls on one rank must come from one CUDA stream, in program order; a call from another stream raises.
    """

    channel = 0   # barrier channel of the context's own signal pad

    def __init__(self, view, rank: int, world: int, cmax: int, owner=None, stream: Optional[int] = None):
        self.view, self.rank, self.world, self.cmax = view, rank, world, cmax
        self._owner = owner      # keeps the peer-mapped memory alive
        self._stream = stream
        # Every kernel variant a rank may launch is loaded now: CUDA loading a module lazily while a peer's sync
        # kernel spins on this rank can deadlock.
        _native.cuda().bn_act_load_kernels()

    @staticmethod
    def window_bytes(world: int, cmax: int) -> int:
        return 4 * int(_native.cuda().bn_sync_window_floats(world, cmax))

    @classmethod
    def create(cls, group, device, cmax: int, mode: str = "auto") -> "SyncBatchNormContext":
        """Collective: a dedicated symmetric-memory context for ``group`` (every rank must call it)."""
        from ..comm.symm import SymmContext

        cmax = max(_UNIT, -(-int(cmax) // _UNIT) * _UNIT)
        symm = SymmContext(group, device, cls.window_bytes(group.world, cmax), mode, "0")
        return cls(symm.view, symm.rank, symm.world, cmax, owner=symm)

    @classmethod
    def from_virtual(cls, cluster, rank: int, cmax: int) -> "SyncBatchNormContext":
        """Rank ``rank`` of a VirtualCluster (window at offset 0 of its arena), bound to that rank's stream."""
        cmax = max(_UNIT, -(-int(cmax) // _UNIT) * _UNIT)
        if cls.window_bytes(cluster.world, cmax) > cluster.data_bytes:
            raise ValueError("VirtualCluster arena of %d bytes is smaller than the %d-byte window" % (
                cluster.data_bytes, cls.window_bytes(cluster.world, cmax)))
        return cls(cluster.views[rank], rank, cluster.world, cmax, owner=cluster,
                   stream=cluster.streams[rank].cuda_stream)

    def stream_for(self, device) -> int:
        s = torch.cuda.current_stream(device).cuda_stream
        if self._stream is None:
            self._stream = s
        elif s != self._stream:
            raise RuntimeError("synchronised batch norm: rank %d was called on stream 0x%x, but its earlier calls used "
                               "0x%x; every call on a rank must come from one stream" % (self.rank, s, self._stream))
        return s

    def __deepcopy__(self, memo):
        return self   # peer-mapped memory is not copied: a deep-copied model keeps its ranks' window


class _SyncBatchNormActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, bias, running_mean, running_var, momentum, eps, relu, sync):
        cu = _native.cuda()
        x, residual = _aligned(x), _aligned(residual)
        n, c, h, w = x.shape
        m = n * h * w
        code = _CODES[x.dtype]
        stream = sync.stream_for(x.device)
        f32 = dict(dtype=torch.float32, device=x.device)
        local = torch.empty(2, c, **f32)               # this rank's mean, M2
        mean, invstd = torch.empty(c, **f32), torch.empty(c, **f32)
        total = torch.empty(1, **f32)                  # row count of all ranks
        nws, nctr = cu.bn_act_workspace(m, c)
        ws = torch.empty(nws, **f32)
        ctr = torch.zeros(nctr, dtype=torch.int32, device=x.device)
        cu.bn_act_fwd_stats_local(x.data_ptr(), code, m, c, local[0].data_ptr(), local[1].data_ptr(), ws.data_ptr(),
                                  ctr.data_ptr(), stream)
        cu.bn_sync_stats(sync.view, sync.channel, 0, sync.cmax, c, local[0].data_ptr(), local[1].data_ptr(), float(m),
                         float(eps), float(momentum), _ptr(running_mean), _ptr(running_var), mean.data_ptr(),
                         invstd.data_ptr(), total.data_ptr(), stream)
        y = torch.empty_like(x)
        mask = torch.empty((m, c // _UNIT), dtype=torch.uint8, device=x.device) if relu else None
        cu.bn_act_fwd_apply(x.data_ptr(), _ptr(residual), code, m, c, mean.data_ptr(), invstd.data_ptr(),
                            weight.data_ptr(), bias.data_ptr(), bool(relu), y.data_ptr(), _ptr(mask), stream)
        ctx.save_for_backward(x, weight, mean, invstd, mask, total)
        ctx.has_residual = residual is not None
        ctx.sync = sync
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, invstd, mask, total = ctx.saved_tensors
        sync = ctx.sync
        cu = _native.cuda()
        n, c, h, w = x.shape
        m = n * h * w
        code = _CODES[x.dtype]
        dy = _aligned(dy.to(x.dtype).contiguous(memory_format=torch.channels_last))
        stream = sync.stream_for(x.device)
        f32 = dict(dtype=torch.float32, device=x.device)
        dweight, dbias = torch.empty(c, **f32), torch.empty(c, **f32)
        nws, nctr = cu.bn_act_workspace(m, c)
        ws = torch.empty(nws, **f32)
        ctr = torch.zeros(nctr, dtype=torch.int32, device=x.device)
        cu.bn_act_bwd_reduce(dy.data_ptr(), x.data_ptr(), _ptr(mask), code, m, c, mean.data_ptr(), invstd.data_ptr(),
                             dweight.data_ptr(), dbias.data_ptr(), ws.data_ptr(), ctr.data_ptr(), stream)
        sums = torch.empty(2, c, **f32)                # sum over ranks of dbias, dweight
        cu.bn_sync_grad(sync.view, sync.channel, 0, sync.cmax, c, dbias.data_ptr(), dweight.data_ptr(),
                        sums[0].data_ptr(), sums[1].data_ptr(), stream)
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if ctx.has_residual else None
        cu.bn_act_bwd_apply(dy.data_ptr(), x.data_ptr(), _ptr(mask), code, m, c, mean.data_ptr(), invstd.data_ptr(),
                            weight.data_ptr(), sums[1].data_ptr(), sums[0].data_ptr(), dx.data_ptr(), _ptr(dres),
                            stream, total.data_ptr())
        # the local sums, as torch.nn.SyncBatchNorm: the gradient exchange averages them over the ranks
        return dx, dres, dweight, dbias, None, None, None, None, None, None


class SyncBatchNormAct2d(BatchNormAct2d):
    """:class:`BatchNormAct2d` whose training-mode statistics are those of all ranks' batches together.

    Forward normalises with the mean and biased variance of the union of the ranks' batches (ranks may hold
    different row counts); the running statistics take the global unbiased variance and are bit-identical on every
    rank.  Backward forms dx from the all-reduced sums and returns the rank's local dweight / dbias.  Training at
    world > 1 needs a fusable input (CUDA, channels_last, C a multiple of 8, fp32/bf16/fp16 activations, fp32
    affine parameters) and raises ``ValueError`` otherwise; eval mode and world 1 are :class:`BatchNormAct2d`.
    """

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True, act=None,
                 sync: Optional[SyncBatchNormContext] = None, device=None, dtype=None):
        super().__init__(num_features, eps, momentum, affine, track_running_stats, act, device, dtype)
        self.sync = sync

    def _synced(self):
        return self.training and self.sync is not None and self.sync.world > 1

    def _unfusable(self, x, residual) -> Optional[str]:
        """Why a training input cannot take the synchronised kernels, or None."""
        if not x.is_cuda:
            return "the input is not a CUDA tensor"
        if x.dtype not in _CODES:
            return "the input dtype %s is not float32, bfloat16 or float16" % x.dtype
        if not self.affine or self.weight.dtype != torch.float32:
            return "the affine parameters must exist and be float32"
        if x.size(1) % _UNIT != 0:
            return "C = %d is not a multiple of %d" % (x.size(1), _UNIT)
        if x.size(1) > self.sync.cmax:
            return "C = %d exceeds the context's %d channels" % (x.size(1), self.sync.cmax)
        if x.numel() == 0:
            return "the input is empty"
        if not _nhwc(x):
            return "the input is not channels_last (NHWC) contiguous"
        if residual is not None and not (residual.shape == x.shape and residual.dtype == x.dtype and _nhwc(residual)):
            return "the residual does not match the input's shape, dtype and channels_last layout"
        return None

    def _fusable(self, x, residual, batch_stats):
        return True if self._synced() else super()._fusable(x, residual, batch_stats)

    def _poolable(self, x, pool):
        return False   # no pooled synchronised kernels: pool of the synchronised (or, at world 1, plain) path

    def _fused(self, x, residual, running_mean, running_var, factor, pair=False):
        if not self._synced():
            return super()._fused(x, residual, running_mean, running_var, factor, pair)
        y = _SyncBatchNormActFn.apply(x, residual, self.weight, self.bias, running_mean, running_var, factor,
                                      self.eps, self.act == "relu", self.sync)
        return (y, y) if pair else y   # autograd sums the two gradients

    def forward(self, x, residual=None, pair=False, pool=None):
        if self._synced():
            self._check_input_dim(x)
            why = self._unfusable(x, residual)
            if why is not None:
                raise ValueError("SyncBatchNormAct2d: synchronised training needs a fusable input, but %s" % why)
        return super().forward(x, residual, pair, pool)


def convert_sync_batchnorm(module: nn.Module, sync: Optional[SyncBatchNormContext]) -> nn.Module:
    """Replace every ``nn.BatchNorm2d`` in ``module`` (``BatchNormAct2d`` included, keeping its ``act``) by a
    :class:`SyncBatchNormAct2d` on ``sync`` that holds the same Parameter and buffer objects, so optimizers built
    over the original parameters stay valid and state_dict keys and parameter order are unchanged.  Children are
    replaced in place; the converted module is returned."""
    if isinstance(module, nn.BatchNorm2d):
        new = SyncBatchNormAct2d(module.num_features, module.eps, module.momentum, module.affine,
                                 module.track_running_stats, act=getattr(module, "act", None), sync=sync,
                                 device="meta")
        new.weight, new.bias = module.weight, module.bias
        new.running_mean, new.running_var = module.running_mean, module.running_var
        new.num_batches_tracked = module.num_batches_tracked
        new.train(module.training)
        if hasattr(module, "qconfig"):
            new.qconfig = module.qconfig
        return new
    for name, child in module.named_children():
        module.add_module(name, convert_sync_batchnorm(child, sync))
    return module
