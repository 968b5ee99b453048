"""DistributedDataParallel: a module wrapper that averages gradients during
backward, so a plain ``torch.optim`` optimizer can be used unchanged.

Parity: /root/reference/byteps/torch/parallel/distributed.py:122-287 (same
constructor arguments, ``no_sync()``, ``synchronize()``, state broadcast at
construction, buffer broadcast before every forward).  On CUDA the gradients
are exchanged by the zero-copy bucketed kernels
(:class:`byteps_b200.parallel.bucket.BucketedGradSync`); elsewhere by
per-parameter ``push_pull_group_sync_inplace`` like the reference, whose grad
counter tells the wrapper when the last gradient of the iteration was issued.
Clipping inside the exchange (``DistributedOptimizer``'s ``max_grad_norm``) is not offered by this wrapper.
"""
from contextlib import contextmanager

import torch
from torch.nn.modules import Module

from ...common import engine as _engine
from .. import broadcast_parameters
from ..compression import Compression
from ..ops import (byteps_torch_set_num_grads, declare, push_pull_group_sync_inplace, size, synchronize)


class DistributedDataParallel(Module):
    def __init__(self, module, device_ids=None, broadcast_buffers=True, compression=Compression.none,
                 bucket_bytes=None):
        super(DistributedDataParallel, self).__init__()
        if device_ids is not None:
            assert len(device_ids) == 1, ("DistributedDataParallel device_ids contain exactly one entry, "
                                          "but got {}.").format(device_ids)
        self.device_ids = device_ids
        self.module = module
        self.broadcast_buffers = broadcast_buffers
        self.require_forward_param_sync = broadcast_buffers
        self._handles = {}
        self._requires_update = set()
        self._hook_handles = []
        self._compression = compression
        self._enable_async = False
        self._require_backward_grad_sync = True
        named_parameters = list(self.module.named_parameters())
        self._parameter_names = {p: n for n, p in named_parameters}
        self._num_grads = sum(p.requires_grad for _, p in named_parameters)
        for name in sorted(self._parameter_names.values()):
            declare("Gradient." + name)
        for name in sorted(self._parameter_names.values()):
            declare("Parameter." + name)
        self._sync = None
        eng = _engine()
        params = [p for _, p in named_parameters if p.requires_grad]
        if size() > 1 and params:
            if eng.backend == "symm" and all(p.is_cuda for p in params):
                from ...parallel.bucket import BucketedGradSync
                from .. import _wire_of

                self._sync = BucketedGradSync(eng, [{"params": params}], wire_dtype=_wire_of(compression),
                                              bucket_bytes=bucket_bytes)
                self._sync.auto_finish = self._on_all_issued
            else:
                self._register_hooks()
                byteps_torch_set_num_grads(self._num_grads)
        if len(list(self.module.state_dict().values())) > 0:
            broadcast_parameters(self.module.state_dict(), root_rank=0)

    @contextmanager
    def no_sync(self):
        """Disable gradient synchronisation inside the context; gradients
        accumulate locally and are synchronised by the first backward after it."""
        if self._enable_async:
            raise AssertionError("no_sync cannot be used in async training")
        old = self._require_backward_grad_sync
        self._require_backward_grad_sync = False
        if self._sync is not None:
            self._sync.enabled = False
        try:
            yield
        finally:
            self._require_backward_grad_sync = old
            if self._sync is not None:
                self._sync.enabled = old

    def forward(self, *inputs, **kwargs):
        if self.require_forward_param_sync:
            self._sync_params()
        return self.module(*inputs, **kwargs)

    def _sync_params(self):
        with torch.no_grad():
            bufs = [(n, b) for n, b in self.module.named_buffers() if b.is_floating_point()]
            if self.broadcast_buffers and bufs and size() > 1:
                broadcast_parameters(bufs, root_rank=0, prefix="Buffer.")

    def _register_hooks(self):
        for _, p in self.module.named_parameters():
            if p.requires_grad:
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
                self._requires_update.add(p)
                self._hook_handles.append(p.register_post_accumulate_grad_hook(self._make_hook(p)))

    def _push_pull_grad_group_sync(self, p):
        name = self._parameter_names.get(p)
        if p.grad is None:      # unused this iteration and cleared by zero_grad(set_to_none=True): contribute zeros
            p.grad = torch.zeros_like(p)
        tensor_compressed, ctx = self._compression.compress(p.grad)
        handle, grad_count = push_pull_group_sync_inplace(tensor_compressed, average=True, name="Gradient." + name)
        return handle, (ctx, tensor_compressed), grad_count

    def _make_hook(self, p):
        def hook(*ignore):
            if self._require_backward_grad_sync:
                handle, ctx, grad_count = self._push_pull_grad_group_sync(p)
                self._handles[p] = (handle, ctx)
                if grad_count == self._num_grads:   # every gradient of this iteration is in flight
                    self.synchronize()
        return hook

    def _on_all_issued(self):
        self._sync.synchronize()

    def synchronize(self):
        if self._sync is not None:
            self._sync.synchronize()
            return
        if not self._require_backward_grad_sync:
            return
        missing_p = self._requires_update - set(self._handles.keys())
        for p in sorted(missing_p, key=lambda q: self._parameter_names.get(q)):
            handle, ctx, _ = self._push_pull_grad_group_sync(p)
            self._handles[p] = (handle, ctx)
        for p, (handle, ctx) in self._handles.items():
            output = synchronize(handle)
            cctx, _ = ctx
            tmp = self._compression.decompress(output, cctx)
            if tmp.data_ptr() != p.grad.data_ptr():
                p.grad.copy_(tmp)
        self._handles.clear()
