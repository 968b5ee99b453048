"""LARS (You et al., 2017, "Large Batch Training of Convolutional Networks"), in the form of the MLPerf ResNet
reference.

Per parameter tensor, with ``g`` its gradient and ``w`` the weight before the update::

    phi = eta * ||w|| / (||g|| + weight_decay * ||w|| + eps)   if adapt and ||w|| > 0 and ||g|| > 0, else 1
    v  <- momentum * v + lr * phi * (g + weight_decay * w)
    w  <- w - v

The norms run over the whole tensor.  The learning rate sits inside the momentum buffer ``v`` (which starts at zero),
as in the MLPerf reference, so a warm-up or decay schedule scales the new contribution only.  ``adapt=False`` turns
the trust ratio off for a param group (ResNet recipes use it, with ``weight_decay=0``, for batch-norm parameters and
biases).  Because ``v`` includes lr, the state does not carry over to or from ``torch.optim.SGD``, whose buffer does
not; checkpoints move between this class and ``DistributedOptimizer(Lars(...), fused_update=True)``.

This class is the plain per-tensor implementation.  ``DistributedOptimizer(Lars(...), fused_update=True)`` runs the
same rule inside the fused exchange on fp32 master weights instead (``parallel/bucket.py``).
"""
from __future__ import annotations

import torch


class Lars(torch.optim.Optimizer):
    def __init__(self, params, lr=0.1, momentum=0.9, weight_decay=0.0, trust_coefficient=0.001, eps=0.0, adapt=True):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: {}".format(lr))
        if not 0.0 <= momentum:
            raise ValueError("Invalid momentum value: {}".format(momentum))
        if not 0.0 <= weight_decay:
            raise ValueError("Invalid weight_decay value: {}".format(weight_decay))
        if not 0.0 < trust_coefficient:
            raise ValueError("Invalid trust_coefficient value: {}".format(trust_coefficient))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {}".format(eps))
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay,
                                      trust_coefficient=trust_coefficient, eps=eps, adapt=adapt))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            lr, mom, wd = group["lr"], group["momentum"], group["weight_decay"]
            eta, eps = group["trust_coefficient"], group["eps"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                if g.is_sparse:
                    raise RuntimeError("Lars does not support sparse gradients")
                state = self.state[p]
                if not state:
                    state["momentum_buffer"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                buf = state["momentum_buffer"]
                d = g.add(p, alpha=wd) if wd != 0 else g.clone()
                if group["adapt"]:
                    w_norm, g_norm = p.norm(), g.norm()
                    phi = torch.where((w_norm > 0) & (g_norm > 0), eta * w_norm / (g_norm + wd * w_norm + eps),
                                      torch.ones_like(w_norm))
                    buf.mul_(mom).add_(d * (lr * phi))
                else:
                    buf.mul_(mom).add_(d, alpha=lr)
                p.sub_(buf)
        return loss
