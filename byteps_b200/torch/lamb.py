"""LAMB (You et al., 2019, "Large Batch Optimization for Deep Learning: Training BERT in 76 minutes").

Per parameter tensor, at step t of its param group::

    m <- beta1 * m + (1 - beta1) * g
    v <- beta2 * v + (1 - beta2) * g^2
    u  = (m / (1 - beta1^t)) / (sqrt(v / (1 - beta2^t)) + eps) + weight_decay * w
    phi = ||w|| / ||u||   if adapt and ||w|| > 0 and ||u|| > 0, else 1
    w <- w - lr * phi * u

``w`` is the parameter before the update and the norms run over the whole tensor.  ``adapt=False`` turns the trust
ratio off for a param group (BERT recipes use it for biases and LayerNorm weights, with ``weight_decay=0``).

This class is the plain per-tensor implementation.  ``DistributedOptimizer(Lamb(...), fused_update=True)`` runs the
same rule inside the fused exchange on fp32 master weights instead (``parallel/bucket.py``).
"""
from __future__ import annotations

import torch


class Lamb(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, adapt=True):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: {}".format(lr))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {}".format(eps))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter at index 0: {}".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter at index 1: {}".format(betas[1]))
        if not 0.0 <= weight_decay:
            raise ValueError("Invalid weight_decay value: {}".format(weight_decay))
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, adapt=adapt))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            lr, eps, wd = group["lr"], group["eps"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                if g.is_sparse:
                    raise RuntimeError("Lamb does not support sparse gradients")
                state = self.state[p]
                if not state:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                t = int(state["step"].item())
                m, v = state["exp_avg"], state["exp_avg_sq"]
                m.mul_(beta1).add_(g, alpha=1 - beta1)
                v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
                u = (m / (1 - beta1 ** t)) / ((v / (1 - beta2 ** t)).sqrt() + eps)
                if wd != 0:
                    u.add_(p, alpha=wd)
                if group["adapt"]:
                    w_norm, u_norm = p.norm(), u.norm()
                    phi = torch.where((w_norm > 0) & (u_norm > 0), w_norm / u_norm, torch.ones_like(w_norm))
                    p.sub_(u * (lr * phi))
                else:
                    p.sub_(u, alpha=lr)
        return loss
