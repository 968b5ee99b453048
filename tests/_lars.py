"""Float64 reference and rounding bounds for LARS: the rule transcribed element by element (test_lars.py checks the
plain Lars against it), and the bounds of the fused kernels against the float64 Lars (shared by test_gpu_lars.py,
which runs the kernels on virtual ranks, and test_gpu_lars_api.py, which runs DistributedOptimizer(Lars(...),
fused_update=True))."""
import math

import torch

from _fused_opt import _U

# A few ragged parameters in two groups: weights with decay and the trust ratio, the rest with neither (the ResNet
# split of batch-norm parameters and biases).  Their gradients come from loss = sum_i (p_i * G_i).sum(), so
# p_i.grad = G_i whatever the weights are.
SHAPES = [(37, 11), (11,), (200,), (5, 3), (1,), (64, 9)]
KW = dict(lr=0.1, momentum=0.9, trust_coefficient=0.02, eps=1e-6)


def transcribed(ws, grads, groups, lrs):
    """The rule in float64, written out from its definition.  ws[g][p]: flat weights of parameter p of group g;
    grads[t][g][p]: its gradient at step t; lrs: a factor on each group's lr per step.  Returns the final weights."""
    ws = [[list(map(float, w)) for w in g_ws] for g_ws in ws]
    vs = [[[0.0] * len(w) for w in g_ws] for g_ws in ws]
    for t, lr_scale in enumerate(lrs):
        for gi, grp in enumerate(groups):
            lr, mom, wd = grp["lr"] * lr_scale, grp["momentum"], grp["weight_decay"]
            eta, eps, adapt = grp["trust_coefficient"], grp["eps"], grp["adapt"]
            for pi, w in enumerate(ws[gi]):
                g, v = grads[t][gi][pi], vs[gi][pi]
                wn = math.sqrt(sum(x * x for x in w))
                gn = math.sqrt(sum(x * x for x in g))
                phi = eta * wn / (gn + wd * wn + eps) if adapt and wn > 0 and gn > 0 else 1.0
                for k in range(len(w)):
                    v[k] = mom * v[k] + lr * phi * (g[k] + wd * w[k])
                    w[k] -= v[k]
    return ws


def advance(e, g, w_prev, lr, mom, wd, eta, eps, adapt, slices):
    """Advance the elementwise bounds e["w"] on |fp32 master - float64 reference| and e["v"] on the momentum by one
    step; e["vmag"] carries |v| with every term taken positive, so no cancellation hides a rounding.

    The summed gradient is exact (see _fused_grad); scale * grad_scale and the product with it round (4u, as in
    _lamb._advance).  d = fma(wd, w, g) adds the master's error through the decay and rounds once.  phi =
    eta ||w|| / (||g|| + wd ||w|| + eps): by the triangle inequality the computed norms are off by at most ||e_w|| and
    ||e_g||, so to first order phi's relative error is ||e_w|| / ||w|| + (||e_g|| + wd ||e_w||) / D, plus a
    second-order term, the float64 sums and the rounding to fp32 (4u together); lr * phi rounds once more.
    v = fma(lr phi, d, fl(momentum v)) rounds twice and w - v once.  `slices` are the parameters' (first, end of real
    elements, end with padding) in the flat layout; the norms run over the real elements."""
    gmag, wmag = g.abs(), w_prev.abs()
    eg = 4 * _U * gmag
    dmag = gmag + wd * wmag
    ed = eg + wd * e["w"] + _U * dmag
    ev = torch.empty_like(e["v"])
    vnew = torch.empty_like(e["vmag"])
    for lo, hi, pad in slices:
        wn, gn = w_prev[lo:hi].norm().item(), g[lo:hi].norm().item()
        if adapt and wn > 0 and gn > 0:
            den = gn + wd * wn + eps
            phi = eta * wn / den
            rd = (eg[lo:hi].norm().item() + wd * e["w"][lo:hi].norm().item()) / den
            rel = e["w"][lo:hi].norm().item() / wn + rd + 2 * rd * rd + 4 * _U
        else:
            phi, rel = 1.0, 0.0
        s = slice(lo, pad)
        step = lr * phi * dmag[s]
        vnew[s] = mom * e["vmag"][s] + step
        ev[s] = (mom * e["v"][s] + _U * mom * e["vmag"][s] + lr * phi * (ed[s] + dmag[s] * (rel + _U))
                 + _U * vnew[s])
    e["vmag"] = vnew
    e["v"] = ev
    e["w"] = e["w"] + ev + _U * (wmag + vnew)


def make_params(dt, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g, device="cuda").to(dt)) for s in SHAPES]


def groups(ps):
    return [dict(params=[ps[0], ps[2], ps[3], ps[5]], weight_decay=0.01),
            dict(params=[ps[1], ps[4]], weight_decay=0.0, adapt=False)]


def fused_lars(ps, **kw):
    import byteps_b200.torch as bps

    return bps.DistributedOptimizer(bps.Lars(groups(ps), **KW),
                                    named_parameters=[("p%d" % i, p) for i, p in enumerate(ps)], fused_update=True,
                                    **kw)


def grads(step, dt, seed=0):
    """Multiples of 2^-10 below 8 in magnitude: sums of a few of them, and their products with powers of two, are
    exact in fp32, so the exchange hands the optimizer exactly the reference's gradient."""
    g = torch.Generator(device="cuda").manual_seed(1000 * seed + step)
    return [((torch.randn(s, generator=g, device="cuda") * 1024).round().clamp(-8191, 8191) / 1024).to(dt)
            for s in SHAPES]


def backward(ps, gs, opt=None):
    """p.grad += G for every parameter; through opt.scale_loss when opt is given (dynamic loss scaling)."""
    loss = sum((p * g).sum().float() for p, g in zip(ps, gs))
    (opt.scale_loss(loss) if opt is not None else loss).backward()


class Reference:
    """The plain Lars on float64 copies of the parameters, with the bounds of advance per parameter."""

    def __init__(self, ps):
        from byteps_b200.torch import Lars

        self.ps = [torch.nn.Parameter(p.detach().double()) for p in ps]
        self.opt = Lars(groups(self.ps), **KW)
        z = lambda p: torch.zeros(p.numel(), dtype=torch.float64, device=p.device)  # noqa: E731
        self.e = [{k: z(p) for k in ("w", "v", "vmag")} for p in self.ps]

    def set_lr(self, lr):
        for g in self.opt.param_groups:
            g["lr"] = lr

    def step(self, gs):
        """One step on float64 gradients gs (one per parameter)."""
        for p, g in zip(self.ps, gs):
            p.grad = g.double().reshape(p.shape)
        w_prev = [p.detach().flatten().clone() for p in self.ps]
        self.opt.step()
        for grp in self.opt.param_groups:
            for p in grp["params"]:
                i = next(j for j, q in enumerate(self.ps) if q is p)
                advance(self.e[i], p.grad.flatten(), w_prev[i], grp["lr"], grp["momentum"], grp["weight_decay"],
                        grp["trust_coefficient"], grp["eps"], grp["adapt"], [(0, p.numel(), p.numel())])

    def check(self, opt, ps, what=""):
        """The fused optimizer's fp32 state of parameters ps (masters, momentum) within twice the bounds, and every
        parameter equal to its rounded master."""
        full = opt.grad_sync.export_state()
        for i, (p, r) in enumerate(zip(ps, self.ps)):
            ent = full[p]
            assert torch.equal(p.detach().cpu(), ent["master"].to(p.dtype)), (what, i, "parameter != round(master)")
            for key, want, bound in (("master", r.detach(), self.e[i]["w"]),
                                     ("state0", self.opt.state[r]["momentum_buffer"], self.e[i]["v"])):
                err = (ent[key].double().flatten().cuda() - want.flatten()).abs()
                bad = err > 2 * bound
                assert not bad.any(), (what, i, key, int(bad.sum()), err.max().item(),
                                       (err / bound.clamp_min(1e-300)).max().item())
