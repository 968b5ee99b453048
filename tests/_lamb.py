"""Float64 reference and rounding bounds for fused LAMB (shared by test_gpu_lamb.py, which runs the kernels on virtual
ranks, and test_gpu_lamb_api.py, which runs DistributedOptimizer(Lamb(...), fused_update=True))."""
import torch

from _fused_opt import _U

# A few ragged parameters in two groups: weights with decay and the trust ratio, the rest with neither (the BERT
# split).  Their gradients come from loss = sum_i (p_i * G_i).sum(), so p_i.grad = G_i whatever the weights are.
SHAPES = [(37, 11), (11,), (200,), (5, 3), (1,), (64, 9)]
KW = dict(lr=0.01, betas=(0.9, 0.99), eps=1e-6)


def _advance(e, g, w_prev, st, lr, wd, b1, b2, eps, t, adapt, w_norm, u_ref, nparams_slices):
    """Advance the elementwise bound e["w"] on |fp32 master - float64 reference| (and the moment bounds) by step t.

    Each fp32 operation rounds to within u*|result|; "*mag" carries the value with every term taken positive, so no
    cancellation hides a rounding.  The summed gradient is exact (see _fused_grad); scale*grad_scale and the product
    with it round (4u).  The moments follow EpiAdam's analysis.  u = m^/(sqrt(v^)+eps) + wd*w adds its error and that
    of the master through the decay term.  The trust ratio phi = ||w|| / ||u|| is a ratio of square roots of sums of
    non-negative terms: by the triangle inequality | ||w~|| - ||w|| | <= ||e_w|| and likewise for u, so its relative
    error is at most ||e_w||/||w|| + ||e_u||/||u|| to first order, plus the float64 sums and the final rounding to
    fp32 (2u); lr*phi rounds once more."""
    gmag = g.abs()
    eg = 4 * _U * gmag
    c1, c2 = 1 - b1 ** t, 1 - b2 ** t
    e["mmag"] = b1 * e["mmag"] + (1 - b1) * gmag
    e["m"] = b1 * e["m"] + (1 - b1) * eg + 4 * _U * e["mmag"] + _U * b1 * gmag
    e["vmag"] = b2 * e["vmag"] + (1 - b2) * gmag * gmag
    e["v"] = b2 * e["v"] + (1 - b2) * (2 * gmag * eg + eg * eg) + 5 * _U * e["vmag"] + _U * b2 * gmag * gmag
    sv = (st["exp_avg_sq"] / c2).sqrt()
    den = sv + eps
    ua = (st["exp_avg"] / c1).abs() / den
    esqrt = torch.minimum(e["v"] / c2 / (2 * sv).clamp_min(1e-300), (e["v"] / c2).sqrt()) + 4 * _U * sv
    eu = e["m"] / c1 / den + ua * ((esqrt + _U * den) / den + 8 * _U) + wd * e["w"] + 2 * _U * (ua + wd * w_prev.abs())
    step_err = torch.empty_like(eu)
    for (lo, hi), wn in zip(nparams_slices, w_norm):
        un = u_ref[lo:hi].norm()
        if adapt and wn > 0 and un > 0:
            phi = (wn / un).item()
            rel = (e["w"][lo:hi].norm() / wn + eu[lo:hi].norm() / un).item() + 4 * _U
            # the ratio of the perturbed norms: (1 + ew) / (1 - eu) - 1 <= ew + eu + 2 eu^2 (eu <= 1/2)
            rel += 2 * (eu[lo:hi].norm() / un).item() ** 2
        else:
            phi, rel = 1.0, 0.0
        # lr*phi*u with phi and lr*phi perturbed, and the rounding of the fma w - lr*phi*u
        step_err[lo:hi] = (lr * phi * (eu[lo:hi] + u_ref[lo:hi].abs() * (rel + _U))
                           + _U * (w_prev[lo:hi].abs() + lr * phi * u_ref[lo:hi].abs()))
    e["w"] = e["w"] + step_err


def make_params(dt, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g, device="cuda").to(dt)) for s in SHAPES]


def groups(ps):
    return [dict(params=[ps[0], ps[2], ps[3], ps[5]], weight_decay=0.01),
            dict(params=[ps[1], ps[4]], weight_decay=0.0, adapt=False)]


def fused_lamb(ps, **kw):
    import byteps_b200.torch as bps

    return bps.DistributedOptimizer(bps.Lamb(groups(ps), **KW), named_parameters=[("p%d" % i, p) for i, p in
                                                                                  enumerate(ps)],
                                    fused_update=True, **kw)


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
    """The plain Lamb on float64 copies of the parameters, with the bounds of _advance per parameter."""

    def __init__(self, ps):
        from byteps_b200.torch import Lamb

        self.ps = [torch.nn.Parameter(p.detach().double()) for p in ps]
        self.opt = Lamb(groups(self.ps), **KW)
        z = lambda p: torch.zeros(p.numel(), dtype=torch.float64, device=p.device)  # noqa: E731
        self.e = [{k: z(p) for k in ("w", "m", "mmag", "v", "vmag")} for p in self.ps]
        self.t = 0

    def set_lr(self, lr):
        for g in self.opt.param_groups:
            g["lr"] = lr

    def step(self, gs):
        """One step on float64 gradients gs (one per parameter)."""
        self.t += 1
        for p, g in zip(self.ps, gs):
            p.grad = g.double().reshape(p.shape)
        w_prev = [p.detach().flatten().clone() for p in self.ps]
        self.opt.step()
        for grp in self.opt.param_groups:
            b1, b2 = grp["betas"]
            c1, c2 = 1 - b1 ** self.t, 1 - b2 ** self.t
            for p in grp["params"]:
                i = next(j for j, q in enumerate(self.ps) if q is p)
                st = {k: self.opt.state[p][k].flatten() for k in ("exp_avg", "exp_avg_sq")}
                u = (st["exp_avg"] / c1) / ((st["exp_avg_sq"] / c2).sqrt() + grp["eps"]) + grp["weight_decay"] * w_prev[i]
                _advance(self.e[i], p.grad.flatten(), w_prev[i], st, grp["lr"], grp["weight_decay"], b1, b2,
                         grp["eps"], self.t, grp["adapt"], [w_prev[i].norm()], u, [(0, p.numel())])

    def check(self, opt, ps, what=""):
        """The fused optimizer's fp32 state of parameters ps (masters, moments) within twice the bounds, and every
        parameter equal to its rounded master."""
        full = opt.grad_sync.export_state()
        for i, (p, r) in enumerate(zip(ps, self.ps)):
            ent = full[p]
            assert torch.equal(p.detach().cpu(), ent["master"].to(p.dtype)), (what, i, "parameter != round(master)")
            for key, want, bound in (("master", r.detach(), self.e[i]["w"]),
                                     ("state0", self.opt.state[r]["exp_avg"], self.e[i]["m"]),
                                     ("state1", self.opt.state[r]["exp_avg_sq"], self.e[i]["v"])):
                err = (ent[key].double().flatten().cuda() - want.flatten()).abs()
                bad = err > 2 * bound
                assert not bad.any(), (what, i, key, int(bad.sum()), err.max().item(),
                                       (err / bound.clamp_min(1e-300)).max().item())
