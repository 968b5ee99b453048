"""Float64 reference of "average, clip, step" for DistributedOptimizer(..., max_grad_norm=...) on the GPU
(test_gpu_clip_api.py): every fused kind in float64, with torch.nn.utils.clip_grad_norm_ on float64 gradients."""
import torch

# ragged parameters in two groups; the gradients come from loss = sum_i (p_i * G_i).sum(), so p_i.grad = G_i
SHAPES = [(37, 11), (11,), (200,), (5, 3), (1,), (64, 9)]
# the gradients' size per step: the clipping coefficient changes from step to step, and one step is not clipped,
# so Adam's and LAMB's moments mix gradients of different scales and a wrong coefficient shows
STEP_SCALE = [1.0, 8.0, 0.02, 3.0, 0.5, 5.0]
MAX_NORM = 4.0


def optimizer(kind, ps):
    """The wrapped optimizer of `kind` over ps in two groups (the second without weight decay, and for LAMB and LARS
    without the trust ratio)."""
    import byteps_b200.torch as bps

    g0, g1 = [ps[0], ps[2], ps[3], ps[5]], [ps[1], ps[4]]
    if kind == "sgd":
        return torch.optim.SGD([dict(params=g0, weight_decay=0.01), dict(params=g1)], lr=0.05, momentum=0.9)
    if kind == "adam":
        return torch.optim.Adam([dict(params=g0, weight_decay=0.01), dict(params=g1)], lr=0.01, eps=1e-6)
    if kind == "adamw":
        return torch.optim.AdamW([dict(params=g0, weight_decay=0.01), dict(params=g1, weight_decay=0.0)], lr=0.01)
    if kind == "lamb":
        return bps.Lamb([dict(params=g0, weight_decay=0.01), dict(params=g1, weight_decay=0.0, adapt=False)],
                        lr=0.01, eps=1e-6)
    if kind == "lars":
        return bps.Lars([dict(params=g0, weight_decay=0.01), dict(params=g1, weight_decay=0.0, adapt=False)],
                        lr=0.1, momentum=0.9, trust_coefficient=0.02, eps=1e-6)
    raise ValueError(kind)


KINDS = ("sgd", "adam", "adamw", "lamb", "lars")


def make_params(dt, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g, device="cuda").to(dt)) for s in SHAPES]


def grads(step, dt, seed=0):
    """Multiples of 2^-7 below 1 in magnitude (seven significant bits: exact in bf16 and fp16, and sums of a few
    are exact in fp32), times a power of two near STEP_SCALE[step]."""
    g = torch.Generator(device="cuda").manual_seed(1000 * seed + step)
    k = 2.0 ** round(torch.log2(torch.tensor(STEP_SCALE[step % len(STEP_SCALE)])).item())
    return [((torch.randn(s, generator=g, device="cuda") * 16).round().clamp(-127, 127) / 128 * k).to(dt)
            for s in SHAPES]


def backward(ps, gs, opt=None):
    loss = sum((p * g).sum().float() for p, g in zip(ps, gs))
    (opt.scale_loss(loss) if opt is not None else loss).backward()


def fused(kind, ps, **kw):
    import byteps_b200.torch as bps

    return bps.DistributedOptimizer(optimizer(kind, ps), named_parameters=[("p%d" % i, p) for i, p in enumerate(ps)],
                                    fused_update=True, **kw)


class Reference:
    """The wrapped optimizer on float64 copies of the parameters: step(gs) sets the averaged gradients, clips them with
    clip_grad_norm_ over every parameter of every group, and steps."""

    def __init__(self, kind, ps, max_norm=MAX_NORM):
        self.ps = [torch.nn.Parameter(p.detach().double()) for p in ps]
        self.opt = optimizer(kind, self.ps)
        self.max_norm = max_norm
        self.norms = []

    def step(self, gs):
        for p, g in zip(self.ps, gs):
            p.grad = g.double().reshape(p.shape).clone()
        ordered = [p for grp in self.opt.param_groups for p in grp["params"]]
        self.norms.append(float(torch.nn.utils.clip_grad_norm_(ordered, self.max_norm)))
        self.opt.step()

    def check(self, opt, ps, what=""):
        """Every fp32 master within 1e-5 relative (plus 1e-6 absolute) of the float64 reference, every parameter equal
        to its rounded master, and grad_norm within 1e-6 of the reference's last norm.  A coefficient that was not
        applied, or applied twice, moves the masters by about lr times the gradient."""
        full = opt.grad_sync.export_state()
        for i, (p, r) in enumerate(zip(ps, self.ps)):
            m = full[p]["master"]
            assert torch.equal(p.detach().cpu(), m.to(p.dtype)), (what, i, "parameter != round(master)")
            want = r.detach().cpu()
            err = (m.double() - want).abs()
            tol = 1e-5 * want.abs() + 1e-6
            assert bool((err <= tol).all()), (what, i, err.max().item(), (err / tol).max().item())
        n = opt.grad_norm.item()
        assert abs(n - self.norms[-1]) <= 1e-6 * self.norms[-1], (what, n, self.norms[-1])
