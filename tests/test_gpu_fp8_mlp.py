"""BERT's FP8 feed-forward block with the GELU inside the casts (ops/fp8.py::fp8_gelu_mlp, kernels/fp8.cu ACT_*).

GPU tests:

* the ``ACT_GELU`` cast of every finite bf16 / fp16 value, and the ``ACT_DGELU`` cast of every finite value against a
  set of gradients (zero, +-1, +-tiny, large, E5M2-saturating), equal bit for bit today's cast of torch's own
  ``F.gelu`` / ``gelu_backward`` output: rows, transposed copy, bias gradient, inverse scale and state;
* an inf or NaN in either input gives a NaN inverse scale and leaves the state alone;
* ``fp8_gelu_mlp`` equals ``fc2(F.gelu(fc1(x)))`` on copies of the same modules bit for bit over several calls
  (the seeding one included), in y, every gradient and all six scaling-state rows; run to run and under a CUDA graph;
* a graphed bert_tiny ``fp8_linear=True`` training run equals the same run with the composition patched in;
* the profiler sees two fewer launches per direction and no GELU kernel on the fused path.

CPU tests: inputs off the fast path are exactly the composition, the model's parameters and state_dict do not
change, the binding rejects bad activation arguments, and ptxas reports no spills for the new instantiations.
"""
import copy
import os
import re
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from byteps_b200.models import bert_tiny
from byteps_b200.ops import fp8
from byteps_b200.ops.fp8 import E4M3, E5M2, FP8_DTYPES, FP8_MAX, Fp8Linear, fp8_gelu_mlp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUSED = "_Fp8GeluMlpFnBackward"


def _dt_id(d):
    return str(d).replace("torch.", "")


def _finite_values(dtype):
    """every finite value of dtype, as a 1-D tensor on the GPU"""
    v = torch.arange(-2 ** 15, 2 ** 15, dtype=torch.int32).to(torch.int16).view(dtype)
    return v[torch.isfinite(v.float())].cuda()


def _grid(v):
    """v as [M, K] with M and K multiples of 16"""
    n = v.numel()
    k = [k for k in (272, 496, 256) if n % (16 * k) == 0][0]   # bf16: 255 * 256 finite values, fp16: 31 * 2048
    return v.view(-1, k)


def _state(scale):
    st = torch.zeros(fp8.STATE_WORDS, dtype=torch.int32, device="cuda")
    st.view(torch.float32)[fp8.HISTORY] = scale
    return st


def _u8(t):
    return t.view(torch.uint8)


def _same(a, b):
    """bitwise equality of two tensors (NaN-safe)"""
    if a is None or b is None:
        return a is None and b is None
    if a.dtype.is_floating_point:
        w = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[a.element_size()]
        a, b = a.view(w), b.view(w)
    return a.shape == b.shape and torch.equal(a, b)


def _ref_cast(x, s, fmt):
    fmax = FP8_MAX[fmt]
    return torch.clamp(x.float() * s, -fmax, fmax).to(FP8_DTYPES[fmt])


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=_dt_id)
def test_gelu_cast_exhaustive(dtype, fmt):
    z = _grid(_finite_values(dtype))
    h = F.gelu(z)
    for s in (1.0, FP8_MAX[fmt] / 3.0, 2.0 ** -12, 1e-30, 1e30):
        s = torch.tensor(s, dtype=torch.float32)
        st, st_ref = _state(s), _state(s)
        rows, cols, inv, db = fp8.cast(z, st, fmt, fp8.BOTH, act=fp8.ACT_GELU)
        ref = _ref_cast(h, s, fmt)
        assert db is None
        assert torch.equal(_u8(rows), _u8(ref)), s
        assert torch.equal(_u8(cols), _u8(ref.t().contiguous())), s
        r_rows, r_cols, r_inv, _ = fp8.cast(h, st_ref, fmt, fp8.BOTH)
        assert torch.equal(_u8(rows), _u8(r_rows)) and torch.equal(_u8(cols), _u8(r_cols))
        assert _same(inv, r_inv) and torch.equal(st, st_ref), s


def _grad_values(dtype):
    fi = torch.finfo(dtype)
    large = 1e30 if dtype == torch.bfloat16 else 3e4
    return [0.0, 1.0, -1.0, fi.tiny, -fi.tiny, fi.tiny * 2.0 ** -6, 1e-3, -0.37, 7.5, large, -large, 300.0]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=_dt_id)
def test_gelu_gradient_cast_exhaustive(dtype):
    z1 = _finite_values(dtype)
    vals = torch.tensor(_grad_values(dtype), dtype=dtype, device="cuda")
    z = _grid(z1.repeat(vals.numel()))
    dh = _grid(vals.repeat_interleave(z1.numel()))
    dz = torch.ops.aten.gelu_backward(dh, z)
    assert torch.isfinite(dz.float()).all()
    for s in (57344.0 / 4, 57344.0 / 100, 1.0, 2.0 ** -20):   # 57344 / 100: every |dz| > 100 saturates
        s = torch.tensor(s, dtype=torch.float32)
        for layout in (fp8.BOTH, fp8.ROWS, fp8.COLS):
            st, st_ref = _state(s), _state(s)
            out = fp8.cast(dh, st, E5M2, layout, dtype, act=fp8.ACT_DGELU, aux=z)
            ref = fp8.cast(dz, st_ref, E5M2, layout, dtype)
            for a, b in zip(out, ref):
                assert _same(a, b), (s, layout)
            assert torch.equal(st, st_ref), (s, layout)
            if out[0] is not None:
                assert torch.equal(_u8(out[0]), _u8(_ref_cast(dz, s, E5M2))), (s, layout)


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["z_inf", "z_nan", "dh_inf", "dh_nan"])
def test_non_finite_inputs_poison_the_call_and_leave_the_state(where):
    g = torch.Generator(device="cuda").manual_seed(0)
    z = torch.randn(96, 160, device="cuda", generator=g).to(torch.bfloat16)
    dh = torch.randn(96, 160, device="cuda", generator=g).to(torch.bfloat16)
    bad = float("inf") if where.endswith("inf") else float("nan")
    (z if where.startswith("z") else dh)[37, 101] = bad
    st = _state(3.0)
    st.view(torch.float32)[:4] = torch.tensor([1.0, 2.0, 0.5, 0.25])
    st[fp8.HISTORY + 1] = 4
    before = st.clone()
    if where.startswith("z"):
        _, _, inv, _ = fp8.cast(z, st, E4M3, fp8.BOTH, act=fp8.ACT_GELU)
        assert torch.isnan(inv).item() and torch.equal(st, before)
    _, _, inv, _ = fp8.cast(dh, st, E5M2, fp8.BOTH, torch.bfloat16, act=fp8.ACT_DGELU, aux=z)
    assert torch.isnan(inv).item() and torch.equal(st, before)


def _pair(k, i, n, bias, dtype, seed):
    torch.manual_seed(seed)
    fc1, fc2 = Fp8Linear(k, i, bias=bias), Fp8Linear(i, n, bias=bias)
    if bias:
        nn.init.normal_(fc1.bias, std=0.5)
        nn.init.normal_(fc2.bias, std=0.1)
    return fc1.cuda().to(dtype), fc2.cuda().to(dtype)


GRADS = {"all": (True, True, True), "x_frozen": (False, True, True), "weights_frozen": (True, False, False),
         "fc2_only": (False, False, True)}


def _mods_state(fc1, fc2):
    return torch.cat([fc1.scaling_state("cuda").buf, fc2.scaling_state("cuda").buf])


@pytest.mark.gpu
@pytest.mark.parametrize("grads", list(GRADS))
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=_dt_id)
@pytest.mark.parametrize("shape,i,n", [((8192, 1024), 4096, 1024), ((2, 64, 128), 512, 128), ((48, 256), 96, 64)])
def test_block_equals_composition(shape, i, n, dtype, bias, grads):
    x_grad, fc1_grad, fc2_grad = GRADS[grads]
    a1, a2 = _pair(shape[-1], i, n, bias, dtype, seed=i + n)
    for p in a1.parameters():
        p.requires_grad_(fc1_grad)
    for p in a2.parameters():
        p.requires_grad_(fc2_grad)
    b1, b2 = copy.deepcopy(a1), copy.deepcopy(a2)
    g = torch.Generator(device="cuda").manual_seed(7)
    for call in range(3):
        x = (torch.randn(*shape, device="cuda", generator=g) * (1 + call)).to(dtype)
        dy = torch.randn(*shape[:-1], n, device="cuda", generator=g).to(dtype)
        xa, xb = x.clone().requires_grad_(x_grad), x.clone().requires_grad_(x_grad)
        ya = fp8_gelu_mlp(xa, a1, a2)
        yb = b2(F.gelu(b1(xb)))
        assert type(ya.grad_fn).__name__ == FUSED
        ya.backward(dy)
        yb.backward(dy)
        assert _same(ya, yb), call
        assert _same(xa.grad, xb.grad), call
        for (na, pa), pb in zip(list(a1.named_parameters()) + list(a2.named_parameters()),
                                list(b1.parameters()) + list(b2.parameters())):
            assert _same(pa.grad, pb.grad), (call, na)
            pa.grad = pb.grad = None
        assert torch.equal(_mods_state(a1, a2), _mods_state(b1, b2)), call


@pytest.mark.gpu
def test_block_deterministic_and_graph_replay():
    from byteps_b200.torch.graph import GraphedStep

    fc1, fc2 = _pair(1024, 4096, 1024, True, torch.bfloat16, seed=3)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(4, 256, 1024, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    dy = torch.randn(4, 256, 1024, device="cuda", generator=g).to(torch.bfloat16)
    mods = [(copy.deepcopy(fc1), copy.deepcopy(fc2)) for _ in range(3)]

    def run(m1, m2):
        x.grad = None
        for p in list(m1.parameters()) + list(m2.parameters()):
            p.grad = None
        y = fp8_gelu_mlp(x, m1, m2)
        y.backward(dy)
        return [y.detach().clone(), x.grad.clone()] + [p.grad.clone() for p in list(m1.parameters()) +
                                                        list(m2.parameters())]

    eager = [run(*mods[0]) for _ in range(4)]
    again = [run(*mods[1]) for _ in range(4)]
    for a, b in zip(eager, again):
        assert all(torch.equal(u, v) for u, v in zip(a, b)), "run-to-run"
    m1, m2 = mods[2]
    params = list(m1.parameters()) + list(m2.parameters())
    xg = x.detach().clone().requires_grad_(True)

    def step():
        y = fp8_gelu_mlp(xg, m1, m2)
        y.backward(dy)
        return y

    for i in range(2):
        assert torch.equal(step(), eager[i][0]), i
    for t in [xg] + params:
        t.grad = torch.zeros_like(t)
    graphed = GraphedStep(step, warmup=1)
    for t in [xg] + params:
        t.grad.zero_()
    y = graphed()
    torch.cuda.synchronize()
    assert torch.equal(y, eager[3][0]) and torch.equal(xg.grad, eager[3][1])
    assert all(torch.equal(p.grad, e) for p, e in zip(params, eager[3][2:]))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fp32", "rows_not_16", "fc1_plain", "fc2_plain", "noncontig"])
def test_off_fast_path_on_gpu_is_the_composition(case):
    dtype = torch.float32 if case == "fp32" else torch.bfloat16
    a1, a2 = _pair(64, 128, 64, True, dtype, seed=5)
    if case in ("fc1_plain", "fc2_plain"):
        m = a1 if case == "fc1_plain" else a2
        plain = nn.Linear(m.in_features, m.out_features).cuda().to(dtype)
        plain.load_state_dict(m.state_dict())
        a1, a2 = (plain, a2) if case == "fc1_plain" else (a1, plain)
    b1, b2 = copy.deepcopy(a1), copy.deepcopy(a2)
    x = torch.randn(40 if case == "rows_not_16" else 32, 64, device="cuda").to(dtype)
    if case == "noncontig":
        x = torch.randn(64, 32, device="cuda").to(dtype).t()
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    if case == "noncontig":
        xa = x.detach().requires_grad_(True)
        xb = x.detach().clone().t().contiguous().t().requires_grad_(True)
    ya, yb = fp8_gelu_mlp(xa, a1, a2), b2(F.gelu(b1(xb)))
    assert type(ya.grad_fn).__name__ != FUSED
    dy = torch.randn_like(ya)
    ya.backward(dy)
    yb.backward(dy)
    assert _same(ya, yb) and _same(xa.grad, xb.grad)
    for pa, pb in zip(list(a1.parameters()) + list(a2.parameters()), list(b1.parameters()) + list(b2.parameters())):
        assert _same(pa.grad, pb.grad)


def _launches(fn):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return names


@pytest.mark.gpu
def test_fusion_removes_the_gelu_launches():
    a1, a2 = _pair(128, 512, 128, True, torch.bfloat16, seed=9)
    b1, b2 = copy.deepcopy(a1), copy.deepcopy(a2)
    x = torch.randn(256, 128, device="cuda").to(torch.bfloat16).requires_grad_(True)
    dy = torch.randn(256, 128, device="cuda").to(torch.bfloat16)
    paths = {"fused": lambda v: fp8_gelu_mlp(v, a1, a2), "composed": lambda v: b2(F.gelu(b1(v)))}
    counts = {}
    for name, f in paths.items():
        for _ in range(2):   # the seeding calls
            f(x).backward(dy)
        params = list(a1.parameters()) + list(a2.parameters()) + list(b1.parameters()) + list(b2.parameters())
        for p in params + [x]:
            p.grad = None
        out = {}
        fwd = _launches(lambda: out.setdefault("y", f(x)))
        bwd = _launches(lambda: out["y"].backward(dy))
        counts[name] = (fwd, bwd)
    (ff, fb), (cf, cb) = counts["fused"], counts["composed"]
    assert any("gelu" in n.lower() for n in cf) and any("gelu" in n.lower() for n in cb), (cf, cb)
    assert not any("gelu" in n.lower() for n in ff + fb), (ff, fb)
    assert len(ff) == len(cf) - 2, (ff, cf)
    assert len(fb) == len(cb) - 2, (fb, cb)


def _run_py(body: str, timeout=900):
    code = "import sys; sys.path.insert(0, %r)\n" % ROOT + textwrap.dedent(body)
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "DMLC_ROLE", "DMLC_NUM_WORKER", "DMLC_NUM_SERVER"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
    return r.stdout


_BERT = """
import torch
import torch.nn.functional as F
import byteps_b200.models.bert as bert
import byteps_b200.torch as bps
from byteps_b200.torch.graph import GraphedStep
COMPOSED, FUSED, OUT = %r, %r, %r
if COMPOSED:
    bert.fp8_gelu_mlp = lambda x, fc1, fc2: fc2(F.gelu(fc1(x)))
bps.init()
torch.manual_seed(0)
model = bert.bert_tiny(fp8_linear=True, fused_loss=FUSED, fused_norm=FUSED, dropout=0.0).cuda().to(torch.bfloat16)
model.train()
opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=0.01),
                               named_parameters=model.named_parameters(), fused_update=True)
g = torch.Generator().manual_seed(1)
ids = torch.randint(0, 30522, (4, 64), generator=g).cuda()
labels = torch.randint(0, 30522, (4, 64), generator=g)
labels[torch.rand(4, 64, generator=g) > 0.15] = -100
labels = labels.cuda()

def step():
    opt.zero_grad()
    loss = model(ids, mlm_labels=labels)
    loss.backward()
    opt.step()
    return loss

stepper = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams)
losses = [stepper().detach().float().clone() for _ in range(4)]
torch.cuda.synchronize()
torch.save({"losses": torch.stack(losses).cpu(),
            "params": {n: p.detach().cpu() for n, p in model.named_parameters()},
            "fp8": [m.scaling_state("cuda").buf.cpu() for m in model.modules() if type(m).__name__ == "Fp8Linear"]},
           OUT)
print("OK")
bps.shutdown()
"""


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [False, True], ids=["stock_norm_loss", "fused_norm_loss"])
def test_bert_tiny_graphed_equals_composition(tmp_path, fused):
    runs = {}
    for composed in (False, True):
        out = str(tmp_path / ("composed.pt" if composed else "fused.pt"))
        assert "OK" in _run_py(_BERT % (composed, fused, out))
        runs[composed] = torch.load(out)
    a, b = runs[False], runs[True]
    assert torch.isfinite(a["losses"]).all() and torch.equal(a["losses"], b["losses"]), (a["losses"], b["losses"])
    for n, p in a["params"].items():
        assert _same(p, b["params"][n]), n
    assert all(torch.equal(u, v) for u, v in zip(a["fp8"], b["fp8"]))


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("kinds", ["fp8_fp8", "fp8_linear", "linear_fp8", "linear_linear"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=_dt_id)
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
def test_cpu_is_the_composition(kinds, dtype, bias):
    torch.manual_seed(0)
    k1, k2 = kinds.split("_")
    fc1 = (Fp8Linear if k1 == "fp8" else nn.Linear)(64, 128, bias=bias).to(dtype)
    fc2 = (Fp8Linear if k2 == "fp8" else nn.Linear)(128, 48, bias=bias).to(dtype)
    x = torch.randn(2, 16, 64).to(dtype).requires_grad_(True)
    y = fp8_gelu_mlp(x, fc1, fc2)
    ref = fc2(F.gelu(fc1(x)))
    assert type(y.grad_fn).__name__ != FUSED and torch.equal(y, ref)
    params = [x] + list(fc1.parameters()) + list(fc2.parameters())
    gy = torch.randn_like(y)
    assert all(torch.equal(a, b) for a, b in zip(torch.autograd.grad(y, params, gy),
                                                 torch.autograd.grad(ref, params, gy)))
    assert all(getattr(m, "_fp8", None) is None for m in (fc1, fc2)), "no scaling state off the fast path"


@pytest.mark.parametrize("fused_norm", [False, True], ids=["stock_norm", "fused_norm"])
def test_bert_fp8_keeps_the_stock_parameters_and_matches_on_cpu(fused_norm):
    torch.manual_seed(0)
    stock, ours = bert_tiny(fused_norm=fused_norm), bert_tiny(fused_norm=fused_norm, fp8_linear=True)
    assert [(n, p.shape) for n, p in ours.named_parameters()] == [(n, p.shape) for n, p in stock.named_parameters()]
    assert list(ours.state_dict()) == list(stock.state_dict())
    ours.load_state_dict(stock.state_dict(), strict=True)
    ids, labels = torch.randint(0, 30522, (2, 16)), torch.randint(0, 30522, (2, 16))
    for training in (True, False):
        stock.train(training)
        ours.train(training)
        torch.manual_seed(2)
        l1 = stock(ids, mlm_labels=labels)
        torch.manual_seed(2)
        l2 = ours(ids, mlm_labels=labels)
        assert torch.equal(l1, l2), training


def test_binding_rejects_bad_activation_arguments():
    from byteps_b200 import _native

    cu = _native.cuda()
    assert (cu.FP8_ACT_NONE, cu.FP8_ACT_GELU, cu.FP8_ACT_DGELU) == (fp8.ACT_NONE, fp8.ACT_GELU, fp8.ACT_DGELU)
    p = 1 << 20   # never dereferenced: every call below is refused before a launch
    bf16 = 1

    def call(act, aux, dbias=0, fmt=E4M3):
        cu.fp8_cast(p, bf16, 64, 64, fmt, fp8.BOTH, p, p, p, p, dbias, p, p, 0, act, aux)

    for act, aux, dbias in ((3, 0, 0), (-1, 0, 0), (fp8.ACT_DGELU, 0, 0), (fp8.ACT_DGELU, p + 8, 0),
                            (fp8.ACT_GELU, p, 0), (fp8.ACT_NONE, p, 0), (fp8.ACT_GELU, 0, p)):
        with pytest.raises(RuntimeError, match="invalid argument"):
            call(act, aux, dbias)
    assert cu.fp8_cast_workspace(64, 64, bf16, E4M3, fp8.BOTH, False, 3) == (0, 0)
    assert cu.fp8_cast_workspace(64, 64, bf16, E4M3, fp8.BOTH, True, fp8.ACT_GELU) == (0, 0)
    assert cu.fp8_cast_workspace(64, 64, bf16, E5M2, fp8.BOTH, True, fp8.ACT_DGELU)[1] > 0


def test_activation_casts_compile_without_spills(tmp_path):
    from byteps_b200 import _build

    nvcc = _build._nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "byteps_b200", "csrc", "kernels", "fp8.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + _build.ARCH_FLAGS + ["-Xptxas", "-v", "-c", src, "-o",
                                                                         str(tmp_path / "fp8.o")],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    found = {1: 0, 2: 0}
    for block in r.stderr.split("Compiling entry function '")[1:]:
        m = re.match(r"_ZN\S*fp8_cast_kernel\S*ELb[01]ELi(\d)EEEv", block)
        if not m or m.group(1) == "0":
            continue
        act = int(m.group(1))
        found[act] += 1
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block[:400]
        regs = int(re.search(r"Used (\d+) registers", block).group(1))
        assert regs <= 128, (block[:200], regs)    # two 256-thread blocks per SM at least
    assert found == {1: 12, 2: 24}, found
