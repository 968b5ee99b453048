"""Single-launch fused batch norm (bn_act_fwd / bn_act_bwd of kernels/bn_act.cu) against the float64 reference of
test_gpu_bn_act.py, with every row of a block's chunk held in shared memory, part of them, or none.

``ops.bn_act.RESIDENT_CAP`` caps the bytes a block holds, so small shapes reach all three cases; the batch-64 stem
and 256x56x56 layer are only partly held under the default budget.
"""
import copy

import pytest
import torch

from byteps_b200 import _native
from byteps_b200.ops import bn_act as bn_mod
from test_gpu_bn_act import ACTS, DTYPES, RESNET50_BN_SHAPES, _check_bn_act, _dt_id, _make, _run

CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
CAPS = ["full", "part", "none"]


def _plans(n, c, h, w, dtype):
    cu = _native.cuda()
    return [cu.bn_act_plan(d, CODES[dtype], n * h * w, c, bn_mod._cap()) for d in (0, 1)]


@pytest.fixture
def cap():
    """Sets RESIDENT_CAP for one shape ("full": default, "part": half the default bytes, "none": 0) and checks
    that the plans of both directions hold all, some or none of a chunk's rows."""

    def set_cap(mode, n, c, h, w, dtype):
        bn_mod.RESIDENT_CAP = None
        full = _plans(n, c, h, w, dtype)
        assert all(p is not None for p in full), "single-launch plan refused at %s" % ((n, c, h, w),)
        if mode == "part":
            bn_mod.RESIDENT_CAP = min(p["held_bytes"] for p in full) // 2
        elif mode == "none":
            bn_mod.RESIDENT_CAP = 0
        plans = _plans(n, c, h, w, dtype)
        for p in plans:
            if mode == "full":
                assert p["held_rows"] == p["rows_per_chunk"]
            elif mode == "part":
                assert p["held_rows"] < p["rows_per_chunk"]
            else:
                assert p["held_rows"] == 0
        return plans

    yield set_cap
    bn_mod.RESIDENT_CAP = None


def _single_launch_taken(n, c, h, w, dtype):
    bn, x, r, dy = _make(n, c, h, w, dtype, "relu", True)
    y = bn(x.clone().requires_grad_(True), r)
    return y.grad_fn.single_launch_fwd


@pytest.mark.gpu
@pytest.mark.parametrize("mode", CAPS)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("chw", RESNET50_BN_SHAPES, ids=lambda s: "%dx%dx%d" % s)
def test_single_launch_resnet50_shapes(chw, dtype, mode, cap):
    c, h, w = chw
    cap(mode, 2, c, h, w, dtype)
    assert _single_launch_taken(2, c, h, w, dtype)
    for _, act, residual in ACTS:
        _check_bn_act(2, c, h, w, dtype, act, residual)


@pytest.mark.gpu
@pytest.mark.parametrize("chw", [(64, 112, 112), (256, 56, 56)], ids=["stem", "256x56x56"])
def test_single_launch_batch64_partly_held(chw):
    c, h, w = chw
    for p in _plans(64, c, h, w, torch.bfloat16):
        assert p is not None and 0 < p["held_rows"] < p["rows_per_chunk"]
    assert _single_launch_taken(64, c, h, w, torch.bfloat16)
    for _, act, residual in ACTS:
        _check_bn_act(64, c, h, w, torch.bfloat16, act, residual)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["full", "none"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("case,shape,kw", [
    ("c8", (4, 8, 9, 9), {}),
    ("odd_rows", (3, 24, 5, 7), {}),
    ("c40_odd_rows", (1, 40, 37, 3), {}),
    ("mean_100_std", (2, 64, 28, 28), dict(mean_shift=100.0)),
    ("zero_gamma", (2, 128, 14, 14), dict(zero_gamma=True)),
], ids=lambda p: p if isinstance(p, str) else None)
def test_single_launch_edge_cases(case, shape, kw, dtype, mode, cap):
    cap(mode, *shape, dtype)
    for _, act, residual in ACTS:
        _check_bn_act(*shape, dtype, act, residual, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["full", "part"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_single_launch_deterministic_and_graphed(dtype, mode, cap):
    from byteps_b200.torch.graph import GraphedStep

    cap(mode, 8, 256, 28, 28, dtype)
    bn, x, r, dy = _make(8, 256, 28, 28, dtype, "relu", True, seed=3)
    state = copy.deepcopy(bn.state_dict())
    a = _run(bn, x, r, dy)
    bn.load_state_dict(state)
    bn.weight.grad = None
    bn.bias.grad = None
    b = _run(bn, x, r, dy)
    for k in a:
        assert torch.equal(a[k], b[k]), k

    xs, rs = x.detach().clone().requires_grad_(True), r.detach().clone().requires_grad_(True)
    outs = {}

    def step():
        xs.grad = None
        rs.grad = None
        bn.weight.grad = None
        bn.bias.grad = None
        y = bn(xs, rs)
        y.backward(dy)
        outs.update(y=y.detach(), dx=xs.grad, dres=rs.grad, dw=bn.weight.grad, db=bn.bias.grad)
        return y

    g = GraphedStep(step, warmup=2)
    bn.load_state_dict(state)
    g()
    torch.cuda.synchronize()
    for k in ("y", "dx", "dres", "dw", "db"):
        assert torch.equal(outs[k], a[k]), k
    running_mean = bn.running_mean.clone()
    bn.load_state_dict(state)
    _run(bn, x, r, dy)
    assert torch.equal(running_mean, bn.running_mean), "running_mean"


@pytest.mark.gpu
def test_two_pass_when_the_plan_rules_it_out():
    """More channel groups than a wave has blocks: no single-launch plan, and the two-pass kernels run."""
    cu = _native.cuda()
    blocks = cu.bn_act_plan(0, CODES[torch.bfloat16], 2, 256)["wave_blocks"]
    c = 64 * (blocks + 1)      # 8-unit channel groups of 64 channels
    assert _plans(1, c, 1, 2, torch.bfloat16) == [None, None]
    assert not _single_launch_taken(1, c, 1, 2, torch.bfloat16)
    _check_bn_act(1, c, 1, 2, torch.bfloat16, "relu", True)
