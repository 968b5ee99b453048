"""The streaming ring of the single-launch batch-norm kernels (bn_act_fwd / bn_act_bwd of kernels/bn_act.cu).

Rows a block does not hold in shared memory pass through a ring of a few row-steps fed by asynchronous copies, and
each thread pushes its rows into the statistics in row order whatever their source.  So every output must be
bit-identical whether a chunk is held whole, in part or not at all (``ops.bn_act.RESIDENT_CAP``): a row read from
the wrong ring slot shows up as an exact-equality failure.
"""
import copy

import pytest
import torch

from byteps_b200 import _native
from byteps_b200.ops import bn_act as bn_mod
from test_gpu_bn_act import ACTS, DTYPES, _check_bn_act, _dt_id, _make, _run

CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def _plans(m, c, dtype):
    cu = _native.cuda()
    return [cu.bn_act_plan(d, CODES[dtype], m, c, bn_mod._cap()) for d in (0, 1)]


def _outputs(bn, state, x, r, dy, cap):
    bn_mod.RESIDENT_CAP = cap
    try:
        bn.load_state_dict(state)
        bn.weight.grad = None
        bn.bias.grad = None
        out = _run(bn, x, r, dy)
    finally:
        bn_mod.RESIDENT_CAP = None
    out.update(running_mean=bn.running_mean.clone(), running_var=bn.running_var.clone())
    return out


# (N, C, H, W) and how a thread's row-steps per chunk compare with the ring depth when nothing is held
RING_SHAPES = [
    ("fewer", (2, 64, 8, 8)),            # 1 row-step per thread
    ("c40", (3, 40, 37, 29)),            # a partial channel group: threads without channels
    ("not_multiple", (2, 64, 208, 208)),  # 11 row-steps per thread, 10 in the last chunk
    ("far_more", (6, 256, 125, 125)),    # 45 row-steps per thread
]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("case,shape", RING_SHAPES, ids=[c for c, _ in RING_SHAPES])
def test_ring_bit_identical_across_held_rows(case, shape, dtype):
    n, c, h, w = shape
    m = n * h * w
    full = _plans(m, c, dtype)
    assert all(p is not None for p in full)
    part_cap = min(p["held_bytes"] for p in full) // 2
    bn_mod.RESIDENT_CAP = 0
    none = _plans(m, c, dtype)
    bn_mod.RESIDENT_CAP = part_cap
    part = _plans(m, c, dtype)
    bn_mod.RESIDENT_CAP = None
    rl = 256 // min(8 if c >= 256 else 4, 1 << ((c // 8).bit_length() - 1))
    for f, p, z in zip(full, part, none):
        assert p["held_rows"] < f["held_rows"] or f["held_rows"] == 0
        assert z["held_rows"] == 0 and z["ring_depth"] > 0
        steps, depth = z["rows_per_chunk"] // rl, z["ring_depth"]
        if case in ("fewer", "c40"):
            assert steps < depth
        elif case == "not_multiple":
            assert steps > depth and steps % depth != 0
        else:
            assert steps >= 4 * depth
    for _, act, residual in ACTS:
        bn, x, r, dy = _make(n, c, h, w, dtype, act, residual, seed=5)
        state = copy.deepcopy(bn.state_dict())
        ref = _outputs(bn, state, x, r, dy, None)
        for cap in (part_cap, 0):
            out = _outputs(bn, state, x, r, dy, cap)
            for k, v in ref.items():
                if v is None:
                    assert out[k] is None
                else:
                    assert torch.equal(out[k], v), "%s differs at RESIDENT_CAP=%d (%s)" % (k, cap, act)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=_dt_id)
@pytest.mark.parametrize("chw", [(64, 112, 112), (256, 56, 56)], ids=["stem", "256x56x56"])
def test_ring_batch64_against_float64(chw, dtype):
    """The two largest ResNet-50 layers at batch 64 stream most of their rows through the ring (bf16 is checked in
    test_gpu_bn_act_resident.py)."""
    c, h, w = chw
    for p in _plans(64 * h * w, c, dtype):
        assert p is not None and p["ring_depth"] > 0 and 0 < p["held_rows"] < p["rows_per_chunk"]
    for _, act, residual in ACTS:
        _check_bn_act(64, c, h, w, dtype, act, residual)


@pytest.mark.gpu
@pytest.mark.parametrize("chw", [(64, 56, 56), (256, 28, 28), (1024, 14, 14)], ids=lambda s: "%dx%dx%d" % s)
def test_forward_holds_the_25mb_layers_whole(chw):
    """x of the batch-64 layers of 25.7 MB (bf16) fits on chip across the 132 SMs of an H100: a forward block
    holds its whole chunk, so x is read from HBM once."""
    c, h, w = chw
    cu = _native.cuda()
    p = cu.bn_act_plan(0, CODES[torch.bfloat16], 64 * h * w, c)
    if p["wave_blocks"] != 264:
        pytest.skip("the figures are for 132 SMs")
    assert p["held_rows"] == p["rows_per_chunk"] and p["ring_depth"] == 0
    assert p["bytes_moved"] == 64 * h * w * c * 2 * 2
