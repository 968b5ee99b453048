"""Batch norm (kernels/bn_act.cu) and LayerNorm (kernels/ln.cu) at every launch geometry their planners produce.

The other test files pick their shapes from ResNet-50 and BERT-base, so they only launch the geometries those shapes
produce.  Here the shapes are chosen by geometry: the width of a block's channel group and whether the last group is
partial, the row chunking of a launch, each LayerNorm row layout with a full and a partial last pass, more than 2^31
elements, and inputs whose data does not start on a 16-byte boundary.  Every numerical check reuses the float64
references and bounds of test_gpu_bn_act.py, test_gpu_ln.py and test_gpu_sync_bn.py, or requires bit-identity with
a path those files check.

Batch-norm geometry (kernels/bn_act.cu): a thread covers one unit of 8 channels; a block covers CB units of one
channel group (CB the largest power of two <= min(units, max CB)) times RL = 256 / CB rows.  The reductions and the
single-launch kernels use max CB = 8 from C = 256 up and 4 below it; the elementwise passes of the two-pass and
synchronised kernels use max CB = 32.  A single launch cuts the M rows into G chunks, one per block of a channel
group.
"""
import copy
import types

import pytest
import torch
import torch.nn as nn

import test_gpu_bn_act as tb
import test_gpu_bn_act_junction as tj
import test_gpu_bn_act_pool as tp
import test_gpu_ln as tl
from byteps_b200 import _native
from byteps_b200.ops import bn_act as bn_mod
from byteps_b200.ops.bn_act import BatchNormAct2d, SyncBatchNormAct2d
from byteps_b200.ops.ln import dropout_add_layer_norm
from test_gpu_bn_act import ACTS, C_ACC, DTYPES, TINY, U32, UNIT, _check_bn_act, _dt_id, _run
from test_gpu_bn_act_junction import summed_in_kernel  # noqa: F401  (fixture)
from test_gpu_bn_act_resident import _single_launch_taken, cap  # noqa: F401  (cap: fixture)
from test_gpu_sync_bn import _check_against_float64, _cluster, _launch_bwd, _launch_fwd, _RankBufs, _rows

CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
CAPS = ["full", "part", "none"]
PATHS = ["single_launch", "two_pass"]


def _shape_id(s):
    return "x".join(map(str, s))


# ------------------------------------------------------------------------------------------ batch-norm geometry
# (N, C, H, W) and the geometry classes each reaches (G and chunk lengths on a 132-SM H100)
BN_SHAPES = [
    (4, 8, 9, 9),       # reduce CB 1 (RL 256); M = 324: G = 2, the last chunk 68 rows
    (4, 16, 9, 9),      # reduce CB 2, full
    (2, 24, 37, 3),     # reduce CB 2, partial (3 units)
    (2, 64, 28, 28),    # reduce CB 4, full; G = 25, the last chunk 32 of 64 rows
    (3, 200, 7, 9),     # reduce CB 4, partial (25 units); apply CB 16, partial (16 + 9 units)
    (1, 40, 1, 2),      # M = 2, the fewest rows the fused kernels take: G = 1, M < RL; reduce CB 4, partial
    (2, 256, 7, 7),     # reduce CB 8, full (4 groups); apply CB 32, full
    (2, 264, 9, 11),    # reduce CB 8, partial (33 units: 4 x 8 + 1); apply CB 32, partial (32 + 1)
    (2, 1000, 7, 7),    # reduce CB 8, partial (125 units: 15 x 8 + 5); apply CB 32, partial (3 x 32 + 29)
    (1, 2056, 3, 5),    # 33 reduce groups of 8 units, the last of 1; M = 15 < RL = 32: G = 1
]
# every class the single-launch and apply grids can take; a CB-1 group is one unit, so it is never partial
BN_CLASSES = {"reduce CB %d, %s" % (cb, kind) for cb in (2, 4, 8) for kind in ("full", "partial")} | {
    "reduce CB 1, full", "apply CB 16, partial", "apply CB 32, partial", "G = 1, M < RL",
    "G > 1, short last chunk", "M = 2"}
# the shapes whose last 8-unit reduction group is partial (C >= 256, C % 64 != 0)
PARTIAL_8 = [s for s in BN_SHAPES if s[1] >= 256 and s[1] % 64]


def _cb(c, max_cb):
    """geo() of kernels/bn_act.cu: units per block row of a channel group."""
    units, cb = c // 8, 1
    while 2 * cb <= units and 2 * cb <= max_cb:
        cb *= 2
    return cb


def _red_cb(c):
    return 8 if c >= 256 else 4


def _partial(c):
    units = c // 8
    return units % _cb(c, _red_cb(c)) != 0 or units % _cb(c, 32) != 0


# the shapes with a partial reduction or apply group
PARTIAL = [s for s in BN_SHAPES if _partial(s[1])]


def _bn_classes(shape):
    """The geometry classes the single-launch plans of both directions, and the apply grid, take at `shape`."""
    n, c, h, w = shape
    m, units = n * h * w, c // 8
    cb = _cb(c, _red_cb(c))
    seen = set()
    for d in (0, 1):
        p = _native.cuda().bn_act_plan(d, CODES[torch.bfloat16], m, c)
        assert p is not None, "no single-launch plan at %s" % (shape,)
        assert p["counters"] == -(-units // cb), "the planner's channel groups are not geo()'s"
        g, rpc = p["ws_floats"] // (2 * c), p["rows_per_chunk"]
        assert g == -(-m // rpc) and rpc % (256 // cb) == 0
        seen.add("reduce CB %d, %s" % (cb, "full" if units % cb == 0 else "partial"))
        if g == 1 and m < 256 // cb:
            seen.add("G = 1, M < RL")
        if g > 1 and m % rpc:
            seen.add("G > 1, short last chunk")
    acb = _cb(c, 32)
    if acb >= 16 and units % acb:
        seen.add("apply CB %d, partial" % acb)
    if m == 2:
        seen.add("M = 2")
    return seen


@pytest.mark.gpu
def test_bn_shapes_cover_every_geometry_class():
    per_shape = {s: _bn_classes(s) for s in BN_SHAPES}
    table = "\n".join("%-16s %s" % (_shape_id(s), ", ".join(sorted(k))) for s, k in per_shape.items())
    print("\n" + table)
    seen = set().union(*per_shape.values())
    assert seen >= BN_CLASSES, "classes no shape reaches: %s\n%s" % (sorted(BN_CLASSES - seen), table)


class _NoPlan:
    """``_native.cuda()`` whose ``bn_act_plan`` finds no single-launch plan, as on a device without cooperative
    launch: the module runs the two-pass kernels.  Records the batch-norm launchers called."""

    def __init__(self, cu):
        self._cu, self.calls = cu, []

    def bn_act_plan(self, *args, **kwargs):
        return None

    def __getattr__(self, name):
        fn = getattr(self._cu, name)
        if not name.startswith("bn_act_") or name in ("bn_act_workspace", "bn_act_load_kernels"):
            return fn

        def call(*args, **kwargs):
            self.calls.append(name)
            return fn(*args, **kwargs)

        return call


@pytest.fixture
def two_pass(monkeypatch):
    proxy = _NoPlan(_native.cuda())
    monkeypatch.setattr(bn_mod, "_native", types.SimpleNamespace(cuda=lambda: proxy))
    return proxy


TWO_PASS_CALLS = ["bn_act_fwd_stats", "bn_act_fwd_apply", "bn_act_bwd_reduce", "bn_act_bwd_apply"]


@pytest.fixture(params=PATHS)
def path(request):
    """The single-launch kernels, or the two-pass kernels (``two_pass``)."""
    if request.param == "two_pass":
        request.getfixturevalue("two_pass")
    return request.param


@pytest.fixture
def cap_reset():
    yield
    bn_mod.RESIDENT_CAP = None


@pytest.mark.gpu
@pytest.mark.parametrize("mode", CAPS)
@pytest.mark.parametrize("shape", BN_SHAPES, ids=_shape_id)
def test_single_launch_geometry(shape, mode, cap):
    for dtype in DTYPES:
        cap(mode, *shape, dtype)
        assert _single_launch_taken(*shape, dtype)
        for _, act, residual in ACTS:
            _check_bn_act(*shape, dtype, act, residual)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("shape", BN_SHAPES, ids=_shape_id)
def test_two_pass_geometry(shape, dtype, two_pass):
    for _, act, residual in ACTS:
        two_pass.calls.clear()
        _check_bn_act(*shape, dtype, act, residual)
        assert two_pass.calls == TWO_PASS_CALLS


@pytest.mark.gpu
@pytest.mark.parametrize("mode", CAPS)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("shape", PARTIAL_8, ids=_shape_id)
def test_junction_sum_partial_groups(shape, dtype, mode, summed_in_kernel):  # noqa: F811
    """Two gradients summed in the kernel: bit-identical to the backward fed torch's sum of them."""
    bn, x, r, g1, g2 = tj._make(shape, dtype, seed=2)
    state = copy.deepcopy(bn.state_dict())
    tj._set_cap(mode, shape, dtype)
    want = tj._backward(bn, state, x, r, (g1 + g2,), pair=False)
    got = tj._backward(bn, state, x, r, (g1, g2), pair=True)
    assert summed_in_kernel == [True]
    tj._assert_same(got, want)


POOL_SHAPE = (2, 264, 9, 7)   # partial 8-unit group, odd H and W


@pytest.mark.gpu
@pytest.mark.parametrize("mode", CAPS)
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_pooled_stem_partial_group(dtype, mode, cap_reset):
    """The pooled kernels: bit-identical to the batch norm followed by torch's max pool and gradient add."""
    bn, x, g1, g2 = tp._make(POOL_SHAPE, dtype, seed=1)
    state = copy.deepcopy(bn.state_dict())
    tp._set_cap(mode, POOL_SHAPE, dtype)
    for grads in ((g1, g2), (g1, None)):
        want, kind = tp._run(bn, state, x, grads, pooled=False)
        assert kind != "_BatchNormActPoolFnBackward"
        got, kind = tp._run(bn, state, x, grads, pooled=True)
        assert kind == "_BatchNormActPoolFnBackward", "pooled path not taken"
        tp._assert_same(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("world", [2, 3])
def test_sync_kernels_partial_groups(world, dtype):
    """The synchronised kernels (two-pass reductions, apply grids of up to 32 units) at every shape with a partial
    group, through the virtual-rank harness of test_gpu_sync_bn.py."""
    cu = _native.cuda()
    vc, ctxs = _cluster(world, max(s[1] for s in PARTIAL))
    for i, (n, c, h, w_) in enumerate(PARTIAL):
        for j, (_, act, residual) in enumerate(ACTS):
            g = torch.Generator(device="cuda").manual_seed(100 * world + 10 * i + j)
            bufs = [_RankBufs(m, c, dtype, act, residual, g) for m in _rows(world, n * h * w_)]
            w = torch.randn(c, device="cuda", generator=g)
            bias = torch.randn(c, device="cuda", generator=g) * 0.5
            rm0, rv0 = torch.randn(c, device="cuda", generator=g), torch.rand(c, device="cuda", generator=g) + 0.5
            rms, rvs = [rm0.clone() for _ in range(world)], [rv0.clone() for _ in range(world)]
            vc.run(lambda r, view, arena, s: _launch_fwd(cu, ctxs[r], bufs[r], w, bias, rms[r], rvs[r], s))
            vc.run(lambda r, view, arena, s: _launch_bwd(cu, ctxs[r], bufs[r], w, s))
            torch.cuda.synchronize()
            _check_against_float64(bufs, w, bias, rms, rvs, rm0, rv0, act)


# ---------------------------------------------------------------------------------------------- module options
OPT_SHAPE = (2, 264, 9, 11)


def _same(got, want):
    for k, v in want.items():
        assert (v is None and got[k] is None) or torch.equal(got[k], v), k


def _check_running(bn, x, rm0, rv0, factor):
    """The running statistics after one step from (rm0, rv0) with averaging factor `factor`, against a float64
    F.batch_norm on the same input, within the bounds of test_gpu_bn_act._check_bn_act."""
    dims = (0, 2, 3)
    xd = x.double()
    rm_ref, rv_ref = rm0.clone(), rv0.clone()
    torch.nn.functional.batch_norm(xd, rm_ref, rv_ref, None, None, True, factor, bn.eps)
    mu, var = xd.mean(dims), xd.var(dims, unbiased=False)
    shift = mu.abs() / torch.sqrt(var + bn.eps) + 1.0
    assert torch.all((bn.running_mean.double() - rm_ref).abs() <= C_ACC * U32 * (rm0.abs() + mu.abs() + var.sqrt()))
    assert torch.all((bn.running_var.double() - rv_ref).abs() <= C_ACC * U32 * (rv0.abs() + var * shift))


def _module_like(ref, **kw):
    bn = BatchNormAct2d(ref.num_features, act=ref.act, **kw).cuda().train()
    with torch.no_grad():
        bn.weight.copy_(ref.weight)
        bn.bias.copy_(ref.bias)
    return bn


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_momentum_none_three_steps(dtype, path):
    """momentum=None averages the running statistics with factor 1 / num_batches_tracked.  Each step's outputs and
    gradients equal, bit for bit, those of the float64-checked step of _check_bn_act on the same inputs."""
    bn = None
    for step in (1, 2, 3):
        ref, x, r, dy, want = _check_bn_act(*OPT_SHAPE, dtype, "relu", True, seed=step)
        if bn is None:
            bn = _module_like(ref, momentum=None)
            with torch.no_grad():
                bn.running_mean.copy_(ref.running_mean * 3.0)
                bn.running_var.copy_(ref.running_var + 1.0)
        with torch.no_grad():   # an optimizer step between batches
            bn.weight.copy_(ref.weight)
            bn.bias.copy_(ref.bias)
        bn.weight.grad = bn.bias.grad = None
        rm0, rv0 = bn.running_mean.double(), bn.running_var.double()
        _same(_run(bn, x, r, dy), want)
        assert int(bn.num_batches_tracked) == step
        _check_running(bn, x, rm0, rv0, 1.0 / step)


@pytest.mark.gpu
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_without_running_stats(dtype, training, path):
    """track_running_stats=False: the kernels get no running-statistics pointers, and eval mode still normalises
    with the batch statistics on the fused path."""
    ref, x, r, dy, want = _check_bn_act(*OPT_SHAPE, dtype, "relu", True, seed=4)
    bn = _module_like(ref, track_running_stats=False).train(training)
    assert bn.running_mean is None and bn.running_var is None and bn.num_batches_tracked is None
    _same(_run(bn, x, r, dy), want)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_non_default_eps(dtype, path, monkeypatch):
    """eps = 0.1: comparable with the batch variances of _make (0.25 to 6.25), so a kernel that used another eps
    would miss the float64 reference of _check_bn_act by far more than its bounds."""
    make = tb._make

    def with_eps(*args, **kwargs):
        bn, x, r, dy = make(*args, **kwargs)
        bn.eps = 0.1
        return bn, x, r, dy

    monkeypatch.setattr(tb, "_make", with_eps)
    for _, act, residual in ACTS:
        bn = _check_bn_act(*OPT_SHAPE, dtype, act, residual)[0]
        assert bn.eps == 0.1


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_pooled_momentum_none_three_steps(dtype):
    """The pooled stem with momentum=None over three steps: bit-identical to the unpooled module followed by torch's
    max pool, running statistics and num_batches_tracked included."""
    ref, _, _, _ = tp._make(POOL_SHAPE, dtype)
    pooled = _module_like(ref, momentum=None)
    chain = copy.deepcopy(pooled)
    for step in (1, 2, 3):
        _, x, g1, g2 = tp._make(POOL_SHAPE, dtype, seed=step)
        rm0, rv0 = pooled.running_mean.double(), pooled.running_var.double()
        want, _ = tp._run(chain, copy.deepcopy(chain.state_dict()), x, (g1, g2), pooled=False)
        got, kind = tp._run(pooled, copy.deepcopy(pooled.state_dict()), x, (g1, g2), pooled=True)
        assert kind == "_BatchNormActPoolFnBackward", "pooled path not taken"
        tp._assert_same(got, want)
        assert int(pooled.num_batches_tracked) == int(chain.num_batches_tracked) == step
        _check_running(pooled, x, rm0, rv0, 1.0 / step)


# ---------------------------------------------------------------------------------------------- LayerNorm layouts
# LN_LAYOUT of kernels/ln.cu: (largest H, units a thread holds (NU), threads per row (TPR)).  A row's TPR threads
# take units l, l + TPR, ...; the last of the NU passes is full only at the layout's largest H.
LN_LAYOUTS = [(128, 1, 16), (256, 1, 32), (512, 2, 32), (1024, 2, 64), (2048, 2, 128)]
LN_H = [8, 24, 120, 128, 136, 200, 256, 264, 392, 512, 520, 1000, 1024, 1032, 1544, 2040, 2048]
LN_DROPOUT_H = [120, 200, 392, 1000, 1544]   # one partial width per layout
K_GROUP = 16   # kGroup of kernels/ln.cu: the backward sums its block partials in runs of 16 blocks


def _ln_layout(h):
    return next((nu, tpr) for top, nu, tpr in LN_LAYOUTS if h <= top)


def _ln_rows(h):
    """M = 1, one row short of and one past a block's rows per step (RPB), and 16 RPB + 1: a backward of 17 blocks,
    one run of kGroup blocks and a run of one."""
    rpb = 256 // _ln_layout(h)[1]
    return sorted({1, max(rpb - 1, 1), rpb + 1, K_GROUP * rpb + 1})


def test_ln_widths_cover_every_layout():
    seen = {(_ln_layout(h), "full" if h == next(t for t, _, _ in LN_LAYOUTS if h <= t) else "partial") for h in LN_H}
    want = {((nu, tpr), kind) for _, nu, tpr in LN_LAYOUTS for kind in ("full", "partial")}
    assert seen == want, sorted(want - seen)
    assert {_ln_layout(h) for h in LN_DROPOUT_H} == {(nu, tpr) for _, nu, tpr in LN_LAYOUTS}


@pytest.mark.gpu
def test_ln_rows_end_on_a_partial_block_run():
    cu = _native.cuda()
    for h in LN_H:
        m = _ln_rows(h)[-1]
        ws, ctr = cu.ln_workspace(m, h)
        g = ws // (2 * h) - (ctr - 1)    # workspace: (G + runs) * 2H floats; counters: runs + 1
        assert g > K_GROUP and g % K_GROUP != 0, (h, m, g)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,wdtype", tl.WDTYPES, ids=["%s-w%s" % (_dt_id(a), _dt_id(b)) for a, b in tl.WDTYPES])
@pytest.mark.parametrize("h", LN_H)
def test_ln_layout_matches_float64(h, dtype, wdtype):
    for m in _ln_rows(h):
        for residual in (False, True):
            tl._check(m, h, dtype, wdtype, residual)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,wdtype", tl.WDTYPES, ids=["%s-w%s" % (_dt_id(a), _dt_id(b)) for a, b in tl.WDTYPES])
@pytest.mark.parametrize("h", LN_DROPOUT_H)
def test_ln_layout_dropout_matches_float64(h, dtype, wdtype):
    for residual in (False, True):
        tl._check(_ln_rows(h)[-1], h, dtype, wdtype, residual, p=0.1, seed=3)


# ---------------------------------------------------------------------------------------------- > 2^31 elements
def _chunks(m, step):
    return ((r0, min(m, r0 + step)) for r0 in range(0, m, step))


@pytest.mark.gpu
def test_bn_act_more_than_2_31_elements():
    """The stem's batch norm at batch 2676 in bf16 (2.15e9 elements), in one launch per direction.  Statistics,
    running statistics and parameter gradients against float64 sums over all rows, y and dx on the rows on both sides
    of element 2^31, all within the bounds of test_gpu_bn_act._check_bn_act."""
    n, c, h, w = 2676, 64, 112, 112
    m = n * h * w
    assert m * c > 2 ** 31
    dtype, cu = torch.bfloat16, _native.cuda()
    assert all(cu.bn_act_plan(d, CODES[dtype], m, c) is not None for d in (0, 1))
    g = torch.Generator(device="cuda").manual_seed(12)
    bn = BatchNormAct2d(c, act="relu").cuda().train()
    with torch.no_grad():
        bn.weight.copy_(torch.randn(c, device="cuda", generator=g))
        bn.bias.copy_(torch.randn(c, device="cuda", generator=g) * 0.5)
        bn.running_mean.copy_(torch.randn(c, device="cuda", generator=g))
        bn.running_var.copy_(torch.rand(c, device="cuda", generator=g) + 0.5)
    rm0, rv0 = bn.running_mean.double(), bn.running_var.double()
    scale = (torch.rand(c, device="cuda", generator=g) * 2 + 0.5).to(dtype)
    loc = torch.randn(c, device="cuda", generator=g).to(dtype)
    rows = torch.randn(m, c, device="cuda", generator=g, dtype=dtype).mul_(scale).add_(loc)   # x as (M, C)
    dy_rows = torch.randn(m, c, device="cuda", generator=g, dtype=dtype)
    nchw = lambda t: t.view(n, h, w, c).permute(0, 3, 1, 2)  # noqa: E731  (channels_last)
    x = nchw(rows).requires_grad_(True)
    y = bn(x)
    assert type(y.grad_fn).__name__ == "_BatchNormActFnBackward" and y.grad_fn.single_launch_fwd
    _, _, mean, invstd, _ = y.grad_fn.saved_tensors
    y.backward(nchw(dy_rows))
    y_rows = y.detach().permute(0, 2, 3, 1).reshape(m, c)
    dx_rows = x.grad.permute(0, 2, 3, 1).reshape(m, c)
    assert y_rows.data_ptr() == y.data_ptr() and dx_rows.data_ptr() == x.grad.data_ptr()
    x, y = None, None

    # float64 sums in chunks of rows: the mean, then the centred sums
    step = 1 << 20
    mu = sum(rows[a:b].double().sum(0) for a, b in _chunks(m, step)) / m
    q = torch.zeros(c, dtype=torch.float64, device="cuda")
    db_ref, sgd, sg, sgd_abs = q.clone(), q.clone(), q.clone(), q.clone()
    for a, b in _chunks(m, step):
        d = rows[a:b].double() - mu
        q += (d * d).sum(0)
        gd = dy_rows[a:b].double() * (y_rows[a:b] > 0)
        db_ref += gd.sum(0)
        sg += gd.abs().sum(0)
        gd *= d
        sgd += gd.sum(0)
        sgd_abs += gd.abs().sum(0)
        del d, gd
    var = q / m
    inv = 1.0 / torch.sqrt(var + bn.eps)
    dw_ref, sgx = sgd * inv, sgd_abs * inv
    shift = mu.abs() * inv + 1.0
    assert torch.all((mean.double() - mu).abs() <= C_ACC * U32 * (mu.abs() + var.sqrt()))
    assert torch.all((invstd.double() - inv).abs() <= C_ACC * U32 * inv * shift)
    rm_ref = 0.9 * rm0 + 0.1 * mu
    rv_ref = 0.9 * rv0 + 0.1 * var * m / (m - 1)
    assert torch.all((bn.running_mean.double() - rm_ref).abs() <= C_ACC * U32 * (rm0.abs() + mu.abs() + var.sqrt()))
    assert torch.all((bn.running_var.double() - rv_ref).abs() <= C_ACC * U32 * (rv0.abs() + var * shift))
    assert torch.all((bn.bias.grad.double() - db_ref).abs() <= C_ACC * U32 * sg), "dbias"
    assert torch.all((bn.weight.grad.double() - dw_ref).abs() <= C_ACC * U32 * (sgx + shift * sg + dw_ref.abs()))

    # y and dx on the rows around element 2^31 (row 2^31 / C starts at it)
    edge = 2 ** 31 // c
    pick = torch.tensor([0, 1, edge - 2, edge - 1, edge, edge + 1, m - 2, m - 1], device="cuda")
    ut = UNIT[dtype]
    wd, bd = bn.weight.detach().double(), bn.bias.detach().double()
    xhat = (rows[pick].double() - mu) * inv
    y_ref = torch.relu(xhat * wd + bd)
    mag = (xhat.abs() * shift + shift) * wd.abs() + bd.abs()
    tol_y = C_ACC * U32 * mag + ut * (y_ref.abs() + C_ACC * U32 * mag) + TINY[dtype]
    err_y = (y_rows[pick].double() - y_ref).abs()
    assert (err_y <= tol_y).all(), "y: worst excess %g" % (err_y - tol_y).max().item()
    gd = dy_rows[pick].double() * (y_rows[pick] > 0)
    a = wd * inv
    dx_ref = a * (gd - db_ref / m - xhat * dw_ref / m)
    mag_dx = a.abs() * (gd.abs() + (xhat.abs() * shift + shift) * ((sgx + shift * sg + dw_ref.abs()) / m) + sg / m)
    tol_dx = C_ACC * U32 * mag_dx * (1 + ut) + ut * dx_ref.abs() + TINY[dtype]
    err_dx = (dx_rows[pick].double() - dx_ref).abs()
    assert (err_dx <= tol_dx).all(), "dx: worst excess %g" % (err_dx - tol_dx).max().item()


@pytest.mark.gpu
def test_ln_more_than_2_31_elements():
    """bf16 rows of H = 1024 (2.15e9 elements), fp32 parameters: out and dy on the rows on both sides of element 2^31,
    dgamma and dbeta against float64 sums over all rows in chunks, within the bounds of test_gpu_ln._check."""
    h, dtype, wdtype = 1024, torch.bfloat16, torch.float32
    m = 2 ** 31 // h + 4096
    assert m * h > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(13)
    y = torch.randn(m, h, device="cuda", generator=g, dtype=dtype).mul_(2).add_(
        torch.randn(m, 1, device="cuda", generator=g, dtype=dtype))
    dout = torch.randn(m, h, device="cuda", generator=g, dtype=dtype)
    w = torch.randn(h, device="cuda", generator=g).requires_grad_(True)
    b = (torch.randn(h, device="cuda", generator=g) * 0.5).requires_grad_(True)
    yg = y.requires_grad_(True)
    out = dropout_add_layer_norm(yg, None, w, b, 0.0, tl.EPS, True)
    assert type(out.grad_fn).__name__ == "_DropoutAddLayerNormFnBackward"
    out.backward(dout)
    out, dy = out.detach(), yg.grad
    y = yg.detach()
    yg = None

    def reference(zb, gb):
        """Per row of the chunk: xhat, shift and rstd of the float64 LayerNorm, as test_gpu_ln._check forms them."""
        zd = zb.double()
        mu = zd.mean(-1, keepdim=True)
        rstd = 1.0 / torch.sqrt(zd.var(-1, unbiased=False, keepdim=True) + tl.EPS)
        return (zd - mu) * rstd, mu.abs() * rstd + 1.0, rstd, gb.double()

    ut, uw = UNIT[dtype], UNIT[wdtype]
    wd, bd = w.detach().double(), b.detach().double()
    edge = 2 ** 31 // h
    pick = torch.tensor([0, 1, edge - 2, edge - 1, edge, edge + 1, m - 2, m - 1], device="cuda")
    xhat, shift, rstd, gd = reference(y[pick], dout[pick])
    out_ref = xhat * wd + bd
    mag = (xhat.abs() + shift) * wd.abs() + bd.abs()
    tol = C_ACC * U32 * mag + ut * (out_ref.abs() + C_ACC * U32 * mag) + TINY[dtype]
    err = (out[pick].double() - out_ref).abs()
    assert (err <= tol).all(), "out: worst excess %g" % (err - tol).max().item()
    gw = gd * wd
    ma, mb = gw.mean(-1, keepdim=True), (gw * xhat).mean(-1, keepdim=True)
    dz_ref = rstd * (gw - ma - xhat * mb)
    big_a = gw.abs().mean(-1, keepdim=True)
    big_b = (gw.abs() * (xhat.abs() + shift)).mean(-1, keepdim=True)
    mag_dz = rstd * (gw.abs() + big_a + (xhat.abs() + shift) * big_b)
    tol_dz = C_ACC * U32 * mag_dz + ut * (dz_ref.abs() + C_ACC * U32 * mag_dz) + TINY[dtype]
    err = (dy[pick].double() - dz_ref).abs()
    assert (err <= tol_dz).all(), "dy: worst excess %g" % (err - tol_dz).max().item()

    dw_ref, db_ref, tol_dw, tol_db = (torch.zeros(h, dtype=torch.float64, device="cuda") for _ in range(4))
    for a, b_ in _chunks(m, 1 << 16):
        xhat, shift, _, gd = reference(y[a:b_], dout[a:b_])
        dw_ref += (gd * xhat).sum(0)
        db_ref += gd.sum(0)
        tol_dw += (gd.abs() * (xhat.abs() + shift)).sum(0)
        tol_db += gd.abs().sum(0)
    tol_dw = C_ACC * U32 * tol_dw
    tol_db = C_ACC * U32 * tol_db
    tol_dw = tol_dw + uw * (dw_ref.abs() + tol_dw) + TINY[wdtype]
    tol_db = tol_db + uw * (db_ref.abs() + tol_db) + TINY[wdtype]
    assert ((w.grad.double() - dw_ref).abs() <= tol_dw).all(), "dgamma"
    assert ((b.grad.double() - db_ref).abs() <= tol_db).all(), "dbeta"


# ---------------------------------------------------------------------------------------------- misaligned inputs
def _misaligned_rows(t):
    """A contiguous copy of t whose data starts one element past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


def _bn_step(bn, state, x, r, grads, pair=False):
    """y, running statistics and every gradient of one step from `state`; x, r and the gradients are used as given
    (views keep their offset)."""
    bn.load_state_dict(state)
    bn.weight.grad = bn.bias.grad = None
    xg, rg = x.detach().requires_grad_(True), r.detach().requires_grad_(True)
    out = bn(xg, rg, pair=pair)
    outs = list(out) if pair else [out]
    assert type(outs[0].grad_fn).__name__ == "_BatchNormActFnBackward", "fused path not taken"
    torch.autograd.backward(outs[:len(grads)], list(grads))
    return dict(y=outs[0].detach().clone(), rm=bn.running_mean.clone(), rv=bn.running_var.clone(), dx=xg.grad,
                dres=rg.grad, dw=bn.weight.grad.clone(), db=bn.bias.grad.clone())


BN_MISALIGNED = [(case, p) for p in PATHS for case in ("x", "residual", "dy")] + [("first_of_pair", "single_launch")]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
@pytest.mark.parametrize("case,route", BN_MISALIGNED, ids=["%s-%s" % c for c in BN_MISALIGNED])
def test_bn_misaligned_input_is_copied(case, route, dtype, request):
    """A channels_last view one element past a 16-byte boundary gives, bit for bit, what its aligned copy gives."""
    if route == "two_pass":
        request.getfixturevalue("two_pass")
    bn, x, r, dy = tb._make(*OPT_SHAPE, dtype, "relu", True, seed=5)
    dy2 = torch.randn_like(dy)
    state = copy.deepcopy(bn.state_dict())
    pair = case == "first_of_pair"
    grads = (dy, dy2) if pair else (dy,)
    want = _bn_step(bn, state, x, r, grads, pair)
    odd = {"x": x, "residual": r, "dy": dy, "first_of_pair": dy}[case]
    mis = tj._misaligned(odd)
    assert torch.equal(mis, odd) and mis.data_ptr() % 16 != 0 and bn_mod._nhwc(mis)
    x2, r2 = (mis if case == "x" else x), (mis if case == "residual" else r)
    got = _bn_step(bn, state, x2, r2, (mis, dy2) if pair else ((mis,) if case == "dy" else grads), pair)
    _same(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt_id)
def test_pooled_misaligned_input_is_copied(dtype, cap_reset):
    bn, x, g1, g2 = tp._make(POOL_SHAPE, dtype, seed=6)
    state = copy.deepcopy(bn.state_dict())
    want, _ = tp._run(bn, state, x, (g1, g2), pooled=True)
    mis = tj._misaligned(x)
    assert torch.equal(mis, x) and mis.data_ptr() % 16 != 0
    bn.load_state_dict(state)
    bn.weight.grad = bn.bias.grad = None
    xg = mis.detach().requires_grad_(True)
    p, alias = bn(xg, pool=nn.MaxPool2d(3, 2, 1), pair=True)
    assert type(p.grad_fn).__name__ == "_BatchNormActPoolFnBackward", "pooled path not taken"
    torch.autograd.backward([p, alias], [g1, g2])
    got = dict(p=p.detach(), rm=bn.running_mean.clone(), rv=bn.running_var.clone(), dx=xg.grad,
               dw=bn.weight.grad.clone(), db=bn.bias.grad.clone())
    tp._assert_same(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["x", "residual", "dy"])
def test_sync_misaligned_input_is_copied(case):
    """Synchronised batch norm at world 2 on virtual ranks: a misaligned x, residual or dy on every rank gives, bit for
    bit, what aligned copies give.  The run follows the hang-safe pattern of test_gpu_sync_bn.py's module test: a
    local warm-up on every rank's stream first loads every kernel the synchronised runs launch."""
    world, c, ns = 2, 264, [2, 3]
    vc, ctxs = _cluster(world, c)
    torch.manual_seed(0)
    base = SyncBatchNormAct2d(c, act="relu").cuda().train()
    with torch.no_grad():
        base.weight.copy_(torch.randn(c) * 0.5 + 1.0)
        base.bias.copy_(torch.randn(c) * 0.5)
    state = copy.deepcopy(base.state_dict())
    bns = [copy.deepcopy(base) for _ in range(world)]
    nhwc = lambda t: t.contiguous(memory_format=torch.channels_last)  # noqa: E731
    xs = [nhwc(torch.randn(n, c, 5, 3, device="cuda") * 2 + 1) for n in ns]
    rs = [nhwc(torch.randn(n, c, 5, 3, device="cuda")) for n in ns]
    dys = [nhwc(torch.randn(n, c, 5, 3, device="cuda")) for n in ns]
    odd = {"x": xs, "residual": rs, "dy": dys}[case]
    mis = [tj._misaligned(t) for t in odd]
    assert all(torch.equal(a, b) and a.data_ptr() % 16 != 0 for a, b in zip(mis, odd))

    def inputs(misaligned):
        ins = dict(x=xs, residual=rs, dy=dys)
        if misaligned:
            ins[case] = mis
        return ins["x"], ins["residual"], ins["dy"]

    for misaligned in (False, True):   # warm-up with local statistics: loads every kernel, both ways
        x_, r_, dy_ = inputs(misaligned)
        for r in range(world):
            with torch.cuda.stream(vc.streams[r]):
                xg = x_[r].detach().requires_grad_(True)
                bns[r](xg, r_[r]).backward(dy_[r])
    torch.cuda.synchronize()

    runs = []
    for misaligned in (False, True):
        x_, r_, dy_ = inputs(misaligned)
        for r, bn in enumerate(bns):
            bn.load_state_dict(state)
            bn.zero_grad(set_to_none=True)
            bn.sync = ctxs[r]
        xg = [x_[r].detach().requires_grad_(True) for r in range(world)]
        rg = [r_[r].detach().requires_grad_(True) for r in range(world)]
        ys = [None] * world
        cur = torch.cuda.current_stream()
        for s in vc.streams:
            s.wait_stream(cur)
        for r in range(world):
            with torch.cuda.stream(vc.streams[r]):
                ys[r] = bns[r](xg[r], rg[r])
        for r in range(world):
            with torch.cuda.stream(vc.streams[r]):
                ys[r].backward(dy_[r])
        for s in vc.streams:
            cur.wait_stream(s)
        torch.cuda.synchronize()
        assert all(type(y.grad_fn).__name__ == "_SyncBatchNormActFnBackward" for y in ys)
        runs.append([[ys[r].detach(), xg[r].grad, rg[r].grad, bns[r].weight.grad.clone(), bns[r].bias.grad.clone(),
                      bns[r].running_mean.clone(), bns[r].running_var.clone()] for r in range(world)])
        for bn in bns:
            bn.sync = None
    for r, (a, b) in enumerate(zip(*runs)):
        for i, (u, v) in enumerate(zip(a, b)):
            assert torch.equal(u, v), "rank %d output %d" % (r, i)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,wdtype", tl.WDTYPES, ids=["%s-w%s" % (_dt_id(a), _dt_id(b)) for a, b in tl.WDTYPES])
@pytest.mark.parametrize("case", ["y", "residual", "dout", "weight"])
def test_ln_misaligned_input_is_copied(case, dtype, wdtype):
    """A view one element past a 16-byte boundary gives, bit for bit, what its aligned copy gives (dropout 0.1 with
    the same seed, so the keep masks agree too)."""
    m, h = 65, 1000
    y, r, dout, w, b = tl._make(m, h, dtype, wdtype, True, seed=7)

    def run(y, r, dout, w):
        yg, rg = y.detach().requires_grad_(True), r.detach().requires_grad_(True)
        wg, bg = w.detach().requires_grad_(True), b.detach().clone().requires_grad_(True)
        torch.manual_seed(5)
        out, mask = dropout_add_layer_norm(yg, rg, wg, bg, 0.1, tl.EPS, True, return_mask=True)
        assert type(out.grad_fn).__name__ == "_DropoutAddLayerNormFnBackward", "fused path not taken"
        out.backward(dout)
        return dict(out=out.detach(), mask=mask, dy=yg.grad, dres=rg.grad, dw=wg.grad, db=bg.grad)

    want = run(y, r, dout, w)
    odd = {"y": y, "residual": r, "dout": dout, "weight": w}[case]
    mis = _misaligned_rows(odd)
    assert torch.equal(mis, odd) and mis.data_ptr() % 16 != 0
    ins = dict(y=y, residual=r, dout=dout, weight=w)
    ins[case] = mis
    _same(run(ins["y"], ins["residual"], ins["dout"], ins["weight"]), want)
