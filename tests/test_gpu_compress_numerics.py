"""The GPU gradient compressors against a float64 reference, stage by stage.

Every stage is checked one step deep: its inputs are what the previous stage left on the device (or a snapshot
of the state before the step), its output is compared with the same operation in float64.  For a value computed
with c fp32 roundings from terms whose absolute values add up to A (the stage's formula evaluated on |terms|),

    |out - e| <= c 2^-24 A + c 2^-150

and where the kernel stores a bf16 or f16 result, half an ulp of that dtype plus its smallest half-subnormal on
top (`_bounds.stored`).  The constants c, per stage:

    corrected gradient   m' = mu m + g           2            p = g + mu m' + ratio e     2 + 2 + 2
                         (with or without FMA contraction; terms that are off drop out)
    sums over n          (per-thread trips + 8 tree levels + partial trips + 8 tree levels [+ 1 division])
    onebit consumer      sum_p +-scale_p (+ err2): P    out = mult sum: P + 1    worker error: 1
    top-k / random-k     sparse or dense sum of P payloads (+ err2): P          mult x value: 1
    dithering            level x scale: 2 (+1 for q / s)  error: 3  slot sum: P + 1  unpack: 3

Onebit signs, top-k selections and random-k indices are exact claims on the kernel's own fp32 values.  Dithering
levels are reproduced from the counter-based splitmix64 draws; a level may differ from the float64 model only
where the model is ambiguous within the fp32 bound of t, and those are counted.  `test_bounds_reject_wrong_models`
shows on the CPU that the bounds tell the kernels' arithmetic from nearby wrong models.

Kernel-level cases call the bindings directly and fill one buffer with P payloads from P producer calls, so the
consumers (which read local slots) run at any size without a cross-rank kernel.  Pipeline cases run
`GpuCompressor` on virtual ranks of one GPU in lockstep with world x blocks <= 64, after every configuration has
run once on a single rank, so no module loads while a rank spins on its peers' flags.
"""
import math

import numpy as np
import pytest
import torch
from _bounds import BF16, DT, F16, F32, HALF_MIN_SUB, UNIT, stored

U = UNIT[F32]
TINY = HALF_MIN_SUB[F32]
DTYPES = ["f32", "bf16", "f16"]
SIZES = [1, 3, 31, 33, 127, 129, 5000, 65_537, 1_081_345, 4_194_305, 31_254_528]
BIG = 31_254_528                 # BERT-large's 30522 x 1024 embedding
P = 3                            # payloads summed by the kernel-level consumers
MULT = 1.0 / 3.0
GUARD = 4096


def _cu():
    from byteps_b200 import _native

    return _native.cuda()


def _code(dt):
    from byteps_b200.comm.symm import wire_code

    return wire_code(dt)


def f32(x):
    return float(torch.tensor(x, dtype=F32))


def bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def report(kind, what, ratio):
    print("compress-numerics: %-9s %-52s max err/bound = %.4f" % (kind, what, ratio))


def check(out, e, b, what, dt=F32):
    """|out - e| <= b elementwise (b widened by the store to dt); returns max err/bound."""
    if dt != F32:
        b = stored(e.abs(), b, dt)
    err = (out.double() - e).abs()
    bad = ~(err <= b)
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: %d of %d out of bound, first at %d: got %r, want %r, bound %r" % (
            what, int(bad.sum()), out.numel(), i, out.reshape(-1)[i].item(), e.reshape(-1)[i].item(),
            b.reshape(-1)[i].item()))
    return (err / b).max().item() if out.numel() else 0.0


def sum_depth(n, items_per_thread, grid, threads=256):
    """fp32 roundings on the way from n terms to one sum: per-thread trips, warp + block tree (8 levels),
    per-thread trips over the grid's partials, tree again."""
    trips = -(-n // (grid * threads * items_per_thread)) * items_per_thread
    return trips + 8 + -(-grid // 256) + 8


def grid_fused(items):
    return max(1, min(1056, -(-items // 256)))


# ------------------------------------------------------------------------------------------------ inputs
def make_grad(n, dt, seed):
    """Normals over 13 binades; from 64 elements on: [0:2) +0, [2:4) -0, [4:12) subnormals of dt, [12:20) values
    one ulp of dt above [20:28)."""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    x = torch.randn(n, generator=g, device="cuda") * torch.exp2(
        torch.randint(-6, 7, (n,), generator=g, device="cuda").float())
    x = x.to(dt)
    if n >= 64:
        kmax, emin = {F16: (1023, -24), BF16: (127, -133), F32: (1 << 22, -149)}[dt]
        x[0:2] = 0.0
        x[2:4] = -0.0
        k = torch.randint(-kmax, kmax + 1, (8,), generator=g, device="cuda").double()
        x[4:12] = (k * 2.0 ** emin).to(dt)
        x[12:20] = x[20:28]
        bits(x[12:20]).add_(1)
    return x


def make_state(n, seed, scale=0.5):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    s = torch.randn(n, generator=g, device="cuda") * scale
    s[:4] = 0.0
    return s


def corrected_ref(g, mom, mu, err, ratio):
    """float64 p = g + mu m' + ratio e with m' = mu m + g; returns (p, bound of p, m', bound of m')."""
    g64 = g.double()
    p, a, c = g64.clone(), g64.abs(), 0
    m_new = mb = None
    if mom is not None:
        mu = f32(mu)
        m_new = mu * mom.double() + g64
        am = mu * mom.double().abs() + g64.abs()
        mb = 2 * U * am + 2 * TINY
        p = g64 + mu * m_new
        a = g64.abs() + mu * am
        c += 4
    if err is not None:
        ratio = f32(ratio)
        p = p + ratio * err.double()
        a = a + ratio * err.double().abs()
        c += 2
    return p, c * U * a + c * TINY, m_new, mb


# ------------------------------------------------------------------------------------------------ onebit
def decode_signs(words, n):
    """Bit j of the MSB-first words: element j is negative."""
    w = words[: (n + 31) // 32].long() & 0xFFFFFFFF
    sh = 31 - torch.arange(32, device=w.device)
    return ((w[:, None] >> sh) & 1).reshape(-1)[:n].bool()


def check_signs(neg, p_gpu, p64, pb, what):
    """bit == (p_gpu < 0) where p_gpu is known, else bit == (p64 < 0) wherever |p64| exceeds its bound."""
    if p_gpu is not None:
        want = p_gpu < 0
        bad = neg != want
    else:
        bad = (neg != (p64 < 0)) & (p64.abs() > pb)
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: sign bit of element %d is %d for p = %r" % (
            what, i, int(neg[i]), (p_gpu if p_gpu is not None else p64)[i].item()))


def check_mean_abs(got, vals, n, depth, what, extra=0.0):
    """got = mean |vals| after `depth` fp32 roundings (and one division)."""
    s = vals.double().abs().sum()
    e = s / n
    b = ((depth + 1) * U * s + extra) / n + TINY
    return check(torch.tensor([got], dtype=torch.float64, device=e.device), e.reshape(1), b.reshape(1), what)


ONEBIT_OPTS = [   # (mom, ef, scaled, p_out written, two-stage consumer)
    (False, False, False, True, False),
    (True, True, True, True, True),
    (False, True, True, False, True),
    (True, False, False, False, False),
    (True, True, False, True, False),
    (False, False, True, True, True),
]


def _cases(n_opts):
    out = []
    for i, n in enumerate(SIZES):
        for j, dt in enumerate(DTYPES):
            if n == BIG and dt == "f16":
                continue
            out.append((n, dt, (i + j) % n_opts if n != BIG else 1))
    return out


def _ids(cases):
    return ["n%d-%s-o%d" % c for c in cases]


ONEBIT_CASES = _cases(len(ONEBIT_OPTS))


@pytest.mark.gpu
@pytest.mark.parametrize("n,dt,opt", ONEBIT_CASES, ids=_ids(ONEBIT_CASES))
def test_onebit_kernels(n, dt, opt):
    cu, d = _cu(), DT[dt]
    use_mom, use_ef, scaled, write_p, two = ONEBIT_OPTS[opt]
    mu, ratio = 0.9, (2.0 if opt % 2 else 0.25)
    s = torch.cuda.current_stream().cuda_stream
    from byteps_b200.ops.compress import GpuCompressor

    slot = GpuCompressor.slot_bytes_for({"compressor_type": "onebit"}, n)
    nwords = (n + 31) // 32
    slots = torch.zeros(P * slot // 4, dtype=torch.int32, device="cuda")
    parts = torch.zeros(cu.FUSED_MAX_BLOCKS, dtype=F32, device="cuda")
    counter = torch.zeros(4, dtype=torch.int32, device="cuda")
    grid = grid_fused((n + 127) // 128 * 32)
    depth = sum_depth(n, 4, grid) + 1      # chunks of 4 per lane, one lane per 4 elements: 4 per trip
    worst = {}
    ps, p64s, pbs = [], [], []
    for r in range(P):
        g = make_grad(n, d, 10 * n + r)
        mom = make_state(n, 11 + r) if use_mom else None
        err = make_state(n, 21 + r) if use_ef else None
        p64, pb, m64, mb = corrected_ref(g, mom, mu, err, ratio)
        # with error feedback p replaces the error state in place, as in the pipeline
        p_out = err if use_ef else (torch.full((n,), 7.0, device="cuda") if write_p else None)
        words_ptr = slots.data_ptr() + r * slot
        cu.onebit_pre(g.data_ptr(), _code(d), mom.data_ptr() if use_mom else 0, mu, err.data_ptr() if use_ef else 0,
                      ratio, p_out.data_ptr() if p_out is not None else 0, n, words_ptr, scaled, parts.data_ptr(),
                      counter.data_ptr(), s)
        torch.cuda.synchronize()
        what = "onebit_pre %s n=%d rank %d" % (dt, n, r)
        if p_out is not None:
            worst["p"] = max(worst.get("p", 0), check(p_out, p64, pb, what + " p"))
        if use_mom:
            worst["mom"] = max(worst.get("mom", 0), check(mom, m64, mb, what + " momentum"))
        w = slots[r * slot // 4: r * slot // 4 + nwords + 1]
        neg = decode_signs(w, n)
        check_signs(neg, p_out, p64, pb, what)
        tail = n % 32
        if tail:
            assert (w[nwords - 1].item() & ((1 << (32 - tail)) - 1)) == 0, what + ": bits past n are set"
        sc = w[nwords:nwords + 1].view(F32).item()
        if scaled:
            src = p_out if p_out is not None else p64
            extra = 0.0 if p_out is not None else pb.sum().item()
            worst["scale"] = max(worst.get("scale", 0), check_mean_abs(sc, src, n, depth, what + " scale", extra))
        else:
            assert sc == 1.0, what
        ps.append(p_out.clone() if p_out is not None else None)
        p64s.append(p64)
        pbs.append(pb)

    # consumer: rank `me` finishes its error feedback, the sum goes to c2 (two-stage) or to out
    me = 1
    scs = torch.tensor([slots[r * slot // 4 + nwords].view(F32).item() for r in range(P)], dtype=torch.float64,
                       device="cuda")
    negs = [decode_signs(slots[r * slot // 4: r * slot // 4 + nwords], n) for r in range(P)]
    e_sum = sum(torch.where(negs[r], -scs[r], scs[r]) for r in range(P))
    a_sum = scs.sum().expand(n)
    err_me = ps[me].clone() if use_ef else None
    err_me0 = err_me.clone() if use_ef else None
    what = "onebit consumer %s n=%d" % (dt, n)
    if two:
        err2 = make_state(n, 99) if use_ef else None
        c2 = err2 if use_ef else torch.empty(n, device="cuda")
        err2_0 = err2.clone() if use_ef else None
        scale2 = torch.zeros(4, device="cuda")
        cu.onebit_sum(slots.data_ptr(), slot, P, me, n, err_me.data_ptr() if use_ef else 0,
                      err2.data_ptr() if use_ef else 0, c2.data_ptr(), 0, _code(d), MULT, scaled, parts.data_ptr(),
                      counter.data_ptr(), scale2.data_ptr(), s)
        torch.cuda.synchronize()
        e_c2 = e_sum + (err2_0.double() if use_ef else 0)
        a_c2 = a_sum + (err2_0.double().abs() if use_ef else 0)
        worst["c2"] = check(c2, e_c2, P * U * a_c2 + P * TINY, what + " c2")
        c2_gpu = c2.clone()
        sc2 = scale2[0].item()
        if scaled:
            worst["scale2"] = check_mean_abs(sc2, c2_gpu, n, depth, what + " scale2")
        else:
            assert sc2 == 1.0
        out = torch.empty(n, dtype=d, device="cuda")
        cu.onebit_out(c2.data_ptr(), n, scale2.data_ptr(), err2.data_ptr() if use_ef else 0, out.data_ptr(),
                      _code(d), MULT, s)
        torch.cuda.synchronize()
        dsign = torch.where(c2_gpu < 0, -1.0, 1.0).double()
        e_out = dsign * f32(MULT) * sc2
        worst["out"] = check(out, e_out, U * e_out.abs() + TINY, what + " out", d)
        if use_ef:
            e_e2 = c2_gpu.double() - dsign * sc2
            worst["err2"] = check(err2, e_e2, U * (c2_gpu.double().abs() + sc2) + TINY, what + " err2")
    else:
        out = torch.empty(n, dtype=d, device="cuda")
        cu.onebit_sum(slots.data_ptr(), slot, P, me, n, err_me.data_ptr() if use_ef else 0, 0, 0, out.data_ptr(),
                      _code(d), MULT, scaled, parts.data_ptr(), counter.data_ptr(), 0, s)
        torch.cuda.synchronize()
        m = f32(MULT)
        worst["out"] = check(out, m * e_sum, (P + 1) * U * m * a_sum + TINY, what + " out", d)
    if use_ef:
        pme = err_me0.double()
        sgn = torch.where(negs[me], -1.0, 1.0).double()
        worst["err"] = check(err_me, pme - sgn * scs[me], U * (pme.abs() + scs[me]) + TINY, what + " worker error")
        assert torch.equal(negs[me], err_me0 < 0), what + ": consumer sign differs from the payload's"
    for k, v in worst.items():
        report("onebit", "%s %s n=%d opt %d" % (k, dt, n, opt), v)


# ------------------------------------------------------------------------------------------------ top-k
def check_topk_selection(x, pairs, k, what):
    """k unique indices below n, every kept |x| >= every dropped |x|, values bit-equal to x[idx]."""
    n = x.numel()
    idx = pairs[0::2].long()
    vals = pairs[1::2]
    assert idx.min().item() >= 0 and idx.max().item() < n, what + ": index out of range"
    kept = torch.zeros(n, dtype=torch.bool, device=x.device)
    kept[idx] = True
    assert int(kept.sum()) == k, what + ": %d unique indices for k = %d" % (int(kept.sum()), k)
    assert torch.equal(vals, bits(x)[idx]), what + ": values differ from the kernel's own p at their index"
    if k < n:
        lo = x.abs()[kept].min().item()
        hi = x.abs()[~kept].max().item()
        assert lo >= hi, what + ": kept |x| %r below dropped |x| %r" % (lo, hi)
        # ties at the threshold are kept lowest index first, so every rank selecting from the same sum agrees
        tie = (x.abs() == lo).nonzero().flatten()
        n_kept = int(kept[tie].sum())
        assert kept[tie[:n_kept]].all(), what + ": tied entries are not kept lowest index first"
    return idx, kept


def topk_ks(n):
    return sorted({k for k in (1, 37, max(1, n // 100), max(1, n // 5), n) if k <= n})


TOPK_OPTS = [   # (mom, ef, input: normal | ties, two-stage consumer)
    (False, False, "normal", False),
    (True, True, "normal", True),
    (False, True, "ties", True),
    (False, False, "ties", False),
]
TOPK_CASES = _cases(len(TOPK_OPTS))


def _ties(n, dt, seed):
    """Few distinct magnitudes: every threshold has many ties."""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    v = torch.tensor([0.5, 1.0, -1.0, 2.0, -2.0, 0.0], device="cuda")
    return v[torch.randint(0, 6, (n,), generator=g, device="cuda")].to(dt)


@pytest.mark.gpu
@pytest.mark.parametrize("n,dt,opt", TOPK_CASES, ids=_ids(TOPK_CASES))
def test_topk_kernels(n, dt, opt):
    cu, d = _cu(), DT[dt]
    use_mom, use_ef, kind, two = TOPK_OPTS[opt]
    mu, ratio = 0.9, (2.0 if opt % 2 else 0.25)
    s = torch.cuda.current_stream().cuda_stream
    tk = torch.zeros(cu.TOPK_SCRATCH_BYTES // 4, dtype=torch.int32, device="cuda")
    ks = topk_ks(n) if n != BIG else [n // 100, n // 5]
    worst = {}
    for k in ks:
        slot = (k * 8 + 255) // 256 * 256
        slots = torch.zeros(P * slot // 4, dtype=torch.int32, device="cuda")
        for r in range(P):
            g = make_grad(n, d, 7 * n + r) if kind == "normal" else _ties(n, d, 7 * n + r)
            mom = make_state(n, 31 + r) if use_mom else None
            # ties survive the correction when the error state is a power-of-two multiple of the gradient
            err = (g.float() * 0.5 if kind == "ties" else make_state(n, 41 + r)) if use_ef else None
            p64, pb, m64, mb = corrected_ref(g, mom, mu, err, ratio)
            p_buf = err if use_ef else torch.empty(n, device="cuda")
            cu.topk_pre(g.data_ptr(), _code(d), mom.data_ptr() if use_mom else 0, mu, err.data_ptr() if use_ef else 0,
                        ratio, p_buf.data_ptr(), n, k, tk.data_ptr(), s)
            torch.cuda.synchronize()
            what = "topk_pre %s n=%d k=%d rank %d" % (dt, n, k, r)
            p_gpu = p_buf.clone()
            worst["p"] = max(worst.get("p", 0), check(p_gpu, p64, pb, what + " p"))
            if use_mom:
                worst["mom"] = max(worst.get("mom", 0), check(mom, m64, mb, what + " momentum"))
            pairs = slots[r * slot // 4: r * slot // 4 + 2 * k]
            cu.topk_finish(p_buf.data_ptr(), n, k, 1, pairs.data_ptr(), use_ef, tk.data_ptr(), s)
            torch.cuda.synchronize()
            idx, kept = check_topk_selection(p_gpu, pairs, k, what)
            exp = p_gpu.clone()
            if use_ef:
                exp[idx] = 0.0
            assert torch.equal(bits(p_buf), bits(exp)), what + ": bytes other than the kept entries changed"
        # consumer: sparse add of the P payloads in rank order, then the second stage or the cast
        what = "topk consumer %s n=%d k=%d" % (dt, n, k)
        err2 = make_state(n, 77) if (use_ef and two) else None
        acc = err2 if err2 is not None else torch.zeros(n, device="cuda")
        e = acc.double().clone()
        a = acc.double().abs()
        for r in range(P):
            pr = slots[r * slot // 4: r * slot // 4 + 2 * k]
            cu.sparse_add_pairs(pr.data_ptr(), k, n, acc.data_ptr(), s)
            i, v = pr[0::2].long(), pr[1::2].view(F32).double()
            e.index_add_(0, i, v)
            a.index_add_(0, i, v.abs())
        torch.cuda.synchronize()
        worst["sum"] = max(worst.get("sum", 0), check(acc, e, P * U * a + P * TINY, what + " sum"))
        out = torch.empty(n, dtype=d, device="cuda")
        m = f32(MULT)
        if two:
            acc_gpu = acc.clone()
            local2 = torch.zeros(2 * k, dtype=torch.int32, device="cuda")
            cu.topk_finish(acc.data_ptr(), n, k, 0, local2.data_ptr(), err2 is not None, tk.data_ptr(), s)
            torch.cuda.synchronize()
            idx, kept = check_topk_selection(acc_gpu, local2, k, what + " second stage")
            if err2 is not None:
                exp = acc_gpu.clone()
                exp[idx] = 0.0
                assert torch.equal(bits(acc), bits(exp)), what + ": err2 changed outside the kept entries"
            cu.scatter_pairs(local2.data_ptr(), k, n, out.data_ptr(), _code(d), MULT, s)
            torch.cuda.synchronize()
            e_out = torch.where(kept, m * acc_gpu.double(), torch.zeros_like(e))
        else:
            cu.cast_scale4(acc.data_ptr(), n, out.data_ptr(), _code(d), MULT, s)
            torch.cuda.synchronize()
            e_out = m * acc.double()
        worst["out"] = max(worst.get("out", 0), check(out, e_out, U * e_out.abs() + TINY, what + " out", d))
        del slots
    for key, v in worst.items():
        report("topk", "%s %s n=%d opt %d" % (key, dt, n, opt), v)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_topk_pre_redoes_a_too_optimistic_sampled_filter(dt):
    """Large values sit exactly on the sample stride, so the sampled threshold is too high and the producer's
    filtered level-0 histogram holds fewer than k keys: the unfiltered redo must run on the producer path."""
    cu, d = _cu(), DT[dt]
    n = 131072 * 2 + 5
    k = n // 100
    g = torch.Generator(device="cuda")
    g.manual_seed(8)
    x = torch.rand(n, generator=g, device="cuda") * 1e-3
    pos = torch.arange(0, 2000, device="cuda") * (n // 32768)
    x[pos] = 10.0 + torch.rand(2000, generator=g, device="cuda")
    x = x.to(d)
    err = make_state(n, 5, 1e-4)
    p64, pb, _, _ = corrected_ref(x, None, 0.0, err, 2.0)
    p = err
    tk = torch.zeros(cu.TOPK_SCRATCH_BYTES // 4, dtype=torch.int32, device="cuda")
    pairs = torch.zeros(2 * k, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    cu.topk_pre(x.data_ptr(), _code(d), 0, 0.0, err.data_ptr(), 2.0, p.data_ptr(), n, k, tk.data_ptr(), s)
    torch.cuda.synchronize()
    p_gpu = p.clone()
    r = check(p_gpu, p64, pb, "adversarial p")
    cu.topk_finish(p.data_ptr(), n, k, 1, pairs.data_ptr(), True, tk.data_ptr(), s)
    torch.cuda.synchronize()
    check_topk_selection(p_gpu, pairs, k, "adversarial sample %s" % dt)
    report("topk", "p %s adversarial sample n=%d" % (dt, n), r)


# ------------------------------------------------------------------------------------------------ random-k
def _sseed(seed):
    return seed - (1 << 64) if seed >= (1 << 63) else seed


def cpu_stream(rng, k, n):
    buf = np.zeros(k, dtype=np.uint32)
    rng.fill_randint_u32(buf.ctypes.data, k, n)
    return torch.from_numpy(buf.astype(np.int64)).cuda()


def last_occurrence(idx, n):
    """For every index, the position of its last draw (or -1)."""
    k = idx.numel()
    last = torch.full((n,), -1, dtype=torch.int64, device=idx.device)
    last.scatter_reduce_(0, idx, torch.arange(k, device=idx.device), reduce="amax")
    return last


RANDOMK_OPTS = [  # (mom, ef, two-stage)
    (False, False, False),
    (True, True, True),
    (False, True, True),
    (True, False, False),
]
RANDOMK_CASES = _cases(len(RANDOMK_OPTS))


@pytest.mark.gpu
@pytest.mark.parametrize("n,dt,opt", RANDOMK_CASES, ids=_ids(RANDOMK_CASES))
def test_randomk_kernels(n, dt, opt):
    from byteps_b200 import _native

    cu, core, d = _cu(), _native.core(), DT[dt]
    use_mom, use_ef, two = RANDOMK_OPTS[opt]
    mu, ratio = 0.9, (2.0 if opt % 2 else 0.25)
    s = torch.cuda.current_stream().cuda_stream
    seed = 0x9E3779B97F4A7C15 + n
    seed &= (1 << 64) - 1
    jump = torch.frombuffer(bytearray(cu.xorshift_jump_table()), dtype=torch.int64).cuda()
    ks = sorted({max(1, n // 100), max(1, n // 5)})
    worst = {}
    far = 0
    for k in ks:
        state = torch.tensor([_sseed(seed)] * 2, dtype=torch.int64, device="cuda")
        state2 = torch.tensor([_sseed(seed)] * 2, dtype=torch.int64, device="cuda")
        rng = core.XorShift128Plus()
        rng.set_seed(seed)
        idx = torch.empty(k, dtype=torch.int32, device="cuda")
        # two draws: the second continues the stream
        for rep in range(2):
            cu.randomk_draw(state.data_ptr(), jump.data_ptr(), k, n, idx.data_ptr(), s)
            torch.cuda.synchronize()
            want = cpu_stream(rng, k, n)
            assert torch.equal(idx.long(), want), "randomk_draw n=%d k=%d draw %d differs from the CPU stream" % (
                n, k, rep)
        il = idx.long()
        slot = (k * 4 + 255) // 256 * 256
        slots = torch.zeros(P * slot // 4, dtype=F32, device="cuda")
        for r in range(P):
            g = make_grad(n, d, 3 * n + r)
            mom = make_state(n, 51 + r) if use_mom else None
            err = make_state(n, 61 + r) if use_ef else None
            p64, pb, m64, mb = corrected_ref(g, mom, mu, err, ratio)
            vals = slots[r * slot // 4: r * slot // 4 + k]
            cu.randomk_pre(g.data_ptr(), _code(d), mom.data_ptr() if use_mom else 0, mu,
                           err.data_ptr() if use_ef else 0, ratio, n, idx.data_ptr(), k, vals.data_ptr(), s)
            torch.cuda.synchronize()
            what = "randomk_pre %s n=%d k=%d rank %d" % (dt, n, k, r)
            worst["vals"] = max(worst.get("vals", 0), check(vals, p64[il], pb[il], what + " vals"))
            if use_mom:
                worst["mom"] = max(worst.get("mom", 0), check(mom, m64, mb, what + " momentum"))
            if use_ef:
                drawn = torch.zeros(n, dtype=torch.bool, device="cuda")
                drawn[il] = True
                assert (bits(err)[drawn] == 0).all(), what + ": a drawn entry of err is not +0"
                worst["err"] = max(worst.get("err", 0), check(err[~drawn], p64[~drawn], pb[~drawn], what + " err"))
        what = "randomk consumer %s n=%d k=%d" % (dt, n, k)
        vsum = torch.empty(k, device="cuda")
        cu.dense_sum_slots(slots.data_ptr(), slot, P, k, vsum.data_ptr(), s)
        torch.cuda.synchronize()
        vs = [slots[r * slot // 4: r * slot // 4 + k].double() for r in range(P)]
        worst["sum"] = max(worst.get("sum", 0), check(vsum, sum(vs), (P - 1) * U * sum(v.abs() for v in vs) + TINY,
                                                      what + " sum"))
        last = last_occurrence(il, n)
        pos = torch.arange(k, device="cuda")
        prev = torch.full((n,), -1, dtype=torch.int64, device="cuda")
        first = prev.scatter_reduce(0, il, pos, reduce="amin", include_self=False)
        far += int(((last - first) > 64).sum())
        m = f32(MULT)

        def scattered(values, mult):
            e = torch.zeros(n, dtype=torch.float64, device="cuda")
            hit = last >= 0
            e[hit] = mult * values.double()[last[hit]]
            return e

        if two:
            sm = torch.empty(n, device="cuda")
            cu.index_scatter(idx.data_ptr(), vsum.data_ptr(), k, n, sm.data_ptr(), 0, 1.0, s)
            torch.cuda.synchronize()
            assert torch.equal(sm.double(), scattered(vsum, 1.0)), what + ": fp32 scatter"
            idx2 = torch.empty(k, dtype=torch.int32, device="cuda")
            rng2 = core.XorShift128Plus()
            rng2.set_seed(seed)
            cu.randomk_draw(state2.data_ptr(), jump.data_ptr(), k, n, idx2.data_ptr(), s)
            torch.cuda.synchronize()
            assert torch.equal(idx2.long(), cpu_stream(rng2, k, n)), what + ": second-stage stream"
            err2 = make_state(n, 88) if use_ef else None
            e2_0 = err2.clone() if use_ef else None
            vals2 = torch.empty(k, device="cuda")
            cu.randomk_pre(sm.data_ptr(), 0, 0, 0.0, err2.data_ptr() if use_ef else 0, 1.0, n, idx2.data_ptr(), k,
                           vals2.data_ptr(), s)
            torch.cuda.synchronize()
            i2 = idx2.long()
            c2 = sm.double() + (e2_0.double() if use_ef else 0)
            ac2 = sm.double().abs() + (e2_0.double().abs() if use_ef else 0)
            worst["vals2"] = check(vals2, c2[i2], U * ac2[i2] + TINY, what + " vals2")
            if use_ef:
                drawn = torch.zeros(n, dtype=torch.bool, device="cuda")
                drawn[i2] = True
                assert (bits(err2)[drawn] == 0).all(), what + ": a drawn entry of err2 is not +0"
                worst["err2"] = check(err2[~drawn], c2[~drawn], U * ac2[~drawn] + TINY, what + " err2")
            out = torch.empty(n, dtype=d, device="cuda")
            cu.index_scatter(idx2.data_ptr(), vals2.data_ptr(), k, n, out.data_ptr(), _code(d), MULT, s)
            torch.cuda.synchronize()
            last = last_occurrence(i2, n)
            e_out = scattered(vals2, m)
        else:
            out = torch.empty(n, dtype=d, device="cuda")
            cu.index_scatter(idx.data_ptr(), vsum.data_ptr(), k, n, out.data_ptr(), _code(d), MULT, s)
            torch.cuda.synchronize()
            e_out = scattered(vsum, m)
        worst["out"] = max(worst.get("out", 0), check(out, e_out, U * e_out.abs() + TINY, what + " out", d))
    for key, v in worst.items():
        report("randomk", "%s %s n=%d opt %d" % (key, dt, n, opt), v)
    print("compress-numerics: randomk   %s n=%d: %d indices drawn again more than 64 draws later" % (dt, n, far))


# ------------------------------------------------------------------------------------------------ dithering
M64 = (1 << 64) - 1
SM_A, SM_B, SM_C, SM_D = 0x9E3779B97F4A7C15, 0xBF58476D1CE4E5B9, 0x94D049BB133111EB, 0x2545F4914F6CDD1D


def _lsr(z, s):
    return (z >> s) & ((1 << (64 - s)) - 1)


def splitmix_uniform(seed, step, idx):
    """rng_uniform of compress.cu for int64 indices, in wrapping int64 arithmetic: (z >> 40) * 2^-24."""
    base = (seed * SM_A + step * SM_B + SM_D) & M64
    z = idx * _sseed(SM_C) + _sseed(base)
    z = (z ^ _lsr(z, 30)) * _sseed(SM_B)
    z = (z ^ _lsr(z, 27)) * _sseed(SM_C)
    z = z ^ _lsr(z, 31)
    return _lsr(z, 40).double() * 2.0 ** -24


def splitmix_uniform_int(seed, step, i):
    """The same draw with Python integers."""
    z = (seed * SM_A + step * SM_B + i * SM_C + SM_D) & M64
    z = ((z ^ (z >> 30)) * SM_B) & M64
    z = ((z ^ (z >> 27)) * SM_C) & M64
    z ^= z >> 31
    return (z >> 40) / 2.0 ** 24


def _circ(u, f):
    d = (u - f).abs()
    return torch.minimum(d, 1.0 - d)


def dither_model(v, scale, s, partition, u):
    """float64 levels (non-negative index q) of v / scale with draws u, and where the model is ambiguous within
    the fp32 rounding of t."""
    a = v.double().abs() / scale if scale > 0 else torch.zeros_like(v, dtype=torch.float64)
    if partition == 0:
        t = a * s
        fl = t.floor()
        frac = t - fl
        q = fl + (u < frac).double()
        amb = _circ(u, frac) <= 8 * U * torch.clamp(t, min=1.0)
    else:
        t = a * 2.0 ** (s - 1)
        small = t < 1.0
        lo_idx = torch.floor(torch.log2(torch.clamp(t, min=1.0)))
        lo = torch.exp2(lo_idx)
        frac = torch.where(small, t, (t - lo) / lo)
        q = torch.where(small, (u < t).double(), lo_idx + 1 + (u < frac).double())
        near = t.clamp(min=1e-300)
        pow2 = torch.exp2(torch.round(torch.log2(near)))
        amb = (_circ(u, frac) <= 16 * U) | ((near / pow2 - 1.0).abs() <= 64 * U)
        q = torch.where(t <= 0, torch.zeros_like(q), q)
    return q.clamp(max=s), amb


def level_value(q, s, partition):
    q = q.double()
    if partition == 0:
        return q / s
    return torch.where(q == 0, torch.zeros_like(q), torch.exp2(q - 1) / 2.0 ** (s - 1))


DITHER_OPTS = [  # (mom, ef, partition, normalize, levels, two-stage)
    (False, False, 0, 0, 8, False),
    (True, True, 1, 1, 6, True),
    (False, True, 0, 1, 127 // 2, True),
    (True, False, 1, 0, 3, False),
    (True, True, 0, 0, 4, True),
    (False, False, 1, 1, 8, False),
]
DITHER_CASES = _cases(len(DITHER_OPTS))


def check_levels(lv, x, scale, s, partition, seed, step, what):
    n = x.numel()
    u = splitmix_uniform(seed, step, torch.arange(n, device="cuda", dtype=torch.int64))
    q, amb = dither_model(x, scale, s, partition, u)
    want = torch.where(x < 0, -q, q)
    got = lv.double()
    mism = got != want
    bad = mism & ~amb
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: %d levels differ from the model, first at %d: got %d, want %d (x %r, u %r)" % (
            what, int(bad.sum()), i, int(got[i]), int(want[i]), x[i].item(), u[i].item()))
    accepted = int((mism & amb).sum())
    assert accepted <= 1e-4 * n, "%s: %d ambiguous levels accepted" % (what, accepted)
    return accepted


@pytest.mark.gpu
@pytest.mark.parametrize("n,dt,opt", DITHER_CASES, ids=_ids(DITHER_CASES))
def test_dithering_kernels(n, dt, opt):
    cu, d = _cu(), DT[dt]
    use_mom, use_ef, partition, normalize, s_lv, two = DITHER_OPTS[opt]
    mu, ratio = 0.9, (2.0 if opt % 2 else 0.25)
    seed, step = 12345 + opt, 3
    st = torch.cuda.current_stream().cuda_stream
    lv_bytes = (n + 15) // 16 * 16
    slot = (lv_bytes + 16 + 255) // 256 * 256
    slots = torch.zeros(P * slot, dtype=torch.uint8, device="cuda")
    acc = torch.zeros(4 + 3 * 132 * 8, device="cuda")
    grid = max(1, min(1056, -(-n // 1024)))
    depth = sum_depth(n, 1, grid)
    worst, accepted = {}, 0
    for r in range(P):
        g = make_grad(n, d, 5 * n + r)
        g0 = g.clone()
        mom = make_state(n, 71 + r) if use_mom else None
        err = make_state(n, 81 + r) if use_ef else None
        p64, pb, m64, mb = corrected_ref(g, mom, mu, err, ratio)
        cor = torch.empty(n, device="cuda")
        cu.ef_correct(g.data_ptr(), _code(d), mom.data_ptr() if use_mom else 0, mu, err.data_ptr() if use_ef else 0,
                      ratio, cor.data_ptr(), n, acc.data_ptr(), st)
        torch.cuda.synchronize()
        what = "ef_correct %s n=%d rank %d" % (dt, n, r)
        assert torch.equal(bits(g), bits(g0)), what + ": the gradient changed"
        worst["p"] = max(worst.get("p", 0), check(cor, p64, pb, what + " p"))
        if use_mom:
            worst["mom"] = max(worst.get("mom", 0), check(mom, m64, mb, what + " momentum"))
        c64 = cor.double()
        assert acc[2].item() == cor.abs().max().item(), what + ": max |p|"
        sa, sq = c64.abs().sum(), (c64 * c64).sum()
        worst["sum|p|"] = max(worst.get("sum|p|", 0), check(acc[0:1], sa.reshape(1), (depth * U * sa + TINY).reshape(1),
                                                            what + " sum |p|"))
        worst["sum p^2"] = max(worst.get("sum p^2", 0), check(acc[1:2], sq.reshape(1),
                                                              ((depth + 1) * U * sq + TINY).reshape(1), what + " sum p^2"))
        pay = slots[r * slot: r * slot + lv_bytes]
        sc_t = slots[r * slot + lv_bytes: r * slot + lv_bytes + 4].view(F32)
        err_out = err if use_ef else torch.empty(n, device="cuda")
        cu.dither_quantize(cor.data_ptr(), n, acc.data_ptr(), s_lv, partition, normalize, seed, step, pay.data_ptr(),
                           sc_t.data_ptr(), err_out.data_ptr(), st)
        torch.cuda.synchronize()
        sc = sc_t.item()
        want_sc = acc[2].item() if normalize == 0 else torch.sqrt(acc[1:2]).item()
        assert sc == want_sc, what + ": scale %r, want %r" % (sc, want_sc)
        lv = pay[:n].view(torch.int8)
        accepted += check_levels(lv, cor, sc, s_lv, partition, seed, step, what)
        vl = level_value(lv.abs(), s_lv, partition) * sc
        e_err = c64 - torch.where(lv < 0, -vl, vl)
        worst["err"] = max(worst.get("err", 0), check(err_out, e_err, 3 * U * (c64.abs() + vl) + 3 * TINY,
                                                      what + " error"))
    what = "dithering consumer %s n=%d" % (dt, n)
    sm = torch.empty(n, device="cuda")
    cu.dither_sum_slots(slots.data_ptr(), slot, P, n, s_lv, partition, sm.data_ptr(), st)
    torch.cuda.synchronize()
    e, a = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    for r in range(P):
        lv = slots[r * slot: r * slot + n].view(torch.int8)
        sc = slots[r * slot + lv_bytes: r * slot + lv_bytes + 4].view(F32).item()
        v = level_value(lv.abs(), s_lv, partition) * sc
        e += torch.where(lv < 0, -v, v)
        a += v
    worst["sum"] = check(sm, e, (P + 1) * U * a + P * TINY, what + " slot sum")
    m = f32(MULT)
    out = torch.empty(n, dtype=d, device="cuda")
    if two:
        lv2 = torch.empty(lv_bytes, dtype=torch.int8, device="cuda")
        sc2 = torch.empty(4, device="cuda")
        cor = torch.empty(n, device="cuda")
        cu.ef_correct(sm.data_ptr(), 0, 0, 0.0, 0, 1.0, cor.data_ptr(), n, acc.data_ptr(), st)
        cu.dither_quantize(cor.data_ptr(), n, acc.data_ptr(), s_lv, partition, normalize, seed ^ 0x5555, step,
                           lv2.data_ptr(), sc2.data_ptr(), 0, st)
        cu.dither_unpack(lv2.data_ptr(), sc2.data_ptr(), n, s_lv, partition, out.data_ptr(), _code(d), MULT, st)
        torch.cuda.synchronize()
        assert torch.equal(cor, sm), what + ": correction without state must copy"
        accepted += check_levels(lv2[:n], cor, sc2[0].item(), s_lv, partition, seed ^ 0x5555, step, what)
        v = level_value(lv2[:n].abs(), s_lv, partition) * sc2[0].item() * m
        e_out = torch.where(lv2[:n] < 0, -v, v)
        worst["out"] = check(out, e_out, 3 * U * e_out.abs() + TINY, what + " unpack", d)
    else:
        cu.cast_scale(sm.data_ptr(), n, out.data_ptr(), _code(d), MULT, st)
        torch.cuda.synchronize()
        e_out = m * sm.double()
        worst["out"] = check(out, e_out, U * e_out.abs() + TINY, what + " cast", d)
    for key, v in worst.items():
        report("dithering", "%s %s n=%d opt %d" % (key, dt, n, opt), v)
    print("compress-numerics: dithering %s n=%d opt %d: %d ambiguous levels accepted" % (dt, n, opt, accepted))


# ------------------------------------------------------------------------------------------------ pipeline
class _RankCtx:
    """SymmContext look-alike for one virtual rank."""

    def __init__(self, vc, r):
        self.cu, self.device, self.world, self.rank = vc.cu, vc.device, vc.world, r
        self.view, self.arena, self.data_bytes = vc.views[r], vc.arenas[r], vc.data_bytes


def _run_lockstep(vc, comps, grads, outs, average):
    """Issue every pipeline phase for ALL virtual ranks before the next phase (see GpuCompressor.phases)."""
    cur = torch.cuda.current_stream()
    for st in vc.streams:
        st.wait_stream(cur)
    plans = []
    for r, c in enumerate(comps):
        with torch.cuda.stream(vc.streams[r]):
            plans.append(c.phases(grads[r], outs[r], average, vc.streams[r].cuda_stream))
    for i in range(len(plans[0])):
        for r in range(len(comps)):
            with torch.cuda.stream(vc.streams[r]):
                plans[r][i]()
    for st in vc.streams:
        cur.wait_stream(st)


# per compressor: (two_stage, average, ef, nesterov, kind-specific kwargs); every option is on and off somewhere
PIPE_OPTS = {
    "onebit": [(True, True, True, False, {"compressor_onebit_scaling": "true"}),
               (False, False, False, True, {}),
               (True, False, False, True, {"compressor_onebit_scaling": "true"}),
               (False, True, True, True, {})],
    "topk": [(True, True, True, False, {"compressor_k": "0.01"}),
             (False, False, False, True, {"compressor_k": "37"}),
             (True, False, False, True, {"compressor_k": "0.2"}),
             (False, True, True, True, {"compressor_k": "0.01"})],
    "randomk": [(True, True, True, False, {"compressor_k": "0.2", "seed": "17"}),
                (False, False, False, True, {"compressor_k": "37", "seed": "5"}),
                (True, False, False, True, {"compressor_k": "0.01"}),
                (False, True, True, True, {"compressor_k": "0.2", "seed": "9"})],
    "dithering": [(True, True, True, False, {"compressor_k": "8", "dithering_partition": "0",
                                             "dithering_normalize": "0"}),
                  (False, False, False, True, {"compressor_k": "4", "dithering_partition": "1",
                                               "dithering_normalize": "1"}),
                  (True, False, False, True, {"compressor_k": "6", "dithering_partition": "0",
                                              "dithering_normalize": "1"}),
                  (False, True, True, True, {"compressor_k": "3", "dithering_partition": "1",
                                             "dithering_normalize": "0"})],
}
LRS = [1.0, 0.5, 0.5, 2.0]          # ratio lr_prev / lr = 1, 2, 1, 0.25
PIPE_CASES = [(kind, i) for kind in PIPE_OPTS for i in range(len(PIPE_OPTS[kind]))]
WORLDS = [1, 2, 3, 5, 8]


def _kwargs(kind, opt):
    two, avg, ef, nest, extra = PIPE_OPTS[kind][opt]
    kw = {"compressor_type": kind}
    kw.update(extra)
    if ef:
        kw["ef_type"] = "vanilla"
    if nest:
        kw["momentum_type"] = "nesterov"
        kw["momentum_mu"] = "0.9"
    return kw, two, avg


def _pipe_n(world):
    return 4099 + 37 * world


def _make_comps(vc, kind, opt, dt, n):
    from byteps_b200.ops.compress import GpuCompressor

    kw, two, _ = _kwargs(kind, opt)
    return [GpuCompressor(_RankCtx(vc, r), kw, n, dt, payload_off=GUARD, two_stage=two) for r in range(vc.world)]


@pytest.fixture(scope="module")
def warm_pipeline():
    """Every pipeline configuration once on a single rank, so that no kernel module loads while ranks spin."""
    from byteps_b200.comm.symm import VirtualCluster

    for kind, opt in PIPE_CASES:
        for dt in DTYPES:
            n = _pipe_n(1)
            vc = VirtualCluster(1, "cuda:0", 1 << 22)
            comps = _make_comps(vc, kind, opt, DT[dt], n)
            _, _, avg = _kwargs(kind, opt)
            g = make_grad(n, DT[dt], 1)
            _run_lockstep(vc, comps, [g], [torch.empty_like(g)], avg)
    torch.cuda.synchronize()


def _snap(c):
    keep = {}
    for name in ("mom", "err", "err2", "rng_state", "rng_state2"):
        t = getattr(c, name, None)
        keep[name] = t.clone() if t is not None else None
    return keep


def _slots(c, vc, step):
    """This step's payload slots as read from rank 0's window (every rank's payload has landed there)."""
    off = c.off + (step & 1) * vc.world * c.slot_bytes
    return [vc.arenas[0][off + p * c.slot_bytes: off + (p + 1) * c.slot_bytes] for p in range(vc.world)]


def _pipe_check(kind, comps, snaps, grads, outs, slots, ratio, mult, n, dt, world, what):
    """One step deep: producer state and payload of every rank, then the consumer from the payloads."""
    c0 = comps[0]
    mu = c0.mu or 0.0
    worst = {}

    def upd(key, v):
        worst[key] = max(worst.get(key, 0.0), v)

    p64s, pbs = [], []
    for r, c in enumerate(comps):
        sn = snaps[r]
        p64, pb, m64, mb = corrected_ref(grads[r], sn["mom"], mu, sn["err"], ratio)
        p64s.append(p64)
        pbs.append(pb)
        if sn["mom"] is not None:
            upd("mom", check(c.mom, m64, mb, "%s rank %d momentum" % (what, r)))
    m = f32(mult)
    if kind == "onebit":
        nwords = (n + 31) // 32
        negs = [decode_signs(sl.view(torch.int32)[:nwords], n) for sl in slots]
        scs = [sl[nwords * 4: nwords * 4 + 4].view(F32).item() for sl in slots]
        for r, c in enumerate(comps):
            check_signs(negs[r], None, p64s[r], pbs[r], "%s rank %d signs" % (what, r))
            if c0.scaled:
                check_mean_abs(scs[r], p64s[r], n, sum_depth(n, 4, grid_fused((n + 127) // 128 * 32)) + 1,
                               "%s rank %d scale" % (what, r), pbs[r].sum().item())
            if c.err is not None:
                sgn = torch.where(negs[r], -1.0, 1.0).double()
                upd("err", check(c.err, p64s[r] - sgn * scs[r], pbs[r] + U * (p64s[r].abs() + scs[r]) + TINY,
                                 "%s rank %d error" % (what, r)))
        e_sum = sum(torch.where(negs[r], -scs[r], scs[r]).double() for r in range(world))
        a_sum = sum(scs)
        if c0.two_stage:
            e2 = snaps[0]["err2"]
            e_c2 = e_sum + (e2.double() if e2 is not None else 0)
            b_c2 = world * U * (a_sum + (e2.double().abs() if e2 is not None else torch.zeros_like(e_c2))) + world * TINY
            sc2 = c0.scale2[0].item()
            if c0.scaled:
                check_mean_abs(sc2, e_c2, n, sum_depth(n, 4, grid_fused((n + 127) // 128 * 32)) + 1,
                               what + " scale2", b_c2.sum().item())
            sure = e_c2.abs() > b_c2
            o = outs[0].double()
            e_out = torch.where(e_c2 < 0, -m * sc2, m * sc2)
            upd("out", check(o.abs(), e_out.abs(), U * e_out.abs() + TINY, what + " out", dt))
            assert ((o < 0) == (e_c2 < 0))[sure].all(), what + ": output sign"
            if e2 is not None:
                d_ = torch.where(o < 0, -sc2, sc2)
                upd("err2", check(comps[0].err2, e_c2 - d_, b_c2 + U * (e_c2.abs() + sc2) + TINY, what + " err2"))
        else:
            upd("out", check(outs[0], m * e_sum, (world + 1) * U * m * a_sum + TINY, what + " out", dt))
    elif kind == "topk":
        k = c0.k
        e = torch.zeros(n, dtype=torch.float64, device="cuda")
        a = torch.zeros_like(e)
        for r, (c, sl) in enumerate(zip(comps, slots)):
            pr = sl.view(torch.int32)[:2 * k]
            i, v = pr[0::2].long(), pr[1::2].view(F32).double()
            assert i.unique().numel() == k, "%s rank %d: indices not unique" % (what, r)
            upd("vals", check(v, p64s[r][i], pbs[r][i], "%s rank %d payload" % (what, r)))
            if c.err is not None:
                kept = torch.zeros(n, dtype=torch.bool, device="cuda")
                kept[i] = True
                assert (bits(c.err)[kept] == 0).all(), "%s rank %d: kept error not zeroed" % (what, r)
                upd("err", check(c.err[~kept], p64s[r][~kept], pbs[r][~kept], "%s rank %d error" % (what, r)))
            e.index_add_(0, i, v)
            a.index_add_(0, i, v.abs())
        e2 = snaps[0]["err2"]
        if e2 is not None:
            e += e2.double()
            a += e2.double().abs()
        b = world * U * a + world * TINY
        o = outs[0].double()
        if c0.two_stage:
            sup = o != 0
            assert int(sup.sum()) <= k, what + ": more than k outputs"
            upd("out", check(outs[0][sup], m * e[sup], m * b[sup] + U * m * e[sup].abs() + TINY, what + " out", dt))
            if e2 is not None:
                z = comps[0].err2
                assert (bits(z)[sup] == 0).all(), what + ": kept err2 not zeroed"
                upd("err2", check(z[~sup], e[~sup], b[~sup], what + " err2"))
        else:
            upd("out", check(outs[0], m * e, m * b + U * m * e.abs() + TINY, what + " out", dt))
    elif kind == "randomk":
        from byteps_b200 import _native

        k = c0.k
        core = _native.core()
        seed = (int(c0.kw.get("seed", "0")) or 0x9E3779B97F4A7C15) & M64
        rng = core.XorShift128Plus()
        st0 = snaps[0]["rng_state"].tolist()
        want = None
        for r, c in enumerate(comps):
            assert snaps[r]["rng_state"].tolist() == st0, what + ": ranks' streams diverged"
        # the stream continues from the state before the step: the CPU generator replays it from the seed
        rng.set_seed(seed)
        drawn_before = (c0.step - 1) * k
        if drawn_before:
            cpu_stream(rng, drawn_before, n)
        want = cpu_stream(rng, k, n)
        assert torch.equal(c0.idx.long(), want), what + ": indices differ from the CPU stream"
        drawn = torch.zeros(n, dtype=torch.bool, device="cuda")
        drawn[want] = True
        vsum = 0
        vabs = 0
        for r, (c, sl) in enumerate(zip(comps, slots)):
            v = sl.view(F32)[:k].double()
            upd("vals", check(v, p64s[r][want], pbs[r][want], "%s rank %d payload" % (what, r)))
            if c.err is not None:
                assert (bits(c.err)[drawn] == 0).all(), "%s rank %d: drawn error not zeroed" % (what, r)
                upd("err", check(c.err[~drawn], p64s[r][~drawn], pbs[r][~drawn], "%s rank %d error" % (what, r)))
            vsum = vsum + v
            vabs = vabs + v.abs()
        last = last_occurrence(want, n)
        hit = last >= 0
        e = torch.zeros(n, dtype=torch.float64, device="cuda")
        a = torch.zeros_like(e)
        e[hit] = vsum[last[hit]]
        a[hit] = vabs[last[hit]]
        b = (world - 1) * U * a + TINY
        if c0.two_stage:
            assert torch.equal(c0.idx2.long(), want), what + ": second-stage indices"
            e2 = snaps[0]["err2"]
            if e2 is not None:
                b = b + U * (a + e2.double().abs())
                e = e + e2.double()
                a = a + e2.double().abs()
                z = comps[0].err2
                assert (bits(z)[drawn] == 0).all(), what + ": drawn err2 not zeroed"
                upd("err2", check(z[~drawn], e[~drawn], b[~drawn], what + " err2"))
            e = torch.where(drawn, e, torch.zeros_like(e))
        upd("out", check(outs[0], m * e, m * b + U * m * e.abs() + TINY, what + " out", dt))
    else:
        lvb = c0.lv_bytes
        e = torch.zeros(n, dtype=torch.float64, device="cuda")
        a = torch.zeros_like(e)
        for r, (c, sl) in enumerate(zip(comps, slots)):
            lv = sl[:n].view(torch.int8)
            sc = sl[lvb:lvb + 4].view(F32).item()
            v = level_value(lv.abs(), c.s, c.partition) * sc
            if c.err is not None:
                upd("err", check(c.err, p64s[r] - torch.where(lv < 0, -v, v),
                                 pbs[r] + 3 * U * (p64s[r].abs() + v) + 3 * TINY, "%s rank %d error" % (what, r)))
            e += torch.where(lv < 0, -v, v)
            a += v
        upd("sum", check(c0.sum, e, (world + 1) * U * a + world * TINY, what + " slot sum"))
        if c0.two_stage:
            lv2 = c0.levels2[:n]
            sc2 = c0.scale2[0].item()
            v = level_value(lv2.abs(), c0.s, c0.partition) * sc2 * m
            e_out = torch.where(lv2 < 0, -v, v)
            upd("out", check(outs[0], e_out, 3 * U * e_out.abs() + TINY, what + " out", dt))
        else:
            e_out = m * c0.sum.double()
            upd("out", check(outs[0], e_out, U * e_out.abs() + TINY, what + " out", dt))
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("kind,opt", PIPE_CASES, ids=["%s-%d" % c for c in PIPE_CASES])
def test_pipeline(kind, opt, dt, world, warm_pipeline):
    """Four steps of GpuCompressor on `world` virtual ranks with the lr changing between steps; the gradients
    stay untouched (outputs are separate tensors), nothing outside the payload window changes, every rank's
    output is the same bits, and every step matches the reference started from the state before it."""
    from byteps_b200.comm.symm import VirtualCluster

    d = DT[dt]
    n = _pipe_n(world)
    kw, two, avg = _kwargs(kind, opt)
    from byteps_b200.ops.compress import GpuCompressor

    pay = GpuCompressor.payload_bytes_for(kw, n, world)
    end = GUARD + pay + GUARD
    vc = VirtualCluster(world, "cuda:0", end)
    from test_gpu_exchange_numerics import check_unchanged, sentinel

    for r in range(world):
        vc.arenas[r][:end].copy_(sentinel(end, 40 + r))
    bands = [vc.arenas[r][:end].clone() for r in range(world)]
    comps = _make_comps(vc, kind, opt, d, n)
    assert world * comps[0].blocks <= 64
    mult = 1.0 / world if avg else 1.0
    worst = {}
    for step, lr in enumerate(LRS, 1):
        for c in comps:
            c.set_lr(lr)
        ratio = comps[0].lr_prev / comps[0].lr_cur
        grads = [make_grad(n, d, 1000 * step + r) for r in range(world)]
        g0 = [g.clone() for g in grads]
        outs = [torch.full((n,), 3.0, dtype=d, device="cuda") for _ in range(world)]
        snaps = [_snap(c) for c in comps]
        torch.cuda.synchronize()
        _run_lockstep(vc, comps, grads, outs, avg)
        torch.cuda.synchronize()
        what = "%s opt %d %s world %d step %d" % (kind, opt, dt, world, step)
        for r in range(world):
            assert torch.equal(bits(grads[r]), bits(g0[r])), "%s rank %d: the gradient changed" % (what, r)
            assert torch.equal(bits(outs[r]), bits(outs[0])), "%s: rank %d output differs from rank 0" % (what, r)
            check_unchanged(vc.arenas[r][:end], bands[r], [(GUARD, GUARD + pay)], "%s rank %d" % (what, r))
            if comps[r].err2 is not None:
                assert torch.equal(bits(comps[r].err2), bits(comps[0].err2)), what + ": server states differ"
        for key, v in _pipe_check(kind, comps, snaps, grads, outs, _slots(comps[0], vc, step), ratio, mult, n, d,
                                  world, what).items():
            worst[key] = max(worst.get(key, 0.0), v)
    for key, v in worst.items():
        report(kind, "pipeline %s %s opt %d world %d" % (key, dt, opt, world), v)


# ------------------------------------------------------------------------------------------------ CPU self-test
def test_bounds_reject_wrong_models():
    """On the CPU: the bounds accept the kernels' arithmetic and reject an fp32 sum done in bf16, a dropped lr
    ratio, a sign taken with <= 0 and momentum rounded to the gradient dtype; the splitmix64 reproduction and the
    dithering level model agree with direct evaluation."""
    torch.manual_seed(0)
    n = 1 << 14
    g = (torch.randn(n) * 4).to(BF16)
    mom, err = torch.randn(n), torch.randn(n)
    g[:2], mom[:2], err[:2] = 0.0, 0.0, 0.0
    mu, ratio = 0.9, 2.0
    p64, pb, m64, mb = corrected_ref(g, mom, mu, err, ratio)
    # the fp32 arithmetic of corrected4, without FMA contraction
    gf = g.float()
    m32 = torch.tensor(mu, dtype=F32) * mom + gf
    p32 = gf + torch.tensor(mu, dtype=F32) * m32 + torch.tensor(ratio, dtype=F32) * err
    assert not (((p32.double() - p64).abs() > pb).any()), "fp32 model rejected"
    assert not (((m32.double() - m64).abs() > mb).any()), "fp32 momentum rejected"
    # momentum rounded to the gradient dtype (the old dithering path)
    pr = (gf + torch.tensor(mu, dtype=F32) * m32).to(BF16).float() + torch.tensor(ratio, dtype=F32) * err
    assert ((pr.double() - p64).abs() > pb).any(), "bound accepts momentum rounded to bf16"
    # lr ratio dropped
    pn = gf + torch.tensor(mu, dtype=F32) * m32 + err
    assert ((pn.double() - p64).abs() > pb).any(), "bound accepts a dropped lr ratio"
    # signs: <= 0 sets the bit of +0.0
    neg_right = p32 < 0
    check_signs(neg_right, p32, p64, pb, "fp32 model")
    with pytest.raises(AssertionError):
        check_signs(p32 <= 0, p32, p64, pb, "<= 0 model")
    # a slot sum done in bf16 instead of fp32
    P_ = 3
    xs = [torch.randn(n) for _ in range(P_)]
    e = sum(x.double() for x in xs)
    a = sum(x.double().abs() for x in xs)
    s32 = xs[0] + xs[1] + xs[2]
    s16 = ((xs[0].to(BF16) + xs[1].to(BF16)).float() + xs[2]).float()
    b = P_ * U * a + P_ * TINY
    check(s32, e, b, "fp32 sum")
    with pytest.raises(AssertionError):
        check(s16, e, b, "bf16 sum")
    # one rounding to the user dtype after the fp32 scale, and not two
    m = f32(1.0 / 3.0)
    check((s32 * m).to(BF16), m * s32.double(), U * m * s32.double().abs() + TINY, "one rounding", BF16)
    with pytest.raises(AssertionError):
        twice = (s32.to(BF16).float() * m).to(BF16)
        check(twice, m * s32.double(), U * m * s32.double().abs() + TINY, "two roundings", BF16)
    # splitmix64 reproduction against Python integers, including a step and an index past 2^32
    for seed, step in ((12345, 3), (0xFFFFFFFFFFFFFFFF, 1 << 40), (0, 0)):
        idx = torch.tensor([0, 1, 2, 77, (1 << 32) + 5, 31_254_527], dtype=torch.int64)
        got = splitmix_uniform(seed, step, idx)
        want = [splitmix_uniform_int(seed, step, int(i)) for i in idx]
        assert got.tolist() == want
    # the level model against direct evaluation
    for partition in (0, 1):
        s_lv = 5
        x = torch.tensor([0.0, -0.3, 0.51, 1.0, -0.07, 0.9999], dtype=F32)
        u = torch.tensor([0.5, 0.2, 0.9, 0.1, 0.3, 0.99], dtype=torch.float64)
        q, amb = dither_model(x, 1.0, s_lv, partition, u)
        for xi, ui, qi in zip(x.tolist(), u.tolist(), q.tolist()):
            t = abs(xi) * (s_lv if partition == 0 else 2 ** (s_lv - 1))
            if partition == 0:
                want = math.floor(t) + (ui < t - math.floor(t))
            elif t == 0:
                want = 0
            elif t < 1:
                want = int(ui < t)
            else:
                lo = 2 ** math.floor(math.log2(t))
                want = math.floor(math.log2(t)) + 1 + (ui < (t - lo) / lo)
            assert qi == min(want, s_lv), (partition, xi, ui, qi, want)
