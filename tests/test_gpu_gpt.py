"""GPT-2-style decoder (models/gpt.py) on the GPU: graphed bf16 gpt_tiny steps with fused AdamW, with the causal
fused attention alone and together with the fused loss and FP8 linears, track the stock model (SDPA with the causal
mask, F.cross_entropy, nn.Linear) on padded batches and packed streams; the packed step runs without a host
synchronisation; and 300 steps at dropout 0.1 stay next to the stock loss curve."""
import numpy as np
import pytest
import torch

from test_gpu_attn import _run_py

_GPT_STEPS = """
import torch
import byteps_b200.torch as bps
from byteps_b200.models import gpt_tiny
from byteps_b200.torch.graph import GraphedStep
FLAGS, PACKED, DROPOUT, STEPS, OUT = %r, %r, %r, %r, %r
bps.init()
torch.manual_seed(0)
model = gpt_tiny(dropout=DROPOUT, **FLAGS).cuda().to(torch.bfloat16).train()
opt = bps.DistributedOptimizer(torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=0.01),
                               named_parameters=model.named_parameters(), fused_update=True)
g = torch.Generator().manual_seed(1)
b, s = 8, 256
# a learnable stream: each sequence counts up from a random start modulo 1000
lengths = torch.randint(16, s + 1, (b,), generator=g)
start = torch.randint(0, 1000, (b, 1), generator=g)
ids = (start + torch.arange(s)[None, :]) %% 1000
attend = torch.arange(s)[None, :] < lengths[:, None]
labels = torch.where(attend, ids, torch.full_like(ids, -100)).cuda()
ids = ids.cuda()
cu = [0]
for n in lengths.tolist():
    cu += [cu[-1] + n, cu[-1] + s]
cu = torch.tensor(cu, dtype=torch.int32).cuda()
calls = [0]

def step():
    opt.zero_grad()
    # the second eager warm-up step reports any host synchronisation of the fused packed step as an error
    check = PACKED and FLAGS and calls[0] == 1
    calls[0] += 1
    if check:
        torch.cuda.set_sync_debug_mode("error")
    if PACKED:
        # padding runs are sequences of their own, whose targets are all -100
        loss = model(ids, labels, cu_seqlens=cu, max_seqlen=s)
    else:
        loss = model(ids, labels)
    loss.backward()
    if check:
        torch.cuda.set_sync_debug_mode(0)
    opt.step()
    return loss

stepper = GraphedStep(step, warmup=2, pre_replay=opt.refresh_hparams)
losses = [stepper().detach().float().item() for _ in range(STEPS)]
torch.save({"losses": losses, "params": {n: p.detach().float().cpu() for n, p in model.named_parameters()}}, OUT)
print("OK")
bps.shutdown()
"""

FLAG_SETS = {"attn": dict(fused_attention=True),
             "attn_loss_fp8": dict(fused_attention=True, fused_loss=True, fp8_linear=True)}


def _run(tmp_path, name, flags, packed, dropout, steps):
    out = str(tmp_path / ("%s_%d.pt" % (name, packed)))
    assert "OK" in _run_py(_GPT_STEPS % (flags, packed, dropout, steps, out))
    return torch.load(out)


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
@pytest.mark.parametrize("flags", list(FLAG_SETS), ids=list(FLAG_SETS))
def test_gpt_tiny_graphed_steps_track_stock(tmp_path, flags, packed):
    """bf16, dropout 0, one CUDA graph per step: the losses track the stock model's within 1 %."""
    s = _run(tmp_path, "stock", {}, packed, 0.0, 8)
    f = _run(tmp_path, flags, FLAG_SETS[flags], packed, 0.0, 8)
    for a, c in zip(s["losses"], f["losses"]):
        assert abs(a - c) <= 1e-2 * abs(a), (s["losses"], f["losses"])
    assert f["losses"][-1] < f["losses"][0]
    assert all(torch.isfinite(p).all() for p in f["params"].values())


@pytest.mark.gpu
def test_gpt_tiny_dropout_loss_curve_tracks_stock(tmp_path):
    """300 graphed packed steps at dropout 0.1 with every flag on: the loss falls, and the means of the last 50
    steps are within 2 % of the stock model's."""
    s = _run(tmp_path, "stock", {}, True, 0.1, 300)
    f = _run(tmp_path, "all", FLAG_SETS["attn_loss_fp8"], True, 0.1, 300)
    ls, lf = np.array(s["losses"]), np.array(f["losses"])
    assert np.isfinite(lf).all()
    assert lf[-50:].mean() < lf[:10].mean() * 0.9
    assert abs(lf[-50:].mean() - ls[-50:].mean()) <= 0.02 * ls[-50:].mean(), (ls[-50:].mean(), lf[-50:].mean())
