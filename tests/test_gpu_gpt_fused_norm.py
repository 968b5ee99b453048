"""GPT-2-style decoder with fused_norm (models/gpt.py) on the GPU: graphed bf16 gpt_tiny steps with fused AdamW,
with fused_norm alone and with every flag, track the stock model on padded batches and packed streams; the fused
packed step runs without a host synchronisation (checked inside test_gpu_gpt's step script whenever a flag is on);
and 300 packed steps at dropout 0.1 with every flag on stay next to the stock loss curve."""
import numpy as np
import pytest
import torch

from test_gpu_gpt import _run

FLAG_SETS = {"norm": dict(fused_norm=True),
             "all": dict(fused_attention=True, fused_loss=True, fp8_linear=True, fused_norm=True)}


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["padded", "packed"])
@pytest.mark.parametrize("flags", list(FLAG_SETS), ids=list(FLAG_SETS))
def test_gpt_tiny_fused_norm_graphed_steps_track_stock(tmp_path, flags, packed):
    """bf16, dropout 0, one CUDA graph per step: the losses track the stock model's within 1 %."""
    s = _run(tmp_path, "stock", {}, packed, 0.0, 8)
    f = _run(tmp_path, flags, FLAG_SETS[flags], packed, 0.0, 8)
    for a, c in zip(s["losses"], f["losses"]):
        assert abs(a - c) <= 1e-2 * abs(a), (s["losses"], f["losses"])
    assert f["losses"][-1] < f["losses"][0]
    assert all(torch.isfinite(p).all() for p in f["params"].values())


@pytest.mark.gpu
def test_gpt_tiny_fused_norm_dropout_loss_curve_tracks_stock(tmp_path):
    """300 graphed packed steps at dropout 0.1 with every flag on, fused_norm included: the loss falls, and the
    means of the last 50 steps are within 2 % of the stock model's."""
    s = _run(tmp_path, "stock", {}, True, 0.1, 300)
    f = _run(tmp_path, "all", FLAG_SETS["all"], True, 0.1, 300)
    ls, lf = np.array(s["losses"]), np.array(f["losses"])
    assert np.isfinite(lf).all()
    assert lf[-50:].mean() < lf[:10].mean() * 0.9
    assert abs(lf[-50:].mean() - ls[-50:].mean()) <= 0.02 * ls[-50:].mean(), (ls[-50:].mean(), lf[-50:].mean())
