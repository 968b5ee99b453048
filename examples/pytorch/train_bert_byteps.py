#!/usr/bin/env python
"""BERT-large pre-training step loop (the reference's bandwidth-bound headline
workload) with the fused AdamW or LAMB exchange: bf16 parameters/gradients, fp32
master weights and moments sharded over the GPUs, updated inside the exchange."""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))
import byteps_b200.torch as bps  # noqa: E402
from byteps_b200.models import get_model  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--model", default="bert_large")
p.add_argument("--batch-size", type=int, default=16)
p.add_argument("--seq-len", type=int, default=128)
p.add_argument("--steps", type=int, default=20)
p.add_argument("--warmup-steps", type=int, default=5)
p.add_argument("--no-cuda", action="store_true", help="CPU run over gloo (unfused optimizer, fp32)")
p.add_argument("--fused-norm", action="store_true",
               help="fused dropout + residual add + LayerNorm kernels at the encoder layers' junctions")
p.add_argument("--fused-attention", action="store_true",
               help="fused self-attention kernels reading Q, K and V in place from the qkv projection")
p.add_argument("--fused-loss", action="store_true",
               help="fused softmax cross-entropy kernels for the masked-LM loss")
p.add_argument("--fp8-linear", action="store_true",
               help="FP8 GEMMs with delayed scaling for the encoder layers' linear layers (sm_90)")
p.add_argument("--optimizer", choices=("adamw", "lamb"), default="adamw",
               help="lamb: weights with decay and the trust ratio; biases and LayerNorm weights without either")
p.add_argument("--max-grad-norm", type=float, default=None,
               help="clip the averaged gradients by their global 2-norm before every update (BERT recipes use 1.0)")
p.add_argument("--max-predictions-per-seq", type=int, default=None,
               help="label 15 %% of the positions and run the masked-LM head on at most this many per sequence "
                    "(BERT recipes use 20 at 128 tokens, 80 at 512)")
args = p.parse_args()
bps.init()
cuda = torch.cuda.is_available() and not args.no_cuda
if cuda:
    torch.cuda.set_device(bps.local_rank())
dev = torch.device("cuda", bps.local_rank()) if cuda else torch.device("cpu")
model = get_model(args.model, fused_norm=args.fused_norm, fused_loss=args.fused_loss,
                  fp8_linear=args.fp8_linear, fused_attention=args.fused_attention,
                  max_predictions_per_seq=args.max_predictions_per_seq or 0).to(dev)
if cuda:
    model = model.to(torch.bfloat16)
if args.optimizer == "lamb":
    # the usual BERT split: 1-D parameters (biases, LayerNorm weights) take neither decay nor adaptation
    decay = [p for p in model.parameters() if p.dim() > 1]
    plain = [p for p in model.parameters() if p.dim() <= 1]
    inner = bps.Lamb([dict(params=decay, weight_decay=0.01),
                      dict(params=plain, weight_decay=0.0, adapt=False)], lr=1e-3)
else:
    inner = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01)
opt = bps.DistributedOptimizer(inner, named_parameters=model.named_parameters(), fused_update=cuda,
                               max_grad_norm=args.max_grad_norm)
bps.broadcast_parameters(model.state_dict(), root_rank=0)
ids = torch.randint(0, 30522, (args.batch_size, args.seq_len), device=dev)
labels = torch.randint(0, 30522, (args.batch_size, args.seq_len), device=dev)
if args.max_predictions_per_seq:
    labels[torch.rand(labels.shape, device=dev) >= 0.15] = -100


def sync():
    if cuda:
        torch.cuda.synchronize()


for i in range(args.steps + args.warmup_steps):
    if i == args.warmup_steps:
        sync()
        t0 = time.time()
    opt.zero_grad()
    loss = model(ids, mlm_labels=labels)
    loss.backward()
    opt.step()
sync()
if bps.rank() == 0:
    dt = time.time() - t0
    print("tokens/sec on %d %s(s): %.0f (loss %.3f)" % (bps.size(), "GPU" if cuda else "CPU worker",
                                                         bps.size() * args.batch_size * args.seq_len * args.steps / dt,
                                                         loss.item()))
bps.shutdown()
