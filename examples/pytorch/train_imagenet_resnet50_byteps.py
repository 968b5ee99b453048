#!/usr/bin/env python
"""ImageNet-style ResNet-50 loop with the reference's checkpoint/resume pattern
(example/pytorch/train_imagenet_resnet50_byteps.py:70-80,145-155,245-252): rank 0
saves/loads with torch.save/load, everybody receives the state through
broadcast_parameters + broadcast_optimizer_state; gradient accumulation with
backward_passes_per_step; lr warm-up; metrics averaged by push_pull.  Synthetic
data stands in for the dataset (no network).

With --fused-update the optimizer state lives in per-rank shards of the exchange; its
state_dict() gathers the full state and is collective, so every rank calls it and
rank 0 alone saves."""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))
import byteps_b200.torch as bps  # noqa: E402
from byteps_b200.models import get_model  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--checkpoint-format", default="./checkpoint-{epoch}.pth.tar")
p.add_argument("--batch-size", type=int, default=32)
p.add_argument("--batches-per-pushpull", type=int, default=1)
p.add_argument("--epochs", type=int, default=2)
p.add_argument("--steps-per-epoch", type=int, default=20)
p.add_argument("--base-lr", type=float, default=0.0125)
p.add_argument("--warmup-epochs", type=float, default=1)
p.add_argument("--model", default="resnet50")
p.add_argument("--image-size", type=int, default=224)
p.add_argument("--no-cuda", action="store_true")
p.add_argument("--fused-update", action="store_true",
               help="optimizer step inside the exchange kernels (fp32 master shards)")
p.add_argument("--optimizer", choices=("sgd", "lars"), default="sgd",
               help="lars: byteps_b200.torch.Lars, with batch-norm parameters and biases in an adapt=False, "
                    "weight_decay=0 group")
p.add_argument("--sync-bn", action="store_true",
               help="batch-norm statistics over all ranks' batches (bps.convert_sync_batchnorm; CUDA channels_last)")
args = p.parse_args()
bps.init()
cuda = torch.cuda.is_available() and not args.no_cuda
if cuda:
    torch.cuda.set_device(bps.local_rank())
dev = torch.device("cuda", bps.local_rank()) if cuda else torch.device("cpu")
resume_from = 0
for e in range(args.epochs, 0, -1):
    if os.path.exists(args.checkpoint_format.format(epoch=e)):
        resume_from = e
        break
resume_from = int(bps.broadcast_object(resume_from, 0, name="resume_from_epoch"))
model = get_model(args.model).to(dev)
if args.sync_bn:
    # synchronised training takes NHWC (channels_last) activations; converting is collective
    model = bps.convert_sync_batchnorm(model.to(memory_format=torch.channels_last))
lr = args.base_lr * args.batches_per_pushpull * bps.size()
if args.optimizer == "lars":
    # the large-batch recipe: no trust ratio and no decay for batch-norm parameters and biases (1-d tensors)
    decayed = [q for q in model.parameters() if q.dim() > 1]
    plain = [q for q in model.parameters() if q.dim() <= 1]
    opt = bps.Lars([dict(params=decayed, weight_decay=5e-5), dict(params=plain, weight_decay=0.0, adapt=False)],
                   lr=lr, momentum=0.9)
else:
    opt = torch.optim.SGD(model.parameters(), lr=lr, momentum=0.9, weight_decay=5e-5)
opt = bps.DistributedOptimizer(opt, named_parameters=model.named_parameters(),
                               backward_passes_per_step=args.batches_per_pushpull,
                               fused_update=args.fused_update and cuda)
if resume_from > 0 and bps.rank() == 0:
    ck = torch.load(args.checkpoint_format.format(epoch=resume_from), map_location=dev)
    model.load_state_dict(ck["model"])
    opt.load_state_dict(ck["optimizer"])
bps.broadcast_parameters(model.state_dict(), root_rank=0)
bps.broadcast_optimizer_state(opt, root_rank=0)
for epoch in range(resume_from, args.epochs):
    for step in range(args.steps_per_epoch):
        frac = epoch + step / args.steps_per_epoch
        scale = min(1.0, (frac * (bps.size() - 1) / max(args.warmup_epochs, 1e-9) + 1) / bps.size())
        for g in opt.param_groups:
            g["lr"] = args.base_lr * bps.size() * args.batches_per_pushpull * scale
        opt.zero_grad()
        for _ in range(args.batches_per_pushpull):
            x = torch.rand(args.batch_size, 3, args.image_size, args.image_size, device=dev)
            if args.sync_bn:
                x = x.contiguous(memory_format=torch.channels_last)
            y = torch.randint(0, 1000, (args.batch_size,), device=dev)
            loss = F.cross_entropy(model(x), y) / args.batches_per_pushpull
            loss.backward()
        opt.step()
    avg = bps.push_pull(loss.detach(), name="train_loss").item()
    opt_state = opt.state_dict()            # collective with --fused-update: every rank takes part
    if bps.rank() == 0:
        print("epoch %d: avg loss %.4f%s" % (epoch + 1, avg, " (resumed from epoch %d)" % resume_from if resume_from else ""))
        torch.save({"model": model.state_dict(), "optimizer": opt_state}, args.checkpoint_format.format(epoch=epoch + 1))
bps.shutdown()
