"""Transports behind push_pull.

``symm``  - hand-written sm_90a kernels over symmetric NVLink peer memory (the product)
``nccl``  - reference-style per-partition ncclReduceScatter/ncclAllGather path (the baseline)
``gloo``  - CPU plumbing through torch.distributed (runs without a GPU)
``ps``    - push/pull against the CPU summation server (CPU-server mode)
``local`` - single process
"""
