"""byteps_b200 - a Hopper-native gradient synchronisation engine with the
capabilities and Horovod-style API of bytedance/byteps.

Layer map (see SURVEY.md section 1 for the reference's):

* ``byteps_b200.torch``     - user API: init/push_pull/DistributedOptimizer/DDP/...
* ``byteps_b200.common``    - process-wide state: ranks, config, engine lifecycle
* ``byteps_b200.comm``      - transports: symmetric-memory CUDA kernels, NCCL
                              baseline, gloo plumbing, parameter-server client
* ``byteps_b200.ops``       - python wrappers of the sm_90a kernels
* ``byteps_b200.parallel``  - DistributedDataParallel, CrossBarrier, sharded fused optimizers
* ``byteps_b200.models``    - benchmark model zoo (ResNet/VGG/BERT/MNIST)
* ``byteps_b200.server``    - the CPU summation server (``import byteps_b200.server`` runs it)
* ``byteps_b200.launcher``  - bpslaunch / dist_launcher
* ``byteps_b200._core``     - native C++ runtime   (csrc/core, cpu, compress, net, server)
* ``byteps_b200._cuda``     - native CUDA kernels  (csrc/kernels, comm)
"""
__version__ = "0.1.0"

from . import _native  # noqa: F401  (locates / builds the extension modules)
