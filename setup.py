#!/usr/bin/env python
"""Build / install byteps_b200.

    python setup.py build_ext --inplace      # compile _core (g++) and _cuda (nvcc sm_90a) next to the sources
    pip install --no-build-isolation -e .     # editable install; the .so files stay in-tree

The reference's setup.py (/root/reference/setup.py:177-1075) builds ps-lite with make (downloading
ZeroMQ), then one extension per framework against TH/THC, TF and MXNet headers.  Here there are two
framework-independent modules driven by byteps_b200/_build.py: `_core` (C++17 runtime: registry,
scheduler, reducer, compressors, transport, server, PS worker; also linked as libbyteps_b200.so for the C API) and
`_cuda` (sm_90a kernels, symmetric memory, NCCL baseline manager), plus `_torch_ops` (the native torch adapter,
pybind over at::Tensor); the other framework front ends are python over the same engine.
Environment: BYTEPS_WITHOUT_CUDA=1 skips the CUDA module (CPU-only boxes without nvcc).
"""
import os
import sys

from setuptools import Command, find_packages, setup
from setuptools.command.build_ext import build_ext as _build_ext
from setuptools.command.build_py import build_py as _build_py

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def _compile():
    from byteps_b200 import _build

    _build.build_core(verbose=True)
    if os.environ.get("BYTEPS_WITHOUT_CUDA", "0") in ("0", ""):
        _build.build_cuda(verbose=True)       # _cuda + the C API's CUDA half (libbyteps_b200_cuda.so)
        _build.build_torch(verbose=True)      # _torch_ops: the native torch adapter


class build_ext(_build_ext):
    def run(self):
        _compile()


class build_py(_build_py):
    def run(self):
        _compile()
        super().run()


class BuildNative(Command):
    description = "compile the native modules in-tree"
    user_options = []

    def initialize_options(self):
        pass

    def finalize_options(self):
        pass

    def run(self):
        _compile()


setup(
    name="byteps_b200",
    version="0.1.0",
    description="Hopper-native gradient synchronisation with the capabilities of bytedance/byteps",
    packages=find_packages(include=["byteps_b200", "byteps_b200.*"]),
    package_data={"byteps_b200": ["*.so", "csrc/*/*"]},
    scripts=["bin/bpslaunch"],
    python_requires=">=3.9",
    install_requires=["torch", "numpy", "cloudpickle"],
    cmdclass={"build_ext": build_ext, "build_py": build_py, "build_native": BuildNative},
    zip_safe=False,
)
