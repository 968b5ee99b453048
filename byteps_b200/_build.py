"""In-tree native build for byteps_b200.

Two extension modules are produced next to this file:

* ``_core``  - pure C++17 runtime (registry, scheduler, CPU reducer, compressors,
  KV transport, server).  No CUDA, no torch headers: builds and runs on a CPU box.
* ``_cuda``  - sm_90a CUDA kernels (fused push-pull over NVLink peer memory,
  compression, fused optimizers) + symmetric-memory setup.  Cross-compiled with
  ``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo``.

The reference builds everything through one ``setup.py`` with host-only flags
(/root/reference/setup.py:177-230); we keep builds incremental and in-tree so
the ``.so`` files travel with the repo snapshot to the GPU box.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
EXT = sysconfig.get_config_var("EXT_SUFFIX")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _py_includes():
    import pybind11

    return ["-I" + pybind11.get_include(), "-I" + sysconfig.get_paths()["include"]]


def _nvcc():
    for cand in (os.environ.get("BYTEPS_NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def _cudart_dirs():
    dirs = []
    try:
        import nvidia.cuda_runtime as rt  # the runtime torch itself loads

        dirs.append(os.path.join(list(rt.__path__)[0], "lib"))
    except Exception:
        pass
    dirs.append("/usr/local/cuda/lib64")
    return [d for d in dirs if os.path.isdir(d)]


def _sources(sub, exts):
    out = []
    for root, _, files in os.walk(os.path.join(CSRC, sub)):
        for f in sorted(files):
            if f.endswith(exts):
                out.append(os.path.join(root, f))
    return sorted(out)


def _headers_stamp():
    h = hashlib.sha1()
    for root, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith((".h", ".cuh", ".hpp")):
                p = os.path.join(root, f)
                h.update(p.encode())
                h.update(str(os.path.getmtime(p)).encode())
    return h.hexdigest()


def _need(obj, src, stamp_key, stamps):
    if not os.path.exists(obj):
        return True
    if os.path.getmtime(obj) < os.path.getmtime(src):
        return True
    return stamps.get(obj) != stamp_key


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed:\n%s\n%s" % (" ".join(cmd), r.stdout))
    return r.stdout


def _compile_all(jobs, verbose):
    if not jobs:
        return
    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
        for out in ex.map(lambda c: _run(c, verbose), jobs):
            if verbose and out.strip():
                print(out)


def _load_stamps():
    p = os.path.join(BUILD, "stamps.json")
    if os.path.exists(p):
        try:
            return json.load(open(p))
        except Exception:
            return {}
    return {}


def _save_stamps(s):
    os.makedirs(BUILD, exist_ok=True)
    json.dump(s, open(os.path.join(BUILD, "stamps.json"), "w"))


import platform

_X86 = platform.machine().lower() in ("x86_64", "amd64", "i386", "i686")
# BYTEPS_NO_X86_SIMD=1: build the scalar fallbacks only (what an aarch64 host - e.g. a Grace Hopper system -
# gets automatically); used by the tests to check that the fallbacks are complete
_SIMD = _X86 and os.environ.get("BYTEPS_NO_X86_SIMD", "0") in ("0", "")
CXX_FLAGS = [
    "-O3", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-fopenmp", "-pthread",
    "-Wall", "-Wno-unused-function", "-Wno-sign-compare", "-I" + CSRC,
    # baseline ISA kept portable (AVX2 + FMA + F16C on x86; AVX-512 paths are function-level target attributes and
    # selected at run time); no -m flags elsewhere
] + (["-mavx2", "-mfma", "-mf16c"] if _SIMD else ["-DBPS_NO_X86_SIMD"])


def build_core(verbose=False, force=False):
    os.makedirs(BUILD, exist_ok=True)
    stamps = _load_stamps()
    hs = _headers_stamp()
    srcs = []
    for sub in ("core", "cpu", "compress", "net", "server", "capi"):
        srcs += _sources(sub, (".cc",))
    srcs = [s for s in srcs if os.path.basename(s) != "byteps_cuda_helper.cc"]     # CUDA half: built by build_cuda
    srcs += [s for s in _sources("bind", (".cc",)) if os.path.basename(s).startswith("core_")]
    flags = CXX_FLAGS + _py_includes()
    key = hashlib.sha1((" ".join(flags) + hs).encode()).hexdigest()
    objs, jobs = [], []
    for s in srcs:
        o = os.path.join(BUILD, "core_" + os.path.relpath(s, CSRC).replace("/", "_") + ".o")
        objs.append(o)
        if force or _need(o, s, key, stamps):
            jobs.append(["g++"] + flags + ["-c", s, "-o", o])
            stamps[o] = key
    target = os.path.join(HERE, "_core" + EXT)
    _compile_all(jobs, verbose)
    if jobs or not os.path.exists(target):
        _run(["g++", "-shared", "-o", target] + objs + ["-fopenmp", "-pthread", "-lrt", "-ldl"], verbose)
    # the same runtime without the Python bindings: what C/C++ framework plugins link against (capi/byteps_c_api.h)
    lib = os.path.join(HERE, "libbyteps_b200.so")
    if jobs or not os.path.exists(lib):
        native = [o for o in objs if not os.path.basename(o).startswith("core_bind_")]
        _run(["g++", "-shared", "-o", lib] + native + ["-fopenmp", "-pthread", "-lrt", "-ldl"], verbose)
    _save_stamps(stamps)
    return target


NVCC_FLAGS = [
    "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden", "-I" + CSRC, "-cudart", "shared",
]


def build_cuda(verbose=False, force=False, ptxas_verbose=False):
    nvcc = _nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found; cannot build the sm_90a extension")
    os.makedirs(BUILD, exist_ok=True)
    stamps = _load_stamps()
    hs = _headers_stamp()
    cus = _sources("kernels", (".cu",)) + _sources("comm", (".cu",))
    ccs = _sources("comm", (".cc",)) + [os.path.join(CSRC, "core", "log.cc")]
    ccs += [s for s in _sources("bind", (".cc",)) if os.path.basename(s).startswith("cuda_")]
    nv_flags = NVCC_FLAGS + ARCH_FLAGS + (["-Xptxas", "-v"] if ptxas_verbose else [])
    cc_flags = CXX_FLAGS + _py_includes() + ["-I/usr/local/cuda/include"]
    nkey = hashlib.sha1((" ".join(nv_flags) + hs).encode()).hexdigest()
    ckey = hashlib.sha1((" ".join(cc_flags) + hs).encode()).hexdigest()
    objs, jobs = [], []
    for s in cus:
        o = os.path.join(BUILD, "cuda_" + os.path.relpath(s, CSRC).replace("/", "_") + ".o")
        objs.append(o)
        if force or _need(o, s, nkey, stamps):
            jobs.append([nvcc] + nv_flags + ["-c", s, "-o", o])
            stamps[o] = nkey
    for s in ccs:
        o = os.path.join(BUILD, "cuda_" + os.path.relpath(s, CSRC).replace("/", "_") + ".o")
        objs.append(o)
        if force or _need(o, s, ckey, stamps):
            jobs.append(["g++"] + cc_flags + ["-c", s, "-o", o])
            stamps[o] = ckey
    target = os.path.join(HERE, "_cuda" + EXT)
    _compile_all(jobs, verbose)
    if jobs or not os.path.exists(target):
        link = ["g++", "-shared", "-o", target] + objs
        for d in _cudart_dirs():
            link += ["-L" + d, "-Wl,-rpath," + d]
        link += ["-l:libcudart.so.12", "-pthread", "-ldl", "-lrt"]
        _run(link, verbose)
    # the CUDA half of the C API: what libbyteps_b200.so dlopens for byteps_push_pull_device (no python, no torch)
    helper = os.path.join(HERE, "libbyteps_b200_cuda.so")
    hsrc = os.path.join(CSRC, "capi", "byteps_cuda_helper.cc")
    hobj = os.path.join(BUILD, "cuda_capi_byteps_cuda_helper.cc.o")
    if force or _need(hobj, hsrc, ckey, stamps) or not os.path.exists(helper) or jobs:
        _run(["g++"] + cc_flags + ["-c", hsrc, "-o", hobj], verbose)
        stamps[hobj] = ckey
        # gpu_stage.cc launches the in-place scale kernel of kernels/misc.cu behind a COPYH2D
        link = ["g++", "-shared", "-Wl,--no-undefined", "-o", helper, hobj,
                os.path.join(BUILD, "cuda_comm_gpu_stage.cc.o"), os.path.join(BUILD, "cuda_kernels_misc.cu.o")]
        for d in _cudart_dirs():
            link += ["-L" + d, "-Wl,-rpath," + d]
        link += ["-l:libcudart.so.12", "-pthread", "-ldl", "-lstdc++", "-lm", "-lc"]
        _run(link, verbose)
    _save_stamps(stamps)
    return target


def build_torch(verbose=False, force=False):
    """The native torch adapter (csrc/torch/native_ops.cc -> byteps_b200/_torch_ops*.so): pybind over
    at::Tensor, built against the torch headers/libraries of the running interpreter (no TH/THC).  It links its
    own copies of the runtime pieces it drives (registry, scheduler) and of the exchange kernels, so it has no
    load-time dependency on the other two modules."""
    import torch
    from torch.utils import cpp_extension as ce

    nvcc = _nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found; cannot build the torch adapter")
    os.makedirs(BUILD, exist_ok=True)
    stamps = _load_stamps()
    hs = _headers_stamp()
    tinc = [p for p in ce.include_paths() if "cuda" not in os.path.basename(p.rstrip("/"))]
    tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cc_flags = ["-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-pthread", "-Wall", "-Wno-unused-function",
                "-Wno-sign-compare", "-I" + CSRC, "-I/usr/local/cuda/include", abi,
                "-DTORCH_EXTENSION_NAME=_torch_ops", "-DTORCH_API_INCLUDE_EXTENSION_H"]
    cc_flags += ["-isystem" + p for p in tinc] + ["-I" + sysconfig.get_paths()["include"]]
    nv_flags = NVCC_FLAGS + ARCH_FLAGS
    ckey = hashlib.sha1((" ".join(cc_flags) + hs + torch.__version__).encode()).hexdigest()
    nkey = hashlib.sha1((" ".join(nv_flags) + hs).encode()).hexdigest()
    ccs = [os.path.join(CSRC, "torch", "native_ops.cc"), os.path.join(CSRC, "core", "registry.cc"),
           os.path.join(CSRC, "core", "scheduler.cc"), os.path.join(CSRC, "core", "log.cc")]
    cus = [os.path.join(CSRC, "kernels", "pushpull.cu")]
    objs, jobs = [], []
    for s in ccs:
        o = os.path.join(BUILD, "torch_" + os.path.relpath(s, CSRC).replace("/", "_") + ".o")
        objs.append(o)
        if force or _need(o, s, ckey, stamps):
            jobs.append(["g++"] + cc_flags + ["-c", s, "-o", o])
            stamps[o] = ckey
    for s in cus:
        o = os.path.join(BUILD, "torch_" + os.path.relpath(s, CSRC).replace("/", "_") + ".o")
        objs.append(o)
        if force or _need(o, s, nkey, stamps):
            jobs.append([nvcc] + nv_flags + ["-c", s, "-o", o])
            stamps[o] = nkey
    target = os.path.join(HERE, "_torch_ops" + EXT)
    _compile_all(jobs, verbose)
    if jobs or not os.path.exists(target):
        link = ["g++", "-shared", "-o", target] + objs + ["-L" + tlib, "-Wl,-rpath," + tlib]
        for d in _cudart_dirs():
            link += ["-L" + d, "-Wl,-rpath," + d]
        link += ["-ltorch_python", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10", "-lc10_cuda",
                 "-l:libcudart.so.12", "-pthread", "-ldl", "-lrt"]
        _run(link, verbose)
    _save_stamps(stamps)
    return target


def build_all(verbose=False, force=False):
    a = build_core(verbose, force)
    b = build_cuda(verbose, force)
    c = build_torch(verbose, force)
    return a, b, c


if __name__ == "__main__":
    v = "-v" in sys.argv
    f = "-f" in sys.argv
    if "core" in sys.argv:
        print(build_core(v, f))
    elif "cuda" in sys.argv:
        print(build_cuda(v, f, ptxas_verbose="--ptxas" in sys.argv))
    elif "torch" in sys.argv:
        print(build_torch(v, f))
    else:
        print(build_all(v, f))
