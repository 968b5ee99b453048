"""Worker-side client of the CPU summation server (CPU-server mode).

Parity: the distributed stage lists of the reference
(/root/reference/byteps/common/operations.cc:429-485): for a GPU tensor
``REDUCE -> COPYD2H -> [COMPRESS] -> PUSH -> PULL -> [DECOMPRESS] -> COPYH2D ->
BROADCAST``, for a host tensor just the middle part.  Here

* the middle part is the native pipeline in csrc/core/ps_worker.cc,
* COPYD2H / COPYH2D are ``cudaMemcpyAsync`` on side streams into pinned host
  staging, chained by events (the native pipeline polls the D2H event instead
  of a blocking ``cudaStreamSynchronize``, core_loops.cc:431-435),
* REDUCE / BROADCAST are the reduce-scatter / all-gather halves of the fused
  NVLink kernel when several GPUs of one box share a worker ("hierarchical"
  mode): every GPU then pushes ITS shard under its own key, so the host path
  runs 8-wide instead of funnelling through one root process.
"""
from __future__ import annotations

import ctypes
import itertools
import os
import threading
from typing import Dict, Optional

import torch

from .. import _native
from ..config import Config

_PS_DT = None


def _dt(dtype):
    from .engine import core_dtype

    return core_dtype(dtype)


_MEMMOVE_MAX = int(os.environ.get("BYTEPS_STAGING_MEMMOVE_MAX", 2 << 20))


def _host_copy(dst: torch.Tensor, src: torch.Tensor):
    """Byte copy between two host tensors of equal size (either may be the uint8 staging window).  Small and medium
    tensors take a plain memmove (ctypes releases the GIL): torch's copy_ wakes its whole intra-op thread team per
    call, ~300 us for the typical gradient tensor (measured on ResNet-like sets: 1.4 GB/s).  Large ones keep copy_,
    whose parallel memcpy beats one thread (100 MB: ~2 ms vs ~11 ms)."""
    nbytes = dst.numel() * dst.element_size()
    if (nbytes <= _MEMMOVE_MAX and dst.is_contiguous() and src.is_contiguous()
            and nbytes == src.numel() * src.element_size()):
        if nbytes:
            ctypes.memmove(dst.data_ptr(), src.data_ptr(), nbytes)
    elif dst.dtype == torch.uint8:
        dst.copy_(src.reshape(-1).view(torch.uint8))
    else:                                   # strided output: let torch scatter from a typed view of the window
        dst.copy_(src.view(dst.dtype).reshape(dst.shape))


def _gpu_numa_node(core, index: int) -> int:
    """NUMA node the GPU's PCIe root hangs off, from sysfs (-1 when the host does not say)."""
    try:
        p = torch.cuda.get_device_properties(index)
        bus = "%04x:%02x:%02x.0" % (getattr(p, "pci_domain_id", 0), p.pci_bus_id, p.pci_device_id)
        return int(core.numa_node_of_pci(bus))
    except Exception:  # noqa: BLE001
        return -1


class _Staging:
    """Pinned host staging buffer for one named GPU tensor."""

    def __init__(self, nbytes: int, name: str, use_shm: bool, numa_node: int = -1):
        self.nbytes = nbytes
        core = _native.core()
        self.shm_name = None
        if use_shm:
            # POSIX shm so a colocated server can read/write it without a socket copy
            self.shm_name = "BytePS_ShM_%d_%s" % (os.getpid(), abs(hash(name)) % (1 << 40))
            ptr = core.shm_create(self.shm_name, max(nbytes, 4096))
            if numa_node >= 0:
                # BYTEPS_NUMA_AWARE=1: the window the GPU DMAs into / out of lives on the GPU's node (core/numa.h)
                core.numa_bind_memory(ptr, max(nbytes, 4096), numa_node)
            from .symm import _RawCuda  # noqa: F401

            import ctypes

            buf = (ctypes.c_uint8 * nbytes).from_address(ptr)
            self.host = torch.frombuffer(buf, dtype=torch.uint8)
            self.pinned = False
            if torch.cuda.is_available():
                try:
                    rc = torch.cuda.cudart().cudaHostRegister(ptr, (max(nbytes, 4096) + 4095) // 4096 * 4096, 0)
                    self.pinned = int(rc) == 0
                except Exception:  # noqa: BLE001
                    self.pinned = False
                if not self.pinned:
                    # pageable staging turns every COPYD2H / COPYH2D into a synchronous bounce through the driver
                    core.log(3, "cudaHostRegister failed for the staging window of %s: D2H/H2D copies will be "
                                "pageable (slow, not overlapped)" % name)
        else:
            self.pinned = torch.cuda.is_available()
            self.host = torch.empty(nbytes, dtype=torch.uint8).pin_memory() if torch.cuda.is_available() \
                else torch.empty(nbytes, dtype=torch.uint8)

    def release(self):
        if self.shm_name:
            _native.core().shm_release(self.shm_name)


class PSClient:
    def __init__(self, cfg: Config, engine):
        core = _native.core()
        self.core = core
        self.cfg = cfg
        self.engine = engine
        # every process is a PS worker node; servers/scheduler are told the same count
        self.num_nodes = cfg.size
        # the shm van only exists between colocated processes: registered windows always go by reference there
        extra = {"enable_ipc": os.environ.get("BYTEPS_ENABLE_IPC", "0") not in ("0", "")
                 or os.environ.get("DMLC_PS_VAN_TYPE", "") == "shm"}
        self.ipc = extra["enable_ipc"]
        if self.ipc and os.environ.get("BYTEPS_SHM_REAP_STALE", "0") not in ("0", ""):
            core.shm_reap_stale()      # staging windows / server stores of byteps processes that were killed
        self.po = core.Postoffice("worker", self.num_nodes, cfg.num_server, cfg.root_uri, cfg.root_port,
                                  os.environ.get("DMLC_NODE_HOST", ""), cfg.rank, extra)
        credit = cfg.scheduling_credit * cfg.partition_bound() if cfg.scheduling_credit > 0 else 0
        self.worker = core.PSWorker(self.po, cfg.key_hash_fn, credit, cfg.min_compress_bytes, cfg.threadpool_size,
                                    self.num_nodes)
        self.worker.set_timeline(engine.timeline)
        # BYTEPS_NUMA_AWARE=1: tell the servers which NUMA node my GPU hangs off (they place the key stores there),
        # and keep my own staging windows on it (csrc/core/numa.h; BYTEPS_NUMA_NODE overrides the sysfs lookup)
        self.numa_node = -1
        if core.numa_aware() and core.numa_num_nodes() > 1:
            self.numa_node = self.worker.numa_node()
            if self.numa_node < 0 and torch.cuda.is_available():
                self.numa_node = _gpu_numa_node(core, torch.cuda.current_device())
            self.worker.set_numa_node(self.numa_node)
        self._gpu_ctx: Dict[int, int] = {}          # device index -> native staging context (two side streams)
        self._pipelined = os.environ.get("BYTEPS_PS_PIPELINE", "1") not in ("0", "")
        if torch.cuda.is_available():
            try:
                cu = _native.cuda()
                self.worker.set_event_query(cu.event_query_fn())
                self.worker.set_gpu_stage(cu.gpu_stage_fns())
            except Exception:  # noqa: BLE001
                self._pipelined = False
        # several processes per box + CPU tensors: reduce inside the box through shared memory first, only the box's
        # root talks to the servers (csrc/core/host_reduce.h - the reference's PCIE_REDUCE / CPU reducer path with
        # its Unix-datagram READY / DO signals).  Created before the start barrier so every rank's socket exists
        # when the first signal is sent.
        self._hr = None
        self._hr_pool = None
        self._hr_futures: Dict[int, object] = {}
        self._hr_ids = itertools.count(1 << 30)
        self._hr_timeout = int(os.environ.get("BYTEPS_HOST_REDUCE_TIMEOUT_MS", "300000"))
        # default (auto): on for CPU-only jobs whose servers are reached over sockets - L local ranks then cost the
        # wire one push per box (4 processes, 100 MB, TCP: 81 -> 67 ms).  With colocated servers and IPC every rank
        # already pushes and pulls by reference and the flat path is as fast (42 vs 40-50 ms); a GPU job pushes CPU
        # tensors only for small things (broadcast_object, metric averages).  BYTEPS_PS_HOST_HIERARCHICAL=1 forces it.
        want = os.environ.get("BYTEPS_PS_HOST_HIERARCHICAL", "auto").lower()
        if want in ("auto", ""):
            want = "0" if (torch.cuda.is_available() or self.ipc) else "1"
        if cfg.local_size > 1 and want != "0":
            from concurrent.futures import ThreadPoolExecutor

            self._hr = core.HostLocalReduce(cfg.local_rank, cfg.local_size, "%d_%d" % (cfg.root_port, cfg.worker_id),
                                            int(os.environ.get("BYTEPS_OMP_THREAD_PER_GPU", "0") or 0))
            self._hr_pool = ThreadPoolExecutor(max_workers=4, thread_name_prefix="bps-hostreduce")
        self.po.start(0, True)
        self._inited = set()
        self._shapes: Dict[str, tuple] = {}      # name -> (nbytes, dtype code) of its first use
        self._plans: Dict[str, tuple] = {}
        self._staging: Dict[str, _Staging] = {}
        self._d2h = None
        self._h2d = None
        self._lock = threading.Lock()
        self._kwargs: Dict[str, dict] = {}

    # ------------------------------------------------------------------ compression config
    def set_compression(self, name: str, kwargs: Optional[dict]):
        """Per-tensor compressor kwargs (the reference only exposes this through
        MXNet's declare_tensor; here every framework-facing declare can pass it)."""
        if kwargs:
            self._kwargs["byteps." + name if not name.startswith("byteps.") else name] = {
                str(k): str(v) for k, v in kwargs.items()}

    def set_learning_rate(self, lr: float):
        self.worker.set_learning_rate(float(lr))

    # ------------------------------------------------------------------ push_pull
    def _key_name(self, name: str, nbytes: int, code: int) -> str:
        """The name whose keys carry this tensor.  Server keys are sized by their init push, so a tensor
        that comes back under the same name with another size or dtype (a second `broadcast_object`, a
        resized embedding) is keyed as a new generation `name#<bytes>.<dtype>` - declared, initialised
        and barriered like any first use, identically on every worker."""
        first = self._shapes.setdefault(name, (nbytes, code))
        if first == (nbytes, code):
            return name
        alias = "%s#%d.%d" % (name, nbytes, code)
        if alias not in self._shapes:
            self._shapes[alias] = (nbytes, code)
            self.engine.registry.declare(alias)
            kw = self._kwargs.get(name)
            if kw:
                self._kwargs[alias] = kw
        return alias

    def _ensure_keys(self, name, host_ptr, nbytes, dtype_code, parts, keys, pushers, is_float=True):
        if name in self._inited:
            return
        for (off, ln), k in zip(parts, keys):
            self.worker.init_key(k, host_ptr + off, ln, dtype_code, pushers)
            kw = self._kwargs.get(name)
            if kw and is_float:
                self.worker.register_compressor(k, kw, ln, dtype_code)
        self._inited.add(name)

    def init_tensor(self, name: str, tensor: torch.Tensor):
        """Run the init push of `name` with THIS content (a barrier over all workers).  In synchronous
        mode the stored value is irrelevant (every round starts with COPY_FIRST); in asynchronous mode it
        is the base the server accumulates weight deltas onto, so the optimizer seeds it with the weights."""
        if name in self._inited:
            return
        host = tensor.detach().to("cpu").contiguous()
        code = _dt(host.dtype)
        nbytes = host.numel() * host.element_size()
        name = self._key_name(name, nbytes, code)
        if name in self._inited:
            return
        keys = self.engine.registry.init_tensor(name, nbytes, code, self.cfg.partition_bound(), 4096)
        parts = self.engine.registry.partitions(name)
        pushers = 0
        if self._hr is not None and not tensor.is_cuda:
            # box-local reduction: only the box's root ever pushes these keys
            if not self._hr.is_root():
                return
            pushers = self.cfg.num_worker
        self._ensure_keys(name, host.data_ptr(), nbytes, code, parts, keys, pushers, host.dtype.is_floating_point)

    def push_pull(self, st, priority: int, version: int) -> int:
        """st: engine._HandleState.  Returns the native handle."""
        eng = self.engine
        t, out = st.tensor, st.output
        code = _dt(t.dtype)
        nbytes = t.numel() * t.element_size()
        kname = self._key_name(st.name, nbytes, code)
        plan = self._plans.get(kname)
        if plan is None:
            # keys and partitions of (name, size, dtype) never change: look them up once
            keys = eng.registry.init_tensor(kname, nbytes, code, self.cfg.partition_bound(), 4096)
            parts = eng.registry.partitions(kname)
            plan = (nbytes, code, keys, parts)
            self._plans[kname] = plan
        keys, parts = plan[2], plan[3]
        is_float = t.dtype.is_floating_point
        scale = (1.0 / self.cfg.size) if (st.average and is_float) else 1.0
        if st.average and not is_float:
            st.post.append(lambda o=out: o.copy_(torch.floor_divide(o, self.cfg.size)))
        if not t.is_cuda:
            if self._hr is not None:
                return self._push_pull_host_hier(st, kname, nbytes, code, keys, parts, priority, version, scale,
                                                 is_float)
            if self.ipc and nbytes >= (1 << 16):
                # colocated server + CPU tensor: stage through a registered shm window so the payload never
                # crosses a socket (two memcpys instead of two TCP round trips; 100 MB: ~2x faster on loopback)
                stg = self._staging.get(kname)
                if stg is None or stg.nbytes != nbytes:
                    stg = _Staging(nbytes, kname, True)
                    self._staging[kname] = stg
                host = stg.host
                _host_copy(host, t)
                self._ensure_keys(kname, host.data_ptr(), nbytes, code, parts, keys, 0, is_float)
                plist = [(k, off, ln) for (off, ln), k in zip(parts, keys)]
                # the result is delivered into `out` per partition by the worker's pool - straight out of the
                # server's shared-memory store when the server is colocated (pull by reference), so neither the
                # server nor this process copies it a second time
                st._keep = (host, out)
                return self.worker.push_pull(kname, host.data_ptr(), code, plist, priority, version, scale, 0,
                                             out.data_ptr())
            if out.data_ptr() != t.data_ptr():
                out.copy_(t)
            self._ensure_keys(kname, out.data_ptr(), nbytes, code, parts, keys, 0, is_float)
            plist = [(k, off, ln) for (off, ln), k in zip(parts, keys)]
            return self.worker.push_pull(kname, out.data_ptr(), code, plist, priority, version, scale, 0)
        if (self.cfg.local_size > 1 and is_float and t.dtype in (torch.float32, torch.bfloat16, torch.float16)
                and os.environ.get("BYTEPS_PS_HIERARCHICAL", "1") not in ("0", "")):
            return self._push_pull_hier(st, priority, version, code)
        # ---- GPU tensor: COPYD2H -> PUSH -> PULL -> COPYH2D per partition, chained by events
        dev = t.device
        stg = self._staging.get(kname)
        if stg is None or stg.nbytes != nbytes:
            stg = _Staging(nbytes, kname, self.ipc, self.numa_node)
            self._staging[kname] = stg
        host = stg.host
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(dev))
        first = kname not in self._inited
        plist = [(k, off, ln) for (off, ln), k in zip(parts, keys)]
        if self._pipelined and not first:
            # native pipeline (csrc/core/ps_worker.cc::PushPullDevice): the D2H copy of partition i is pushed as soon
            # as it has landed, the H2D copy of partition j is issued from its pull completion, the 1/size scale is
            # applied on the host per partition - D2H, PUSH, PULL and H2D of different partitions overlap
            cu = _native.cuda()
            di = dev.index if dev.index is not None else torch.cuda.current_device()
            gctx = self._gpu_ctx.get(di)
            if gctx is None:
                gctx = cu.gpu_stage_create(di)
                self._gpu_ctx[di] = gctx
            h = self.worker.push_pull_device(kname, t.data_ptr(), out.data_ptr(), host.data_ptr(), code, plist,
                                             priority, version, scale, ready.cuda_event, gctx)
            st._keep = (ready, host, t, out)

            def _wait_h2d(hh=h, d=dev):
                ev = self.worker.take_done_event(hh)        # recorded after the last partition's H2D was enqueued
                if ev:
                    cu.stream_wait_event(torch.cuda.current_stream(d).cuda_stream, ev)

            st.post.insert(0, _wait_h2d)
            return h
        if self._d2h is None:
            self._d2h = torch.cuda.Stream(device=dev)
            self._h2d = torch.cuda.Stream(device=dev)
        self._d2h.wait_event(ready)
        with torch.cuda.stream(self._d2h):
            host.copy_(t.view(-1).view(torch.uint8), non_blocking=True)
            copied = torch.cuda.Event()
            copied.record(self._d2h)
        if first:
            copied.synchronize()   # the init push reads the buffer on the host
        self._ensure_keys(kname, host.data_ptr(), nbytes, code, parts, keys, 0, is_float)
        h = self.worker.push_pull(kname, host.data_ptr(), code, plist, priority, version, scale,
                                  copied.cuda_event)
        st._keep = (copied, ready, host)

        def _h2d(o=out, hb=host, s=self._h2d, d=dev):
            with torch.cuda.stream(s):
                o.view(-1).view(torch.uint8).copy_(hb, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(s)
            torch.cuda.current_stream(d).wait_event(ev)

        st.post.insert(0, _h2d)
        return h

    def _push_pull_hier(self, st, priority: int, version: int, code: int) -> int:
        """Hierarchical CPU-server mode for the GPUs of one box (reference stage list
        REDUCE -> COPYD2H -> PUSH -> PULL -> COPYH2D -> BROADCAST, operations.cc:429-485):

          REDUCE    reduce-scatter half of the NVLink kernel: my shard = box-local sum
          COPYD2H   my shard -> pinned host staging (side stream, event chained)
          PUSH/PULL my shard under MY key (key | (local_rank+1) << 40); the server sums it
                    over the boxes (pushers = DMLC_NUM_WORKER), all 8 host paths run in parallel
          COPYH2D   shard back to the arena
          BROADCAST all-gather half of the kernel, fused with the 1/size scale
        """
        from ..ops.pushpull import all_gather, reduce_scatter, shard_elems

        eng = self.engine
        t, out = st.tensor, st.output
        dev = t.device
        kname = self._key_name(st.name, t.numel() * t.element_size(), code)
        ctx = eng._ensure_symm(dev)
        cs = eng.comm_stream
        n, es = t.numel(), t.element_size()
        nbytes = (n + 7) // 8 * 8 * es
        off = eng._native.alloc_stage(nbytes, True)
        window = ctx.tensor(off, n, t.dtype)
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(dev))
        cs.wait_event(ready)
        b, e = shard_elems(ctx, n)
        with torch.cuda.stream(cs):
            window.copy_(t.view(-1))
            reduce_scatter(ctx, off, n, t.dtype, stream=cs)
            eng.launches += 1
            sbytes = max(e - b, 0) * es
            stg = self._staging.get(kname)
            if stg is None or stg.nbytes != max(sbytes, 16):
                stg = _Staging(max(sbytes, 16), kname, self.ipc, self.numa_node)
                self._staging[kname] = stg
            host = stg.host[:sbytes]
            if sbytes:
                host.copy_(window[b:e].view(torch.uint8), non_blocking=True)
            copied = torch.cuda.Event()
            copied.record(cs)
        # keys of MY shard: one per partition of the shard, tagged with my local rank
        bound = self.cfg.partition_bound()
        parts = self.core.partition_bytes(sbytes, bound) if sbytes else []
        base = eng.registry.declare(kname)
        tag = (self.cfg.local_rank + 1) << 40
        plist = [(self.core.make_key(base, i) | tag, o, ln) for i, (o, ln) in enumerate(parts)]
        if kname not in self._inited:
            copied.synchronize()
            for k, o, ln in plist:
                self.worker.init_key(k, host.data_ptr() + o, ln, code, self.cfg.num_worker)
            self._inited.add(kname)
        scale = (1.0 / self.cfg.size) if st.average else 1.0
        h = self.worker.push_pull(kname, host.data_ptr(), code, plist, priority, version, 1.0,
                                  copied.cuda_event) if plist else -1
        st._keep = (copied, ready, host, window)

        def _finish(o=out, w=window, hb=host, d=dev):
            with torch.cuda.stream(cs):
                if sbytes:
                    w[b:e].view(torch.uint8).copy_(hb, non_blocking=True)
                all_gather(ctx, off, n, t.dtype, scale=scale, stream=cs)
                eng.launches += 1
                o.view(-1).copy_(w)
                ev = torch.cuda.Event()
                ev.record(cs)
            torch.cuda.current_stream(d).wait_event(ev)

        st.post.insert(0, _finish)
        return h

    def _push_pull_host_hier(self, st, kname, nbytes, code, keys, parts, priority, version, scale, is_float) -> int:
        """CPU tensor on a box with several local ranks: contribute to the box's shared-memory slots, the root sums
        them (CpuReducer), pushes the box sum under the tensor's keys (pushers = number of boxes), pulls the global
        sum back into the shared window and tells the other ranks to copy it out.  Runs on a small thread pool so
        `push_pull_async` returns at once; the handle completes when `out` holds the result."""
        hr, t, out = self._hr, st.tensor, st.output
        if not t.is_contiguous() or not out.is_contiguous():
            raise ValueError("Tensor is required to be contiguous.")
        key0 = keys[0]
        plist = [(k, off, ln) for (off, ln), k in zip(parts, keys)]
        tmo = self._hr_timeout

        def job(t=t, out=out):
            if not hr.contribute(key0, t.data_ptr(), nbytes, tmo):
                raise RuntimeError("host reduce: could not reach the box's shared region / root for %s" % kname)
            if hr.is_root():
                win = hr.reduce(key0, nbytes, code, tmo)
                if not win:
                    raise RuntimeError("host reduce: timed out waiting for the local ranks' copies of %s" % kname)
                # no lock: the init push of a key is a barrier over the boxes' roots, and two roots may reach the
                # init pushes of two tensors in opposite order - serialising them would dead-lock
                self._ensure_keys(kname, win, nbytes, code, parts, keys, self.cfg.num_worker, is_float)
                h = self.worker.push_pull(kname, win, code, plist, priority, version, scale, 0)
                self.worker.wait(h, -1)
                if not hr.publish(key0, out.data_ptr(), nbytes, tmo):
                    raise RuntimeError("host reduce: local ranks did not collect %s" % kname)
            elif not hr.collect(key0, out.data_ptr(), nbytes, tmo, code, 1.0):
                raise RuntimeError("host reduce: no result from the box's root for %s" % kname)

        hid = next(self._hr_ids)
        self._hr_futures[hid] = self._hr_pool.submit(job)
        return hid

    def poll(self, h: int) -> bool:
        f = self._hr_futures.get(h)
        if f is not None:
            return f.done()
        return h < 0 or self.worker.poll(h)

    def wait(self, h: int):
        f = self._hr_futures.pop(h, None)
        if f is not None:
            f.result()          # re-raises what the job raised
            return
        if h >= 0:
            self.worker.wait(h, -1)

    def barrier(self):
        self.po.barrier(0, self.core.GROUP_WORKER)

    def close(self):
        try:
            if self._hr_pool is not None:
                self._hr_pool.shutdown(wait=True)
            self._hr = None
            self.worker.stop()
            self.po.finalize(0, True)
        finally:
            for s in self._staging.values():
                s.release()
            self._staging.clear()
            for g in self._gpu_ctx.values():
                try:
                    _native.cuda().gpu_stage_destroy(g)
                except Exception:  # noqa: BLE001
                    pass
            self._gpu_ctx.clear()
