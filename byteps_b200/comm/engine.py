"""The push-pull engine: name registry, partitioning, priority/credit scheduling,
handles, and dispatch to a transport.

Host-side shape of the reference runtime (SURVEY 3.2/3.3):
``EnqueueTensor`` partitions a tensor and feeds 12 stage queues polled by up to
15 threads (/root/reference/byteps/common/operations.cc:182-281,
core_loops.cc).  On one NVSwitch box the GPU path needs none of that: a
push_pull is *stream ordered*.  The comm stream waits on an event recorded on
the producer stream, ONE fused kernel per batch of partitions does
pack+reduce-scatter+all-gather+unpack, and completion is another event that
``synchronize`` makes the consumer stream wait on - no host thread, no 1 us
polling, and the whole thing can be captured into a CUDA graph.  The native
scheduler still decides the ORDER of partitions inside a flush window
(priority desc, key asc, byte credits), exactly like the reference's
BytePSScheduledQueue.
"""
from __future__ import annotations

import threading
from dataclasses import dataclass, field
from typing import Dict, Optional

import torch

from .. import _native
from ..config import Config
from .symm import SymmContext

_CORE_DT = None
_SYMM_DTYPES = (torch.float32, torch.bfloat16, torch.float16)    # what the symmetric-memory kernels reduce


def core_dtype(dtype: torch.dtype) -> int:
    global _CORE_DT
    if _CORE_DT is None:
        c = _native.core()
        _CORE_DT = {
            torch.float32: c.F32, torch.float64: c.F64, torch.float16: c.F16, torch.uint8: c.U8,
            torch.int32: c.I32, torch.int8: c.I8, torch.int64: c.I64, torch.bfloat16: c.BF16,
        }
    try:
        return _CORE_DT[dtype]
    except KeyError:
        raise ValueError("Tensor type %s is not supported." % dtype)


@dataclass
class _HandleState:
    tensor: torch.Tensor
    output: torch.Tensor
    name: str
    average: bool
    done_event: Optional[torch.cuda.Event] = None
    work: list = field(default_factory=list)    # torch.distributed Work objects
    post: list = field(default_factory=list)    # callables run at synchronize
    native: int = -1                            # native handle id (host pipeline)
    start_us: int = 0


class PushPullEngine:
    def __init__(self, cfg: Config, group, pg=None):
        self.cfg = cfg
        self.group = group
        self.pg = pg
        self.core = _native.core()
        self.registry = self.core.Registry()
        self.timeline = self.core.Timeline()
        self.timeline.configure(cfg.trace_on, cfg.trace_start_step, cfg.trace_end_step, cfg.trace_dir, cfg.local_rank)
        self.telemetry = self.core.Telemetry(cfg.telemetry_on, 10.0)
        self._handles: Dict[int, _HandleState] = {}
        self._next_handle = 0
        self._lock = threading.RLock()
        self._noname = 0
        self._step_of: Dict[str, int] = {}
        self.rank, self.size = cfg.rank, cfg.size
        self.symm: Optional[SymmContext] = None
        self.comm_stream = None
        self._native_meta: Dict[int, tuple] = {}
        self._trace_native = bool(cfg.trace_on or cfg.debug_sample_tensor)
        self._launches = 0         # kernels of OURS launched (bench 'gpu_launches'), see the `launches` property
        self._native = None        # csrc/torch/native_ops.cc: the per-tensor symmetric-memory push_pull
        self._compress_kwargs: Dict[str, Dict[str, str]] = {}   # per-tensor compressor config (declare kwargs)
        self._gpu_compressors: Dict[str, object] = {}
        self._compress_ctx: Optional[SymmContext] = None
        self._compress_cursor = 0
        self._lr = None
        self._hostshm = None       # same-host CPU jobs: box-local reduction instead of gloo (csrc/core/host_reduce.h)
        self._hostshm_state = None
        self.backend = self._pick_backend()

    @property
    def launches(self) -> int:
        return self._launches + (self._native.launches if self._native is not None else 0)

    @launches.setter
    def launches(self, value: int):
        self._launches = value - (self._native.launches if self._native is not None else 0)

    # ------------------------------------------------------------------ setup
    def _pick_backend(self) -> str:
        b = self.cfg.backend
        if self.size == 1:
            return "local"
        if b == "auto":
            b = "symm" if torch.cuda.is_available() else "gloo"
        return b

    def _ensure_symm(self, device):
        if self.symm is None:
            self.symm = SymmContext(self.group, device, self.cfg.arena_bytes, self.cfg.symm_mode, self.cfg.use_nvls)
            if self.comm_stream is None:
                self.comm_stream = torch.cuda.Stream(device=device, priority=-1)
            self._make_native(device)
        return self.symm

    def _make_native(self, device):
        """The native torch adapter drives the generic per-tensor path: declare -> partition -> priority /
        credit queue -> fused pack+exchange+unpack launches, with cudaStreamWaitEvent readiness and native
        handles (reference: byteps/torch/ops.cc:54-135, ready_event.cc, handle_manager.cc)."""
        mod = _native.torch_ops()
        import os as _os

        cfg, ctx = self.cfg, self.symm
        view = ctx.view
        wire = {"bf16": 1, "bfloat16": 1, "fp16": 2, "float16": 2, "half": 2}.get(str(cfg.wire_dtype).lower(), -1)
        credit = cfg.scheduling_credit * cfg.partition_bound() if cfg.scheduling_credit > 0 else 0
        dev_index = device.index if device.index is not None else torch.cuda.current_device()
        self._native = mod.NativeSymmOps(
            data=[view.data_ptr(r) for r in range(self.size)], sig=[view.sig_ptr(r) for r in range(self.size)],
            mc=view.mc_ptr if ctx.nvls else 0, epoch=view.epoch_ptr, rank=self.rank, world=self.size,
            arena_bytes=int(ctx.data_bytes), comm_stream=self.comm_stream.cuda_stream, device=dev_index,
            partition_bytes=cfg.partition_bound(), group_bytes=cfg.group_bytes, one_shot_bytes=cfg.one_shot_bytes,
            flush_bytes=int(_os.environ.get("BYTEPS_FLUSH_BYTES", str(16 << 20))), credit_bytes=credit,
            blocks=cfg.comm_blocks, threads=cfg.comm_threads, nvls=bool(ctx.nvls), wire_override=wire)
        for name in self.registry.declared_names():     # same declaration order -> same keys as the python registry
            self._native.declare(name)

    # ------------------------------------------------------------------ names
    def declare(self, name: str) -> int:
        if self._native is not None:
            self._native.declare(name)
        return self.registry.declare(name)

    def _auto_name(self) -> str:
        self._noname += 1
        return "push_pull.noname.%d" % self._noname

    # ------------------------------------------------------------------ gradient compression config
    def set_compression(self, name: str, kwargs: Optional[dict]):
        """Per-tensor compressor kwargs (``compressor_type``, ``compressor_k``, ``ef_type``,
        ``momentum_type``, ... - docs/gradient-compression.md).  The reference takes them at
        declare time from the MXNet plugin only (mxnet/ops.py:82-123, operations.cc:396-408);
        here every front end can pass them.  NVLink backend: GPU compressors exchanging payloads
        through symmetric memory; CPU-server backend: the native worker/server compressors."""
        if not kwargs:
            return
        full = name if name.startswith("byteps.") else "byteps." + name
        self._compress_kwargs[full] = {str(k): str(v) for k, v in kwargs.items()}
        if self._ps is not None:
            self._ps.set_compression(full, kwargs)

    def set_learning_rate(self, lr: float):
        """Error feedback rescales the residual by lr_prev/lr (the reference reads the rate from
        the mmap'd file ``lr.s`` written by the MXNet trainer, vanilla_error_feedback.cc:42-64)."""
        self._lr = float(lr)
        for c in self._gpu_compressors.values():
            c.set_lr(self._lr)
        if self._ps is not None:
            self._ps.set_learning_rate(self._lr)

    def _new_gpu_compressor(self, name: str, t: torch.Tensor):
        """Payload windows are bump-allocated from dedicated symmetric arenas (created
        collectively, so every rank must compress the same tensors in the same order)."""
        import os as _os

        from ..ops.compress import GpuCompressor

        kw = self._compress_kwargs[name]
        probe = GpuCompressor.payload_bytes_for(kw, t.numel(), self.size)
        ctx = self._compress_ctx
        if ctx is None or self._compress_cursor + probe > ctx.data_bytes:
            nbytes = max(int(_os.environ.get("BYTEPS_COMPRESS_ARENA_BYTES", str(64 << 20))), probe + 4096)
            ctx = SymmContext(self.group, t.device, nbytes, self.cfg.symm_mode, "0")
            self._compress_ctx = ctx
            self._compress_cursor = 0
        comp = GpuCompressor(ctx, kw, t.numel(), t.dtype, payload_off=self._compress_cursor)
        self._compress_cursor += comp.payload_bytes
        if self._lr is not None:
            comp.set_lr(self._lr)
        self._gpu_compressors[name] = comp
        return comp

    def _compressed_symm(self, h: int, st: _HandleState):
        """One compressed tensor over NVLink: momentum/error-feedback/compress, payload exchange,
        decompress-and-sum, (server-stage recompression), all on the communication stream."""
        t, out = st.tensor, st.output
        self.flush()
        self._ensure_symm(t.device)
        comp = self._gpu_compressors.get(st.name)
        if comp is None or comp.n != t.numel() or comp.dtype != t.dtype:
            comp = self._new_gpu_compressor(st.name, t)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(t.device))
        self.comm_stream.wait_event(ev)
        comp.push_pull(t, out, st.average, stream=self.comm_stream)
        self.launches += 1
        st.done_event = torch.cuda.Event()
        st.done_event.record(self.comm_stream)

    # ------------------------------------------------------------------ API
    def push_pull_async(self, tensor: torch.Tensor, output: torch.Tensor, average: bool, name: Optional[str],
                        version: int = 0, priority: int = 0, flush: bool = True) -> int:
        if not tensor.is_contiguous() or not output.is_contiguous():
            raise ValueError("Tensor is required to be contiguous.")
        core_dtype(tensor.dtype)  # validates dtype
        name = "byteps." + (self._auto_name() if name is None else name)
        nbytes = tensor.numel() * tensor.element_size()
        symm = self.backend == "symm" and tensor.is_cuda and tensor.dtype in _SYMM_DTYPES and tensor.numel() > 0
        if symm and not (name in self._compress_kwargs and nbytes >= self.cfg.min_compress_bytes):
            # the native adapter: declare -> partition -> priority/credit queue -> fused launches
            self._ensure_symm(tensor.device)
            h = self._native.try_push_pull_async(tensor, output, average, name[7:], priority, version, flush)
            if h < 0:
                raise ValueError("push_pull of a CUDA tensor needs a CUDA output of the same dtype and size")
            if self._trace_native:
                self._native_meta[h] = (name, self.core.now_us())
            return -(h + 1)          # handles of the native adapter are negative on this side
        with self._lock:
            self.registry.declare(name)
            h = self._next_handle
            self._next_handle += 1
            st = _HandleState(tensor, output, name, average, start_us=self.core.now_us())
            self._handles[h] = st
        if self.telemetry.should_record():
            self.telemetry.record(nbytes)
        if self.backend == "local" or tensor.numel() == 0:
            self._local(st)
        elif symm:
            self._compressed_symm(h, st)
        elif self.backend == "ps":
            self._enqueue_ps(h, st, priority, version)
        else:
            self._collective(h, st, priority)
        return h

    def poll(self, h: int) -> bool:
        if h < 0:
            return self._native.poll(-h - 1)
        st = self._handles.get(h)
        if st is None:
            return True
        if st.native >= 0:
            return self._ps.poll(st.native)
        if st.done_event is not None and not st.done_event.query():
            return False
        return all(w.is_completed() for w in st.work)

    def synchronize(self, h: int, block_host: bool = False):
        if h < 0:
            out = self._native.synchronize(-h - 1, block_host)
            if self.telemetry.should_record():
                nb = self._native.take_bytes()
                if nb:
                    self.telemetry.record(nb)
            meta = self._native_meta.pop(-h - 1, None) if self._native_meta else None
            if meta is not None:
                st = _HandleState(out, out, meta[0], False, start_us=meta[1])
                self._sample(st)
                self._finish_trace(st)
            return out
        st = self._handles.get(h)
        if st is None:
            return None
        if st.native >= 0:
            self._ps.wait(st.native)
        for w in st.work:
            w.wait()
        if st.done_event is not None:
            if block_host:
                st.done_event.synchronize()
            else:
                torch.cuda.current_stream(st.output.device).wait_event(st.done_event)
        for fn in st.post:
            fn()
        self._sample(st)
        with self._lock:
            self._handles.pop(h, None)
        self._finish_trace(st)
        return st.output

    def _sample(self, st):
        if self.cfg.debug_sample_tensor and self.cfg.debug_sample_tensor in st.name:
            # BYTEPS_DEBUG_SAMPLE_TENSOR: first/last element after the operation (the host pipeline of the
            # CPU-server mode prints them after every stage like the reference, core_loops.cc:37-67)
            flat = st.output.detach().view(-1)
            if flat.numel():
                print("[byteps_b200] sample %s rank=%d first=%s last=%s" % (
                    st.name, self.rank, flat[0].item(), flat[-1].item()), flush=True)

    def outstanding(self) -> int:
        return len(self._handles) + (self._native.outstanding() if self._native is not None else 0)

    # ------------------------------------------------------------------ local
    def _local(self, st: _HandleState):
        if st.output.data_ptr() != st.tensor.data_ptr():
            st.output.copy_(st.tensor)

    # ------------------------------------------------------------------ torch.distributed transports
    def _collective(self, h: int, st: _HandleState, priority: int):
        """gloo plumbing / reference-style NCCL path: one all-reduce (or RS+AG)
        per partition, issued in (priority, key) order."""
        import torch.distributed as dist

        t, out = st.tensor, st.output
        if out.data_ptr() != t.data_ptr():
            out.copy_(t)
        if self.backend == "nccl" and out.is_cuda and out.is_floating_point():
            # the reference's own single-box path (baseline arm): per-partition RS+AG in groups of 4, then div_
            if self._nccl_ref is None:
                from .nccl_baseline import NativeNcclReferencePath, NcclReferencePath

                import os as _os

                if _os.environ.get("BYTEPS_NCCL_NATIVE", "1") not in ("0", ""):
                    self._nccl_ref = NativeNcclReferencePath(self.group, out.device, self.cfg.partition_bytes)
                else:
                    self._nccl_ref = NcclReferencePath(self.pg, self.cfg.partition_bytes)
            st.done_event = self._nccl_ref.push_pull_([out], average=st.average)
            return
        keys = self.registry.init_tensor(st.name, out.numel() * out.element_size(), core_dtype(out.dtype),
                                         self.cfg.partition_bound(), 4096)
        if not out.is_cuda and self._host_shm_reduce(st, keys[0]):
            return
        flat = out.view(-1)
        es = out.element_size()
        for (off, ln), _k in zip(self.registry.partitions(st.name), keys):
            part = flat[off // es:(off + ln) // es]
            st.work.append(dist.all_reduce(part, op=dist.ReduceOp.SUM, group=self.pg, async_op=True))
        if st.average:
            st.post.append(lambda o=out: _divide(o, self.size))

    def _host_shm_reduce(self, st: _HandleState, key0: int) -> bool:
        """CPU tensor, several ranks per host: sum inside every host through shared-memory slots and the CPU reducer
        (csrc/core/host_reduce.h: READY / DO_BROADCAST datagrams, root = highest local rank) instead of sending
        everything through gloo's ring.  One host: that is the whole exchange.  Several hosts: the hosts' roots
        all-reduce the box sums over gloo (1/local_size of the traffic) before they publish.  False -> the caller
        falls back to plain gloo (disabled, one rank per host, tensor too large for /dev/shm)."""
        import os as _os

        import torch.distributed as dist

        if self._hostshm_state is None:
            want = _os.environ.get("BYTEPS_HOST_SHM_REDUCE", "auto").lower()
            L = self.cfg.local_size
            regular = L > 1 and self.size % L == 0 and self.rank == self.cfg.worker_id * L + self.cfg.local_rank
            free = 0
            if want not in ("0", "") and self.backend == "gloo" and self.size > 1:
                # every rank must take the same decision (for the job and for every tensor): the smallest /dev/shm
                # and "is the rank layout box-major everywhere" are agreed on once
                try:
                    vfs = _os.statvfs("/dev/shm")
                    mine = vfs.f_bavail * vfs.f_frsize
                except OSError:
                    mine = 0
                box = torch.tensor([mine if regular else 0, L], dtype=torch.int64)
                lo, hi = box.clone(), box.clone()
                dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=self.pg)
                dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=self.pg)
                free = int(lo[0]) if int(lo[1]) == int(hi[1]) else 0      # same local size on every host
            enabled = free >= (256 << 20) or (want == "1" and free > 0)
            self._hostshm_state = {"enabled": enabled, "budget": free // 2, "used": 0, "keys": {}, "seq": 0}
            if enabled:
                import threading
                from concurrent.futures import ThreadPoolExecutor

                boxes = self.size // L
                tag = "g%s_%d" % (_os.environ.get("MASTER_PORT", str(self.cfg.root_port)), self.cfg.worker_id)
                try:          # binds a Unix datagram socket under BYTEPS_SOCKET_PATH (/tmp)
                    self._hostshm = self.core.HostLocalReduce(self.cfg.local_rank, L, tag, 0)
                    ok = 1
                except Exception as e:  # noqa: BLE001
                    self.core.log(3, "host shm reduce unavailable on rank %d (%s): using gloo" % (self.rank, e))
                    ok = 0
                agreed = torch.tensor([ok], dtype=torch.int64)
                dist.all_reduce(agreed, op=dist.ReduceOp.MIN, group=self.pg)
                if int(agreed[0]) == 0:          # one rank could not set it up: nobody uses it
                    self._hostshm = None
                    state = self._hostshm_state
                    state["enabled"] = False
                    return False
                self._hostshm_reducer = self.core.CpuReducer(0)
                self._hostshm_pool = ThreadPoolExecutor(max_workers=4, thread_name_prefix="bps-hostshm")
                # the hosts' roots exchange the box sums; collectives of one group must be issued in the same order
                # everywhere, so the pool's jobs take turns (submission order) for that one call
                self._hostshm_roots = (dist.new_group(ranks=[b * L + L - 1 for b in range(boxes)], backend="gloo")
                                       if boxes > 1 else None)
                self._hostshm_turn = 0
                self._hostshm_cv = threading.Condition()
                dist.barrier(group=self.pg)          # every rank's datagram socket exists from here on
        state = self._hostshm_state
        if not state["enabled"]:
            return False
        t, out = st.tensor, st.output
        nbytes = out.numel() * out.element_size()
        L = self.cfg.local_size
        known = state["keys"].get(key0)
        if known is None:
            cost = (L + 1) * ((nbytes + 4095) // 4096 * 4096)
            known = state["used"] + cost <= state["budget"]        # same arithmetic on every rank
            if known:
                state["used"] += cost
            state["keys"][key0] = known
        if not known:
            return False
        hr, code, size = self._hostshm, core_dtype(out.dtype), self.size
        scale_on_root = st.average and out.is_floating_point()
        roots = self._hostshm_roots
        seq = state["seq"]
        state["seq"] += 1

        def across_hosts(win):
            """gloo all-reduce of the box sum in the window, enqueued in submission order on every root"""
            import ctypes

            view = torch.frombuffer((ctypes.c_uint8 * nbytes).from_address(win), dtype=torch.uint8).view(out.dtype)
            with self._hostshm_cv:
                self._hostshm_cv.wait_for(lambda: self._hostshm_turn == seq)
                try:
                    work = dist.all_reduce(view, op=dist.ReduceOp.SUM, group=roots, async_op=True)
                finally:
                    self._hostshm_turn = seq + 1
                    self._hostshm_cv.notify_all()
            work.wait()

        def skip_turn():
            with self._hostshm_cv:
                self._hostshm_cv.wait_for(lambda: self._hostshm_turn == seq)
                self._hostshm_turn = seq + 1
                self._hostshm_cv.notify_all()

        def job():
            took_turn = roots is None or not hr.is_root()
            try:
                if not hr.contribute(key0, out.data_ptr(), nbytes, 300000):
                    raise RuntimeError("host shm reduce: cannot reach the shared region of %s" % st.name)
                # one host: every rank scales the shard it summed; several hosts: the root scales after the exchange
                alpha = (1.0 / size) if (scale_on_root and roots is None) else 1.0
                if hr.is_root():
                    win = hr.reduce(key0, nbytes, code, 300000, alpha)
                    if not win:
                        raise RuntimeError("host shm reduce: timed out waiting for the local ranks' %s" % st.name)
                    if roots is not None:
                        took_turn = True
                        across_hosts(win)
                        if scale_on_root:
                            self._hostshm_reducer.scale(win, nbytes, code, 1.0 / size)
                    if not hr.publish(key0, out.data_ptr(), nbytes, 300000):
                        raise RuntimeError("host shm reduce: local ranks did not collect %s" % st.name)
                elif not hr.collect(key0, out.data_ptr(), nbytes, 300000, code, alpha):
                    raise RuntimeError("host shm reduce: no result from the root for %s" % st.name)
            finally:
                if not took_turn:
                    skip_turn()          # a failed root job must not block the jobs queued behind it

        st.work.append(_FutureWork(self._hostshm_pool.submit(job)))
        if st.average and not scale_on_root:
            st.post.append(lambda o=out: _divide(o, size))
        return True

    # ------------------------------------------------------------------ symmetric-memory transport
    def flush(self):
        """Drain the native scheduler into fused launches (deterministic on every rank
        as long as ranks enqueue the same tensors between flush points)."""
        if self._native is not None:
            self._native.flush()

    # ------------------------------------------------------------------ parameter-server transport
    _ps = None
    _nccl_ref = None

    def attach_ps(self, ps_client):
        self._ps = ps_client
        for name, kw in self._compress_kwargs.items():
            ps_client.set_compression(name, kw)

    def init_tensor(self, name: str, tensor: torch.Tensor):
        """Seed the server-side copy of `name` (CPU-server backend; a no-op elsewhere)."""
        if self.backend == "ps" and self._ps is not None:
            full = name if name.startswith("byteps.") else "byteps." + name
            self.registry.declare(full)
            self._ps.init_tensor(full, tensor)

    def _enqueue_ps(self, h: int, st: _HandleState, priority: int, version: int):
        if self._ps is None:
            raise RuntimeError("backend 'ps' selected but no parameter-server client is attached")
        st.native = self._ps.push_pull(st, priority, version)

    # ------------------------------------------------------------------ tracing
    def _finish_trace(self, st: _HandleState):
        if not self.timeline.enabled():
            return
        step = self._step_of.get(st.name, 0)
        self._step_of[st.name] = step + 1
        if self.timeline.active(step):
            now = self.core.now_us()
            self.timeline.record(st.name, "", (1 << 64) - 1, st.start_us, max(1, now - st.start_us))
        if step + 1 == self.timeline.end_step() and all(
                v >= self.timeline.end_step() for v in self._step_of.values()):
            self.timeline.dump()

    def shutdown(self):
        for h in list(self._handles):
            try:
                self.synchronize(h)
            except Exception:  # noqa: BLE001
                pass
        if self.timeline.enabled() and self.timeline.num_events():
            self.timeline.dump()
        if self.comm_stream is not None:
            self.comm_stream.synchronize()
        if self._hostshm is not None:
            self._hostshm_pool.shutdown(wait=True)
            self._hostshm = None
        self._native = None
        if self.symm is not None:
            if self.size > 1:
                try:
                    self.group.barrier()
                except Exception:  # noqa: BLE001
                    pass
            ctxs = {id(c.ctx): c.ctx for c in self._gpu_compressors.values()}
            self._gpu_compressors.clear()
            self._compress_ctx = None
            for c in ctxs.values():
                c.close()
            self.symm.close()
            self.symm = None


class _FutureWork:
    """concurrent.futures.Future behind the wait() / is_completed() face of a torch.distributed Work."""

    def __init__(self, fut):
        self._f = fut

    def wait(self):
        self._f.result()

    def is_completed(self) -> bool:
        return self._f.done()


def _divide(t: torch.Tensor, n: int):
    if t.is_floating_point():
        t.div_(n)
    else:
        t.copy_(torch.floor_divide(t, n))
