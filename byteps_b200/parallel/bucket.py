"""Zero-copy bucketed gradient synchronisation over symmetric memory.

This is the H100-first replacement for the reference's per-parameter
``push_pull_async_inplace`` hooks (/root/reference/byteps/torch/__init__.py:117-158)
and its per-<=4MB-partition NCCL reduce-scatter/all-gather launches
(core_loops.cc:190-269): gradients LIVE in a peer-mapped arena (``p.grad`` are
strided views into it), buckets are contiguous byte ranges laid out in
backward order, and one fused kernel per bucket does the whole exchange in
place - optionally fused with the fp32 master-weight optimizer step, in which
case the updated parameters (not the gradients) are what is all-gathered.

Everything is stream ordered: a bucket launch waits on an event recorded on the
autograd stream, completion is an event the optimizer step waits on.  No host
thread takes part, so the step can be captured in one CUDA graph.
"""
from __future__ import annotations

import os
import struct
import weakref
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from ..comm.symm import SymmContext, pick_blocks, wire_code
from ..utils.timing import stamp


def _env_int(name, default):
    v = os.environ.get(name)
    return int(v) if v else default


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


REDUCE_ENGINES = ("auto", "nvls", "lsu", "tma", "wgmma")


def _strided_view(flat: torch.Tensor, p: torch.Tensor, offset: int) -> torch.Tensor:
    """A view of `flat` with p's sizes and strides (keeps channels_last etc.)."""
    if p.is_contiguous():
        return flat[offset:offset + p.numel()].view(p.shape)
    return torch.as_strided(flat, p.size(), p.stride(), offset)


def _dense(p: torch.Tensor) -> bool:
    """True if p's storage footprint equals numel (a permutation of contiguous)."""
    if p.numel() == 0:
        return True
    span = 1 + sum((s - 1) * st for s, st in zip(p.size(), p.stride()))
    return span == p.numel()


def shard_bounds(numel: int, world: int, rank: int):
    """Element range [begin, end) of the shard `rank` owns in a bucket of `numel` (padded) elements: the bucket
    is cut into `world` equal runs of 8-element units; trailing ranks of a small bucket own an empty shard."""
    units = numel // 8
    per = (units + world - 1) // world
    s0 = min(per * rank, units)
    s1 = min(s0 + per, units)
    return s0 * 8, s1 * 8


def copy_bucket_state(shard: torch.Tensor, span, starts: List[int], tensors: List[torch.Tensor], to_shard: bool):
    """Copy between one shard of a bucket's flat state and per-parameter tensors - the one place that knows how
    the optimizer state of a bucket is laid out.

    `shard` holds elements [span[0], span[1]) of the flat bucket layout: parameter i occupies
    [starts[i], starts[i] + numel) in storage order (as `_strided_view` maps it, so a channels_last weight is
    stored NHWC), padded to a multiple of 8 elements.  `tensors[i]` has parameter i's shape AND strides, so its
    own storage order is the bucket's.  to_shard=True scatters the tensors into the shard and leaves every
    element no parameter covers (padding, the tail of an over-allocated shard) zero; to_shard=False gathers the
    shard's part of each parameter into its tensor and leaves the rest of the tensor as it was."""
    s0, s1 = span
    if to_shard:
        shard.zero_()
    for t, st in zip(tensors, starts):
        n = t.numel()
        lo, hi = max(st, s0), min(st + n, s1)
        if lo >= hi:
            continue
        flat = torch.as_strided(t, (n,), (1,), t.storage_offset())
        if to_shard:
            shard[lo - s0:hi - s0].copy_(flat[lo - st:hi - st])
        else:
            flat[lo - st:hi - st].copy_(shard[lo - s0:hi - s0])


@dataclass
class Bucket:
    index: int
    group_index: int
    dtype: torch.dtype
    params: List[torch.nn.Parameter] = field(default_factory=list)
    starts: List[int] = field(default_factory=list)    # element offsets inside the bucket
    numel: int = 0                                     # padded element count (multiple of 8)
    grad_off: int = 0                                  # byte offset of the gradient window in the arena
    param_off: int = -1                                # byte offset of the parameter window (fused mode)
    pending: int = 0
    launched: bool = False
    flat_grad: Optional[torch.Tensor] = None
    flat_param: Optional[torch.Tensor] = None
    master: Optional[torch.Tensor] = None              # fp32 shard
    state0: Optional[torch.Tensor] = None
    state1: Optional[torch.Tensor] = None
    done: Optional[torch.cuda.Event] = None
    priority: int = 0                                  # max priority of the parameters inside (scheduling)
    ring_cls: Optional[tuple] = None                   # (wire code, ring kind) of the ring table it belongs to
    ring_pos: int = -1                                 # position inside that table
    lamb_win_off: int = -1                             # byte offset of the norm window (fused LAMB and LARS)
    lamb_params: Optional[torch.Tensor] = None         # LAMB, LARS, clipping: (start, numel) per parameter, int64
    normed: bool = False                               # clipping: this step's norm pass has been issued

    @property
    def nbytes(self) -> int:
        return self.numel * torch.empty((), dtype=self.dtype).element_size()


_LIVE = weakref.WeakSet()


def resync_fused_masters():
    """Re-derive fp32 master shards from the (just broadcast / just loaded)
    parameters of every live fused synchroniser."""
    for s in list(_LIVE):
        if s.fused:
            s.sync_master_from_params()


_HP_FMT = "<9f3if2if"   # matches csrc/kernels/pushpull.cuh::OptHParams (64 bytes)
_TRUST_KINDS = ("lamb", "lars")   # fused optimizers with per-parameter trust ratios: three launches per bucket
_LS_STATE_FMT = "<2df5i"   # csrc/kernels/loss_scale.cuh::LossScaleState (40 bytes)
_LS_ENTRY_FMT = "<2Q4i"    # csrc/kernels/loss_scale.cuh::LossScaleCheckEntry (32 bytes)


class BucketedGradSync:
    """Owns the arena, the buckets and the hooks for one set of parameters."""

    def __init__(self, engine, param_groups, *, fused: Optional[str] = None, wire_dtype: Optional[torch.dtype] = None,
                 bucket_bytes: Optional[int] = None, backward_passes_per_step: int = 1, average: bool = True,
                 priority_of: Optional[Dict] = None, loss_scaler: Optional[Dict] = None,
                 max_grad_norm: Optional[float] = None):
        """loss_scaler (fused mode only): dynamic loss scaling on the device, a dict with GradScaler's
        init_scale, growth_factor, backoff_factor and growth_interval (see `_issue_deferred_step`).
        max_grad_norm (fused mode only): clip the averaged gradients by their global 2-norm before the update, as
        torch.nn.utils.clip_grad_norm_ does (see `_issue_deferred_step`)."""
        self.engine = engine
        self.world, self.rank = engine.size, engine.rank
        self.fused = fused                     # None | "sgd" | "adam" | "adamw" | "lamb" | "lars"
        if loss_scaler is not None and not fused:
            raise ValueError("dynamic loss scaling needs the fused optimizer")
        self.loss_scaler = dict(loss_scaler) if loss_scaler is not None else None
        if max_grad_norm is not None and not fused:
            raise ValueError("max_grad_norm in the exchange needs the fused optimizer")
        self.max_grad_norm = max_grad_norm
        reduce_engine = os.environ.get("BYTEPS_REDUCE_ENGINE", "auto").lower()
        if reduce_engine not in REDUCE_ENGINES:
            raise ValueError("BYTEPS_REDUCE_ENGINE=%s: expected one of %s (the tensor-core engine of sm_90a is 'wgmma')"
                             % (reduce_engine, "|".join(REDUCE_ENGINES)))
        self.average = average
        self.bpps = backward_passes_per_step
        self.bucket_bytes = bucket_bytes or _env_int("BYTEPS_BUCKET_BYTES", 16 << 20)
        self.param_groups = param_groups
        self.wire_override = wire_dtype
        params = [(gi, p) for gi, g in enumerate(param_groups) for p in g["params"] if p.requires_grad]
        if not params:
            raise ValueError("no parameters require gradients")
        self.device = params[0][1].device
        for _, p in params:
            if p.device != self.device or not p.is_cuda:
                raise ValueError("the symmetric-memory path needs all parameters on one CUDA device")
            if not _dense(p):
                raise ValueError("parameters must be dense (contiguous up to a permutation)")
        # backward order ~ reverse of registration order
        order = list(reversed(params))
        self.buckets: List[Bucket] = []
        open_buckets: Dict = {}       # one open bucket per (param group, dtype)
        for gi, p in order:
            es = p.element_size()
            cur = open_buckets.get((gi, p.dtype))
            if cur is None or ((cur.numel + _pad8(p.numel())) * es > self.bucket_bytes and cur.params):
                cur = Bucket(len(self.buckets), gi, p.dtype)
                self.buckets.append(cur)
                open_buckets[(gi, p.dtype)] = cur
            cur.params.append(p)
            cur.starts.append(cur.numel)
            cur.numel += _pad8(p.numel())
        # ---- arena layout: [grad windows][param windows (fused)][staging (wire cast)]
        off = 0
        for b in self.buckets:
            b.grad_off = off
            off = (off + b.nbytes + 255) // 256 * 256
        if fused:
            for b in self.buckets:
                b.param_off = off
                off = (off + b.nbytes + 255) // 256 * 256
        if fused in _TRUST_KINDS:
            # every rank stores its partial norms of each parameter into its slot of every peer's window
            from .. import _native

            for b in self.buckets:
                b.lamb_win_off = off
                off += (_native.cuda().lamb_window_bytes(len(b.params), self.world) + 255) // 256 * 256
        self.stage_off = off
        self.stage_bytes = 0
        if self._needs_stage():
            self.stage_bytes = max(self._wire_bytes(b) for b in self.buckets)
            off += (self.stage_bytes + 255) // 256 * 256
        self.ls_win_off = -1
        if self.loss_scaler is not None:
            # the overflow flags every rank publishes to every peer (loss_scale_update), only in this mode
            self.ls_win_off = off
            off += 256
        self.clip_win_off = -1
        if max_grad_norm is not None:
            # every rank's float64 sum of squares, published to every peer (clip_norm_update), only in this mode
            self.clip_win_off = off
            off += 256
        cfg = engine.cfg
        stamp("buckets: layout of %d buckets, arena %d MiB" % (len(self.buckets), off >> 20))
        self.ctx = SymmContext(engine.group, self.device, max(off, 4096), cfg.symm_mode, cfg.use_nvls)
        stamp("buckets: symmetric arena ready")
        if engine.comm_stream is None:
            engine.comm_stream = torch.cuda.Stream(device=self.device, priority=-1)
        self.comm_stream = engine.comm_stream
        self.threads = cfg.comm_threads
        self._param_bucket: Dict[torch.nn.Parameter, Bucket] = {}
        self._delay: Dict[torch.nn.Parameter, int] = {}
        self._grad_views: Dict[torch.nn.Parameter, torch.Tensor] = {}
        for b in self.buckets:
            b.flat_grad = self.ctx.tensor(b.grad_off, b.numel, b.dtype)
            if fused:
                b.flat_param = self.ctx.tensor(b.param_off, b.numel, b.dtype)
            for p, st in zip(b.params, b.starts):
                gv = _strided_view(b.flat_grad, p, st)
                if p.grad is not None:
                    gv.copy_(p.grad)
                p.grad = gv
                self._grad_views[p] = gv
                self._param_bucket[p] = b
                self._delay[p] = self.bpps
                if fused:
                    pv = _strided_view(b.flat_param, p, st)
                    pv.copy_(p.data)
                    p.data = pv
            b.pending = len(b.params)
        if fused:
            self._init_fused_state()
        if self.loss_scaler is not None:
            self._init_loss_scaler()
        if max_grad_norm is not None:
            self._init_clip()
        self._next = 0          # strict mode: next bucket index allowed to launch
        self._strict = os.environ.get("BYTEPS_STRICT_ORDER", "0") not in ("0", "")
        self._hooks = []
        self._step = 0
        self._hp_dirty = True
        self._seg_tables: Dict[int, torch.Tensor] = {}
        self._last_done = None
        self._trace_t0 = None
        self._trace_spans = []
        # which engine moves the NVLink bytes of plain (unfused) buckets:
        #   auto/nvls: multimem.ld_reduce/st when available, else LSU P2P; lsu: force P2P loads/stores;
        #   tma: cp.async.bulk ring; wgmma: TMA + tensor-core reduction with a register accumulator
        self._reduce_engine = reduce_engine
        # fused optimizer kernels: "tma" streams the fp32 state through shared memory with bulk copies,
        # "lsu" keeps it in registers (also used whenever the gradients need a wire cast)
        self._fused_engine = os.environ.get("BYTEPS_FUSED_ENGINE", "auto").lower()
        if self._fused_engine == "auto":
            # the TMA kernel keeps more bytes in flight per SM (shared-memory ring instead of registers) and runs
            # solo; the register kernel stays the multi-GPU default and handles every wire cast
            self._fused_engine = "tma" if self.world == 1 else "lsu"
        # CTAs of the TMA variant: its bytes in flight live in shared memory, so a fraction of the SMs
        # saturates HBM/NVLink and the rest stays free for the backward kernels it overlaps with
        self._fused_tma_blocks = _env_int("BYTEPS_FUSED_TMA_BLOCKS", 128)
        self._umma_maps = {}
        self._xlaunches = 0
        self._last_step_launches = 0
        self._priority_of = priority_of or {}
        for b in self.buckets:
            b.priority = max([int(self._priority_of.get(p, 0)) for p in b.params] or [0])
        self._setup_ring()
        self.enabled = True            # DDP.no_sync() turns hooks into local accumulation
        self.auto_finish = None        # DDP: called when every bucket of the iteration was launched
        self._launched = 0
        self._register_hooks()
        _LIVE.add(self)
        torch.cuda.current_stream(self.device).synchronize()
        if self.world > 1:
            engine.group.barrier()
        stamp("buckets: views, fused state, hooks")

    # ------------------------------------------------------------------ layout helpers
    def _wire(self, b: Bucket) -> torch.dtype:
        w = self.wire_override
        if w is not None and b.dtype == torch.float32 and w in (torch.bfloat16, torch.float16):
            return w
        return b.dtype

    def _wire_bytes(self, b: Bucket) -> int:
        return b.numel * torch.empty((), dtype=self._wire(b)).element_size()

    def _needs_stage(self) -> bool:
        return any(self._wire(b) != b.dtype for b in self.buckets)

    def shard_range(self, b: Bucket):
        """Element range [begin, end) of the shard this rank owns in bucket b."""
        return shard_bounds(b.numel, self.world, self.rank)

    # ------------------------------------------------------------------ fused optimizer state
    def _init_fused_state(self):
        kind = self.fused
        for b in self.buckets:
            s0, s1 = self.shard_range(b)
            n = max(s1 - s0, 8)
            b.master = torch.zeros(n, dtype=torch.float32, device=self.device)
            b.master[: s1 - s0].copy_(b.flat_param[s0:s1].float())
            b.state0 = torch.zeros(n, dtype=torch.float32, device=self.device)
            b.state1 = torch.zeros(n, dtype=torch.float32, device=self.device) if kind not in ("sgd", "lars") else None
        ng = len(self.param_groups)
        self._hp_dev = torch.zeros((ng, 64), dtype=torch.uint8, device=self.device)
        self._group_step = [0] * ng      # steps run (with dynamic loss scaling: attempted, skipped ones included)
        self.loss_scale = 1.0
        if kind in _TRUST_KINDS:
            self._init_lamb()

    def _init_lamb(self):
        """The device memory of a trust-ratio optimizer (LAMB, LARS) besides its SGD or Adam state: a (start, numel)
        table per bucket, the float64 scratch of the partial norms and one float trust ratio per parameter.  The
        buckets of a step run in order on the comm stream, so the scratch and the ratios of the largest bucket serve
        them all."""
        cu = self.ctx.cu
        # loaded before any launch that spins on a peer (DESIGN 1.6)
        if self.fused == "lamb":
            cu.lamb_load_kernels()
        else:
            cu.lars_load_kernels()
        self._build_param_tables()
        nmax = max(len(b.params) for b in self.buckets)
        shard_max = max(s1 - s0 for s0, s1 in map(self.shard_range, self.buckets))
        self._lamb_scratch = torch.zeros(cu.lamb_scratch_bytes(shard_max, nmax) // 8, dtype=torch.float64,
                                         device=self.device)
        self._lamb_phi = torch.ones(nmax, dtype=torch.float32, device=self.device)

    def _build_param_tables(self):
        """Every bucket's (start, numel) table on the device: the parameter cursor of the norm kernels keeps padding
        out of every norm with it."""
        for b in self.buckets:
            if b.lamb_params is None:
                b.lamb_params = torch.tensor([[st, p.numel()] for p, st in zip(b.params, b.starts)],
                                             dtype=torch.int64, device=self.device)

    def lamb_device_bytes(self) -> int:
        """Device bytes fused LAMB adds to fused Adam, or fused LARS to fused SGD, on this rank: tables, scratch,
        trust ratios, norm windows."""
        if self.fused not in _TRUST_KINDS:
            return 0
        windows = sum(self.ctx.cu.lamb_window_bytes(len(b.params), self.world) for b in self.buckets)
        return (sum(b.lamb_params.nbytes for b in self.buckets) + self._lamb_scratch.nbytes + self._lamb_phi.nbytes
                + windows)

    # ------------------------------------------------------------------ gradient clipping (fused mode)
    def _init_clip(self):
        """Device state of global gradient-norm clipping: the (start, numel) tables, one float64 scratch row per bucket
        (one entry per CTA of its norm pass; entries no CTA writes stay zero and add nothing), the total norm and
        the agreement window."""
        cu = self.ctx.cu
        cu.clip_load_kernels()           # loaded before any launch that spins on a peer (DESIGN 1.6)
        self._build_param_tables()
        row = max(self._blocks(b) for b in self.buckets)
        self._clip_scratch = torch.zeros((len(self.buckets), row), dtype=torch.float64, device=self.device)
        self._grad_norm = torch.zeros((), dtype=torch.float32, device=self.device)
        self.ctx.tensor(self.clip_win_off, 256, torch.uint8).zero_()

    def grad_norm_tensor(self) -> torch.Tensor:
        """0-dim float32 device tensor: the last step's total gradient norm before clipping, written by the kernels
        (so also by every replay of a captured step)."""
        return self._grad_norm

    def clip_device_bytes(self) -> int:
        """Device bytes clipping adds on this rank: the (start, numel) tables (unless LAMB or LARS has them anyway),
        the scratch rows, the total norm and the agreement window."""
        if self.max_grad_norm is None:
            return 0
        tables = 0 if self.fused in _TRUST_KINDS else sum(b.lamb_params.nbytes for b in self.buckets)
        return tables + self._clip_scratch.nbytes + self._grad_norm.nbytes + self.ctx.cu.CLIP_WINDOW_BYTES

    def _launch_norm(self, b: Bucket, wait: bool = True):
        """The norm pass of bucket b on the comm stream (clip_norm_partial): this rank's shard of the reduced gradient,
        one float64 sum of squares per CTA into the bucket's scratch row."""
        cu = self.ctx.cu
        cs = self.comm_stream
        if wait:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.device))
            cs.wait_event(ev)
        wire = self._wire(b)
        if wire == b.dtype:
            segs, nsegs, stage = 0, 0, b.grad_off
        else:
            segs, nsegs, stage = self._seg_table(b).data_ptr(), 1, self.stage_off
        scale = (1.0 / self.world) if self.average else 1.0
        row = self._clip_scratch[b.index].data_ptr()
        cu.clip_norm_partial(self.ctx.view, wire_code(b.dtype), wire_code(wire), segs, nsegs, stage, b.numel, scale,
                             b.lamb_params.data_ptr(), len(b.params), row, self._hp_dev.data_ptr() + 64 * b.group_index,
                             self._blocks(b), self.threads, 0, self._nvls_for(wire), cs.cuda_stream)
        b.normed = True
        self._count_launch()

    # ------------------------------------------------------------------ dynamic loss scaling (fused mode)
    def _init_loss_scaler(self):
        """Device state of dynamic loss scaling: the scaler (LossScaleState), the applied-step count of every param
        group, the float64 Adam betas the device forms the bias corrections from, and the check table, one entry
        (gradient window, length, gradient dtype, wire dtype) per bucket."""
        cu = self.ctx.cu
        cu.loss_scale_load_kernels()     # loaded before any launch that spins on a peer (DESIGN 1.6)
        ng = len(self.param_groups)
        self._ls_state = torch.zeros(cu.LOSS_SCALE_STATE_BYTES, dtype=torch.uint8, device=self.device)
        self._ls_steps = torch.zeros(ng, dtype=torch.int32, device=self.device)
        self._ls_betas = torch.zeros((ng, 2), dtype=torch.float64, device=self.device)
        blob = b"".join(struct.pack(_LS_ENTRY_FMT, b.grad_off, b.numel, wire_code(b.dtype), wire_code(self._wire(b)),
                                    0, 0) for b in self.buckets)
        self._ls_table = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(self.device)
        self._ls_max_vectors = max(b.nbytes // 16 for b in self.buckets)
        self.ctx.tensor(self.ls_win_off, 256, torch.uint8).zero_()
        self.reset_loss_scaler()

    def reset_loss_scaler(self):
        """Scaler back to its initial values: scale = init_scale, growth tracker and skipped count 0."""
        c = self.loss_scaler
        self.set_loss_scaler_state(c["init_scale"], c["growth_factor"], c["backoff_factor"], c["growth_interval"], 0,
                                   skipped=0)

    def set_loss_scaler_state(self, scale, growth_factor, backoff_factor, growth_interval, growth_tracker,
                              skipped=None):
        """Install a scaler state (GradScaler.state_dict()'s values); skipped=None keeps the skipped count."""
        if skipped is None:
            skipped = self.loss_scaler_state()["skipped"]
        vals = (float(growth_factor), float(backoff_factor), float(scale), int(growth_interval), int(growth_tracker),
                int(skipped), 0, 0)
        self._ls_state.copy_(torch.frombuffer(bytearray(struct.pack(_LS_STATE_FMT, *vals)), dtype=torch.uint8))

    def loss_scaler_state(self) -> Dict:
        """The scaler as the device holds it: scale, growth_factor, backoff_factor, growth_interval, tracker,
        skipped, and steps (applied steps per group).  Synchronises with the current stream, which every step's
        synchronize() has made wait for the exchanges."""
        raw = self._ls_state.cpu().numpy().tobytes()
        growth, backoff, scale, interval, tracker, skipped, _, _ = struct.unpack(_LS_STATE_FMT, raw)
        return {"scale": scale, "growth_factor": growth, "backoff_factor": backoff, "growth_interval": interval,
                "tracker": tracker, "skipped": skipped, "steps": self._ls_steps.tolist()}

    def scale_tensor(self) -> torch.Tensor:
        """0-dim float32 view of the device scale S (what the coming step's loss is multiplied by)."""
        return self._ls_state[16:20].view(torch.float32)[0]

    def applied_steps(self) -> List[int]:
        """Steps the optimizer has applied per param group: with dynamic loss scaling the device's count (skipped
        steps excluded; synchronises), otherwise the steps run."""
        if self.loss_scaler is not None:
            return self._ls_steps.tolist()
        return list(self._group_step)

    def sync_master_from_params(self):
        for b in self.buckets:
            s0, s1 = self.shard_range(b)
            b.master[: s1 - s0].copy_(b.flat_param[s0:s1].float())

    def step_done(self):
        """Eager mode, end of optimizer.step(): count the step and publish the
        hyper-parameters of the next one."""
        if not self.fused or torch.cuda.is_current_stream_capturing():
            return
        for gi in range(len(self._group_step)):
            self._group_step[gi] += 1
        self.refresh_hparams()

    def pre_replay(self):
        """CUDA-graph mode, before every replay: publish the hyper-parameters of
        the step about to run, then count it."""
        if not self.fused:
            return
        self.refresh_hparams()
        for gi in range(len(self._group_step)):
            self._group_step[gi] += 1

    def refresh_hparams(self):
        """Send the param-group hyper-parameters (lr, momentum, Adam bias
        corrections, ...) of the NEXT step to the device block the fused kernels
        read.  The values ride in the argument space of a tiny kernel on the
        current stream, so they are ordered before the next exchange kernels and
        a captured CUDA graph sees fresh values on every replay."""
        if not self.fused:
            return
        cur = torch.cuda.current_stream(self.device)
        if torch.cuda.is_current_stream_capturing():
            return   # replays are fed from outside the graph
        blob = b""
        for gi, g in enumerate(self.param_groups):
            t = self._group_step[gi] + 1     # the step that is about to run
            if self.fused == "sgd":
                vals = (float(g.get("lr", 0.0)), float(g.get("weight_decay", 0.0)), float(g.get("momentum", 0.0)),
                        float(g.get("dampening", 0.0)), 0.0, 0.0, 0.0, 1.0, 1.0,
                        int(bool(g.get("nesterov", False))), 0, int(t == 1), 1.0 / self.loss_scale, 0, 0, 0.0)
            elif self.fused == "lars":
                vals = (float(g.get("lr", 0.0)), float(g.get("weight_decay", 0.0)), float(g.get("momentum", 0.0)),
                        0.0, 0.0, 0.0, float(g.get("eps", 0.0)), 1.0, 1.0, 0, 0, int(t == 1), 1.0 / self.loss_scale,
                        0, int(bool(g.get("adapt", True))), float(g.get("trust_coefficient", 0.001)))
            else:
                b1, b2 = g.get("betas", (0.9, 0.999))
                adapt = int(bool(g.get("adapt", True))) if self.fused == "lamb" else 0
                vals = (float(g.get("lr", 0.0)), float(g.get("weight_decay", 0.0)), 0.0, 0.0, float(b1), float(b2),
                        float(g.get("eps", 1e-8)), 1.0 - b1 ** t, 1.0 - b2 ** t, 0,
                        int(self.fused == "adamw"), int(t == 1), 1.0 / self.loss_scale, 0, adapt, 0.0)
            blob += struct.pack(_HP_FMT, *vals)
        self.ctx.cu.write_blob(self._hp_dev.data_ptr(), blob, cur.cuda_stream)
        self.engine.launches += 1
        if self.loss_scaler is not None and self.fused not in ("sgd", "lars"):
            # loss_scale_update forms Adam's bias corrections on the device, from the betas as the host holds them
            betas = b"".join(struct.pack("<2d", *map(float, g.get("betas", (0.9, 0.999)))) for g in self.param_groups)
            self.ctx.cu.write_blob(self._ls_betas.data_ptr(), betas, cur.cuda_stream)
            self.engine.launches += 1

    # ------------------------------------------------------------------ hooks
    def _register_hooks(self):
        for b in self.buckets:
            for p in b.params:
                self._hooks.append(p.register_post_accumulate_grad_hook(self._make_hook(p)))

    def _make_hook(self, p):
        def hook(param):
            if not self.enabled:
                return
            self._delay[p] -= 1
            if self._delay[p] > 0:
                return
            if self._delay[p] < 0:
                raise AssertionError(
                    "Gradients were computed more than backward_passes_per_step times before call to step(). "
                    "Increase backward_passes_per_step to accumulate gradients locally.")
            gv = self._grad_views[p]
            if p.grad is not gv:
                # someone replaced .grad (e.g. zero_grad(set_to_none=True)): fold it back into the arena
                if p.grad is not None and p.grad.data_ptr() != gv.data_ptr():
                    gv.copy_(p.grad)
                p.grad = gv
            b = self._param_bucket[p]
            b.pending -= 1
            if b.pending == 0 and self.loss_scaler is None:   # dynamic loss scaling: launched at the step
                if self.max_grad_norm is None:
                    self._launch_ready(b)
                elif not self._strict:
                    self._launch_norm(b)        # clipping: the norm pass now, the exchange at the step
        return hook

    def set_backward_passes_per_step(self, n: int):
        self.bpps = n
        for p in self._delay:
            self._delay[p] = n

    # ------------------------------------------------------------------ launching
    def _launch_ready(self, b: Optional[Bucket] = None):
        """Launch a bucket whose gradients are complete.  By default buckets go
        out in completion order - identical on every rank because autograd
        executes the same graph in the same order (the assumption DDP also
        makes); BYTEPS_STRICT_ORDER=1 forces creation order instead."""
        if b is not None and not self._strict:
            if not b.launched:
                self._issue(b)
            return
        while self._next < len(self.buckets) and self.buckets[self._next].pending == 0:
            if not self.buckets[self._next].launched:
                self._issue(self.buckets[self._next])
            self._next += 1

    def _issue(self, b: Bucket):
        if self._ring_mode == "off" or b.ring_cls is None:
            self._ring_flush()          # keep the comm stream in issue order
            self._launch(b)
        elif self._ring_mode == "persistent" and self._step >= self._ring_persistent_after:
            self._ring_persistent_ready(b)
        else:
            self._ring_enqueue(b)

    def _nvls_for(self, wire: torch.dtype) -> bool:
        """Whether exchanges on this wire dtype use the in-switch (NVLS) reduction.  Not for an fp16 wire under dynamic
        loss scaling: multimem.ld_reduce returns the rank sum in fp16, where values the overflow check passed can add
        up to inf; the peer-load path sums them in fp32 registers instead (see loss_scale.cuh)."""
        return bool(self.ctx.nvls) and not (self.loss_scaler is not None and wire == torch.float16)

    def _seg_table(self, b: Bucket) -> torch.Tensor:
        t = self._seg_tables.get(b.index)
        if t is None:
            ptr = b.flat_grad.data_ptr()
            t = torch.tensor([[ptr, ptr, 0, b.numel]], dtype=torch.int64, device=self.device)
            self._seg_tables[b.index] = t
        return t

    def _blocks(self, b: Bucket) -> int:
        """CTAs of bucket b's exchange (and norm pass): a function of the bucket, the same on every rank."""
        shard = (self._wire_bytes(b) + self.world - 1) // self.world
        return self.engine.cfg.comm_blocks or pick_blocks(shard, self.threads, 32, cap=64)

    def _launch(self, b: Bucket):
        cu = self.ctx.cu
        view = self.ctx.view
        cur = torch.cuda.current_stream(self.device)
        tracing = (self.engine.timeline.enabled() and self.engine.timeline.active(self._step)
                   and not torch.cuda.is_current_stream_capturing())
        ev = torch.cuda.Event(enable_timing=tracing)
        ev.record(cur)
        cs = self.comm_stream
        cs.wait_event(ev)
        ev_t = None
        if tracing:
            ev_t = torch.cuda.Event(enable_timing=True)
            ev_t.record(cs)
        wire = self._wire(b)
        world = self.world
        scale = (1.0 / world) if self.average else 1.0
        shard = (self._wire_bytes(b) + world - 1) // world
        blocks = self._blocks(b)
        nvls = self._nvls_for(wire)
        if self.fused in _TRUST_KINDS:
            self._launch_trust(b, wire, scale, blocks, nvls, cs)
            self._after_launch(b, cur, cs, ev_t)
            return
        if self.fused:
            kind = cu.OPT_SGD if self.fused == "sgd" else cu.OPT_ADAM
            hp_ptr = self._hp_dev.data_ptr() + 64 * b.group_index
            if wire == b.dtype and self._fused_engine == "tma":
                # optimizer state streamed through shared memory with bulk copies (pushpull.cu, TMA variant)
                es = 4 if b.dtype == torch.float32 else 2
                per_stage = (2 if kind == cu.OPT_SGD else 3) * 256 * (16 // es) * 4
                stages = max(2, min(8, (96 << 10) // per_stage))
                shard_units = (shard + 15) // 16
                cap = self._fused_tma_blocks
                tblocks = self.engine.cfg.comm_blocks or max(1, min(cap, (shard_units + 255) // 256))
                cu.pushpull_fused_opt_tma(view, wire_code(wire), kind, b.grad_off, b.param_off, b.numel, scale,
                                          b.master.data_ptr(), b.state0.data_ptr(),
                                          b.state1.data_ptr() if b.state1 is not None else 0, hp_ptr, tblocks, stages,
                                          nvls, 0, cs.cuda_stream)
                self._after_launch(b, cur, cs, ev_t)
                return
            if wire == b.dtype:
                segs, nsegs, stage = 0, 0, b.grad_off
            else:
                segs, nsegs, stage = self._seg_table(b).data_ptr(), 1, self.stage_off
            cu.pushpull_fused_opt(view, wire_code(b.dtype), wire_code(wire), wire_code(b.dtype), kind, segs, nsegs,
                                  stage, b.param_off, b.numel, scale, b.master.data_ptr(), b.state0.data_ptr(),
                                  b.state1.data_ptr() if b.state1 is not None else 0, hp_ptr, blocks, self.threads, 0,
                                  nvls, cs.cuda_stream)
        elif wire == b.dtype:
            eng_kind = self._reduce_engine
            if eng_kind == "wgmma" and b.dtype in (torch.bfloat16, torch.float16) and world <= 8:
                # tensor-core reduction: TMA-fed [I|..|I] x [X_0;..;X_{P-1}] accumulated in registers
                maps = self._umma_maps.get(b.index)
                if maps is None:
                    maps = cu.make_umma_maps(view, wire_code(wire), b.grad_off, b.numel)
                    self._umma_maps[b.index] = maps
                ublocks = max(1, min(64, (shard + 16383) // 16384))
                cu.pushpull_inplace_umma(view, maps, wire_code(wire), b.grad_off, b.numel, scale, ublocks, 0,
                                         cs.cuda_stream)
            elif eng_kind == "tma":
                tblocks = pick_blocks(shard, 256, 16, cap=64)
                cu.pushpull_inplace_tma(view, wire_code(wire), b.grad_off, b.numel, scale, tblocks, 4, 0,
                                        cs.cuda_stream)
            else:
                cu.pushpull_inplace(view, wire_code(wire), b.grad_off, b.numel, scale, blocks, self.threads, 0,
                                    nvls and eng_kind != "lsu", cs.cuda_stream)
        else:
            cu.pushpull_packed(view, wire_code(b.dtype), wire_code(wire), self._seg_table(b).data_ptr(), 1,
                               self.stage_off, b.numel, scale, blocks, self.threads, 0, nvls, False, True,
                               cs.cuda_stream)
        self._after_launch(b, cur, cs, ev_t)

    def _launch_trust(self, b: Bucket, wire, scale, blocks, nvls, cs):
        """LAMB and LARS: three kernels per bucket.  LAMB (pushpull_lamb.cuh): lamb_moments reduces this rank's shard,
        updates the moments and sums w^2 and u^2 per parameter; lamb_norms trades those sums with the peers and forms
        the trust ratios; lamb_apply updates the masters and all-gathers the parameters.  LARS (pushpull_lars.cuh):
        lars_norms_partial reduces the shard and sums w^2 and g^2; lars_norms forms the ratios as lamb_norms does;
        lars_apply reduces the shard again, updates the momentum and the masters and all-gathers the parameters.  The
        grids depend on the bucket only."""
        cu = self.ctx.cu
        if wire == b.dtype:
            segs, nsegs, stage = 0, 0, b.grad_off
        else:
            segs, nsegs, stage = self._seg_table(b).data_ptr(), 1, self.stage_off
        hp = self._hp_dev.data_ptr() + 64 * b.group_index
        n, table = len(b.params), b.lamb_params.data_ptr()
        scratch, phi = self._lamb_scratch.data_ptr(), self._lamb_phi.data_ptr()
        g, w = wire_code(b.dtype), wire_code(wire)
        if self.fused == "lars":
            cu.lars_norms_partial(self.ctx.view, g, w, segs, nsegs, stage, b.numel, scale, b.master.data_ptr(), table, n,
                                  scratch, hp, blocks, self.threads, 0, nvls, cs.cuda_stream)
            cu.lars_norms(self.ctx.view, w, b.numel, table, n, scratch, b.lamb_win_off, phi, hp, min(n, 32), 0,
                          cs.cuda_stream)
            cu.lars_apply(self.ctx.view, g, w, stage, b.param_off, b.numel, scale, b.master.data_ptr(),
                          b.state0.data_ptr(), table, n, phi, hp, blocks, self.threads, 0, nvls, cs.cuda_stream)
            self._count_launch(2)        # _after_launch counts the third
            return
        cu.lamb_moments(self.ctx.view, g, w, segs, nsegs, stage, b.numel, scale, b.master.data_ptr(),
                        b.state0.data_ptr(), b.state1.data_ptr(), table, n, scratch, hp, blocks, self.threads, 0, nvls,
                        cs.cuda_stream)
        cu.lamb_norms(self.ctx.view, w, b.numel, table, n, scratch, b.lamb_win_off, phi, hp, min(n, 32), 0,
                      cs.cuda_stream)
        cu.lamb_apply(self.ctx.view, g, w, b.param_off, b.numel, b.master.data_ptr(), b.state0.data_ptr(),
                      b.state1.data_ptr(), table, n, phi, hp, blocks, self.threads, 0, nvls, cs.cuda_stream)
        self._count_launch(2)            # _after_launch counts the third

    # ------------------------------------------------------------------ descriptor ring
    def _setup_ring(self):
        """BYTEPS_RING: how bucket exchanges reach the GPU.

        off         one kernel per bucket (two cross-rank barriers each);
        batch       buckets that became ready are handed to ONE descriptor-ring launch per flush window
                    (BYTEPS_RING_BATCH_BYTES, or the end of backward): flags instead of barriers, no
                    launch gaps, CTAs flow from one bucket into the next;
        persistent  one ring launch per step (per dtype class), issued when the first bucket is ready;
                    later buckets are announced by a `ring_mark` on the autograd stream.
        With BYTEPS_SCHEDULING_CREDIT > 0 the ring's root scheduler picks the ready bucket with the
        highest priority inside a byte-credit window (reference: scheduled_queue.cc:82-163)."""
        from ..ops.ring import RingEntry, RingTable

        cu = self.ctx.cu
        mode = os.environ.get("BYTEPS_RING", "auto").lower()
        if mode in ("0", "no", "false"):
            mode = "off"
        if mode in ("1", "yes", "true", "on"):
            mode = "batch"
        self._ring_tables = {}
        self._ring_pending: List[Bucket] = []
        self._ring_pending_bytes = 0
        self._ring_started = False
        self._ring_batch_bytes = _env_int("BYTEPS_RING_BATCH_BYTES", 64 << 20)
        # persistent launches spin while backward is still producing gradients.  CUDA loads kernels lazily and
        # a first-time load can wait for running kernels, so the first steps (which load cuDNN/cuBLAS/ATen
        # kernels) go through the batch path; the same step count on every rank keeps launches aligned.
        self._ring_persistent_after = _env_int("BYTEPS_RING_PERSISTENT_AFTER", 2)
        self._ring_blocks = _env_int("BYTEPS_RING_BLOCKS", 0)
        credit = self.engine.cfg.scheduling_credit
        self._ring_sched = credit > 0
        self._ring_credit = credit * self.engine.cfg.partition_bound() if credit > 0 else 0
        self._stamps = os.environ.get("BYTEPS_COMM_STAMPS", "1") not in ("0", "")
        self._stamp_base = None
        # LAMB and LARS need every rank's partial norms between the reduction and the update: per-bucket launches only
        eligible = (self._reduce_engine in ("auto", "nvls", "lsu") and len(self.buckets) <= cu.RING_SLOTS
                    and self.fused not in _TRUST_KINDS
                    and not (self.fused and self._fused_engine == "tma" and self.world == 1 and mode == "auto"))
        if mode == "auto":
            # one rank: nothing to wait for, the TMA-streamed optimizer kernel per bucket is the fastest;
            # several ranks: the ring removes two NVLink barrier round trips and a launch per bucket
            mode = "batch" if (self.world > 1 and eligible) else "off"
        if mode != "off" and not eligible:
            mode = "off"
        if mode == "persistent" and (self.loss_scaler is not None or self.max_grad_norm is not None):
            mode = "batch"      # every exchange waits for a decision at the step (overflow, norm): nothing to start early
        self._ring_mode = mode
        if mode == "off":
            return
        kind = {None: cu.RING_ALLREDUCE, "sgd": cu.RING_SGD}.get(self.fused, cu.RING_ADAM)
        scale = (1.0 / self.world) if self.average else 1.0
        by_cls = {}
        for b in self.buckets:
            if self._wire(b) != b.dtype:
                continue            # needs a wire cast: stays on the per-bucket packed kernel
            cls = (wire_code(b.dtype), kind)
            by_cls.setdefault(cls, []).append(b)
        for cls, bs in by_cls.items():
            entries = []
            for pos, b in enumerate(bs):
                b.ring_cls, b.ring_pos = cls, pos
                entries.append(RingEntry(
                    grad_off=b.grad_off, param_off=max(b.param_off, 0), numel=b.numel, wire=cls[0], slot=b.index,
                    kind=kind, scale=scale, priority=b.priority,
                    master=b.master.data_ptr() if b.master is not None else 0,
                    state0=b.state0.data_ptr() if b.state0 is not None else 0,
                    state1=b.state1.data_ptr() if b.state1 is not None else 0,
                    hp=(self._hp_dev.data_ptr() + 64 * b.group_index) if self.fused else 0))
            self._ring_tables[cls] = (RingTable(entries, self.device), bs)

    def _ring_grid(self, nbytes: int) -> int:
        if self._ring_blocks:
            return self._ring_blocks
        if self.engine.cfg.comm_blocks:
            return self.engine.cfg.comm_blocks
        shard = (nbytes + self.world - 1) // self.world
        return pick_blocks(shard, 512, 32, cap=64 if self._ring_mode == "batch" else 24)

    def _ring_enqueue(self, b: Bucket):
        """batch mode: remember the bucket; flush when enough bytes are waiting."""
        self._ring_pending.append(b)
        self._ring_pending_bytes += b.nbytes
        b.launched = True
        self._launched += 1
        if self._ring_pending_bytes >= self._ring_batch_bytes:
            self._ring_flush()
        elif self.auto_finish is not None and self._launched == len(self.buckets):
            self._ring_flush()
            self.auto_finish()

    def _ring_flush(self):
        """One ring launch per run of pending buckets that are consecutive in their class table."""
        pend = self._ring_pending
        if not pend:
            return
        self._ring_pending = []
        self._ring_pending_bytes = 0
        cur = torch.cuda.current_stream(self.device)
        cs = self.comm_stream
        ev = torch.cuda.Event()
        ev.record(cur)
        cs.wait_event(ev)
        i = 0
        while i < len(pend):
            b0 = pend[i]
            nvls = self._nvls_for(self._wire(b0)) and self._reduce_engine != "lsu"
            j = i + 1
            while (j < len(pend) and pend[j].ring_cls == b0.ring_cls
                   and pend[j].ring_pos == pend[j - 1].ring_pos + 1):
                j += 1
            table, _ = self._ring_tables[b0.ring_cls]
            nbytes = sum(x.nbytes for x in pend[i:j])
            table.launch(self.ctx.view, self._ring_grid(nbytes // max(1, j - i)), cs.cuda_stream, nvls=nvls,
                         sched=self._ring_sched and j - i > 1, self_mark=True, credit_bytes=self._ring_credit,
                         first=b0.ring_pos, count=j - i)
            self._count_launch()
            i = j
        done = torch.cuda.Event()
        done.record(cs)
        for b in pend:
            b.done = done
            if self.engine.telemetry.should_record():
                self.engine.telemetry.record(b.nbytes)
        self._last_done = done
        self._ring_traced = True

    def _ring_persistent_ready(self, b: Bucket):
        """persistent mode: the first ready bucket of a step starts one ring launch per class (they
        consume their tables in order and wait on flags); every ready bucket is announced by a mark
        kernel on the producing stream."""
        cur = torch.cuda.current_stream(self.device)
        cs = self.comm_stream
        self.ctx.cu.ring_mark(self.ctx.view, [b.index], cur.cuda_stream)
        self._count_launch()
        if not self._ring_started:
            self._ring_started = True
            ev = torch.cuda.Event()
            ev.record(cur)
            cs.wait_event(ev)
            nvls = bool(self.ctx.nvls) and self._reduce_engine != "lsu"
            for cls, (table, bs) in self._ring_tables.items():
                nbytes = sum(x.nbytes for x in bs) // len(bs)
                table.launch(self.ctx.view, self._ring_grid(nbytes), cs.cuda_stream, nvls=nvls,
                             sched=self._ring_sched and len(bs) > 1, self_mark=False,
                             credit_bytes=self._ring_credit)
                self._count_launch()
            done = torch.cuda.Event()
            done.record(cs)
            self._last_done = done
            for x in self.buckets:
                if x.ring_cls is not None:
                    x.done = done
        if self.engine.telemetry.should_record():
            self.engine.telemetry.record(b.nbytes)
        b.launched = True
        self._launched += 1
        self._ring_traced = True
        if self.auto_finish is not None and self._launched == len(self.buckets):
            self.auto_finish()

    def exposed_comm_ms(self) -> Optional[float]:
        """Device-measured communication time that was NOT hidden behind the backward pass in the
        last step: (comm stream idle after the last exchange) - (autograd stream reached
        optimizer.step), both stamped with the GPU's globaltimer by one-thread kernels, so the
        figure also exists for CUDA-graph replays.  None before the first step."""
        if not self._stamps:
            return None
        torch.cuda.synchronize(self.device)
        _, stamps = self.ctx.cu.ring_trace(self.ctx.view, [])
        if stamps[0] == 0 or stamps[1] == 0:
            return None
        return max(0.0, (stamps[1] - stamps[0]) / 1e6)

    def ring_spans(self):
        """[(bucket index, order position, start ns, end ns)] of the last ring launches (globaltimer)."""
        torch.cuda.synchronize(self.device)
        idx = [b.index for b in self.buckets if b.ring_cls is not None]
        rows, _ = self.ctx.cu.ring_trace(self.ctx.view, idx)
        return [(i, pos, t0, t1) for i, (pos, t0, t1) in zip(idx, rows)]

    def _count_launch(self, n: int = 1):
        self.engine.launches += n
        self._xlaunches += n

    def launches_per_step(self) -> int:
        """Kernels of ours (exchange launches + marks) the last completed step issued; what one
        CUDA-graph replay of that step launches."""
        return self._last_step_launches

    def _after_launch(self, b: Bucket, cur, cs, ev_t):
        self._count_launch()
        if self.engine.telemetry.should_record():
            self.engine.telemetry.record(b.nbytes)
        tl = self.engine.timeline
        if tl.enabled() and tl.active(self._step) and not torch.cuda.is_current_stream_capturing():
            # device-timed span of this bucket's exchange (the reference's timeline uses host wall-clock)
            if self._trace_t0 is None:
                self._trace_t0 = (torch.cuda.Event(enable_timing=True), self.engine.core.now_us())
                self._trace_t0[0].record(cur)
            b.done = torch.cuda.Event(enable_timing=True)
            b.done.record(cs)
            self._trace_spans.append((b, ev_t, b.done))
        else:
            b.done = torch.cuda.Event()
            b.done.record(cs)
        b.launched = True
        self._last_done = b.done
        self._launched += 1
        if self.auto_finish is not None and self._launched == len(self.buckets):
            self.auto_finish()

    def synchronize(self):
        """Issue whatever has not been launched (unused parameters) and make the
        current stream wait for every bucket of this step."""
        cur = torch.cuda.current_stream(self.device)
        if self._stamps:
            self.ctx.cu.ring_stamp(self.ctx.view, 0, cur.cuda_stream)       # backward (and everything before) done
            self._count_launch()
        self._issue_remaining()
        if self._stamps and self._last_done is not None:
            self.ctx.cu.ring_stamp(self.ctx.view, 1, self.comm_stream.cuda_stream)   # last exchange finished
            self._count_launch()
            self._last_done = torch.cuda.Event()
            self._last_done.record(self.comm_stream)
        if self._last_done is not None:
            # the comm stream executes in order: the most recent event covers every bucket
            torch.cuda.current_stream(self.device).wait_event(self._last_done)
            self._last_done = None
        self._reset()

    def _zero_unused(self, b: Bucket):
        """A parameter whose hook did not fire in this iteration contributes zeros (like a fresh zero gradient in the
        reference), not whatever an earlier iteration left in its arena window - `model.zero_grad()` only drops the
        `.grad` references, it does not clear the arena."""
        for p in b.params:
            if self._delay.get(p) == self.bpps:
                self._grad_views[p].zero_()

    def _issue_remaining(self):
        """Issue every bucket that has not gone out yet (unused parameters), in index order on every rank."""
        if self.loss_scaler is not None or self.max_grad_norm is not None:
            self._issue_deferred_step()
            return
        for b in self.buckets:
            if not b.launched:
                self._zero_unused(b)
                b.pending = 0
                self._issue(b)
        self._ring_flush()

    def _issue_deferred_step(self):
        """Dynamic loss scaling and gradient clipping: the exchanges of the step, issued at the step on the comm
        stream, after a decision every rank takes on the device.

        1. dynamic loss scaling: loss_scale_check (does any element of this rank's gradient windows overflow on its
           wire?) and loss_scale_update (every rank learns every rank's flag by barrier_peers and an OR in rank
           order, updates the scale, counts the step per group if it is applied, and writes grad_scale = 1/S, skip,
           first_step and the Adam bias corrections into the hyper-parameter blocks, over what refresh_hparams put
           there).
        2. clipping: clip_norm_partial for every bucket whose hook has not launched it during backward (all of them
           with loss scaling, which must unscale first), in bucket order; then clip_norm_update, which sums the
           squares over every bucket and rank, writes the norm and multiplies every group's grad_scale by
           min(1, max_grad_norm / (norm + 1e-6)).  grad_scale is rewritten before every step (refresh_hparams,
           pre_replay or loss_scale_update), so the coefficient never compounds.
        3. every bucket's fused exchange in bucket order: one ring flush (BYTEPS_RING=batch, and persistent, which
           behaves as batch here) or one launch per bucket; a skipped step leaves the optimizer state as it is.
        No exchange went out during backward, so the update no longer overlaps with it."""
        for b in self.buckets:
            if not b.launched:
                self._zero_unused(b)
                b.pending = 0
        cu = self.ctx.cu
        cur = torch.cuda.current_stream(self.device)
        cs = self.comm_stream
        ev = torch.cuda.Event()
        ev.record(cur)
        cs.wait_event(ev)
        if self.loss_scaler is not None:
            state = self._ls_state.data_ptr()
            cu.loss_scale_check(self.ctx.view, self._ls_table.data_ptr(), len(self.buckets), self._ls_max_vectors,
                                state, cs.cuda_stream)
            cu.loss_scale_update(self.ctx.view, 0, self.ls_win_off, state, self._ls_steps.data_ptr(),
                                 self._ls_betas.data_ptr(), self._hp_dev.data_ptr(), len(self.param_groups),
                                 self.fused not in ("sgd", "lars"), cs.cuda_stream)
            self._count_launch(2)
        if self.max_grad_norm is not None:
            for b in self.buckets:
                if not b.normed:
                    self._launch_norm(b, wait=False)
            cu.clip_norm_update(self.ctx.view, 0, self.clip_win_off, self._clip_scratch.data_ptr(), len(self.buckets),
                                self._clip_scratch.shape[1], float(self.max_grad_norm), self._grad_norm.data_ptr(),
                                self._hp_dev.data_ptr(), len(self.param_groups), cs.cuda_stream)
            self._count_launch()
        for b in self.buckets:
            if self._ring_mode != "off" and b.ring_cls is not None:
                self._ring_pending.append(b)
                b.launched = True
                self._launched += 1
            else:
                self._ring_flush()          # keep the comm stream in bucket order
                self._launch(b)
        self._ring_flush()

    def finish_launches(self):
        """Launch every bucket that has not gone out yet, without waiting."""
        self._issue_remaining()
        if self._stamps and self._last_done is not None:
            self.ctx.cu.ring_stamp(self.ctx.view, 1, self.comm_stream.cuda_stream)   # last exchange finished
            self._count_launch()
        self._reset(keep_events=True)

    def _flush_trace(self):
        """Turn the timing events of this step into Chrome-trace spans (device time, anchored at
        the host timestamp of the step's first launch)."""
        if not self._trace_spans:
            return
        tl = self.engine.timeline
        t0_ev, t0_us = self._trace_t0
        self._trace_spans[-1][2].synchronize()
        for b, start, end in self._trace_spans:
            ts = t0_us + int(t0_ev.elapsed_time(start) * 1000)
            dur = max(1, int(start.elapsed_time(end) * 1000))
            name = "bucket%d[%s x%d]" % (b.index, str(b.dtype)[6:], len(b.params))
            stage = "PUSHPULL_FUSED_OPT" if self.fused else "PUSHPULL"
            tl.record(name, stage, b.index, ts, dur)
            tl.record(name, "", (1 << 64) - 1, ts, dur)
        self._trace_spans = []
        self._trace_t0 = None
        if self._step + 1 >= tl.end_step():
            tl.dump()

    def record_ring_trace(self, dump: bool = False):
        """Chrome-trace spans of the last step's ring launches.  The kernels stamp the GPU's
        globaltimer when the first CTA picks a bucket up and when the last CTA finishes it, so the
        spans exist for CUDA-graph replays too (the reference's timeline is host wall-clock only,
        docs/timeline.md; events cannot be recorded inside a captured graph)."""
        tl = self.engine.timeline
        if not tl.enabled() or not getattr(self, "_ring_traced", False):
            return
        if self._stamp_base is None:
            # anchor: one stamp kernel + the host clock right after it completed
            self.ctx.cu.ring_stamp(self.ctx.view, 15, torch.cuda.current_stream(self.device).cuda_stream)
            torch.cuda.synchronize(self.device)
            host_us = self.engine.core.now_us()
            _, st = self.ctx.cu.ring_trace(self.ctx.view, [])
            self._stamp_base = (host_us, st[15])
        host_us, gt0 = self._stamp_base
        by_index = {b.index: b for b in self.buckets}
        for idx, pos, t0, t1 in self.ring_spans():
            if t1 <= t0 or t0 == 0:
                continue
            b = by_index[idx]
            ts = host_us + (int(t0) - int(gt0)) // 1000
            dur = max(1, (int(t1) - int(t0)) // 1000)
            name = "bucket%d[%s x%d prio %d #%d]" % (b.index, str(b.dtype)[6:], len(b.params), b.priority, pos)
            tl.record(name, "PUSHPULL_FUSED_OPT" if self.fused else "PUSHPULL", b.index, ts, dur)
            tl.record(name, "", (1 << 64) - 1, ts, dur)
        self._ring_traced = False
        if dump or self._step + 1 >= tl.end_step():
            tl.dump()

    def _reset(self, keep_events: bool = False):
        self._flush_trace()
        if (self._ring_mode != "off" and self.engine.timeline.enabled() and self.engine.timeline.active(self._step)
                and not torch.cuda.is_current_stream_capturing()):
            self.record_ring_trace()
        self._launched = 0
        self._next = 0
        self._step += 1
        self._ring_started = False
        self._last_step_launches, self._xlaunches = self._xlaunches, 0
        for b in self.buckets:
            b.pending = len(b.params)
            b.launched = False
            b.normed = False
        for p in self._delay:
            self._delay[p] = self.bpps

    def zero_grad(self):
        for b in self.buckets:
            b.flat_grad.zero_()

    def remove_hooks(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []

    # ------------------------------------------------------------------ state access (fused mode)
    def master_params(self) -> Dict[torch.nn.Parameter, torch.Tensor]:
        """fp32 master values of THIS rank's shard, keyed by parameter (partial views)."""
        out = {}
        for b in self.buckets:
            s0, s1 = self.shard_range(b)
            for p, st in zip(b.params, b.starts):
                lo, hi = max(st, s0), min(st + p.numel(), s1)
                if lo < hi:
                    out[p] = (lo - st, b.master[lo - s0:hi - s0])
        return out

    _STATE_KEYS = ("master", "state0", "state1")

    def export_state(self) -> Dict[torch.nn.Parameter, Dict[str, torch.Tensor]]:
        """The full fp32 optimizer state, {param: {"master", "state0"[, "state1"]: CPU tensor}}, each tensor with
        its parameter's shape and strides.  Collective when world > 1: every rank must call it, and every rank
        gets the whole state.  Per bucket and buffer, this rank's shard goes into a zero host buffer of the
        bucket's length, and the buffers' bit patterns are summed over ranks as int32 through the engine's host
        collective, one bucket at a time.  Every element is non-zero on one rank at most, so the sum reproduces each
        rank's bits exactly (negative zeros and NaN payloads included); no float arithmetic and no wire cast
        (BYTEPS_WIRE_DTYPE applies to float32 exchanges on the device) touches the state."""
        if not self.fused:
            raise RuntimeError("export_state needs the fused optimizer")
        out: Dict[torch.nn.Parameter, Dict[str, torch.Tensor]] = {p: {} for b in self.buckets for p in b.params}
        for b in self.buckets:
            s0, s1 = self.shard_range(b)
            for key in self._STATE_KEYS:
                buf = getattr(b, key)
                if buf is None:
                    continue
                host = torch.zeros(b.numel, dtype=torch.float32)
                host[s0:s1].copy_(buf[:s1 - s0])
                if self.world > 1:
                    bits = host.view(torch.int32)
                    h = self.engine.push_pull_async(bits, bits, False, "FusedState.%d.%d.%s" % (b.index, b.numel, key))
                    self.engine.synchronize(h)
                tensors = [torch.empty_strided(p.size(), p.stride(), dtype=torch.float32) for p in b.params]
                copy_bucket_state(host, (0, b.numel), b.starts, tensors, to_shard=False)
                for p, t in zip(b.params, tensors):
                    out[p][key] = t
        return out

    def import_state(self, state: Dict[torch.nn.Parameter, Dict[str, torch.Tensor]], group_steps: List[int]):
        """Install full per-parameter state (as `export_state` returns it; any shape-matching dtype and layout)
        and the per-group step counts.  Each rank copies its own slice IN PLACE into the existing shard buffers,
        whose addresses a captured CUDA graph or ring table may hold.  A missing entry takes the initial value:
        the master from the current parameter, zero moments / momentum."""
        if not self.fused:
            raise RuntimeError("import_state needs the fused optimizer")
        if len(group_steps) != len(self._group_step):
            raise ValueError("expected %d group step counts, got %d" % (len(self._group_step), len(group_steps)))
        for p, ent in state.items():
            for key, v in ent.items():
                if v is not None and tuple(v.shape) != tuple(p.shape):
                    raise ValueError("state %r has shape %s, its parameter %s" % (key, tuple(v.shape), tuple(p.shape)))
        for b in self.buckets:
            s0, s1 = self.shard_range(b)
            for key in self._STATE_KEYS:
                buf = getattr(b, key)
                if buf is None:
                    continue
                tensors = []
                for p in b.params:
                    v = state.get(p, {}).get(key)
                    t = torch.empty_strided(p.size(), p.stride(), dtype=torch.float32)
                    if v is not None:
                        t.copy_(v)
                    elif key == "master":
                        t.copy_(p.detach())
                    else:
                        t.zero_()
                    tensors.append(t)
                stage = torch.empty(buf.numel(), dtype=torch.float32)
                copy_bucket_state(stage, (s0, s1), b.starts, tensors, to_shard=True)
                buf.copy_(stage)
        self._group_step = [int(t) for t in group_steps]
        if self.loss_scaler is not None:
            self._ls_steps.copy_(torch.tensor(self._group_step, dtype=torch.int32))
        self.refresh_hparams()

    def close(self):
        self.remove_hooks()
        torch.cuda.synchronize(self.device)
        for b in self.buckets:
            for p in b.params:
                if p.grad is not None:
                    p.grad = p.grad.detach().clone()
                if self.fused:
                    p.data = p.data.clone()
        if self.world > 1:
            self.engine.group.barrier()
        self.ctx.close()
