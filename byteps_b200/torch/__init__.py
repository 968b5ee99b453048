"""byteps_b200.torch - the user-facing API (drop-in for ``byteps.torch``).

Parity: /root/reference/byteps/torch/__init__.py:23-466.  Same entry points:
``init/shutdown/suspend/resume/rank/size/local_rank/local_size``,
``push_pull[_async][_inplace]``, ``poll/synchronize/declare``,
``DistributedOptimizer``, ``broadcast_parameters/optimizer_state/object``,
``Compression``; ``parallel.DistributedDataParallel`` and
``cross_barrier.CrossBarrier`` live in their sub-modules like in the reference.

What is different underneath: on CUDA the optimizer does not issue one
push_pull per parameter.  Gradients live in a symmetric NVLink-mapped arena and
are exchanged bucket by bucket by one fused sm_90a kernel each
(:mod:`byteps_b200.parallel.bucket`); with ``fused_update=True`` the kernel also
applies the SGD/Adam/LAMB/LARS step on fp32 master weights and all-gathers the new
parameters instead of the gradients.
"""
from __future__ import annotations

import io
import math
import os
from contextlib import contextmanager

import cloudpickle
import torch

from ..common import config as _config
from ..common import engine as _engine
from .compression import Compression
from .lamb import Lamb
from .lars import Lars
from .ops import (byteps_torch_set_num_grads, declare, get_pushpull_speed, init, local_rank, local_size, poll,
                  push_pull, push_pull_async, push_pull_async_inplace, push_pull_group_sync_inplace,
                  push_pull_inplace, rank, resume, set_learning_rate, shutdown, size, suspend, synchronize)
from .ops import push_pull_async_inplace as byteps_push_pull

__all__ = [
    "init", "shutdown", "suspend", "resume", "rank", "size", "local_rank", "local_size", "get_pushpull_speed",
    "push_pull", "push_pull_async", "push_pull_inplace", "push_pull_async_inplace", "push_pull_group_sync_inplace",
    "poll", "synchronize", "declare", "byteps_torch_set_num_grads", "DistributedOptimizer", "broadcast_parameters",
    "broadcast_optimizer_state", "broadcast_object", "Compression", "set_learning_rate", "convert_sync_batchnorm",
    "Lamb", "Lars",
]


def _wire_of(compression):
    if compression is Compression.fp16:
        return torch.float16
    if compression is getattr(Compression, "bf16", None):
        return torch.bfloat16
    return None


def _fused_kind(optimizer_cls, param_groups):
    name = optimizer_cls.__name__
    if issubclass(optimizer_cls, Lamb):
        return "lamb"
    if issubclass(optimizer_cls, Lars):
        return "lars"
    if issubclass(optimizer_cls, torch.optim.SGD):
        return "sgd"
    if issubclass(optimizer_cls, torch.optim.AdamW):
        return "adamw"
    if issubclass(optimizer_cls, torch.optim.Adam):
        if any(g.get("amsgrad", False) for g in param_groups):
            return None
        return "adam"
    del name
    return None


# torch.amp.GradScaler's defaults, by its names
_LOSS_SCALE_DEFAULTS = {"init_scale": 65536.0, "growth_factor": 2.0, "backoff_factor": 0.5, "growth_interval": 2000}


def _loss_scale_config(option):
    """The dynamic_loss_scale argument as a complete dict of GradScaler's parameters, or None when it is off."""
    if option is None or option is False:
        return None
    if option is True:
        return dict(_LOSS_SCALE_DEFAULTS)
    if not isinstance(option, dict):
        raise ValueError("dynamic_loss_scale must be a bool or a dict of %s" % ", ".join(_LOSS_SCALE_DEFAULTS))
    unknown = sorted(set(option) - set(_LOSS_SCALE_DEFAULTS))
    if unknown:
        raise ValueError("dynamic_loss_scale: unknown key(s) %s; expected some of %s"
                         % (", ".join(map(repr, unknown)), ", ".join(_LOSS_SCALE_DEFAULTS)))
    cfg = dict(_LOSS_SCALE_DEFAULTS, **option)
    return dict(zip(_LOSS_SCALE_DEFAULTS, _checked_scaler_values(
        "dynamic_loss_scale", cfg["init_scale"], cfg["growth_factor"], cfg["backoff_factor"], cfg["growth_interval"])))


def _checked_max_grad_norm(value):
    """max_grad_norm as a float, or ValueError: None (no clipping) or a finite number > 0."""
    if value is None:
        return None
    if isinstance(value, bool):
        raise ValueError("max_grad_norm must be a finite number > 0, got %r" % (value,))
    try:
        v = float(value)
    except (TypeError, ValueError):
        raise ValueError("max_grad_norm must be a finite number > 0, got %r" % (value,)) from None
    if not (math.isfinite(v) and v > 0):
        raise ValueError("max_grad_norm must be a finite number > 0, got %r" % (value,))
    return v


def _checked_scaler_entry(ls):
    """A loaded "loss_scaler" entry (GradScaler.state_dict()'s keys) as (scale, growth_factor, backoff_factor,
    growth_interval, growth_tracker), checked like the constructor's options, or ValueError."""
    missing = sorted({"scale", "growth_factor", "backoff_factor", "growth_interval", "_growth_tracker"} - set(ls))
    if missing:
        raise ValueError("loaded loss_scaler entry lacks %s" % ", ".join(missing))
    vals = _checked_scaler_values("loaded loss_scaler", ls["scale"], ls["growth_factor"], ls["backoff_factor"],
                                  ls["growth_interval"])
    tracker = ls["_growth_tracker"]
    if isinstance(tracker, bool) or int(tracker) != tracker or not 0 <= tracker < vals[3]:
        raise ValueError("loaded loss_scaler: _growth_tracker must be an integer in [0, growth_interval), got %r"
                         % (tracker,))
    return vals + (int(tracker),)


def _checked_scaler_values(what, scale, growth, backoff, interval):
    """(scale, growth_factor, backoff_factor, growth_interval) as float, float, float, int, or ValueError."""
    scale, growth, backoff = float(scale), float(growth), float(backoff)
    # the device holds S as a float32 and multiplies the gradients by the float32 1/S
    s32 = float(torch.tensor(scale, dtype=torch.float32))
    if not (math.isfinite(s32) and s32 > 0 and math.isfinite(float(torch.tensor(1.0 / s32, dtype=torch.float32)))):
        raise ValueError("%s: the scale must be positive with S and 1/S finite in float32, got %r" % (what, scale))
    if not growth > 1 or not math.isfinite(growth):
        raise ValueError("%s: growth_factor must be finite and > 1, got %r" % (what, growth))
    if not 0 < backoff < 1:
        raise ValueError("%s: backoff_factor must be in (0, 1), got %r" % (what, backoff))
    if isinstance(interval, bool) or int(interval) != interval or interval < 1:
        raise ValueError("%s: growth_interval must be an integer >= 1, got %r" % (what, interval))
    return scale, growth, backoff, int(interval)


class _DistributedOptimizer(torch.optim.Optimizer):
    def __init__(self, params, named_parameters, compression, backward_passes_per_step=1, fused_update=None,
                 bucket_bytes=None, compression_params=None, dynamic_loss_scale=None, max_grad_norm=None):
        super(self.__class__, self).__init__(params)
        if fused_update is None:
            fused_update = os.getenv("BYTEPS_FUSED_OPTIMIZER", "0") not in ("0", "")
        loss_scaler = _loss_scale_config(dynamic_loss_scale)
        self._max_grad_norm = _checked_max_grad_norm(max_grad_norm)
        if loss_scaler is not None and not fused_update:
            raise ValueError("dynamic_loss_scale needs fused_update=True")
        self._compression = compression
        from ..common.compression_params import translate

        self._compress_kwargs = translate(compression_params, self.defaults)
        named_parameters = list(named_parameters) if named_parameters is not None else []
        self._enable_async = (int(os.getenv('BYTEPS_ENABLE_ASYNC', 0)) != 0)
        self._async_seeded = False
        if self._enable_async:
            assert int(os.getenv('DMLC_NUM_WORKER', 1)) > 1, "Async is only valid for distributed training"
            if self._max_grad_norm is not None:
                raise ValueError("max_grad_norm clips the averaged gradients; BYTEPS_ENABLE_ASYNC never averages them")
        if any(not isinstance(p, tuple) for p in named_parameters):
            raise ValueError('named_parameters should be a sequence of tuples (name, parameter), '
                             'usually produced by model.named_parameters().')
        dups = _DistributedOptimizer.find_duplicates([k for k, _ in named_parameters])
        if dups:
            raise ValueError('Parameter names in named_parameters must be unique. '
                             'Found duplicates: %s' % ', '.join(dups))
        all_params = [p for g in self.param_groups for p in g['params']]
        if named_parameters:
            self._parameter_names = {p: n for n, p in named_parameters}
        else:
            self._parameter_names = {p: 'push_pull.noname.%s' % i for i, p in enumerate(all_params)}
        self.backward_passes_per_step = backward_passes_per_step
        self._push_pull_delay = {p: backward_passes_per_step for p in all_params if p.requires_grad}
        self._handles = {}
        self._grad_accs = []
        self._hook_handles = []
        self._requires_update = set()
        self._should_sync = True
        self._sync = None        # BucketedGradSync on the symmetric-memory path
        self._fused = None
        # priority: parameters needed first by the next forward go first
        self._priority = {p: -i for i, p in enumerate(all_params)}

        # declare in sorted-name order, gradients first then parameters, so
        # keys are identical on all ranks (reference: "two loops for load-balancing")
        for name in sorted(self._parameter_names.values()):
            declare("Gradient." + name, **self._compress_kwargs)
        for name in sorted(self._parameter_names.values()):
            declare("Parameter." + name)
        if self._compress_kwargs:
            # error feedback rescales its residual by lr_prev / lr: the compressors must know the rate BEFORE the
            # first exchange, not from the first step() on (the residual of step 1 was scaled by 1 / lr otherwise)
            set_learning_rate(self.param_groups[0]["lr"])

        eng = _engine()
        on_cuda = all(p.is_cuda for p in all_params) and torch.cuda.is_available()
        # lossy compressors work per tensor (own error-feedback state): they take the per-parameter path
        want_symm = on_cuda and not self._enable_async and not self._compress_kwargs and (
            eng.backend == "symm" or (eng.backend == "local" and fused_update))
        if loss_scaler is not None and not want_symm:
            raise ValueError("dynamic_loss_scale needs the fused update on the symmetric-memory or local backend "
                             "(CUDA parameters, no lossy compression, no BYTEPS_ENABLE_ASYNC); this job uses the %r "
                             "backend" % eng.backend)
        if want_symm:
            from ..parallel.bucket import BucketedGradSync

            kind = _fused_kind(self.__class__.__mro__[1], self.param_groups) if fused_update else None
            if fused_update and kind is None:
                raise ValueError("fused_update supports SGD, Adam, AdamW (no amsgrad), byteps_b200.torch.Lamb and "
                                 "byteps_b200.torch.Lars")
            self._fused = kind
            self._sync = BucketedGradSync(eng, self.param_groups, fused=kind, wire_dtype=_wire_of(compression),
                                          bucket_bytes=bucket_bytes,
                                          backward_passes_per_step=backward_passes_per_step,
                                          priority_of=self._priority, loss_scaler=loss_scaler,
                                          max_grad_norm=self._max_grad_norm if kind else None)
            if kind:
                self._sync.refresh_hparams()
        elif size() > 1 or eng.backend == "ps":
            # one worker behind a server (BYTEPS_FORCE_DISTRIBUTED=1, the reference's test harness) still goes
            # through the servers: that is what applies the two compression stages
            self._register_hooks()
        if self._max_grad_norm is not None and not self._fused:
            # the unfused paths clip with torch itself and keep its result here
            self._grad_norm = torch.zeros((), dtype=torch.float32, device=all_params[0].device)

    @staticmethod
    def find_duplicates(lst):
        seen, dups = set(), set()
        for el in lst:
            if el in seen:
                dups.add(el)
            seen.add(el)
        return dups

    def set_backward_passes_per_step(self, passes):
        self.backward_passes_per_step = passes
        for p in self._push_pull_delay:
            self._push_pull_delay[p] = passes
        if self._sync is not None:
            self._sync.set_backward_passes_per_step(passes)

    # ---- generic (per-parameter) path: gloo / nccl / ps transports -------------
    def _register_hooks(self):
        for param_group in self.param_groups:
            for p in param_group['params']:
                if p.requires_grad:
                    if p.grad is None:
                        p.grad = torch.zeros_like(p)
                    self._requires_update.add(p)
                    self._hook_handles.append(p.register_post_accumulate_grad_hook(self._make_hook(p)))

    def _push_pull_grad_async(self, p):
        name = self._parameter_names.get(p)
        if self._enable_async:
            return None, None   # the real handle is created in step()
        if p.grad is None:      # unused this iteration and cleared by zero_grad(set_to_none=True): contribute zeros
            p.grad = torch.zeros_like(p)
        tensor = p.grad
        if not tensor.is_contiguous() and _dense_tensor(tensor):
            # channels_last & co: the sum is elementwise, exchange the dense storage as a flat view
            tensor = torch.as_strided(tensor, (tensor.numel(),), (1,), tensor.storage_offset())
        tensor_compressed, ctx = self._compression.compress(tensor)
        handle = byteps_push_pull(tensor_compressed, average=True, name="Gradient." + name,
                                  priority=self._priority.get(p, 0))
        return handle, (ctx, tensor_compressed)

    def _make_hook(self, p):
        def hook(*ignore):
            if p in self._handles and self._handles[p][0] is not None:
                if self._push_pull_delay[p] <= 0:
                    raise AssertionError(
                        "Gradients were computed more than backward_passes_per_step times before call "
                        "to step(). Increase backward_passes_per_step to accumulate gradients locally.")
            assert not p.grad.requires_grad
            assert self._push_pull_delay[p] > 0
            handle, ctx = None, None
            self._push_pull_delay[p] -= 1
            if self._push_pull_delay[p] == 0:
                handle, ctx = self._push_pull_grad_async(p)
            self._handles[p] = (handle, ctx)
        return hook

    def synchronize(self):
        if self._sync is not None:
            self._sync.synchronize()
            return
        missing_p = self._requires_update - set(self._handles.keys())
        for p in sorted(missing_p, key=lambda q: self._parameter_names.get(q)):
            self._handles[p] = self._push_pull_grad_async(p)
        for p, (handle, ctx) in list(self._handles.items()):
            if handle is None:
                self._handles[p] = self._push_pull_grad_async(p)
        for p, (handle, ctx) in self._handles.items():
            output = synchronize(handle)
            self._push_pull_delay[p] = self.backward_passes_per_step
            if not self._enable_async and ctx is not None:
                cctx, _ = ctx
                tmp = self._compression.decompress(output, cctx)
                if tmp.data_ptr() != p.grad.data_ptr():
                    if tmp.shape != p.grad.shape:   # flat view of a dense, permuted gradient
                        torch.as_strided(p.grad, (p.grad.numel(),), (1,), p.grad.storage_offset()).copy_(tmp)
                    else:
                        p.grad.copy_(tmp)
        self._handles.clear()

    @contextmanager
    def skip_synchronize(self):
        if self._enable_async:
            raise AssertionError("skip_synchronize cannot be used in async training")
        self._should_sync = False
        try:
            yield
        finally:
            self._should_sync = True

    def zero_grad(self, set_to_none=False):
        if self._sync is not None:
            self._sync.zero_grad()      # one memset per bucket; .grad stays an arena view
            return
        return super(self.__class__, self).zero_grad(set_to_none=set_to_none)

    def refresh_hparams(self):
        """Fused mode + CUDA graphs: call before every replay of a captured step
        so lr/momentum/Adam bias corrections of that step reach the kernels
        (eager ``step()`` does the equivalent by itself)."""
        if self._sync is not None:
            self._drop_loaded_state()
            self._sync.pre_replay()

    def step(self, closure=None):
        if self._enable_async:
            old_weight_map = {p: p.data.clone().detach() for p in self._handles}
            if not self._async_seeded:
                # the server accumulates deltas ONTO its stored copy: seed it with the weights (in name order, the
                # same on every worker; workers are expected to start from broadcast parameters).  The reference
                # seeds it with whatever the first push_pull of that name carries, i.e. a delta.
                for p in sorted(old_weight_map, key=lambda q: self._parameter_names.get(q)):
                    _engine().init_tensor("AsyncParam." + self._parameter_names.get(p), old_weight_map[p])
                self._async_seeded = True
            loss = super(self.__class__, self).step(closure)
            for p, (h, _) in list(self._handles.items()):
                p.data.sub_(old_weight_map.get(p))   # weight delta, pushed in place
                if h is None:
                    name = self._parameter_names.get(p)
                    handle = byteps_push_pull(p, average=False, name="AsyncParam." + name)
                    self._handles[p] = (handle, None)
            self.synchronize()
            return loss
        if self._fused:
            self._drop_loaded_state()
            loss = closure() if closure is not None else None
            # the update already happened inside the exchange kernels
            if self._should_sync:
                self.synchronize()
            self._sync.step_done()
            return loss
        if self._compress_kwargs:
            set_learning_rate(self.param_groups[0]["lr"])     # error feedback rescales by lr_prev/lr
        if self._should_sync:
            self.synchronize()
        if self._max_grad_norm is not None:
            params = [p for g in self.param_groups for p in g["params"]]
            self._grad_norm.copy_(torch.nn.utils.clip_grad_norm_(params, self._max_grad_norm))
        return super(self.__class__, self).step(closure)

    @property
    def grad_sync(self):
        return self._sync

    @property
    def grad_norm(self):
        """The last step's total gradient norm before clipping, as ``clip_grad_norm_`` returns it: a 0-dim float32
        tensor.  With ``fused_update=True`` it is a device tensor the kernels write (a captured step updates it on
        every replay); reading it does not synchronise, ``.item()`` does.  On a step dynamic loss scaling skipped it
        holds the non-finite norm that was computed."""
        if self._max_grad_norm is None:
            raise RuntimeError("this optimizer was built without max_grad_norm")
        return self._sync.grad_norm_tensor() if self._fused else self._grad_norm

    # ---- dynamic loss scaling (fused mode) ------------------------------------------
    def _scaler(self):
        if self._sync is None or self._sync.loss_scaler is None:
            raise RuntimeError("this optimizer was built without dynamic_loss_scale")
        return self._sync

    def scale_loss(self, loss):
        """``loss * S``, S being the current loss scale as a device scalar: no host synchronisation, so it can be
        captured into a CUDA graph.  Use ``opt.scale_loss(loss).backward()``; ``step()`` unscales, skips a step
        whose gradients overflowed and updates S."""
        return loss * self._scaler().scale_tensor()

    @property
    def loss_scale(self):
        """The current loss scale S (a float).  Reads it from the device: synchronises."""
        return self._scaler().loss_scaler_state()["scale"]

    @property
    def skipped_steps(self):
        """Steps this optimizer skipped because a gradient overflowed.  Reads the count from the device:
        synchronises.  The count is not part of a checkpoint: after ``load_state_dict`` it continues from this
        optimizer's own count, not from the saved run's."""
        return self._scaler().loss_scaler_state()["skipped"]

    def _drop_loaded_state(self):
        """Fused mode: forget the full copies of a load that no broadcast_optimizer_state consumed.  Training has
        moved on from them (a later broadcast must offer the live state, not roll back to the checkpoint)."""
        if self._fused and self.state:
            self.state.clear()

    # ---- checkpoints of the fused optimizer ----------------------------------------
    # With fused_update the state lives in the exchange's fp32 shards, not in self.state.  state_dict() gathers it
    # into the layout torch.optim uses (SGD and Lars: momentum_buffer; Adam/AdamW/Lamb: step, exp_avg, exp_avg_sq), plus
    # master_param for 16-bit parameters; load_state_dict() takes that layout, from this class or from torch.optim.
    _FUSED_KEYS = {"sgd": ("momentum_buffer",), "adam": ("exp_avg", "exp_avg_sq"), "adamw": ("exp_avg", "exp_avg_sq"),
                   "lamb": ("exp_avg", "exp_avg_sq"), "lars": ("momentum_buffer",)}

    def state_dict(self):
        """The optimizer state in ``torch.optim``'s format.

        With ``fused_update=True`` and more than one process this call is collective, like FSDP's optimizer
        state dict: every rank must call it (and every rank gets the full state); save it on one rank only.
        The state is full, not sharded, so it loads at any world size and into a plain ``torch.optim``
        optimizer.  Tensors are fp32 CPU tensors with their parameter's shape and strides.  16-bit parameters
        get one extra entry, ``master_param``, the fp32 master weights.
        """
        sd = super(self.__class__, self).state_dict()
        if not self._fused:
            return sd
        full = self._sync.export_state()
        steps = self._sync.applied_steps()
        state = {}
        idx = 0
        for gi, g in enumerate(self.param_groups):
            t = steps[gi]
            for p in g["params"]:
                ent = full.get(p)
                if ent is not None:
                    e = {}
                    if t > 0 and self._fused in ("sgd", "lars"):
                        # Lars keeps its buffer whatever the momentum, as the plain optimizer does
                        if self._fused == "lars" or g.get("momentum", 0) != 0:
                            e["momentum_buffer"] = ent["state0"]
                    elif t > 0:
                        e["step"] = torch.tensor(float(t), dtype=torch.float32)
                        e["exp_avg"], e["exp_avg_sq"] = ent["state0"], ent["state1"]
                    # torch's Adam creates its state only for a parameter without any: an entry holding only the
                    # masters (nothing has been stepped yet, so they equal the weights) would stop it
                    if p.dtype != torch.float32 and (t > 0 or self._fused in ("sgd", "lars")):
                        e["master_param"] = ent["master"]
                    if e:
                        state[idx] = e
                idx += 1
        sd["state"] = state
        if self._sync.loss_scaler is not None:
            sd["loss_scaler"] = self._loss_scaler_entry()
        return sd

    def _loss_scaler_entry(self):
        """torch.amp.GradScaler.state_dict() of the device scaler."""
        st = self._sync.loss_scaler_state()
        return {"scale": st["scale"], "growth_factor": st["growth_factor"], "backoff_factor": st["backoff_factor"],
                "growth_interval": st["growth_interval"], "_growth_tracker": st["tracker"]}

    def load_state_dict(self, state_dict):
        """Load a state dict of ``state_dict()`` or of the matching ``torch.optim`` optimizer.

        With ``fused_update=True`` the state is copied in place into this rank's shards (CUDA graphs captured
        earlier stay valid) and the full tensors are also kept in ``self.state`` until
        ``broadcast_optimizer_state`` hands them to the other ranks, so loading on rank 0 only works.  The next
        ``step()`` (or ``refresh_hparams()`` before a graph replay) drops them if no broadcast came first.  A
        ``momentum_buffer`` means SGD or Lars has taken a step; Adam's ``step`` must be equal within a param group.
        A Lars buffer includes the learning rate, so it does not move between Lars and ``torch.optim.SGD``.
        Missing entries start fresh: master weights from the current parameters (load the model first),
        zero moments.
        """
        if not self._fused:
            return super(self.__class__, self).load_state_dict(state_dict)
        ls_vals = None
        if self._sync.loss_scaler is not None and state_dict.get("loss_scaler") is not None:
            ls_vals = _checked_scaler_entry(state_dict["loss_scaler"])    # before anything is installed
        live = [p for g in self.param_groups for p in g["params"]]
        saved = [i for g in state_dict["param_groups"] for i in g["params"]]
        by_id = dict(zip(saved, live))
        full = {}
        for i, ent in state_dict["state"].items():
            p = by_id.get(i)
            if p is None:
                continue
            full[p] = {k: (_full_like(p, v) if torch.is_tensor(v) and v.dim() > 0 else v) for k, v in ent.items()}
        steps = []
        for g in self.param_groups:
            ents = [full[p] for p in g["params"] if p in full]
            if self._fused in ("sgd", "lars"):
                steps.append(1 if any("momentum_buffer" in e for e in ents) else 0)
                continue
            vals = sorted({float(e["step"]) for e in ents if "step" in e})
            if len(vals) > 1:
                raise ValueError("loaded state dict has different Adam step counts in one parameter group: %s"
                                 % vals)
            steps.append(int(vals[0]) if vals else 0)
        # torch rebuilds param_groups as new dicts: put the loaded options into the live ones instead, which the
        # wrapped optimizer and the exchange's hyper-parameter feed hold
        groups = self.param_groups
        super(self.__class__, self).load_state_dict({"state": {}, "param_groups": state_dict["param_groups"]})
        for old, new in zip(groups, self.param_groups):
            old.update(new)
        self.param_groups = groups
        self.state.update(full)
        if self._sync.loss_scaler is not None:
            if ls_vals is None:
                self._sync.reset_loss_scaler()
            else:
                self._sync.set_loss_scaler_state(*ls_vals)
        keys = self._FUSED_KEYS[self._fused]
        self._sync.import_state({p: dict({"master": e.get("master_param")},
                                         **{"state%d" % i: e.get(k) for i, k in enumerate(keys)})
                                 for p, e in full.items()}, steps)


def DistributedOptimizer(optimizer, named_parameters=None, compression=Compression.none,
                         backward_passes_per_step=1, fused_update=None, bucket_bytes=None, compression_params=None,
                         dynamic_loss_scale=False, max_grad_norm=None):
    """Wrap ``optimizer`` so gradients are averaged over all processes before
    ``step()``; communication overlaps with ``loss.backward()``.

    Arguments match the reference (optimizer, named_parameters, compression,
    backward_passes_per_step).  Extras: ``fused_update=True`` applies the
    SGD, Adam(W), :class:`Lamb` or :class:`Lars` step on fp32 master weights inside the
    exchange kernels;
    ``bucket_bytes`` sets the fusion granularity; ``compression_params`` (e.g.
    ``{"compressor": "topk", "k": 0.01, "ef": "vanilla"}``, docs/gradient-compression.md)
    turns on lossy gradient compression per tensor - GPU kernels over NVLink, or the
    worker/server compressors in CPU-server mode.

    ``synchronize()`` forces completion, ``skip_synchronize()`` lets a following ``step()`` skip it.

    ``max_grad_norm`` (a finite float > 0): clip the gradients by their global 2-norm before every update, with
    ``torch.nn.utils.clip_grad_norm_``'s rule.  The norm N is taken over every parameter of every param group, on
    the averaged gradient (with ``dynamic_loss_scale``, the unscaled one), and the update runs on
    ``min(1, max_grad_norm / (N + 1e-6)) * g``.  Only the 2-norm is supported.  ``grad_norm`` holds N of the last
    step.  With ``fused_update=True`` the norm is taken and applied inside the exchange on the device, with no host
    synchronisation, so the step still captures into a CUDA graph; the exchanges then wait for the last gradient,
    so the update no longer overlaps with backward.  Every other configuration runs ``synchronize()``,
    ``clip_grad_norm_`` over all parameters and the wrapped ``step()``.  With ``fused_update=True``, a
    ``clip_grad_norm_`` of your own between ``synchronize()`` and ``step()`` has no effect: the update has already
    happened, and ``.grad`` holds this rank's unreduced gradients.

    ``dynamic_loss_scale`` (with ``fused_update=True``, symmetric-memory or local backend): dynamic loss scaling
    for fp16 training, decided on the device.  ``True`` uses ``torch.amp.GradScaler``'s defaults; a dict overrides
    any of ``init_scale``, ``growth_factor``, ``backoff_factor`` and ``growth_interval`` (GradScaler's meanings).
    The loop is ``opt.zero_grad(); opt.scale_loss(loss).backward(); opt.step()``: a step whose gradients hold an
    inf or NaN on any rank (as they go onto the wire) is skipped on every rank and the scale backs off; the scale
    grows after ``growth_interval`` clean steps.  Nothing synchronises with the host, so the step captures into a
    CUDA graph.  ``loss_scale`` and ``skipped_steps`` read the state (and synchronise); ``state_dict()`` carries
    it as ``"loss_scaler"`` in GradScaler's format.  Do not combine ``fused_update=True`` with a
    ``torch.amp.GradScaler``: the update happens inside the exchange, before the scaler could unscale or skip it.
    """
    cls = type(optimizer.__class__.__name__, (optimizer.__class__,), dict(_DistributedOptimizer.__dict__))
    return cls(optimizer.param_groups, named_parameters, compression, backward_passes_per_step, fused_update,
               bucket_bytes, compression_params, dynamic_loss_scale, max_grad_norm)


def broadcast_parameters(params, root_rank, prefix="Parameter."):
    """Broadcast parameters from ``root_rank`` (dict such as ``state_dict()``,
    or a list of tensors / (name, tensor) pairs).  Implemented, like the
    reference, as zero-on-non-root followed by a sum push_pull."""
    if isinstance(params, dict):
        params = sorted(params.items())
    elif isinstance(params, list):
        params = [p if isinstance(p, tuple) else (None, p) for p in params]
    else:
        raise ValueError('invalid params of type: %s' % type(params))
    handles = []
    for name, p in params:
        if not torch.is_tensor(p):
            continue
        t = p.detach()
        if not t.is_contiguous():
            # e.g. channels_last weights: exchange the dense storage instead
            if not _dense_tensor(t):
                raise ValueError("cannot broadcast non-dense tensor %s" % name)
            t = torch.as_strided(t, (t.numel(),), (1,), t.storage_offset())
        if rank() != root_rank:
            t.zero_()
        handles.append(byteps_push_pull(t, average=False, name=(prefix + name) if name else None))
    for h in handles:
        synchronize(h)
    from ..parallel.bucket import resync_fused_masters

    resync_fused_masters()


def _dense_tensor(t):
    if t.numel() == 0:
        return True
    span = 1 + sum((s - 1) * st for s, st in zip(t.size(), t.stride()))
    return span == t.numel()


def _full_like(p, value=None):
    """An fp32 CPU tensor with p's shape and strides holding `value` (zeros if None).  Every rank lays the
    state tensors of a broadcast out like this, so their flat storage views line up."""
    t = torch.empty_strided(p.size(), p.stride(), dtype=torch.float32)
    if value is None:
        return t.zero_()
    if tuple(value.shape) != tuple(p.shape):
        raise ValueError("loaded state of shape %s for a parameter of shape %s"
                         % (tuple(value.shape), tuple(p.shape)))
    return t.copy_(value)


def _fused_broadcast_source(optimizer, root_rank):
    """Fused mode: the state dict every rank feeds into the in-place broadcast.  A root that loaded a state dict
    offers the full tensors load_state_dict() kept in ``optimizer.state``, and the other ranks zero tensors of the
    same keys, shapes and strides.  A root that loaded nothing offers its live state, which every rank exports
    together (after the layout's broadcast has re-derived the masters from the parameters)."""
    base = super(optimizer.__class__, optimizer).state_dict()     # param_groups, and what self.state holds
    layout = None
    if rank() == root_rank and base["state"]:
        layout = {i: {k: torch.is_tensor(v) and v.dim() > 0 for k, v in ent.items()}
                  for i, ent in base["state"].items()}
    layout = broadcast_object(layout, root_rank, name="optimizer_state.layout")
    if layout is None:
        return optimizer.state_dict()
    if rank() != root_rank:
        live = [p for g in optimizer.param_groups for p in g["params"]]
        base["state"] = {i: {k: _full_like(live[i]) if is_tensor else torch.tensor(0.0)
                             for k, is_tensor in ent.items()} for i, ent in layout.items()}
    return base


def _materialised_state(optimizer, root_rank=0):
    """state_dict of an optimizer whose per-parameter state exists.  A fresh optimizer has none until its first
    step: take one step of the INNER optimizer on zero gradients and undo whatever it did to the weights
    (weight decay moves them even with a zero gradient)."""
    if getattr(optimizer, "_fused", None):
        return _fused_broadcast_source(optimizer, root_rank)
    sd = optimizer.state_dict()
    if sd["state"]:
        return sd
    weights = [p for g in optimizer.param_groups for p in g["params"]]
    for p in weights:
        if p.requires_grad and p.grad is None:
            p.grad = torch.zeros_like(p)
    keep = [p.detach().clone() for p in weights]
    inner = super(optimizer.__class__, optimizer) if hasattr(optimizer, "_push_pull_delay") else optimizer
    inner.step()
    for p, v in zip(weights, keep):
        p.data.copy_(v)
    return optimizer.state_dict()


def broadcast_optimizer_state(optimizer, root_rank, prefix="Parameter."):
    """Make every process's optimizer state equal to ``root_rank``'s: tensor entries (momentum buffers, Adam
    moments, ...) are broadcast in place like parameters, everything else - python / 0-dim state entries such as
    ``step`` and the options of every param group (lr, betas, ...) - travels as one pickled tree.
    (Reference: byteps/torch/__init__.py:302-424.)

    With ``fused_update=True`` the root's state is what its last ``load_state_dict`` loaded (so loading on the
    root only is enough), or else its live state.  Every rank installs its shard of it, and the full copies
    ``load_state_dict`` kept are dropped.  ``broadcast_parameters`` re-derives the fp32 master weights from the
    parameters, so call it first: this call then puts the loaded masters back.  Without a loaded state the
    masters stay re-derived from the parameters, as after any ``broadcast_parameters``."""
    if isinstance(optimizer, torch.optim.LBFGS):
        raise ValueError("cannot broadcast torch.optim.LBFGS state")
    fused = getattr(optimizer, "_fused", None)
    sd = _materialised_state(optimizer, root_rank)
    if not sd["state"] and not fused:
        return
    tensors = []                                     # (name, tensor); names are equal on all ranks by construction
    plain = {"groups": [{k: v for k, v in g.items() if k != "params"} for g in sd["param_groups"]], "state": {}}
    for g in sd["param_groups"]:
        for pid in g["params"]:
            for field, val in sd["state"].get(pid, {}).items():
                if torch.is_tensor(val) and val.dim() > 0 and val.numel() > 0:
                    tensors.append(("%s.%s" % (field, pid), val))
                else:
                    plain["state"].setdefault(pid, {})[field] = val
    broadcast_parameters(tensors, root_rank, prefix)
    if fused and optimizer.grad_sync.loss_scaler is not None:
        # the root's scaler: what its load_state_dict installed, or its live state
        plain["loss_scaler"] = optimizer._loss_scaler_entry() if rank() == root_rank else None
    plain = broadcast_object(plain, root_rank, name="optimizer_state.plain")
    if "loss_scaler" in plain:
        sd["loss_scaler"] = plain["loss_scaler"]
    for live, stored, opts in zip(optimizer.param_groups, sd["param_groups"], plain["groups"]):
        live.update(opts)
        stored.update(opts)             # load_state_dict below must not put the old options back
    for pid, fields in plain["state"].items():
        sd["state"][pid].update(fields)
    # tensors were overwritten in place; the plain entries reach the optimizer through load_state_dict (torch
    # casts a python `step` back to the tensor form the optimizer keeps)
    optimizer.load_state_dict(sd)
    if fused:
        optimizer.state.clear()         # every rank holds its shard now


def broadcast_object(obj, root_rank=0, name=None):
    """Pickle ``obj`` on ``root_rank`` and return it on every process."""
    if name is None:
        name = type(obj).__name__
    if rank() == root_rank:
        b = io.BytesIO()
        cloudpickle.dump(obj, b)
        t = torch.frombuffer(bytearray(b.getvalue()), dtype=torch.uint8).clone()
        sz = torch.tensor([t.shape[0]], dtype=torch.int32)
        broadcast_parameters([(name + '.sz', sz)], root_rank, prefix="Size.")
    else:
        sz = torch.tensor([0], dtype=torch.int32)
        broadcast_parameters([(name + '.sz', sz)], root_rank, prefix="Size.")
        t = torch.zeros(int(sz.item()), dtype=torch.uint8)
    broadcast_parameters([(name + '.t', t)], root_rank, prefix="Parameter.")
    if rank() != root_rank:
        obj = cloudpickle.load(io.BytesIO(t.numpy().tobytes()))
    return obj


def convert_sync_batchnorm(module):
    """Synchronised batch norm: the counterpart of ``torch.nn.SyncBatchNorm.convert_sync_batchnorm``.

    Replaces every ``nn.BatchNorm2d`` of ``module`` (the models' ``BatchNormAct2d`` included, keeping their
    activation and residual input) by :class:`~byteps_b200.ops.bn_act.SyncBatchNormAct2d`, which normalises with
    the statistics of all ranks' batches in training.  The new modules hold the same Parameter and buffer objects,
    so a ``DistributedOptimizer`` built before or after the call stays valid.  Call it after ``init()``; it is
    collective (every rank calls it on the same model) and needs the symmetric-memory backend.  Returns the
    converted module."""
    from ..ops.bn_act import SyncBatchNormContext
    from ..ops.bn_act import convert_sync_batchnorm as _convert

    eng = _engine()
    if eng.backend not in ("local", "symm"):
        raise ValueError("convert_sync_batchnorm needs the symmetric-memory backend; this job uses %r" % eng.backend)
    sync = None
    if eng.size > 1:
        cmax = max([m.num_features for m in module.modules() if isinstance(m, torch.nn.BatchNorm2d)] or [8])
        sync = SyncBatchNormContext.create(eng.group, torch.device("cuda", torch.cuda.current_device()), cmax,
                                           eng.cfg.symm_mode)
    return _convert(module, sync)
