"""``tf.distribute`` integration: ``MirroredStrategy`` whose cross-replica reduction ends in a push_pull
(parity: /root/reference/byteps/tensorflow/distribute/cross_device_ops.py:585-627 ``BytepsAllReduce`` /
``BytepsCrossDeviceOps`` and mirrored_strategy.py:349-387 ``MirroredStrategy``).

The reference vendors 1.6 kLoC of TensorFlow-internal strategy code (tied to TF 1.15 / 2.1) to change one line:
after the replicas of a process have been reduced onto one device, the result is summed over all worker
processes with ``_push_pull``.  Here the same behaviour is built on TensorFlow's PUBLIC extension points only:

* ``BytepsCrossDeviceOps`` subclasses ``tf.distribute.CrossDeviceOps`` and implements the three abstract
  methods (``reduce_implementation``, ``batch_reduce_implementation``, ``broadcast_implementation``): local
  replicas are combined by a ``tf.distribute.ReductionToOneDevice`` (or whatever ``local_ops`` is given),
  then each component is exchanged through the shared engine - on an H100 that is the NVLink push-pull
  kernel, reached zero-copy through DLPack (ops.py).
* ``BytepsAllReduce(num_packs)`` keeps the reference's constructor; ``num_packs`` groups the tensors of a
  ``batch_reduce`` into that many concatenated exchanges (1 = everything in one launch, 0 = one per tensor).
* ``MirroredStrategy(devices=None, cross_device_ops=None)`` subclasses ``tf.distribute.MirroredStrategy``.
  One process drives one GPU here, so ``devices`` defaults to this process's GPU (``/gpu:<local_rank>``, or
  the CPU when TensorFlow sees no GPU) and ``cross_device_ops`` to ``BytepsAllReduce()``.

``ReduceOp.MEAN`` yields the mean over ALL replicas of ALL workers (the reference divides by the local
replica count only and leaves the division by the worker count to the training script).
"""
from __future__ import annotations

import tensorflow as tf

from ..ops import _push_pull, broadcast as _broadcast, local_rank, rank, size

__all__ = ["BytepsCrossDeviceOps", "BytepsAllReduce", "MirroredStrategy"]


def _is_mean(reduce_op) -> bool:
    name = getattr(reduce_op, "name", None) or str(reduce_op)
    return name.upper().endswith("MEAN")


def _components(value):
    """Per-device tensors of a (possibly distributed) value."""
    vals = getattr(value, "values", None)
    if isinstance(vals, (tuple, list)):
        return list(vals)
    return [value]


def _rebuild(value, comps):
    """A value of the same kind as `value` holding `comps` (Mirrored / PerReplica take the tuple of
    per-device tensors as their only constructor argument; plain tensors pass through)."""
    if isinstance(getattr(value, "values", None), (tuple, list)):
        return type(value)(tuple(comps))
    return comps[0]


class BytepsCrossDeviceOps(tf.distribute.CrossDeviceOps):
    """Reduce the replicas of this process locally, then sum over all worker processes by push_pull."""

    def __init__(self, local_ops=None, num_packs: int = 1, scope: str = "MirroredStrategy."):
        super().__init__()
        if num_packs < 0:
            raise ValueError("push_pull all-reduce requires num_packs >= 0, but {} is specified".format(num_packs))
        self._local = local_ops if local_ops is not None else tf.distribute.ReductionToOneDevice()
        self._num_packs = int(num_packs)
        self._scope = scope

    # -- helpers -------------------------------------------------------------------------------------------
    def _name(self, kind: str, tensor) -> str:
        # dtype + shape + kind (the anonymous-eager-tensor rule of ops._stable_name): the same name every step, the
        # same on every worker; exchanges are synchronous, so tensors of one shape may share it
        shape = "x".join(str(int(d)) for d in tensor.shape)
        return "%s%s_%s_%s" % (self._scope, kind, getattr(tensor.dtype, "name", tensor.dtype), shape or "scalar")

    def _exchange_one(self, tensor, kind, mean, tag=""):
        out = _push_pull(tensor, name=self._name(kind, tensor) + tag)
        if mean:
            out = out / tf.cast(size(), out.dtype)
        return out

    def _global(self, reduce_op, reduced, kind, tag=""):
        if size() <= 1:
            return reduced
        mean = _is_mean(reduce_op)
        comps = _components(reduced)
        # every local device holds the same locally-reduced value: exchange it once, mirror the result
        first = self._exchange_one(comps[0], kind, mean, tag)
        return _rebuild(reduced, [first] * len(comps))

    # -- tf.distribute.CrossDeviceOps ------------------------------------------------------------------------
    def reduce_implementation(self, reduce_op, per_replica_value, destinations, options=None):
        reduced = self._call_local("reduce_implementation", reduce_op, per_replica_value, destinations, options)
        return self._global(reduce_op, reduced, "reduce")

    def batch_reduce_implementation(self, reduce_op, value_destination_pairs, options=None):
        pairs = list(value_destination_pairs)
        local = [self._call_local("reduce_implementation", reduce_op, v, d, options) for v, d in pairs]
        if size() <= 1 or not local:
            return local
        if self._num_packs == 0 or len(local) == 1:
            return [self._global(reduce_op, r, "batch", ".%d" % i) for i, r in enumerate(local)]
        return self._packed(reduce_op, local)

    def broadcast_implementation(self, tensor, destinations):
        return self._local.broadcast_implementation(tensor, destinations)

    def _gather_implementation(self, per_replica_value, destinations, axis, options=None):
        """All-gather along `axis`: local replicas first (TensorFlow's own implementation), then the workers.  The
        cross-worker step is a push_pull of a buffer that is zero except for this worker's block, so every worker
        must contribute the same shape (what `strategy.gather` of per-replica batches produces)."""
        try:
            local = self._local._gather_implementation(per_replica_value, destinations, axis, options)
        except TypeError:
            local = self._local._gather_implementation(per_replica_value, destinations, axis)
        if size() <= 1:
            return local
        comps = _components(local)
        mine = comps[0]
        blocks = [mine if r == rank() else tf.zeros_like(mine) for r in range(size())]
        gathered = _push_pull(tf.concat(blocks, axis=axis), name=self._name("gather", mine) + ".ax%d" % axis)
        return _rebuild(local, [gathered] * len(comps))

    def _call_local(self, method, reduce_op, value, destinations, options):
        fn = getattr(self._local, method)
        try:
            return fn(reduce_op, value, destinations, options)
        except TypeError:          # TF < 2.4: no `options` argument
            return fn(reduce_op, value, destinations)

    def _packed(self, reduce_op, local):
        """Concatenate the flattened gradients of one dtype into `num_packs` exchanges (the reference's
        `num_packs` aggregation, cross_device_ops.py:585-606), split the results back."""
        mean = _is_mean(reduce_op)
        firsts = [_components(r)[0] for r in local]
        by_dtype = {}
        for i, t in enumerate(firsts):
            by_dtype.setdefault(getattr(t.dtype, "name", str(t.dtype)), []).append(i)
        outs = [None] * len(local)
        for dname in sorted(by_dtype):
            idx = by_dtype[dname]
            packs = max(1, min(self._num_packs, len(idx)))
            per = -(-len(idx) // packs)
            for pk in range(packs):
                chunk = idx[pk * per:(pk + 1) * per]
                if not chunk:
                    continue
                flat = tf.concat([tf.reshape(firsts[i], [-1]) for i in chunk], axis=0)
                summed = self._exchange_one(flat, "pack", mean, ".%s.%d" % (dname, pk))
                off = 0
                for i in chunk:
                    n = 1
                    for d in firsts[i].shape:
                        n *= int(d)
                    piece = tf.reshape(summed[off:off + n], firsts[i].shape)
                    off += n
                    outs[i] = _rebuild(local[i], [piece] * len(_components(local[i])))
        return outs


class BytepsAllReduce(BytepsCrossDeviceOps):
    """``cross_device_ops=BytepsAllReduce(num_packs=1)`` - the reference's spelling."""

    def __init__(self, num_packs: int = 1):
        super().__init__(num_packs=num_packs)


def _default_devices():
    try:
        gpus = tf.config.list_logical_devices("GPU")
    except Exception:  # noqa: BLE001 - very old TF
        gpus = []
    if gpus:
        return ["/gpu:%d" % (local_rank() % len(gpus))]
    return ["/cpu:0"]


class MirroredStrategy(tf.distribute.MirroredStrategy):
    """``tf.distribute.MirroredStrategy`` over the GPUs of this process, synchronised with every other worker
    process by push_pull.  Variables created under ``scope()`` are additionally made identical across workers
    by ``broadcast_variables`` (call it once after building the model, or use the keras
    ``BroadcastGlobalVariablesCallback``)."""

    def __init__(self, devices=None, cross_device_ops=None):
        if devices is None:
            devices = _default_devices()
        if cross_device_ops is None:
            cross_device_ops = BytepsAllReduce()
        super().__init__(devices=devices, cross_device_ops=cross_device_ops)

    def broadcast_variables(self, variables, root_rank: int = 0):
        """Make `variables` (mirrored or plain) equal to `root_rank`'s on every worker."""
        for i, var in enumerate(variables):
            comps = _components(var)
            value = _broadcast(comps[0], root_rank, name="MirroredStrategy.bcast.%d" % i)
            for c in comps:
                c.assign(value)
