"""TensorFlow front end: ``push_pull``, ``broadcast_variables``, ``DistributedOptimizer``,
``DistributedGradientTape``, ``BroadcastGlobalVariablesHook``
(parity: /root/reference/byteps/tensorflow/__init__.py:40-417).

TensorFlow is not part of this image; the module binds to whatever ``tensorflow`` is importable
and is exercised in tests/test_plugins.py against a minimal stand-in.  The exchange itself runs in
the shared engine (ops.py), so TF gradients on an H100 ride the same NVLink kernels as torch ones.
"""
from __future__ import annotations

import os

try:
    import tensorflow as tf
except ImportError as e:  # pragma: no cover
    raise ImportError("byteps_b200.tensorflow needs the `tensorflow` package (not shipped in this image); "
                      "`byteps_b200.torch` and `byteps_b200.dlpack` are always available") from e

from .compression import Compression
from .ops import (ReduceOps, _push_pull, broadcast, get_pushpull_speed, handle_average_backwards_compatibility,
                  init, local_rank, local_size, rank, resume, shutdown, size, suspend)

Average = ReduceOps.Average
Sum = ReduceOps.Sum
Adasum = ReduceOps.Adasum       # accepted as a name, rejected where a reduction would have to run it


def _resolve_op(op, average):
    op = handle_average_backwards_compatibility(op, average)
    if op == Adasum or op == "Adasum":
        raise ValueError("op == Adasum is not supported yet")
    return op


def push_pull(tensor, scope="", average=None, device_dense="", device_sparse="", compression=Compression.none,
              op=None, enable_async=False, name=None):
    """Average (default) or sum a tf.Tensor / tf.Variable over all workers.  ``tf.IndexedSlices``
    are densified first (the exchange kernels are dense)."""
    op = _resolve_op(op, average)
    if isinstance(tensor, tf.IndexedSlices):
        tensor = tf.convert_to_tensor(tensor)
    with tf.device(device_dense):
        compressed, ctx = compression.compress(tensor)
        summed = compression.decompress(_push_pull(compressed, scope, name=name), ctx)
        if op == Average and not enable_async:     # async training exchanges weight deltas: no averaging
            summed = summed / tf.cast(size(), summed.dtype)
    return summed


def broadcast_variables(variables, root_rank, scope=""):
    """Assign root's value to every variable on every worker."""
    variables = list(variables)
    if size() > 1:
        for i, var in enumerate(variables):
            var.assign(broadcast(var, root_rank, scope, name="bcast_%d_%s" % (i, getattr(var, "name", "var"))))
    return variables


def broadcast_global_variables(root_rank):
    """TF1-style graphs only; eager programs call broadcast_variables(model.variables, ...)."""
    if tf.executing_eagerly():
        raise RuntimeError("bps.broadcast_global_variables() does not support eager execution. "
                           "Please use `bps.broadcast_variables(<model/optimizer variables>)` instead.")
    return broadcast_variables(tf.compat.v1.global_variables(), root_rank)


class BroadcastGlobalVariablesHook(object):
    """SessionRunHook-compatible object (estimator / MonitoredTrainingSession): broadcasts all
    global variables from ``root_rank`` right after the session is created, so every worker starts
    from the same random init or restored checkpoint."""

    def __init__(self, root_rank, device=""):
        self.root_rank, self.device = root_rank, device
        self.bcast_op = None

    def begin(self):
        self.bcast_op = None

    def after_create_session(self, session, coord):
        with tf.device(self.device):
            self.bcast_op = broadcast_variables(tf.compat.v1.global_variables(), self.root_rank)

    def before_run(self, run_context):
        return None

    def after_run(self, run_context, run_values):
        return None

    def end(self, session):
        return None


def _reduce_grads(grads, names, device_dense, device_sparse, compression, sparse_as_dense, enable_async, scope):
    out = []
    for g, n in zip(grads, names):
        if g is None:
            out.append(None)
            continue
        if sparse_as_dense and isinstance(g, tf.IndexedSlices):
            g = tf.convert_to_tensor(g)
        out.append(push_pull(g, scope, device_dense=device_dense, device_sparse=device_sparse,
                             compression=compression, enable_async=enable_async, name=n))
    return out


def DistributedOptimizer(optimizer, name=None, use_locking=False, device_dense="", device_sparse="",
                         compression=Compression.none, sparse_as_dense=False, op=Average):
    """Wrap a TF/Keras optimizer: gradients are averaged over all workers before being applied
    (``compute_gradients``/``_compute_gradients``/``apply_gradients`` are intercepted, whichever the
    wrapped class has).  With ``BYTEPS_ENABLE_ASYNC=1`` the local update runs first and weight deltas
    are exchanged instead."""
    enable_async = int(os.getenv("BYTEPS_ENABLE_ASYNC", 0)) != 0
    if op == Adasum or op == "Adasum":
        raise ValueError("op == Adasum is not supported yet with DistributedOptimizer")
    base = optimizer.__class__
    scope = (name or "Distributed%s" % base.__name__) + "."

    def _names(grads_and_vars):
        return ["grad_%d_%s" % (i, getattr(v, "name", "var")) for i, (_, v) in enumerate(grads_and_vars)]

    class _Distributed(base):
        _bps_reduced = False

        def _bps_reduce(self, grads_and_vars):
            gv = list(grads_and_vars)
            if size() <= 1 or enable_async:
                return gv
            grads = _reduce_grads([g for g, _ in gv], _names(gv), device_dense, device_sparse, compression,
                                  sparse_as_dense, enable_async, scope)
            return list(zip(grads, [v for _, v in gv]))

        def compute_gradients(self, *args, **kwargs):           # tf.compat.v1 optimizers
            self._bps_reduced = True
            return self._bps_reduce(super().compute_gradients(*args, **kwargs))

        def _compute_gradients(self, *args, **kwargs):          # keras OptimizerV2.minimize
            self._bps_reduced = True
            return self._bps_reduce(super()._compute_gradients(*args, **kwargs))

        def apply_gradients(self, grads_and_vars, *args, **kwargs):
            gv = list(grads_and_vars)
            if not self._bps_reduced:                           # custom loops calling apply_gradients directly
                gv = self._bps_reduce(gv)
            self._bps_reduced = False
            if not enable_async:
                return super().apply_gradients(gv, *args, **kwargs)
            old = [tf.identity(v) for _, v in gv]
            result = super().apply_gradients(gv, *args, **kwargs)
            for i, ((_, v), o) in enumerate(zip(gv, old)):      # push the delta, adopt the server's weights
                v.assign(o + push_pull(v - o, scope, op=Sum, enable_async=True,
                                       name="AsyncParam_%d_%s" % (i, getattr(v, "name", "var"))))
            return result

    obj = _Distributed.__new__(_Distributed)
    obj.__dict__.update(optimizer.__dict__)
    return obj


class _DistributedGradientTape(object):
    def __init__(self, tape, device_dense, device_sparse, compression, sparse_as_dense):
        self._tape = tape
        self._args = (device_dense, device_sparse, compression, sparse_as_dense)

    def __getattr__(self, item):
        return getattr(self._tape, item)

    def __enter__(self):
        self._tape.__enter__()
        return self

    def __exit__(self, *exc):
        return self._tape.__exit__(*exc)

    def gradient(self, target, sources, output_gradients=None):
        grads = self._tape.gradient(target, sources, output_gradients)
        if size() <= 1:
            return grads
        flat = list(grads) if isinstance(grads, (list, tuple)) else [grads]
        srcs = list(sources) if isinstance(sources, (list, tuple)) else [sources]
        names = ["tape_grad_%d_%s" % (i, getattr(s, "name", "src")) for i, s in enumerate(srcs)]
        d, s, c, sad = self._args
        red = _reduce_grads(flat, names, d, s, c, sad, False, "DistributedGradientTape.")
        return red if isinstance(grads, (list, tuple)) else red[0]


def DistributedGradientTape(gradtape, device_dense="", device_sparse="", compression=Compression.none,
                            sparse_as_dense=False):
    """Wrap a ``tf.GradientTape``: ``gradient()`` returns gradients averaged over all workers."""
    return _DistributedGradientTape(gradtape, device_dense, device_sparse, compression, sparse_as_dense)


__all__ = ["init", "shutdown", "suspend", "resume", "size", "rank", "local_size", "local_rank", "push_pull",
           "broadcast", "broadcast_variables", "broadcast_global_variables", "BroadcastGlobalVariablesHook",
           "DistributedOptimizer", "DistributedGradientTape", "Compression", "Average", "Sum", "Adasum", "ReduceOps",
           "get_pushpull_speed", "handle_average_backwards_compatibility"]
