"""GPU gradient compression with error feedback, exchanged over NVLink.

Same algorithms and kwargs as the CPU compressors in csrc/compress (and the
reference's /root/reference/byteps/common/compressor): onebit (+scaling), topk,
randomk, dithering (linear|natural x max|l2), vanilla error feedback with the
lr ratio, nesterov momentum.  Pipeline for one tensor, all on one stream:

    producer  ONE pass: momentum + error feedback + compress (sign words / first radix
              histogram); the corrected value replaces the error state in place; norms and
              histogram picks are finished by the last block to leave, in a fixed order
    push      the payload is copied into EVERY peer's window (coalesced 16-byte stores over
              NVLink) and the same kernel ends in the flag barrier
    consumer  reads local memory only: decompress all payloads + sum + the "server" stage
              (second error feedback + recompression) + the worker's own error update in one
              sweep, then one pass that writes the user's tensor (x 1/size when averaging)

(csrc/kernels/compress_fused.cu; dithering quantises with the kernels of compress.cu and uses the same
push + local-sum exchange, and random-k scatters its sums with compress.cu's index_scatter.)

The second stage reproduces the reference's server-side compression
(server.cc:92-118) so results follow the same two-stage contract its tests
check; every rank computes it redundantly from the same data, bit-identically.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from ..comm.symm import SymmContext, wire_code


def _k_of(kw: Dict[str, str], numel: int) -> int:
    f = float(kw["compressor_k"])
    if f <= 0:
        raise ValueError("compressor_k must be positive")
    if f < 1:
        return max(1, int(f * numel))
    return min(int(f), int(numel))        # an absolute k larger than a small tensor keeps everything


class GpuCompressor:
    @staticmethod
    def payload_bytes_for(kwargs: Dict[str, str], numel: int, world: int = 1) -> int:
        """Bytes of symmetric memory one tensor's payload window needs: `world` slots (one per
        sender), double buffered by step parity."""
        return 2 * max(1, world) * GpuCompressor.slot_bytes_for(kwargs, numel)

    @staticmethod
    def slot_bytes_for(kwargs: Dict[str, str], numel: int) -> int:
        kw = {str(k): str(v) for k, v in kwargs.items()}
        kind, n = kw.get("compressor_type"), int(numel)
        if kind == "onebit":
            b = (n + 31) // 32 * 4 + 4
        elif kind == "topk":
            b = _k_of(kw, n) * 8
        elif kind == "randomk":
            b = _k_of(kw, n) * 4
        elif kind == "dithering":
            b = (n + 15) // 16 * 16 + 16
        else:
            raise ValueError("unknown compressor_type %r" % kind)
        return (b + 255) // 256 * 256

    def __init__(self, ctx: SymmContext, kwargs: Dict[str, str], numel: int, dtype: torch.dtype, payload_off: int = 0,
                 two_stage: bool = True):
        self.ctx, self.cu = ctx, ctx.cu
        self.kw = {str(k): str(v) for k, v in kwargs.items()}
        self.kind = self.kw.get("compressor_type")
        if self.kind not in ("onebit", "topk", "randomk", "dithering"):
            raise ValueError("unknown compressor_type %r" % self.kind)
        self.n, self.dtype, self.off = int(numel), dtype, int(payload_off)
        self.code = wire_code(dtype)
        dev = ctx.device
        cu = self.cu
        self.use_ef = self.kw.get("ef_type") == "vanilla"
        self.mu = float(self.kw["momentum_mu"]) if self.kw.get("momentum_type") == "nesterov" else None
        self.two_stage = two_stage
        f32 = dict(dtype=torch.float32, device=dev)
        n = self.n
        self.err = torch.zeros(n, **f32) if self.use_ef else None
        self.err2 = torch.zeros(n, **f32) if (self.use_ef and two_stage) else None
        self.mom = torch.zeros(n, **f32) if self.mu is not None else None
        self.lr_prev = self.lr_cur = 1.0
        self.step = 0
        self.slot_bytes = self.slot_bytes_for(self.kw, n)
        self.payload_bytes = 2 * ctx.world * self.slot_bytes          # whole window: [parity][sender]
        if self.off % 256 or self.off + self.payload_bytes > ctx.data_bytes:
            raise ValueError("payload window does not fit in the arena")
        self.parts = torch.zeros(cu.FUSED_MAX_BLOCKS, **f32)
        self.counter = torch.zeros(4, dtype=torch.int32, device=dev)
        # CTAs of the push kernel (each owns a flag-barrier slot); payloads are small
        self.blocks = 1
        if self.kind == "onebit":
            self.scaled = self.kw.get("compressor_onebit_scaling", "false").lower() in ("1", "true", "yes")
            self.wire_bytes = (n + 31) // 32 * 4 + 4
            self.scratch = None if self.use_ef else torch.empty(n, **f32)     # c2 when there is no err2 to hold it
            self.scale2 = torch.zeros(4, **f32)
        elif self.kind == "topk":
            self.k = _k_of(self.kw, n)
            self.wire_bytes = self.k * 8
            self.scratch = torch.empty(n, **f32)          # corrected tensor without EF / summed payloads without err2
            self.tk = torch.zeros(cu.TOPK_SCRATCH_BYTES // 4, dtype=torch.int32, device=dev)
            self.local2 = torch.empty(2 * self.k, dtype=torch.int32, device=dev)
        elif self.kind == "randomk":
            self.k = _k_of(self.kw, n)
            self.wire_bytes = self.k * 4
            seed = (int(self.kw.get("seed", "0")) or 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
            sseed = seed - (1 << 64) if seed >= (1 << 63) else seed
            # the CPU compressors' xorshift128+ streams (worker stage and "server" stage), advanced ON THE
            # DEVICE: the generator is linear over GF(2), so every thread jumps to its chunk of the stream
            self.rng_state = torch.tensor([sseed, sseed], dtype=torch.int64, device=dev)
            self.rng_state2 = torch.tensor([sseed, sseed], dtype=torch.int64, device=dev)
            self.jump = torch.frombuffer(bytearray(cu.xorshift_jump_table()), dtype=torch.int64).to(dev)
            self.idx = torch.empty(self.k, dtype=torch.int32, device=dev)
            self.idx2 = torch.empty(self.k, dtype=torch.int32, device=dev)
            self.vals = torch.empty(self.k, **f32)
            self.vals2 = torch.empty(self.k, **f32)
            self.scratch = torch.empty(n, **f32)
        else:
            self.s = int(float(self.kw["compressor_k"]))
            self.partition = int(self.kw.get("dithering_partition", "0"))
            self.normalize = int(self.kw.get("dithering_normalize", "0"))
            self.seed = int(self.kw.get("seed", "0")) or 12345
            self.lv_bytes = (n + 15) // 16 * 16
            self.wire_bytes = self.lv_bytes + 16
            self.levels2 = torch.empty(self.lv_bytes, dtype=torch.int8, device=dev)
            self.scale2 = torch.empty(4, **f32)
            self.corrected = torch.empty(n, **f32)
            self.sum = torch.empty(n, **f32)
            self.acc = torch.zeros(4 + 3 * 132 * 8, **f32)   # results + per-block partials (kEfAccFloats)
        self.blocks = max(1, min(128, (self.wire_bytes + 65535) // 65536))
        self.payload = ctx.arena[self.off:self.off + self.payload_bytes]

    def set_lr(self, lr: float):
        self.lr_cur = float(lr)

    def _window(self, parity: int):
        """(arena offset of the window of this parity, device pointer of its first slot, of my slot)"""
        off = self.off + parity * self.ctx.world * self.slot_bytes
        base = self.ctx.arena.data_ptr() + off
        return off, base, base + self.ctx.rank * self.slot_bytes

    # ------------------------------------------------------------------
    def push_pull(self, grad: torch.Tensor, out: Optional[torch.Tensor] = None, average: bool = True, stream=None):
        """grad -> out (defaults to grad, in place)."""
        st = stream or torch.cuda.current_stream(self.ctx.device)
        with torch.cuda.stream(st):
            for phase in self.phases(grad, out, average, st.cuda_stream):
                phase()
        return grad if out is None else out

    def phases(self, grad, out, average, s):
        """The pipeline as a list of closures.  Odd entries are the cross-rank kernels (they
        spin on peer flags); a single-process multi-rank harness must issue each phase for ALL
        virtual ranks before the next one, so no spinning kernel sits in front of a peer's work
        in a shared hardware queue."""
        cu, ctx, n = self.cu, self.ctx, self.n
        out = grad if out is None else out
        assert grad.numel() == n and grad.dtype == self.dtype and grad.is_contiguous() and out.is_contiguous()
        if grad.data_ptr() % 16 or out.data_ptr() % 16:
            raise ValueError("compressed push_pull needs 16-byte aligned tensors")
        world, me = ctx.world, ctx.rank
        mult = (1.0 / world) if average else 1.0
        ratio = (self.lr_prev / self.lr_cur) if self.lr_cur > 0 else 1.0
        self.lr_prev = self.lr_cur
        self.step += 1
        step = self.step
        err = self.err.data_ptr() if self.err is not None else 0
        e2 = self.err2.data_ptr() if self.err2 is not None else 0
        mom = self.mom.data_ptr() if self.mom is not None else 0
        mu = self.mu or 0.0
        kind = self.kind
        g, o = grad.data_ptr(), out.data_ptr()
        win_off, slots, mine = self._window(step & 1)
        parts, counter = self.parts.data_ptr(), self.counter.data_ptr()

        def push():
            cu.payload_push(ctx.view, win_off, self.slot_bytes, self.wire_bytes, self.blocks, 0, s)

        if kind == "onebit":
            c2 = (e2 or self.scratch.data_ptr()) if self.two_stage else 0

            def pre():
                # p -> err (in place), sign words + mean|p| -> my slot
                cu.onebit_pre(g, self.code, mom, mu, err, ratio, err, n, mine, self.scaled, parts, counter, s)

            def post():
                cu.onebit_sum(slots, self.slot_bytes, world, me, n, err, e2, c2, o, self.code, mult, self.scaled,
                              parts, counter, self.scale2.data_ptr(), s)
                if self.two_stage:
                    cu.onebit_out(c2, n, self.scale2.data_ptr(), e2, o, self.code, mult, s)
            return [pre, push, post]
        if kind == "topk":
            p_buf = err or self.scratch.data_ptr()
            tk = self.tk.data_ptr()

            def pre():
                cu.topk_pre(g, self.code, mom, mu, err, ratio, p_buf, n, self.k, tk, s)
                cu.topk_finish(p_buf, n, self.k, 1, mine, bool(err), tk, s)     # kept entries zeroed: err is final

            def post():
                # c2 = sum of the payloads (+ err2): scatter-added in rank order, unique indices per payload
                if e2:
                    acc = e2
                else:
                    acc = self.scratch.data_ptr()
                    self.scratch.zero_()
                for p in range(world):
                    cu.sparse_add_pairs(slots + p * self.slot_bytes, self.k, n, acc, s)
                if self.two_stage:
                    cu.topk_finish(acc, n, self.k, 0, self.local2.data_ptr(), bool(e2), tk, s)
                    cu.scatter_pairs(self.local2.data_ptr(), self.k, n, o, self.code, mult, s)
                else:
                    cu.cast_scale4(acc, n, o, self.code, mult, s)
            return [pre, push, post]
        if kind == "randomk":
            def pre():
                cu.randomk_draw(self.rng_state.data_ptr(), self.jump.data_ptr(), self.k, n, self.idx.data_ptr(), s)
                cu.randomk_pre(g, self.code, mom, mu, err, ratio, n, self.idx.data_ptr(), self.k, mine, s)

            def post():
                cu.dense_sum_slots(slots, self.slot_bytes, world, self.k, self.vals.data_ptr(), s)
                if self.two_stage:
                    # server: D(worker payloads) summed = scatter(idx, vals); then its own random-k draw
                    sm = self.scratch.data_ptr()
                    cu.index_scatter(self.idx.data_ptr(), self.vals.data_ptr(), self.k, n, sm, 0, 1.0, s)
                    cu.randomk_draw(self.rng_state2.data_ptr(), self.jump.data_ptr(), self.k, n,
                                    self.idx2.data_ptr(), s)
                    # err2 += sum (dense), gather at idx2, zero the kept entries of err2
                    cu.randomk_pre(sm, 0, 0, 0.0, e2, 1.0, n, self.idx2.data_ptr(), self.k, self.vals2.data_ptr(), s)
                    cu.index_scatter(self.idx2.data_ptr(), self.vals2.data_ptr(), self.k, n, o, self.code, mult, s)
                else:
                    cu.index_scatter(self.idx.data_ptr(), self.vals.data_ptr(), self.k, n, o, self.code, mult, s)
            return [pre, push, post]

        # ---- dithering: quantise into my slot, push, sum the local slots
        pay = mine
        cor, acc, sm = self.corrected.data_ptr(), self.acc.data_ptr(), self.sum.data_ptr()

        def pre():
            cu.ef_correct(g, self.code, mom, mu, err, ratio, cor, n, acc, s)
            cu.dither_quantize(cor, n, acc, self.s, self.partition, self.normalize, self.seed, step, pay,
                               pay + self.lv_bytes, err, s)

        def post():
            cu.dither_sum_slots(slots, self.slot_bytes, world, n, self.s, self.partition, sm, s)
            if self.two_stage:
                cu.ef_correct(sm, 0, 0, 0.0, e2, 1.0, cor, n, acc, s)
                cu.dither_quantize(cor, n, acc, self.s, self.partition, self.normalize, self.seed ^ 0x5555, step,
                                   self.levels2.data_ptr(), self.scale2.data_ptr(), e2, s)
                cu.dither_unpack(self.levels2.data_ptr(), self.scale2.data_ptr(), n, self.s, self.partition,
                                 o, self.code, mult, s)
            else:
                cu.cast_scale(sm, n, o, self.code, mult, s)
        return [pre, push, post]
