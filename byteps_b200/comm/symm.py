"""Symmetric-memory contexts: the python side of csrc/comm/symm_mem.cc.

A :class:`SymmContext` is one peer-mapped device allocation (data window +
signal pad) shared by all ranks of a job, plus the ``PeerView`` the kernels
take.  Creation is collective.  :class:`VirtualCluster` builds N "virtual
ranks" inside ONE process on ONE GPU, which lets the multi-peer kernels be
tested for numerics on a single H100 (the N kernels run concurrently on N
streams and synchronise through the same flag protocol).
"""
from __future__ import annotations

import uuid

import torch

from .. import _native
from ..utils.timing import stamp

_DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def wire_code(dtype: torch.dtype) -> int:
    try:
        return _DT[dtype]
    except KeyError:
        raise TypeError("push_pull on the CUDA path supports float32/bfloat16/float16, got %s" % dtype)


class _RawCuda:
    """Exposes a raw device pointer through __cuda_array_interface__ so torch
    can alias it without a C++ extension built against torch headers."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self.owner = owner
        self.__cuda_array_interface__ = {
            "shape": (nbytes,),
            "typestr": "|u1",
            "data": (ptr, False),
            "version": 2,
            "strides": None,
        }


def alias_tensor(ptr: int, nbytes: int, device: torch.device, owner=None) -> torch.Tensor:
    return torch.as_tensor(_RawCuda(ptr, nbytes, owner), device=device)


class SymmContext:
    def __init__(self, group, device: torch.device, data_bytes: int, mode: str = "auto", use_nvls: str = "auto"):
        cu = _native.cuda()
        self.cu = cu
        self.group = group
        self.rank, self.world = group.rank, group.world
        self.device = torch.device(device)
        dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        token = group.broadcast_object(uuid.uuid4().hex[:12] if group.rank == 0 else None, 0)
        if self.world == 1:
            mode = "local"
        stamp("symm: token broadcast")
        self.mem = cu.SymmMem(self.rank, self.world, dev_index, int(data_bytes), mode, token)
        stamp("symm: local allocation of %d MiB (%s)" % (int(data_bytes) >> 20, self.mem.mode))
        if self.world > 1:
            modes = group.all_gather_object(self.mem.mode)
            if len(set(modes)) != 1:  # someone fell back: everybody uses legacy IPC
                self.mem.close_server()
                group.barrier()
                self.mem = cu.SymmMem(self.rank, self.world, dev_index, int(data_bytes), "ipc", token + "x")
            infos = group.all_gather_object(self.mem.export_info())
            self.mem.import_peers(infos)
            stamp("symm: peers imported")
            group.barrier()
        self.nvls = False
        # auto: in-switch reduction from 4 peers up; with 2 peers plain P2P loads (fewer multimem protocol bytes
        # per useful byte)
        want_nvls = use_nvls in ("1", "try") or (use_nvls == "auto" and self.world >= 4)
        if self.world > 1 and want_nvls and self.mem.mode == "vmm":
            self._setup_multicast(required=(use_nvls == "1"))
        stamp("symm: multicast setup (nvls=%s)" % self.nvls)
        if self.world > 1:
            group.barrier()
            self.mem.close_server()
        self.view = self.mem.view()
        self.data_bytes = self.mem.data_bytes
        try:   # INFO: how the peers are mapped (docs/troubleshooting.md, docs/faq.md)
            _native.core().log(2, "symmetric memory: %d MiB, mode=%s, nvls=%s, world=%d" % (
                int(self.data_bytes) >> 20, self.mem.mode, self.nvls, self.world))
        except Exception:  # noqa: BLE001 - logging must never break set-up
            pass
        self.arena = alias_tensor(self.mem.local_ptr(), self.data_bytes, self.device, owner=self.mem)

    def _setup_multicast(self, required: bool):
        g = self.group
        ok = all(g.all_gather_object(bool(self.mem.mc_supported())))
        if ok:
            info = self.mem.mc_create() if self.rank == 0 else b""
            info = g.broadcast_object(info, 0)
            ok = len(info) > 0
        if ok:
            err = None
            try:
                self.mem.mc_join(info)
            except Exception as e:  # noqa: BLE001
                err = str(e)
            ok = all(e is None for e in g.all_gather_object(err))
        if ok:
            err = None
            try:
                self.mem.mc_bind()
            except Exception as e:  # noqa: BLE001
                err = str(e)
            ok = all(e is None for e in g.all_gather_object(err))
        self.nvls = bool(ok and self.mem.has_multicast())
        if required and not self.nvls:
            raise RuntimeError("BYTEPS_USE_NVLS=1 but NVLS multicast could not be set up")

    def tensor(self, off: int, numel: int, dtype: torch.dtype) -> torch.Tensor:
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        return self.arena[off:off + nbytes].view(dtype)

    def close(self):
        self.arena = None
        self.mem = None


class VirtualCluster:
    """N virtual ranks on one device, one process (tests / single-GPU numerics)."""

    def __init__(self, world: int, device, data_bytes: int):
        cu = _native.cuda()
        self.cu = cu
        self.world = world
        self.device = torch.device(device)
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.mems = [cu.SymmMem(0, 1, idx, int(data_bytes), "local", "v%d" % r) for r in range(world)]
        views = [m.view() for m in self.mems]
        data = [v.data_ptr(0) for v in views]
        sig = [v.sig_ptr(0) for v in views]
        self.views = [cu.PeerView(data=data, sig=sig, mc=0, epoch=views[r].epoch_ptr, rank=r, world=world)
                      for r in range(world)]
        self.data_bytes = self.mems[0].data_bytes
        self.arenas = [alias_tensor(m.local_ptr(), self.data_bytes, self.device, owner=m) for m in self.mems]
        self.streams = [torch.cuda.Stream(device=self.device) for _ in range(world)]

    def run(self, fn):
        """fn(rank, view, arena, stream_handle) launches one rank's kernel."""
        cur = torch.cuda.current_stream(self.device)
        for s in self.streams:
            s.wait_stream(cur)
        for r in range(self.world):
            fn(r, self.views[r], self.arenas[r], self.streams[r].cuda_stream)
        for s in self.streams:
            cur.wait_stream(s)


def pick_blocks(shard_bytes: int, threads: int, unroll_bytes: int, cap: int, sm_count: int = 132) -> int:
    """CTAs for an exchange: enough tiles in flight to cover the NVLink
    bandwidth-delay product (~2 us x 450 GB/s of NVLink 4 = 0.9 MB per GPU) without
    taking every SM away from the backward pass."""
    tile = threads * unroll_bytes
    need = max(1, (shard_bytes + tile - 1) // tile)
    return int(max(1, min(need, cap, sm_count)))
