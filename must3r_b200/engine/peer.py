"""Peer-visible device memory for the multi-GPU schedule: buffers allocated by the library (cudaMalloc), exported as CUDA
IPC handles, exchanged with torch.distributed and mapped by every other rank of the node, so that a GEMM epilogue on one
GPU can store K|V rows straight into the memory buffers of all GPUs over NVLink (SURVEY.md §8e)."""
from __future__ import annotations

import ctypes as C
from typing import List

import torch
import torch.distributed as dist

from .. import _lib


class _RawCudaBuffer:
    """Minimal __cuda_array_interface__ holder so torch can view library-owned device memory without copying."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}


class PeerArena:
    """`nbytes` of device memory on every rank; ``local`` is a uint8 torch view of this rank's block,
    ``ptrs[r]`` the address of rank r's block as seen from this process (own block: the local address).
    Behind the block sit `FLAG_BYTES` of barrier flags: a uint32 slot per rank (m3r_peer_signal / m3r_peer_wait)."""

    FLAG_BYTES = 256

    def __init__(self, nbytes: int, device: torch.device):
        lib = _lib.lib()
        rank, world = dist.get_rank(), dist.get_world_size()
        self.nbytes, self.device, self._opened = nbytes, device, []
        self.rank, self.world, self.epoch = rank, world, 0
        nbytes_al = (nbytes + 255) // 256 * 256
        p = C.c_void_p()
        _lib.check(lib.m3r_peer_alloc(nbytes_al + self.FLAG_BYTES, C.byref(p)), "peer_alloc")
        self.ptr = p.value
        self.flag_off = nbytes_al
        whole = torch.as_tensor(_RawCudaBuffer(self.ptr, nbytes_al + self.FLAG_BYTES), device=device)
        whole[nbytes_al:].zero_()
        torch.cuda.synchronize(device)
        self.local = whole[:nbytes]
        handle = (C.c_uint8 * 64)()
        _lib.check(lib.m3r_ipc_export(C.c_void_p(self.ptr), handle), "ipc_export")
        mine = torch.tensor(list(handle), dtype=torch.uint8, device=device)
        allh = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(allh, mine)
        self.ptrs: List[int] = []
        for r in range(world):
            if r == rank:
                self.ptrs.append(self.ptr)
                continue
            hb = (C.c_uint8 * 64)(*allh[r].cpu().tolist())
            q = C.c_void_p()
            _lib.check(lib.m3r_ipc_open(hb, C.byref(q)), "ipc_open")
            self.ptrs.append(q.value)
            self._opened.append(q.value)
        dist.barrier()
        self._slots = (C.c_void_p * world)(*[self.ptrs[r] + self.flag_off + 4 * rank for r in range(world)])

    # ---- device-side barrier: no host synchronisation, the launch thread keeps enqueueing
    def signal(self, stream_ptr):
        """Publish the next epoch to every rank once the work enqueued so far on the stream has completed."""
        self.epoch += 1
        _lib.check(_lib.lib().m3r_peer_signal(self._slots, self.world, self.epoch, stream_ptr), "peer_signal")

    def skip_epoch(self):
        """A round this rank sits out: keep the epoch counters of all ranks in step."""
        self.epoch += 1

    def wait(self, ranks, stream_ptr):
        """Work enqueued after this sees everything the given ranks stored before signalling the current epoch."""
        mask = 0
        for r in ranks:
            mask |= 1 << r
        if mask:
            _lib.check(_lib.lib().m3r_peer_wait(C.c_void_p(self.ptr + self.flag_off), mask, self.epoch, stream_ptr), "peer_wait")

    def close(self):
        lib = _lib.lib()
        torch.cuda.synchronize(self.device)
        dist.barrier()
        for q in self._opened:
            lib.m3r_ipc_close(C.c_void_p(q))
        self._opened = []
        dist.barrier()
        if self.ptr:
            self.local = None
            lib.m3r_peer_free(C.c_void_p(self.ptr))
            self.ptr = 0
