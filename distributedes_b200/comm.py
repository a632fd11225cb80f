"""Peer-memory exchange for a sharded generation (csrc/des_comm.cu): one process per GPU on one node.

torch.distributed is used once, to hand every rank the 64-byte cudaIpc handles of the others; after that the two
exchange steps of a generation (fitness all-gather, partial all-reduce) are kernels of this library storing into the
peers' memory over NVLink — no NCCL call on the hot path, and the whole generation can be captured in a CUDA graph.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.distributed as dist

from . import _lib
from .ops import _ptr


class _DevArray:
    """Exposes a raw device pointer through __cuda_array_interface__ so torch can alias it (no copy, no ownership)."""

    def __init__(self, ptr, n, owner):
        self.__cuda_array_interface__ = {'shape': (int(n),), 'typestr': '<f4', 'data': (int(ptr), False), 'version': 2}
        self._owner = owner


class PeerComm:
    """The exchange among the ranks of `group` (an engine.RankGroup)."""

    def __init__(self, N, P, device, group):
        self.lib = _lib.load()
        self.rank, self.world = group.rank, group.world
        self.device = torch.device(device)
        self.N, self.P = int(N), int(P)
        self._h = C.c_void_p()
        handle = (C.c_ubyte * 64)()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.des_comm_create(C.byref(self._h), self.rank, self.world, self.N, self.P, handle), 'des_comm_create')
            mine = torch.tensor(list(bytes(handle)), dtype=torch.uint8, device=self.device)
            every = [torch.empty_like(mine) for _ in range(self.world)]
            dist.all_gather(every, mine, group=group.pg)
            blob = b''.join(bytes(t.cpu().numpy().tobytes()) for t in every)
            buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
            _lib.check(self.lib.des_comm_connect(self._h, buf), 'des_comm_connect')
            ptr = self.lib.des_comm_fitness_all_dev(self._h)
            self.fitness_all = torch.as_tensor(_DevArray(ptr, self.N, self), device=self.device)
            dist.barrier(group=group.pg)                 # every block is mapped before anyone stores into a peer

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def allgather_fitness(self, member_offset, n_local):
        _lib.check(self.lib.des_comm_allgather_fitness(self._h, int(member_offset), int(n_local), self._stream()),
                   'des_comm_allgather_fitness')

    def allreduce_partial(self, partial_local, out):
        dev = self.fitness_all.device
        _lib.check(self.lib.des_comm_allreduce_partial(self._h, _ptr(out, 'out', torch.float32, self.P, dev),
                                                       _ptr(partial_local, 'partial_local', torch.float32, self.P, dev),
                                                       self.P, self._stream()), 'des_comm_allreduce_partial')

    def close(self):
        if self._h:
            self.fitness_all = None
            self.lib.des_comm_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
