"""Multi-GPU sharding of the two hot paths (SURVEY.md §8e) — one process per GPU.

* HGEMM: row-sharded.  Rank r owns rows [r*rows, (r+1)*rows) of A and of C, B is
  replicated; after the step every rank holds the full C ("a single all-gather of C
  over NVLink").  Two transports:
    - ``nccl``  : GEMM into the rank's slice of C, then one in-place ncclAllGather
                  (the baseline the north star names);
    - ``fused`` : the GEMM epilogue stores every finished C tile straight into
                  the C buffer of every peer through NVLink-mapped pointers
                  (torch symmetric memory provides the peer mappings), so the transfer
                  overlaps the remaining MMA work tile by tile; a symmetric-memory
                  barrier closes the step.  Two symmetric C buffers alternate (see
                  ``RowShardedHgemm.fused`` for the ownership rule).
* Attention: the (batch x head) axis is embarrassingly parallel: `shard_heads` slices it,
  no collective.

The reference has no distributed layer at all (SURVEY §2.6); this file is new design,
not a port.
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch
import torch.distributed as dist

from . import _capi


def shard_range(n_units: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous, balanced [begin, end) slice of `n_units` independent units for `rank`."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError(f"bad world/rank {world}/{rank}")
    base, rem = divmod(n_units, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def shard_heads(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, world: int, rank: int):
    """Slice [B,H,N,D] tensors on the flattened (batch x head) axis; returns contiguous
    [1, units, N, D] views for this rank (attention needs no collective)."""
    B, H, N, D = q.shape
    b, e = shard_range(B * H, world, rank)
    f = lambda t: t.reshape(B * H, N, D)[b:e].unsqueeze(0)
    return f(q), f(k), f(v)


class RowShardedHgemm:
    """C[world*rows, N] = A[world*rows, K] @ B[K, N] with A/C row-sharded over ranks."""

    def __init__(self, rows: int, N: int, K: int, world: int, rank: int, device: torch.device,
                 transport: str = "nccl", group: Optional[dist.ProcessGroup] = None):
        if transport not in ("nccl", "fused"):
            raise ValueError(f"unknown transport {transport!r}")
        self.rows, self.N, self.K, self.world, self.rank = rows, N, K, world, rank
        self.device = device
        self.group = group
        self.transport = transport if world > 1 else "nccl"
        self._bufs = []       # fused: [(c_full, symm handle, multicast ptr, ctypes peer array)] x 2
        self._turn = 0
        if self.transport == "fused":
            # symmetric allocations: every rank's C buffer is mapped into every other rank
            # (NVLink P2P) and, where the fabric supports it, bound to one NVLS multicast object
            import ctypes
            import torch.distributed._symmetric_memory as symm_mem
            for _ in range(2):
                c = symm_mem.empty(rows * world, N, dtype=torch.half, device=device)
                h = symm_mem.rendezvous(c, group if group is not None else dist.group.WORLD)
                use_mc = bool(getattr(h, "has_multicast_support", False)) and \
                    os.environ.get("B200_FUSED_NO_MULTICAST", "0") != "1"
                mc = int(h.multicast_ptr) if use_mc else 0
                peers = [int(p_) for r, p_ in enumerate(h.buffer_ptrs) if r != rank]
                self._bufs.append((c, h, mc, (ctypes.c_void_p * max(1, len(peers)))(*peers)))
            self._n_peers = world - 1
            self.c_full = self._bufs[0][0]
        else:
            self.c_full = torch.empty(rows * world, N, dtype=torch.half, device=device)
        self.c_mine = self.c_full[rank * rows:(rank + 1) * rows]

    def compute_only(self, a_shard: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        rc = _capi.lib().b200_hgemm_f16_rows(a_shard.data_ptr(), b.data_ptr(), self.c_full.data_ptr(),
                                             self.rows, self.N, self.K, _capi.B_ROW_MAJOR_KN,
                                             self.rank * self.rows,
                                             torch.cuda.current_stream(self.device).cuda_stream)
        _capi.check(rc, "hgemm_rows")
        return self.c_mine

    def gather(self) -> torch.Tensor:
        """The exchange step: one in-place all-gather of the C row shards (the send buffer is this
        rank's slice of the receive buffer).  Device-agnostic (NCCL on GPUs, gloo in the CPU tests)."""
        if self.world > 1:
            dist.all_gather_into_tensor(self.c_full, self.c_mine, group=self.group)
        return self.c_full

    def fused(self, a_shard: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        """GEMM whose epilogue delivers each finished tile to every GPU (stores to the peer
        mappings, or through the NVLS multicast mapping), closed by a symmetric-memory barrier:
        after it, the returned [world*rows, N] tensor holds the complete C on every rank.

        Ownership rule.  Peers write into this rank's C while THEIR step runs, so a C buffer must
        not be handed back to the peers while this rank still reads it.  Two symmetric buffers
        alternate: step i writes buffer i % 2 and closes with barrier channel i % 2.  A peer can
        start step i+2 (which overwrites buffer i % 2) only after it passed the closing barrier of
        step i+1, which this rank enters — in stream order — only after everything it queued on
        the result of step i.  So: the tensor returned by a call stays valid until the call after
        the next one is issued; consume it (on the same stream) before then."""
        c_full, symm, mc_ptr, peer_array = self._bufs[self._turn]
        rc = _capi.lib().b200_hgemm_f16_rows_fused(
            a_shard.data_ptr(), b.data_ptr(), c_full.data_ptr(), mc_ptr,
            peer_array, self._n_peers, self.rows, self.N, self.K, _capi.B_ROW_MAJOR_KN,
            self.rank * self.rows, torch.cuda.current_stream(self.device).cuda_stream)
        _capi.check(rc, "hgemm_rows_fused")
        symm.barrier(channel=self._turn)
        self._turn ^= 1
        self.c_full = c_full
        self.c_mine = c_full[self.rank * self.rows:(self.rank + 1) * self.rows]
        return c_full

    def __call__(self, a_shard: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        if self.transport == "fused":
            return self.fused(a_shard, b)
        self.compute_only(a_shard, b)
        return self.gather()
