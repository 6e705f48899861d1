"""Symmetric (peer-mapped) workspaces for one NVSwitch box.

Every rank of a ring set allocates identically sized device regions through the C++ runtime
(``csrc/symm.cpp`` – cudaMalloc + CUDA IPC handles), exchanges the 64-byte handles once over
``torch.distributed`` and maps every peer's region.  After that the hot path never touches NCCL:

* kernels read peer K/V slots with bulk-TMA copies over NVLink (``attn_fwd_sm90.cu`` fetch warp);
* copy engines pull peer Q/dO/stat slots on a side stream in the backward;
* ranks synchronise with a device-side barrier on peer-mapped signal pads
  (``elementwise_sm90.cu:device_barrier_kernel``, ``st.release.sys`` / ``ld.acquire.sys``).

The reference does all of this with ``batch_isend_irecv`` + ``dist.barrier()`` per hop (ring.py:51-60).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from ring_attention_pytorch_b200.ops import _ext


@dataclass
class SymmRegion:
    """One symmetric allocation: local tensor (uint8) + base address of the same region on every ring rank."""
    local: torch.Tensor
    peer_ptrs: List[int]  # index = ring-local rank; own entry = local.data_ptr()
    nbytes: int


class RingWorkspace:
    """Symmetric staging buffers + signal pads shared by the ranks of one ring set."""

    def __init__(self, ring_ranks: List[int], device: torch.device, group=None):
        self.ring_ranks = list(ring_ranks)  # global ranks, ring order
        self.ring_size = len(ring_ranks)
        self.global_rank = dist.get_rank() if dist.is_initialized() else 0
        self.ring_rank = self.ring_ranks.index(self.global_rank)
        self.device = device
        self.group = group
        self.regions: Dict[str, SymmRegion] = {}
        self.uses: Dict[str, int] = {}
        self.epoch = 0
        self.side_stream = torch.cuda.Stream(device=device)
        self.pads = self._alloc("__pads__", 256)

    # -- allocation ---------------------------------------------------------------------------
    def _alloc(self, name: str, nbytes: int) -> SymmRegion:
        ops = _ext.ops()
        nbytes = (nbytes + 255) // 256 * 256
        local, handle = ops.symm_alloc(nbytes)
        if self.ring_size == 1:
            region = SymmRegion(local, [local.data_ptr()], nbytes)
        else:
            world = dist.get_world_size()
            gathered: List[Optional[Tuple[int, bytes]]] = [None] * world
            dist.all_gather_object(gathered, (self.global_rank, bytes(handle.numpy().tobytes())), group=self.group)
            by_rank = {r: h for r, h in gathered}
            ptrs = []
            for r in self.ring_ranks:
                if r == self.global_rank:
                    ptrs.append(local.data_ptr())
                else:
                    h = torch.frombuffer(bytearray(by_rank[r]), dtype=torch.uint8).clone()
                    ptrs.append(int(ops.symm_open(h)))
            region = SymmRegion(local, ptrs, nbytes)
        self.regions[name] = region
        return region

    def region(self, name: str, nbytes: int) -> SymmRegion:
        """Return a symmetric region of at least ``nbytes`` (collective on first use / growth).

        Growth retires the old region first.  Peers may still be reading it over NVLink (fused kernels, copy-engine
        pulls of the previous call), and freeing IPC-exported memory under an importer is undefined, so the retirement
        is a collective fence: every rank drains its own device work, all ranks meet, imports are closed, and only then
        is the exporting allocation released."""
        reg = self.regions.get(name)
        if reg is not None and reg.nbytes >= nbytes:
            return reg
        if reg is not None:
            self._retire(name)
        return self._alloc(name, nbytes)

    def _retire(self, name: str) -> None:
        reg = self.regions.pop(name)
        self.uses.pop(name, None)
        torch.cuda.synchronize(self.device)
        if self.ring_size > 1:
            dist.barrier(group=self.group)  # every rank has finished all work that could touch the old region
        ops = _ext.ops()
        for r, ptr in enumerate(reg.peer_ptrs):
            if r != self.ring_rank:
                ops.symm_close(ptr)
        if self.ring_size > 1:
            dist.barrier(group=self.group)  # all imports are closed: the exporters may free
        del reg  # drops the local tensor -> cudaFree through the from_blob deleter

    def close(self) -> None:
        """Release every region (collective).  Called at interpreter exit for the cached workspaces."""
        for name in list(self.regions):
            if name != "__pads__":
                self._retire(name)
        if "__pads__" in self.regions:
            self._retire("__pads__")

    def staging(self, name: str, nbytes: int) -> Tuple[torch.Tensor, List[int]]:
        """Double-buffered staging slot: returns (local uint8 view, peer base pointers of the same half).

        Alternating halves lets one cross-rank barrier per call suffice: a half is rewritten only two
        calls later, after every peer has signalled a barrier that it could only reach once its reads of
        that half were complete.
        """
        nbytes = (nbytes + 255) // 256 * 256
        reg = self.region(name, 2 * nbytes)
        half_bytes = reg.nbytes // 2
        use = self.uses.get(name, 0)
        self.uses[name] = use + 1
        off = (use % 2) * half_bytes
        return reg.local[off:off + nbytes], [p + off for p in reg.peer_ptrs]

    # -- synchronisation ----------------------------------------------------------------------
    def barrier(self) -> None:
        """Device-side barrier over the ring set on the current stream (no host sync, no NCCL)."""
        if self.ring_size == 1:
            return
        self.epoch += 1
        _ext.ops().device_barrier(self.pads.peer_ptrs, self.ring_rank, self.epoch)


_workspaces: Dict[Tuple[int, int, int], RingWorkspace] = {}


def close_workspaces() -> None:
    """Collective: retire every cached workspace (tests call it before tearing the process group down)."""
    for key in list(_workspaces):
        ws = _workspaces.pop(key)
        try:
            ws.close()
        except Exception:  # noqa: BLE001 - best effort at shutdown (the process group may already be gone)
            pass


def get_workspace(ring_size: int, device: torch.device) -> RingWorkspace:
    """Workspace of the ring set this rank belongs to (ranks ``[k*ring, (k+1)*ring)`` form ring set k,
    reference ring.py:35-47)."""
    rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
    ring_set = rank // ring_size
    key = (ring_size, ring_set, device.index if device.index is not None else torch.cuda.current_device())
    ws = _workspaces.get(key)
    if ws is None:
        ranks = list(range(ring_set * ring_size, (ring_set + 1) * ring_size))
        ws = RingWorkspace(ranks, device)
        _workspaces[key] = ws
    return ws
