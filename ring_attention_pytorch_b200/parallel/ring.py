"""Host-driven P2P ring for the portable (CPU / gloo, or NCCL without the sm_90a kernels) path.

The sm_90a path never touches this module: there the ring is a *schedule* evaluated inside the kernels
(``layout.ring_hop_owners`` -> ``hop_owner[]``) and K/V move with in-kernel bulk-TMA copies over NVLink.  The
portable path follows the same schedule — hop ``s`` of ring rank ``r`` holds the data of owner ``(r - s) mod W`` —
and realises it by actually rotating the tensors with point-to-point messages, so both backends share one definition
of "who is visited when" (:class:`RingTopology`).

The reference's functional surface (reference ring.py:27-124: ``circular_*``, ``ring_pass``, ``one_ring_pass``,
``null_ring_pass``, ``all_ring_pass``, ``RingInfo``) is kept for users that built on it.  Differences in behaviour:

* no ``dist.barrier()`` after every exchange (reference ring.py:57-60): a matched isend / irecv pair that has been
  waited on is already a complete point-to-point synchronisation;
* ``ring_pass`` honours ``num_ring_passes`` (reference ring.py:62-77 always moves one position);
* ranks and owners handed to callers are ring-local, also for ring sets (``ring_size < world_size``).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Iterator, List, NamedTuple, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
from torch import Tensor

from ring_attention_pytorch_b200.parallel.distributed import default, exists, get_rank, get_world_size


@dataclass(frozen=True)
class RingTopology:
    """One ring set: global ranks ``[base, base + size)``; ``local`` is this rank's position inside it."""
    size: int
    base: int
    local: int

    @classmethod
    def of(cls, rank: Optional[int] = None, ring_size: Optional[int] = None) -> "RingTopology":
        rank = default(rank, get_rank())
        size = max(1, default(ring_size, get_world_size()))
        return cls(size=size, base=(rank // size) * size, local=rank % size)

    def shifted(self, steps: int) -> int:
        """Ring-local index ``steps`` positions to the right (negative: left)."""
        return (self.local + steps) % self.size

    def to_global(self, local_index: int) -> int:
        return self.base + local_index % self.size

    def owner_at_hop(self, hop: int) -> int:
        """Ring-local rank whose shard this rank holds after ``hop`` exchanges (same rule as the kernels' schedule)."""
        return self.shifted(-hop)


# ---- reference-compatible index helpers (reference ring.py:27-47) -----------------------------------------------------
def circular_index_left(pos: int, ring_size: int, num: int = 1) -> int:
    return (pos - num) % ring_size


def circular_index_right(pos: int, ring_size: int, num: int = 1) -> int:
    return (pos + num) % ring_size


def circular_rank_left(rank: Optional[int] = None, ring_size: Optional[int] = None, num: int = 1) -> int:
    topo = RingTopology.of(rank, ring_size)
    return topo.to_global(topo.shifted(-num))


def circular_rank_right(rank: Optional[int] = None, ring_size: Optional[int] = None, num: int = 1) -> int:
    topo = RingTopology.of(rank, ring_size)
    return topo.to_global(topo.shifted(num))


# ---- data movement ---------------------------------------------------------------------------------------------------
def send_and_receive_(x: Tensor, receive_buffer: Tensor, send_to_rank: int, receive_from_rank: int) -> None:
    """One matched exchange; returns when both directions have completed."""
    work = dist.batch_isend_irecv([
        dist.P2POp(dist.isend, x, send_to_rank),
        dist.P2POp(dist.irecv, receive_buffer, receive_from_rank),
    ])
    for w in work:
        w.wait()


def ring_pass(num_ring_passes: int, x: Tensor, receive_buffer: Optional[Tensor] = None, ring_size: Optional[int] = None):
    """Move ``x`` ``num_ring_passes`` positions to the right around this rank's ring set.

    Returns ``(received, sent)``: the sent tensor can serve as the next receive buffer, which is how the portable ring
    op ping-pongs two allocations through all hops.
    """
    topo = RingTopology.of(ring_size=ring_size)
    x = x.contiguous()
    receive_buffer = torch.empty_like(x) if not exists(receive_buffer) else receive_buffer.contiguous()
    steps = num_ring_passes % topo.size
    if steps == 0:
        receive_buffer.copy_(x)
        return receive_buffer, x
    send_and_receive_(x, receive_buffer, topo.to_global(topo.shifted(steps)), topo.to_global(topo.shifted(-steps)))
    return receive_buffer, x


def one_ring_pass(x: Tensor, receive_buffer: Optional[Tensor] = None, ring_size: Optional[int] = None):
    return ring_pass(1, x, receive_buffer, ring_size)


class RingInfo(NamedTuple):
    ring_rank: int                 # ring-local rank of the shard currently held
    iter_info: Tuple[bool, bool]   # (first hop, last hop)


def null_ring_pass(*tensors, max_iters=None, receive_buffers=None, ring_size=None):
    """Degenerate ring of one hop (no communication): what the ring iterator yields without sequence parallelism."""
    yield RingInfo(0, (True, True)), (tensors, receive_buffers)


def all_ring_pass(*tensors, max_iters: Optional[int] = None, receive_buffers: Optional[Sequence] = None,
                  ring_size: Optional[int] = None) -> Iterator:
    """Visit the ring: yields, hop by hop, the tensors currently held and the ring-local rank that owns them.

    ``max_iters`` truncates the walk (causal look-back limits); ``None`` entries in ``tensors`` travel as ``None``.
    """
    topo = RingTopology.of(ring_size=ring_size)
    hops = max(1, min(topo.size, default(max_iters, topo.size)))
    held: List[Optional[Tensor]] = list(tensors)
    spare: List[Optional[Tensor]] = list(default(receive_buffers, (None,) * len(tensors)))
    for hop in range(hops):
        last = hop == hops - 1
        yield RingInfo(topo.owner_at_hop(hop), (hop == 0, last)), (held, spare)
        if last:
            break
        moved = [ring_pass(1, t, buf, topo.size) if exists(t) else (None, None) for t, buf in zip(held, spare)]
        held = [m[0] for m in moved]
        spare = [m[1] for m in moved]
