"""Sequence layouts as position maps.

A *layout* says which global token position local index ``i`` on ring rank ``r`` holds.  Every layout
the reference supports is a piecewise-affine map with at most two segments, which is exactly what the
sm_90a kernels evaluate in registers (``csrc/attn_common.cuh``):

    i <  seg_len : base0[r] + stride * i
    i >= seg_len : base1[r] + stride * (i - seg_len)

* ``plain``   – rank r holds the contiguous chunk ``[r*n, (r+1)*n)``   (reference ring_attention.py:253-255)
* ``striped`` – rank r holds tokens ``i*W + r``                         (reference ring_attention.py:397-401 with
  ``striped_bucket_size = ring_seq_size``, the CUDA flavour; ring_flash_attention_cuda.py:157-160)
* ``zigzag``  – rank r holds chunks ``r`` and ``2W-1-r`` of ``2W``      (reference zig_zag_attention.py:62-69)
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List

import torch

LAYOUTS = ("plain", "striped", "zigzag")


@dataclass
class PositionMap:
    layout: str
    world: int
    n: int
    stride: int
    seg_len: int
    base0: List[int] = field(default_factory=list)
    base1: List[int] = field(default_factory=list)

    def positions(self, rank: int, device=None) -> torch.Tensor:
        i = torch.arange(self.n, device=device)
        first = self.base0[rank] + self.stride * i
        second = self.base1[rank] + self.stride * (i - self.seg_len)
        return torch.where(i < self.seg_len, first, second)

    def pos_range(self, rank: int):
        p = self.positions(rank)
        return int(p.min()), int(p.max())


def make_position_map(layout: str, world: int, n: int) -> PositionMap:
    assert layout in LAYOUTS, f"unknown layout {layout}"
    if layout == "plain":
        return PositionMap(layout, world, n, 1, n, [r * n for r in range(world)], [0] * world)
    if layout == "striped":
        return PositionMap(layout, world, n, world, n, list(range(world)), [0] * world)
    assert n % 2 == 0, "zig-zag layout needs an even local length"
    c = n // 2
    return PositionMap(layout, world, n, 1, c, [r * c for r in range(world)],
                       [(2 * world - 1 - r) * c for r in range(world)])


def ring_hop_owners(pm: PositionMap, rank: int, causal: bool, window: int | None, max_hops: int | None = None) -> List[int]:
    """Owners ring rank ``rank`` must visit, in ring order (itself first, then r-1, r-2, ...).

    An owner is dropped when no (query, key) pair between the two ranks can be visible, e.g. ranks
    ``> r`` under the plain causal layout (reference ring_flash_attention_cuda.py:161-165 skips their
    compute but still moves the data) or ranks beyond the look-back window.
    """
    owners = []
    qlo, qhi = pm.pos_range(rank)
    for s in range(pm.world):
        if max_hops is not None and s >= max_hops:
            break
        o = (rank - s) % pm.world
        if s > 0 and causal:
            klo, khi = pm.pos_range(o)
            if klo > qhi:
                continue
            if window is not None and window > 0 and qlo - khi > window:
                continue
        owners.append(o)
    return owners


def ring_query_owners(pm: PositionMap, rank: int, causal: bool, window: int | None) -> List[int]:
    """Ranks whose queries can see keys held by ``rank`` (itself first, then r+1, r+2, ...).

    Used by the KV-stationary backward kernel, which pulls Q / dO / lse / delta instead of K / V.
    """
    owners = []
    klo, khi = pm.pos_range(rank)
    for s in range(pm.world):
        o = (rank + s) % pm.world
        if s > 0 and causal:
            qlo, qhi = pm.pos_range(o)
            if klo > qhi:
                continue
            if window is not None and window > 0 and qlo - khi > window:
                continue
        owners.append(o)
    return owners


def to_layout(x: torch.Tensor, layout: str, world: int, dim: int = 1) -> torch.Tensor:
    """Permute a full sequence so that chunk ``r`` of the result is what rank ``r`` holds."""
    n_total = x.shape[dim]
    assert n_total % world == 0
    n = n_total // world
    pm = make_position_map(layout, world, n)
    idx = torch.cat([pm.positions(r, x.device) for r in range(world)])
    return x.index_select(dim, idx)


def from_layout(x: torch.Tensor, layout: str, world: int, dim: int = 1) -> torch.Tensor:
    """Inverse of :func:`to_layout`."""
    n_total = x.shape[dim]
    n = n_total // world
    pm = make_position_map(layout, world, n)
    idx = torch.cat([pm.positions(r, x.device) for r in range(world)])
    inv = torch.empty_like(idx)
    inv[idx] = torch.arange(n_total, device=x.device)
    return x.index_select(dim, inv)
