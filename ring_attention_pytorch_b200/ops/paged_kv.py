"""Paged KV caches for tree decode: K / V live in a pool of fixed-size pages and a per-sequence block table maps local
key ``j`` of sequence ``b`` to slot ``j % page_size`` of page ``block_table[b, j // page_size]``.

A pool is ``[num_pages, hk, page_size, d]`` (HND), or an NHD pool ``[num_pages, page_size, hk, d]`` passed as
``.transpose(1, 2)``; ``block_table`` is int32 ``[b, max_pages]``.  Both helpers are plain PyTorch, hide the page
arithmetic and make no host sync, so they can run inside a decode loop that replays a captured CUDA graph.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor


def _bits(t: Tensor) -> Tensor:
    """The same memory as an integer tensor of the same element size: indexing copies the bits of any dtype (the
    float8 types have no CPU gather / index_put)."""
    if t.is_floating_point() and t.element_size() == 1:
        return t.view(torch.uint8)
    return t


def gather_paged_kv(pool: Tensor, block_table: Tensor, n: Optional[int] = None) -> Tensor:
    """``pool [num_pages, hk, page_size, d]`` and ``block_table [b, max_pages]`` -> the contiguous cache
    ``[b, hk, n, d]`` (default ``n = max_pages * page_size``) whose key ``j`` is ``pool[block_table[b, j // page_size],
    :, j % page_size]``.  A paged decode call computes exactly what the contiguous call on this cache computes."""
    num_pages, hk, ps, d = pool.shape
    b, max_pages = block_table.shape
    n = max_pages * ps if n is None else n
    if not 0 <= n <= max_pages * ps:
        raise ValueError(f"gather_paged_kv: n must be in [0, max_pages * page_size = {max_pages * ps}], got {n}")
    pages = _bits(pool)[block_table.long()]  # [b, max_pages, hk, page_size, d]
    out = pages.permute(0, 2, 1, 3, 4).reshape(b, hk, max_pages * ps, d)[:, :, :n]
    return out.contiguous().view(pool.dtype)


@torch.no_grad()
def write_paged_kv(k_pool: Tensor, v_pool: Tensor, block_table: Tensor, start: Tensor, k_new: Tensor,
                   v_new: Tensor) -> None:
    """Write ``t`` new tokens per sequence, ``k_new`` / ``v_new [b, hk, t, d]``, at local positions ``start[b] ..
    start[b] + t - 1`` (``start``: integer ``[b]`` on the pools' device) into the pages the table maps them to.  The
    values are cast to the pools' dtype.  The pages must already be in the table."""
    ps = k_pool.shape[2]
    b, hk, t, d = k_new.shape
    pos = start.to(torch.int64)[:, None] + torch.arange(t, device=start.device)[None]  # [b, t]
    page = block_table.long().gather(1, pos // ps)
    slot = pos % ps
    for pool, new in ((k_pool, k_new), (v_pool, v_new)):
        # advanced indices around a slice: the indexed view is [b, t, hk, d]
        _bits(pool)[page, :, slot] = _bits(new.to(pool.dtype)).permute(0, 2, 1, 3)
