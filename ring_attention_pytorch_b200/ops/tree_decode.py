"""Tree-attention decoding: single-query attention over a KV cache sharded along the sequence across ranks
(reference tree_attn_decoding.py:23-104, Algorithm 3 of https://arxiv.org/abs/2408.04093).

Layout is head-first like the reference: ``q [b, h, m, d]`` (``m`` query tokens per sequence, 1 for plain decode),
``k [b, hk, n, d]``, ``v [b, hk, n, dv]``.

* CUDA path: ``csrc/tree_decode_tc_sm90.cu`` (head dim 128) / ``csrc/tree_decode_sm90.cu`` – ONE persistent cooperative kernel per rank and step computes the
  split-KV partials of its KV shard, merges the splits, publishes ``(out, lse)`` in symmetric memory, signals the
  peers and merges all ranks' partials in-kernel (NVLink peer loads, or ``multimem.ld_reduce`` through the NVSwitch
  when the buffers have a multicast mapping), replacing the reference's Triton launch padded to a 128-row tile plus
  three latency-bound all-reduces (MAX, SUM, SUM).
* portable path (CPU / gloo): local einsum attention + one MAX and one packed SUM all-reduce.

Fixes vs. the reference: ``shard_kv_seq=False`` with ``k=None`` works (reference uses an undefined ``dim_v``
– tree_attn_decoding.py:46 vs 84) by taking ``dim_v`` explicitly; grouped-query heads are supported.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist
from torch import Tensor

from ring_attention_pytorch_b200.parallel.distributed import default, exists, get_rank, get_world_size, is_distributed
from ring_attention_pytorch_b200.ops.paged_kv import gather_paged_kv
from ring_attention_pytorch_b200.utils.validate import (check_decode_query, check_decode_ranges, check_paged_kv, check_sinks,
                                                         typecheck)


def _visible_keys(n: int, cache_seqlens: Optional[Tensor], q_pos: Optional[Tensor], window: Optional[int],
                  kv_pos: tuple[int, int], b: int, device, m: int = 1) -> Tensor:
    """bool [b, m, n]: local key j of sequence b is visible to its query token t (see :func:`tree_attn_decode`)."""
    j = torch.arange(n, device=device, dtype=torch.int64)
    vis = torch.ones(b, m, n, dtype=torch.bool, device=device)
    if cache_seqlens is not None:
        vis &= j[None, None] < cache_seqlens.to(torch.int64)[:, None, None]
    if q_pos is not None:
        t = torch.arange(m, device=device, dtype=torch.int64)
        rel = (q_pos.to(torch.int64)[:, None] + t[None])[:, :, None] - (kv_pos[0] + kv_pos[1] * j)[None, None]
        vis &= rel >= 0
        if window is not None and window > 0:
            vis &= rel <= window
    return vis


def _local_attention(q: Tensor, k: Tensor, v: Tensor, visible: Optional[Tensor] = None, softclamp_value: float = 0.0):
    """q [b,h,m,d], k [b,hk,n,d], v [b,hk,n,dv] -> (out [b,h,m,dv] fp32, lse [b,h,m,1] fp32).  ``visible`` (bool
    [b, m, n]) masks keys per query token; a row that sees none gives out 0 and the finite sentinel lse
    ``-finfo.max``, so that the cross-rank merge of a row empty on every rank computes exp(0), never -inf - -inf."""
    b, h, m, d = q.shape
    hk = k.shape[1]
    g = h // hk
    scale = d ** -0.5
    qf = q.float().view(b, g, hk, m, d)  # query head j uses kv head j % hk
    sim = torch.einsum("bghid,bhjd->bghij", qf, k.float()) * scale
    if visible is not None:
        if softclamp_value > 0:
            sim = (sim / softclamp_value).tanh() * softclamp_value
        sim = sim.masked_fill(~visible[:, None, None, :, :], -float("inf"))
        lse = sim.logsumexp(dim=-1, keepdim=True)
        lse = torch.where(lse == -float("inf"), torch.full_like(lse, -torch.finfo(torch.float32).max), lse)
        # 0 * NaN is NaN: keys no token sees may hold anything
        vf = v.float().masked_fill(~visible.any(1)[:, None, :, None], 0.0)
        out = torch.einsum("bghij,bhjd->bghid", (sim - lse).exp(), vf)
        return out.reshape(b, h, m, -1), lse.reshape(b, h, m, 1)
    lse = sim.logsumexp(dim=-1, keepdim=True)
    attn = (sim - lse).exp()
    out = torch.einsum("bghij,bhjd->bghid", attn, v.float())
    return out.reshape(b, h, m, -1), lse.reshape(b, h, m, 1)


@torch.no_grad()
@typecheck
def tree_attn_decode(
    q: Tensor,
    k: Optional[Tensor] = None,
    v: Optional[Tensor] = None,
    eps: float = 1e-8,
    shard_kv_seq: bool = True,
    use_triton: Optional[bool] = None,
    dim_v: Optional[int] = None,
    sinks: Optional[Tensor] = None,
    cache_seqlens: Optional[Tensor] = None,
    q_pos: Optional[Tensor] = None,
    window: Optional[int] = None,
    softclamp_value: float = 0.0,
    kv_pos: Optional[tuple[int, int]] = None,
    block_table: Optional[Tensor] = None,
) -> Tensor:
    """``q [b, h, m, d]``; returns ``[b, h, m, dv]`` in ``q.dtype``.

    ``shard_kv_seq=True``: every rank passes the *full* K/V and attends to its own ``chunk(world)`` slice
    (ranks beyond the number of chunks contribute nothing).  ``shard_kv_seq=False``: K/V are already this
    rank's shard (``None`` for an empty shard).  ``use_triton`` is kept for signature parity and selects the
    sm_90a kernel (default: on CUDA inputs).

    ``sinks`` (floating ``[h]``): learned attention sinks, one logit per query head with a zero value vector.  The
    softmax runs over the keys of every rank and the sink, which is added once, in the cross-rank merge.

    Ragged and windowed decode: key ``j`` of a rank's K/V sits at global position ``P(j) = offset + stride * j`` and is
    visible to sequence ``b`` iff ``j < cache_seqlens[b]`` (int32 ``[b]``, the keys held), ``P(j) <= q_pos[b]``
    (integer ``[b]``) and, with ``window > 0``, ``q_pos[b] - P(j) <= window`` -- the look-back rule of the ring op.
    With ``shard_kv_seq=True`` the lengths and positions are global and each rank derives its own from its
    ``chunk`` (``offset = rank * chunk``, ``stride = 1``); with ``shard_kv_seq=False`` they are this rank's and
    ``kv_pos = (offset, stride)`` places its keys (required with ``q_pos`` on more than one rank; e.g. ``(rank,
    world)`` for round-robin appends).  ``softclamp_value > 0``: logits ``c * tanh(s / c)`` (the sink is not clamped).
    A row that sees no key on any rank and has no sink gives 0.

    Multi-token decode (``m > 1``, e.g. verifying ``m`` draft tokens in one pass over the cache): query token ``t``
    sits at ``q_pos[b] + t`` and sees key ``j`` iff the rule above holds at that position, so the tokens are causal
    among themselves.  The caller appends the tokens' K/V first and counts them in ``cache_seqlens``.  Without
    ``q_pos`` there is no position rule and every token sees every held key -- speculative verification needs
    ``q_pos``.  GQA, softclamp, sinks (once per token row) and the cache formats apply per token row.

    Paged KV cache: with ``block_table`` (int32 ``[b, max_pages]``) ``k`` / ``v`` are this rank's page pools
    ``[num_pages, hk, page_size, d]`` (or an NHD pool passed as ``.transpose(1, 2)``), and local key ``j`` of sequence
    ``b`` is ``pool[block_table[b, j // page_size], :, j % page_size]``: the call equals the one on
    ``gather_paged_kv(pool, block_table)`` (``ops/paged_kv.py``).  It needs ``shard_kv_seq=False`` (each rank passes
    its own pools, table, ``cache_seqlens`` and ``kv_pos``) and ``cache_seqlens``; ``page_size`` is 16, 32 or a
    multiple of 64.  Entries of pages that hold no key visible to any token of the call are never read (they may name a
    freed page); entries are not checked and must lie in ``[0, num_pages)``.
    """
    assert not (exists(k) ^ exists(v)), "keys and values are either both None, or both present"
    check_decode_query(q, name="tree_attn_decode")
    dtype = q.dtype
    b, h, m = q.shape[:3]
    check_sinks(sinks, h, q.device, name="tree_attn_decode")
    check_decode_ranges(b, q.device, cache_seqlens, q_pos, window, kv_pos, softclamp_value, name="tree_attn_decode")
    if exists(block_table) and shard_kv_seq:
        raise ValueError("tree_attn_decode: a paged cache (block_table) needs shard_kv_seq=False: each rank passes its "
                         "own page pools and table")
    check_paged_kv(b, q.device, k, v, block_table, cache_seqlens, name="tree_attn_decode")
    ranged = exists(cache_seqlens) or exists(q_pos) or softclamp_value > 0
    if exists(v):
        dim_v = v.shape[-1]

    if shard_kv_seq:
        assert exists(k), "keys and values must be passed if not already sharded across sequence"
        if exists(kv_pos):
            raise ValueError("tree_attn_decode: kv_pos is derived from the chunk with shard_kv_seq=True")
        rank, world = get_rank(), get_world_size()
        ks, vs = k.chunk(world, dim=-2), v.chunk(world, dim=-2)
        k, v = (ks[rank], vs[rank]) if rank < len(ks) else (None, None)
        if ranged and exists(k):
            offset = rank * ks[0].shape[-2]
            kv_pos = (offset, 1)
            if exists(cache_seqlens):
                cache_seqlens = (cache_seqlens - offset).clamp(0, k.shape[-2]).to(torch.int32)
    elif exists(q_pos) and not exists(kv_pos) and is_distributed() and get_world_size() > 1:
        raise ValueError("tree_attn_decode: kv_pos = (offset, stride) of this rank's keys is required with q_pos "
                         "when the cache is sharded over more than one rank")
    kv_pos = default(kv_pos, (0, 1))
    assert exists(dim_v), "dim_v is required when this rank holds no keys"

    use_kernel = default(use_triton, q.is_cuda)
    assert not (use_kernel and not q.is_cuda), "input needs to be on cuda to use the sm_90a kernel"

    if use_kernel:
        from ring_attention_pytorch_b200.ops.tree_decode_cuda import tree_decode_cuda

        if ranged:
            return tree_decode_cuda(q, k, v, dim_v=dim_v, eps=eps, sinks=sinks, cache_seqlens=cache_seqlens, q_pos=q_pos,
                                    window=window, kv_pos=kv_pos, softclamp_value=softclamp_value,
                                    block_table=block_table).to(dtype)
        return tree_decode_cuda(q, k, v, dim_v=dim_v, eps=eps, sinks=sinks).to(dtype)

    if exists(block_table):
        k, v = gather_paged_kv(k, block_table), gather_paged_kv(v, block_table)
    if exists(k) and k.shape[-2] > 0 and ranged:
        visible = _visible_keys(k.shape[-2], cache_seqlens, q_pos, window, kv_pos, b, q.device, m)
        local_out, lse = _local_attention(q, k, v, visible, softclamp_value)
    elif exists(k) and k.shape[-2] > 0:
        local_out, lse = _local_attention(q, k, v)
    else:
        local_out = q.new_zeros((b, h, m, dim_v), dtype=torch.float32)
        lse = torch.full((b, h, m, 1), -torch.finfo(torch.float32).max, device=q.device, dtype=torch.float32)

    if not is_distributed() and not exists(sinks):
        return local_out.to(dtype)

    max_lse = lse.clone()
    if is_distributed():
        dist.all_reduce(max_lse, dist.ReduceOp.MAX)
    if exists(sinks):
        sink = sinks.float().view(1, h, 1, 1)
        max_lse = torch.maximum(max_lse, sink)
    den = (lse - max_lse).exp()
    packed = torch.cat((local_out * den, den), dim=-1)  # numerator | denominator in one collective
    if is_distributed():
        dist.all_reduce(packed)
    num, den = packed[..., :-1], packed[..., -1:]
    if exists(sinks):  # the sink joins the merged denominator once, after the reduction
        den = den + (sink - max_lse).exp()
    return (num / den.clamp(min=eps)).to(dtype)
