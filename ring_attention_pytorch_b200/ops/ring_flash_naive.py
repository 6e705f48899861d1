"""Portable ring flash attention (pure PyTorch autograd Function, CPU/gloo or any device).

This is the semantic specification of the framework and the path that runs without a GPU
(CPU or any device).  Capability parity with reference ring_flash_attention.py:60-406, re-derived around position
maps instead of bucket bookkeeping:

* one code path for plain, striped and zig-zag layouts (visibility = ``pos_q >= pos_k``);
* exact token look-back windows (``pos_q - pos_k <= max_lookback_seq_len``);
* grouped-query attention without materialising repeated K/V on the ring (only kv heads travel);
* **correct dK/dV**: the (k, v, dk, dv) packet rides the ring and is sent home once, after the last hop,
  by the exact remaining distance (the reference sends it every iteration and mis-unpacks the result –
  reference ring_flash_attention.py:377-385, SURVEY defect D1/D2/D3);
* fully masked rows give 0 output (never NaN);
* document masking for packed sequences (``document_ids``, see :mod:`ring_attention_pytorch_b200.parallel.documents`);
* learned attention sinks (``sinks``): folded into each row's softmax state once, after the last hop.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor
from torch.autograd import Function

from ring_attention_pytorch_b200.parallel.distributed import default, exists, get_rank, get_world_size, is_distributed
from ring_attention_pytorch_b200.parallel.documents import check_document_ids, document_mask, ring_document_spans
from ring_attention_pytorch_b200.parallel.layout import PositionMap, make_position_map, ring_hop_owners
from ring_attention_pytorch_b200.parallel.ring import all_ring_pass, null_ring_pass, ring_pass
from ring_attention_pytorch_b200.utils.validate import check_attention_inputs, check_sinks, typecheck

EPSILON = 1e-10


def ring_num_hops(pm: PositionMap, causal: bool, window: Optional[int]) -> int:
    """Uniform number of ring iterations every rank must take part in (max over ranks of the furthest
    hop that still contains a visible key)."""
    if not causal:
        return pm.world
    hops = 1
    for r in range(pm.world):
        owners = set(ring_hop_owners(pm, r, causal, window))
        for s in range(pm.world - 1, 0, -1):
            if ((r - s) % pm.world) in owners:
                hops = max(hops, s + 1)
                break
    return hops


def _visibility(q_pos: Tensor, k_pos: Tensor, causal: bool, window: Optional[int]) -> Optional[Tensor]:
    if not causal:
        return None
    rel = q_pos[:, None] - k_pos[None, :]
    vis = rel >= 0
    if exists(window) and window > 0:
        vis = vis & (rel <= window)
    return vis


def _group_q(t: Tensor, kv_heads: int) -> Tensor:
    """[b, n, h, d] -> [b, n, g, hk, d] with h = g * hk + hk_index (query head j uses kv head j % hk)."""
    b, n, h, d = t.shape
    return t.view(b, n, h // kv_heads, kv_heads, d)


class RingFlashAttentionFunction(Function):
    @staticmethod
    @torch.no_grad()
    def forward(
        ctx,
        q: Tensor,
        k: Tensor,
        v: Tensor,
        mask: Optional[Tensor],
        causal: bool,
        bucket_size: int,
        ring_reduce_col: bool,
        striped_ring_attn: bool,
        max_lookback_seq_len: Optional[int],
        ring_size: Optional[int],
        softclamp_qk_sim: bool = False,
        softclamp_value: float = 50.0,
        layout: Optional[str] = None,
        document_ids: Optional[Tensor] = None,
        sinks: Optional[Tensor] = None,
    ):
        check_document_ids(document_ids, q, k)
        ring_size = default(ring_size, get_world_size())
        cross_attn = q.shape[-3] != k.shape[-3]
        ring_reduce_col = ring_reduce_col and is_distributed() and not cross_attn and ring_size > 1
        striped_ring_attn = striped_ring_attn and ring_reduce_col
        layout = default(layout, "striped" if striped_ring_attn else "plain")
        if not ring_reduce_col:
            layout, ring_size = "plain", 1

        assert k.shape[-2] == v.shape[-2] and q.shape[-2] % k.shape[-2] == 0
        assert not (exists(max_lookback_seq_len) and not causal), "look-back windows need causal attention"
        if causal:
            mask = None  # reference ring_flash_attention.py:107-108

        b, n, h, d = q.shape
        n_k, hk = k.shape[1], k.shape[2]
        scale = d ** -0.5
        rank = get_rank() % ring_size if ring_reduce_col else 0
        pm = make_position_map(layout, ring_size, n_k)
        q_pos = pm.positions(rank, q.device) if not cross_attn else torch.arange(n, device=q.device) + (n_k - n)
        owners = set(ring_hop_owners(pm, rank, causal, max_lookback_seq_len))
        max_iters = ring_num_hops(pm, causal, max_lookback_seq_len) if ring_reduce_col else 1
        # this rank's query rows: [b, n, 2] intervals of their documents (None: no document masking)
        q_spans = ring_document_spans(document_ids, pm, ring_reduce_col)[rank] if exists(document_ids) else None

        qf = _group_q(q.float() * scale, hk)  # [b, n, g, hk, d]
        o = torch.zeros_like(qf)
        row_max = torch.full((b, n, qf.shape[2], hk, 1), -torch.finfo(torch.float32).max, device=q.device)
        row_sum = torch.zeros_like(row_max)
        bucket = max(1, min(n, bucket_size))

        ring_iter = all_ring_pass if ring_reduce_col else null_ring_pass
        kv = torch.stack((k, v))
        mask_u8 = mask.to(torch.uint8) if exists(mask) else None  # bool tensors do not travel over every backend
        for (ring_rank, _), ((kv_cur, mask_cur), _bufs) in ring_iter(kv, mask_u8, max_iters=max_iters, ring_size=ring_size):
            if ring_rank not in owners and ring_reduce_col:
                continue
            mask_cur = mask_cur.bool() if exists(mask_cur) else None
            kc, vc = kv_cur[0].float(), kv_cur[1].float()
            k_pos = pm.positions(ring_rank, q.device)
            for s in range(0, n, bucket):
                e = min(s + bucket, n)
                vis = _visibility(q_pos[s:e], k_pos, causal, max_lookback_seq_len)
                if exists(vis) and not bool(vis.any()):
                    continue
                sim = torch.einsum("bighd,bjhd->bighj", qf[:, s:e], kc)
                if softclamp_qk_sim:
                    sim = (sim / softclamp_value).tanh() * softclamp_value
                keep = None
                if exists(vis):
                    keep = vis[None, :, None, None, :]
                if exists(mask_cur):
                    km = mask_cur[:, None, None, None, :]
                    keep = km if keep is None else (keep & km)
                if exists(q_spans):
                    dm = document_mask(q_spans[:, s:e], k_pos)[:, :, None, None, :]
                    keep = dm if keep is None else (keep & dm)
                if exists(keep):
                    sim = sim.masked_fill(~keep, -torch.finfo(torch.float32).max)
                blk_max = sim.amax(dim=-1, keepdim=True)
                new_max = torch.maximum(row_max[:, s:e], blk_max)
                p = (sim - new_max).exp()
                if exists(keep):
                    p = p.masked_fill(~keep, 0.0)
                corr = (row_max[:, s:e] - new_max).exp()
                row_sum[:, s:e] = row_sum[:, s:e] * corr + p.sum(dim=-1, keepdim=True)
                o[:, s:e] = o[:, s:e] * corr + torch.einsum("bighj,bjhd->bighd", p, vc)
                row_max[:, s:e] = new_max

        if exists(sinks):
            # the sink logit joins every row's denominator once, with a zero value vector
            sink = sinks.float().view(1, 1, qf.shape[2], hk, 1)
            new_max = torch.maximum(row_max, sink)
            corr = (row_max - new_max).exp()
            row_sum = row_sum * corr + (sink - new_max).exp()
            o = o * corr
            row_max = new_max

        has_any = row_sum > 0
        o = torch.where(has_any, o / row_sum.clamp(min=EPSILON), torch.zeros_like(o))
        lse = torch.where(has_any, row_sum.clamp(min=EPSILON).log() + row_max, torch.full_like(row_max, float("inf")))
        out = o.reshape(b, n, h, d).to(q.dtype)

        ctx.args = (causal, scale, mask, bucket, ring_reduce_col, ring_size, max_iters, max_lookback_seq_len,
                    softclamp_qk_sim, softclamp_value, layout, cross_attn, rank, q_spans)
        ctx.save_for_backward(q, k, v, out, lse, sinks if exists(sinks) else torch.empty(0))
        return out

    @staticmethod
    @torch.no_grad()
    def backward(ctx, do: Tensor):
        (causal, scale, mask, bucket, ring_reduce_col, ring_size, max_iters, window, softclamp_qk_sim,
         softclamp_value, layout, cross_attn, rank, q_spans) = ctx.args
        q, k, v, o, lse, sinks = ctx.saved_tensors
        b, n, h, d = q.shape
        n_k, hk = k.shape[1], k.shape[2]
        pm = make_position_map(layout, ring_size, n_k)
        q_pos = pm.positions(rank, q.device) if not cross_attn else torch.arange(n, device=q.device) + (n_k - n)
        owners = set(ring_hop_owners(pm, rank, causal, window))

        qf = _group_q(q.float(), hk)
        dof = _group_q(do.float(), hk)
        of = _group_q(o.float(), hk)
        delta = (dof * of).sum(dim=-1, keepdim=True)
        dq = torch.zeros_like(qf)
        dsinks = None
        if sinks.numel() > 0:  # d lse / d sink = exp(sink - lse); this rank's rows only
            sink = sinks.float().view(1, 1, qf.shape[2], hk, 1)
            dsinks = -((sink - lse).exp() * delta).sum(dim=(0, 1)).reshape(h).to(sinks.dtype)

        # (k, v, dk, dv) ride the ring together in fp32 (reference carries them in the activation dtype)
        packet = torch.stack((k.float(), v.float(), torch.zeros_like(k, dtype=torch.float32),
                              torch.zeros_like(v, dtype=torch.float32)))
        ring_iter = all_ring_pass if ring_reduce_col else null_ring_pass
        last_packet = packet
        mask_u8 = mask.to(torch.uint8) if exists(mask) else None
        for (ring_rank, _), ((packet_cur, mask_cur), _bufs) in ring_iter(packet, mask_u8, max_iters=max_iters,
                                                                          ring_size=ring_size):
            last_packet = packet_cur
            if ring_rank not in owners and ring_reduce_col:
                continue
            mask_cur = mask_cur.bool() if exists(mask_cur) else None
            kc, vc, dkc, dvc = packet_cur
            k_pos = pm.positions(ring_rank, q.device)
            for s in range(0, n, bucket):
                e = min(s + bucket, n)
                vis = _visibility(q_pos[s:e], k_pos, causal, window)
                if exists(vis) and not bool(vis.any()):
                    continue
                sim = torch.einsum("bighd,bjhd->bighj", qf[:, s:e], kc) * scale
                if softclamp_qk_sim:
                    t = (sim / softclamp_value).tanh()
                    sim = t * softclamp_value
                keep = None
                if exists(vis):
                    keep = vis[None, :, None, None, :]
                if exists(mask_cur):
                    km = mask_cur[:, None, None, None, :]
                    keep = km if keep is None else (keep & km)
                if exists(q_spans):
                    dm = document_mask(q_spans[:, s:e], k_pos)[:, :, None, None, :]
                    keep = dm if keep is None else (keep & dm)
                lse_blk = lse[:, s:e]
                p = (sim - torch.where(torch.isfinite(lse_blk), lse_blk, torch.zeros_like(lse_blk))).exp()
                p = torch.where(torch.isfinite(lse_blk), p, torch.zeros_like(p))
                if exists(keep):
                    p = p.masked_fill(~keep, 0.0)
                dvc += torch.einsum("bighj,bighd->bjhd", p, dof[:, s:e])
                dp = torch.einsum("bighd,bjhd->bighj", dof[:, s:e], vc)
                ds = p * (dp - delta[:, s:e]) * scale
                if softclamp_qk_sim:
                    ds = ds * (1.0 - t * t)
                dq[:, s:e] += torch.einsum("bighj,bjhd->bighd", ds, kc)
                dkc += torch.einsum("bighj,bighd->bjhd", ds, qf[:, s:e])

        if ring_reduce_col and max_iters > 0:
            # after `max_iters - 1` hops this rank holds the packet of owner (rank - (max_iters-1)); send it
            # the remaining way round so every packet ends at its owner.
            remaining = (ring_size - (max_iters - 1)) % ring_size
            dkv = last_packet[2:].contiguous()
            if remaining != 0:
                dkv, _ = ring_pass(remaining, dkv, None, ring_size)
            dk, dv = dkv[0], dkv[1]
        else:
            dk, dv = last_packet[2], last_packet[3]

        dq = dq.reshape(b, n, h, d).to(q.dtype)
        return (dq, dk.to(k.dtype), dv.to(v.dtype), None, None, None, None, None, None, None, None, None, None, None,
                dsinks)


ring_flash_attn_ = RingFlashAttentionFunction.apply


@typecheck
def ring_flash_attn(
    q: Tensor,
    k: Tensor,
    v: Tensor,
    mask: Optional[Tensor] = None,
    causal: bool = False,
    bucket_size: int = 1024,
    ring_reduce_col: bool = False,
    striped_ring_attn: bool = False,
    max_lookback_seq_len: Optional[int] = None,
    ring_size: Optional[int] = None,
    softclamp_qk_sim: bool = False,
    softclamp_value: float = 50.0,
    layout: Optional[str] = None,
    document_ids: Optional[Tensor] = None,
    sinks: Optional[Tensor] = None,
) -> Tensor:
    """Reference-compatible signature (ring_flash_attention.py:391-406) + ``layout`` ('plain'|'striped'|'zigzag').

    ``document_ids`` (integer ``[b, n]``, sharded and laid out like ``q``): document masking for packed sequences.  A
    document is a maximal run of equal ids in global position order (two separate runs sharing an id are two
    documents); a query sees only keys of its own document, on top of ``causal``, the look-back window and ``mask``.
    Unlike ``mask`` it is kept under ``causal=True``.  Self-attention only.

    ``sinks`` (floating ``[h]``): learned attention sinks, one logit per query head (not softclamped) that joins every
    row's softmax denominator once, with a zero value vector.  A row that sees no key gives 0.  Its gradient is this
    rank's partial sum over its own rows, like every other parameter's."""
    check_attention_inputs(q, k, v, mask, name="ring_flash_attn")
    check_sinks(sinks, q.shape[2], q.device, name="ring_flash_attn")
    return ring_flash_attn_(q, k, v, mask, causal, bucket_size, ring_reduce_col, striped_ring_attn,
                            max_lookback_seq_len, ring_size, softclamp_qk_sim, softclamp_value, layout, document_ids,
                            sinks)
