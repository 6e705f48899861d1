"""Thin Python wrappers over the sm_90a kernels (``torch.ops.rab.*``).

These are the building blocks the autograd ops in :mod:`ring_attention_pytorch_b200.ops.ring_cuda`
compose; they are also what the GPU unit tests drive directly.  ``emulate_ring_forward`` runs a whole
W-rank ring on ONE device by giving every emulated rank its own K/V gather buffer and pointing the
"peer" addresses at the other ranks' buffers – the kernel cannot tell the difference, which lets the
multi-hop fetch/ready-flag protocol be tested on a single GPU.

``doc_spans`` (every wrapper) is the int32 ``[world, b, n, 2]`` document interval table of
:mod:`ring_attention_pytorch_b200.parallel.documents`; ``None`` launches the kernels without document masking.

``sinks`` (the forwards) is the contiguous fp32 ``[h]`` tensor of learned attention sinks, one logit per query head
that joins every row's softmax denominator with a zero value vector; ``None`` launches the kernels without sinks.
The forward counts it in the launch that starts a row (the single launch, or hop 0 of the hop-wise mode).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from ring_attention_pytorch_b200.ops import _ext
from ring_attention_pytorch_b200.parallel.documents import document_spans
from ring_attention_pytorch_b200.parallel.layout import (PositionMap, make_position_map, ring_hop_owners,
                                                          ring_query_owners)


def pack_key_mask_bits(mask: torch.Tensor) -> torch.Tensor:
    """[world, b, n] bool (True = keep) -> [world, b, words] int32 bit-packed, words % 4 == 0."""
    world, b, n = mask.shape
    words = ((n + 127) // 128) * 4
    padded = torch.zeros(world, b, words * 32, dtype=torch.bool, device=mask.device)
    padded[..., :n] = mask
    bits = padded.view(world, b, words, 32).to(torch.int64)
    weights = (1 << torch.arange(32, device=mask.device, dtype=torch.int64))
    packed = (bits * weights).sum(-1)
    packed = torch.where(packed >= 2 ** 31, packed - 2 ** 32, packed)
    return packed.to(torch.int32).contiguous()


def alloc_kv_buffer(world: int, batch: int, kv_heads: int, n_k: int, d: int, dtype, device) -> torch.Tensor:
    return torch.empty(world, 2, batch * kv_heads, n_k, d, dtype=dtype, device=device)


def fused_attn_fwd(
    q: torch.Tensor,
    kv_buf: torch.Tensor,
    peer_ptrs: Sequence[int],
    ready: torch.Tensor,
    kmask_bits: Optional[torch.Tensor],
    *,
    kv_heads: int,
    rank: int,
    pm: PositionMap,
    causal: bool,
    window: Optional[int],
    scale: float,
    softclamp: float = 0.0,
    q_pos_offset: int = 0,
    hop_owner: Optional[List[int]] = None,
    doc_spans: Optional[torch.Tensor] = None,
    sinks: Optional[torch.Tensor] = None,
):
    if hop_owner is None:
        hop_owner = ring_hop_owners(pm, rank, causal, window)
    return _ext.ops().attn_fwd(
        q, kv_buf, list(peer_ptrs), ready, kmask_bits, kv_heads, rank, bool(causal), int(window or 0), float(scale),
        float(softclamp), pm.stride, pm.seg_len, pm.base0, pm.base1, int(q_pos_offset), list(hop_owner), doc_spans,
        sinks)


def fused_attn_fwd_hop(
    q: torch.Tensor,
    kv_slot: torch.Tensor,
    owner: int,
    world: int,
    carry_o: torch.Tensor,
    carry_ml: torch.Tensor,
    kmask_bits: Optional[torch.Tensor],
    *,
    carry_in: bool,
    carry_out: bool,
    kv_heads: int,
    rank: int,
    pm: PositionMap,
    causal: bool,
    window: Optional[int],
    scale: float,
    softclamp: float = 0.0,
    q_pos_offset: int = 0,
    doc_spans: Optional[torch.Tensor] = None,
    sinks: Optional[torch.Tensor] = None,
):
    """ONE ring hop of the forward (``memory="ring"``): ``q`` against owner ``owner``'s K/V slot ``[2, b*hk, n_k, d]``.

    The online-softmax state travels between the per-hop launches in ``carry_o`` (fp32 ``[b, n_q, h, d]``, the
    un-normalised O) and ``carry_ml`` (fp32 ``[2, b*h, n_q]``: running maximum / sum); the launch with
    ``carry_out=False`` returns the final (o, lse).  The reference carries (o, m, lse) between its per-hop Triton
    launches the same way (ring_flash_attention_cuda.py:143-173)."""
    return _ext.ops().attn_fwd_hop(
        q, kv_slot[None], int(owner), int(world), carry_o, carry_ml, bool(carry_in), bool(carry_out), kmask_bits,
        kv_heads, rank, bool(causal), int(window or 0), float(scale), float(softclamp), pm.stride, pm.seg_len, pm.base0,
        pm.base1, int(q_pos_offset), doc_spans, sinks)


def alloc_fwd_carry(q: torch.Tensor):
    b, n_q, h, d = q.shape
    return (torch.empty(b, n_q, h, d, dtype=torch.float32, device=q.device),
            torch.empty(2, b * h, n_q, dtype=torch.float32, device=q.device))


def emulate_ring_forward(
    qs: Sequence[torch.Tensor],
    ks: Sequence[torch.Tensor],
    vs: Sequence[torch.Tensor],
    *,
    layout: str = "plain",
    causal: bool = False,
    window: Optional[int] = None,
    softclamp: float = 0.0,
    key_masks: Optional[Sequence[torch.Tensor]] = None,
    scale: Optional[float] = None,
    hopwise: bool = False,
    document_ids: Optional[Sequence[torch.Tensor]] = None,
    sinks: Optional[torch.Tensor] = None,
):
    """Run the fused forward for every rank of a W-rank ring on the current device.

    qs/ks/vs: per-rank shards ``[b, n, h, d]`` / ``[b, n, hk, d]``.  Returns (outs, lses) lists.
    ``hopwise``: one launch per hop with carried softmax state (the ``memory="ring"`` schedule).
    ``document_ids``: per-rank ``[b, n]`` document ids (in the ring's layout) for document masking.
    ``sinks``: fp32 ``[h]`` attention sinks.
    """
    ops = _ext.ops()
    world = len(qs)
    b, n, h, d = qs[0].shape
    hk = ks[0].shape[2]
    dev, dt = qs[0].device, qs[0].dtype
    pm = make_position_map(layout, world, n)
    scale = d ** -0.5 if scale is None else scale
    bufs = [alloc_kv_buffer(world, b, hk, n, d, dt, dev) for _ in range(world)]
    for r in range(world):
        bufs[r].zero_()
        ops.pack_kv(ks[r], vs[r], bufs[r][r])
    kbits = None
    if key_masks is not None:
        kbits = pack_key_mask_bits(torch.stack(list(key_masks), 0))
    spans = None if document_ids is None else document_spans(torch.stack(list(document_ids), 0), pm)
    outs, lses = [], []
    if hopwise:
        for r in range(world):
            q = qs[r].contiguous()
            carry_o, carry_ml = alloc_fwd_carry(q)
            hops = ring_hop_owners(pm, r, causal, window)
            for s_, owner in enumerate(hops):
                o, lse = fused_attn_fwd_hop(q, bufs[owner][owner], owner, world, carry_o, carry_ml, kbits,
                                            carry_in=s_ > 0, carry_out=s_ + 1 < len(hops), kv_heads=hk, rank=r, pm=pm,
                                            causal=causal, window=window, scale=scale, softclamp=softclamp,
                                            doc_spans=spans, sinks=sinks)
            outs.append(o)
            lses.append(lse)
        return outs, lses
    for r in range(world):
        ready = torch.zeros(world, dtype=torch.int32, device=dev)
        peers = [bufs[o][o].data_ptr() for o in range(world)]  # owner o's own slot
        o, lse = fused_attn_fwd(qs[r].contiguous(), bufs[r], peers, ready, kbits, kv_heads=hk, rank=r, pm=pm,
                                causal=causal, window=window, scale=scale, softclamp=softclamp, doc_spans=spans,
                                sinks=sinks)
        outs.append(o)
        lses.append(lse)
    return outs, lses


# ------------------------------------------------------------------------------------------------
# fp8 (e4m3) forward, head dim 128
# ------------------------------------------------------------------------------------------------
def alloc_kv_buffer_fp8(world: int, batch: int, kv_heads: int, n_k: int, device) -> torch.Tensor:
    """``world`` fp8 slots ``[world, 2, b*hk, pad128(n_k), 128]`` uint8 (layout: ``csrc/kernels.h``, pack_kv_fp8)."""
    return torch.empty(world, 2, batch * kv_heads, pad128(n_k), 128, dtype=torch.uint8, device=device)


def pack_kv_fp8(k: torch.Tensor, v: torch.Tensor, slot: torch.Tensor) -> None:
    """k, v e4m3 ``[b, n, hk, 128]`` -> one fp8 slot ``[2, b*hk, pad128(n), 128]``: K, then V^T per 128-key tile in the
    key order of :func:`ring_attention_pytorch_b200.ops.ring_fp8.v8_key_of_slot`; keys past ``n`` are zero."""
    _ext.ops().pack_kv_fp8(k, v, slot)


def fused_attn_fwd_fp8(
    q: torch.Tensor,
    kv_buf: torch.Tensor,
    n_k: int,
    descales,
    peer_ptrs: Sequence[int],
    ready: torch.Tensor,
    kmask_bits: Optional[torch.Tensor],
    *,
    kv_heads: int,
    rank: int,
    pm: PositionMap,
    causal: bool,
    window: Optional[int],
    scale: float,
    softclamp: float = 0.0,
    q_pos_offset: int = 0,
    hop_owner: Optional[List[int]] = None,
    doc_spans: Optional[torch.Tensor] = None,
    sinks: Optional[torch.Tensor] = None,
):
    """:func:`fused_attn_fwd` on e4m3 operands: ``q`` e4m3 ``[b, n_q, h, 128]``, ``kv_buf`` the fp8 slots of
    :func:`alloc_kv_buffer_fp8` holding ``n_k`` keys each, ``descales`` = (q [b*h], k [b*hk], v [b*hk]) fp32.
    Returns bf16 o and the fp32 lse."""
    if hop_owner is None:
        hop_owner = ring_hop_owners(pm, rank, causal, window)
    qd, kd, vd = descales
    return _ext.ops().attn_fwd_fp8(
        q, kv_buf, int(n_k), qd, kd, vd, list(peer_ptrs), ready, kmask_bits, kv_heads, rank, bool(causal),
        int(window or 0), float(scale), float(softclamp), pm.stride, pm.seg_len, pm.base0, pm.base1, int(q_pos_offset),
        list(hop_owner), doc_spans, sinks)


def fused_attn_fwd_hop_fp8(
    q: torch.Tensor,
    kv_slot: torch.Tensor,
    n_k: int,
    descales,
    owner: int,
    world: int,
    carry_o: torch.Tensor,
    carry_ml: torch.Tensor,
    kmask_bits: Optional[torch.Tensor],
    *,
    carry_in: bool,
    carry_out: bool,
    kv_heads: int,
    rank: int,
    pm: PositionMap,
    causal: bool,
    window: Optional[int],
    scale: float,
    softclamp: float = 0.0,
    q_pos_offset: int = 0,
    doc_spans: Optional[torch.Tensor] = None,
    sinks: Optional[torch.Tensor] = None,
):
    """:func:`fused_attn_fwd_hop` on e4m3 operands (see :func:`fused_attn_fwd_fp8`).  The carried O is not scaled by
    ``v_descale`` (it is the same for every owner); the final launch applies it."""
    qd, kd, vd = descales
    return _ext.ops().attn_fwd_hop_fp8(
        q, kv_slot[None], int(n_k), qd, kd, vd, int(owner), int(world), carry_o, carry_ml, bool(carry_in),
        bool(carry_out), kmask_bits, kv_heads, rank, bool(causal), int(window or 0), float(scale), float(softclamp),
        pm.stride, pm.seg_len, pm.base0, pm.base1, int(q_pos_offset), doc_spans, sinks)


def emulate_ring_forward_fp8(
    qs: Sequence[torch.Tensor],
    ks: Sequence[torch.Tensor],
    vs: Sequence[torch.Tensor],
    q_descales: Sequence[torch.Tensor],
    k_descale: torch.Tensor,
    v_descale: torch.Tensor,
    *,
    layout: str = "plain",
    causal: bool = False,
    window: Optional[int] = None,
    softclamp: float = 0.0,
    key_masks: Optional[Sequence[torch.Tensor]] = None,
    scale: Optional[float] = None,
    hopwise: bool = False,
    document_ids: Optional[Sequence[torch.Tensor]] = None,
    sinks: Optional[torch.Tensor] = None,
):
    """:func:`emulate_ring_forward` for the fp8 forward: e4m3 shards, per-rank ``q_descales`` ``[b, h]`` and the
    ring-wide ``k_descale`` / ``v_descale`` ``[b, hk]`` (fp32).  Returns (outs, lses), outs in bf16."""
    world = len(qs)
    b, n, h, d = qs[0].shape
    hk = ks[0].shape[2]
    dev = qs[0].device
    pm = make_position_map(layout, world, n)
    scale = d ** -0.5 if scale is None else scale
    bufs = [alloc_kv_buffer_fp8(world, b, hk, n, dev) for _ in range(world)]
    for r in range(world):
        bufs[r].zero_()
        pack_kv_fp8(ks[r], vs[r], bufs[r][r])
    kd, vd = (t.float().expand(b, hk).contiguous() for t in (k_descale, v_descale))
    kbits = None
    if key_masks is not None:
        kbits = pack_key_mask_bits(torch.stack(list(key_masks), 0))
    spans = None if document_ids is None else document_spans(torch.stack(list(document_ids), 0), pm)
    outs, lses = [], []
    for r in range(world):
        q = qs[r].contiguous()
        descales = (q_descales[r].float().expand(b, h).contiguous(), kd, vd)
        if hopwise:
            carry_o, carry_ml = alloc_fwd_carry(q)
            hops = ring_hop_owners(pm, r, causal, window)
            for s_, owner in enumerate(hops):
                o, lse = fused_attn_fwd_hop_fp8(q, bufs[owner][owner], n, descales, owner, world, carry_o, carry_ml,
                                                kbits, carry_in=s_ > 0, carry_out=s_ + 1 < len(hops), kv_heads=hk,
                                                rank=r, pm=pm, causal=causal, window=window, scale=scale,
                                                softclamp=softclamp, doc_spans=spans, sinks=sinks)
        else:
            ready = torch.zeros(world, dtype=torch.int32, device=dev)
            peers = [bufs[o][o].data_ptr() for o in range(world)]  # owner o's own slot
            o, lse = fused_attn_fwd_fp8(q, bufs[r], n, descales, peers, ready, kbits, kv_heads=hk, rank=r, pm=pm,
                                        causal=causal, window=window, scale=scale, softclamp=softclamp,
                                        doc_spans=spans, sinks=sinks)
        outs.append(o)
        lses.append(lse)
    return outs, lses


def pad64(n: int) -> int:
    return (n + 63) // 64 * 64


def alloc_qdo_buffer(world: int, batch: int, heads: int, n_q: int, d: int, dtype, device) -> torch.Tensor:
    return torch.empty(world, 2, batch * heads, n_q, d, dtype=dtype, device=device)


def alloc_stat_buffer(world: int, batch: int, heads: int, n_q: int, device) -> torch.Tensor:
    return torch.zeros(world, 2, batch * heads, pad64(n_q), dtype=torch.float32, device=device)


def fused_attn_bwd(
    qdo_buf: torch.Tensor,
    kv_buf: torch.Tensor,
    stat_buf: torch.Tensor,
    kmask_bits: Optional[torch.Tensor],
    *,
    batch: int,
    heads: int,
    kv_heads: int,
    rank: int,
    pm: PositionMap,
    causal: bool,
    window: Optional[int],
    scale: float,
    softclamp: float = 0.0,
    q_pos_offset: int = 0,
    ready_kv: Optional[torch.Tensor] = None,
    ready_q: Optional[torch.Tensor] = None,
    ready_target: int = 0,
    doc_spans: Optional[torch.Tensor] = None,
):
    """Run both backward kernels on already gathered buffers; returns (dq, dk, dv)."""
    ops = _ext.ops()
    kv_owners = ring_hop_owners(pm, rank, causal, window)
    q_owners = ring_query_owners(pm, rank, causal, window)
    common = (kmask_bits, batch, heads, kv_heads, rank, bool(causal), int(window or 0), float(scale), float(softclamp),
              pm.stride, pm.seg_len, pm.base0, pm.base1, int(q_pos_offset))
    dq = ops.attn_bwd_dq(qdo_buf, kv_buf, stat_buf, ready_kv, ready_target, *common, kv_owners, doc_spans)
    dk, dv = ops.attn_bwd_dkdv(qdo_buf, kv_buf, stat_buf, ready_q, ready_target, *common, q_owners, doc_spans)
    return dq, dk, dv


def pad128(n: int) -> int:
    return (n + 127) // 128 * 128


def fused_attn_bwd_ring(
    qdo: torch.Tensor,
    stat: torch.Tensor,
    kv_buf: torch.Tensor,
    kmask_bits: Optional[torch.Tensor],
    *,
    batch: int,
    heads: int,
    kv_heads: int,
    rank: int,
    pm: PositionMap,
    causal: bool,
    window: Optional[int],
    scale: float,
    softclamp: float = 0.0,
    q_pos_offset: int = 0,
    dq_acc: Optional[torch.Tensor] = None,
    dkv_acc_ptrs: Sequence[int] = (),
    nk_pad: int = 0,
    ready: Optional[torch.Tensor] = None,
    ready_target: int = 0,
    hop_owner: Optional[List[int]] = None,
    world: int = 0,
    slot_owner: int = -1,
    doc_spans: Optional[torch.Tensor] = None,
):
    """The one-kernel (5-GEMM) backward, head dim 128 (``csrc/attn_bwd_sm90.cu``, KV-stationary kernel in its one-pass form).

    ``slot_owner >= 0`` (``memory="ring"``): ``kv_buf`` is ONE owner's slot ``[1, 2, b*hk, n_k, d]`` of a ``world``
    rank ring and the launch covers that hop only; ``dq_acc`` and the dK/dV accumulators add up across the launches.

    ``qdo`` [2, b*h, n_q, d] / ``stat`` [2, b*h, n_pad] are this rank's ``bwd_prep`` output, ``kv_buf`` the K/V gather.
    dQ (unscaled) is added into ``dq_acc`` (fp32 [b*h, n_pad, d], allocated zeroed when not given).  Without
    ``dkv_acc_ptrs`` dK / dV come back as 16-bit tensors; with them (one fp32 [2, b*hk, nk_pad, d] accumulator address
    per ring rank) the kernel adds its tiles into the owners' accumulators and returns empty tensors.
    Returns (dq_acc, dk, dv)."""
    ops = _ext.ops()
    d = kv_buf.shape[-1]
    if dq_acc is None:
        dq_acc = torch.zeros(batch * heads, stat.shape[-1], d, dtype=torch.float32, device=kv_buf.device)
    if hop_owner is None:
        hop_owner = ring_hop_owners(pm, rank, causal, window)
    dk, dv = ops.attn_bwd_ring(qdo, kv_buf, stat, dq_acc, ready, int(ready_target), kmask_bits, batch, heads, kv_heads,
                               rank, bool(causal), int(window or 0), float(scale), float(softclamp), pm.stride,
                               pm.seg_len, pm.base0, pm.base1, int(q_pos_offset), list(hop_owner),
                               list(dkv_acc_ptrs), int(nk_pad), int(world), int(slot_owner), doc_spans)
    return dq_acc, dk, dv


def emulate_ring_backward(
    qs, ks, vs, outs, lses, douts, *,
    layout: str = "plain",
    causal: bool = False,
    window: Optional[int] = None,
    softclamp: float = 0.0,
    key_masks=None,
    scale: Optional[float] = None,
    fused: Optional[bool] = None,
    hopwise: bool = False,
    document_ids=None,
    sinks: Optional[torch.Tensor] = None,
):
    """Backward of :func:`emulate_ring_forward` for every emulated rank on the current device.
    ``hopwise`` (fused only): one launch per hop against a single K/V slot (the ``memory="ring"`` schedule).
    ``sinks`` (fp32 ``[h]``): every rank's tuple gains a fourth entry, that rank's fp32 sink gradient ``[h]``.

    ``fused`` (default: head dim 128) selects the one-kernel backward: every emulated rank adds its dK / dV tiles into
    the owners' fp32 accumulators, exactly what the ranks of a real ring do over NVLink."""
    ops = _ext.ops()
    world = len(qs)
    b, n, h, d = qs[0].shape
    hk = ks[0].shape[2]
    dev, dt = qs[0].device, qs[0].dtype
    pm = make_position_map(layout, world, n)
    scale = d ** -0.5 if scale is None else scale
    kv_all = alloc_kv_buffer(world, b, hk, n, d, dt, dev)
    qdo_all = alloc_qdo_buffer(world, b, h, n, d, dt, dev)
    stat_all = alloc_stat_buffer(world, b, h, n, dev)
    dsinks = [None if sinks is None else torch.empty(h, dtype=torch.float32, device=dev) for _ in range(world)]
    for r in range(world):
        ops.pack_kv(ks[r], vs[r], kv_all[r])
        ops.bwd_prep(qs[r].contiguous(), outs[r].contiguous(), douts[r].contiguous(), lses[r].contiguous(), qdo_all,
                     stat_all, r, sinks, dsinks[r])
    kbits = None
    if key_masks is not None:
        kbits = pack_key_mask_bits(torch.stack(list(key_masks), 0))
    spans = None if document_ids is None else document_spans(torch.stack(list(document_ids), 0), pm)
    if fused is None:
        fused = d == 128
    res = []
    if fused:
        nk_pad = pad128(n)
        ring = world > 1
        accs = [torch.zeros(2, b * hk, nk_pad, d, dtype=torch.float32, device=dev) for _ in range(world)] if ring else []
        ptrs = [a.data_ptr() for a in accs]
        dqs, direct = [], []
        for r in range(world):
            if hopwise and ring:
                dq_acc = None
                for owner in ring_hop_owners(pm, r, causal, window):
                    dq_acc, dk, dv = fused_attn_bwd_ring(
                        qdo_all[r], stat_all[r], kv_all[owner:owner + 1], kbits, batch=b, heads=h, kv_heads=hk, rank=r,
                        pm=pm, causal=causal, window=window, scale=scale, softclamp=softclamp, dq_acc=dq_acc,
                        dkv_acc_ptrs=ptrs, nk_pad=nk_pad, hop_owner=[owner], world=world, slot_owner=owner,
                        doc_spans=spans)
            else:
                dq_acc, dk, dv = fused_attn_bwd_ring(qdo_all[r], stat_all[r], kv_all, kbits, batch=b, heads=h,
                                                     kv_heads=hk, rank=r, pm=pm, causal=causal, window=window,
                                                     scale=scale, softclamp=softclamp, dkv_acc_ptrs=ptrs, nk_pad=nk_pad,
                                                     doc_spans=spans)
            dqs.append(dq_acc)
            direct.append((dk, dv))
        for r in range(world):
            dq = torch.empty(b, n, h, d, dtype=dt, device=dev)
            ops.acc_convert(dqs[r], dq, scale)
            if ring:
                dk = torch.empty(b, n, hk, d, dtype=dt, device=dev)
                dv = torch.empty_like(dk)
                ops.acc_convert(accs[r][0], dk, 1.0)
                ops.acc_convert(accs[r][1], dv, 1.0)
            else:
                dk, dv = direct[r]
            res.append((dq, dk, dv))
    else:
        for r in range(world):
            # every emulated rank sees the same fully gathered buffers (what the NVLink gather produces)
            res.append(fused_attn_bwd(qdo_all, kv_all, stat_all, kbits, batch=b, heads=h, kv_heads=hk, rank=r, pm=pm,
                                      causal=causal, window=window, scale=scale, softclamp=softclamp, doc_spans=spans))
    if sinks is not None:
        res = [(*g, ds) for g, ds in zip(res, dsinks)]
    return res
