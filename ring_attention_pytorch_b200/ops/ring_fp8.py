"""fp8 (e4m3) forward of ring attention, for long-context prefill.

``quantize_fp8`` turns q, k, v into e4m3 with one fp32 scale per (batch, head), taken over the whole ring set, and
``ring_flash_attn_fp8`` runs the ring forward on them: the same schedule, masks, layouts, memory modes and in-kernel
NVLink fetch as :func:`ring_flash_attn_cuda`, with both attention matmuls as e4m3 wgmma and half the K/V bytes moved.
Forward only: there is no backward, and inputs that require grad are refused.

Semantics: ``ring_flash_attn_fp8(q, k, v, qd, kd, vd, ...)`` is ``ring_flash_attn(q.float() * qd, k.float() * kd,
v.float() * vd, ...)`` (descales broadcast over tokens and head dim) returned as bf16.  On CPU tensors that is exactly
what runs; on CUDA tensors the sm_90a kernel computes it with S = Q K^T in fp32 from e4m3 products and P quantised to
e4m3 for P V.

``k_descale`` and ``v_descale`` must be the same on every rank of a ring (``quantize_fp8`` with the ring's size gives
that): O accumulates across owners without a per-owner rescale, and ``v_descale`` is applied once, in the epilogue.
The K/V scales have the ``[b * hk]`` convention of ``tree_decode_cuda(k_scale=, v_scale=)``, so the quantised K/V of a
prefill can go into the decode cache unchanged.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist
from torch import Tensor

from ring_attention_pytorch_b200.parallel.distributed import default, exists, get_rank, get_world_size, is_distributed
from ring_attention_pytorch_b200.parallel.documents import check_document_ids
from ring_attention_pytorch_b200.utils.validate import check_fp8_attention_inputs, typecheck

E4M3_MAX = 448.0


def v8_key_of_slot(kappa: int) -> int:
    """Key held by slot ``kappa`` of a V^T tile in the fp8 K/V slot: Python mirror of ``v8_key_of_slot`` in
    ``csrc/attn_common.cuh``.  A permutation of every 32-key group that lets the e4m3 P operand come straight from the
    registers of the S accumulator."""
    return ((kappa & ~31) + 16 * ((kappa >> 4) & 1) + 8 * ((kappa >> 1) & 1) + 2 * ((kappa >> 2) & 3)
            + (kappa & 1))


def _ring_amax(amax: Tensor, ring_size: int) -> Tensor:
    """Elementwise max of ``amax`` over this rank's ring set (the all-gather-and-slice of ``_gather_ring_masks``)."""
    world = get_world_size()
    gathered = [torch.empty_like(amax) for _ in range(world)]
    dist.all_gather(gathered, amax.contiguous())
    ring_set = get_rank() // ring_size
    return torch.stack(gathered[ring_set * ring_size:(ring_set + 1) * ring_size]).amax(0)


@torch.no_grad()
def quantize_fp8(t: Tensor, ring_size: Optional[int] = None):
    """``t`` ``[b, n, heads, d]`` -> (``t_fp8`` e4m3 ``[b, n, heads, d]``, ``descale`` fp32 ``[b, heads]``).

    ``descale = amax / 448`` with ``amax`` the absolute maximum of each (batch, head) over tokens and head dim, taken over
    every rank of this rank's ring set when torch.distributed is initialised (``ring_size`` defaults to the world size;
    ``ring_size=1`` keeps the scales local).  An all-zero (batch, head) gets descale 1.  The cast saturates at +-448.
    ``t_fp8.float() * descale[:, None, :, None]`` approximates ``t`` within one e4m3 step."""
    if t.dim() != 4:
        raise ValueError(f"quantize_fp8: t must be [b, n, heads, d], got {tuple(t.shape)}")
    amax = t.abs().amax(dim=(1, 3)).float()
    ring_size = default(ring_size, get_world_size())
    if is_distributed() and ring_size > 1:
        amax = _ring_amax(amax, ring_size)
    descale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    scaled = t.float() / descale[:, None, :, None]
    return scaled.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn), descale


def _dequantize(t: Tensor, descale: Tensor) -> Tensor:
    b, heads = t.shape[0], t.shape[2]
    return t.float() * descale.float().expand(b, heads)[:, None, :, None]


def dequantized_ring_flash_attn(q, k, v, q_descale, k_descale, v_descale, *args, **kwargs) -> Tensor:
    """The definition of the fp8 op: the portable ring op on the dequantised inputs, as bf16."""
    from ring_attention_pytorch_b200.ops.ring_flash_naive import ring_flash_attn

    out = ring_flash_attn(_dequantize(q, q_descale), _dequantize(k, k_descale), _dequantize(v, v_descale), *args,
                          **kwargs)
    return out.to(torch.bfloat16)


@torch.no_grad()
def _ring_flash_attn_fp8_cuda(q, k, v, q_descale, k_descale, v_descale, mask, causal, ring_reduce_col,
                              striped_ring_attn, max_lookback_seq_len, ring_size, softclamp_qk_sim, softclamp_value,
                              layout, document_ids, sinks) -> Tensor:
    from ring_attention_pytorch_b200.ops import _ext, ring_cuda
    from ring_attention_pytorch_b200.ops.fused import (alloc_fwd_carry, alloc_kv_buffer_fp8, fused_attn_fwd_fp8,
                                                       fused_attn_fwd_hop_fp8, pack_key_mask_bits, pack_kv_fp8, pad128)
    from ring_attention_pytorch_b200.parallel.documents import ring_document_spans
    from ring_attention_pytorch_b200.parallel.layout import make_position_map, ring_hop_owners
    from ring_attention_pytorch_b200.parallel.symm import get_workspace
    from ring_attention_pytorch_b200.utils.timing import nvtx_range

    ops = _ext.ops()
    ring_size = default(ring_size, get_world_size())
    cross_attn = q.shape[1] != k.shape[1]
    use_ring = bool(ring_reduce_col) and is_distributed() and not cross_attn and ring_size > 1
    layout = default(layout, "striped" if (striped_ring_attn and use_ring) else "plain")
    if not use_ring:
        layout, ring_size = "plain", 1
    assert not (exists(max_lookback_seq_len) and not causal), "look-back windows need causal attention"
    if causal:
        mask = None

    b, n_q, h, d = q.shape
    n_k, hk = k.shape[1], k.shape[2]
    scale = d ** -0.5
    q = q.contiguous()
    descales = (q_descale.float().expand(b, h).contiguous(), k_descale.float().expand(b, hk).contiguous(),
                v_descale.float().expand(b, hk).contiguous())
    rank = get_rank() % ring_size if use_ring else 0
    # max(n_q, n_k): a map of n_k rows would wrap query row i >= n_k of a cross-attention to position i - n_k
    pm = make_position_map(layout, ring_size, max(n_q, n_k))
    q_off = (n_k - n_q) if (cross_attn and causal) else 0
    dev = q.device
    spans = ring_document_spans(document_ids.to(dev), pm, use_ring) if exists(document_ids) else None
    sinks = sinks.float().contiguous() if exists(sinks) else None

    # an fp8 slot [2, b*hk, n_pad, 128] has the bytes of a bf16 slot of n_pad / 2 keys: the workspaces, the copy-engine
    # window and the fetcher warps only move bytes
    n_pad = pad128(n_k)

    def as_fp8_slots(t: Tensor, lead) -> Tensor:
        return t.view(torch.uint8).view(*lead, 2, b * hk, n_pad, 128)

    ready = torch.zeros(ring_size, dtype=torch.int32, device=dev)
    peers = [0] * ring_size
    kbits = None
    hop_mode = use_ring and ring_cuda._use_hop_window(2 * b * hk * n_pad * 128)
    with nvtx_range("rab.fwd8.pack+barrier"):
        if hop_mode:
            ws = get_workspace(ring_size, dev)
            own, own_ptrs, slot_bytes = ring_cuda._own_slot_workspace(ws, b, hk, n_pad // 2, 128, torch.bfloat16)
            own = as_fp8_slots(own, ())
            pack_kv_fp8(k, v, own)
            ws.barrier()  # every peer's own slot is complete
            ring_cuda._count(2)
        elif use_ring:
            ws = get_workspace(ring_size, dev)
            kv_gather, own_slot_ptrs, _ = ring_cuda._ring_gather_workspace(ws, ring_size, b, hk, n_pad // 2, 128,
                                                                          torch.bfloat16)
            kv_gather = as_fp8_slots(kv_gather, (ring_size,))
            pack_kv_fp8(k, v, kv_gather[rank])
            ws.barrier()  # every peer's own slot is complete
            ring_cuda._count(2)
            peers = [0 if o == rank else own_slot_ptrs[o] for o in range(ring_size)]
        else:
            kv_gather = alloc_kv_buffer_fp8(1, b, hk, n_k, dev)
            pack_kv_fp8(k, v, kv_gather[0])
            ring_cuda._count()
        if exists(mask):
            kbits = pack_key_mask_bits(ring_cuda._gather_ring_masks(mask, ring_size) if use_ring else mask[None])

    softclamp = float(softclamp_value) if softclamp_qk_sim else 0.0
    with nvtx_range("rab.fwd8.kernel"):
        if hop_mode:
            hops = ring_hop_owners(pm, rank, causal, max_lookback_seq_len)
            window_slots = ring_cuda._HopWindow(ops, ws, own, own_ptrs, slot_bytes, hops)
            carry_o, carry_ml = alloc_fwd_carry(q)
            for s_, owner in enumerate(hops):
                o, _ = fused_attn_fwd_hop_fp8(q, window_slots.slot(s_), n_k, descales, owner, ring_size, carry_o,
                                              carry_ml, kbits, carry_in=s_ > 0, carry_out=s_ + 1 < len(hops),
                                              kv_heads=hk, rank=rank, pm=pm, causal=causal,
                                              window=max_lookback_seq_len, scale=scale, softclamp=softclamp,
                                              q_pos_offset=q_off, doc_spans=spans, sinks=sinks)
                window_slots.launched(s_)
                ring_cuda._count()
        else:
            o, _ = fused_attn_fwd_fp8(q, kv_gather, n_k, descales, peers, ready, kbits, kv_heads=hk, rank=rank, pm=pm,
                                      causal=causal, window=max_lookback_seq_len, scale=scale, softclamp=softclamp,
                                      q_pos_offset=q_off, doc_spans=spans, sinks=sinks)
            ring_cuda._count()
    return o


@torch.no_grad()
@typecheck
def ring_flash_attn_fp8(
    q: Tensor,
    k: Tensor,
    v: Tensor,
    q_descale: Tensor,
    k_descale: Tensor,
    v_descale: Tensor,
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
    rotary_freqs: Optional[Tensor] = None,
    sinks: Optional[Tensor] = None,
) -> Tensor:
    """Ring attention forward on e4m3 inputs (see the module docstring for the exact semantics).

    q ``[b, n, h, 128]``, k / v ``[b, n, hk, 128]`` ``float8_e4m3fn``, sharded and laid out as for
    :func:`ring_flash_attn_cuda`; ``q_descale`` fp32 ``[b, h]``, ``k_descale`` / ``v_descale`` fp32 ``[b, hk]`` (one
    element broadcasts).  Every other argument has the meaning it has there.  Returns bf16 ``[b, n, h, 128]``.
    ``rotary_freqs`` is refused: rotate q and k before quantising them.  ``sinks`` (floating ``[h]``, not requiring
    grad): learned attention sinks in the logits' natural-log units, as in :func:`ring_flash_attn`."""
    check_fp8_attention_inputs(q, k, v, q_descale, k_descale, v_descale, mask, name="ring_flash_attn_fp8",
                               rotary_freqs=rotary_freqs, sinks=sinks)
    check_document_ids(document_ids, q, k)
    kwargs = dict(mask=mask, causal=causal, bucket_size=bucket_size, ring_reduce_col=ring_reduce_col,
                  striped_ring_attn=striped_ring_attn, max_lookback_seq_len=max_lookback_seq_len, ring_size=ring_size,
                  softclamp_qk_sim=softclamp_qk_sim, softclamp_value=softclamp_value, layout=layout,
                  document_ids=document_ids, sinks=sinks)
    if not q.is_cuda:
        return dequantized_ring_flash_attn(q, k, v, q_descale, k_descale, v_descale, **kwargs)
    if q.shape[3] != 128:
        raise ValueError(f"ring_flash_attn_fp8: the CUDA kernel needs head dim 128, got {q.shape[3]}")
    kwargs.pop("bucket_size")  # tiling is fixed by the kernel (128 x 128)
    return _ring_flash_attn_fp8_cuda(q, k, v, q_descale, k_descale, v_descale, **kwargs)
