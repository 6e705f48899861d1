"""sm_90a tree-attention decode: ONE persistent cooperative kernel per rank and step (``csrc/tree_decode_tc_sm90.cu``,
``csrc/tree_decode_sm90.cu``).

The kernel computes the split-KV partials of this rank's shard, merges the splits, publishes ``(out, lse)`` in a
symmetric buffer, signals the peers and merges all ranks' partials — over NVLink peer loads, or, when the buffers have a
multicast (NVLS) mapping, with ``multimem.ld_reduce`` inside the NVSwitch.  This wrapper only owns the buffers: they are
cached per (device, world, rows, head dim), every counter is self-resetting and the cross-rank epoch lives in device
memory, so a decode step allocates nothing and is CUDA-graph capturable.  Reference: tree_attn_decoding.py:60-102 (one
Triton launch padded to 128 rows + three all-reduces).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
from torch import Tensor

from ring_attention_pytorch_b200.ops import _ext
from ring_attention_pytorch_b200.parallel.distributed import get_rank, get_world_size, is_distributed
from ring_attention_pytorch_b200.utils.validate import check_decode_query, check_decode_ranges, check_paged_kv

LAUNCHES = {"count": 0}
# nvls "auto": use the NVSwitch multicast mapping when torch's symmetric memory can provide one, else NVLink peer loads
# tensor_core "auto": head dim 128 runs the wgmma kernel (K / V tiles go from TMA straight into the MMA, read in place
#                     from the cache; an fp8 cache is widened to bf16 in shared memory), everything else the CUDA-core kernel
CONFIG = {"nvls": "auto", "tensor_core": "auto"}
K_MAX_WORLD = 16
PAD_WORDS = 2 * K_MAX_WORLD  # two signal rounds
TILE = 64  # keys per tile in both kernels; unit ranges start on a multiple of it


def _choose_splits(n: int, groups: int, resident_ctas: int) -> int:
    """Enough work units to fill the persistent grid about twice, at least 256 keys per split."""
    if n <= 0:
        return 1
    want = max(1, (2 * resident_ctas + groups - 1) // groups)
    return max(1, min(want, (n + 255) // 256))


@dataclass(frozen=True)
class DecodePlan:
    tensor_core: bool  # which kernel runs: the wgmma kernel or the CUDA-core kernel
    groups: int        # (batch, kv head, head chunk) groups; work units = groups * splits
    resident: int      # co-resident CTAs of the kernel on this device (the persistent grid's size limit)
    splits: int        # key splits per group


def decode_span(n: int, window: Optional[int] = None, kv_pos_stride: int = 1, tokens: int = 1) -> int:
    """The most keys, with the up-to-63-key slack of tile alignment, that one sequence's visible range can touch: the
    ranged kernels split this span, not ``n``.  With a look-back window a query sees at most ``window // stride + 1``
    local keys, so the splits cover O(window) keys; ``tokens`` consecutive queries see the union of their ranges, at
    most ``(window + tokens - 1) // stride + 1`` keys."""
    if window is None or window <= 0:
        return n
    return min(n, (window + tokens - 1) // kv_pos_stride + TILE)


def decode_plan(b: int, h: int, hk: int, n: int, d: int, kv_kind: int, *, ranged: bool = False,
                span: Optional[int] = None, tokens: int = 1, paged: bool = False) -> DecodePlan:
    """The kernel and the work split a decode call of these sizes gets (``kv_kind``: 0 bf16, 1 fp16, 2 fp8 cache).
    ``ranged``: the instantiations with per-sequence key ranges / softclamp; ``span`` (default ``n``): the keys the
    splits are planned over (:func:`decode_span`).  ``tokens > 1``: a multi-token call (always ranged), whose work
    units hold ``NH`` (query head, token) columns of one kv head -- 8, 16 or 32 for ``g * tokens`` up to 8, up to 16,
    larger on the tensor-core kernel, 4 on the CUDA-core kernel -- planned with that variant's residency.
    ``paged`` (always ranged; ``n = max_pages * page_size``): the splits are those of a contiguous cache of ``n`` keys,
    so the paged call computes bitwise what that call computes; the grid is bounded by the paged variant's residency."""
    assert ranged or tokens > 1 or not paged, "a paged call is ranged"
    tc = CONFIG["tensor_core"]
    use_tc = tc in ("auto", True, "on") and d == 128 and n >= 1
    g = h // hk
    if tokens > 1:
        cols = g * tokens
        gm = (8 if cols <= 8 else (16 if cols <= 16 else 32)) if use_tc else 4
        groups = b * hk * ((cols + gm - 1) // gm)
        resident = int(_ext.ops().tree_decode_max_ctas(d, kv_kind, use_tc, True, cols))
        splits = _choose_splits(n if span is None else span, groups, resident)
        if paged:
            resident = int(_ext.ops().tree_decode_max_ctas(d, kv_kind, use_tc, True, cols, True))
        return DecodePlan(use_tc, groups, resident, splits)
    gm = (8 if g <= 8 else 16) if use_tc else 4  # query heads per work unit (tensor-core kernel: MMA N)
    groups = b * hk * ((g + gm - 1) // gm)
    resident = int(_ext.ops().tree_decode_max_ctas(d, kv_kind, use_tc))
    if ranged:
        # the splits follow the plain kernel's residency, so full-length ranges split exactly like the plain call;
        # the grid is bounded by the ranged kernel's own residency (cooperative launch)
        splits = _choose_splits(n if span is None else span, groups, resident)
        return DecodePlan(use_tc, groups, int(_ext.ops().tree_decode_max_ctas(d, kv_kind, use_tc, True, 0, paged)),
                          splits)
    return DecodePlan(use_tc, groups, resident, _choose_splits(n, groups, resident))


@dataclass
class _Buffers:
    rows: int
    d: int
    world: int
    rank: int
    partial_ptrs: List[int]
    aux_local_ptr: int
    pad_ptrs: List[int]
    mc_partial_ptr: int
    mc_aux_ptr: int
    counters: Tensor
    keep: tuple  # owners of the memory above
    scratch: Optional[Tensor] = None
    group_done: Optional[Tensor] = None


_cache: Dict[Tuple, _Buffers] = {}


def _layout(rows: int, d: int) -> Tuple[int, int, int, int]:
    """Byte offsets of (partials, aux, pads) inside one symmetric allocation and its total size."""
    partial_bytes = 2 * rows * (d + 4) * 4
    aux_bytes = 2 * 2 * rows * 4
    pad_bytes = PAD_WORDS * 4
    a = (partial_bytes + 255) // 256 * 256
    b = a + (aux_bytes + 255) // 256 * 256
    return 0, a, b, b + (pad_bytes + 255) // 256 * 256


def _alloc_symmetric(nbytes: int, dev: torch.device, world: int, rank: int):
    """(local uint8 tensor, per-rank base addresses, multicast base or 0, owner).  Tries torch's symmetric memory first
    (it can bind the allocation to an NVSwitch multicast object); falls back to the package's own IPC regions."""
    if world == 1:
        t = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        return t, [t.data_ptr()], 0, t
    if CONFIG["nvls"] in ("auto", True, "on"):
        try:
            import torch.distributed._symmetric_memory as symm_mem

            t = symm_mem.empty(nbytes, dtype=torch.uint8, device=dev)
            hdl = symm_mem.rendezvous(t, dist.group.WORLD)
            t.zero_()
            torch.cuda.synchronize(dev)
            dist.barrier()
            mc = int(getattr(hdl, "multicast_ptr", 0) or 0)
            return t, [int(x) for x in hdl.buffer_ptrs], mc, (t, hdl)
        except Exception as e:  # noqa: BLE001 - no fabric / multicast support: plain peer mappings still work
            if CONFIG["nvls"] in (True, "on"):
                raise
            _alloc_symmetric.last_error = f"{type(e).__name__}: {e}"
    from ring_attention_pytorch_b200.parallel.symm import get_workspace

    ws = get_workspace(world, dev)
    reg = ws.region(f"tree_decode_{nbytes}", nbytes)
    reg.local.zero_()
    torch.cuda.synchronize(dev)
    dist.barrier()
    return reg.local, list(reg.peer_ptrs), 0, reg


_alloc_symmetric.last_error = None


def _buffers(rows: int, d: int, dev: torch.device) -> _Buffers:
    world = get_world_size() if is_distributed() else 1
    rank = get_rank() if world > 1 else 0
    key = (dev.index, world, rows, d)
    buf = _cache.get(key)
    if buf is None:
        off_p, off_a, off_s, total = _layout(rows, d)
        local, bases, mc, owner = _alloc_symmetric(total, dev, world, rank)
        buf = _Buffers(rows=rows, d=d, world=world, rank=rank, partial_ptrs=[x + off_p for x in bases],
                       aux_local_ptr=bases[rank] + off_a, pad_ptrs=[x + off_s for x in bases],
                       mc_partial_ptr=(mc + off_p) if mc else 0, mc_aux_ptr=(mc + off_a) if mc else 0,
                       counters=torch.zeros(4, dtype=torch.int32, device=dev), keep=(local, owner))
        _cache[key] = buf
    return buf


def uses_nvls(q: Tensor) -> bool:
    """True when the decode of this (shape, device) merges through the NVSwitch multicast mapping."""
    b, h, m, d = q.shape
    key = (q.device.index, get_world_size() if is_distributed() else 1, b * h * m, d)
    return key in _cache and _cache[key].mc_partial_ptr != 0


def _is_cache_prefix(t: Tensor) -> bool:
    """[b, hk, n, d] with dense rows and uniformly strided (batch, head) planes: the filled prefix of a growing
    [b, hk, capacity, d] cache.  The tensor-core kernel reads it in place (tensor-map plane stride), no copy."""
    b, hk, n, d = t.shape
    sb, sh, sn, sd = t.stride()
    if t.is_contiguous():
        return True
    return (b > 1 and hk > 1 and sd == 1 and sn == d and sb == hk * sh and sh >= n * d
            and (sh * t.element_size()) % 16 == 0)


@torch.no_grad()
def tree_decode_cuda(
    q: Tensor,
    k: Optional[Tensor],
    v: Optional[Tensor],
    *,
    dim_v: int,
    eps: float = 1e-8,
    k_scale: Optional[Tensor] = None,
    v_scale: Optional[Tensor] = None,
    scale_block_keys: int = 0,
    out: Optional[Tensor] = None,
    sinks: Optional[Tensor] = None,
    cache_seqlens: Optional[Tensor] = None,
    q_pos: Optional[Tensor] = None,
    window: Optional[int] = None,
    kv_pos: Tuple[int, int] = (0, 1),
    softclamp_value: float = 0.0,
    block_table: Optional[Tensor] = None,
) -> Tensor:
    """q [b, h, m, d] (bf16 / fp16 / fp32; m >= 1 query tokens per sequence); k, v [b, hk, n, d] this rank's shard
    (bf16 / fp16 / float8_e4m3fn) or None.
    k / v may be the filled prefix ``cache[:, :, :n]`` of a larger ``[b, hk, capacity, d]`` buffer: the tensor-core kernel
    (head dim 128, n >= 128) reads it in place; other cases are made contiguous first.

    ``k_scale`` / ``v_scale``: optional fp32 dequantisation scales for the fp8 path, either per (batch, kv head)
    (``numel == b*hk``) or block-scaled ``[b*hk, n_blocks]`` with one scale per ``scale_block_keys`` keys
    (a multiple of 64).  ``out`` ([b, h, m, d]) may be passed to make the call allocation free (CUDA graphs).
    ``sinks`` (``[h]``, fp32 contiguous for an allocation-free call): learned attention sinks, added once per token row,
    in the kernel's cross-rank merge.  Returns [b, h, m, d] in q's dtype.

    Ragged and windowed decode.  Local key ``j`` sits at global position ``P(j) = kv_pos[0] + kv_pos[1] * j`` and is
    visible iff ``j < min(cache_seqlens[b], n)`` (int32 ``[b]``; None: every key), ``P(j) <= q_pos[b]`` (integer
    ``[b]``; int32 keeps the call allocation free) and, with ``window > 0``, ``q_pos[b] - P(j) <= window``.  The
    kernel derives each sequence's key range from the device tensors, so a decode loop can update them in place and
    replay a captured graph; the whole ``[b, hk, capacity, d]`` buffers may be passed.  ``softclamp_value > 0`` turns
    the logits into ``c * tanh(s / c)`` (not the sink).  A row that sees no key and has no sink gives 0.

    Multi-token decode (``m > 1``, e.g. verifying ``m`` draft tokens): query token ``t`` sits at ``q_pos[b] + t`` and
    each token applies the rule above at its own position, so the tokens are causal among themselves; their K / V are
    appended (and counted in ``cache_seqlens``) before the call.  Without ``q_pos`` there is no position rule: every
    token sees every held key.  One pass over the cache serves all ``m`` tokens.  ``q_pos + m - 1`` must fit in int32.

    Paged KV cache (``block_table``, int32 ``[b, max_pages]``, contiguous for an allocation-free call): ``k`` / ``v``
    are page pools ``[num_pages, hk, page_size, d]`` (an NHD pool ``[num_pages, page_size, hk, d]`` passed as
    ``.transpose(1, 2)`` works too) and local key ``j`` of sequence ``b`` is ``pool[block_table[b, j // page_size], :,
    j % page_size]``.  The call computes exactly the contiguous call on ``gather_paged_kv(pool, block_table)``
    (``ops/paged_kv.py``), ``n = max_pages * page_size``, with every rule above.  ``cache_seqlens`` is required;
    ``page_size`` is 16, 32 or a multiple of 64.  Table entries of pages that hold no key visible to a token of the
    call are never read, so they may point at any page (e.g. one freed behind a window and reused).  Entries are not
    checked (that would need a host sync) and must lie in ``[0, num_pages)``.
    """
    check_decode_query(q, out, dim_v, name="tree_decode_cuda")
    b, h, m, d = q.shape
    check_decode_ranges(b, q.device, cache_seqlens, q_pos, window, kv_pos, softclamp_value, name="tree_decode_cuda")
    check_paged_kv(b, q.device, k, v, block_table, cache_seqlens, name="tree_decode_cuda")
    ops = _ext.ops()
    paged = block_table is not None and block_table.shape[1] > 0
    ranged = cache_seqlens is not None or q_pos is not None or softclamp_value > 0 or m > 1 or paged
    assert dim_v == d, "the decode kernel assumes dim_v == dim_qk"
    dev = q.device
    q3 = q.reshape(b, h, d) if m == 1 else q
    if not q3.is_contiguous():
        q3 = q3.contiguous()
    if q3.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        q3 = q3.float()
    n, hk = 0, h
    if paged:
        if k.dtype == torch.float32:
            k, v = k.to(torch.bfloat16), v.to(torch.bfloat16)
        hk, n = k.shape[1], block_table.shape[1] * k.shape[2]
        block_table = block_table.contiguous()
    elif block_table is not None:  # no pages: this rank holds no keys
        k = v = None
    elif k is not None and k.shape[-2] > 0:
        if k.dtype == torch.float32:
            k, v = k.to(torch.bfloat16), v.to(torch.bfloat16)
        hk, n = k.shape[1], k.shape[2]
    else:
        k = v = None
    g = h // hk
    kv_kind = 0 if k is None or k.dtype == torch.bfloat16 else (1 if k.dtype == torch.float16 else 2)
    if m > 1:
        plan = decode_plan(b, h, hk, n, d, kv_kind, ranged=True, span=decode_span(n, window, int(kv_pos[1]), m),
                           tokens=m, paged=paged)
    elif ranged:
        plan = decode_plan(b, h, hk, n, d, kv_kind, ranged=True, span=decode_span(n, window, int(kv_pos[1])),
                           paged=paged)
    else:
        plan = decode_plan(b, h, hk, n, d, kv_kind)
    use_tc, groups, resident, splits = plan.tensor_core, plan.groups, plan.resident, plan.splits
    if k is not None and not paged and not (use_tc and _is_cache_prefix(k) and v.stride() == k.stride()):
        k, v = k.contiguous(), v.contiguous()  # no-op for dense inputs
    buf = _buffers(b * h * m, d, dev)
    need = b * hk * splits * g * m * (d + 4)  # scratch rows: (b, kv head, split, column), g * m columns
    if buf.scratch is None or buf.scratch.numel() < need:
        buf.scratch = torch.empty(need, dtype=torch.float32, device=dev)
    if buf.group_done is None or buf.group_done.numel() < b * hk * ((g * m + 3) // 4):
        buf.group_done = torch.zeros(b * hk * ((g * m + 3) // 4), dtype=torch.int32, device=dev)
    if out is None:
        out_dtype = q.dtype if q.dtype in (torch.bfloat16, torch.float16) else torch.float32
        out = torch.empty(b, h, m, d, dtype=out_dtype, device=dev)
    if sinks is not None:
        sinks = sinks.float().contiguous()
    units = groups * splits if n > 0 else 0
    grid = max(1, min(resident, max(units, (b * h * m + 3) // 4)))
    out_k = out.view(b, h, d) if m == 1 else out
    if ranged:
        if q_pos is not None and q_pos.dtype != torch.int32:
            q_pos = q_pos.to(torch.int32)
        ops.tree_decode(q3, k, v, k_scale, v_scale, buf.scratch, buf.group_done, buf.counters, buf.partial_ptrs,
                        buf.aux_local_ptr, buf.pad_ptrs, buf.mc_partial_ptr, buf.mc_aux_ptr, buf.rank, out_k,
                        hk, splits, d ** -0.5, scale_block_keys, eps, grid, use_tc, sinks,
                        cache_seqlens.contiguous() if cache_seqlens is not None else None, q_pos.contiguous()
                        if q_pos is not None else None, window or 0, int(kv_pos[0]), int(kv_pos[1]),
                        float(softclamp_value), block_table if paged else None)
    else:
        ops.tree_decode(q3, k, v, k_scale, v_scale, buf.scratch, buf.group_done, buf.counters, buf.partial_ptrs,
                        buf.aux_local_ptr, buf.pad_ptrs, buf.mc_partial_ptr, buf.mc_aux_ptr, buf.rank, out_k,
                        hk, splits, d ** -0.5, scale_block_keys, eps, grid, use_tc, sinks)
    LAUNCHES["count"] += 1
    return out
