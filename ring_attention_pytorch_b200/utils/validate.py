"""Runtime argument validation for the public constructors and ops.

The reference type-checks every public entry point with ``beartype`` (ring_attention.py:47, 103, 284, 489;
ring_flash_attention.py:391).  ``typecheck`` is that decorator when beartype is importable (it is a declared dependency and
listed in ``requirements.txt``) and a no-op otherwise, so the package stays importable on a bare PyTorch install.  On top
of the annotation checks, ``check_attention_inputs`` validates what annotations cannot express: tensor ranks, matching
batch / head-dim sizes, grouped-query divisibility and mask shapes — failing with a message that names the argument
instead of a kernel-launch assertion.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

try:  # pragma: no cover - exercised implicitly by every decorated call
    from beartype import BeartypeConf
    from beartype import beartype as _beartype

    # PEP 484 numeric tower: an int is accepted where a float is annotated (``theta=10000``, ``softclamp_value=50``)
    _checked = _beartype(conf=BeartypeConf(is_pep484_tower=True))

    def typecheck(fn):
        return _checked(fn)

    HAVE_BEARTYPE = True
except Exception:  # noqa: BLE001

    def typecheck(fn):
        return fn

    HAVE_BEARTYPE = False


def check_attention_inputs(q: Tensor, k: Tensor, v: Tensor, mask: Optional[Tensor] = None, *, name: str = "attention",
                           head_dim_first: bool = False, max_head_dim: Optional[int] = None) -> None:
    """q [b, n, h, d], k / v [b, n_k, hk, d] (or head-first).  Raises ValueError naming the offending argument."""
    for nm, t in (("q", q), ("k", k), ("v", v)):
        if not torch.is_tensor(t) or t.dim() != 4:
            raise ValueError(f"{name}: {nm} must be a 4-D tensor, got {tuple(t.shape) if torch.is_tensor(t) else type(t)}")
    hd, sd = (1, 2) if head_dim_first else (2, 1)
    if k.shape != v.shape:
        raise ValueError(f"{name}: k and v must have the same shape, got {tuple(k.shape)} and {tuple(v.shape)}")
    if q.shape[0] != k.shape[0]:
        raise ValueError(f"{name}: batch sizes differ: q {q.shape[0]}, k {k.shape[0]}")
    if q.shape[3] != k.shape[3]:
        raise ValueError(f"{name}: head dims differ: q {q.shape[3]}, k {k.shape[3]}")
    if q.shape[hd] % k.shape[hd] != 0:
        raise ValueError(f"{name}: query heads ({q.shape[hd]}) must be a multiple of key/value heads ({k.shape[hd]})")
    if max_head_dim is not None and q.shape[3] > max_head_dim:
        raise ValueError(f"{name}: head dim {q.shape[3]} exceeds the supported maximum {max_head_dim}")
    if not (q.device == k.device == v.device):
        raise ValueError(f"{name}: q, k, v must live on one device, got {q.device}, {k.device}, {v.device}")
    if mask is not None:
        if mask.dtype != torch.bool or mask.dim() != 2 or mask.shape[0] != k.shape[0] or mask.shape[1] != k.shape[sd]:
            raise ValueError(f"{name}: mask must be bool [batch, keys] = [{k.shape[0]}, {k.shape[sd]}], got "
                             f"{mask.dtype} {tuple(mask.shape)}")


def check_sinks(sinks: Optional[Tensor], heads: int, device, *, name: str = "attention") -> None:
    """Learned attention sinks: a floating ``[heads]`` tensor (one logit per query head) on the inputs' device."""
    if sinks is None:
        return
    if not torch.is_tensor(sinks) or sinks.dim() != 1 or sinks.shape[0] != heads:
        raise ValueError(f"{name}: sinks must be a 1-D tensor of one logit per query head [{heads}], got "
                         f"{tuple(sinks.shape) if torch.is_tensor(sinks) else type(sinks)}")
    if not sinks.is_floating_point():
        raise ValueError(f"{name}: sinks must be a floating tensor, got {sinks.dtype}")
    if sinks.device != torch.device(device):
        raise ValueError(f"{name}: sinks must live on {device}, got {sinks.device}")


def check_decode_query(q, out=None, dim_v: Optional[int] = None, *, name: str = "decode") -> None:
    """The query of a decode call: a 4-D ``[b, h, m, d]`` tensor with ``m >= 1`` query tokens per sequence, and
    ``out`` (when given) ``[b, h, m, dim_v]``."""
    if not torch.is_tensor(q) or q.dim() != 4:
        raise ValueError(f"{name}: q must be a 4-D tensor [batch, heads, tokens, dim], got "
                         f"{tuple(q.shape) if torch.is_tensor(q) else type(q)}")
    if q.shape[2] < 1:
        raise ValueError(f"{name}: q needs at least one query token per sequence, got shape {tuple(q.shape)}")
    if out is not None:
        want = (*q.shape[:3], q.shape[3] if dim_v is None else dim_v)
        if not torch.is_tensor(out) or tuple(out.shape) != want:
            raise ValueError(f"{name}: out must be {list(want)}, got "
                             f"{tuple(out.shape) if torch.is_tensor(out) else type(out)}")


def check_decode_ranges(batch: int, device, cache_seqlens: Optional[Tensor], q_pos: Optional[Tensor],
                        window: Optional[int], kv_pos, softclamp_value: float, *, name: str = "decode") -> None:
    """Per-sequence key ranges of a decode call: ``cache_seqlens`` int32 ``[batch]``, ``q_pos`` integer ``[batch]``,
    both on the inputs' device; ``window`` (>= 0) only with ``q_pos``; ``kv_pos = (offset >= 0, stride >= 1)``;
    ``softclamp_value >= 0``.  Values inside the tensors are not read (no host sync): lengths are clamped to the cache."""
    for nm, t, dtypes in (("cache_seqlens", cache_seqlens, (torch.int32,)),
                          ("q_pos", q_pos, (torch.int8, torch.int16, torch.int32, torch.int64, torch.uint8))):
        if t is None:
            continue
        if not torch.is_tensor(t) or t.dim() != 1 or t.shape[0] != batch:
            raise ValueError(f"{name}: {nm} must be a 1-D tensor of one entry per sequence [{batch}], got "
                             f"{tuple(t.shape) if torch.is_tensor(t) else type(t)}")
        if t.dtype not in dtypes:
            raise ValueError(f"{name}: {nm} must be {'int32' if len(dtypes) == 1 else 'an integer tensor'}, got {t.dtype}")
        if t.device != torch.device(device):
            raise ValueError(f"{name}: {nm} must live on {device}, got {t.device}")
    if window is not None:
        if q_pos is None:
            raise ValueError(f"{name}: a look-back window needs q_pos, the position of each sequence's query")
        if window < 0 or window >= 2 ** 31:
            raise ValueError(f"{name}: window must be in [0, 2**31), got {window}")
    if kv_pos is not None:
        if len(kv_pos) != 2 or not 0 <= int(kv_pos[0]) < 2 ** 31 or not 1 <= int(kv_pos[1]) < 2 ** 31:
            raise ValueError(f"{name}: kv_pos must be (offset >= 0, stride >= 1), got {tuple(kv_pos)}")
    if not softclamp_value >= 0.0:
        raise ValueError(f"{name}: softclamp_value must be >= 0, got {softclamp_value}")


def check_paged_kv(batch: int, device, k, v, block_table: Optional[Tensor], cache_seqlens: Optional[Tensor], *,
                   name: str = "decode") -> None:
    """A paged decode call: ``block_table`` int32 ``[batch, max_pages]`` on the inputs' device, ``cache_seqlens``
    given, and ``k`` / ``v`` page pools ``[num_pages, hk, page_size, d]`` of one shape, dtype and strides, with unit
    ``d`` stride, strides that are multiples of 16 bytes, ``page_size`` 16, 32 or a multiple of 64 and
    ``max_pages * page_size < 2**31``.  The table's entries are not read (no host sync); they must lie in
    ``[0, num_pages)``."""
    if block_table is None:
        return
    if not torch.is_tensor(block_table) or block_table.dim() != 2 or block_table.shape[0] != batch:
        raise ValueError(f"{name}: block_table must be a 2-D tensor [batch = {batch}, max_pages], got "
                         f"{tuple(block_table.shape) if torch.is_tensor(block_table) else type(block_table)}")
    if block_table.dtype != torch.int32:
        raise ValueError(f"{name}: block_table must be int32, got {block_table.dtype}")
    if block_table.device != torch.device(device):
        raise ValueError(f"{name}: block_table must live on {device}, got {block_table.device}")
    if cache_seqlens is None:
        raise ValueError(f"{name}: a paged cache (block_table) needs cache_seqlens, the keys held by each sequence")
    if not torch.is_tensor(k) or not torch.is_tensor(v):
        raise ValueError(f"{name}: block_table needs the k and v page pools")
    if k.dim() != 4 or k.shape != v.shape or k.dtype != v.dtype or k.stride() != v.stride():
        raise ValueError(f"{name}: the k and v page pools [num_pages, hk, page_size, d] must share shape, dtype and "
                         f"strides, got {k.dtype} {tuple(k.shape)} {k.stride()} and {v.dtype} {tuple(v.shape)} "
                         f"{v.stride()}")
    if k.stride(3) != 1:
        raise ValueError(f"{name}: the page pools need unit stride on the head dim, got strides {k.stride()}")
    ps = k.shape[2]
    if ps not in (16, 32) and not (ps > 0 and ps % 64 == 0):
        raise ValueError(f"{name}: page_size (pool dim 2) must be 16, 32 or a multiple of 64, got {ps}")
    if any(s * k.element_size() % 16 for s in k.stride()[:3]):
        raise ValueError(f"{name}: the page pools' strides must be multiples of 16 bytes, got {k.stride()} elements "
                         f"of {k.element_size()} bytes")
    if block_table.shape[1] * ps >= 2 ** 31:
        raise ValueError(f"{name}: max_pages * page_size must be below 2**31, got {block_table.shape[1]} * {ps}")


def check_fp8_attention_inputs(q: Tensor, k: Tensor, v: Tensor, q_descale, k_descale, v_descale,
                               mask: Optional[Tensor] = None, *, name: str = "attention",
                               rotary_freqs: Optional[Tensor] = None, sinks: Optional[Tensor] = None) -> None:
    """Inputs of the fp8 forward: e4m3 q / k / v with the shapes of :func:`check_attention_inputs`, fp32 descales
    ``[b, h]`` (q) and ``[b, hk]`` (k, v) or one element each, sinks as :func:`check_sinks`, nothing that requires
    grad, no rotary angles."""
    check_attention_inputs(q, k, v, mask, name=name)
    for nm, t in (("q", q), ("k", k), ("v", v)):
        if t.dtype != torch.float8_e4m3fn:
            raise ValueError(f"{name}: {nm} must be torch.float8_e4m3fn, got {t.dtype}")
    b, h, hk = q.shape[0], q.shape[2], k.shape[2]
    for nm, t, heads in (("q_descale", q_descale, h), ("k_descale", k_descale, hk), ("v_descale", v_descale, hk)):
        if not torch.is_tensor(t) or t.dtype != torch.float32:
            raise ValueError(f"{name}: {nm} must be a float32 tensor")
        if t.numel() != 1 and tuple(t.shape) != (b, heads):
            raise ValueError(f"{name}: {nm} must be [batch, heads] = [{b}, {heads}] or have one element, got "
                             f"{tuple(t.shape)}")
        if t.device != q.device:
            raise ValueError(f"{name}: {nm} must live on {q.device}, got {t.device}")
    check_sinks(sinks, h, q.device, name=name)
    if any(t is not None and t.requires_grad for t in (q, k, v, q_descale, k_descale, v_descale, sinks)):
        raise ValueError(f"{name}: the fp8 attention is forward only; an input requires grad")
    if rotary_freqs is not None:
        raise ValueError(f"{name}: rotary_freqs is not accepted; rotate q and k first, then quantise them")
