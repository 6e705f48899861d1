"""Dense attention oracles (plain PyTorch, any device, any float dtype).

``default_attention`` mirrors the public oracle of the reference (ring_attention.py:47-98) including its
grouped-query head mapping (query head ``j`` reads kv head ``j % kv_heads``) and its "mask is ignored
when causal" rule.  ``attention_with_positions`` is the general oracle every kernel and every ring
schedule in this repository is validated against: visibility is decided from explicit global token
positions, so plain / striped / zig-zag shards, look-back windows and key padding are all one code
path.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from ring_attention_pytorch_b200.utils.tensor_typing import Bool, Float
from ring_attention_pytorch_b200.utils.validate import typecheck


def softclamp(t: Tensor, value: float) -> Tensor:
    return (t / value).tanh() * value


def expand_kv_heads(t: Tensor, heads: int) -> Tensor:
    """[b, n, hk, d] -> [b, n, h, d] with query head j <- kv head j % hk (reference '(g h)' repeat)."""
    hk = t.shape[-2]
    assert heads % hk == 0
    if hk == heads:
        return t
    g = heads // hk
    return t.repeat(*([1] * (t.ndim - 2)), g, 1)


def attention_with_positions(
    q: Tensor,
    k: Tensor,
    v: Tensor,
    q_pos: Optional[Tensor] = None,
    k_pos: Optional[Tensor] = None,
    *,
    causal: bool = False,
    window: Optional[int] = None,
    key_mask: Optional[Tensor] = None,
    softclamp_value: float = 0.0,
    scale: Optional[float] = None,
    return_lse: bool = False,
    q_doc: Optional[Tensor] = None,
    k_doc: Optional[Tensor] = None,
    sinks: Optional[Tensor] = None,
):
    """q [b, i, h, d]; k, v [b, j, hk, d]; q_pos [i], k_pos [j] integer global positions.

    ``q_doc`` [b, i] / ``k_doc`` [b, j]: document labels, a query sees only keys with its label (on top of every other
    rule).  Labels must be unique per document, e.g. the start column of ``parallel.documents.document_spans``.
    Rows with no visible key produce zeros (and ``lse = +inf``).

    ``sinks`` [h]: learned attention sinks, one logit per query head (not softclamped) that joins every row's softmax
    denominator with a zero value vector: ``lse = log(exp(sinks[h]) + sum_j exp(s_ij))``, ``out = sum_j exp(s_ij -
    lse) v_j``.  A row with no visible key gives zeros and ``lse = sinks[h]``.
    """
    b, i, h, d = q.shape
    j = k.shape[1]
    scale = d ** -0.5 if scale is None else scale
    kx, vx = expand_kv_heads(k, h), expand_kv_heads(v, h)
    sim = torch.einsum("bihd,bjhd->bhij", q, kx) * scale
    if softclamp_value and softclamp_value > 0:
        sim = softclamp(sim, softclamp_value)
    visible = torch.ones(b, 1, i, j, dtype=torch.bool, device=q.device)
    if causal:
        if q_pos is None:
            q_pos = torch.arange(i, device=q.device) + (j - i)
        if k_pos is None:
            k_pos = torch.arange(j, device=q.device)
        rel = q_pos[:, None] - k_pos[None, :]
        vis = rel >= 0
        if window is not None and window > 0:
            vis = vis & (rel <= window)
        visible = visible & vis[None, None]
    if key_mask is not None:
        visible = visible & key_mask[:, None, None, :]
    if q_doc is not None:
        visible = visible & (q_doc[:, None, :, None] == k_doc[:, None, None, :])
    neg = torch.finfo(sim.dtype).min
    sim = sim.masked_fill(~visible, neg)
    if sinks is not None:  # one more column per row: the sink logit, always visible, with a zero value
        sim = torch.cat((sim, sinks.to(sim.dtype)[None, :, None, None].expand(b, h, i, 1)), dim=-1)
        visible = torch.cat((visible.expand(b, h, i, j), visible.new_ones(b, h, i, 1)), dim=-1)
    any_vis = visible.any(dim=-1, keepdim=True)
    m = sim.amax(dim=-1, keepdim=True)
    p = (sim - m).exp().masked_fill(~visible, 0.0)
    l = p.sum(dim=-1, keepdim=True)
    attn = torch.where(any_vis, p / l.clamp(min=torch.finfo(sim.dtype).tiny), torch.zeros_like(p))
    out = torch.einsum("bhij,bjhd->bihd", attn[..., :j], vx)
    if return_lse:
        lse = torch.where(any_vis, m + l.clamp(min=torch.finfo(sim.dtype).tiny).log(),
                          torch.full_like(m, float("inf"))).squeeze(-1)
        return out, lse
    return out


@typecheck
def default_attention(
    q: Float["b i h d"],
    k: Float["b j hk d"],
    v: Float["b j hk d"],
    mask: Optional[Bool["b j"]] = None,
    causal: bool = False,
    softclamp_qk_sim: bool = False,
    softclamp_value: float = 50.0,
) -> Tensor:
    """Reference-compatible dense attention, layout (b, n, h, d) (ring_attention.py:47-98)."""
    return attention_with_positions(
        q, k, v,
        causal=causal,
        key_mask=None if causal else mask,
        softclamp_value=softclamp_value if softclamp_qk_sim else 0.0,
    )
