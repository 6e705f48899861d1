"""Document masking for packed sequences: document ids -> per-token intervals of global positions.

Many documents packed into one row must not attend across their boundaries.  A *document* is a maximal run
of equal ids in **global** position order (two separate runs that happen to share an id are two documents);
query ``i`` may see key ``j`` only if both lie in the same run.  The rule is applied on top of the causal
rule, the look-back window and the key mask.

This module is the one place that turns ids into the representation every attention path consumes: for
every ring rank ``r``, batch row ``b`` and local index ``i``, the half-open interval ``[start, end)`` of
global positions of the document holding token ``pos(r, i)``, as an int32 table ``[ring, b, n, 2]``.
q and k share a document iff ``pos(k)`` lies in q's interval iff ``pos(q)`` lies in k's, so the kernels
only ever read the intervals of their own stationary rows (``csrc/attn_common.cuh``).

Everything here runs as device tensor ops without host synchronisation.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist
from torch import Tensor

from ring_attention_pytorch_b200.parallel.distributed import get_rank, get_world_size
from ring_attention_pytorch_b200.parallel.layout import PositionMap, make_position_map


def document_spans(ids: Tensor, pm: PositionMap) -> Tensor:
    """Every ring rank's document ids ``[ring, b, n]`` (each in the layout of ``pm``) -> int32 ``[ring, b, n, 2]``
    intervals ``[start, end)`` of global positions of each token's document."""
    world, b, n = ids.shape
    assert world == pm.world and n == pm.n, "ids must be [ring, b, n] in the layout of the position map"
    dev = ids.device
    total = world * n
    pos = torch.cat([pm.positions(r, dev) for r in range(world)])            # [ring * n]: local slot -> position
    glob = torch.empty(b, total, dtype=ids.dtype, device=dev)
    glob[:, pos] = ids.permute(1, 0, 2).reshape(b, total)                    # ids in global position order
    idx = torch.arange(total, device=dev).expand(b, total)
    first = torch.ones(b, total, dtype=torch.bool, device=dev)
    first[:, 1:] = glob[:, 1:] != glob[:, :-1]                               # a run starts here
    last = torch.ones_like(first)
    last[:, :-1] = first[:, 1:]                                              # a run ends here
    start = torch.where(first, idx, torch.zeros_like(idx)).cummax(dim=1).values
    end = torch.where(last, idx + 1, torch.full_like(idx, total)).flip(1).cummin(dim=1).values.flip(1)
    spans = torch.stack((start, end), dim=-1)[:, pos]                        # back to the layout: [b, ring * n, 2]
    return spans.view(b, world, n, 2).permute(1, 0, 2, 3).to(torch.int32).contiguous()


def _gather_ring_ids(ids: Tensor, ring_size: int) -> Tensor:
    """[b, n] ids on every rank -> [ring, b, n] for this rank's ring set (cold path, one all-gather)."""
    world = get_world_size()
    local = ids.to(torch.int32).contiguous()
    gathered = [torch.empty_like(local) for _ in range(world)]
    dist.all_gather(gathered, local)
    ring_set = get_rank() // ring_size
    return torch.stack(gathered[ring_set * ring_size:(ring_set + 1) * ring_size])


def ring_document_spans(document_ids: Tensor, pm: PositionMap, use_ring: bool) -> Tensor:
    """This rank's ``document_ids`` ``[b, n]`` (laid out like ``q``) -> the ``[ring, b, n, 2]`` interval table of
    the whole ring.  ``use_ring``: gather the other ranks' ids over this rank's ring set, else ``pm`` is a
    one-rank map and the local ids are the whole sequence."""
    assert document_ids.dim() == 2 and document_ids.shape[1] == pm.n, "document_ids must be [b, n] like q"
    assert not document_ids.is_floating_point() and document_ids.dtype != torch.bool, "document_ids must be integers"
    ids = _gather_ring_ids(document_ids, pm.world) if use_ring else document_ids[None]
    return document_spans(ids, pm)


def document_mask(q_spans: Tensor, k_pos: Tensor) -> Tensor:
    """``[b, i, 2]`` query intervals and ``[j]`` key positions -> bool ``[b, i, j]``: key in the query's document."""
    return (q_spans[..., 0:1] <= k_pos) & (k_pos < q_spans[..., 1:2])


def document_runs(document_ids: Tensor) -> Tensor:
    """Unsharded ``[b, n]`` ids -> ``[b, n]`` labels, equal iff two tokens are in the same run (its start)."""
    return document_spans(document_ids[None], make_position_map("plain", 1, document_ids.shape[1]))[0, ..., 0]


def check_document_ids(document_ids: Optional[Tensor], q: Tensor, k: Tensor) -> None:
    if document_ids is None:
        return
    if q.shape[1] != k.shape[1]:
        raise ValueError("document_ids needs self-attention: q and k must have the same sequence length")
    if tuple(document_ids.shape) != tuple(q.shape[:2]):
        raise ValueError(f"document_ids must be [b, n] = {tuple(q.shape[:2])}, got {tuple(document_ids.shape)}")
