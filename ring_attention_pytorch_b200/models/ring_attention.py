"""nn modules: RingAttention, RingTransformer, RingRotaryEmbedding, RMSNorm, FeedForward and the
batch<->sequence resharding helpers.

Capability and state-dict parity with reference ring_attention.py (file:lines cited per symbol); the
parameter names (``to_qkv.0.gamma``, ``to_qkv.1.weight``, ``to_out.weight``, ``token_emb.weight``,
``layers.N.0/1...``, ``to_logits.*``) are identical, so a reference checkpoint loads unchanged.

Differences, all of them fixes of behaviour the reference gets wrong (SURVEY.md §2.8):

* one striping permutation for every backend (rank r holds tokens ``i*W + r`` – the reference uses a
  different, bucket-granular permutation on its CPU path);
* rotary positions come from the same position map the attention kernels use and are **ring-local**
  (reference ring_attention.py:143-150 uses the global rank / world size, wrong for ring sets – D6);
* ``RingAttention(auto_shard_seq=True)`` derives the ring size from the number of sharded batches (D5);
* the batch/sequence all-gathers back-propagate with a reduce-scatter (D8);
* ``return_loss`` with no padding mask works (D10).
"""
from __future__ import annotations

from typing import Optional, Union

import torch
import torch.nn.functional as F
from torch import Tensor, nn
from torch.nn import Module, ModuleList

from ring_attention_pytorch_b200.ops.oracle import attention_with_positions, default_attention
from ring_attention_pytorch_b200.ops.ring_flash_naive import ring_flash_attn
from ring_attention_pytorch_b200.parallel.distributed import (
    AllGather,
    default,
    divisible_by,
    exists,
    get_rank,
    get_world_size,
    is_distributed,
    split_by_rank,
)
from ring_attention_pytorch_b200.parallel.documents import document_runs
from ring_attention_pytorch_b200.parallel.layout import make_position_map
from ring_attention_pytorch_b200.utils.validate import typecheck


def cuda_kernels_usable(dim_head: int = 64) -> bool:
    """Default of ``use_cuda_kernel``: the hand-written kernels are built for sm_90a (Hopper) only and cover head dims up
    to 128; on any other GPU (or larger heads) the modules use the portable ring op instead of failing at launch."""
    if not torch.cuda.is_available() or dim_head > 128:
        return False
    try:
        return torch.cuda.get_device_capability() == (9, 0)
    except Exception:  # noqa: BLE001
        return False


def cast_tuple(t, length: int = 1):
    return t if isinstance(t, tuple) else ((t,) * length)


# ------------------------------------------------------------------------------------------------
# rotary embeddings aware of the sequence layout (reference ring_attention.py:102-172)
# ------------------------------------------------------------------------------------------------
class RingRotaryEmbedding(Module):
    @typecheck
    def __init__(self, dim: int, ring: bool = False, striped: bool = False, buckets: int = 1, theta: float = 10000):
        super().__init__()
        self.ring = ring
        self.striped = striped
        self.buckets = buckets  # kept for signature parity; striping is always token-granular here
        inv_freq = theta ** -(torch.arange(0, dim, 2).float() / dim)
        self.register_buffer("inv_freq", inv_freq)

    @property
    def device(self):
        return self.inv_freq.device

    def positions(self, seq: int, ring_size: Optional[int] = None, layout: Optional[str] = None) -> Tensor:
        """Global token positions of the ``seq`` local indices held by this rank."""
        if not (self.ring and is_distributed()):
            return torch.arange(seq, device=self.device)
        ring_size = default(ring_size, get_world_size())
        layout = default(layout, "striped" if self.striped else "plain")
        pm = make_position_map(layout, ring_size, seq)
        return pm.positions(get_rank() % ring_size, self.device)

    @torch.autocast("cuda", enabled=False)
    def forward(self, seq: Union[int, Tensor], ring_size: Optional[int] = None, layout: Optional[str] = None) -> Tensor:
        pos = seq if torch.is_tensor(seq) else self.positions(seq, ring_size, layout)
        pos = pos.to(self.inv_freq.dtype)
        freqs = torch.einsum("i,j->ij", pos, self.inv_freq)
        return torch.cat((freqs, freqs), dim=-1)


@torch.autocast("cuda", enabled=False)
def apply_rotary_pos_emb(pos: Tensor, t: Tensor, head_dim_first: bool = False) -> Tensor:
    """Rotate feature pairs ``(i, i + d/2)`` of ``t`` ([b, n, h, d], or [b, h, n, d] with ``head_dim_first``) by the
    angles ``pos`` [n, d] (both halves of ``pos`` carry the same d/2 angles).  Same convention as the reference
    (ring_attention.py:160-172) and as ``csrc/elementwise_sm90.cu::rotary_kernel``; computed in fp32."""
    ang = pos if head_dim_first else pos.unsqueeze(1)
    half = t.shape[-1] // 2
    cos, sin = ang.cos(), ang.sin()
    lo, hi = t[..., :half].float(), t[..., half:].float()
    out = torch.cat((lo * cos[..., :half] - hi * sin[..., :half], hi * cos[..., half:] + lo * sin[..., half:]), dim=-1)
    return out.to(t.dtype)


# ------------------------------------------------------------------------------------------------
# padding and batch <-> sequence resharding (reference ring_attention.py:176-279)
# ------------------------------------------------------------------------------------------------
def _pad_tokens(t: Tensor, multiple: int, value) -> Tensor:
    """Right-pad axis 1 (tokens) of ``t`` to the next multiple of ``multiple``."""
    missing = -t.shape[1] % multiple
    if missing == 0:
        return t
    filler = t.new_full((t.shape[0], missing, *t.shape[2:]), value)
    return torch.cat((t, filler), dim=1)


def maybe_pad_seq_and_mask(x: Tensor, mask: Optional[Tensor], seq_size: int):
    """Pad tokens (and the key mask, created on demand so that the padding is masked out) to a multiple of ``seq_size``."""
    if x.shape[1] % seq_size == 0:
        return x, mask
    if mask is None:
        mask = torch.ones(x.shape[:2], device=x.device, dtype=torch.bool)
    return _pad_tokens(x, seq_size, 0), _pad_tokens(mask, seq_size, False)


def pad_document_ids(document_ids: Tensor, seq_size: int) -> Tensor:
    """Right-pad ``[b, n]`` document ids to a multiple of ``seq_size`` with an id that differs from each row's last one,
    so the padding is a document of its own."""
    missing = -document_ids.shape[1] % seq_size
    if missing == 0:
        return document_ids
    return torch.cat((document_ids, (document_ids[:, -1:] + 1).expand(-1, missing)), dim=1)


def stripe(t: Tensor, ring_seq_size: int) -> Tensor:
    """'b (i j) ... -> b (j i) ...' with i = ring_seq_size: chunk r of the result holds tokens i*W + r."""
    b, n = t.shape[:2]
    j = n // ring_seq_size
    return t.reshape(b, ring_seq_size, j, *t.shape[2:]).transpose(1, 2).reshape(b, n, *t.shape[2:])


def unstripe(t: Tensor, ring_seq_size: int) -> Tensor:
    b, n = t.shape[:2]
    j = n // ring_seq_size
    return t.reshape(b, j, ring_seq_size, *t.shape[2:]).transpose(1, 2).reshape(b, n, *t.shape[2:])


def sharded_batch_to_sharded_seq(x: Tensor, mask: Optional[Tensor], seq_size: int):
    """All-gather the (possibly uneven) batch, fold ``num_sharded_batches`` rows into the sequence axis and
    take this rank's ``seq_size`` chunk (reference ring_attention.py:223-262)."""
    assert is_distributed()
    all_gather = AllGather(dim=0)
    x, sizes = all_gather(x)
    if exists(mask):
        mask, _ = all_gather(mask)

    world_size = get_world_size()
    total_split_seq = x.shape[1] // seq_size
    assert divisible_by(world_size, total_split_seq), (
        f"world size {world_size} must be divisible by the number of sequence chunks {total_split_seq}")
    num_sharded_batches = world_size // total_split_seq
    assert divisible_by(x.shape[0], num_sharded_batches), "total batch must be divisible by the number of ring sets"

    def fold(t: Tensor) -> Tensor:
        bs = t.shape[0] // num_sharded_batches
        return t.reshape(bs, num_sharded_batches * t.shape[1], *t.shape[2:])

    x = fold(x).split(seq_size, dim=1)
    x, _ = split_by_rank(x)
    if exists(mask):
        mask = fold(mask).split(seq_size, dim=1)
        mask, _ = split_by_rank(mask)
    return (x, mask), sizes, num_sharded_batches


def sharded_seq_to_sharded_batch(logits: Tensor, sizes: Tensor, num_sharded_batches: int = 1) -> Tensor:
    """reference ring_attention.py:264-279"""
    all_gather = AllGather(dim=-2)
    logits, _ = all_gather(logits)
    b, n = logits.shape[:2]
    logits = logits.reshape(b * num_sharded_batches, n // num_sharded_batches, *logits.shape[2:])
    logits = logits.split(sizes.tolist(), dim=0)
    logits, _ = split_by_rank(logits)
    return logits


# ------------------------------------------------------------------------------------------------
# layers
# ------------------------------------------------------------------------------------------------
class RMSNorm(Module):
    """x / rms(x) * gamma, written as unit-normalise times sqrt(dim) (parameter name ``gamma`` as in the reference,
    ring_attention.py:470-477, so that its checkpoints load)."""

    def __init__(self, dim: int):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(dim))
        self.sqrt_dim = float(dim) ** 0.5

    def forward(self, x: Tensor) -> Tensor:
        unit = x / x.norm(dim=-1, keepdim=True).clamp_min(1e-12)  # what F.normalize computes
        return unit * (self.sqrt_dim * self.gamma)


class BlockwiseSequential(nn.Sequential):
    """``nn.Sequential`` applied to the sequence axis in blocks of ``chunk_size`` tokens, each block recomputed in
    the backward (blockwise feed-forward of the Ring Attention paper, which the reference only draws in
    ``ring.png``): the ``[b, n, 4 * dim]`` inner activation never exists for more than one block.  Child indices,
    hence state-dict keys, are those of a plain ``nn.Sequential``."""

    def __init__(self, *mods, chunk_size: Optional[int] = None):
        super().__init__(*mods)
        self.chunk_size = chunk_size

    def forward(self, x: Tensor) -> Tensor:
        run = super().forward
        if not self.chunk_size or x.shape[-2] <= self.chunk_size:
            return run(x)
        if torch.is_grad_enabled() and x.requires_grad:
            from torch.utils.checkpoint import checkpoint

            outs = [checkpoint(run, c, use_reentrant=False) for c in x.split(self.chunk_size, dim=-2)]
        else:
            outs = [run(c) for c in x.split(self.chunk_size, dim=-2)]
        return torch.cat(outs, dim=-2)


def FeedForward(dim: int, mult: int = 4, chunk_size: Optional[int] = None) -> nn.Sequential:
    """reference ring_attention.py:479-486; ``chunk_size`` (extra) makes it blockwise over the sequence."""
    dim_inner = int(dim * mult)
    return BlockwiseSequential(RMSNorm(dim), nn.Linear(dim, dim_inner), nn.GELU(), nn.Linear(dim_inner, dim),
                               chunk_size=chunk_size)


class RingAttention(Module):
    """Multi-head / grouped-query attention whose sequence dimension may be sharded over a ring of ranks
    (reference ring_attention.py:283-466, same constructor and forward signature)."""

    @typecheck
    def __init__(
        self,
        dim: int,
        *,
        dim_head: int = 64,
        heads: int = 8,
        num_grouped_query_heads: int = 1,
        causal: bool = False,
        eps: float = 1e-10,
        bucket_size: int = 512,
        ring_attn: bool = False,
        ring_seq_size: int = 512,
        max_lookback_seq_len: Optional[int] = None,
        striped_ring_attn: bool = False,
        auto_shard_seq: bool = False,
        prenorm: bool = True,
        force_regular_attn: bool = False,
        rotary_embed: bool = False,
        rotary_embed_theta: int = 10000,
        use_cuda_kernel: Optional[bool] = None,
        fp8_attn: bool = False,
        attn_sinks: bool = False,
    ):
        """``fp8_attn``: forward-only e4m3 attention for inference prefill (call under ``torch.no_grad()``).  q, k and v
        are quantised with :func:`ring_attention_pytorch_b200.ops.ring_fp8.quantize_fp8` (per-(batch, head) scales over
        the ring set) and attended with ``ring_flash_attn_fp8``; rotary embedding is applied before the quantisation.

        ``attn_sinks``: a learned attention sink per query head, the parameter ``sinks`` ``[heads]`` (initialised to
        zero), which every attention path honours (see :func:`ring_attention_pytorch_b200.ops.ring_flash_naive.
        ring_flash_attn`).  Without it the module has no such parameter, so checkpoints without sinks load unchanged."""
        super().__init__()
        use_cuda_kernel = default(use_cuda_kernel, cuda_kernels_usable(dim_head))
        assert not (use_cuda_kernel and not torch.cuda.is_available())
        self.use_cuda_kernel = use_cuda_kernel
        assert not (fp8_attn and force_regular_attn), "fp8_attn runs the ring op, not the regular attention"
        self.fp8_attn = fp8_attn

        self.eps = eps
        self.heads = heads
        self.dim_head = dim_head
        assert divisible_by(heads, num_grouped_query_heads), (
            f"number of query heads ({heads}) must be divisible by the groups ({num_grouped_query_heads})")
        kv_heads = heads // num_grouped_query_heads
        self.num_grouped_query_heads = num_grouped_query_heads
        self.qkv_head_breakdown = (heads, kv_heads, kv_heads)
        self.scale = dim_head ** -0.5
        self.causal = causal

        assert (not ring_attn) or divisible_by(ring_seq_size, bucket_size), (
            f"ring seq size {ring_seq_size} is not divisible by bucket size {bucket_size}")
        self.ring_attn = ring_attn
        self.max_lookback_seq_len = max_lookback_seq_len
        self.striped_ring_attn = striped_ring_attn
        self.force_regular_attn = force_regular_attn
        self.auto_shard_seq = default(auto_shard_seq, ring_attn)
        assert not (not self.ring_attn and self.auto_shard_seq)
        self.ring_seq_size = ring_seq_size
        self.bucket_size = bucket_size

        self.rotary_embed = None
        if rotary_embed:
            self.rotary_embed = RingRotaryEmbedding(dim=dim_head, ring=ring_attn, striped=striped_ring_attn,
                                                    theta=rotary_embed_theta, buckets=ring_seq_size // bucket_size)

        dim_inner = dim_head * heads
        dim_kv_inner = dim_head * kv_heads
        self.to_qkv_split = (dim_inner, dim_kv_inner, dim_kv_inner)
        self.to_qkv = nn.Sequential(
            RMSNorm(dim) if prenorm else nn.Identity(),
            nn.Linear(dim, dim_inner + (dim_kv_inner * 2), bias=False),
        )
        self.to_out = nn.Linear(dim_inner, dim, bias=False)
        self.sinks = nn.Parameter(torch.zeros(heads)) if attn_sinks else None

    def forward(
        self,
        x: Tensor,
        mask: Optional[Tensor] = None,
        rotary_emb: Optional[Tensor] = None,
        force_ring_reduce_off: bool = False,
        ring_size: Optional[int] = None,
        document_ids: Optional[Tensor] = None,
    ) -> Tensor:
        """``document_ids`` (integer ``[b, n]``, laid out like ``x``): document masking for packed sequences, see
        :func:`ring_attention_pytorch_b200.ops.ring_cuda.ring_flash_attn_cuda`.  It follows ``x`` through the padding,
        striping and sharding, and is honoured by every attention path."""
        ring_size = default(ring_size, get_world_size())
        ring_attn = self.ring_attn and is_distributed()
        auto_shard_seq = self.auto_shard_seq and is_distributed()
        seq_len = x.shape[1]

        if auto_shard_seq:
            x, mask = maybe_pad_seq_and_mask(x, mask, self.ring_seq_size)
            if exists(document_ids):
                document_ids = pad_document_ids(document_ids, self.ring_seq_size)
            if self.striped_ring_attn:
                x = stripe(x, self.ring_seq_size)
                if exists(mask):
                    mask = stripe(mask, self.ring_seq_size)
                if exists(document_ids):
                    document_ids = stripe(document_ids, self.ring_seq_size)
            (x, mask), batch_sizes, num_sharded_batches = sharded_batch_to_sharded_seq(x, mask, self.ring_seq_size)
            if exists(document_ids):
                (document_ids, _), *_ = sharded_batch_to_sharded_seq(document_ids, None, self.ring_seq_size)
            ring_size = get_world_size() // num_sharded_batches

        qkv = self.to_qkv(x)
        b, n = qkv.shape[:2]
        q, k, v = qkv.view(b, n, -1, self.dim_head).split(self.qkv_head_breakdown, dim=-2)

        use_ring = ring_attn and not force_ring_reduce_off
        if self.fp8_attn and torch.is_grad_enabled():
            raise ValueError("RingAttention(fp8_attn=True) is forward only: call it under torch.no_grad()")
        if not exists(rotary_emb) and exists(self.rotary_embed):
            rotary_emb = self.rotary_embed(n, ring_size if use_ring else 1) if use_ring else \
                self.rotary_embed(torch.arange(n, device=x.device))
        any_cuda_inputs = any(t.is_cuda for t in (q, k, v))
        kernel_path = any_cuda_inputs and self.use_cuda_kernel and not self.force_regular_attn
        # On the sm_90a path the rotation of q and k happens inside the op's pack kernels (fp32 sincos from the same
        # angles, fused with the head-major repack): no eager elementwise passes over q and k.
        fuse_rotary = kernel_path and exists(rotary_emb) and self.dim_head % 16 == 0 and not self.fp8_attn
        if exists(rotary_emb) and not fuse_rotary:
            q = apply_rotary_pos_emb(rotary_emb, q)
            k = apply_rotary_pos_emb(rotary_emb, k)

        sinks = self.sinks
        if self.force_regular_attn and (exists(document_ids) or exists(sinks)):
            runs = document_runs(document_ids) if exists(document_ids) else None
            out = attention_with_positions(q, k, v, causal=self.causal, key_mask=None if self.causal else mask,
                                           q_doc=runs, k_doc=runs, sinks=sinks)
        elif self.force_regular_attn:
            out = default_attention(q, k, v, mask=mask, causal=self.causal)
        elif self.fp8_attn:
            from ring_attention_pytorch_b200.ops.ring_fp8 import (dequantized_ring_flash_attn, quantize_fp8,
                                                                  ring_flash_attn_fp8)

            (q8, qd), (k8, kd), (v8, vd) = (quantize_fp8(t, ring_size if use_ring else 1) for t in (q, k, v))
            args = (mask, self.causal, self.bucket_size, use_ring, self.striped_ring_attn and use_ring,
                    self.max_lookback_seq_len, ring_size)
            # off the kernel path the op's definition runs: the portable ring op on the dequantised inputs
            attn = ring_flash_attn_fp8 if kernel_path else dequantized_ring_flash_attn
            out = attn(q8, k8, v8, qd, kd, vd, *args, document_ids=document_ids,
                       sinks=sinks.detach() if exists(sinks) else None).to(q.dtype)
        elif kernel_path:
            from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda

            out = ring_flash_attn_cuda(q, k, v, mask, self.causal, self.bucket_size, use_ring,
                                       self.striped_ring_attn and use_ring, self.max_lookback_seq_len, ring_size,
                                       rotary_freqs=rotary_emb if fuse_rotary else None, document_ids=document_ids,
                                       sinks=sinks)
        else:
            out = ring_flash_attn(q, k, v, mask, self.causal, self.bucket_size, use_ring,
                                  self.striped_ring_attn and use_ring, self.max_lookback_seq_len, ring_size,
                                  document_ids=document_ids, sinks=sinks)

        out = out.reshape(b, n, -1)
        out = self.to_out(out)

        if auto_shard_seq:
            out = sharded_seq_to_sharded_batch(out, batch_sizes, num_sharded_batches)
            if self.striped_ring_attn:
                out = unstripe(out, self.ring_seq_size)
            out = out[:, :seq_len]
        return out


class RingTransformer(Module):
    """Small decoder/encoder stack for end-to-end tests and benchmarks (reference ring_attention.py:488-685)."""

    @typecheck
    def __init__(
        self,
        *,
        num_tokens: int,
        dim: int,
        depth: int,
        causal: bool = False,
        dim_head: int = 64,
        heads: int = 8,
        ff_mult: int = 4,
        num_grouped_query_heads: int = 1,
        bucket_size: int = 512,
        ring_attn: bool = False,
        striped_ring_attn: bool = False,
        ring_seq_size: int = 512,
        auto_shard_seq: Optional[bool] = None,
        max_lookback_seq_len: Union[tuple[Optional[int], ...], int, None] = None,
        rotary_embed_theta: int = 10000,
        ignore_index: int = -1,
        force_regular_attn: bool = False,
        use_cuda_kernel: Optional[bool] = None,
        ff_chunk_size: Optional[int] = None,
        fp8_attn: bool = False,
        attn_sinks: bool = False,
    ):
        """``attn_sinks``: a learned attention sink per query head in every layer (see :class:`RingAttention`)."""
        super().__init__()
        use_cuda_kernel = default(use_cuda_kernel, cuda_kernels_usable(dim_head))
        self.use_cuda_kernel = use_cuda_kernel
        assert not (use_cuda_kernel and not torch.cuda.is_available())

        self.ring_attn = ring_attn
        self.striped_ring_attn = striped_ring_attn
        self.ring_seq_size = ring_seq_size
        self.bucket_size = bucket_size
        assert (not ring_attn) or divisible_by(ring_seq_size, bucket_size), (
            f"ring seq size {ring_seq_size} is not divisible by bucket size {bucket_size}")
        self.auto_shard_seq = default(auto_shard_seq, ring_attn)
        assert not (not self.ring_attn and self.auto_shard_seq)
        assert not (not self.ring_attn and self.striped_ring_attn)
        assert not (self.striped_ring_attn and not causal), "striped ring attention only applies to autoregressive models"

        self.token_emb = nn.Embedding(num_tokens, dim)
        self.rotary_emb = RingRotaryEmbedding(dim=dim_head, ring=ring_attn, striped=striped_ring_attn,
                                              theta=rotary_embed_theta, buckets=ring_seq_size // bucket_size)
        self.layers = ModuleList([])
        max_lookback_seq_len = cast_tuple(max_lookback_seq_len, depth)
        assert len(max_lookback_seq_len) == depth
        for layer_max_lookback_seq_len in max_lookback_seq_len:
            self.layers.append(ModuleList([
                RingAttention(dim=dim, causal=causal, dim_head=dim_head, heads=heads,
                              num_grouped_query_heads=num_grouped_query_heads, bucket_size=bucket_size,
                              ring_attn=ring_attn, ring_seq_size=ring_seq_size,
                              max_lookback_seq_len=layer_max_lookback_seq_len, striped_ring_attn=striped_ring_attn,
                              force_regular_attn=force_regular_attn, use_cuda_kernel=self.use_cuda_kernel,
                              auto_shard_seq=False, fp8_attn=fp8_attn, attn_sinks=attn_sinks),
                FeedForward(dim=dim, mult=ff_mult, chunk_size=ff_chunk_size),
            ]))
        self.to_logits = nn.Sequential(RMSNorm(dim), nn.Linear(dim, num_tokens, bias=False))
        self.ignore_index = ignore_index

    def forward(
        self,
        x: Tensor,
        mask: Optional[Tensor] = None,
        labels: Optional[Tensor] = None,
        return_loss: bool = False,
        force_ring_reduce_off: bool = False,
        ring_size: Optional[int] = None,
        document_ids: Optional[Tensor] = None,
    ):
        """``document_ids`` (integer ``[b, n]``, like ``x``): packed-sequence document masking in every layer (see
        :class:`RingAttention`); with ``return_loss`` it is shifted together with the input."""
        seq_len = x.shape[-1]
        auto_shard_seq = not force_ring_reduce_off and self.auto_shard_seq and is_distributed()
        use_ring = self.ring_attn and is_distributed() and not force_ring_reduce_off

        return_loss = return_loss or exists(labels)
        label_mask = None
        if return_loss and not exists(labels):
            # label i is token i + 1: its validity is the mask of token i + 1 (reference ring_attention.py:614 uses
            # mask[:, 1:] as well); the input mask loses its last position together with the input
            x, labels = x[:, :-1], x[:, 1:]
            if exists(document_ids):
                document_ids = document_ids[:, :-1]
            if exists(mask):
                label_mask = mask[:, 1:]
                mask = mask[:, :-1]
        elif exists(labels) and exists(mask):
            label_mask = mask[:, : labels.shape[1]]

        ring_size = default(ring_size, get_world_size())

        if auto_shard_seq:
            x, mask = maybe_pad_seq_and_mask(x, mask, self.ring_seq_size)
            if exists(document_ids):
                document_ids = pad_document_ids(document_ids, self.ring_seq_size)
            if exists(labels):
                labels, label_mask = maybe_pad_seq_and_mask(labels, label_mask, self.ring_seq_size)
                if exists(label_mask):
                    labels = labels.masked_fill(~label_mask, self.ignore_index)
                    label_mask = None
            if self.striped_ring_attn:
                x = stripe(x, self.ring_seq_size)
                if exists(labels):
                    labels = stripe(labels, self.ring_seq_size)
                if exists(mask):
                    mask = stripe(mask, self.ring_seq_size)
                if exists(document_ids):
                    document_ids = stripe(document_ids, self.ring_seq_size)
            (x, mask), batch_sizes, num_sharded_batches = sharded_batch_to_sharded_seq(x, mask, self.ring_seq_size)
            if exists(labels):
                (labels, _), *_ = sharded_batch_to_sharded_seq(labels, None, self.ring_seq_size)
            if exists(document_ids):
                (document_ids, _), *_ = sharded_batch_to_sharded_seq(document_ids, None, self.ring_seq_size)
            ring_size = get_world_size() // num_sharded_batches

        if exists(labels) and exists(label_mask):  # not auto-sharded: padded targets are ignored as well
            labels = labels.masked_fill(~label_mask, self.ignore_index)

        n = x.shape[-1]
        if use_ring:
            rotary_emb = self.rotary_emb(n, ring_size)
        else:
            rotary_emb = self.rotary_emb(torch.arange(n, device=x.device))

        x = self.token_emb(x)
        for attn, ff in self.layers:
            x = attn(x, mask=mask, rotary_emb=rotary_emb, force_ring_reduce_off=force_ring_reduce_off,
                     ring_size=ring_size, document_ids=document_ids) + x
            x = ff(x) + x
        logits = self.to_logits(x)

        if return_loss:
            # local mean over this rank's shard; DDP's gradient averaging reduces across ranks
            # (reference ring_attention.py:664-673)
            return F.cross_entropy(logits.transpose(1, 2), labels, ignore_index=self.ignore_index)

        if not auto_shard_seq:
            return logits
        logits = sharded_seq_to_sharded_batch(logits, batch_sizes, num_sharded_batches)
        if self.striped_ring_attn:
            logits = unstripe(logits, self.ring_seq_size)
        return logits[:, :seq_len]
