"""Ring attention with the same capabilities and public API as lucidrains/ring-attention-pytorch
(reference ``ring_attention_pytorch/__init__.py:1-21``), rebuilt around hand-written sm_90a kernels.

Public exports mirror the reference and add the pieces it only exposes through sub-modules.
"""
from ring_attention_pytorch_b200.models.ring_attention import (
    FeedForward,
    RingAttention,
    RingRotaryEmbedding,
    RingTransformer,
    RMSNorm,
    apply_rotary_pos_emb,
)
from ring_attention_pytorch_b200.ops.flash_attn import flash_attn_backward, flash_attn_forward
from ring_attention_pytorch_b200.ops.oracle import attention_with_positions, default_attention
from ring_attention_pytorch_b200.ops.paged_kv import gather_paged_kv, write_paged_kv
from ring_attention_pytorch_b200.ops.ring_flash_naive import ring_flash_attn, ring_flash_attn_
from ring_attention_pytorch_b200.ops.tree_decode import tree_attn_decode
from ring_attention_pytorch_b200.ops.zig_zag import zig_zag_attn, zig_zag_pad_seq, zig_zag_shard


def __getattr__(name):
    # the CUDA op imports the extension lazily so that CPU-only users never touch it
    if name in ("ring_flash_attn_cuda", "ring_flash_attn_cuda_"):
        from ring_attention_pytorch_b200.ops import ring_cuda

        return getattr(ring_cuda, name)
    if name in ("ring_flash_attn_fp8", "quantize_fp8"):
        from ring_attention_pytorch_b200.ops import ring_fp8

        return getattr(ring_fp8, name)
    raise AttributeError(name)


__all__ = [
    "RingAttention",
    "RingTransformer",
    "RingRotaryEmbedding",
    "RMSNorm",
    "FeedForward",
    "apply_rotary_pos_emb",
    "default_attention",
    "attention_with_positions",
    "ring_flash_attn",
    "ring_flash_attn_",
    "ring_flash_attn_cuda",
    "ring_flash_attn_cuda_",
    "ring_flash_attn_fp8",
    "quantize_fp8",
    "tree_attn_decode",
    "gather_paged_kv",
    "write_paged_kv",
    "flash_attn_forward",
    "flash_attn_backward",
    "zig_zag_attn",
    "zig_zag_pad_seq",
    "zig_zag_shard",
]

__version__ = "0.1.0"
