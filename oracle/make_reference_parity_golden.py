"""Regenerate ``tests/golden/reference_parity.pt``: the outputs of the original ``ring_attention_pytorch`` package on the
inputs that ``tests/test_reference_parity.py`` feeds this package, so that the parity tests run without it.

    python oracle/make_reference_parity_golden.py /path/to/ring-attention-pytorch

Every input is rebuilt from the same seeds inside the tests; only the reference's results (and the reference model
weights that must load into this package's modules) are stored.  CPU only.
"""
from __future__ import annotations

import inspect
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "reference_parity.pt")


def _zigzag_worker(rank, world, tmp):
    import ring_attention_pytorch.zig_zag_attention as theirs

    torch.manual_seed(0)
    x = torch.randn(2, 29, 16)
    pb, inv_b = theirs.zig_zag_pad_seq(x)
    (sb, qb, kb), gather_b = theirs.zig_zag_shard(pb)
    h, d = 4, 8
    q = torch.randn(2, h, sb.shape[1], d)
    k = torch.randn(2, 2, sb.shape[1], d)
    v = torch.randn(2, 2, sb.shape[1], d)
    mask = qb[:, None] >= kb[None, :]
    want = theirs.zig_zag_attn(q, k, v, attn_mask=mask)
    torch.save({"padded": pb, "shard": sb, "q_idx": qb, "k_idx": kb, "roundtrip": inv_b(gather_b(sb)), "attn": want},
               os.path.join(tmp, f"zigzag_{rank}.pt"))


def _ring_transformer_worker(rank, world, striped, tmp):
    import ring_attention_pytorch as theirs

    torch.manual_seed(0)
    kw = dict(num_tokens=64, dim=32, depth=2, causal=True, dim_head=8, heads=4, num_grouped_query_heads=2, bucket_size=4,
              ring_attn=True, striped_ring_attn=striped, ring_seq_size=8, use_cuda_kernel=False)
    b = theirs.RingTransformer(**kw)
    torch.manual_seed(1)
    x = torch.randint(0, 64, (2, 15))
    with torch.no_grad():
        lb = b(x)
    torch.save({"state_dict": b.state_dict(), "logits": lb}, os.path.join(tmp, f"ringtf_{int(striped)}_{rank}.pt"))


def _tree_worker(rank, world, seq_len, tmp):
    import ring_attention_pytorch as theirs

    torch.manual_seed(0)
    q, k, v = torch.randn(2, 4, 1, 8), torch.randn(2, 4, seq_len, 8), torch.randn(2, 4, seq_len, 8)
    want = theirs.tree_attn_decode(q, k, v, use_triton=False)
    torch.save(want, os.path.join(tmp, f"tree_{seq_len}_{rank}.pt"))


def main(ref_dir: str) -> None:
    sys.path.insert(0, ref_dir)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ring_attention_pytorch as ref
    import ring_attention_pytorch.distributed as r_dist
    import ring_attention_pytorch.ring as r_ring
    import ring_attention_pytorch.zig_zag_attention as r_zz
    from dist_utils import run_distributed

    g = {}
    # RingTransformer: weights, logits, loss and gradients
    torch.manual_seed(0)
    kw = dict(num_tokens=64, dim=32, depth=2, causal=True, dim_head=8, heads=4, num_grouped_query_heads=2,
              bucket_size=4, ring_attn=False, use_cuda_kernel=False)
    theirs = ref.RingTransformer(**kw)
    x = torch.randint(0, 64, (2, 17))
    lb = theirs(x, return_loss=True)
    lb.backward()
    g["transformer"] = {"state_dict": theirs.state_dict(), "x": x, "logits": theirs(x).detach(), "loss": lb.detach(),
                        "grads": {n: p.grad.clone() for n, p in theirs.named_parameters()}}

    # RingAttention module with rotary embeddings
    g["attention"] = {}
    for causal in (False, True):
        torch.manual_seed(1)
        kw = dict(dim=32, dim_head=8, heads=4, num_grouped_query_heads=2, causal=causal, bucket_size=4, ring_attn=False,
                  rotary_embed=True, use_cuda_kernel=False)
        theirs = ref.RingAttention(**kw)
        x = torch.randn(2, 19, 32)
        mask = None if causal else (torch.rand(2, 19) > 0.25)
        g["attention"][causal] = {"state_dict": theirs.state_dict(), "out": theirs(x, mask).detach()}

    # functional ops
    torch.manual_seed(2)
    q = torch.randn(2, 21, 4, 8, requires_grad=True)
    k = torch.randn(2, 21, 2, 8, requires_grad=True)
    v = torch.randn(2, 21, 2, 8, requires_grad=True)
    mask = torch.rand(2, 21) > 0.3
    fn = {}
    for causal in (False, True):
        m = None if causal else mask
        fb = ref.ring_flash_attn(q, k, v, m, causal, 4)
        gr = torch.randn_like(fb)
        fn[causal] = {"default": ref.default_attention(q, k, v, m, causal).detach(), "flash": fb.detach(), "g": gr,
                      "grads": [t.detach() for t in torch.autograd.grad(fb, (q, k, v), gr)]}
    pb = ref.RingRotaryEmbedding(8)(21)
    fn["rotary_pos"] = pb.detach()
    fn["rotary_q"] = ref.ring_attention.apply_rotary_pos_emb(pb, q).detach()
    import torch.distributed as dist

    with tempfile.TemporaryDirectory() as tmp:
        import socket

        with socket.socket() as sock:
            sock.bind(("127.0.0.1", 0))
            port = sock.getsockname()[1]
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
        try:
            dq, dk, dv = torch.randn(2, 4, 1, 8), torch.randn(2, 4, 33, 8), torch.randn(2, 4, 33, 8)
            fn["decode"] = {"q": dq, "k": dk, "v": dv, "out": ref.tree_attn_decode(dq, dk, dv, use_triton=False)}
        finally:
            dist.destroy_process_group()
        g["functional"] = fn

        run_distributed(_zigzag_worker, 2, tmp)
        g["zigzag"] = [torch.load(os.path.join(tmp, f"zigzag_{r}.pt")) for r in range(2)]
        g["ring_transformer"] = {}
        for striped in (False, True):
            run_distributed(_ring_transformer_worker, 2, striped, tmp)
            g["ring_transformer"][striped] = [torch.load(os.path.join(tmp, f"ringtf_{int(striped)}_{r}.pt"))
                                              for r in range(2)]
        g["tree"] = {}
        for seq_len in (2, 31):
            run_distributed(_tree_worker, 3, seq_len, tmp)
            g["tree"][seq_len] = [torch.load(os.path.join(tmp, f"tree_{seq_len}_{r}.pt")) for r in range(3)]

    # public API: parameter names of every callable the reference exports
    def params(f):
        target = f.__init__ if inspect.isclass(f) else f
        try:
            sig = inspect.signature(target)
        except (TypeError, ValueError):
            return None
        return [p for p in sig.parameters if p not in ("self", "args", "kwargs")]

    api = {}
    for key, mod, names in [("", ref, ["RingAttention", "RingTransformer", "RingRotaryEmbedding", "apply_rotary_pos_emb",
                                        "default_attention", "ring_flash_attn", "ring_flash_attn_cuda",
                                        "tree_attn_decode"]),
                            ("distributed", r_dist, ["all_gather_variable_dim", "split_by_rank", "get_rank",
                                                     "get_world_size", "is_distributed", "pad_dim_to"]),
                            ("ring", r_ring, ["ring_pass", "all_ring_pass", "null_ring_pass", "one_ring_pass",
                                              "get_rank", "get_world_size"]),
                            ("zig_zag", r_zz, ["zig_zag_pad_seq", "zig_zag_shard", "zig_zag_attn"])]:
        api[key] = {n: params(getattr(mod, n)) for n in names if hasattr(mod, n)}
    g["api"] = api

    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    torch.save(g, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ.get("RING_ATTENTION_REFERENCE", "."))
