#!/usr/bin/env python
"""Decoding against a KV cache that is sharded along the sequence across ranks (tree attention decoding,
reference ``tree_attn_decoding.py``; https://arxiv.org/abs/2408.04093).

Every rank keeps ITS slice of the cache for all layers / heads; a decode step sends the (tiny) query to every rank,
each rank attends to its slice and the partial results are merged — on the GPU in ONE kernel launch per rank and step
(split-KV attention + in-kernel cross-rank merge over NVLink / NVLS), on CPU with two gloo all-reduces.  New
tokens are appended round-robin so that the shards stay balanced.

    # 8 x H100 (80 GB): 32 query / 8 KV heads, 1M cached tokens (131072 per rank), batch 16, bf16 or fp8-e4m3 cache
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29500 \
        examples/decode_tree_attention.py --context 1048576 --batch 16 --heads 32 --kv-heads 8 --steps 64 [--fp8]

    # no GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29500 \
        examples/decode_tree_attention.py --device cpu --context 512 --batch 2 --heads 4 --kv-heads 2 --dim-head 16 --steps 8 --check
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--device", default="cuda", choices=["cuda", "cpu"])
    ap.add_argument("--context", type=int, default=1 << 20, help="cached tokens (whole job) before the first step")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--heads", type=int, default=32)
    ap.add_argument("--kv-heads", type=int, default=8)
    ap.add_argument("--dim-head", type=int, default=128)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--fp8", action="store_true", help="float8_e4m3fn cache with per-(batch, head) scales (CUDA only)")
    ap.add_argument("--check", action="store_true", help="compare every step with dense attention over the gathered cache")
    ap.add_argument("--seed", type=int, default=0)
    return ap.parse_args(argv)


class ShardedKVCache:
    """This rank's slice ``[b, hk, capacity, d]`` of one layer's cache; token t of the stream lives on rank t % world."""

    def __init__(self, batch, kv_heads, dim_head, capacity, dtype, device):
        self.k = torch.empty(batch, kv_heads, capacity, dim_head, dtype=dtype, device=device)
        self.v = torch.empty_like(self.k)
        self.len = 0

    def append(self, k_new: torch.Tensor, v_new: torch.Tensor) -> None:
        n = k_new.shape[2]
        self.k[:, :, self.len:self.len + n] = k_new.to(self.k.dtype)
        self.v[:, :, self.len:self.len + n] = v_new.to(self.v.dtype)
        self.len += n

    def view(self):
        return self.k[:, :, :self.len], self.v[:, :, :self.len]


def run(args) -> float:
    """Inside an initialised process group.  Returns the largest error seen with ``--check`` (0.0 otherwise)."""
    from ring_attention_pytorch_b200 import tree_attn_decode

    rank, world = dist.get_rank(), dist.get_world_size()
    cuda = args.device == "cuda"
    dev = torch.device("cuda", torch.cuda.current_device()) if cuda else torch.device("cpu")
    dt = torch.bfloat16 if cuda else torch.float32
    b, h, hk, d = args.batch, args.heads, args.kv_heads, args.dim_head
    assert not (args.fp8 and not cuda), "the fp8 cache needs the sm_90a kernel"

    gen = torch.Generator().manual_seed(args.seed)  # decode-time stream: the same on every rank (queries, new tokens)

    def stream(n):  # n new tokens for every (batch, kv head): keys, values
        return (torch.randn(b, hk, n, d, generator=gen), torch.randn(b, hk, n, d, generator=gen))

    # prefill: every rank creates ITS slice of the context on its own device (tokens rank, rank + world, ...)
    n_local = len(range(rank, args.context, world))
    per_rank = n_local + args.steps // world + 2
    cache_dtype = torch.float8_e4m3fn if args.fp8 else dt
    cache = ShardedKVCache(b, hk, d, per_rank, cache_dtype, dev)
    dgen = torch.Generator(device=dev).manual_seed(args.seed * 7919 + 1 + rank)
    prefill_k = torch.randn(b, hk, n_local, d, generator=dgen, device=dev)
    prefill_v = torch.randn(b, hk, n_local, d, generator=dgen, device=dev)
    k_scale = v_scale = None
    if args.fp8:  # one scale per (batch, kv head): global maximum of the prefill, e4m3 tops out at 448
        k_scale = prefill_k.abs().amax(dim=(2, 3)).reshape(-1) * (1.25 / 448.0)
        v_scale = prefill_v.abs().amax(dim=(2, 3)).reshape(-1) * (1.25 / 448.0)
        dist.all_reduce(k_scale, dist.ReduceOp.MAX)
        dist.all_reduce(v_scale, dist.ReduceOp.MAX)
        prefill_k = prefill_k / k_scale.view(b, hk, 1, 1)
        prefill_v = prefill_v / v_scale.view(b, hk, 1, 1)
    cache.append(prefill_k, prefill_v)
    del prefill_k, prefill_v

    def quantised(t, scale):  # what the cache stores, as fp32 (for --check)
        t = t.to(cache_dtype).float()
        return t * scale.view(b, hk, 1, 1) if scale is not None else t

    full_k = full_v = None
    if args.check:  # small configs only: gather every rank's slice (order does not matter to attention)
        parts_k, parts_v = [None] * world, [None] * world
        dist.all_gather_object(parts_k, quantised(cache.view()[0], k_scale).cpu())
        dist.all_gather_object(parts_v, quantised(cache.view()[1], v_scale).cpu())
        full_k, full_v = torch.cat(parts_k, 2), torch.cat(parts_v, 2)

    worst, times = 0.0, []
    for step in range(args.steps):
        q = torch.randn(b, h, 1, d, generator=gen).to(dev, dt)
        k_new, v_new = (t.to(dev) for t in stream(1))
        if args.fp8:
            k_new, v_new = k_new / k_scale.view(b, hk, 1, 1), v_new / v_scale.view(b, hk, 1, 1)
        if (args.context + step) % world == rank:  # round-robin owner of the new token
            cache.append(k_new, v_new)
        k, v = cache.view()
        if cuda:
            torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        if args.fp8:
            from ring_attention_pytorch_b200.ops.tree_decode_cuda import tree_decode_cuda

            out = tree_decode_cuda(q, k, v, dim_v=d, k_scale=k_scale, v_scale=v_scale)
        else:
            out = tree_attn_decode(q, k, v, shard_kv_seq=False, dim_v=d)
        if cuda:
            torch.cuda.synchronize(dev)
        times.append(time.perf_counter() - t0)
        if args.check:
            full_k = torch.cat([full_k, quantised(k_new, k_scale).cpu()], 2)
            full_v = torch.cat([full_v, quantised(v_new, v_scale).cpu()], 2)
            qf = q.float().cpu().view(b, h // hk, hk, 1, d)  # query head j reads kv head j % hk
            sim = torch.einsum("bghid,bhjd->bghij", qf, full_k) * d ** -0.5
            ref = torch.einsum("bghij,bhjd->bghid", sim.softmax(-1), full_v).reshape(b, h, 1, d)
            worst = max(worst, float((out.float().cpu() - ref).abs().max()))
    if rank == 0:
        ts = sorted(times[min(3, len(times) - 1):])
        med = ts[len(ts) // 2]
        cached = args.context + args.steps
        kv_bytes = 2 * b * hk * cached * d * (1 if args.fp8 else (2 if cuda else 4))
        print(f"[decode] world {world}, {cached} cached tokens ({cache.len} on rank 0), batch {b}, heads {h}/{hk}: "
              f"median step {med * 1e3:.3f} ms, {b / med:.0f} tokens/s, cache read {kv_bytes / med / 1e9:.0f} GB/s whole job"
              + (f", max |err| vs dense {worst:.2e}" if args.check else ""), flush=True)
    return worst


def main(argv=None) -> None:
    args = parse_args(argv)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    if args.device == "cuda":
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        run(args)
    finally:
        if args.device == "cuda":
            from ring_attention_pytorch_b200.parallel.symm import close_workspaces

            close_workspaces()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
