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

    # ragged batch (seeded prompt lengths in [0, context]) and a look-back window of 4096 tokens
    ... examples/decode_tree_attention.py --context 1048576 --batch 16 --ragged --window 4096

    # speculative verification: every step appends 4 draft tokens and checks them in one decode call
    ... examples/decode_tree_attention.py --context 1048576 --batch 16 --draft 4

    # paged KV cache: 16-token pages from a shuffled free list, pages behind the window go back to the list
    ... examples/decode_tree_attention.py --context 1048576 --batch 16 --ragged --window 4096 --page-size 16
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
    ap.add_argument("--ragged", action="store_true", help="per-sequence prompt lengths drawn from the seed in [0, context]")
    ap.add_argument("--window", type=int, default=None, help="look-back window: the query sees positions >= pos - W")
    ap.add_argument("--draft", type=int, default=1,
                    help="query tokens per step: append M tokens and decode them in one call (causal among themselves)")
    ap.add_argument("--page-size", type=int, default=None,
                    help="paged KV cache: each rank keeps a pool of pages of P tokens and a block table per sequence")
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
    if args.ragged or args.window is not None or args.draft > 1 or args.page_size:
        return run_ragged(args)
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


def run_ragged(args) -> float:
    """``--ragged`` / ``--window`` / ``--draft``: every sequence has its own length, the decode passes the whole capacity
    buffers with per-sequence ``cache_seqlens``, query positions and ``kv_pos = (rank, world)`` (token t of a sequence
    lives on rank t % world at local slot t // world).  Slots past a sequence's length hold NaN (0x7F in e4m3): they
    must not matter.  Each step appends ``--draft`` tokens and decodes all of them in one call.

    ``--page-size P``: each rank keeps K / V in a pool of P-token pages and a block table per sequence.  Pages come from
    a seeded, shuffled free list as a sequence grows; with a window, pages wholly behind every future query's window go
    back to the list (and may be handed to another sequence) while the table still names them."""
    from ring_attention_pytorch_b200 import tree_attn_decode
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.ops.tree_decode_cuda import tree_decode_cuda

    rank, world = dist.get_rank(), dist.get_world_size()
    cuda = args.device == "cuda"
    dev = torch.device("cuda", torch.cuda.current_device()) if cuda else torch.device("cpu")
    dt = torch.bfloat16 if cuda else torch.float32
    b, h, hk, d, M = args.batch, args.heads, args.kv_heads, args.dim_head, args.draft
    assert not (args.fp8 and not cuda), "the fp8 cache needs the sm_90a kernel"
    gen = torch.Generator().manual_seed(args.seed)  # the same on every rank: lengths, queries, new tokens
    lens = torch.full((b,), args.context, dtype=torch.int64)
    if args.ragged:
        lens = torch.randint(0, args.context + 1, (b,), generator=gen)
        lens[0] = lens[0] % world  # shorter than the world: some ranks hold none of it
    cache_dtype = torch.float8_e4m3fn if args.fp8 else dt

    def local_len(n):  # tokens rank, rank + world, ... below n
        return (n - rank + world - 1).clamp(min=0) // world

    cap = (args.context + args.steps * M + world - 1) // world + 1
    n0 = (args.context + world - 1) // world
    dgen = torch.Generator(device=dev).manual_seed(args.seed * 7919 + 1 + rank)
    pk = torch.randn(b, hk, n0, d, generator=dgen, device=dev)
    pv = torch.randn(b, hk, n0, d, generator=dgen, device=dev)
    k_scale = v_scale = None
    if args.fp8:
        k_scale = pk.abs().amax(dim=(2, 3)).reshape(-1) * (1.25 / 448.0)
        v_scale = pv.abs().amax(dim=(2, 3)).reshape(-1) * (1.25 / 448.0)
        dist.all_reduce(k_scale, dist.ReduceOp.MAX)
        dist.all_reduce(v_scale, dist.ReduceOp.MAX)
        pk, pv = pk / k_scale.view(b, hk, 1, 1), pv / v_scale.view(b, hk, 1, 1)
    held = local_len(lens)
    P = args.page_size
    if P:
        from ring_attention_pytorch_b200 import write_paged_kv

        max_pages = (cap + P - 1) // P
        # a pool with room for every sequence's pages; ids handed out in a seeded random order
        kc = torch.empty(b * max_pages + 1, hk, P, d, dtype=cache_dtype, device=dev)
        free = torch.randperm(kc.shape[0], generator=torch.Generator().manual_seed(args.seed + 101 + rank)).tolist()
        table = torch.zeros(b, max_pages, dtype=torch.int32)
        owned = [0] * b  # pages [0, owned[i]) of sequence i are in the table
        released = [0] * b  # pages [0, released[i]) went back to the free list

        def grow(i, n):  # sequence i holds n local keys: give it the pages they need
            while owned[i] * P < n:
                table[i, owned[i]] = free.pop()
                owned[i] += 1
    else:
        kc = torch.empty(b, hk, cap, d, dtype=cache_dtype, device=dev)
    vc = torch.empty_like(kc)
    for t in (kc, vc):
        (t.view(torch.uint8).fill_(0x7F) if args.fp8 else t.fill_(float("nan")))
    for i in range(b):
        if P:
            grow(i, int(held[i]))
            tb = table[i:i + 1].to(dev)
            write_paged_kv(kc, vc, tb, torch.zeros(1, dtype=torch.int64, device=dev), pk[i:i + 1, :, :held[i]],
                           pv[i:i + 1, :, :held[i]])
        else:
            kc[i, :, :held[i]] = pk[i, :, :held[i]].to(cache_dtype)
            vc[i, :, :held[i]] = pv[i, :, :held[i]].to(cache_dtype)
    del pk, pv

    def quantised(t, scale):  # what the cache stores, as fp32 (for --check)
        t = t.to(cache_dtype).float()
        return t * scale.view(b, hk, 1, 1) if scale is not None else t

    full_k = full_v = None
    if args.check:  # global [b, hk, max length, d] in position order, from every rank's slots
        total = int(lens.max()) + args.steps * M
        full_k, full_v = torch.zeros(b, hk, total, d), torch.zeros(b, hk, total, d)
        parts = [None] * world
        if P:
            from ring_attention_pytorch_b200 import gather_paged_kv

            kg, vg = gather_paged_kv(kc, table.to(dev)), gather_paged_kv(vc, table.to(dev))
        else:
            kg, vg = kc, vc
        dist.all_gather_object(parts, (quantised(kg.float(), k_scale).cpu(), quantised(vg.float(), v_scale).cpu()))
        for r, (pk_r, pv_r) in enumerate(parts):
            for i in range(b):
                m = len(range(r, int(lens[i]), world))
                full_k[i, :, r:r + world * m:world], full_v[i, :, r:r + world * m:world] = pk_r[i, :, :m], pv_r[i, :, :m]

    worst, times, seen = 0.0, [], 0
    for _ in range(args.steps):
        q = torch.randn(b, h, M, d, generator=gen).to(dev, dt)
        k_new, v_new = torch.randn(b, hk, M, d, generator=gen), torch.randn(b, hk, M, d, generator=gen)
        if args.fp8:
            k_new, v_new = k_new / k_scale.view(b, hk, 1, 1).cpu(), v_new / v_scale.view(b, hk, 1, 1).cpu()
        for u in range(M):  # new token u of sequence i sits at lens[i] + u and goes to rank (lens[i] + u) % world
            pos = lens + u
            mine = (pos % world == rank).nonzero().flatten()
            slot = local_len(pos)[mine]
            if P:
                for i, s_ in zip(mine.tolist(), slot.tolist()):
                    grow(i, s_ + 1)
                write_paged_kv(kc, vc, table[mine].to(dev), slot.to(dev), k_new[mine, :, u:u + 1].to(dev),
                               v_new[mine, :, u:u + 1].to(dev))
                continue
            kc[mine.to(dev), :, slot.to(dev)] = k_new[mine, :, u].to(dev, cache_dtype)
            vc[mine.to(dev), :, slot.to(dev)] = v_new[mine, :, u].to(dev, cache_dtype)
        q_pos = lens.clone()  # the first new token's position
        lens += M
        held = local_len(lens)
        kw = dict(cache_seqlens=held.to(dev, torch.int32), q_pos=q_pos.to(dev, torch.int32), window=args.window,
                  kv_pos=(rank, world))
        if P:
            kw["block_table"] = table.to(dev)
        seen += int(sum(min(int(n), (args.window or int(n)) + M) for n in lens))
        if cuda:
            torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        if args.fp8:
            out = tree_decode_cuda(q, kc, vc, dim_v=d, k_scale=k_scale, v_scale=v_scale, **kw)
        else:
            out = tree_attn_decode(q, kc, vc, shard_kv_seq=False, dim_v=d, **kw)
        if cuda:
            torch.cuda.synchronize(dev)
        times.append(time.perf_counter() - t0)
        if P and args.window is not None:
            # every later query sits at >= lens: local keys before the first one its window reaches are dead, and so
            # is every page that holds only such keys (the table keeps naming it; the kernels never read it)
            first = local_len((lens - args.window).clamp(min=0))
            for i in range(b):
                while (released[i] + 1) * P <= int(first[i]) and released[i] < owned[i]:
                    free.append(int(table[i, released[i]]))  # handed out next, to any sequence
                    released[i] += 1
        if args.check:
            kq = quantised(k_new, k_scale.cpu() if k_scale is not None else None)
            vq = quantised(v_new, v_scale.cpu() if v_scale is not None else None)
            for i in range(b):
                p0 = int(q_pos[i])
                full_k[i, :, p0:p0 + M], full_v[i, :, p0:p0 + M] = kq[i], vq[i]
                n = int(lens[i])
                ref = attention_with_positions(q[i:i + 1].float().cpu().transpose(1, 2),
                                               full_k[i:i + 1, :, :n].transpose(1, 2), full_v[i:i + 1, :, :n].transpose(1, 2),
                                               q_pos=p0 + torch.arange(M), k_pos=torch.arange(n), causal=True,
                                               window=args.window)
                worst = max(worst, float((out[i:i + 1].float().cpu() - ref.transpose(1, 2)).abs().max()))
    if rank == 0:
        ts = sorted(times[min(3, len(times) - 1):])
        med = ts[len(ts) // 2]
        kv_bytes = 2 * hk * d * (seen / args.steps) * (1 if args.fp8 else (2 if cuda else 4))
        print(f"[decode] world {world}, ragged {args.ragged}, window {args.window}, draft {M}, lengths {int(lens.min())}.."
              f"{int(lens.max())}, batch {b}, heads {h}/{hk}: median step {med * 1e3:.3f} ms, {b * M / med:.0f} tokens/s, "
              f"visible cache read {kv_bytes / med / 1e9:.0f} GB/s whole job"
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
