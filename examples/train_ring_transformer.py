#!/usr/bin/env python
"""Long-context language-model training: sequence parallelism (ring attention) x data parallelism.

Every rank feeds ITS OWN batch of full-length sequences; the model all-gathers the batches, splits every sequence over
the ring (``auto_shard_seq``; striped for causal load balance) and returns the rank-local mean loss — the calling
convention of the reference (``ring_attention.py:560-673``).  Parameter gradients are averaged over all ranks with one
coalesced all-reduce after the backward (what DDP does, without its per-bucket hooks).

    # one 8 x H100 box: one ring of 8, 65536 tokens per sequence (8192 per rank)
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29500 \
        examples/train_ring_transformer.py --seq-len 65536 --dim 1024 --depth 8 --heads 8 --dim-head 128 --steps 50

    # the same box as 2 data-parallel replicas x rings of 4 (ring sets, reference ring.py:35-47)
    ... examples/train_ring_transformer.py --seq-len 32768 --batches-per-ring 2

    # no GPU: portable path on gloo
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29500 \
        examples/train_ring_transformer.py --device cpu --seq-len 64 --dim 32 --depth 2 --heads 4 --dim-head 8 --steps 5

``--ckpt PATH`` writes model / optimizer / step after every ``--ckpt-every`` steps (rank 0) and resumes from it when it
exists.  Data is synthetic: a noisy copy task (second half of every sequence repeats the first half), which needs
attention across half the sequence, i.e. across ring ranks, to be learned; ``--task count`` is a local task that is
learned within tens of steps (used by the CPU test).
"""
from __future__ import annotations

import argparse
import os
import sys
import time
from math import ceil

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--device", default="cuda", choices=["cuda", "cpu"])
    ap.add_argument("--seq-len", type=int, default=65536, help="tokens per sequence (sharded over the ring)")
    ap.add_argument("--batch", type=int, default=1, help="sequences per rank and step")
    ap.add_argument("--batches-per-ring", type=int, default=1,
                    help="data-parallel replicas: ring size = world / batches-per-ring")
    ap.add_argument("--vocab", type=int, default=256)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--depth", type=int, default=8)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--kv-heads", type=int, default=None, help="grouped-query attention: number of K/V heads")
    ap.add_argument("--dim-head", type=int, default=128)
    ap.add_argument("--lookback", type=int, default=None, help="causal look-back window in tokens (all layers)")
    ap.add_argument("--no-striped", action="store_true", help="plain contiguous shards instead of striped")
    ap.add_argument("--ff-chunk", type=int, default=None, help="blockwise feed-forward chunk (tokens)")
    ap.add_argument("--task", default="copy", choices=["copy", "count"], help="synthetic data (see synthetic_batch)")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--lr", type=float, default=3e-4)
    ap.add_argument("--memory", default="auto", choices=["auto", "ring", "gather"], help="ring_cuda.CONFIG['memory']")
    ap.add_argument("--ckpt", default=None)
    ap.add_argument("--ckpt-every", type=int, default=25)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--log-every", type=int, default=1)
    return ap.parse_args(argv)


def synthetic_batch(batch: int, seq_len: int, vocab: int, gen: torch.Generator, device, task: str = "copy") -> torch.Tensor:
    """``copy``: tokens[half:] = tokens[:half] with 2 % noise (needs attention across half the sequence).
    ``count``: tokens[i + 1] = tokens[i] + 1 (mod vocab) with 5 % noise (local; learned within tens of steps)."""
    if task == "count":
        start = torch.randint(0, vocab, (batch, 1), generator=gen)
        jumps = (torch.rand(batch, seq_len, generator=gen) < 0.05) * torch.randint(0, vocab, (batch, seq_len), generator=gen)
        tokens = (start + torch.arange(seq_len)[None] + jumps.cumsum(1)) % vocab
        return tokens.to(device, non_blocking=True)
    half = seq_len // 2
    first = torch.randint(0, vocab, (batch, half), generator=gen)
    second = first.clone()
    noise = torch.rand(batch, half, generator=gen) < 0.02
    second[noise] = torch.randint(0, vocab, (int(noise.sum()),), generator=gen)
    tokens = torch.cat([first, second], 1)
    if tokens.shape[1] < seq_len:  # odd length
        tokens = torch.cat([tokens, tokens[:, :1]], 1)
    return tokens.to(device, non_blocking=True)


def average_gradients(params, world: int) -> None:
    """One coalesced all-reduce over every parameter gradient (ranks that did not touch a parameter contribute zeros)."""
    grads = []
    for p in params:
        if p.grad is None:
            p.grad = torch.zeros_like(p)
        grads.append(p.grad)
    flat = torch.cat([g.reshape(-1).float() for g in grads])
    dist.all_reduce(flat)
    flat /= world
    off = 0
    for g in grads:
        n = g.numel()
        g.copy_(flat[off:off + n].view_as(g))
        off += n


def train(args) -> float:
    """Runs inside an initialised process group; returns the last (rank-averaged) loss."""
    from ring_attention_pytorch_b200 import RingTransformer

    rank, world = dist.get_rank(), dist.get_world_size()
    cuda = args.device == "cuda"
    dev = torch.device("cuda", torch.cuda.current_device()) if cuda else torch.device("cpu")
    assert world % args.batches_per_ring == 0, "world size must be a multiple of --batches-per-ring"
    ring_size = world // args.batches_per_ring
    # the model sees seq_len - 1 inputs (labels are the inputs shifted by one); every rank of a ring gets one chunk
    ring_seq_size = ceil((args.seq_len - 1) / ring_size)
    if cuda:
        from ring_attention_pytorch_b200.ops import ring_cuda

        ring_cuda.CONFIG["memory"] = args.memory

    torch.manual_seed(args.seed)  # identical initial weights on every rank
    heads = args.heads
    groups = 1 if args.kv_heads is None else heads // args.kv_heads
    model = RingTransformer(
        num_tokens=args.vocab, dim=args.dim, depth=args.depth, causal=True, dim_head=args.dim_head, heads=heads,
        num_grouped_query_heads=groups, bucket_size=ring_seq_size, ring_attn=world > 1,
        striped_ring_attn=world > 1 and not args.no_striped, ring_seq_size=ring_seq_size,
        max_lookback_seq_len=args.lookback, ff_chunk_size=args.ff_chunk, use_cuda_kernel=cuda,
    ).to(dev)
    opt = torch.optim.AdamW(model.parameters(), lr=args.lr, betas=(0.9, 0.95), weight_decay=0.0)

    start = 0
    if args.ckpt and os.path.exists(args.ckpt):
        state = torch.load(args.ckpt, map_location=dev)
        model.load_state_dict(state["model"])
        opt.load_state_dict(state["opt"])
        start = int(state["step"])
        if rank == 0:
            print(f"[train] resumed from {args.ckpt} at step {start}", flush=True)

    n_params = sum(p.numel() for p in model.parameters())
    if rank == 0:
        print(f"[train] world {world} = {args.batches_per_ring} replica(s) x ring of {ring_size}; seq {args.seq_len} "
              f"({ring_seq_size} tokens per rank), {n_params / 1e6:.1f} M parameters, "
              f"device {dev}", flush=True)

    loss_avg = float("nan")
    for step in range(start, args.steps):
        gen = torch.Generator().manual_seed(args.seed * 1_000_003 + step * world + rank)  # resumable data stream
        tokens = synthetic_batch(args.batch, args.seq_len, args.vocab, gen, dev, args.task)
        if cuda:
            torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=cuda):
            loss = model(tokens, return_loss=True)
        loss.backward()
        average_gradients(list(model.parameters()), world)
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0)
        opt.step()
        opt.zero_grad(set_to_none=True)
        stat = loss.detach().float().reshape(1).clone()
        dist.all_reduce(stat)
        loss_avg = float(stat.item()) / world
        if cuda:
            torch.cuda.synchronize(dev)
        dt = time.perf_counter() - t0
        if rank == 0 and (step % args.log_every == 0 or step + 1 == args.steps):
            tok_s = world * args.batch * args.seq_len / dt
            print(f"[train] step {step + 1:5d}  loss {loss_avg:.4f}  {dt * 1e3:9.1f} ms  {tok_s:12.0f} tokens/s",
                  flush=True)
        if args.ckpt and ((step + 1) % args.ckpt_every == 0 or step + 1 == args.steps):
            if rank == 0:
                tmp = args.ckpt + ".tmp"
                torch.save({"model": model.state_dict(), "opt": opt.state_dict(), "step": step + 1}, tmp)
                os.replace(tmp, args.ckpt)  # atomic: a killed run never leaves a torn checkpoint
            dist.barrier()
    return loss_avg


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
        train(args)
    finally:
        if args.device == "cuda":
            from ring_attention_pytorch_b200.parallel.symm import close_workspaces

            close_workspaces()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
