"""Secondary benchmarks (run under torchrun for N > 1):

    zigzag   GQA Llama-style heads=32 kv_heads=8, total seq 1 048 576, zig-zag schedule, fwd (+bwd with --bwd)
    decode   tree_attn_decode, 8192 keys per rank, batch 256, 32/8 heads, d=128, bf16 and fp8-e4m3 KV
    sweep    ring forward/backward sweep over total sequence lengths, reports K/V bytes over NVLink per second

Every number: CUDA events, barrier + synchronize on both sides, max over ranks, >= 3 warm-up iterations.
Prints one JSON line per measurement on rank 0.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def setup():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    return world, rank, torch.device("cuda", local)


def timed(fn, world, warmup=3, iters=5):
    for _ in range(warmup):
        fn()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda", dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def emit(rank, **kw):
    if rank == 0:
        print(json.dumps(kw), flush=True)


def bench_zigzag(world, rank, dev, total, bwd, iters):
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda

    h, hk, d = 32, 8, 128
    n = total // world
    q = torch.randn(1, n, h, d, device=dev, dtype=torch.bfloat16, requires_grad=bwd)
    k = torch.randn(1, n, hk, d, device=dev, dtype=torch.bfloat16, requires_grad=bwd)
    v = torch.randn(1, n, hk, d, device=dev, dtype=torch.bfloat16, requires_grad=bwd)
    w = torch.randn(1, n, h, d, device=dev, dtype=torch.bfloat16)
    layout = "zigzag" if world > 1 else None

    def step():
        out = ring_flash_attn_cuda(q, k, v, None, True, 1024, world > 1, False, None, world, False, 50.0, layout)
        if bwd:
            out.backward(w)
            q.grad = k.grad = v.grad = None

    ms = timed(step, world, warmup=3, iters=iters)
    flops = 4.0 * h * float(total) ** 2 * d * 0.5 * (3.5 if bwd else 1.0)
    kv_bytes = (world - 1) * 2 * n * hk * d * 2  # K/V bytes each rank pulls over NVLink in the forward
    emit(rank, bench="zigzag_gqa", n_gpus=world, seq_len=total, heads=h, kv_heads=hk, bwd=bwd, ms=ms,
         tflops=flops / ms / 1e9, tokens_per_s=total / (ms * 1e-3), kv_pull_gb_per_rank=kv_bytes / 1e9)


def bench_decode(world, rank, dev, n_per_rank, batch, iters):
    from ring_attention_pytorch_b200.ops.tree_decode_cuda import tree_decode_cuda

    h, hk, d = 32, 8, 128
    q = torch.randn(batch, h, 1, d, device=dev, dtype=torch.bfloat16)
    k = torch.randn(batch, hk, n_per_rank, d, device=dev, dtype=torch.bfloat16)
    v = torch.randn(batch, hk, n_per_rank, d, device=dev, dtype=torch.bfloat16)
    for name, kk, vv, ks, vs in (
        ("bf16", k, v, None, None),
        ("fp8_e4m3", k.to(torch.float8_e4m3fn), v.to(torch.float8_e4m3fn),
         torch.ones(batch * hk, device=dev), torch.ones(batch * hk, device=dev)),
    ):
        ms = timed(lambda: tree_decode_cuda(q, kk, vv, dim_v=d, k_scale=ks, v_scale=vs), world, warmup=5, iters=iters)
        kv_bytes = 2 * kk.numel() * kk.element_size()
        from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc

        emit(rank, bench="tree_decode", kv_dtype=name, n_gpus=world, keys_per_rank=n_per_rank, batch=batch, ms=ms,
             local_kv_gb_per_s=kv_bytes / ms / 1e6, hbm_frac_of_datasheet_3350=kv_bytes / ms / 1e6 / 3350.0,
             tokens_per_s=batch / (ms * 1e-3), launches_per_step=1, merge="nvls multimem" if tdc.uses_nvls(q) else "nvlink peer loads",
             nvls_unavailable_because=tdc._alloc_symmetric.last_error)


def bench_sweep(world, rank, dev, iters, sizes=(4096, 16384, 65536, 262144, 1048576)):
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda

    h, d = 32, 128
    for total in sizes:
        n = total // world
        if n < 128:
            continue
        q = torch.randn(1, n, h, d, device=dev, dtype=torch.bfloat16, requires_grad=True)
        k = torch.randn(1, n, h, d, device=dev, dtype=torch.bfloat16, requires_grad=True)
        v = torch.randn(1, n, h, d, device=dev, dtype=torch.bfloat16, requires_grad=True)
        w = torch.randn(1, n, h, d, device=dev, dtype=torch.bfloat16)

        def fwd():
            return ring_flash_attn_cuda(q, k, v, None, True, 1024, world > 1, world > 1, None, world)

        def fwdbwd():
            fwd().backward(w)
            q.grad = k.grad = v.grad = None

        it = max(2, min(iters, 20 if total <= 65536 else 3))
        ms_f = timed(lambda: fwd(), world, warmup=3, iters=it)
        ms_fb = timed(fwdbwd, world, warmup=3, iters=it)
        kv_bytes = (world - 1) * 2 * n * h * d * 2
        f = 4.0 * h * float(total) ** 2 * d * 0.5
        emit(rank, bench="ring_sweep", n_gpus=world, seq_len=total, ms_fwd=ms_f, ms_fwd_bwd=ms_fb,
             fwd_tflops=f / ms_f / 1e9, fwd_bwd_tflops=3.5 * f / ms_fb / 1e9,
             kv_gb_per_s_per_rank_fwd=kv_bytes / ms_f / 1e6)
        del q, k, v, w
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", default="zigzag,decode")
    ap.add_argument("--total-seq", type=int, default=1048576)
    ap.add_argument("--bwd", action="store_true")
    ap.add_argument("--keys-per-rank", type=int, default=8192)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--sweep-sizes", default="4096,16384,65536,262144,1048576")
    args = ap.parse_args()
    world, rank, dev = setup()
    for which in args.which.split(","):
        if which == "zigzag":
            bench_zigzag(world, rank, dev, args.total_seq, args.bwd, args.iters)
        elif which == "decode":
            bench_decode(world, rank, dev, args.keys_per_rank, args.batch, max(args.iters, 10))
        elif which == "sweep":
            bench_sweep(world, rank, dev, args.iters, tuple(int(x) for x in args.sweep_sizes.split(",")))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
