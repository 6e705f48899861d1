#!/usr/bin/env python
"""Ragged and windowed tree decode on one GPU: the cases of the README's Status table, each group timed with its cases
alternating, the median of ``--reps`` launches per case after warm-up (CUDA events around each call).

  (a) README decode shape (b 256, 32 / 8 heads, 8192 keys, d 128, bf16): the plain call against cache_seqlens = n
  (b) a ragged batch of the same heads, capacity 16384, seeded lengths uniform in [1, 16384]: visible K/V bytes per
      second, against those of (a)
  (c) windowed decode (b 16, 32 / 8 heads, 131072 keys, window 4096), bf16 and fp8: against the same call without a
      window and against a dense 4097-key decode

    python tools/bench_decode_ragged.py [--reps 9] [--warmup 3]

Prints the card's name and power limit first, then one line per case.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"{torch.cuda.get_device_name()}, power limit unknown ({type(e).__name__})"
    return q


def alternate(cases: dict, reps: int, warmup: int) -> dict:
    """{name: callable} -> {name: median ms}, the cases interleaved launch by launch."""
    for _ in range(warmup):
        for fn in cases.values():
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in cases}
    for _ in range(reps):
        for name, fn in cases.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    return {k: statistics.median(v) for k, v in times.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    from ring_attention_pytorch_b200.ops.tree_decode_cuda import tree_decode_cuda

    print(f"[card] {card()}", flush=True)
    dev = torch.device("cuda")
    gen = torch.Generator(dev).manual_seed(0)
    h, hk, d = 32, 8, 128
    rows = []

    def report(case, ms, **extra):
        rows.append(dict(case=case, ms=round(ms, 4), **extra))
        print(json.dumps(rows[-1]), flush=True)

    # (a) and (b)
    b, n = 256, 8192
    q = torch.randn(b, h, 1, d, device=dev, dtype=torch.bfloat16, generator=gen)
    k = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
    v = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
    full = torch.full((b,), n, dtype=torch.int32, device=dev)
    med = alternate({"plain": lambda: tree_decode_cuda(q, k, v, dim_v=d),
                     "seqlens_n": lambda: tree_decode_cuda(q, k, v, dim_v=d, cache_seqlens=full)}, args.reps, args.warmup)
    bytes_a = 2 * b * hk * n * d * 2
    report("a_plain", med["plain"], gbps=round(bytes_a / med["plain"] / 1e6, 1))
    report("a_seqlens_n", med["seqlens_n"], gbps=round(bytes_a / med["seqlens_n"] / 1e6, 1),
           ratio_to_plain=round(med["seqlens_n"] / med["plain"], 4))
    gbps_a = bytes_a / med["plain"] / 1e6
    del k, v
    cap = 16384
    k = torch.randn(b, hk, cap, d, device=dev, dtype=torch.bfloat16, generator=gen)
    v = torch.randn(b, hk, cap, d, device=dev, dtype=torch.bfloat16, generator=gen)
    lens = torch.randint(1, cap + 1, (b,), generator=torch.Generator().manual_seed(1)).to(dev, torch.int32)
    med = alternate({"ragged": lambda: tree_decode_cuda(q, k, v, dim_v=d, cache_seqlens=lens)}, args.reps, args.warmup)
    bytes_b = 2 * hk * d * 2 * int(lens.sum())
    gbps_b = bytes_b / med["ragged"] / 1e6
    report("b_ragged", med["ragged"], visible_gbps=round(gbps_b, 1), ratio_to_a=round(gbps_b / gbps_a, 3))
    del q, k, v

    # (c)
    b, n, window = 16, 131072, 4096
    q = torch.randn(b, h, 1, d, device=dev, dtype=torch.bfloat16, generator=gen)
    for cache in ("bf16", "fp8"):
        k = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
        v = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
        kw = {}
        if cache == "fp8":
            k, v = k.to(torch.float8_e4m3fn), v.to(torch.float8_e4m3fn)
            kw = dict(k_scale=torch.ones(b * hk, device=dev), v_scale=torch.ones(b * hk, device=dev))
        kd, vd = k[:, :, n - window - 1:].contiguous(), v[:, :, n - window - 1:].contiguous()
        qp = torch.full((b,), n - 1, dtype=torch.int32, device=dev)
        med = alternate({"window": lambda: tree_decode_cuda(q, k, v, dim_v=d, q_pos=qp, window=window, **kw),
                         "full": lambda: tree_decode_cuda(q, k, v, dim_v=d, **kw),
                         "dense4097": lambda: tree_decode_cuda(q, kd, vd, dim_v=d, **kw)}, args.reps, args.warmup)
        report(f"c_{cache}_window4096", med["window"], ratio_to_dense4097=round(med["window"] / med["dense4097"], 3),
               ratio_to_full=round(med["window"] / med["full"], 4))
        report(f"c_{cache}_full131072", med["full"])
        report(f"c_{cache}_dense4097", med["dense4097"])
        del k, v, kd, vd


if __name__ == "__main__":
    main()
