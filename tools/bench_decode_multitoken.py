#!/usr/bin/env python
"""Multi-token tree decode on one GPU (speculative verification: m draft tokens per sequence in one call), each group
timed with its cases alternating call by call, the median of ``--reps`` calls per case after warm-up (CUDA events
around each call).  Every call passes ``cache_seqlens`` and ``q_pos`` (the m tokens are the last m keys held).

  (a) README decode shape (b 256, 32 / 8 heads, 8192 keys, d 128), bf16 and fp8 caches, tensor-core kernel: one call
      with m = 1, 2, 4, 8, and 4 sequential single-token calls
  (b) long context (b 16, 32 / 8 heads, 131072 keys, d 128, bf16): m = 1, 4, 8, with and without a 4096-token window

    python tools/bench_decode_multitoken.py [--reps 9] [--warmup 3]

Prints the card's name and power limit first, then one JSON line per case.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_decode_ragged import alternate, card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    assert args.reps >= 9, "at least 9 timed calls per case"
    from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc

    tdc.CONFIG["tensor_core"] = "on"
    print(f"[card] {card()}", flush=True)
    dev = torch.device("cuda")
    gen = torch.Generator(dev).manual_seed(0)
    h, hk, d = 32, 8, 128

    def report(case, ms, **extra):
        print(json.dumps(dict(case=case, ms=round(ms, 4), **extra)), flush=True)

    def calls(q, k, v, n, b, ms_, kw):
        lens = torch.full((b,), n, dtype=torch.int32, device=dev)
        out = {}
        for m in ms_:
            qp = torch.full((b,), n - m, dtype=torch.int32, device=dev)
            qm = q[:, :, :m].contiguous()
            out[f"m{m}"] = (lambda qm=qm, qp=qp: tdc.tree_decode_cuda(qm, k, v, dim_v=d, cache_seqlens=lens, q_pos=qp,
                                                                      **kw))
        return out, lens

    # (a)
    b, n = 256, 8192
    q = torch.randn(b, h, 8, d, device=dev, dtype=torch.bfloat16, generator=gen)
    for cache in ("bf16", "fp8"):
        k = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
        v = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
        kw = {}
        if cache == "fp8":
            k, v = k.to(torch.float8_e4m3fn), v.to(torch.float8_e4m3fn)
            kw = dict(k_scale=torch.ones(b * hk, device=dev), v_scale=torch.ones(b * hk, device=dev))
        cases, lens = calls(q, k, v, n, b, (1, 2, 4, 8), kw)
        singles = [(q[:, :, t:t + 1].contiguous(), torch.full((b,), n - 4 + t, dtype=torch.int32, device=dev))
                   for t in range(4)]

        def seq4():
            for qt, qp in singles:
                tdc.tree_decode_cuda(qt, k, v, dim_v=d, cache_seqlens=lens, q_pos=qp, **kw)

        cases["seq4"] = seq4
        med = alternate(cases, args.reps, args.warmup)
        kv_bytes = 2 * b * hk * n * d * (1 if cache == "fp8" else 2)
        for m in (1, 2, 4, 8):
            report(f"a_{cache}_m{m}", med[f"m{m}"], gbps=round(kv_bytes / med[f"m{m}"] / 1e6, 1),
                   ratio_to_m1=round(med[f"m{m}"] / med["m1"], 4))
        report(f"a_{cache}_4x_single", med["seq4"], m4_speedup=round(med["seq4"] / med["m4"], 3))
        del k, v

    # (b)
    b, n, window = 16, 131072, 4096
    q = torch.randn(b, h, 8, d, device=dev, dtype=torch.bfloat16, generator=gen)
    k = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
    v = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
    for w in (None, window):
        cases, _ = calls(q, k, v, n, b, (1, 4, 8), dict(window=w))
        med = alternate(cases, args.reps, args.warmup)
        for m in (1, 4, 8):
            report(f"b_window{w or 0}_m{m}", med[f"m{m}"], ratio_to_m1=round(med[f"m{m}"] / med["m1"], 4))


if __name__ == "__main__":
    main()
