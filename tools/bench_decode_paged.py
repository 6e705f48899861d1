#!/usr/bin/env python
"""Paged KV cache in tree decode on one GPU: the contiguous call against paged calls on the same keys, each group timed
with its cases alternating call by call, the median of ``--reps`` calls per case after warm-up (CUDA events around each
call).  Every call passes ``cache_seqlens``; page ids are a seeded random permutation of the pool, so consecutive pages
of a sequence are scattered over it.

  (a) README decode shape (b 256, 32 / 8 heads, 8192 keys, d 128), bf16 and fp8 caches: contiguous, P = 16, 32, 64, 256
  (b) b 16, 131072 keys, window 4096, bf16: contiguous against P = 64 whose pages wholly before the window all name one
      poison (NaN) page -- the pool holds only the pages the window reaches
  (c) m = 4 draft tokens at the (a) shape, bf16: contiguous against P = 16

    python tools/bench_decode_paged.py [--reps 9] [--warmup 3]

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


def _bits(t):
    return t.view(torch.uint8) if t.element_size() == 1 else t


def to_pool(cache: torch.Tensor, ps: int, gen: torch.Generator, table=None):
    """cache [b, hk, n, d] -> (pool [b * n / ps, hk, ps, d], table int32 [b, n / ps]) with shuffled page ids (or the
    given table's)."""
    b, hk, n, d = cache.shape
    mp = n // ps
    perm = torch.randperm(b * mp, device=cache.device, generator=gen) if table is None else table.flatten().long()
    pool = torch.empty(b * mp, hk, ps, d, dtype=cache.dtype, device=cache.device)
    _bits(pool)[perm] = _bits(cache).view(b, hk, mp, ps, d).permute(0, 2, 1, 3, 4).reshape(b * mp, hk, ps, d)
    return pool, perm.view(b, mp).to(torch.int32)


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

    def report(case, ms, base, **extra):
        print(json.dumps(dict(case=case, ms=round(ms, 4), ratio_to_contiguous=round(ms / base, 4), **extra)),
              flush=True)

    # (a) and (c)
    b, n = 256, 8192
    lens = torch.full((b,), n, dtype=torch.int32, device=dev)
    q = torch.randn(b, h, 1, d, device=dev, dtype=torch.bfloat16, generator=gen)
    q4 = torch.randn(b, h, 4, d, device=dev, dtype=torch.bfloat16, generator=gen)
    q4_pos = torch.full((b,), n - 4, dtype=torch.int32, device=dev)
    for cache in ("bf16", "fp8"):
        k = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
        v = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
        kw = dict(dim_v=d, cache_seqlens=lens)
        if cache == "fp8":
            k, v = k.to(torch.float8_e4m3fn), v.to(torch.float8_e4m3fn)
            kw.update(k_scale=torch.ones(b * hk, device=dev), v_scale=torch.ones(b * hk, device=dev))
        cases = {"contiguous": lambda: tdc.tree_decode_cuda(q, k, v, **kw)}
        pools = {}
        for ps in (16, 32, 64, 256):
            kp, table = to_pool(k, ps, gen)
            vp, _ = to_pool(v, ps, gen, table)
            pools[ps] = (kp, vp, table)
            cases[f"P{ps}"] = (lambda kp=kp, vp=vp, table=table:
                               tdc.tree_decode_cuda(q, kp, vp, block_table=table, **kw))
        out = {name: fn() for name, fn in cases.items()}
        assert all(torch.equal(o, out["contiguous"]) for o in out.values()), "paged and contiguous calls differ"
        med = alternate(cases, args.reps, args.warmup)
        kv_bytes = 2 * b * hk * n * d * (1 if cache == "fp8" else 2)
        for name in cases:
            report(f"a_{cache}_{name}", med[name], med["contiguous"], gbps=round(kv_bytes / med[name] / 1e6, 1))
        if cache == "bf16":  # (c)
            kp, vp, table = pools[16]
            kw4 = dict(kw, q_pos=q4_pos)
            cases = {"contiguous": lambda: tdc.tree_decode_cuda(q4, k, v, **kw4),
                     "P16": lambda: tdc.tree_decode_cuda(q4, kp, vp, block_table=table, **kw4)}
            assert torch.equal(cases["contiguous"](), cases["P16"]()), "paged and contiguous calls differ"
            med = alternate(cases, args.reps, args.warmup)
            for name in cases:
                report(f"c_m4_{name}", med[name], med["contiguous"])
        del k, v, pools, cases, out
        torch.cuda.empty_cache()

    # (b)
    b, n, window, ps = 16, 131072, 4096, 64
    lens = torch.full((b,), n, dtype=torch.int32, device=dev)
    q_pos = lens - 1
    q = torch.randn(b, h, 1, d, device=dev, dtype=torch.bfloat16, generator=gen)
    k = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
    v = torch.randn(b, hk, n, d, device=dev, dtype=torch.bfloat16, generator=gen)
    first = (n - 1 - window) // ps  # the first page the window reaches
    live = n // ps - first
    kp = torch.full((b * live + 1, hk, ps, d), float("nan"), device=dev, dtype=torch.bfloat16)  # page 0: poison
    vp = kp.clone()
    perm = torch.randperm(b * live, device=dev, generator=gen) + 1
    table = torch.zeros(b, n // ps, dtype=torch.int32, device=dev)
    table[:, first:] = perm.view(b, live).to(torch.int32)
    for pool, src in ((kp, k), (vp, v)):
        pool[perm] = src[:, :, first * ps:].reshape(b, hk, live, ps, d).permute(0, 2, 1, 3, 4).reshape(-1, hk, ps, d)
    kw = dict(dim_v=d, cache_seqlens=lens, q_pos=q_pos, window=window)
    cases = {"contiguous": lambda: tdc.tree_decode_cuda(q, k, v, **kw),
             "P64": lambda: tdc.tree_decode_cuda(q, kp, vp, block_table=table, **kw)}
    assert torch.equal(cases["contiguous"](), cases["P64"]()), "paged and contiguous calls differ"
    med = alternate(cases, args.reps, args.warmup)
    for name in cases:
        report(f"b_window{window}_{name}", med[name], med["contiguous"])


if __name__ == "__main__":
    main()
