"""Cost of learned attention sinks: the same workloads with and without ``sinks``.

    python tools/bench_attn_sinks.py [--seq 262144] [--heads 32] [--steps 5] [--warmup 1]

Cases, run alternately in the same process (one call of each per round, CUDA-event timed, median of ``--steps``):
  full      causal training step (forward + backward) of ring_flash_attn_cuda, S tokens, bf16, head dim 128, batch 1
  window128 the same with max_lookback_seq_len=128, the sliding-window-plus-sink shape
  decode    tree_decode_cuda, batch 256, 32 query / 8 KV heads, 8192 keys, head dim 128, bf16 cache
each ``plain`` (sinks=None) and ``sinks`` (fp32 [h] sinks that require grad).  Prints the card name and power limit
with the result (one JSON line).  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_documents import power_limit_w  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=262144)
    ap.add_argument("--heads", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attn_sinks needs a CUDA device")
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda
    from ring_attention_pytorch_b200.ops.tree_decode_cuda import tree_decode_cuda

    torch.manual_seed(0)
    S, h, d = args.seq, args.heads, 128
    dt = torch.bfloat16
    q, k, v, do = (torch.randn(1, S, h, d, device="cuda", dtype=dt) for _ in range(4))
    q, k, v = (t.requires_grad_() for t in (q, k, v))
    sinks = torch.zeros(h, device="cuda", requires_grad=True)
    dq_ = torch.randn(256, 32, 1, d, device="cuda", dtype=dt)
    dk_, dv_ = (torch.randn(256, 8, 8192, d, device="cuda", dtype=dt) for _ in range(2))
    dsinks = torch.zeros(32, device="cuda")
    dout = torch.empty(256, 32, 1, d, device="cuda", dtype=dt)

    def train(window, with_sinks):
        def fn():
            out = ring_flash_attn_cuda(q, k, v, None, True, 1024, max_lookback_seq_len=window,
                                       sinks=sinks if with_sinks else None)
            torch.autograd.grad(out, (q, k, v, sinks) if with_sinks else (q, k, v), do)
        return fn

    def decode(with_sinks):
        def fn():
            for _ in range(20):  # 20 decode steps per timed call
                tree_decode_cuda(dq_, dk_, dv_, dim_v=d, out=dout, sinks=dsinks if with_sinks else None)
        return fn

    cases = {"full/plain": train(None, False), "full/sinks": train(None, True),
             "window128/plain": train(128, False), "window128/sinks": train(128, True),
             "decode/plain": decode(False), "decode/sinks": decode(True)}
    times = {c: [] for c in cases}
    for it in range(args.warmup + args.steps):
        for c, fn in cases.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if it >= args.warmup:
                times[c].append(e0.elapsed_time(e1) / (20 if c.startswith("decode") else 1))
    res = {c: {"ms": round(statistics.median(ts), 4), "ms_min": round(min(ts), 4), "ms_max": round(max(ts), 4)}
           for c, ts in times.items()}
    for w in ("full", "window128", "decode"):
        res[f"{w}/sinks_over_plain"] = round(res[f"{w}/sinks"]["ms"] / res[f"{w}/plain"]["ms"], 4)
    dev = torch.cuda.current_device()
    res.update(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(dev), seq=S, heads=h,
               steps=args.steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
