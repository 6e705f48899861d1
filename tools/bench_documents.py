"""Packed-sequence document masking on one GPU: step time of causal fwd+bwd with and without ``document_ids``.

    python tools/bench_documents.py [--seq 262144] [--heads 32] [--dim-head 128] [--steps 5] [--warmup 2] [--profile]

Cases, run alternately in the same process (one fwd+bwd step of each per round, CUDA-event timed):
  (a) no document_ids                      (b) document_ids with one document
  (c) documents of 8192 tokens             (d) random document lengths in [1K, 64K] (seeded)
TFLOP/s counts the visible pairs only: bench.py's 4*B*H*D*S^2/2*3.5 with S^2/2 replaced by sum(L_i^2)/2.

Before timing, case (c)'s out / dQ / dK / dV are checked against running each document on its own through the same
op (the documents as a batch, no document_ids).  Prints the card name and power limit with the result (one JSON
line) and exits non-zero if the check fails.  ``--profile`` adds the CUDA time per kernel of one step of cases (a) and
(b) (torch.profiler), to show which kernel a difference between them comes from.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit_w(index: int):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out)
    except Exception:  # noqa: BLE001
        return None


def document_lengths(kind: str, S: int, seed: int = 0):
    if kind in ("none", "one"):
        return [S]
    if kind == "8k":
        return [8192] * (S // 8192)
    g = torch.Generator().manual_seed(seed)
    lens, left = [], S
    while left > 0:
        L = min(int(torch.randint(1024, 65536 + 1, (1,), generator=g)), left)
        lens.append(L)
        left -= L
    return lens


def ids_of(lens, device):
    return torch.repeat_interleave(torch.arange(len(lens), device=device), torch.tensor(lens, device=device))[None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=262144)
    ap.add_argument("--heads", type=int, default=32)
    ap.add_argument("--dim-head", type=int, default=128)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()

    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda

    dev = torch.device("cuda", torch.cuda.current_device())
    S, H, D, B = args.seq, args.heads, args.dim_head, 1
    torch.manual_seed(0)
    q, k, v, g = (torch.randn(B, S, H, D, device=dev, dtype=torch.bfloat16) for _ in range(4))
    q, k, v = (t.requires_grad_() for t in (q, k, v))

    def step(ids):
        out = ring_flash_attn_cuda(q, k, v, None, True, document_ids=ids)
        grads = torch.autograd.grad(out, (q, k, v), g)
        return out, grads

    # ---- correctness of case (c): packed equals every document on its own
    L = 8192
    ids_c = ids_of(document_lengths("8k", S), dev)
    out_p, grads_p = step(ids_c)
    nd = S // L
    qs, ks, vs = (t.detach().view(nd, L, H, D).clone().requires_grad_() for t in (q, k, v))
    out_s = ring_flash_attn_cuda(qs, ks, vs, None, True)
    grads_s = torch.autograd.grad(out_s, (qs, ks, vs), g.view(nd, L, H, D))
    check = {}
    for name, a, b in (("out", out_p, out_s), ("dq", grads_p[0], grads_s[0]), ("dk", grads_p[1], grads_s[1]),
                       ("dv", grads_p[2], grads_s[2])):
        a, b = a.reshape(-1).float(), b.reshape(-1).float()
        check[name] = float((a - b).detach().abs().max() / b.detach().abs().max().clamp_min(1e-6))
    check_ok = all(e < 2e-2 for e in check.values())
    del out_p, grads_p, out_s, grads_s, qs, ks, vs

    # ---- timing, cases alternating
    cases = {"a_none": None, "b_one_doc": "one", "c_8k_docs": "8k", "d_random_1k_64k": "random"}
    lens = {c: document_lengths(kind or "none", S) for c, kind in cases.items()}
    ids = {c: (None if kind is None else ids_of(lens[c], dev)) for c, kind in cases.items()}
    times = {c: [] for c in cases}
    for it in range(args.warmup + args.steps):
        for c in cases:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(ids[c])
            e1.record()
            torch.cuda.synchronize()
            if it >= args.warmup:
                times[c].append(e0.elapsed_time(e1))
    res = {}
    for c in cases:
        ms = statistics.median(times[c])
        flops = 4.0 * B * H * D * sum(float(x) ** 2 for x in lens[c]) * 0.5 * 3.5
        res[c] = {"ms_per_step": round(ms, 3), "ms_min": round(min(times[c]), 3), "ms_max": round(max(times[c]), 3),
                  "documents": len(lens[c]), "visible_tflops": round(flops / (ms * 1e-3) / 1e12, 1)}
    profile = {}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile as torch_profile

        for c in ("a_none", "b_one_doc"):
            with torch_profile(activities=[ProfilerActivity.CUDA]) as prof:
                step(ids[c])
                torch.cuda.synchronize()
            per_kernel = {}
            for ev in prof.key_averages():
                if ev.device_type.name == "CUDA" and ev.device_time_total > 0:
                    per_kernel[ev.key[:60]] = round(ev.device_time_total / 1e3, 2)  # ms
            profile[c] = dict(sorted(per_kernel.items(), key=lambda kv: -kv[1])[:6])
    print(json.dumps({
        "workload": {"seq": S, "heads": H, "dim_head": D, "batch": B, "dtype": "bf16", "causal": True,
                     "pass": "fwd+bwd", "steps": args.steps, "warmup": args.warmup},
        "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
        "cases": res,
        "speedup_c_over_a": round(res["a_none"]["ms_per_step"] / res["c_8k_docs"]["ms_per_step"], 2),
        "check_8k_docs_vs_separate": {"max_rel_err": check, "ok": check_ok},
        **({"profile_ms_per_kernel": profile} if profile else {}),
    }))
    sys.exit(0 if check_ok else 1)


if __name__ == "__main__":
    main()
