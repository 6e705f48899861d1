"""fp8 (e4m3) prefill forward against the bf16 forward: one causal forward pass at long context, no backward.

    python tools/bench_fp8_prefill.py [--seq 262144] [--heads 32] [--steps 5] [--warmup 2] [--profile]

Cases, run alternately in the same process (one call of each per round, CUDA-event timed, median of ``--steps``):
  bf16      ring_flash_attn_cuda on bf16 q, k, v under no_grad
  fp8       ring_flash_attn_fp8 on q, k, v quantised beforehand (quantize_fp8)
  fp8+quant quantize_fp8 of q, k, v and ring_flash_attn_fp8, as a prefill that starts from bf16 activations does
TFLOP/s counts the causal forward's matmuls: 4*B*H*D*S^2/2.  Head dim 128, batch 1, N(0, 1) inputs.

Each case's output is checked on 64 sampled rows against the fp32 oracle (utils/check.py): the bf16 op against the bf16
inputs, the fp8 op against its dequantised inputs.  With two or more GPUs it also times the same workload as a 2-GPU
ring (striped layout, S/2 tokens per rank).  Prints the card name and power limit with the result (one JSON line) and
exits non-zero if a check fails.  ``--profile`` adds the CUDA time per kernel of one call of each case
(torch.profiler).  Writes nothing.
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


def make_cases(q, k, v, causal=True, ring=None):
    """{name: fn() -> out} for one rank; ``ring`` = (ring_size, layout) runs the ring op."""
    from ring_attention_pytorch_b200 import quantize_fp8, ring_flash_attn_fp8
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda

    ring_args = () if ring is None else (None, causal, 1024, True, ring[1] == "striped", None, ring[0])
    plain_args = (None, causal) if ring is None else ring_args
    ring_size = 1 if ring is None else ring[0]
    (q8, qd), (k8, kd), (v8, vd) = (quantize_fp8(t, ring_size) for t in (q, k, v))

    def bf16():
        with torch.no_grad():
            return ring_flash_attn_cuda(q, k, v, *plain_args)

    def fp8():
        return ring_flash_attn_fp8(q8, k8, v8, qd, kd, vd, *plain_args)

    def fp8_quant():
        (a, ad), (b, bd), (c, cd) = (quantize_fp8(t, ring_size) for t in (q, k, v))
        return ring_flash_attn_fp8(a, b, c, ad, bd, cd, *plain_args)

    deq = [t.float() * s[:, None, :, None] for t, s in ((q8, qd), (k8, kd), (v8, vd))]
    return {"bf16": bf16, "fp8": fp8, "fp8+quant": fp8_quant}, deq


def time_cases(cases, steps, warmup):
    times = {c: [] for c in cases}
    for it in range(warmup + steps):
        for c, fn in cases.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if it >= warmup:
                times[c].append(e0.elapsed_time(e1))
    return times


def summarise(times, flops):
    res = {}
    for c, ts in times.items():
        ms = statistics.median(ts)
        res[c] = {"ms": round(ms, 3), "ms_min": round(min(ts), 3), "ms_max": round(max(ts), 3),
                  "tflops": round(flops / (ms * 1e-3) / 1e12, 1)}
    res["speedup_fp8_over_bf16"] = round(res["bf16"]["ms"] / res["fp8"]["ms"], 3)
    res["speedup_fp8_quant_over_bf16"] = round(res["bf16"]["ms"] / res["fp8+quant"]["ms"], 3)
    res["quantize_share_of_fp8_quant"] = round(1.0 - res["fp8"]["ms"] / res["fp8+quant"]["ms"], 3)
    return res


def out_check(q, k, v, out, world=1, rank=0, layout="plain"):
    from ring_attention_pytorch_b200.utils.check import sampled_check

    zq, zk = torch.zeros_like(q), torch.zeros_like(k)  # forward only: dout = 0, so only `out` is compared
    res = sampled_check(q, k, v, zq, out, zq, zk, zk, causal=True, layout=layout, world=world, rank=rank)
    return {"max_abs_over_max": round(res["out"]["max_abs_over_max"], 5),
            "frac_elements_out_of_tol": res["out"]["frac_elements_out_of_tol"], "nan": res["out"]["nan"]}


def _ring_worker(rank, world, S, H, D, steps, warmup, out_q):
    import torch.distributed as dist

    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, init_method="tcp://127.0.0.1:29533")
    try:
        dev = torch.device("cuda", rank)
        torch.manual_seed(0)
        pm = make_position_map("striped", world, S // world)
        idx = pm.positions(rank, dev)
        q, k, v = (torch.randn(1, S, H, D, device=dev, dtype=torch.bfloat16)[:, idx].contiguous() for _ in range(3))
        cases, deq = make_cases(q, k, v, ring=(world, "striped"))
        outs = {c: fn() for c, fn in cases.items()}
        checks = {"bf16": out_check(q, k, v, outs["bf16"], world, rank, "striped"),
                  "fp8": out_check(*deq, outs["fp8"], world, rank, "striped")}
        del outs
        times = time_cases(cases, steps, warmup)
        if rank == 0:
            out_q.put({"times": times, "checks": checks})
        dist.barrier()
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=262144)
    ap.add_argument("--heads", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()

    dev = torch.device("cuda", torch.cuda.current_device())
    S, H, D, B = args.seq, args.heads, 128, 1
    flops = 4.0 * B * H * D * S * S * 0.5
    torch.manual_seed(0)
    q, k, v = (torch.randn(B, S, H, D, device=dev, dtype=torch.bfloat16) for _ in range(3))
    cases, deq = make_cases(q, k, v)

    outs = {c: fn() for c, fn in cases.items()}
    torch.cuda.synchronize()
    checks = {"bf16": out_check(q, k, v, outs["bf16"]), "fp8": out_check(*deq, outs["fp8"]),
              "fp8+quant": out_check(*deq, outs["fp8+quant"])}
    del outs
    ok = all(not c["nan"] and c["max_abs_over_max"] < 3e-2 for c in checks.values())
    one_gpu = summarise(time_cases(cases, args.steps, args.warmup), flops)

    profile = {}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile as torch_profile

        for c, fn in cases.items():
            with torch_profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            per_kernel = {}
            for ev in prof.key_averages():
                if ev.device_type.name == "CUDA" and ev.device_time_total > 0:
                    per_kernel[ev.key[:60]] = round(ev.device_time_total / 1e3, 3)  # ms
            profile[c] = dict(sorted(per_kernel.items(), key=lambda kv: -kv[1])[:8])

    ring = None
    if torch.cuda.device_count() >= 2:
        import torch.multiprocessing as mp

        del q, k, v, deq, cases
        torch.cuda.empty_cache()
        ctx = mp.get_context("spawn")
        out_q = ctx.SimpleQueue()
        procs = [ctx.Process(target=_ring_worker, args=(r, 2, S, H, D, args.steps, args.warmup, out_q))
                 for r in range(2)]
        for p in procs:
            p.start()
        for p in procs:
            p.join()
        if all(p.exitcode == 0 for p in procs) and not out_q.empty():
            got = out_q.get()
            ring = {"world": 2, "layout": "striped", **summarise(got["times"], flops), "out_check": got["checks"]}
            ok = ok and all(not c["nan"] and c["max_abs_over_max"] < 3e-2 for c in got["checks"].values())
        else:
            ring = {"error": "2-GPU ring run failed"}
            ok = False

    print(json.dumps({
        "workload": {"seq": S, "heads": H, "dim_head": D, "batch": B, "causal": True, "pass": "fwd",
                     "steps": args.steps, "warmup": args.warmup},
        "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
        "one_gpu": one_gpu, "out_check_vs_fp32_oracle": checks, "ok": ok,
        **({"ring_2gpu": ring} if ring is not None else {"ring_2gpu": "not run: fewer than 2 GPUs"}),
        **({"profile_ms_per_kernel": profile} if profile else {}),
    }))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
