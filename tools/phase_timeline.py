"""Per-phase CUDA-event timeline of the ring attention op on every rank (run under torchrun).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 \
        tools/phase_timeline.py --seq-len 262144 --out phase_timeline_n8.json

Phases are the ``nvtx_range`` regions of ``ops/ring_cuda.py`` (pack + device barrier, forward kernel, backward prep,
accumulator zero + barrier, backward kernel + dQ convert, final barrier + dK/dV convert).  Every rank reports the
milliseconds of each phase for the timed steps; rank 0 prints a table (median per rank) and writes the JSON.  The wait a
rank spends inside a device barrier shows up in the phase that contains it, which is what attributes multi-GPU scaling
loss to skew between ranks rather than to the kernels.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq-len", type=int, default=262144)
    ap.add_argument("--heads", type=int, default=32)
    ap.add_argument("--kv-heads", type=int, default=None)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)

    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda
    from ring_attention_pytorch_b200.utils import timing

    H, HK, D = args.heads, args.kv_heads or args.heads, 128
    n = args.seq_len // world
    torch.manual_seed(rank)
    q = torch.randn(1, n, H, D, device=dev, dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(1, n, HK, D, device=dev, dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(1, n, HK, D, device=dev, dtype=torch.bfloat16, requires_grad=True)
    w = torch.randn(1, n, H, D, device=dev, dtype=torch.bfloat16)

    def step():
        out = ring_flash_attn_cuda(q, k, v, None, True, 1024, world > 1, world > 1, None, world)
        out.backward(w)
        q.grad = k.grad = v.grad = None

    for _ in range(args.warmup):
        step()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    timing.enable_phase_timing(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    rep = timing.phase_report()
    timing.enable_phase_timing(False)
    mine = {name: statistics.median(ms) for name, ms in rep.items()}
    mine["step_total"] = e0.elapsed_time(e1) / args.steps
    allr = [None] * world
    if world > 1:
        dist.all_gather_object(allr, mine)
    else:
        allr = [mine]
    if rank == 0:
        names = list(mine.keys())
        print(f"{'phase':28s}" + "".join(f"  rank{r:<2d}" for r in range(world)) + "     max    min")
        for nme in names:
            vals = [a.get(nme, 0.0) for a in allr]
            print(f"{nme:28s}" + "".join(f" {x:7.2f}" for x in vals) + f"  {max(vals):7.2f} {min(vals):7.2f}")
        res = {"n_gpus": world, "seq_len": args.seq_len, "heads": H, "kv_heads": HK, "steps": args.steps,
               "unit": "ms (median over steps, per rank)", "phases": {nme: [a.get(nme, 0.0) for a in allr] for nme in names}}
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                json.dump(res, f, indent=1)
        print(json.dumps(res))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
