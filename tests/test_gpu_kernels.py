"""GPU tests (H100): every sm_90a kernel against a plain PyTorch fp32 oracle of the same op.

Run with ``python -m pytest tests -m gpu -x -q`` on a box with a GPU.  The multi-rank ring protocol is
exercised on a single device by emulating W ranks (``ops.fused.emulate_ring_*``) and, when >= 2 GPUs are
visible, for real over NCCL-bootstrapped symmetric memory.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

pytestmark = pytest.mark.gpu


def _cases():
    import gpu_dev_check

    return gpu_dev_check


def test_extension_is_loaded_not_a_fallback():
    from ring_attention_pytorch_b200.ops import _ext

    assert _ext.load()
    assert _ext.extension_path().exists()
    assert hasattr(torch.ops.rab, "attn_fwd")


FWD_CASES = {
    "d128": dict(),
    "d128_n128_h1": dict(n=128, h=1),
    "d128_causal": dict(n=512, causal=True),
    "d128_tail": dict(n=300, b=2),
    "d128_causal_n1000": dict(n=1000, causal=True, h=4),
    "d64": dict(n=512, d=64, h=4),
    "d64_causal_tail": dict(n=777, d=64, h=4, causal=True),
    "gqa_causal": dict(n=512, h=8, hk=2, causal=True),
    "kmask": dict(n=384, h=2, kmask=True, b=2),
    "softclamp": dict(n=384, h=2, softclamp=20.0),
    "window": dict(n=1024, h=2, causal=True, window=200),
    "fp16": dict(n=512, h=2, causal=True, dtype="fp16"),
    "many_items": dict(n=2048, h=16, b=2, causal=True),
    "ring2_plain": dict(world=2, n=256, h=2),
    "ring2_plain_causal": dict(world=2, n=256, h=2, causal=True),
    "ring4_striped_causal_gqa": dict(world=4, n=384, h=4, hk=2, layout="striped", causal=True),
    "ring4_zigzag_causal": dict(world=4, n=512, h=2, layout="zigzag", causal=True),
    "ring4_plain_window": dict(world=4, n=256, h=2, causal=True, window=300),
    "ring3_kmask": dict(world=3, n=200, h=2, kmask=True),
    "ring8_striped_causal": dict(world=8, n=1024, h=8, hk=2, layout="striped", causal=True),
}


@pytest.mark.parametrize("name", list(FWD_CASES))
def test_fused_forward(name):
    res = _cases().case_fwd(**FWD_CASES[name])
    assert res["ok"], res


BWD_CASES = {k: v for k, v in FWD_CASES.items() if k != "ring8_striped_causal"}
BWD_CASES["n64_h1"] = dict(n=64, h=1)
BWD_CASES["ring8_striped_causal_gqa"] = dict(world=8, n=512, h=8, hk=2, layout="striped", causal=True)
# head dim 128 defaults to the one-kernel (5-GEMM) backward; the two-kernel pair stays covered explicitly
BWD_CASES["two_kernel_d128_causal"] = dict(n=1000, causal=True, h=4, fused=False)
BWD_CASES["two_kernel_gqa_causal"] = dict(n=512, h=8, hk=2, causal=True, fused=False)
BWD_CASES["two_kernel_ring4_striped"] = dict(world=4, n=384, h=4, hk=2, layout="striped", causal=True, fused=False)


@pytest.mark.parametrize("name", list(BWD_CASES))
def test_fused_backward(name):
    res = _cases().case_bwd(**BWD_CASES[name])
    assert res["ok"], res


# memory="ring": one launch per hop against a single K/V slot, softmax state / fp32 accumulators carried between launches
HOP_CASES = {k: dict(v, hopwise=True) for k, v in FWD_CASES.items() if k.startswith("ring")}
HOP_CASES["ring4_d64_striped_causal"] = dict(world=4, n=300, h=4, hk=2, d=64, layout="striped", causal=True, hopwise=True)
HOP_CASES["ring8_plain_window_sparse"] = dict(world=8, n=256, h=2, causal=True, window=300, hopwise=True)
HOP_CASES["ring4_softclamp_fp16"] = dict(world=4, n=384, h=2, layout="zigzag", causal=True, softclamp=20.0, dtype="fp16",
                                         hopwise=True)


@pytest.mark.parametrize("name", list(HOP_CASES))
def test_hopwise_forward(name):
    res = _cases().case_fwd(**HOP_CASES[name])
    assert res["ok"], res


@pytest.mark.parametrize("name", [k for k, v in HOP_CASES.items() if v.get("d", 128) == 128])
def test_hopwise_backward(name):
    res = _cases().case_bwd(**HOP_CASES[name])
    assert res["ok"], res


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("d", [32, 64, 128])
def test_autograd_op_matches_oracle(causal, d):
    from ring_attention_pytorch_b200 import default_attention
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda

    torch.manual_seed(0)
    q = torch.randn(2, 200, 4, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(2, 200, 2, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(2, 200, 2, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    g = torch.randn(2, 200, 4, d, device="cuda", dtype=torch.bfloat16)
    out = ring_flash_attn_cuda(q, k, v, None, causal)
    got = torch.autograd.grad(out, (q, k, v), g)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    ref = default_attention(qf, kf, vf, causal=causal)
    want = torch.autograd.grad(ref, (qf, kf, vf), g.float())
    assert (out.float() - ref).abs().max() < 3e-2
    for a, b in zip(got, want):
        assert (a.float() - b).abs().max() / b.abs().max() < 3e-2


def test_cross_attention_and_fp32_inputs():
    from ring_attention_pytorch_b200 import default_attention
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda

    torch.manual_seed(0)
    q = torch.randn(1, 70, 2, 64, device="cuda")
    k = torch.randn(1, 333, 2, 64, device="cuda")
    v = torch.randn(1, 333, 2, 64, device="cuda")
    for causal in (False, True):
        out = ring_flash_attn_cuda(q, k, v, None, causal)
        assert out.dtype == torch.float32
        ref = default_attention(q, k, v, causal=causal)
        assert (out - ref).abs().max() < 3e-2


def test_transformer_cuda_kernel_matches_dense():
    from ring_attention_pytorch_b200 import RingTransformer

    torch.manual_seed(0)
    kw = dict(num_tokens=128, dim=128, depth=2, causal=True, dim_head=64, heads=4, num_grouped_query_heads=2,
              bucket_size=64, ring_attn=False)
    fused = RingTransformer(use_cuda_kernel=True, **kw).cuda()
    dense = RingTransformer(use_cuda_kernel=False, force_regular_attn=True, **kw).cuda()
    dense.load_state_dict(fused.state_dict())
    tokens = torch.randint(0, 128, (2, 257), device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        a = fused(tokens)
        b = dense(tokens)
    assert (a.float() - b.float()).abs().max() < 0.15
    la = fused(tokens, return_loss=True)
    lb = dense(tokens, return_loss=True)
    la.backward()
    lb.backward()
    ga, gb = fused.token_emb.weight.grad, dense.token_emb.weight.grad
    assert (ga - gb).abs().max() / gb.abs().max() < 5e-2


def test_graft_smoke():
    sys.path.insert(0, ROOT)
    import __graft_entry__

    __graft_entry__.smoke()


# ------------------------------------------------------------------------------------------------
# real multi-GPU ring (NVLink, symmetric memory) – needs >= 2 devices
# ------------------------------------------------------------------------------------------------
def _ring_worker(rank, world, layout, causal, hk, kmask=False, backward="fused", memory="gather"):
    import torch.distributed as dist

    from ring_attention_pytorch_b200.ops import ring_cuda

    ring_cuda.CONFIG["backward"] = backward
    ring_cuda.CONFIG["memory"] = memory

    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    torch.manual_seed(0)
    b, n, h, d = 1, 640, 4, 128
    dev = torch.device("cuda", rank)
    qs = [torch.randn(b, n, h, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    ks = [torch.randn(b, n, hk, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    vs = [torch.randn(b, n, hk, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    gs = [torch.randn(b, n, h, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    q, k, v = (t[rank].clone().requires_grad_() for t in (qs, ks, vs))
    masks = [torch.rand(b, n, device=dev) > 0.3 for _ in range(world)] if kmask else None
    for _ in range(2):  # twice: exercises the double-buffered staging + epoch barrier
        out = ring_flash_attn_cuda(q, k, v, masks[rank] if kmask else None, causal, 1024, True, layout == "striped",
                                   None, world, False, 50.0, layout)
        dq, dk, dv = torch.autograd.grad(out, (q, k, v), gs[rank])
    torch.cuda.synchronize()
    pm = make_position_map(layout, world, n)
    qf = [t.float().requires_grad_() for t in qs]
    kf = [t.float().requires_grad_() for t in ks]
    vf = [t.float().requires_grad_() for t in vs]
    k_all, v_all = torch.cat(kf, 1), torch.cat(vf, 1)
    k_pos = torch.cat([pm.positions(r, dev) for r in range(world)])
    loss = 0
    outs = []
    for r in range(world):
        o = attention_with_positions(qf[r], k_all, v_all, pm.positions(r, dev), k_pos, causal=causal,
                                     key_mask=torch.cat(masks, 1) if kmask else None)
        outs.append(o)
        loss = loss + (o * gs[r].float()).sum()
    loss.backward()
    assert (out.float() - outs[rank]).abs().max() < 3e-2
    for got, ref in ((dq, qf[rank].grad), (dk, kf[rank].grad), (dv, vf[rank].grad)):
        assert (got.float() - ref).abs().max() / ref.abs().max() < 3e-2
    dist.barrier()


@pytest.mark.parametrize("layout,causal,hk,kmask,backward,memory", [("plain", False, 4, False, "fused", "gather"),
                                                                    ("striped", True, 2, False, "fused", "gather"),
                                                                    ("zigzag", True, 4, False, "fused", "gather"),
                                                                    ("plain", False, 2, True, "fused", "gather"),
                                                                    ("striped", True, 2, False, "two_kernel", "gather"),
                                                                    ("plain", False, 4, True, "two_kernel", "gather"),
                                                                    ("striped", True, 2, False, "fused", "ring"),
                                                                    ("plain", True, 4, False, "fused", "ring"),
                                                                    ("zigzag", True, 4, False, "fused", "ring"),
                                                                    ("plain", False, 2, True, "fused", "ring"),
                                                                    ("plain", False, 2, True, "two_kernel", "ring")])
def test_real_ring_two_gpus(layout, causal, hk, kmask, backward, memory):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from dist_utils import run_distributed

    world = min(torch.cuda.device_count(), 8)
    world = 2 if world < 4 else 4
    run_distributed(_ring_worker, world, layout, causal, hk, kmask, backward, memory, backend="nccl")


# ------------------------------------------------------------------------------------------------
# tree-attention decode kernel
# ------------------------------------------------------------------------------------------------
def _dense_decode(q, k, v):
    b, h, _, d = q.shape
    hk = k.shape[1]
    kx = k.float().repeat(1, h // hk, 1, 1)
    vx = v.float().repeat(1, h // hk, 1, 1)
    sim = torch.einsum("bhid,bhjd->bhij", q.float(), kx) * d ** -0.5
    return torch.einsum("bhij,bhjd->bhid", sim.softmax(-1), vx)


# The single-GPU decode kernels are tested under the noise-scaled rule in tests/test_decode_kernels.py.
def _tree_worker_gpu(rank, world, seq_len):
    import torch.distributed as dist

    from ring_attention_pytorch_b200 import tree_attn_decode

    torch.manual_seed(0)
    dev = torch.device("cuda", rank)
    q = torch.randn(2, 8, 1, 128, device=dev, dtype=torch.bfloat16)
    k = torch.randn(2, 4, seq_len, 128, device=dev, dtype=torch.bfloat16)
    v = torch.randn(2, 4, seq_len, 128, device=dev, dtype=torch.bfloat16)
    ref = _dense_decode(q, k, v)
    for _ in range(3):
        out = tree_attn_decode(q, k, v)
    torch.cuda.synchronize()
    assert (out.float() - ref).abs().max() < 2e-2
    dist.barrier()


@pytest.mark.parametrize("seq_len", [4099, 1])
def test_tree_decode_multi_gpu(seq_len):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from dist_utils import run_distributed

    run_distributed(_tree_worker_gpu, 2, seq_len, backend="nccl")


def _module_worker_gpu(rank, world, striped):
    import torch.distributed as dist

    from ring_attention_pytorch_b200 import RingTransformer

    torch.manual_seed(0)
    dev = torch.device("cuda", rank)
    seq_len = 1000
    ring_seq = 512
    kw = dict(num_tokens=256, dim=256, depth=2, causal=True, dim_head=64, heads=4, num_grouped_query_heads=2,
              bucket_size=ring_seq)
    ring = RingTransformer(ring_attn=True, striped_ring_attn=striped, ring_seq_size=ring_seq, use_cuda_kernel=True,
                           **kw).to(dev)
    dense = RingTransformer(ring_attn=False, use_cuda_kernel=False, force_regular_attn=True, **kw).to(dev)
    dense.load_state_dict(ring.state_dict())
    torch.manual_seed(10 + rank)
    tokens = torch.randint(0, 256, (2, seq_len), device=dev)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        a = ring(tokens)
        b = dense(tokens)
    assert a.shape == b.shape
    assert (a.float() - b.float()).abs().max() < 0.2
    loss = ring(tokens, return_loss=True)
    loss.backward()
    assert torch.isfinite(loss) and torch.isfinite(ring.token_emb.weight.grad).all()
    dist.barrier()


@pytest.mark.parametrize("striped", [False, True])
def test_ring_transformer_multi_gpu(striped):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from dist_utils import run_distributed

    run_distributed(_module_worker_gpu, 2, striped, backend="nccl")


def _ring_set_worker(rank, world, ring_size):
    """world = ring_sets x ring_size: every ring set runs its own independent striped causal ring."""
    import torch.distributed as dist

    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    torch.manual_seed(0)
    b, n, h, hk, d = 1, 384, 4, 2, 128
    dev = torch.device("cuda", rank)
    qs = [torch.randn(b, n, h, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    ks = [torch.randn(b, n, hk, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    vs = [torch.randn(b, n, hk, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    gs = [torch.randn(b, n, h, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    q, k, v = (t[rank].clone().requires_grad_() for t in (qs, ks, vs))
    out = ring_flash_attn_cuda(q, k, v, None, True, 1024, True, True, None, ring_size)
    dq, dk, dv = torch.autograd.grad(out, (q, k, v), gs[rank])
    torch.cuda.synchronize()

    ring_set = rank // ring_size
    members = list(range(ring_set * ring_size, (ring_set + 1) * ring_size))
    pm = make_position_map("striped", ring_size, n)
    qf = {r: qs[r].float().requires_grad_() for r in members}
    kf = {r: ks[r].float().requires_grad_() for r in members}
    vf = {r: vs[r].float().requires_grad_() for r in members}
    k_all = torch.cat([kf[r] for r in members], 1)
    v_all = torch.cat([vf[r] for r in members], 1)
    k_pos = torch.cat([pm.positions(i, dev) for i in range(ring_size)])
    loss, outs = 0, {}
    for i, r in enumerate(members):
        o = attention_with_positions(qf[r], k_all, v_all, pm.positions(i, dev), k_pos, causal=True)
        outs[r] = o
        loss = loss + (o * gs[r].float()).sum()
    loss.backward()
    assert (out.float() - outs[rank]).abs().max() < 3e-2
    for got, ref in ((dq, qf[rank].grad), (dk, kf[rank].grad), (dv, vf[rank].grad)):
        assert (got.float() - ref).abs().max() / ref.abs().max() < 3e-2
    dist.barrier()


def test_ring_sets_four_gpus():
    if torch.cuda.device_count() < 4:
        pytest.skip("needs >= 4 GPUs")
    from dist_utils import run_distributed

    run_distributed(_ring_set_worker, 4, 2, backend="nccl")


@pytest.mark.parametrize("d", [64, 128])
def test_hop_api_kernel_path_matches_dense_path(d):
    """flash_attn_forward / flash_attn_backward (reference triton_flash_attn.py:304, 988): the sm_90a kernels as
    single-hop building blocks with carried (o, m, lse), vs the dense fp32 path of the same functions."""
    from ring_attention_pytorch_b200.ops import flash_attn as fa

    torch.manual_seed(0)
    b, n, h, hk = 2, 300, 4, 2
    q = torch.randn(b, n, h, d, device="cuda", dtype=torch.bfloat16)
    ks = [torch.randn(b, n, hk, d, device="cuda", dtype=torch.bfloat16) for _ in range(3)]
    vs = [torch.randn(b, n, hk, d, device="cuda", dtype=torch.bfloat16) for _ in range(3)]
    keep = torch.rand(b, n, device="cuda") > 0.3
    bias = torch.where(keep, 0.0, -torch.finfo(torch.float32).max)
    # hop 0: causal incl. diagonal; hop 1: causal, diagonal masked (striped, later rank); hop 2: key padding
    hop_kw = [dict(causal=True), dict(causal=True, causal_mask_diagonal=True), dict(bias=bias)]

    def run(qq, kk, vv):
        o = torch.zeros(b, n, h, d, device="cuda", dtype=torch.float32)
        m = lse = None
        for i, kw in enumerate(hop_kw):
            o, m, lse = fa.flash_attn_forward(qq, kk[i], vv[i], o=o, m=m, lse=lse, load_accumulated=i > 0,
                                              return_normalized_output=i == 2, **kw)
        return o, lse

    assert fa._use_kernel(q, True)
    o_k, lse_k = run(q, ks, vs)
    o_d, lse_d = run(q.float(), [t.float() for t in ks], [t.float() for t in vs])
    assert (o_k - o_d).abs().max() < 3e-2
    assert (lse_k[..., :n] - lse_d[..., :n]).abs().max() < 3e-2

    do = torch.randn(b, n, h, d, device="cuda", dtype=torch.bfloat16)
    for i, kw in enumerate(hop_kw):
        got = [torch.empty_like(q), torch.empty_like(ks[i]), torch.empty_like(vs[i])]
        want = [torch.empty_like(t, dtype=torch.float32) for t in got]
        dl_k = fa.flash_attn_backward(do, q, ks[i], vs[i], o_d.to(q.dtype), lse_d, *got, **kw)
        dl_d = fa.flash_attn_backward(do.float(), q.float(), ks[i].float(), vs[i].float(), o_d, lse_d, *want, **kw)
        assert (dl_k - dl_d).abs().max() < 5e-2
        for a, w in zip(got, want):
            assert (a.float() - w).abs().max() / w.abs().max() < 4e-2, (i, kw.keys())


# ------------------------------------------------------------------------------------------------
# real rings at a size where a localized bug would show: sampled rows against the chunked fp32 oracle
# ------------------------------------------------------------------------------------------------
def _big_ring_worker(rank, world, layout, n, h, hk, ring_size, memory="gather"):
    import torch.distributed as dist

    from ring_attention_pytorch_b200.ops import ring_cuda
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda
    from ring_attention_pytorch_b200.utils.check import sampled_check

    ring_cuda.CONFIG["memory"] = memory
    ring_size = ring_size or world
    torch.manual_seed(100 + rank)
    dev = torch.device("cuda", rank)
    q = torch.randn(1, n, h, 128, device=dev, dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(1, n, hk, 128, device=dev, dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(1, n, hk, 128, device=dev, dtype=torch.bfloat16, requires_grad=True)
    g = torch.randn(1, n, h, 128, device=dev, dtype=torch.bfloat16)
    out = ring_flash_attn_cuda(q, k, v, None, True, 1024, True, layout == "striped", None, ring_size, False, 50.0, layout)
    dq, dk, dv = torch.autograd.grad(out, (q, k, v), g)
    if ring_size == world:
        res = sampled_check(q.detach(), k.detach(), v.detach(), g, out.detach(), dq, dk, dv, causal=True, layout=layout,
                            world=world, rank=rank, head_index=h - 1, samples=48, chunk=1024)
        assert res["ok"], res
        if memory == "ring":
            # the workspace is O(n / W): this rank's own K/V slot (double buffered), never a W-slot gather
            from ring_attention_pytorch_b200.parallel.symm import get_workspace

            regions = get_workspace(ring_size, dev).regions
            slot = 2 * n * hk * 128 * 2
            assert "kv_gather" not in regions and regions["kv_own"].nbytes <= 2 * slot + 1024, list(regions)
    else:
        # ring sets: every set is an independent ring; check inside the set through a sub-group gather
        sets = world // ring_size
        groups = [dist.new_group(list(range(s * ring_size, (s + 1) * ring_size))) for s in range(sets)]
        mine = groups[rank // ring_size]

        def gather(t):
            parts = [torch.empty_like(t) for _ in range(ring_size)]
            dist.all_gather(parts, t.contiguous(), group=mine)
            return parts

        from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
        from ring_attention_pytorch_b200.parallel.layout import make_position_map

        pm = make_position_map(layout, ring_size, n)
        ks, vs = gather(k.detach()), gather(v.detach())
        r = rank % ring_size
        rows = torch.arange(0, n, max(1, n // 64), device=dev)
        k_all, v_all = torch.cat([t.float() for t in ks], 1), torch.cat([t.float() for t in vs], 1)
        k_pos = torch.cat([pm.positions(i, dev) for i in range(ring_size)])
        ref = attention_with_positions(q.detach()[:, rows].float(), k_all, v_all, pm.positions(r, dev)[rows], k_pos,
                                       causal=True)
        assert (out.detach()[:, rows].float() - ref).abs().max() < 3e-2
        assert torch.isfinite(dq.float()).all() and torch.isfinite(dk.float()).all()
    torch.cuda.synchronize()
    dist.barrier()


@pytest.mark.parametrize("layout,hk", [("striped", 2), ("zigzag", 8)])
def test_real_ring_all_gpus_sampled_oracle(layout, hk):
    """Every visible GPU (2, 4 or 8) in one ring, 8192 tokens per rank, GQA, fwd + bwd, sampled rows vs fp32 oracle."""
    world = torch.cuda.device_count()
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    from dist_utils import run_distributed

    world = 8 if world >= 8 else (4 if world >= 4 else 2)
    run_distributed(_big_ring_worker, world, layout, 8192, 8, hk, None, backend="nccl", timeout=600.0)


@pytest.mark.parametrize("layout,hk", [("striped", 2), ("zigzag", 8)])
def test_real_ring_hop_window_memory_mode(layout, hk):
    """``CONFIG["memory"] = "ring"``: per-hop launches against a 2-slot window (copy engines one hop ahead), carried
    softmax state and accumulators; same sampled-oracle check, and the symmetric workspace stays O(n / W)."""
    world = torch.cuda.device_count()
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    from dist_utils import run_distributed

    world = 8 if world >= 8 else (4 if world >= 4 else 2)
    run_distributed(_big_ring_worker, world, layout, 8192, 8, hk, None, "ring", backend="nccl", timeout=600.0)


def test_ring_sets_two_by_four():
    """8 GPUs as 2 independent rings of 4 (reference ring.py:35-47 ring sets)."""
    if torch.cuda.device_count() < 8:
        pytest.skip("needs 8 GPUs")
    from dist_utils import run_distributed

    run_distributed(_big_ring_worker, 8, "striped", 2048, 4, 2, 4, backend="nccl", timeout=600.0)


def _stress_worker(rank, world, iters):
    """Alternating shapes: exercises the double-buffered gather workspace, the symmetric accumulators and the
    region growth / retirement path (a larger shape arrives after smaller ones)."""
    import torch.distributed as dist

    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda
    from ring_attention_pytorch_b200.parallel.symm import close_workspaces

    dev = torch.device("cuda", rank)
    shapes = [(256, 2, 2), (640, 4, 2), (384, 4, 4), (1024, 4, 1)]
    ref = {}
    for it in range(iters):
        n, h, hk = shapes[it % len(shapes)]
        torch.manual_seed(7 + rank + 1000 * (it % len(shapes)))
        q = torch.randn(1, n, h, 128, device=dev, dtype=torch.bfloat16, requires_grad=True)
        k = torch.randn(1, n, hk, 128, device=dev, dtype=torch.bfloat16, requires_grad=True)
        v = torch.randn(1, n, hk, 128, device=dev, dtype=torch.bfloat16, requires_grad=True)
        out = ring_flash_attn_cuda(q, k, v, None, True, 1024, True, True, None, world)
        dq, dk, dv = torch.autograd.grad(out, (q, k, v), out.detach())
        key = it % len(shapes)
        cur = (out.detach().float().sum().item(), dk.float().abs().sum().item(), dq.float().abs().sum().item())
        if key in ref:  # same inputs -> same results up to the (order-dependent) fp32 reductions
            for a, b2 in zip(cur, ref[key]):
                assert abs(a - b2) <= 2e-3 * max(1.0, abs(b2)), (it, cur, ref[key])
        else:
            ref[key] = cur
    torch.cuda.synchronize()
    dist.barrier()
    close_workspaces()


def test_ring_stress_alternating_shapes():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from dist_utils import run_distributed

    run_distributed(_stress_worker, 2, 200, backend="nccl", timeout=600.0)


# ------------------------------------------------------------------------------------------------
# rotary embedding inside the op's pack kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,hk", [(128, 2), (64, 4), (96, 4)])
def test_in_op_rotary_matches_eager(d, hk):
    from ring_attention_pytorch_b200 import RingRotaryEmbedding, apply_rotary_pos_emb
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda

    torch.manual_seed(0)
    b, n, h = 2, 300, 4
    q = torch.randn(b, n, h, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(b, n, hk, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(b, n, hk, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    g = torch.randn(b, n, h, d, device="cuda", dtype=torch.bfloat16)
    freqs = RingRotaryEmbedding(d).cuda()(torch.arange(n, device="cuda") * 37)  # large angles: range reduction matters
    fused = ring_flash_attn_cuda(q, k, v, None, True, rotary_freqs=freqs)
    gf = torch.autograd.grad(fused, (q, k, v), g)
    eager = ring_flash_attn_cuda(apply_rotary_pos_emb(freqs, q), apply_rotary_pos_emb(freqs, k), v, None, True)
    ge = torch.autograd.grad(eager, (q, k, v), g)
    assert (fused.float() - eager.float()).abs().max() < 2e-2
    for a, b2 in zip(gf, ge):
        assert (a.float() - b2.float()).abs().max() / b2.float().abs().max() < 3e-2


def test_rotary_module_launches_no_eager_rotary_kernels():
    """RingAttention(rotary_embed=True) on the kernel path: the only kernels touching q / k before attention are ours."""
    from torch.profiler import ProfilerActivity, profile

    from ring_attention_pytorch_b200 import RingAttention

    torch.manual_seed(0)
    attn = RingAttention(dim=256, dim_head=64, heads=4, causal=True, rotary_embed=True, ring_attn=False,
                         use_cuda_kernel=True).cuda().to(torch.bfloat16)
    x = torch.randn(2, 257, 256, device="cuda", dtype=torch.bfloat16)
    attn(x)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        attn(x)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    assert any("rotary_kernel" in nme for nme in names), names
    assert not any(("sin" in nme.lower() or "cos" in nme.lower()) and "rotary_kernel" not in nme for nme in names), names


@pytest.mark.parametrize("fp8", [False, True])
def test_tree_decode_is_cuda_graph_capturable(fp8):
    """A decode step allocates nothing and keeps its counters / epoch in device memory: capture once, replay with new
    queries, check every replay against the oracle under the noise-scaled rule."""
    from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc
    from ring_attention_pytorch_b200.ops.tree_decode_cuda import tree_decode_cuda

    gdc = _cases()
    old = dict(tdc.CONFIG)
    tdc.CONFIG["tensor_core"] = "auto"
    try:
        torch.manual_seed(0)
        b, h, hk, n, d = 4, 16, 4, 2048, 128
        q = torch.randn(b, h, 1, d, device="cuda", dtype=torch.bfloat16)
        k = torch.randn(b, hk, n, d, device="cuda", dtype=torch.bfloat16)
        v = torch.randn(b, hk, n, d, device="cuda", dtype=torch.bfloat16)
        ks = vs = None
        kk, vv = k, v
        if fp8:
            kk, vv = k.to(torch.float8_e4m3fn), v.to(torch.float8_e4m3fn)
            ks = vs = torch.ones(b * hk, device="cuda")
        out = torch.empty_like(q)
        tree_decode_cuda(q, kk, vv, dim_v=d, k_scale=ks, v_scale=vs, out=out)  # warm-up: creates the cached buffers
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            tree_decode_cuda(q, kk, vv, dim_v=d, k_scale=ks, v_scale=vs, out=out)
        for it in range(3):
            q.copy_(torch.randn_like(q))
            graph.replay()
            torch.cuda.synchronize()
            ref = gdc.decode_reference(q, kk.float(), vv.float())
            lowp = gdc.decode_reference(q, kk.float(), vv.float(), dtype=torch.bfloat16)
            res = gdc.noise_bound(out, ref, lowp, gdc.CAP_OUT)
            assert res["ok"], (it, res)
    finally:
        tdc.CONFIG.update(old)


@pytest.mark.parametrize("fp8", [False, True])
def test_tree_decode_reads_a_growing_cache_in_place(fp8):
    """k / v = filled prefix of a [b, hk, capacity, d] buffer: the tensor-core kernel reads it through the tensor map's
    plane stride (no copy).  Step after step, the result is bitwise the one of the dense copy of the same prefix (same
    kernel, same tiles, sums in the same order: only the source stride differs) and passes the noise-scaled rule."""
    from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc

    gdc = _cases()
    old = dict(tdc.CONFIG)
    tdc.CONFIG["tensor_core"] = "auto"
    try:
        torch.manual_seed(0)
        b, h, hk, d, cap = 3, 8, 2, 128, 1000
        dt = torch.float8_e4m3fn if fp8 else torch.bfloat16
        kc = (torch.randn(b, hk, cap, d, device="cuda") * (0.5 if fp8 else 1.0)).to(dt)
        vc = (torch.randn(b, hk, cap, d, device="cuda") * (0.5 if fp8 else 1.0)).to(dt)
        q = torch.randn(b, h, 1, d, device="cuda", dtype=torch.bfloat16)
        sc = torch.ones(b * hk, device="cuda") if fp8 else None
        for n in (128, 300, 777, cap):
            kp, vp = kc[:, :, :n], vc[:, :, :n]
            assert tdc._is_cache_prefix(kp) and (n == cap or not kp.is_contiguous())
            got = tdc.tree_decode_cuda(q, kp, vp, dim_v=d, k_scale=sc, v_scale=sc)
            want = tdc.tree_decode_cuda(q, kp.contiguous(), vp.contiguous(), dim_v=d, k_scale=sc, v_scale=sc)
            assert torch.equal(got, want), n
            ref = gdc.decode_reference(q, kp.float(), vp.float())
            lowp = gdc.decode_reference(q, kp.float(), vp.float(), dtype=torch.bfloat16)
            res = gdc.noise_bound(got, ref, lowp, gdc.CAP_OUT)
            assert res["ok"], (n, res)
    finally:
        tdc.CONFIG.update(old)
