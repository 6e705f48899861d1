"""fp8 (e4m3) forward for long-context prefill: ``quantize_fp8``, ``ring_flash_attn_fp8``, ``RingAttention(fp8_attn=True)``
and the sm_90a kernels behind them (``pack_kv_fp8`` and the e4m3 instantiation of the forward).

GPU tolerance: relative RMS error of ``out`` against the fp32 oracle on the dequantised inputs (N(0, 1) data, so the
only error is the kernel's: P in e4m3, S accumulated from e4m3 products, bf16 output).  Observed on one H100 80GB HBM3
(700 W power limit) over the single-GPU cases below: 1.6e-2 to 2.67e-2 for fp8, against 3.1e-3 to 4.1e-3 for the bf16
kernel on the same dequantised inputs (fp8 / bf16 ratio 5.3 to 6.6).  The 3e-2 first guess held, with little margin.
Since each tile's P is taken against its own maximum and its P V is added to O in fp32: 1.5e-2 to 2.2e-2 (ratio 4.8 to 5.5), same card.
``REL_RMS_TOL`` is 5e-2, 1.9x the worst observed value (twice it would be 5.3e-2, past the 5e-2 ceiling set for this
bound); ``BF16_RATIO_TOL`` is 13, twice the worst observed ratio, so a layout bug cannot hide behind the loose bound.
"""
import os
import sys

import pytest
import torch
import torch.distributed as dist

from dist_utils import run_distributed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

REL_RMS_TOL = 5e-2
BF16_RATIO_TOL = 13.0
LAYOUTS = ("plain", "striped", "zigzag")


def _rel_rms(got, want):
    got, want = got.float(), want.float()
    return ((got - want).norm() / want.norm().clamp_min(1e-30)).item()


def _quantized(*shapes, device="cpu", seed=0):
    """N(0, 1) tensors of the given shapes and their e4m3 quantisation: [(t8, descale), ...]."""
    from ring_attention_pytorch_b200 import quantize_fp8

    g = torch.Generator().manual_seed(seed)
    return [quantize_fp8(torch.randn(*s, generator=g).to(device), 1) for s in shapes]


def _deq(t8, ds):
    b, heads = t8.shape[0], t8.shape[2]
    return t8.float() * ds.float().expand(b, heads)[:, None, :, None]


# ================================================================================================
# CPU
# ================================================================================================
def test_quantize_fp8_round_trip_and_shapes():
    from ring_attention_pytorch_b200 import quantize_fp8

    torch.manual_seed(0)
    t = torch.randn(2, 50, 3, 16) * torch.tensor([0.01, 1.0, 300.0])[None, None, :, None]
    t8, ds = quantize_fp8(t)
    assert t8.dtype == torch.float8_e4m3fn and t8.shape == t.shape
    assert ds.dtype == torch.float32 and ds.shape == (2, 3)
    amax = t.abs().amax(dim=(1, 3))
    assert torch.allclose(ds, amax / 448)
    assert torch.equal(t8.float().abs().amax(dim=(1, 3)), torch.full((2, 3), 448.0))
    # within one e4m3 step: 2^-3 relative for normals, 2^-9 (in units of the scale) below the normal range
    err = (_deq(t8, ds) - t).abs()
    step = torch.maximum(t.abs() * 2 ** -3, ds[:, None, :, None] * 2 ** -9)
    assert (err <= step).all(), (err / step).max()


def test_quantize_fp8_zero_rows():
    from ring_attention_pytorch_b200 import quantize_fp8

    t = torch.randn(2, 10, 4, 8)
    t[1, :, 2] = 0
    t8, ds = quantize_fp8(t)
    assert ds[1, 2] == 1.0 and (t8[1, :, 2].float() == 0).all()
    assert torch.isfinite(ds).all() and (ds > 0).all()


def test_v8_key_order_makes_register_p_times_vt_equal_p_times_v():
    """Model of the two register fragments of one warp: thread quad q holds S columns {2q, 2q+1, 8+2q, 9+2q, ...} of a
    32-key group (fp32 accumulator) and feeds them, in register order, as A columns {4q..4q+3, 16+4q..16+4q+3} (e4m3
    A operand of m64nNk32).  With V^T slot kappa holding key v8_key_of_slot(kappa) the MMA computes P V exactly."""
    from ring_attention_pytorch_b200.ops.ring_fp8 import v8_key_of_slot

    assert sorted(v8_key_of_slot(k) for k in range(128)) == list(range(128))
    assert all(v8_key_of_slot(k) // 32 == k // 32 for k in range(128))
    torch.manual_seed(0)
    for group in range(4):
        p = torch.randn(32, dtype=torch.float64)  # P of one row over keys 32 group .. 32 group + 31
        v = torch.randn(32, 5, dtype=torch.float64)
        vt = torch.stack([v[v8_key_of_slot(32 * group + k) - 32 * group] for k in range(32)])
        for q in range(4):
            s_cols = [8 * j + 2 * q + e for j in range(4) for e in range(2)]  # accumulator registers, in order
            a_cols = [4 * q + i for i in range(4)] + [16 + 4 * q + i for i in range(4)]  # A operand columns, in order
            p_a = torch.zeros(32, dtype=torch.float64)
            for s_col, a_col in zip(s_cols, a_cols):
                p_a[a_col] = p[s_col]
            # the four threads of the quad each own 8 columns; together they cover the group
            mine_a = torch.zeros(32, dtype=torch.bool)
            mine_a[a_cols] = True
            mine_s = torch.zeros(32, dtype=torch.bool)
            mine_s[s_cols] = True
            assert torch.allclose((p_a[mine_a, None] * vt[mine_a]).sum(0), (p[mine_s, None] * v[mine_s]).sum(0))


@pytest.mark.parametrize("kw", [dict(causal=True), dict(causal=False), dict(causal=True, max_lookback_seq_len=9),
                                dict(softclamp_qk_sim=True, softclamp_value=5.0), dict(mask="keys"),
                                dict(causal=True, document_ids="docs")])
def test_portable_op_is_ring_flash_attn_on_dequantised_inputs(kw):
    from ring_attention_pytorch_b200 import ring_flash_attn, ring_flash_attn_fp8

    kw = dict(kw)
    b, n, h, hk, d = 2, 37, 4, 2, 16
    (q8, qd), (k8, kd), (v8, vd) = _quantized((b, n, h, d), (b, n, hk, d), (b, n, hk, d), seed=3)
    if kw.get("mask") == "keys":
        kw["mask"] = torch.rand(b, n, generator=torch.Generator().manual_seed(1)) > 0.3
    if kw.get("document_ids") == "docs":
        kw["document_ids"] = torch.tensor([[0] * 10 + [1] * 20 + [2] * 7, [5] * 37])
    out = ring_flash_attn_fp8(q8, k8, v8, qd, kd, vd, bucket_size=8, **kw)
    want = ring_flash_attn(_deq(q8, qd), _deq(k8, kd), _deq(v8, vd), bucket_size=8, **kw)
    assert out.dtype == torch.bfloat16 and out.shape == (b, n, h, d)
    assert torch.equal(out, want.to(torch.bfloat16))
    # one descale element broadcasts
    one = torch.ones(1)
    assert torch.equal(ring_flash_attn_fp8(q8, k8, v8, one, one, one, bucket_size=8, **kw),
                       ring_flash_attn(q8.float(), k8.float(), v8.float(), bucket_size=8, **kw).to(torch.bfloat16))


def test_fp8_op_value_errors():
    from ring_attention_pytorch_b200 import ring_flash_attn_fp8

    b, n, h, hk, d = 1, 8, 4, 2, 16
    (q8, qd), (k8, kd), (v8, vd) = _quantized((b, n, h, d), (b, n, hk, d), (b, n, hk, d))
    with pytest.raises(ValueError, match="float8_e4m3fn"):
        ring_flash_attn_fp8(q8.float(), k8, v8, qd, kd, vd)
    with pytest.raises(ValueError, match="float8_e4m3fn"):
        ring_flash_attn_fp8(q8, k8, v8.to(torch.float8_e5m2), qd, kd, vd)
    with pytest.raises(ValueError, match="q_descale"):
        ring_flash_attn_fp8(q8, k8, v8, kd, kd, vd)
    with pytest.raises(ValueError, match="k_descale"):
        ring_flash_attn_fp8(q8, k8, v8, qd, torch.ones(b, hk, 1), vd)
    with pytest.raises(ValueError, match="v_descale"):
        ring_flash_attn_fp8(q8, k8, v8, qd, kd, vd.double())
    with pytest.raises(ValueError, match="forward only"):
        ring_flash_attn_fp8(q8.clone().requires_grad_(), k8, v8, qd, kd, vd)
    with pytest.raises(ValueError, match="forward only"):
        ring_flash_attn_fp8(q8, k8, v8, qd, kd.clone().requires_grad_(), vd)
    with pytest.raises(ValueError, match="rotary"):
        ring_flash_attn_fp8(q8, k8, v8, qd, kd, vd, rotary_freqs=torch.zeros(n, d))


def _ring_set_scale_worker(rank, world):
    from ring_attention_pytorch_b200 import quantize_fp8

    ring_size = 2
    # rank r's tensor has amax 1 + r in every (batch, head) except where it is larger on the other set's ranks
    t = torch.full((2, 6, 3, 4), 1.0 + rank)
    t[0, 0, 0, 0] = -10.0 * (rank + 1)
    _, ds = quantize_fp8(t, ring_size)
    set_ranks = range(rank // ring_size * ring_size, rank // ring_size * ring_size + ring_size)
    want = torch.full((2, 3), max(1.0 + r for r in set_ranks)) / 448
    want[0, 0] = max(10.0 * (r + 1) for r in set_ranks) / 448
    assert torch.allclose(ds, want), (rank, ds, want)
    everyone = [torch.empty_like(ds) for _ in range(world)]
    dist.all_gather(everyone, ds)
    for r in set_ranks:
        assert torch.equal(everyone[r], ds)
    other = everyone[(rank + ring_size) % world]
    assert not torch.equal(other, ds)
    _, local = quantize_fp8(t, 1)
    assert torch.allclose(local, t.abs().amax(dim=(1, 3)) / 448)


def test_quantize_fp8_scales_are_shared_within_a_ring_set_only():
    run_distributed(_ring_set_scale_worker, 4)


def _module_worker(rank, world, striped, docs):
    from math import ceil

    from ring_attention_pytorch_b200 import RingAttention

    torch.manual_seed(0)
    seq_len = 45
    ring_seq_size = ceil(seq_len / world)
    kw = dict(dim=32, dim_head=16, heads=4, num_grouped_query_heads=2, causal=True, bucket_size=ring_seq_size,
              use_cuda_kernel=False)
    ref = RingAttention(ring_attn=True, striped_ring_attn=striped, ring_seq_size=ring_seq_size, **kw)
    ring8 = RingAttention(ring_attn=True, striped_ring_attn=striped, ring_seq_size=ring_seq_size, fp8_attn=True, **kw)
    ring8.load_state_dict(ref.state_dict())
    torch.manual_seed(100)
    x = torch.randn(2, seq_len, 32)
    ids = torch.tensor([[0] * 9 + [1] * 3 + [0] * 11 + [4] * 22, [2] * 1 + [3] * 20 + [5] * 24]) if docs else None
    with torch.no_grad():
        want = ref(x, document_ids=ids)
        got = ring8(x, document_ids=ids)
    assert got.shape == want.shape
    assert _rel_rms(got, want) < 0.05, _rel_rms(got, want)
    with pytest.raises(ValueError, match="no_grad"):
        ring8(x, document_ids=ids)


@pytest.mark.parametrize("striped,docs", [(False, False), (True, False), (False, True), (True, True)])
def test_ring_attention_fp8_module_matches_bf16_module_on_gloo(striped, docs):
    run_distributed(_module_worker, 4, striped, docs)


def test_ring_transformer_threads_fp8_attn():
    from ring_attention_pytorch_b200 import RingTransformer

    torch.manual_seed(0)
    kw = dict(num_tokens=64, dim=32, depth=2, causal=True, dim_head=16, heads=2, use_cuda_kernel=False)
    ref, m8 = RingTransformer(**kw), RingTransformer(fp8_attn=True, **kw)
    m8.load_state_dict(ref.state_dict())
    assert all(layer[0].fp8_attn for layer in m8.layers) and not any(layer[0].fp8_attn for layer in ref.layers)
    tokens = torch.randint(0, 64, (2, 40))
    with torch.no_grad():
        assert _rel_rms(m8(tokens), ref(tokens)) < 0.05
    with pytest.raises(ValueError, match="no_grad"):
        m8(tokens)


# ================================================================================================
# GPU: pack_kv_fp8 and the e4m3 forward kernel
# ================================================================================================
def _pack_reference(k8, v8):
    """Torch model of pack_kv_fp8: uint8 [2, b*hk, n_pad, 128]."""
    from ring_attention_pytorch_b200.ops.ring_fp8 import v8_key_of_slot

    b, n, hk, d = k8.shape
    n_pad = (n + 127) // 128 * 128
    kb, vb = (torch.zeros(b * hk, n_pad, d, dtype=torch.uint8, device=k8.device) for _ in range(2))
    kb[:, :n] = k8.view(torch.uint8).permute(0, 2, 1, 3).reshape(b * hk, n, d)
    vb[:, :n] = v8.view(torch.uint8).permute(0, 2, 1, 3).reshape(b * hk, n, d)
    order = torch.tensor([v8_key_of_slot(kk) for kk in range(128)], device=k8.device)
    tiles = vb.view(b * hk, n_pad // 128, 128, d)[:, :, order]  # [bh, tile, slot, d]
    vt = tiles.transpose(2, 3).reshape(b * hk, n_pad, d)        # [bh, tile * 128 + d row, slot]
    return torch.stack((kb, vt))


@pytest.mark.gpu
def test_pack_kv_fp8_byte_exact():
    from ring_attention_pytorch_b200.ops.fused import alloc_kv_buffer_fp8, pack_kv_fp8

    b, n, hk, d = 2, 1000, 3, 128
    torch.manual_seed(0)
    # strided inputs (a slice of a fused kv projection), and NaN-free garbage in the slot before packing
    kv = (torch.randn(b, n, 2 * hk, d, device="cuda") * 40).to(torch.float8_e4m3fn)
    k8, v8 = kv[:, :, :hk], kv[:, :, hk:]
    slot = alloc_kv_buffer_fp8(1, b, hk, n, "cuda")[0]
    slot.fill_(0x7F)  # 0x7f is NaN in e4m3: the padded keys must be overwritten with zeros
    pack_kv_fp8(k8, v8, slot)
    want = _pack_reference(k8, v8)
    assert slot.shape == want.shape
    assert torch.equal(slot, want)
    assert (slot[0, :, n:] == 0).all()  # K rows of the padded keys
    last = slot[1, :, -128:].view(-1, 128, 128)  # V^T of the last tile: [d row][key slot]
    from ring_attention_pytorch_b200.ops.ring_fp8 import v8_key_of_slot
    pad = torch.tensor([v8_key_of_slot(kk) >= n % 128 for kk in range(128)], device="cuda")
    assert (last[:, :, pad] == 0).all() and (last[:, :, ~pad] != 0).any()


def _oracle_case(b=1, n=1000, h=2, hk=None, causal=False, window=None, kmask=False, softclamp=0.0, docs=False,
                 n_k=None, seed=0):
    """Single-GPU fp8 forward vs the fp32 oracle and vs the bf16 kernel on the same dequantised inputs."""
    from ring_attention_pytorch_b200 import ring_flash_attn_fp8
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda
    from ring_attention_pytorch_b200.parallel.documents import document_runs

    hk = hk or h
    n_k = n_k or n
    d = 128
    (q8, qd), (k8, kd), (v8, vd) = _quantized((b, n, h, d), (b, n_k, hk, d), (b, n_k, hk, d), device="cuda", seed=seed)
    mask = (torch.rand(b, n_k, generator=torch.Generator().manual_seed(seed)) > 0.25).cuda() if kmask else None
    ids = None
    if docs:
        ids = torch.cumsum(torch.rand(b, n, generator=torch.Generator().manual_seed(seed)) < 0.01, 1).cuda()
    kw = dict(causal=causal, max_lookback_seq_len=window, softclamp_qk_sim=softclamp > 0,
              softclamp_value=softclamp or 50.0, document_ids=ids)
    out = ring_flash_attn_fp8(q8, k8, v8, qd, kd, vd, mask, **kw)
    qf, kf, vf = _deq(q8, qd), _deq(k8, kd), _deq(v8, vd)
    runs = document_runs(ids) if docs else None
    ref = attention_with_positions(qf, kf, vf, causal=causal, window=window, key_mask=None if causal else mask,
                                   softclamp_value=softclamp, q_doc=runs, k_doc=runs)
    with torch.no_grad():
        out16 = ring_flash_attn_cuda(qf.bfloat16(), kf.bfloat16(), vf.bfloat16(), mask, **kw)
    torch.cuda.synchronize()
    assert out.dtype == torch.bfloat16 and out.shape == (b, n, h, d)
    assert torch.isfinite(out).all()
    return _rel_rms(out, ref), _rel_rms(out16, ref)


ORACLE_CASES = {
    "causal_n1000": dict(causal=True),
    "noncausal_n1000": dict(),
    "gqa8_2_causal_n4096": dict(n=4096, h=8, hk=2, causal=True),
    "noncausal_n4096_b2": dict(n=4096, b=2, h=4, hk=2),
    "kmask": dict(b=2, kmask=True),
    "window": dict(n=4096, causal=True, window=700),
    "softclamp_causal": dict(causal=True, softclamp=20.0),
    "documents_causal": dict(n=4096, causal=True, docs=True),
    "documents_noncausal_gqa": dict(h=4, hk=2, docs=True),
    "cross_attention_causal": dict(n=700, n_k=1000, causal=True),
    "cross_attention_causal_more_queries": dict(n=1000, n_k=300, causal=True),
    "cross_attention_kmask": dict(n=300, n_k=1000, kmask=True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ORACLE_CASES))
def test_fp8_forward_matches_oracle(name):
    err8, err16 = _oracle_case(**ORACLE_CASES[name])
    print(f"[fp8] {name}: rel_rms fp8 {err8:.3e}, bf16 {err16:.3e}, ratio {err8 / err16:.2f}")
    assert err8 <= REL_RMS_TOL, (err8, err16)
    assert err8 <= BF16_RATIO_TOL * err16, (err8, err16)


@pytest.mark.gpu
def test_fp8_op_rejects_head_dim_64_on_the_kernel_path():
    from ring_attention_pytorch_b200 import ring_flash_attn_fp8

    (q8, qd), (k8, kd), (v8, vd) = _quantized((1, 128, 2, 64), (1, 128, 2, 64), (1, 128, 2, 64), device="cuda")
    with pytest.raises(ValueError, match="head dim 128"):
        ring_flash_attn_fp8(q8, k8, v8, qd, kd, vd)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("hopwise", [False, True])
def test_fp8_emulated_ring_matches_oracle(world, layout, hopwise):
    from ring_attention_pytorch_b200.ops.fused import emulate_ring_forward_fp8
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    b, n, h, hk, d = 1, 384, 4, 2, 128
    causal = layout != "plain" or world == 4
    pm = make_position_map(layout, world, n)
    # ring-wide K/V scales, per-rank Q scales
    (kall, kd), (vall, vd) = _quantized((b, world * n, hk, d), (b, world * n, hk, d), device="cuda", seed=world)
    qs = _quantized(*[(b, n, h, d)] * world, device="cuda", seed=10 + world)
    ks = [kall[:, pm.positions(r, "cuda")] for r in range(world)]
    vs = [vall[:, pm.positions(r, "cuda")] for r in range(world)]
    outs, _ = emulate_ring_forward_fp8([q for q, _ in qs], ks, vs, [s for _, s in qs], kd, vd, layout=layout,
                                       causal=causal, hopwise=hopwise)
    k_pos = torch.cat([pm.positions(r, "cuda") for r in range(world)])
    kf, vf = _deq(torch.cat(ks, 1), kd), _deq(torch.cat(vs, 1), vd)
    for r in range(world):
        ref = attention_with_positions(_deq(*qs[r]), kf, vf, pm.positions(r, "cuda"), k_pos, causal=causal)
        assert torch.isfinite(outs[r]).all()
        err = _rel_rms(outs[r], ref)
        assert err <= REL_RMS_TOL, (r, err)


@pytest.mark.gpu
def test_fp8_hopwise_equals_gather():
    """The per-hop launches carry an unscaled O and apply v_descale once: same result as the one-launch ring."""
    from ring_attention_pytorch_b200.ops.fused import emulate_ring_forward_fp8

    world, b, n, h, d = 4, 1, 256, 2, 128
    (kall, kd), (vall, vd) = _quantized((b, world * n, h, d), (b, world * n, h, d), device="cuda", seed=5)
    qs = _quantized(*[(b, n, h, d)] * world, device="cuda", seed=6)
    args = ([q for q, _ in qs], list(kall.split(n, 1)), list(vall.split(n, 1)), [s for _, s in qs], kd * 3, vd * 5)
    a, _ = emulate_ring_forward_fp8(*args, causal=True)
    g, _ = emulate_ring_forward_fp8(*args, causal=True, hopwise=True)
    for x, y in zip(a, g):
        assert (x.float() - y.float()).abs().max() <= 1e-2 * y.float().abs().max()


def _real_ring_fp8_worker(rank, world, memory):
    from ring_attention_pytorch_b200 import quantize_fp8, ring_flash_attn_fp8
    from ring_attention_pytorch_b200.ops import ring_cuda
    from ring_attention_pytorch_b200.ops.fused import emulate_ring_forward_fp8
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    ring_cuda.CONFIG["memory"] = memory
    dev = torch.device("cuda", rank)
    b, n, h, hk, d = 1, 640, 4, 2, 128
    torch.manual_seed(0)
    full = [torch.randn(b, world * n, heads, d) for heads in (h, hk, hk)]
    pm = make_position_map("striped", world, n)
    mine = [t[:, pm.positions(rank)].to(dev) for t in full]
    (q8, qd), (k8, kd), (v8, vd) = (quantize_fp8(t, world) for t in mine)
    out = ring_flash_attn_fp8(q8, k8, v8, qd, kd, vd, None, True, 1024, True, True, None, world)
    # every rank replays the whole ring on its own GPU from the same quantised shards
    shards = [[None] * world for _ in range(4)]
    for i, t in enumerate((q8.view(torch.uint8), qd, k8.view(torch.uint8), v8.view(torch.uint8))):
        gathered = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(gathered, t.contiguous())
        shards[i] = gathered
    qs = [t.view(torch.float8_e4m3fn) for t in shards[0]]
    ks = [t.view(torch.float8_e4m3fn) for t in shards[2]]
    vs = [t.view(torch.float8_e4m3fn) for t in shards[3]]
    outs, _ = emulate_ring_forward_fp8(qs, ks, vs, shards[1], kd, vd, layout="striped", causal=True,
                                       hopwise=memory == "ring")
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    assert torch.equal(out, outs[rank])
    dist.barrier()


@pytest.mark.gpu
@pytest.mark.parametrize("memory", ["gather", "ring"])
def test_fp8_real_ring_matches_emulated_ring(memory):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    run_distributed(_real_ring_fp8_worker, 2, memory, backend="nccl", timeout=600.0)


@pytest.mark.gpu
def test_ring_attention_fp8_module_on_kernels():
    from ring_attention_pytorch_b200 import RingAttention

    torch.manual_seed(0)
    kw = dict(dim=256, dim_head=128, heads=4, num_grouped_query_heads=2, causal=True, rotary_embed=True)
    ref = RingAttention(use_cuda_kernel=True, **kw).cuda()
    m8 = RingAttention(use_cuda_kernel=True, fp8_attn=True, **kw).cuda()
    m8.load_state_dict(ref.state_dict())
    x = torch.randn(2, 700, 256, device="cuda")
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        want = ref(x)
        got = m8(x)
    assert torch.isfinite(got).all()
    assert _rel_rms(got, want) < 0.1, _rel_rms(got, want)
    with pytest.raises(ValueError, match="no_grad"):
        m8(x)
