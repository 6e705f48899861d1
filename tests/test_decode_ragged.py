"""Ragged and windowed tree decode: per-sequence cache lengths, query positions with a look-back window, and softclamp.

Local key ``j`` of sequence ``b`` sits at global position ``P(j) = offset + stride * j`` and is visible iff
``j < min(cache_seqlens[b], n)``, ``P(j) <= q_pos[b]`` and (window > 0) ``q_pos[b] - P(j) <= window``.

CPU: the portable path on gloo worlds of 1, 2 and 4 (chunked and round-robin shards) against ``attention_with_positions``
in fp64; a hypothesis property test of the kernels' unit-range arithmetic (a Python mirror of ``td_unit_range``); the
example's ragged / windowed loop; argument validation.

GPU: both kernels against the oracle under the noise-scaled rule, with everything outside the visible ranges NaN (0x7F
in e4m3); bitwise identity with the plain call when every length is ``n``; per-sequence calls on sliced caches; CUDA
graph replays with the lengths and positions advanced in place; real rings of 2 and 8 GPUs.
"""
import os
import sys

import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "examples"))

import gpu_dev_check as gdc  # noqa: E402
from dist_utils import run_distributed  # noqa: E402

from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc  # noqa: E402
from ring_attention_pytorch_b200.ops.oracle import attention_with_positions  # noqa: E402

TILE = 64


def visible(n, lens, q_pos, window, offset=0, stride=1):
    """bool [b, n] by the definition above (lens / q_pos: int tensors [b] or None)."""
    b = next((t.shape[0] for t in (lens, q_pos) if t is not None), 1)
    j = torch.arange(n)
    vis = torch.ones(b, n, dtype=torch.bool)
    if lens is not None:
        vis &= j[None] < lens.long().cpu()[:, None]
    if q_pos is not None:
        rel = q_pos.long().cpu()[:, None] - (offset + stride * j)[None]
        vis &= rel >= 0
        if window is not None and window > 0:
            vis &= rel <= window
    return vis


def reference(q, k, v, vis, softclamp=0.0, sinks=None, dtype=torch.float64):
    """q [b, h, 1, d], k / v [b, hk, n, d] (clean values), vis [b, n] -> [b, h, 1, d] through the oracle."""
    outs = []
    for i in range(q.shape[0]):
        o = attention_with_positions(q[i:i + 1].transpose(1, 2).to(dtype), k[i:i + 1].transpose(1, 2).to(dtype),
                                     v[i:i + 1].transpose(1, 2).to(dtype), key_mask=vis[i:i + 1].to(q.device),
                                     softclamp_value=softclamp, sinks=None if sinks is None else sinks.to(dtype))
        outs.append(o.transpose(1, 2))
    return torch.cat(outs)


def nan_fill_invisible(t, vis):
    """A copy of the cache t [b, hk, n, d] with every invisible key NaN (0x7F in e4m3)."""
    t = t.clone()
    mask = ~vis.to(t.device)[:, None, :, None].expand(t.shape)
    if t.dtype == torch.float8_e4m3fn:
        t.view(torch.uint8)[mask] = 0x7F
    else:
        t[mask] = float("nan")
    return t


# ================================================================================================
# CPU: the portable path
# ================================================================================================
N_GLOBAL = 300
LENS = [0, 1, 65, 300, 129, 200]
# (window, softclamp, sinks); q_pos: the last key, except a query past the cache, one before most shards and -1
CASES = [(None, 0.0, False), (5, 0.0, False), (100, 0.0, True), (None, 8.0, False), (37, 5.0, True), (64, 0.0, False)]


def _portable_case(seed, h=4, hk=2, d=16):
    g = torch.Generator().manual_seed(seed)
    b = len(LENS)
    q = torch.randn(b, h, 1, d, generator=g, dtype=torch.float64)
    k = torch.randn(b, hk, N_GLOBAL, d, generator=g, dtype=torch.float64)
    v = torch.randn(b, hk, N_GLOBAL, d, generator=g, dtype=torch.float64)
    lens = torch.tensor(LENS, dtype=torch.int32)
    q_pos = (lens - 1).long()
    q_pos[2], q_pos[4], q_pos[5] = 65 + 40, 1, -1
    return q, k, v, lens, q_pos


def _portable_worker(rank, world, shard):
    from ring_attention_pytorch_b200 import tree_attn_decode

    for ci, (window, clamp, with_sinks) in enumerate(CASES):
        for h, hk in ((4, 2), (8, 8)):
            q, k, v, lens, q_pos = _portable_case(ci, h, hk)
            sinks = torch.linspace(-2.0, 3.0, h) if with_sinks else None
            vis = visible(N_GLOBAL, lens, q_pos, window)
            ref = reference(q, k, v, vis, clamp, sinks)
            kn, vn = nan_fill_invisible(k, vis), nan_fill_invisible(v, vis)
            kw = dict(q_pos=q_pos, window=window, softclamp_value=clamp, sinks=sinks)
            if shard:
                out = tree_attn_decode(q.float(), kn.float(), vn.float(), cache_seqlens=lens, **kw)
            else:  # round-robin: global key t lives on rank t % world at local slot t // world
                kl, vl = kn[:, :, rank::world].float().contiguous(), vn[:, :, rank::world].float().contiguous()
                local = ((lens.long() - rank + world - 1).clamp(min=0) // world).to(torch.int32)
                out = tree_attn_decode(q.float(), kl, vl, shard_kv_seq=False, cache_seqlens=local, kv_pos=(rank, world),
                                       **kw)
            assert torch.isfinite(out).all(), (rank, ci)
            err = (out.double() - ref).abs().max().item()
            assert err < 1e-5, (rank, world, shard, ci, h, err)
            if sinks is None:  # sequence 0 holds no key, sequence 5 queries position -1: exactly zero
                assert torch.equal(out[0], torch.zeros_like(out[0])) and torch.equal(out[5], torch.zeros_like(out[5]))


@pytest.mark.parametrize("shard", [True, False])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_portable_ragged_windowed_decode(world, shard):
    """Lengths 0, 1 and not multiples of 64, windows below a tile and across shard boundaries, a query before a rank's
    first key, softclamp, sinks, GQA and rows empty on every rank; the invisible keys hold NaN."""
    if world == 1:
        _portable_worker(0, 1, shard)
    else:
        run_distributed(_portable_worker, world, shard)


def test_portable_new_arguments_at_defaults_are_bitwise_unchanged():
    from ring_attention_pytorch_b200 import tree_attn_decode

    q, k, v, _, _ = _portable_case(0)
    q, k, v = q.float(), k.float(), v.float()
    assert torch.equal(tree_attn_decode(q, k, v), tree_attn_decode(q, k, v, cache_seqlens=None, q_pos=None,
                                                                     window=None, softclamp_value=0.0, kv_pos=None))


def test_invalid_decode_ranges_raise():
    from ring_attention_pytorch_b200 import tree_attn_decode

    q, k, v, lens, q_pos = _portable_case(0)
    q, k, v = q.float(), k.float(), v.float()
    bad = [dict(window=8), dict(cache_seqlens=lens.long()), dict(cache_seqlens=lens[:3]), dict(q_pos=q_pos.float()),
           dict(q_pos=q_pos[:, None]), dict(q_pos=q_pos, window=-1), dict(softclamp_value=-1.0),
           dict(q_pos=q_pos, kv_pos=(0, 1)), dict(cache_seqlens=lens.to("meta"))]
    for kw in bad:
        with pytest.raises(ValueError):
            tree_attn_decode(q, k, v, **kw)
    for kv_pos in ((-1, 1), (0, 0)):
        with pytest.raises(ValueError):
            tree_attn_decode(q, k, v, shard_kv_seq=False, q_pos=q_pos, kv_pos=kv_pos)


def _needs_kv_pos_worker(rank, world):
    from ring_attention_pytorch_b200 import tree_attn_decode

    q, k, v, lens, q_pos = _portable_case(0)
    with pytest.raises(ValueError):
        tree_attn_decode(q.float(), k.float(), v.float(), shard_kv_seq=False, q_pos=q_pos)


def test_sharded_q_pos_needs_kv_pos():
    run_distributed(_needs_kv_pos_worker, 2)


# ================================================================================================
# CPU: the unit-range arithmetic of the kernels (mirror of tree_decode_common.cuh:td_unit_range)
# ================================================================================================
def _floor_div(a, b):
    return a // b  # Python's // floors for either sign, like td_floor_div


def unit_range(n, splits, length, q_pos, window, offset, stride, split):
    """(lo, k0, k1) of unit (b, split), as the kernels compute it (C integer arithmetic on non-negative operands)."""
    lo, hi = 0, n
    if length is not None:
        hi = min(hi, length)
    span = n
    if q_pos is not None:
        rel = q_pos - offset
        hi = min(hi, _floor_div(rel, stride) + 1)
        if window is not None and window > 0:
            lo = max(lo, -_floor_div(window - rel, stride))
            span = min(span, window // stride + TILE)
    lo = min(lo, n)
    per = ((span + splits - 1) // splits + TILE - 1) // TILE * TILE
    k0 = min((lo & ~(TILE - 1)) + split * per, n)
    k1 = max(min(hi, k0 + per), k0) if lo < hi else k0
    return lo, k0, k1


def test_python_span_matches_kernel_mirror():
    for n, window, stride in ((5000, None, 1), (5000, 4096, 1), (5000, 100, 8), (10, 4096, 1), (131072, 4096, 8)):
        span = tdc.decode_span(n, window, stride)
        assert span == (n if window is None else min(n, window // stride + TILE))


def _check_units(n, length, q_pos, window, offset, stride, splits):
    vis = visible(n, None if length is None else torch.tensor([length]),
                  None if q_pos is None else torch.tensor([q_pos]), window, offset, stride)[0]
    covered = torch.zeros(n, dtype=torch.int64)
    for s in range(splits):
        lo, k0, k1 = unit_range(n, splits, length, q_pos, window, offset, stride, s)
        assert 0 <= k0 <= k1 <= n
        if k0 < k1:
            assert k0 % TILE == 0 and lo <= k1 - 1  # tiles start on 64-key boundaries; clamped loads stay in [lo, k1)
            covered[max(k0, lo):k1] += 1
    assert torch.equal(covered, vis.long()), (n, length, q_pos, window, offset, stride, splits)


def test_unit_ranges_property():
    """Every visible key is covered by exactly one unit, no unit reaches outside [0, n) and every tile start is a
    multiple of 64, over random lengths, positions, windows, position maps and split counts."""
    hyp = pytest.importorskip("hypothesis")
    st = hyp.strategies

    @hyp.settings(max_examples=400, deadline=None)
    @hyp.given(n=st.integers(1, 3000), length=st.one_of(st.none(), st.integers(-5, 3100)),
               q_pos=st.one_of(st.none(), st.integers(-300, 30000)), window=st.one_of(st.none(), st.integers(0, 4000)),
               offset=st.integers(0, 3000), stride=st.integers(1, 9), splits=st.integers(1, 80))
    def prop(n, length, q_pos, window, offset, stride, splits):
        if q_pos is None:
            window = None
        _check_units(n, length, q_pos, window, offset, stride, splits)

    prop()


def test_unit_ranges_edge_cases():
    for args in ((64, 64, 63, None, 0, 1, 1), (65, 65, 64, 0, 0, 1, 3), (1000, 1000, 999, 5, 0, 1, 7),
                 (1000, 1000, 2, 10, 3, 1, 4), (200, 200, 700, 90, 5, 4, 2), (4099, 3000, 5000, 4096, 0, 1, 1),
                 (128, 0, 10, None, 0, 1, 2), (128, 128, -1, 3, 0, 1, 2)):
        _check_units(*args)


def test_windowed_splits_cover_order_window_keys():
    """With a window the splits are planned over window / stride + 64 keys, whatever n is."""
    n, window, splits = 131072, 4096, 4
    for q_pos in (131071, 70000, 5000):
        tiles = 0
        for s in range(splits):
            lo, k0, k1 = unit_range(n, splits, n, q_pos, window, 0, 1, s)
            tiles += -(-(k1 - k0) // TILE)
        assert tiles <= window // TILE + 2, (q_pos, tiles)


# ================================================================================================
# CPU: the example
# ================================================================================================
def _example_worker(rank, world, argv, out_path):
    import decode_tree_attention as ex

    worst = ex.run(ex.parse_args(argv))
    if rank == 0:
        torch.save(torch.tensor(worst), out_path)


@pytest.mark.parametrize("world,context,window", [(2, 301, 37), (4, 3, 2)])
def test_decode_example_ragged_windowed(tmp_path, world, context, window):
    """World 4 with context 3: every prompt is shorter than the world."""
    out = tmp_path / "err.pt"
    run_distributed(_example_worker, world, ["--device", "cpu", "--context", str(context), "--batch", "4", "--heads",
                                             "4", "--kv-heads", "2", "--dim-head", "16", "--steps", "9", "--check",
                                             "--ragged", "--window", str(window)], str(out))
    assert torch.load(out).item() < 1e-4


# ================================================================================================
# GPU
# ================================================================================================
@pytest.fixture
def decode_config():
    old = dict(tdc.CONFIG)
    yield tdc.CONFIG
    tdc.CONFIG.clear()
    tdc.CONFIG.update(old)


def _gpu_case(cache, b_lens, h, hk, n, d, seed=0):
    import test_decode_kernels as tdk

    q, k, v = tdk.make_inputs(None, len(b_lens), h, hk, n, d, seed=seed)
    cc = tdk.make_cache(cache, q, k, v, seed=seed)
    return cc, cc["q"].to(torch.float16 if cache == "fp16" else torch.bfloat16)


def _run_ranged(kernel, cache, d, h, hk, n, lens, q_pos, window, clamp, with_sinks, kv_pos=(0, 1), seed=0, tag=""):
    cc, qc = _gpu_case(cache, lens, h, hk, n, d, seed)
    lens_t = torch.tensor(lens, dtype=torch.int32, device="cuda")
    qpos_t = None if q_pos is None else torch.tensor(q_pos, dtype=torch.int32, device="cuda")
    vis = visible(n, lens_t, qpos_t, window, *kv_pos)
    sinks = gdc.make_sinks("mix", [qc.transpose(1, 2)], [cc["kd"].transpose(1, 2)], clamp) if with_sinks else None
    kn, vn = nan_fill_invisible(cc["k"], vis), nan_fill_invisible(cc["v"], vis)
    out = tdc.tree_decode_cuda(qc, kn, vn, dim_v=d, k_scale=cc["k_scale"], v_scale=cc["v_scale"],
                               scale_block_keys=cc["block"], sinks=sinks, cache_seqlens=lens_t, q_pos=qpos_t,
                               window=window, kv_pos=kv_pos, softclamp_value=clamp)
    ref = reference(qc, cc["kd"], cc["vd"], vis, clamp, sinks, dtype=torch.float32)
    lowp = reference(qc, cc["kd"], cc["vd"], vis, clamp, sinks, dtype=cc["lowp"])
    res = gdc.noise_bound(out, ref, lowp, gdc.CAP_OUT)
    print(f"[ranged {tag} {kernel} {cache} d {d} g {h // hk} n {n} window {window} clamp {clamp} sinks {with_sinks}] "
          f"err {res['err']:.3e} bound {res['bound']:.3e} ratio {res['ratio']:.3f}")
    assert torch.isfinite(out.float()).all() and res["ok"], res
    return out


GPU_CASES = []
for _kern, _d in (("on", 128), ("off", 128), ("off", 64)):
    for _cache in ("bf16", "fp16", "fp8", "fp8_b128"):
        GPU_CASES.append((_kern, _cache, _d, 8, 2, None, 0.0, False))
        GPU_CASES.append((_kern, _cache, _d, 8, 2, 300, 0.0, True))
    for _g, _hk in ((1, 4), (4, 2), (8, 1), (16, 2)):
        GPU_CASES.append((_kern, "bf16", _d, _g * _hk, _hk, 200, 20.0, False))
    GPU_CASES.append((_kern, "fp8_b128", _d, 10, 2, 77, 10.0, True))


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=lambda c: "-".join(str(x) for x in c))
def test_ranged_decode_kernels(case, decode_config):
    """Ragged lengths incl. 0 and 1, a query past its cache and one before every key, windows whose first visible key is
    not 64-aligned, softclamp and sinks; every invisible key holds NaN (0x7F in e4m3)."""
    kernel, cache, d, h, hk, window, clamp, with_sinks = case
    decode_config["tensor_core"] = kernel
    n = 1500
    lens = [0, 1, 700, 1500, 1001, 64, 1200]
    q_pos = [x - 1 for x in lens]
    q_pos[2], q_pos[6] = 900, -1
    _run_ranged(kernel, cache, d, h, hk, n, lens, q_pos, window, clamp, with_sinks)
    # a strided position map (round-robin shard of rank 3 in a world of 5), lengths only, and positions only
    _run_ranged(kernel, cache, d, h, hk, n, lens, [5 * x for x in lens], window, clamp, with_sinks, kv_pos=(3, 5))
    _run_ranged(kernel, cache, d, h, hk, n, lens, None, None, clamp, with_sinks)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["on", "off"])
@pytest.mark.parametrize("cache", ["bf16", "fp8_b128"])
def test_full_lengths_are_bitwise_the_plain_call(kernel, cache, decode_config):
    decode_config["tensor_core"] = kernel
    b, h, hk, n, d = 3, 12, 2, 5000, 128
    cc, qc = _gpu_case(cache, [0] * b, h, hk, n, d, seed=5)
    kw = dict(dim_v=d, k_scale=cc["k_scale"], v_scale=cc["v_scale"], scale_block_keys=cc["block"])
    plain = tdc.tree_decode_cuda(qc, cc["k"], cc["v"], **kw).clone()
    full = tdc.tree_decode_cuda(qc, cc["k"], cc["v"], cache_seqlens=torch.full((b,), n, dtype=torch.int32,
                                                                                 device="cuda"), **kw)
    assert torch.equal(plain, full)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["on", "off"])
def test_ragged_batch_matches_per_sequence_calls(kernel, decode_config):
    decode_config["tensor_core"] = kernel
    h, hk, n, d = 8, 2, 3000, 128
    lens = [3000, 1, 1777, 64, 2049]
    cc, qc = _gpu_case("bf16", lens, h, hk, n, d, seed=7)
    out = tdc.tree_decode_cuda(qc, cc["k"], cc["v"], dim_v=d,
                               cache_seqlens=torch.tensor(lens, dtype=torch.int32, device="cuda"))
    for i, L in enumerate(lens):
        one = tdc.tree_decode_cuda(qc[i:i + 1], cc["k"][i:i + 1, :, :L], cc["v"][i:i + 1, :, :L], dim_v=d)
        kd, vd = cc["kd"][i:i + 1, :, :L], cc["vd"][i:i + 1, :, :L]
        ref = gdc.decode_reference(qc[i:i + 1], kd, vd)
        lowp = gdc.decode_reference(qc[i:i + 1], kd, vd, dtype=torch.bfloat16)
        res = gdc.noise_bound(out[i:i + 1], ref, lowp, gdc.CAP_OUT)
        res1 = gdc.noise_bound(one, ref, lowp, gdc.CAP_OUT)
        assert res["ok"] and res1["ok"], (i, res, res1)
        assert (out[i:i + 1].float() - one.float()).abs().max().item() <= 2 * res["bound"]


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["on", "off"])
def test_cuda_graph_replay_advances_lengths_in_place(kernel, decode_config):
    """Capture one step; advance ``cache_seqlens`` and ``q_pos`` in place and replay: each replay is bitwise the eager
    call on the same inputs."""
    decode_config["tensor_core"] = kernel
    b, h, hk, n, d, window = 4, 16, 4, 4096, 128, 1000
    cc, qc = _gpu_case("bf16", [0] * b, h, hk, n, d, seed=9)
    lens = torch.tensor([100, 1, 2000, 3000], dtype=torch.int32, device="cuda")
    q_pos = (lens - 1).clone()
    out = torch.empty(b, h, 1, d, device="cuda", dtype=qc.dtype)
    kw = dict(dim_v=d, cache_seqlens=lens, q_pos=q_pos, window=window, softclamp_value=30.0)
    tdc.tree_decode_cuda(qc, cc["k"], cc["v"], out=out, **kw)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        tdc.tree_decode_cuda(qc, cc["k"], cc["v"], out=out, **kw)
    for step in range(5):
        lens.add_(37)
        q_pos.add_(37)
        graph.replay()
        torch.cuda.synchronize()
        got = out.clone()
        want = tdc.tree_decode_cuda(qc, cc["k"], cc["v"], **kw)
        assert torch.equal(got, want), step


def _real_ring_worker(rank, world, window):
    from ring_attention_pytorch_b200 import tree_attn_decode

    dev = torch.device("cuda", rank)
    g = torch.Generator().manual_seed(3)
    b, h, hk, d, cap = 5, 8, 2, 128, 700
    lens = torch.tensor([0, 1, 3 * world + 1, cap * world - 3, 1000])  # global lengths
    q = torch.randn(b, h, 1, d, generator=g)
    kg, vg = torch.randn(b, hk, cap * world, d, generator=g), torch.randn(b, hk, cap * world, d, generator=g)
    q_pos = lens - 1
    vis = visible(cap * world, lens, q_pos, window)
    ref = reference(q, kg, vg, vis)
    kl = kg[:, :, rank::world].to(dev, torch.bfloat16).contiguous()
    vl = vg[:, :, rank::world].to(dev, torch.bfloat16).contiguous()
    local = ((lens - rank + world - 1).clamp(min=0) // world).to(dev, torch.int32)
    out = tree_attn_decode(q.to(dev, torch.bfloat16), kl, vl, shard_kv_seq=False, cache_seqlens=local,
                           q_pos=q_pos.to(dev), window=window, kv_pos=(rank, world))
    assert (out.double().cpu() - ref).abs().max() < 2e-2, rank
    dist.barrier()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("window", [None, 333])
def test_real_ring_ragged_windowed(world, window):
    """Round-robin shards on a real ring; the merge is NVLS where the NVSwitch offers multicast, P2P otherwise."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    run_distributed(_real_ring_worker, world, window, backend="nccl", timeout=600.0)
