"""Paged KV caches in tree decode: ``k`` / ``v`` are page pools ``[num_pages, hk, page_size, d]`` (or NHD pools seen
through ``.transpose(1, 2)``) and ``block_table [b, max_pages]`` maps local key ``j`` of sequence ``b`` to slot
``j % page_size`` of page ``block_table[b, j // page_size]``.  The call computes exactly the contiguous call on
``gather_paged_kv(pool, block_table)``.

CPU: gather / write round trips; the portable path on gloo worlds of 1, 2 and 4 with per-rank pools against the
contiguous call and the fp64 oracle; validation; the example's ``--page-size`` loop; the ptxas log of the paged
instantiations.

GPU: both kernels bitwise against the contiguous call on the gathered cache, with every slot and page outside the
visible keys NaN and unused table entries on an all-NaN page; the noise-scaled bound against the oracle; CUDA-graph
replays that append through the table; the benchmark shape; real rings.
"""
import os
import re
import sys

import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "examples"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gpu_dev_check as gdc  # noqa: E402
from dist_utils import run_distributed  # noqa: E402
from test_decode_multitoken import _gpu_case, _ptxas_log, reference_m, visible_m  # noqa: E402

from ring_attention_pytorch_b200 import gather_paged_kv, tree_attn_decode, write_paged_kv  # noqa: E402
from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc  # noqa: E402


def _bits(t):
    return t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t


def poison_(t):
    """Fill with NaN (0x7F in e4m3)."""
    _bits(t).fill_(0x7F) if t.dtype == torch.float8_e4m3fn else t.fill_(float("nan"))
    return t


def to_pool(cache, ps, layout, seed=0, spare=3):
    """cache [b, hk, n, d] (n a multiple of ps) -> (pool, table, spare page ids): the pages of every sequence at shuffled
    ids of a pool with ``spare`` more pages, all NaN.  ``layout`` "nhd": the pool is [num_pages, ps, hk, d] in memory,
    returned as its [num_pages, hk, ps, d] transpose."""
    b, hk, n, d = cache.shape
    mp = n // ps
    num = b * mp + spare
    perm = torch.randperm(num, generator=torch.Generator().manual_seed(seed))
    table = perm[:b * mp].view(b, mp).to(torch.int32).to(cache.device)
    if layout == "hnd":
        pool = torch.empty(num, hk, ps, d, dtype=cache.dtype, device=cache.device)
    else:
        pool = torch.empty(num, ps, hk, d, dtype=cache.dtype, device=cache.device).transpose(1, 2)
    poison_(pool)
    pages = _bits(cache).reshape(b, hk, mp, ps, d).permute(0, 2, 1, 3, 4).reshape(b * mp, hk, ps, d)
    _bits(pool)[table.long().flatten()] = pages
    return pool, table, perm[b * mp:].tolist()


def poisoned(pool, table, spare, vis):
    """(pool, table) with every slot of a key no token sees NaN, and every page that holds none of the visible keys
    (vis: bool [b, n] over the table's keys) renamed to the all-NaN spare page."""
    b, mp = table.shape
    ps = pool.shape[2]
    pool = pool.clone()  # keeps the strides (HND or NHD)
    vis = vis.to(pool.device)
    hidden = (~vis).view(b, mp, ps)
    page_ids = table.long()[:, :, None].expand(b, mp, ps)[hidden]
    slots = torch.arange(ps, device=pool.device)[None, None].expand(b, mp, ps)[hidden]
    if pool.dtype == torch.float8_e4m3fn:
        pool.view(torch.uint8)[page_ids, :, slots] = 0x7F
    else:
        pool[page_ids, :, slots] = float("nan")
    table = table.clone()
    table[~vis.view(b, mp, ps).any(-1)] = spare[0]
    return pool, table


# ================================================================================================
# CPU: the helpers
# ================================================================================================
@pytest.mark.parametrize("layout", ["hnd", "nhd"])
@pytest.mark.parametrize("ps", [16, 32, 64, 128])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float8_e4m3fn])
def test_gather_write_round_trip(layout, ps, dtype):
    g = torch.Generator().manual_seed(ps)
    b, hk, d, n = 5, 3, 16, 4 * ps
    cache = torch.randn(b, hk, n, d, generator=g).to(dtype)
    pool, table, spare = to_pool(cache, ps, layout, seed=ps)
    assert torch.equal(_bits(gather_paged_kv(pool, table)), _bits(cache))
    assert torch.equal(_bits(gather_paged_kv(pool, table, n - 5)), _bits(cache[:, :, :n - 5]))
    # ragged appends of t tokens, some crossing page boundaries; the other slots stay as they were
    vpool = pool.clone()
    start = torch.tensor([0, ps - 1, 2 * ps + 3, 3 * ps - 2, 5])
    for t in (1, 3):
        k_new, v_new = torch.randn(b, hk, t, d, generator=g), torch.randn(b, hk, t, d, generator=g)
        want_k, want_v = cache.clone(), gather_paged_kv(vpool, table).clone()
        write_paged_kv(pool, vpool, table, start, k_new, v_new)
        for i in range(b):
            s = int(start[i])
            want_k[i, :, s:s + t] = k_new[i].to(dtype)
            want_v[i, :, s:s + t] = v_new[i].to(dtype)
        assert torch.equal(_bits(gather_paged_kv(pool, table)), _bits(want_k))
        assert torch.equal(_bits(gather_paged_kv(vpool, table)), _bits(want_v))
        cache = want_k
    for s in spare:  # pages outside the table are untouched
        assert (_bits(pool)[s] == 0x7F).all() if dtype == torch.float8_e4m3fn else torch.isnan(pool[s]).all()


# ================================================================================================
# CPU: the portable path
# ================================================================================================
N_GLOBAL = 300
LENS = [0, 1, 65, 300, 129, 200, 9]
# (use q_pos, window, softclamp, sinks)
CASES = [(True, None, 0.0, False), (True, 5, 0.0, True), (True, 100, 8.0, False), (False, None, 5.0, True),
         (True, 37, 0.0, False), (True, 64, 3.0, True)]


def _portable_worker(rank, world):
    for m in (1, 3):
        for ci, (use_qpos, window, clamp, with_sinks) in enumerate(CASES):
            for ps, layout in ((16, "hnd"), (32, "nhd"), (64, "nhd")):
                g = torch.Generator().manual_seed(ci * 10 + m)
                b, h, hk, d = len(LENS), 4, 2, 16
                q = torch.randn(b, h, m, d, generator=g, dtype=torch.float64)
                kg = torch.randn(b, hk, N_GLOBAL, d, generator=g, dtype=torch.float64)
                vg = torch.randn(b, hk, N_GLOBAL, d, generator=g, dtype=torch.float64)
                lens = torch.tensor(LENS, dtype=torch.int32)
                q_pos = (lens - m).long()
                q_pos[2], q_pos[4], q_pos[5] = 65 + 40, 1 - m, -m
                q_pos = q_pos if use_qpos else None
                sinks = torch.linspace(-2.0, 3.0, h) if with_sinks else None
                vis = visible_m(N_GLOBAL, m, lens, q_pos, window)
                ref = reference_m(q, kg, vg, vis, clamp, sinks)
                # round-robin: global key t on rank t % world at local slot t // world
                cap = (N_GLOBAL + world - 1) // world
                cap = (cap + ps - 1) // ps * ps
                kl = torch.zeros(b, hk, cap, d)
                vl = torch.zeros(b, hk, cap, d)
                held = len(range(rank, N_GLOBAL, world))
                kl[:, :, :held], vl[:, :, :held] = kg[:, :, rank::world].float(), vg[:, :, rank::world].float()
                local = ((lens.long() - rank + world - 1).clamp(min=0) // world).to(torch.int32)
                kp, table, spare = to_pool(kl, ps, layout, seed=rank)
                vp, _, _ = to_pool(vl, ps, layout, seed=rank)
                lvis = visible_m(cap, m, local, None if q_pos is None else q_pos, window, rank, world).any(1)
                kpp, tp = poisoned(kp, table, spare, lvis)
                vpp, _ = poisoned(vp, table, spare, lvis)
                kw = dict(shard_kv_seq=False, cache_seqlens=local, q_pos=q_pos, window=window, softclamp_value=clamp,
                          sinks=sinks, kv_pos=(rank, world))
                out = tree_attn_decode(q.float(), kpp, vpp, block_table=tp, **kw)
                dense = tree_attn_decode(q.float(), kl, vl, **kw)
                assert torch.equal(out, dense), (rank, world, m, ci, ps)
                err = (out.double() - ref).abs().max().item()
                assert err < 1e-5, (rank, world, m, ci, ps, err)


@pytest.mark.parametrize("world", [1, 2, 4])
def test_portable_paged_decode(world):
    """Per-rank pools (HND and NHD, shuffled ids, 16 / 32 / 64-key pages) and round-robin kv_pos; lengths incl. 0 and 1,
    windows, softclamp, sinks, m in {1, 3}; slots and pages no token sees are NaN.  Bitwise the contiguous call on the
    clean cache, within 1e-5 of the fp64 oracle."""
    if world == 1:
        _portable_worker(0, 1)
    else:
        run_distributed(_portable_worker, world)


def test_invalid_paged_calls_raise():
    b, h, hk, d, ps = 3, 4, 2, 16, 16
    q = torch.randn(b, h, 1, d)
    kp = torch.randn(10, hk, ps, d)
    vp = torch.randn(10, hk, ps, d)
    table = torch.zeros(b, 4, dtype=torch.int32)
    lens = torch.full((b,), 20, dtype=torch.int32)
    bad = [
        dict(block_table=table.long(), cache_seqlens=lens),                     # dtype
        dict(block_table=table[0], cache_seqlens=lens),                         # rank
        dict(block_table=table[:2], cache_seqlens=lens),                        # batch
        dict(block_table=table.to("meta"), cache_seqlens=lens),                 # device
        dict(block_table=table),                                                # no cache_seqlens
        dict(block_table=table, cache_seqlens=lens, v=vp[:, :1]),               # unequal shapes
        dict(block_table=table, cache_seqlens=lens, v=vp.double()),             # unequal dtypes
        dict(block_table=table, cache_seqlens=lens, k=kp.transpose(0, 1).contiguous().transpose(0, 1)),  # strides
        dict(block_table=table, cache_seqlens=lens, k=torch.randn(10, hk, ps, 2 * d)[..., ::2],
             v=torch.randn(10, hk, ps, 2 * d)[..., ::2]),                       # d stride
        dict(block_table=table, cache_seqlens=lens, k=torch.randn(10, hk, 48, d), v=torch.randn(10, hk, 48, d)),
        dict(block_table=table, cache_seqlens=lens, k=torch.randn(10, hk, ps, d + 2)[..., :d],
             v=torch.randn(10, hk, ps, d + 2)[..., :d]),                        # 72-byte slot stride
        dict(block_table=torch.zeros(b, 2 ** 15, dtype=torch.int32), cache_seqlens=lens,
             k=torch.randn(1, hk, 2 ** 16, d), v=torch.randn(1, hk, 2 ** 16, d)),  # 2^31 keys
    ]
    for kw in bad:
        args = {"k": kp, "v": vp, **kw}
        k, v = args.pop("k"), args.pop("v")
        with pytest.raises(ValueError):
            tree_attn_decode(q, k, v, shard_kv_seq=False, **args)
        with pytest.raises(ValueError):
            tdc.tree_decode_cuda(q, k, v, dim_v=d, **args)
    with pytest.raises(ValueError, match="shard_kv_seq"):
        tree_attn_decode(q, kp, vp, block_table=table, cache_seqlens=lens)


# ================================================================================================
# CPU: the example, the build
# ================================================================================================
def _example_worker(rank, world, argv, out_path):
    import decode_tree_attention as ex

    worst = ex.run(ex.parse_args(argv))
    if rank == 0:
        torch.save(torch.tensor(worst), out_path)


@pytest.mark.parametrize("extra", [[], ["--draft", "3", "--window", "29"]])
def test_decode_example_paged(tmp_path, extra):
    out = tmp_path / "err.pt"
    argv = ["--device", "cpu", "--context", "301", "--batch", "4", "--heads", "4", "--kv-heads", "2", "--dim-head",
            "16", "--steps", "12", "--check", "--page-size", "16", "--ragged"] + extra
    run_distributed(_example_worker, 2, argv, str(out))
    assert torch.load(out).item() < 1e-4


@pytest.mark.parametrize("src,count", [("tree_decode_tc_sm90.cu", 15), ("tree_decode_sm90.cu", 12)])
def test_paged_instantiations_do_not_spill(src, count, tmp_path):
    """ptxas -v of the decode sources: the paged kernels keep everything in registers, and the tensor-core ones keep
    their wgmma asynchronous."""
    log = _ptxas_log(src, tmp_path)
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", log)[1:]
    paged = {}
    for blk in blocks:
        name = re.match(r"'(\S+)'", blk).group(1)
        if re.search(r"tree_decode(_tc)?_paged_kernelI", name):
            m = re.search(r"(\d+) bytes spill stores", blk)
            paged[name] = int(m.group(1)) if m else None
    assert len(paged) == count, sorted(paged)
    assert all(v == 0 for v in paged.values()), paged
    serialized = re.findall(r"wgmma.mma_async instructions are serialized.*function '(\S+)'", log)
    assert not [f for f in serialized if f in paged], serialized


# ================================================================================================
# GPU
# ================================================================================================
@pytest.fixture
def decode_config():
    old = dict(tdc.CONFIG)
    yield tdc.CONFIG
    tdc.CONFIG.clear()
    tdc.CONFIG.update(old)


N_GPU = 1536
GPU_LENS = [0, 1, 700, 1536, 1001, 64, 1200]
# (m, g, window, softclamp, sinks, kv_pos): windows whose start is not 64-aligned, a strided position map
GPU_CONFIGS = [(1, 4, None, 0.0, False, (0, 1)), (1, 1, 300, 20.0, True, (0, 1)), (4, 8, 200, 0.0, True, (3, 5)),
               (33, 1, None, 0.0, False, (0, 1)), (4, 4, 77, 10.0, False, (0, 1))]


def _paged_vs_dense(cache, d, ps, layout, cfg, seed=0, oracle=False):
    m, g, window, clamp, with_sinks, kv_pos = cfg
    hk = 2
    h = g * hk
    cc, qc = _gpu_case(cache, len(GPU_LENS), h, hk, N_GPU, d, m, seed)
    lens = torch.tensor(GPU_LENS, dtype=torch.int32, device="cuda")
    q_pos = torch.tensor([kv_pos[1] * x + kv_pos[0] - m for x in GPU_LENS], dtype=torch.int32, device="cuda")
    q_pos[2] = kv_pos[1] * 900 + kv_pos[0]
    vis = visible_m(N_GPU, m, lens, q_pos, window, *kv_pos)
    sinks = gdc.make_sinks("mix", [qc.transpose(1, 2)], [cc["kd"].transpose(1, 2)], clamp) if with_sinks else None
    kw = dict(dim_v=d, k_scale=cc["k_scale"], v_scale=cc["v_scale"], scale_block_keys=cc["block"], sinks=sinks,
              cache_seqlens=lens, q_pos=q_pos, window=window, kv_pos=kv_pos, softclamp_value=clamp)
    kp, table, spare = to_pool(cc["k"], ps, layout, seed=seed + ps)
    vp, _, _ = to_pool(cc["v"], ps, layout, seed=seed + ps)
    dense = tdc.tree_decode_cuda(qc, gather_paged_kv(kp, table), gather_paged_kv(vp, table), **kw)
    clean = tdc.tree_decode_cuda(qc, kp, vp, block_table=table, **kw)
    kpp, tp = poisoned(kp, table, spare, vis.any(1))
    vpp, _ = poisoned(vp, table, spare, vis.any(1))
    dirty = tdc.tree_decode_cuda(qc, kpp, vpp, block_table=tp, **kw)
    assert torch.isfinite(dirty.float()).all()
    assert torch.equal(clean, dense), (cache, d, ps, layout, cfg)
    assert torch.equal(dirty, dense), (cache, d, ps, layout, cfg)
    if oracle:
        ref = reference_m(qc, cc["kd"], cc["vd"], vis, clamp, sinks, dtype=torch.float32)
        lowp = reference_m(qc, cc["kd"], cc["vd"], vis, clamp, sinks, dtype=cc["lowp"])
        res = gdc.noise_bound(dirty, ref, lowp, gdc.CAP_OUT)
        print(f"[paged {tdc.CONFIG['tensor_core']} {cache} d {d} P {ps} {layout} {cfg}] err {res['err']:.3e} "
              f"bound {res['bound']:.3e} ratio {res['ratio']:.3f}")
        assert res["ok"], res


GPU_CASES = [(kern, d, cache, ps) for kern, d in (("on", 128), ("off", 128), ("off", 64))
             for cache in ("bf16", "fp16", "fp8", "fp8_b128") for ps in (16, 32, 64, 256)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=lambda c: "-".join(str(x) for x in c))
def test_paged_decode_is_bitwise_the_gathered_call(case, decode_config):
    """HND and NHD pools with shuffled page ids; lengths incl. 0, 1 and non-multiples of the page size; m in {1, 4, 33},
    g in {1, 4, 8}; every slot past the lengths and every page outside the visible keys NaN, unused entries on an
    all-NaN page: the output is finite and bitwise the contiguous call on the gathered clean cache."""
    kernel, d, cache, ps = case
    decode_config["tensor_core"] = kernel
    for layout in ("hnd", "nhd"):
        for i, cfg in enumerate(GPU_CONFIGS):
            _paged_vs_dense(cache, d, ps, layout, cfg, seed=i, oracle=(ps == 16 and i < 3))


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 4])
@pytest.mark.parametrize("kernel", ["on", "off"])
def test_cuda_graph_replay_appends_through_the_table(kernel, m, decode_config):
    """Capture one paged step.  Between replays, outside the graph: write the next m tokens with write_paged_kv, put a
    fresh page id into the table in place when a page fills, advance cache_seqlens and q_pos.  Each replay is bitwise
    the eager call."""
    decode_config["tensor_core"] = kernel
    b, h, hk, d, ps, cap = 4, 16, 4, 128, 16, 4096
    mp = cap // ps
    g = torch.Generator("cuda").manual_seed(5)
    q = torch.randn(b, h, m, d, device="cuda", generator=g, dtype=torch.bfloat16)
    kp = poison_(torch.empty(b * mp + 1, hk, ps, d, device="cuda", dtype=torch.bfloat16))
    vp = poison_(torch.empty_like(kp))
    free = torch.randperm(b * mp + 1, generator=torch.Generator().manual_seed(1)).tolist()
    table = torch.full((b, mp), free[-1], dtype=torch.int32, device="cuda")  # unused entries: an all-NaN page
    free.pop()
    owned = [0] * b
    lens = torch.tensor([100, 4, 2000, 3000], dtype=torch.int32, device="cuda")

    def grow(upto):
        for i in range(b):
            while owned[i] * ps < int(upto[i]):
                table[i, owned[i]] = free.pop()
                owned[i] += 1

    grow(lens)
    for i in range(b):  # the prompt
        n = int(lens[i])
        write_paged_kv(kp, vp, table[i:i + 1], torch.zeros(1, dtype=torch.int32, device="cuda"),
                       torch.randn(1, hk, n, d, device="cuda", generator=g), torch.randn(1, hk, n, d, device="cuda", generator=g))
    q_pos = (lens - m).clone()
    out = torch.empty(b, h, m, d, device="cuda", dtype=torch.bfloat16)
    kw = dict(dim_v=d, cache_seqlens=lens, q_pos=q_pos, window=1000, softclamp_value=30.0, block_table=table)
    tdc.tree_decode_cuda(q, kp, vp, out=out, **kw)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        tdc.tree_decode_cuda(q, kp, vp, out=out, **kw)
    for step in range(6):
        grow(lens + m)
        write_paged_kv(kp, vp, table, lens, torch.randn(b, hk, m, d, device="cuda", generator=g),
                       torch.randn(b, hk, m, d, device="cuda", generator=g))
        lens.add_(m)
        q_pos.add_(m)
        graph.replay()
        torch.cuda.synchronize()
        got = out.clone()
        want = tdc.tree_decode_cuda(q, kp, vp, **kw)
        assert torch.isfinite(got.float()).all()
        assert torch.equal(got, want), step


@pytest.mark.gpu
@pytest.mark.parametrize("ps", [16, 64])
@pytest.mark.parametrize("cache", ["bf16", "fp8"])
def test_benchmark_shape_paged(cache, ps, decode_config):
    """b 256, 32 / 8 heads, 8192 keys: the plan splits like the contiguous call and its grid fits the paged variant's
    residency (cooperative launch); sampled sequences pass the oracle bound."""
    from ring_attention_pytorch_b200.ops import _ext

    decode_config["tensor_core"] = "on"
    b, h, hk, n, d = 256, 32, 8, 8192, 128
    kind = 2 if cache == "fp8" else 0
    plan = tdc.decode_plan(b, h, hk, n, d, kind, ranged=True, span=n, paged=True)
    dense_plan = tdc.decode_plan(b, h, hk, n, d, kind, ranged=True, span=n)
    assert plan.splits == dense_plan.splits and plan.tensor_core
    assert plan.resident == int(_ext.ops().tree_decode_max_ctas(d, kind, True, True, 0, True)) > 0
    cc, qc = _gpu_case(cache, b, h, hk, n, d, 1, seed=11)
    rows = [0, 37, 128, 255]
    kd, vd = cc["kd"][rows].clone(), cc["vd"][rows].clone()
    del cc["kd"], cc["vd"]
    kp, table, _ = to_pool(cc.pop("k"), ps, "hnd", seed=ps)
    vp, _, _ = to_pool(cc.pop("v"), ps, "hnd", seed=ps)
    lens = torch.full((b,), n, dtype=torch.int32, device="cuda")
    out = tdc.tree_decode_cuda(qc, kp, vp, dim_v=d, k_scale=cc["k_scale"], v_scale=cc["v_scale"],
                               scale_block_keys=cc["block"], cache_seqlens=lens, block_table=table)
    torch.cuda.synchronize()
    vis = visible_m(n, 1, lens[rows], None, None)
    ref = reference_m(qc[rows], kd, vd, vis, dtype=torch.float32)
    lowp = reference_m(qc[rows], kd, vd, vis, dtype=cc["lowp"])
    res = gdc.noise_bound(out[rows], ref, lowp, gdc.CAP_OUT)
    assert res["ok"], res


def _real_ring_worker(rank, world):
    dev = torch.device("cuda", rank)
    g = torch.Generator().manual_seed(3)
    b, h, hk, d, cap, m, ps = 5, 8, 2, 128, 704, 1, 16
    lens = torch.tensor([0, 2, 3 * world + 1, cap * world - 3, 1000])
    q = torch.randn(b, h, m, d, generator=g)
    kg, vg = torch.randn(b, hk, cap * world, d, generator=g), torch.randn(b, hk, cap * world, d, generator=g)
    q_pos = lens - m
    sinks = torch.linspace(-1.0, 2.0, h)
    for window in (None, 333):
        vis = visible_m(cap * world, m, lens, q_pos, window)
        ref = reference_m(q, kg, vg, vis, sinks=sinks)
        kp, table, _ = to_pool(kg[:, :, rank::world].to(dev, torch.bfloat16).contiguous(), ps, "nhd", seed=rank)
        vp, _, _ = to_pool(vg[:, :, rank::world].to(dev, torch.bfloat16).contiguous(), ps, "nhd", seed=rank)
        local = ((lens - rank + world - 1).clamp(min=0) // world).to(dev, torch.int32)
        out = tree_attn_decode(q.to(dev, torch.bfloat16), kp, vp, shard_kv_seq=False, cache_seqlens=local,
                               q_pos=q_pos.to(dev), window=window, kv_pos=(rank, world), sinks=sinks.to(dev),
                               block_table=table)
        assert (out.double().cpu() - ref).abs().max() < 2e-2, (rank, window)
    dist.barrier()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
def test_real_ring_paged(world):
    """Per-rank NHD pools and tables with round-robin kv_pos, a window and sinks, against the dense reference; the merge
    is NVLS where the NVSwitch offers multicast, P2P otherwise."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    run_distributed(_real_ring_worker, world, backend="nccl", timeout=600.0)
