"""Multi-token tree decode: ``q [b, h, m, d]``, query token ``t`` of sequence ``b`` at global position ``q_pos[b] + t``.

Local key ``j`` sits at ``P(j) = offset + stride * j`` and is visible to token ``t`` iff ``j < min(cache_seqlens[b], n)``,
``P(j) <= q_pos[b] + t`` and (window > 0) ``q_pos[b] + t - P(j) <= window``; without ``q_pos`` every token sees every
held key.  Everything else (GQA, softclamp, sinks, cache formats) applies per token row.

CPU: the portable path on gloo worlds of 1, 2 and 4 against an fp64 dense reference; one m-token call against m
single-token calls; m = 1 bitwise against results of the single-token implementation (``tests/golden``); a hypothesis
property test of the kernels' multi-token unit and column ranges; validation; the example's ``--draft`` loop; the
ptxas log of the multi-token instantiations.

GPU: both kernels against the oracle under the noise-scaled rule with every key outside the union of the tokens'
ranges NaN; CUDA-graph replays advancing lengths and positions by m; the benchmark shape at m = 8; real rings.
"""
import os
import re
import shutil
import subprocess
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
from test_decode_ragged import nan_fill_invisible, reference  # noqa: E402

from ring_attention_pytorch_b200 import build as ext_build  # noqa: E402
from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc  # noqa: E402

TILE = 64


def visible_m(n, m, lens, q_pos, window, offset=0, stride=1, b=1):
    """bool [b, m, n] by the rule above (lens / q_pos: int tensors [b] or None; ``b`` when both are None)."""
    b = next((t.shape[0] for t in (lens, q_pos) if t is not None), b)
    j = torch.arange(n)
    vis = torch.ones(b, m, n, dtype=torch.bool)
    if lens is not None:
        vis &= (j[None] < lens.long().cpu()[:, None])[:, None]
    if q_pos is not None:
        pos = q_pos.long().cpu()[:, None] + torch.arange(m)[None]
        rel = pos[:, :, None] - (offset + stride * j)[None, None]
        vis &= rel >= 0
        if window is not None and window > 0:
            vis &= rel <= window
    return vis


def reference_m(q, k, v, vis, softclamp=0.0, sinks=None, dtype=torch.float64):
    """q [b, h, m, d], vis [b, m, n] -> [b, h, m, d]: the single-token oracle of each token row."""
    return torch.cat([reference(q[:, :, t:t + 1], k, v, vis[:, t], softclamp, sinks, dtype)
                      for t in range(q.shape[2])], 2)


# ================================================================================================
# CPU: the portable path
# ================================================================================================
N_GLOBAL = 300
LENS = [0, 1, 65, 300, 129, 200, 9]
# (use q_pos, window, softclamp, sinks, use lens)
CASES = [(True, None, 0.0, False, True), (True, 5, 0.0, True, True), (True, 100, 8.0, False, True),
         (False, None, 0.0, False, True), (False, None, 5.0, True, False), (True, 37, 0.0, False, False),
         (True, 64, 3.0, True, True)]


def _portable_case(seed, m, h=4, hk=2, d=16):
    g = torch.Generator().manual_seed(seed)
    b = len(LENS)
    q = torch.randn(b, h, m, d, generator=g, dtype=torch.float64)
    k = torch.randn(b, hk, N_GLOBAL, d, generator=g, dtype=torch.float64)
    v = torch.randn(b, hk, N_GLOBAL, d, generator=g, dtype=torch.float64)
    lens = torch.tensor(LENS, dtype=torch.int32)
    q_pos = (lens - m).long()  # the m draft tokens are the last m keys held
    # a query run past the cache, tokens before every key (some see none), one inside a short window
    q_pos[2], q_pos[4], q_pos[5], q_pos[6] = 65 + 40, 1 - m, -m, 3
    return q, k, v, lens, q_pos


def _portable_worker(rank, world, shard):
    from ring_attention_pytorch_b200 import tree_attn_decode

    for m in (1, 2, 5, 9):
        for ci, (use_qpos, window, clamp, with_sinks, use_lens) in enumerate(CASES):
            for h, hk in ((4, 2), (6, 6)):
                q, k, v, lens, q_pos = _portable_case(ci * 10 + m, m, h, hk)
                q_pos = q_pos if use_qpos else None
                lens_ = lens if use_lens else None
                sinks = torch.linspace(-2.0, 3.0, h) if with_sinks else None
                vis = visible_m(N_GLOBAL, m, lens_, q_pos, window, b=len(LENS))
                ref = reference_m(q, k, v, vis, clamp, sinks)
                union = vis.any(1)
                kn, vn = nan_fill_invisible(k, union), nan_fill_invisible(v, union)
                kw = dict(q_pos=q_pos, window=window, softclamp_value=clamp, sinks=sinks)
                if shard:
                    out = tree_attn_decode(q.float(), kn.float(), vn.float(), cache_seqlens=lens_, **kw)
                else:  # round-robin: global key t lives on rank t % world at local slot t // world
                    kl, vl = kn[:, :, rank::world].float().contiguous(), vn[:, :, rank::world].float().contiguous()
                    src = lens_ if lens_ is not None else torch.full_like(lens, N_GLOBAL)
                    local = ((src.long() - rank + world - 1).clamp(min=0) // world).to(torch.int32)
                    out = tree_attn_decode(q.float(), kl, vl, shard_kv_seq=False, cache_seqlens=local,
                                           kv_pos=(rank, world), **kw)
                assert out.shape == (len(LENS), h, m, 16)
                assert torch.isfinite(out).all(), (rank, m, ci)
                err = (out.double() - ref).abs().max().item()
                assert err < 1e-5, (rank, world, shard, m, ci, h, err)
                if sinks is None:  # rows that see no key anywhere are exactly zero
                    empty = ~vis.any(-1)  # [b, m]
                    assert torch.equal(out.permute(0, 2, 1, 3)[empty], torch.zeros_like(out.permute(0, 2, 1, 3)[empty]))


@pytest.mark.parametrize("shard", [True, False])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_portable_multitoken_decode(world, shard):
    """m in {1, 2, 5, 9} with and without q_pos, windows, lengths, softclamp and sinks; tokens that see no key on a
    rank or none at all; every key outside the union of the tokens' ranges holds NaN."""
    if world == 1:
        _portable_worker(0, 1, shard)
    else:
        run_distributed(_portable_worker, world, shard)


@pytest.mark.parametrize("window", [None, 20])
def test_one_call_equals_single_token_calls(window):
    from ring_attention_pytorch_b200 import tree_attn_decode

    m = 5
    q, k, v, lens, q_pos = _portable_case(3, m)
    sinks = torch.linspace(-1.0, 1.0, 4)
    kw = dict(cache_seqlens=lens, window=window, softclamp_value=4.0, sinks=sinks)
    q, k, v = q.float(), k.float(), v.float()
    multi = tree_attn_decode(q, k, v, q_pos=q_pos, **kw)
    single = torch.cat([tree_attn_decode(q[:, :, t:t + 1], k, v, q_pos=q_pos + t, **kw) for t in range(m)], 2)
    assert (multi - single).abs().max().item() < 1e-6


def test_single_token_is_bitwise_the_previous_result():
    """The fixture holds inputs and outputs of the single-token portable path before multi-token support."""
    from ring_attention_pytorch_b200 import tree_attn_decode

    gold = torch.load(os.path.join(ROOT, "tests", "golden", "decode_single_token_portable.pt"))
    q, k, v, lens, q_pos, sinks = (gold[x] for x in ("q", "k", "v", "lens", "q_pos", "sinks"))
    cases = {
        "plain": dict(),
        "sinks": dict(sinks=sinks),
        "ranged": dict(cache_seqlens=lens, q_pos=q_pos, window=9, softclamp_value=5.0, sinks=sinks),
        "lens_only": dict(cache_seqlens=lens),
        "strided": dict(shard_kv_seq=False, q_pos=q_pos, kv_pos=(2, 3), window=31),
    }
    assert set(cases) == set(gold["results"])
    for name, kw in cases.items():
        assert torch.equal(tree_attn_decode(q, k, v, **kw), gold["results"][name]), name


def test_invalid_queries_raise():
    from ring_attention_pytorch_b200 import tree_attn_decode

    q, k, v, _, _ = _portable_case(0, 2)
    q, k, v = q.float(), k.float(), v.float()
    for bad in (q[:, :, 0], q[:, :, :0], q[None]):
        with pytest.raises(ValueError):
            tree_attn_decode(bad, k, v)
        with pytest.raises(ValueError):
            tdc.tree_decode_cuda(bad, k, v, dim_v=16)
    for out in (torch.empty(7, 4, 1, 16), torch.empty(7, 4, 2, 8), torch.empty(7 * 4 * 2 * 16)):
        with pytest.raises(ValueError):
            tdc.tree_decode_cuda(q, k, v, dim_v=16, out=out)


# ================================================================================================
# CPU: the unit and column ranges of the multi-token kernels (tree_decode_common.cuh)
# ================================================================================================
def unit_range(n, splits, length, q_pos, window, offset, stride, split, m):
    """(lo, k0, k1) of unit (b, split): td_unit_range<TILE, MULTI> (Python's // floors like td_floor_div)."""
    lo, hi = 0, n
    if length is not None:
        hi = min(hi, length)
    span = n
    if q_pos is not None:
        rel = q_pos - offset
        hi = min(hi, (rel + m - 1) // stride + 1)
        if window is not None and window > 0:
            lo = max(lo, -((window - rel) // stride))
            span = min(span, (window + m - 1) // stride + TILE)
    lo = min(lo, n)
    per = ((span + splits - 1) // splits + TILE - 1) // TILE * TILE
    k0 = min((lo & ~(TILE - 1)) + split * per, n)
    k1 = max(min(hi, k0 + per), k0) if lo < hi else k0
    return lo, k0, k1


def col_range(q_pos, window, offset, stride, t, lo, k1):
    """[clo, chi) of token t inside a unit's [lo, k1): td_col_range."""
    clo, chi = lo, k1
    if q_pos is not None:
        rel = q_pos + t - offset
        chi = min(chi, rel // stride + 1)
        if window is not None and window > 0:
            clo = max(clo, -((window - rel) // stride))
    return min(clo, k1), max(chi, lo)


def _check_units(n, length, q_pos, window, offset, stride, splits, m):
    vis = visible_m(n, m, None if length is None else torch.tensor([length]),
                    None if q_pos is None else torch.tensor([q_pos]), window, offset, stride)[0]
    union = vis.any(0)
    covered = torch.zeros(n, dtype=torch.int64)
    per_token = torch.zeros(m, n, dtype=torch.int64)
    for s in range(splits):
        lo, k0, k1 = unit_range(n, splits, length, q_pos, window, offset, stride, s, m)
        assert 0 <= k0 <= k1 <= n
        if k0 < k1:
            assert k0 % TILE == 0 and lo <= k1 - 1  # tiles start on 64-key boundaries; clamped loads stay in [lo, k1)
            covered[max(k0, lo):k1] += 1
            for t in range(m):
                clo, chi = col_range(q_pos, window, offset, stride, t, lo, k1)
                assert lo <= clo <= k1 and lo <= chi <= k1
                keys = torch.arange(k0, k1)
                per_token[t, k0:k1] += ((keys >= clo) & (keys < chi)).long()
    assert torch.equal(covered, union.long()), (n, length, q_pos, window, offset, stride, splits, m)
    assert torch.equal(per_token, vis.long()), (n, length, q_pos, window, offset, stride, splits, m)


def test_multitoken_unit_ranges_property():
    """The units of a multi-token call cover exactly the union of the tokens' visible keys, each key in one split,
    with tiles on 64-key boundaries; inside them, each token's column range is exactly its visible keys."""
    hyp = pytest.importorskip("hypothesis")
    st = hyp.strategies

    @hyp.settings(max_examples=300, deadline=None)
    @hyp.given(n=st.integers(1, 2000), length=st.one_of(st.none(), st.integers(-5, 2100)),
               q_pos=st.one_of(st.none(), st.integers(-300, 20000)), window=st.one_of(st.none(), st.integers(0, 3000)),
               offset=st.integers(0, 2000), stride=st.integers(1, 9), splits=st.integers(1, 60), m=st.integers(1, 40))
    def prop(n, length, q_pos, window, offset, stride, splits, m):
        if q_pos is None:
            window = None
        _check_units(n, length, q_pos, window, offset, stride, splits, m)

    prop()


def test_multitoken_unit_ranges_edge_cases():
    for args in ((64, 64, 56, 7, 0, 1, 1, 8), (200, 200, 100, 1, 0, 2, 3, 2), (1000, 1000, 990, 5, 0, 1, 7, 33),
                 (128, 0, 10, None, 0, 1, 2, 3), (128, 128, -5, 3, 0, 1, 2, 9), (300, 300, 64, 63, 0, 1, 4, 2)):
        _check_units(*args)


def test_python_span_matches_kernel_mirror():
    for n, window, stride, m in ((5000, None, 1, 4), (5000, 4096, 1, 8), (5000, 100, 8, 9), (131072, 4096, 8, 33)):
        span = tdc.decode_span(n, window, stride, m)
        assert span == (n if window is None else min(n, (window + m - 1) // stride + TILE))
        assert tdc.decode_span(n, window, stride, 1) == tdc.decode_span(n, window, stride)


# ================================================================================================
# CPU: the example, the build
# ================================================================================================
def _example_worker(rank, world, argv, out_path):
    import decode_tree_attention as ex

    worst = ex.run(ex.parse_args(argv))
    if rank == 0:
        torch.save(torch.tensor(worst), out_path)


@pytest.mark.parametrize("window", [None, 29])
def test_decode_example_draft_tokens(tmp_path, window):
    out = tmp_path / "err.pt"
    argv = ["--device", "cpu", "--context", "301", "--batch", "4", "--heads", "4", "--kv-heads", "2", "--dim-head",
            "16", "--steps", "5", "--check", "--draft", "3"] + ([] if window is None else ["--window", str(window)])
    run_distributed(_example_worker, 2, argv, str(out))
    assert torch.load(out).item() < 1e-4


def _ptxas_log(src, tmp_path) -> str:
    log = ext_build.BUILD / (src + ".log")
    if log.exists():
        t = log.stat().st_mtime
        if all(f.stat().st_mtime <= t for f in [ext_build.CSRC / src, *ext_build._headers()]):
            return log.read_text()
    if not (shutil.which(ext_build.NVCC) or os.path.exists(ext_build.NVCC)):
        pytest.skip("nvcc not available and no current build log")
    cmd = [ext_build.NVCC, *ext_build.NVCC_FLAGS, "-I", str(ext_build.CSRC), "-c", str(ext_build.CSRC / src),
           "-o", str(tmp_path / (src + ".o"))]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    return proc.stdout + proc.stderr


@pytest.mark.parametrize("src,count", [("tree_decode_tc_sm90.cu", 9), ("tree_decode_sm90.cu", 6)])
def test_multitoken_instantiations_do_not_spill(src, count, tmp_path):
    """ptxas -v of the decode sources: the multi-token instantiations (template flags ranged = multi = true) keep
    everything in registers, and the tensor-core ones keep their wgmma asynchronous."""
    log = _ptxas_log(src, tmp_path)
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", log)[1:]
    multi = {}
    for blk in blocks:
        name = re.match(r"'(\S+)'", blk).group(1)
        if re.search(r"tree_decode(_tc)?_kernelI\S*Lb1ELb1EEEv", name):
            m = re.search(r"(\d+) bytes spill stores", blk)
            multi[name] = int(m.group(1)) if m else None
    assert len(multi) == count, sorted(multi)
    assert all(v == 0 for v in multi.values()), multi
    serialized = re.findall(r"wgmma.mma_async instructions are serialized.*function '(\S+)'", log)
    assert not [f for f in serialized if f in multi], serialized


# ================================================================================================
# GPU
# ================================================================================================
@pytest.fixture
def decode_config():
    old = dict(tdc.CONFIG)
    yield tdc.CONFIG
    tdc.CONFIG.clear()
    tdc.CONFIG.update(old)


def _gpu_case(cache, b, h, hk, n, d, m, seed=0):
    import test_decode_kernels as tdk

    q, k, v = tdk.make_inputs(None, b, h, hk, n, d, seed=seed)
    qm = torch.randn(b, h, m, d, device="cuda", generator=torch.Generator("cuda").manual_seed(seed + 17))
    cc = tdk.make_cache(cache, qm, k, v, seed=seed)  # (the fp8 case rescales every token's query the same way)
    return cc, cc["q"].to(torch.float16 if cache == "fp16" else torch.bfloat16)


def _run_multi(cache, d, h, hk, n, m, lens, q_pos, window, clamp, with_sinks, kv_pos=(0, 1), seed=0, tag=""):
    cc, qc = _gpu_case(cache, len(lens), h, hk, n, d, m, seed)
    lens_t = torch.tensor(lens, dtype=torch.int32, device="cuda")
    qpos_t = None if q_pos is None else torch.tensor(q_pos, dtype=torch.int32, device="cuda")
    vis = visible_m(n, m, lens_t, qpos_t, window, *kv_pos)
    sinks = gdc.make_sinks("mix", [qc.transpose(1, 2)], [cc["kd"].transpose(1, 2)], clamp) if with_sinks else None
    union = vis.any(1)
    kn, vn = nan_fill_invisible(cc["k"], union), nan_fill_invisible(cc["v"], union)
    out = tdc.tree_decode_cuda(qc, kn, vn, dim_v=d, k_scale=cc["k_scale"], v_scale=cc["v_scale"],
                               scale_block_keys=cc["block"], sinks=sinks, cache_seqlens=lens_t, q_pos=qpos_t,
                               window=window, kv_pos=kv_pos, softclamp_value=clamp)
    ref = reference_m(qc, cc["kd"], cc["vd"], vis, clamp, sinks, dtype=torch.float32)
    lowp = reference_m(qc, cc["kd"], cc["vd"], vis, clamp, sinks, dtype=cc["lowp"])
    res = gdc.noise_bound(out, ref, lowp, gdc.CAP_OUT)
    print(f"[multi {tag} {tdc.CONFIG['tensor_core']} {cache} d {d} g {h // hk} m {m} window {window} clamp {clamp} "
          f"sinks {with_sinks}] err {res['err']:.3e} bound {res['bound']:.3e} ratio {res['ratio']:.3f}")
    assert out.shape == (len(lens), h, m, d)
    assert torch.isfinite(out.float()).all() and res["ok"], res
    return out


GPU_CASES = []
for _kern, _d in (("on", 128), ("off", 128), ("off", 64)):
    for _cache in ("bf16", "fp16", "fp8", "fp8_b128"):
        GPU_CASES.append((_kern, _cache, _d, 3, 4, 300, 0.0, True))
    for _m in (2, 8, 33):
        for _g in (1, 4, 8):
            GPU_CASES.append((_kern, "bf16", _d, _m, _g, 200 if _m != 8 else None, 20.0 if _g == 4 else 0.0,
                              _m == 33))


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=lambda c: "-".join(str(x) for x in c))
def test_multitoken_decode_kernels(case, decode_config):
    """Ragged lengths incl. 0 and 1, tokens before every key, windows whose bounds are not 64-aligned, a strided
    position map, softclamp and sinks; g * m crosses 8, 16 and 32 columns and needs several chunks."""
    kernel, cache, d, m, g, window, clamp, with_sinks = case
    decode_config["tensor_core"] = kernel
    hk = 2
    n = 1500
    lens = [0, 1, 700, 1500, 1001, 64, 1200]
    q_pos = [x - m for x in lens]
    q_pos[2], q_pos[6] = 900, 1 - m
    _run_multi(cache, d, g * hk, hk, n, m, lens, q_pos, window, clamp, with_sinks)
    # a strided position map (round-robin shard of rank 3 in a world of 5), and lengths only (no position rule)
    _run_multi(cache, d, g * hk, hk, n, m, lens, [5 * x for x in lens], window, clamp, with_sinks, kv_pos=(3, 5),
               tag="strided")
    _run_multi(cache, d, g * hk, hk, n, m, lens, None, None, clamp, with_sinks, tag="no q_pos")


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["on", "off"])
def test_cuda_graph_replay_advances_by_m(kernel, decode_config):
    """Capture one m-token step; advance ``cache_seqlens`` and ``q_pos`` by m in place and replay: each replay is
    bitwise the eager call on the same inputs."""
    decode_config["tensor_core"] = kernel
    b, h, hk, n, d, m, window = 4, 16, 4, 4096, 128, 4, 1000
    cc, qc = _gpu_case("bf16", b, h, hk, n, d, m, seed=9)
    lens = torch.tensor([100, 4, 2000, 3000], dtype=torch.int32, device="cuda")
    q_pos = (lens - m).clone()
    out = torch.empty(b, h, m, d, device="cuda", dtype=qc.dtype)
    kw = dict(dim_v=d, cache_seqlens=lens, q_pos=q_pos, window=window, softclamp_value=30.0)
    tdc.tree_decode_cuda(qc, cc["k"], cc["v"], out=out, **kw)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        tdc.tree_decode_cuda(qc, cc["k"], cc["v"], out=out, **kw)
    for step in range(5):
        lens.add_(m)
        q_pos.add_(m)
        graph.replay()
        torch.cuda.synchronize()
        got = out.clone()
        want = tdc.tree_decode_cuda(qc, cc["k"], cc["v"], **kw)
        assert torch.equal(got, want), step


@pytest.mark.gpu
@pytest.mark.parametrize("cache", ["bf16", "fp8"])
def test_benchmark_shape_eight_tokens(cache, decode_config):
    """b 256, 32 / 8 heads, 8192 keys, m = 8: 32 columns per unit, a full persistent grid planned with that variant's
    residency (cooperative launch); sampled sequences match the oracle."""
    decode_config["tensor_core"] = "on"
    b, h, hk, n, d, m = 256, 32, 8, 8192, 128, 8
    cc, qc = _gpu_case(cache, b, h, hk, n, d, m, seed=11)
    plan = tdc.decode_plan(b, h, hk, n, d, 2 if cache == "fp8" else 0, ranged=True, span=n, tokens=m)
    assert plan.tensor_core and plan.groups == b * hk and plan.groups * plan.splits >= plan.resident
    lens = torch.full((b,), n, dtype=torch.int32, device="cuda")
    out = tdc.tree_decode_cuda(qc, cc["k"], cc["v"], dim_v=d, k_scale=cc["k_scale"], v_scale=cc["v_scale"],
                               scale_block_keys=cc["block"], cache_seqlens=lens, q_pos=lens - m)
    torch.cuda.synchronize()
    rows = [0, 37, 128, 255]
    vis = visible_m(n, m, lens[rows], (lens - m)[rows], None)
    kd, vd = cc["kd"][rows], cc["vd"][rows]
    ref = reference_m(qc[rows], kd, vd, vis, dtype=torch.float32)
    lowp = reference_m(qc[rows], kd, vd, vis, dtype=cc["lowp"])
    res = gdc.noise_bound(out[rows], ref, lowp, gdc.CAP_OUT)
    assert res["ok"], res


def _real_ring_worker(rank, world):
    from ring_attention_pytorch_b200 import tree_attn_decode

    dev = torch.device("cuda", rank)
    g = torch.Generator().manual_seed(3)
    b, h, hk, d, cap, m = 5, 8, 2, 128, 700, 4
    lens = torch.tensor([0, 2, 3 * world + 1, cap * world - 3, 1000])  # global lengths, the m drafts included
    q = torch.randn(b, h, m, d, generator=g)
    kg, vg = torch.randn(b, hk, cap * world, d, generator=g), torch.randn(b, hk, cap * world, d, generator=g)
    q_pos = lens - m
    sinks = torch.linspace(-1.0, 2.0, h)
    for window in (None, 333):
        vis = visible_m(cap * world, m, lens, q_pos, window)
        ref = reference_m(q, kg, vg, vis, sinks=sinks)
        kl = kg[:, :, rank::world].to(dev, torch.bfloat16).contiguous()
        vl = vg[:, :, rank::world].to(dev, torch.bfloat16).contiguous()
        local = ((lens - rank + world - 1).clamp(min=0) // world).to(dev, torch.int32)
        out = tree_attn_decode(q.to(dev, torch.bfloat16), kl, vl, shard_kv_seq=False, cache_seqlens=local,
                               q_pos=q_pos.to(dev), window=window, kv_pos=(rank, world), sinks=sinks.to(dev))
        assert (out.double().cpu() - ref).abs().max() < 2e-2, (rank, window)
    dist.barrier()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
def test_real_ring_multitoken(world):
    """Round-robin shards on a real ring with sinks; the merge is NVLS where the NVSwitch offers multicast, P2P
    otherwise."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    run_distributed(_real_ring_worker, world, backend="nccl", timeout=600.0)
