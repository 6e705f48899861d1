"""Learned attention sinks: one extra logit per query head that joins every row's softmax denominator with a zero
value vector.  For query row i of head h with visible keys J_i and logits s_ij (after scale and softclamp):

    L_i   = log(exp(sigma_h) + sum_{j in J_i} exp(s_ij))
    out_i = sum_{j in J_i} exp(s_ij - L_i) v_j
    dsigma_h = -sum_{b, i} exp(sigma_h - L_i) (dO_i . out_i)      (this rank's rows)

The CPU half checks the oracle, the portable op on gloo rings, the portable decode and the modules, and shows that
the GPU error rule (``gpu_dev_check.noise_bound``) rejects plausible sink mistakes in a torch model of the kernel's
algorithm.  The GPU half runs the kernels under that rule.
"""
import math
import os
import sys

import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gpu_dev_check as gdc  # noqa: E402
from dist_utils import run_distributed  # noqa: E402

from ring_attention_pytorch_b200.ops.oracle import attention_with_positions  # noqa: E402
from ring_attention_pytorch_b200.parallel.documents import document_runs  # noqa: E402
from ring_attention_pytorch_b200.parallel.layout import make_position_map  # noqa: E402


# ================================================================================================
# CPU: oracle, portable op, portable decode, modules
# ================================================================================================
def test_oracle_matches_explicit_softmax_over_keys_and_sink():
    torch.manual_seed(0)
    b, i, j, h, hk, d = 2, 9, 13, 4, 2, 8
    q, k, v = torch.randn(b, i, h, d, dtype=torch.float64), torch.randn(b, j, hk, d, dtype=torch.float64), \
        torch.randn(b, j, hk, d, dtype=torch.float64)
    sinks = torch.tensor([-3.0, 0.5, 2.0, 9.0], dtype=torch.float64)
    key_mask = torch.rand(b, j) > 0.4
    key_mask[1] = False  # batch 1: every row sees no key
    out, lse = attention_with_positions(q, k, v, key_mask=key_mask, sinks=sinks, return_lse=True, softclamp_value=3.0)
    heads = torch.arange(h) % hk
    s = torch.einsum("bihd,bjhd->bhij", q, k[:, :, heads]) * d ** -0.5
    s = (s / 3.0).tanh() * 3.0  # the keys' logits are softclamped, the sink is not
    s = s.masked_fill(~key_mask[:, None, None, :], -math.inf)
    ext = torch.cat((s, sinks[None, :, None, None].expand(b, h, i, 1)), -1)
    p = ext.softmax(-1)[..., :j]
    want = torch.einsum("bhij,bjhd->bihd", p, v[:, :, heads])
    assert torch.allclose(out, want, atol=1e-12)
    assert torch.allclose(lse, ext.logsumexp(-1), atol=1e-12)
    assert (out[1] == 0).all() and torch.equal(lse[1], sinks[:, None].expand(h, i))


def _global_case(seed, b, total, h, hk, d, docs, kmask, empty):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(b, total, h, d, generator=g)
    k = torch.randn(b, total, hk, d, generator=g)
    v = torch.randn(b, total, hk, d, generator=g)
    do = torch.randn(b, total, h, d, generator=g)
    sinks = torch.randn(h, generator=g) * 2.0
    km = (torch.rand(b, total, generator=g) > 0.3) if kmask else None
    if empty:
        km[0] = False
    ids = gdc.make_document_ids("ragged" if total > 64 else "tiny", b, total, seed, device="cpu") if docs else None
    return q, k, v, do, sinks, km, ids


# (name, causal, window, key mask, documents, GQA, empty rows)
PORTABLE_CASES = [
    ("causal_gqa", True, None, False, False, True, False),
    ("window", True, 5, False, False, False, False),
    ("kmask_empty", False, None, True, False, True, True),
    ("docs", True, None, False, True, False, False),
]


def _portable_worker(rank, world, layout):
    from ring_attention_pytorch_b200.ops.ring_flash_naive import ring_flash_attn

    n, b, h, d = 24, 2, 4, 16
    pm = make_position_map(layout, world, n)
    for ci, (name, causal, window, kmask, docs, gqa, empty) in enumerate(PORTABLE_CASES):
        hk = 2 if gqa else h
        q, k, v, do, sinks, km, ids = _global_case(ci, b, world * n, h, hk, d, docs, kmask, empty)
        pos = pm.positions(rank)
        qs, ks, vs, dos = (t[:, pos].clone() for t in (q, k, v, do))
        qs.requires_grad_(), ks.requires_grad_(), vs.requires_grad_()
        sk = sinks.clone().requires_grad_()
        out = ring_flash_attn(qs, ks, vs, None if km is None else km[:, pos], causal, 8, True,
                              layout == "striped", window, world, layout=layout,
                              document_ids=None if ids is None else ids[:, pos], sinks=sk)
        (out * dos).sum().backward()
        # oracle in fp64 over the whole sequence, global position order; this rank's rows and keys of it
        qf, kf, vf, sf = (t.double().requires_grad_() for t in (q, k, v, sinks))
        runs = document_runs(ids) if docs else None
        ref = attention_with_positions(qf, kf, vf, causal=causal, window=window, key_mask=km, q_doc=runs,
                                       k_doc=runs, sinks=sf)
        (ref[:, pos] * do[:, pos].double()).sum().backward()  # this rank's rows: its share of dsigma
        got_dk = torch.zeros_like(kf.grad)
        got_dk[:, pos] = ks.grad.double()
        dist.all_reduce(got_dk)
        got_dv = torch.zeros_like(vf.grad)
        got_dv[:, pos] = vs.grad.double()
        dist.all_reduce(got_dv)
        # dk / dv of the whole ring come from every rank's rows: compare them against the full loss
        qa, ka, va, sa = (t.double().requires_grad_() for t in (q, k, v, sinks))
        full = attention_with_positions(qa, ka, va, causal=causal, window=window, key_mask=km, q_doc=runs,
                                        k_doc=runs, sinks=sa)
        (full * do.double()).sum().backward()
        for label, got, want in (("out", out.double(), ref[:, pos]), ("dq", qs.grad.double(), qf.grad[:, pos]),
                                 ("dk", got_dk, ka.grad), ("dv", got_dv, va.grad),
                                 ("dsinks", sk.grad.double(), sf.grad)):
            err = (got - want).abs().max().item()
            assert err <= 2e-5 * (1 + want.abs().max().item()), (name, layout, world, rank, label, err)
        dsum = sk.grad.double().clone()
        dist.all_reduce(dsum)
        assert (dsum - sa.grad).abs().max().item() <= 1e-4, (name, "dsinks summed over ranks")


@pytest.mark.parametrize("world,layout", [(2, "plain"), (2, "zigzag"), (4, "striped"), (4, "zigzag")])
def test_portable_ring_matches_fp64_oracle(world, layout):
    run_distributed(_portable_worker, world, layout)


@pytest.mark.parametrize("name", [c[0] for c in PORTABLE_CASES])
def test_portable_single_rank_matches_fp64_oracle(name):
    from ring_attention_pytorch_b200.ops.ring_flash_naive import ring_flash_attn

    ci = [c[0] for c in PORTABLE_CASES].index(name)
    _, causal, window, kmask, docs, gqa, empty = PORTABLE_CASES[ci]
    h = 4
    hk = 2 if gqa else h
    q, k, v, do, sinks, km, ids = _global_case(ci, 2, 40, h, hk, 16, docs, kmask, empty)
    args = [t.clone().requires_grad_() for t in (q, k, v, sinks)]
    out = ring_flash_attn(*args[:3], km, causal, 16, max_lookback_seq_len=window, document_ids=ids, sinks=args[3])
    got = (out, *torch.autograd.grad(out, args, do))
    ref_in = [t.double().requires_grad_() for t in (q, k, v, sinks)]
    runs = document_runs(ids) if docs else None
    ref = attention_with_positions(*ref_in[:3], causal=causal, window=window, key_mask=km, q_doc=runs, k_doc=runs,
                                   sinks=ref_in[3])
    want = (ref, *torch.autograd.grad(ref, ref_in, do.double()))
    for label, g_, w_ in zip(("out", "dq", "dk", "dv", "dsinks"), got, want):
        assert g_.dtype == torch.float32
        assert (g_.double() - w_).abs().max().item() <= 2e-5 * (1 + w_.abs().max().item()), label
    if empty:
        assert (out[0] == 0).all() and (got[1][0] == 0).all()


@pytest.mark.parametrize("causal", [True, False])
def test_portable_cross_attention_more_queries_than_keys(causal):
    from ring_attention_pytorch_b200.ops.ring_flash_naive import ring_flash_attn

    torch.manual_seed(3)
    q, k, v = torch.randn(1, 30, 4, 16), torch.randn(1, 11, 2, 16), torch.randn(1, 11, 2, 16)
    sinks = torch.tensor([0.0, -1.0, 1.0, 3.0])
    do = torch.randn(1, 30, 4, 16)
    args = [t.clone().requires_grad_() for t in (q, k, v, sinks)]
    out = ring_flash_attn(*args[:3], None, causal, 8, sinks=args[3])
    got = (out, *torch.autograd.grad(out, args, do))
    ref_in = [t.double().requires_grad_() for t in (q, k, v, sinks)]
    ref, lse = attention_with_positions(*ref_in[:3], causal=causal, sinks=ref_in[3], return_lse=True)
    want = (ref, *torch.autograd.grad(ref, ref_in, do.double()))
    for label, g_, w_ in zip(("out", "dq", "dk", "dv", "dsinks"), got, want):
        assert (g_.double() - w_).abs().max().item() <= 2e-5 * (1 + w_.abs().max().item()), label
    if causal:  # the first 19 rows see no key: out 0, lse = sigma, dq 0
        assert (out[:, :19] == 0).all() and (got[1][:, :19] == 0).all()
        assert torch.allclose(lse[0, :, :19], sinks.double()[:, None].expand(4, 19))


def _decode_ref(q, k, v, sinks):
    """Head-first decode q [b, h, 1, d], k / v [b, hk, n, d] -> [b, h, 1, d] through the oracle, fp64."""
    out = attention_with_positions(q.double().transpose(1, 2), k.double().transpose(1, 2),
                                   v.double().transpose(1, 2), sinks=sinks.double())
    return out.transpose(1, 2)


def _decode_worker(rank, world, n):
    from ring_attention_pytorch_b200.ops.tree_decode import tree_attn_decode

    g = torch.Generator().manual_seed(7)
    q = torch.randn(2, 4, 1, 32, generator=g)
    k, v = torch.randn(2, 2, n, 32, generator=g), torch.randn(2, 2, n, 32, generator=g)
    sinks = torch.tensor([-2.0, 0.0, 1.5, 4.0])
    out = tree_attn_decode(q, k, v, sinks=sinks)
    assert (out.double() - _decode_ref(q, k, v, sinks)).abs().max() < 1e-5, (rank, n)


@pytest.mark.parametrize("world,n", [(1, 37), (2, 37), (4, 3), (4, 1)])
def test_portable_tree_decode(world, n):
    """``n < world``: some ranks hold no key; the sink still enters once."""
    if world == 1:
        _decode_worker(0, 1, n)
    else:
        run_distributed(_decode_worker, world, n)


def test_sinks_none_is_bitwise_unchanged():
    from ring_attention_pytorch_b200.ops.ring_flash_naive import ring_flash_attn
    from ring_attention_pytorch_b200.ops.ring_fp8 import dequantized_ring_flash_attn, quantize_fp8
    from ring_attention_pytorch_b200.ops.tree_decode import tree_attn_decode

    torch.manual_seed(0)
    q, k, v = torch.randn(1, 20, 4, 16), torch.randn(1, 20, 2, 16), torch.randn(1, 20, 2, 16)
    assert torch.equal(ring_flash_attn(q, k, v, None, True, 8), ring_flash_attn(q, k, v, None, True, 8, sinks=None))
    assert torch.equal(attention_with_positions(q, k, v, causal=True),
                       attention_with_positions(q, k, v, causal=True, sinks=None))
    qd, kd, vd = (t.transpose(1, 2) for t in (q[:, :1], k, v))
    assert torch.equal(tree_attn_decode(qd, kd, vd), tree_attn_decode(qd, kd, vd, sinks=None))
    (q8, sq), (k8, sk), (v8, sv) = (quantize_fp8(t, 1) for t in (q, k, v))
    assert torch.equal(dequantized_ring_flash_attn(q8, k8, v8, sq, sk, sv, causal=True),
                       dequantized_ring_flash_attn(q8, k8, v8, sq, sk, sv, causal=True, sinks=None))


def test_invalid_sinks_raise():
    from ring_attention_pytorch_b200.ops.ring_flash_naive import ring_flash_attn
    from ring_attention_pytorch_b200.ops.ring_fp8 import quantize_fp8, ring_flash_attn_fp8
    from ring_attention_pytorch_b200.ops.tree_decode import tree_attn_decode

    q, k, v = torch.randn(1, 8, 4, 16), torch.randn(1, 8, 2, 16), torch.randn(1, 8, 2, 16)
    for bad in (torch.zeros(2), torch.zeros(4, 1), torch.zeros(4, dtype=torch.int64), torch.zeros(4, device="meta")):
        with pytest.raises(ValueError):
            ring_flash_attn(q, k, v, sinks=bad)
        with pytest.raises(ValueError):
            tree_attn_decode(q[:, :1].transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), sinks=bad)
    (q8, sq), (k8, sk), (v8, sv) = (quantize_fp8(t, 1) for t in (q, k, v))
    with pytest.raises(ValueError):  # the fp8 op is forward only: a sink that requires grad cannot be honoured
        ring_flash_attn_fp8(q8, k8, v8, sq, sk, sv, sinks=torch.zeros(4, requires_grad=True))
    out = ring_flash_attn_fp8(q8, k8, v8, sq, sk, sv, causal=True, sinks=torch.ones(4))
    assert out.dtype == torch.bfloat16 and torch.isfinite(out.float()).all()


def test_module_state_dict_with_and_without_sinks():
    from ring_attention_pytorch_b200 import RingAttention, RingTransformer

    plain = RingAttention(32, heads=4, dim_head=8, use_cuda_kernel=False)
    with_sinks = RingAttention(32, heads=4, dim_head=8, use_cuda_kernel=False, attn_sinks=True)
    assert "sinks" not in plain.state_dict() and with_sinks.state_dict()["sinks"].shape == (4,)
    assert set(with_sinks.state_dict()) - set(plain.state_dict()) == {"sinks"}
    with_sinks.load_state_dict(plain.state_dict(), strict=False)  # a checkpoint without sinks loads
    plain.load_state_dict({k: v for k, v in with_sinks.state_dict().items() if k != "sinks"})
    kw = dict(num_tokens=16, dim=32, depth=2, heads=4, dim_head=8, use_cuda_kernel=False)
    keys = set(RingTransformer(attn_sinks=True, **kw).state_dict()) - set(RingTransformer(**kw).state_dict())
    assert keys == {"layers.0.0.sinks", "layers.1.0.sinks"}


def _module_worker(rank, world):
    from ring_attention_pytorch_b200 import RingAttention

    torch.manual_seed(0)
    kw = dict(dim=32, heads=4, dim_head=8, num_grouped_query_heads=2, causal=True, use_cuda_kernel=False,
              attn_sinks=True, bucket_size=4, ring_seq_size=8)
    ring = RingAttention(ring_attn=True, auto_shard_seq=True, **kw)
    with torch.no_grad():
        ring.sinks.copy_(torch.tensor([-1.0, 0.5, 2.0, 4.0]))
    regular = RingAttention(force_regular_attn=True, **kw)
    regular.load_state_dict(ring.state_dict())
    x = torch.randn(2, 16, 32, generator=torch.Generator().manual_seed(1))
    out_ring, out_reg = ring(x), regular(x)
    assert (out_ring - out_reg).abs().max() < 1e-5
    out_ring.square().sum().backward()
    out_reg.square().sum().backward()
    g_ring, g_reg = ring.sinks.grad.clone(), regular.sinks.grad.clone()
    dist.all_reduce(g_ring)
    dist.all_reduce(g_reg)
    assert (g_ring - g_reg).abs().max() < 1e-4 * (1 + g_reg.abs().max())


def test_module_ring_matches_force_regular_attn():
    run_distributed(_module_worker, 2)


# ================================================================================================
# CPU: the error rule rejects sink mistakes in a torch model of the kernel's algorithm
# ================================================================================================
def emulate_sink_ring(qs, ks, vs, dos, sinks, *, layout, causal, softclamp=0.0, mutant=None):
    """The forward kernel's algorithm with sinks on every rank of an emulated ring: the sink as initial state
    (m = sigma log2 e, l = 1), hops in ``ring_hop_owners`` order, 128-key tiles, the lazy maximum, P rounded to bf16,
    out rounded to bf16; then dsigma from lse and delta = rowsum(dO * out).  ``mutant``: per_hop (the sink re-added at
    every hop), kv_head (sigma indexed by the kv head), softclamp (sigma passed through softclamp), dsink_sign."""
    world, n = len(qs), qs[0].shape[1]
    b, _, h, d = qs[0].shape
    hk = ks[0].shape[2]
    pm = make_position_map(layout, world, n)
    heads = torch.arange(h) % hk
    k_all = torch.cat([k.float() for k in ks], 1)[:, :, heads]
    v_all = torch.cat([v.float() for v in vs], 1)[:, :, heads]
    k_pos = torch.cat([pm.positions(r) for r in range(world)])
    sig = sinks.float()[heads] if mutant == "kv_head" else sinks.float()
    if mutant == "softclamp":
        sig = (sig / softclamp).tanh() * softclamp
    sig2 = (sig / math.log(2.0))[None, :, None, None]
    outs, lses, dsinks = [], [], []
    for r in range(world):
        s = torch.einsum("bihd,bjhd->bhij", qs[r].float(), k_all) * d ** -0.5
        if softclamp:
            s = (s / softclamp).tanh() * softclamp
        s2 = s.masked_fill(~gdc._visible(pm.positions(r), k_pos, causal, None), -math.inf) / math.log(2.0)
        m = sig2.expand(b, h, n, 1).clone()
        l = torch.ones(b, h, n, 1)
        o = torch.zeros(b, h, n, d)
        hop_first = {int(t[0]) // n: int(t[0]) for t in gdc.visit_order(pm, r, causal, None) if int(t[0]) % n == 0}
        for idx in gdc.visit_order(pm, r, causal, None):
            if mutant == "per_hop" and int(idx[0]) in hop_first.values() and int(idx[0]) // n != r:
                l = l + torch.exp2(sig2 - m)
            st = s2[..., idx]
            cmax = st.amax(-1, keepdim=True)
            raise_ = cmax > m + gdc.LAZY_THRESHOLD
            new = torch.where(raise_, torch.maximum(m, cmax), m)
            factor = torch.exp2(m - new)
            l, o, m = l * factor, o * factor, new
            p = torch.exp2(st - m)
            l = l + p.sum(-1, keepdim=True)
            o = o + p.bfloat16().float() @ v_all[:, idx].permute(0, 2, 1, 3)
        out = (o / l).permute(0, 2, 1, 3).bfloat16().float()
        lse = ((m + torch.log2(l)) * math.log(2.0)).squeeze(-1)
        delta = (dos[r].float() * out).sum(-1).transpose(1, 2)  # [b, h, n]
        ds = -(torch.exp(sinks.float()[None, :, None] - lse) * delta).sum(dim=(0, 2))
        outs.append(out)
        lses.append(lse)
        dsinks.append(-ds if mutant == "dsink_sign" else ds)
    return outs, lses, dsinks


def _sink_rule_case(case):
    world, layout, h, hk, softclamp, kind = {
        "ring4_near": (4, "striped", 2, 2, 0.0, "near"),
        "gqa_mix": (1, "plain", 4, 2, 0.0, "mix"),
        "softclamp": (1, "plain", 2, 2, 5.0, "near"),
        "ring2_below": (2, "zigzag", 2, 1, 0.0, "mix"),
    }[case]
    qs, ks, vs, dos = gdc.make_case_inputs(None, world, 1, 256, h, hk, 64, torch.bfloat16, layout, True, None, seed=2,
                                           grad=True, device="cpu")
    sinks = gdc.make_sinks(kind, qs, ks, softclamp)
    if case == "gqa_mix":  # heads sharing a kv head get very different sinks
        sinks = torch.tensor([-4.0, 1.0, 6.0, 3.0]) + sinks.mean()
    if case == "softclamp":
        sinks = torch.full((h,), 4.0)
    args = dict(layout=layout, causal=True, softclamp=softclamp)
    ref = gdc._ref_ring(qs, ks, vs, layout, True, None, softclamp, None, dos=dos, sinks=sinks)
    lowp = gdc._ref_ring(qs, ks, vs, layout, True, None, softclamp, None, dos=dos, dtype=torch.bfloat16, sinks=sinks)
    return (qs, ks, vs, dos, sinks), args, ref, lowp


def _sink_rule(got, ref, lowp):
    res = {"out": gdc.noise_bound(got[0], ref[0], lowp[0]), "lse": gdc.noise_bound(got[1], ref[1], lowp[1]),
           "dsinks": gdc.noise_bound(got[2], [g[3] for g in ref[2]], [g[3] for g in lowp[2]])}
    return max(r["ratio"] for r in res.values()), res


@pytest.mark.parametrize("case", ["ring4_near", "gqa_mix", "softclamp", "ring2_below"])
def test_rule_accepts_the_sink_algorithm(case):
    inputs, args, ref, lowp = _sink_rule_case(case)
    worst, res = _sink_rule(emulate_sink_ring(*inputs, **args), ref, lowp)
    print(f"[accept] sinks {case}: worst error/bound {worst:.3f}")
    assert worst <= 1.0, res


@pytest.mark.parametrize("mutant,case", [("per_hop", "ring4_near"), ("kv_head", "gqa_mix"),
                                         ("softclamp", "softclamp"), ("dsink_sign", "ring2_below")])
def test_rule_rejects_sink_mistakes(mutant, case):
    inputs, args, ref, lowp = _sink_rule_case(case)
    worst, res = _sink_rule(emulate_sink_ring(*inputs, **args, mutant=mutant), ref, lowp)
    print(f"[reject] sinks {mutant} on {case}: worst error/bound {worst:.2f}")
    assert worst >= 3.0, res


# ================================================================================================
# GPU: the kernels under the rule
# ================================================================================================
def _report(name, res):
    for key, r in res.items():
        if isinstance(r, dict) and "bound" in r:
            print(f"[{name}] {key}: err {r['err']:.3e} lowp {r['lowp_err']:.3e} bound {r['bound']:.3e} "
                  f"ratio {r['ratio']:.3f}")


FWD = {
    "below_n257": dict(n=257, h=2, sinks="below"),
    "near_causal_n1000": dict(n=1000, h=2, causal=True, sinks="near"),
    "above_causal": dict(n=384, h=2, causal=True, sinks="above"),
    "mix_gqa_hk1_b3": dict(n=129, h=8, hk=1, b=3, sinks="mix"),
    "mix_d64_fp16": dict(n=127, h=4, hk=2, d=64, dtype="fp16", causal=True, sinks="mix"),
    "above_n1": dict(n=1, h=2, sinks="above"),
    "near_n64_d64": dict(n=64, h=2, d=64, sinks="near"),
    "window1_near": dict(n=257, h=2, causal=True, window=1, sinks="near"),
    "window128_mix": dict(n=300, h=4, causal=True, window=128, sinks="mix"),
    "softclamp_near": dict(n=200, h=2, softclamp=20.0, regime="softclamp_sat", sinks="near"),
    "late_spike_near": dict(n=384, h=2, causal=True, regime="late_spike", sinks="near"),
    "late_spike_above": dict(n=257, h=2, regime="late_spike", sinks="above"),
    "empty_rows_mix": dict(n=200, h=4, b=2, regime="empty_rows", sinks="mix"),
    "docs_masked_near": dict(n=384, h=2, b=2, kmask=True, docs="masked", sinks="near"),
    "docs_ragged_causal_mix": dict(n=300, h=4, causal=True, docs="ragged", sinks="mix"),
    "ring2_causal_near": dict(world=2, n=256, h=2, causal=True, sinks="near"),
    "ring3_empty_above": dict(world=3, n=128, h=2, b=2, regime="empty_rows", sinks="above"),
    "ring4_striped_mix_hk1": dict(world=4, n=256, h=4, hk=1, layout="striped", causal=True, sinks="mix"),
    "ring4_zigzag_fp16_spike": dict(world=4, n=128, h=2, layout="zigzag", causal=True, dtype="fp16",
                                    regime="late_spike", sinks="near"),
    "ring2_docs_window": dict(world=2, n=256, h=2, causal=True, window=128, docs="ragged", sinks="mix"),
}
HOP = {k: v for k, v in FWD.items() if v.get("world", 1) > 1}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FWD))
def test_forward_with_sinks(name):
    res = gdc.case_fwd(**FWD[name])
    _report(name, res)
    assert res["ok"], res


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(HOP))
def test_hopwise_forward_with_sinks(name):
    res = gdc.case_fwd(hopwise=True, **HOP[name])
    _report(f"{name} hop", res)
    assert res["ok"], res


BWD = {
    "near_causal": dict(n=384, h=2, causal=True, sinks="near"),
    "mix_gqa_hk1": dict(n=129, h=8, hk=1, b=3, sinks="mix"),
    "above_causal": dict(n=257, h=2, causal=True, sinks="above"),
    "below_two_kernel": dict(n=257, h=2, causal=True, sinks="below", fused=False),
    "mix_d64_fp16": dict(n=129, h=4, d=64, dtype="fp16", causal=True, sinks="mix"),
    "window1_near_two_kernel": dict(n=257, h=2, causal=True, window=1, sinks="near", fused=False),
    "window128_mix": dict(n=300, h=4, causal=True, window=128, sinks="mix"),
    "spike_near": dict(n=384, h=2, causal=True, regime="late_spike", sinks="near"),
    "empty_rows_mix": dict(n=200, h=4, b=2, regime="empty_rows", sinks="mix"),
    "empty_rows_two_kernel": dict(n=200, h=2, b=2, regime="empty_rows", sinks="above", fused=False),
    "docs_masked_near": dict(n=384, h=2, b=2, kmask=True, docs="masked", sinks="near"),
    "ring2_hop_near": dict(world=2, n=256, h=2, causal=True, sinks="near", hopwise=True),
    "ring4_striped_mix": dict(world=4, n=256, h=4, hk=1, layout="striped", causal=True, sinks="mix"),
    "ring4_zigzag_hop_above": dict(world=4, n=128, h=2, layout="zigzag", causal=True, sinks="above", hopwise=True),
    "ring3_two_kernel_mix": dict(world=3, n=128, h=4, hk=2, causal=True, sinks="mix", fused=False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BWD))
def test_backward_with_sinks(name):
    """dq, dk, dv and every rank's dsigma under the rule; a second backward gives bitwise the same dsigma."""
    res = gdc.case_bwd(**BWD[name])
    _report(name, res)
    assert res["dsinks_deterministic"], res
    assert res["ok"], res


@pytest.mark.gpu
@pytest.mark.parametrize("backward", ["fused", "two_kernel"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_op_with_sinks(backward, dtype):
    """Through the autograd op: the gradient comes back in the sinks' dtype and is bitwise reproducible."""
    from ring_attention_pytorch_b200.ops import ring_cuda

    old = dict(ring_cuda.CONFIG)
    ring_cuda.CONFIG["backward"] = backward
    try:
        torch.manual_seed(0)
        b, n, h, hk, d = 2, 333, 4, 2, 128
        q = torch.randn(b, n, h, d, device="cuda", dtype=dtype, requires_grad=True)
        k = torch.randn(b, n, hk, d, device="cuda", dtype=dtype, requires_grad=True)
        v = torch.randn(b, n, hk, d, device="cuda", dtype=dtype, requires_grad=True)
        sinks = torch.tensor([-2.0, 0.0, 2.0, 12.0], device="cuda", dtype=dtype, requires_grad=True)
        do = torch.randn(b, n, h, d, device="cuda", dtype=dtype)
        out = ring_cuda.ring_flash_attn_cuda(q, k, v, None, True, sinks=sinks)
        got = (out, *torch.autograd.grad(out, (q, k, v, sinks), do))
        again = torch.autograd.grad(ring_cuda.ring_flash_attn_cuda(q, k, v, None, True, sinks=sinks), sinks, do)[0]
        assert got[4].dtype == dtype and torch.equal(got[4], again)

        def oracle(dt):
            xs = [t.detach().to(dt).requires_grad_() for t in (q, k, v, sinks)]
            o = attention_with_positions(*xs[:3], causal=True, sinks=xs[3])
            return (o.detach(), *torch.autograd.grad(o, xs, do.to(dt)))

        ref, lowp = oracle(torch.float32), oracle(dtype)
        for name, g_, r_, l_ in zip(("out", "dq", "dk", "dv", "dsinks"), got, ref, lowp):
            res = gdc.noise_bound(g_, r_, l_, None if name == "out" else gdc.CAP_GRAD_REL * r_.abs().max().item())
            _report(f"op {backward} {dtype}", {name: res})
            assert res["ok"], (name, res)
    finally:
        ring_cuda.CONFIG.update(old)


def _fp8_sink_case(kind, world=1, b=1, n=2048, h=2, hk=None, layout="plain", causal=True, hopwise=False, seed=0):
    from ring_attention_pytorch_b200 import quantize_fp8
    from ring_attention_pytorch_b200.ops.fused import emulate_ring_forward, emulate_ring_forward_fp8

    hk = hk or h
    qs, ks, vs, _ = gdc.make_case_inputs(None, world, b, n, h, hk, 128, torch.float32, layout, causal, None,
                                         seed=seed)
    kq, kd = quantize_fp8(torch.cat(ks, 1), 1)
    vq, vd = quantize_fp8(torch.cat(vs, 1), 1)
    qq = [quantize_fp8(q, 1) for q in qs]
    k8, v8 = list(kq.split(n, 1)), list(vq.split(n, 1))

    def deq(t8, ds):
        return t8.float() * ds[:, None, :, None]

    qf = [deq(q, s) for q, s in qq]
    kf, vf = [deq(t, kd) for t in k8], [deq(t, vd) for t in v8]
    sinks = gdc.make_sinks(kind, qf, kf)
    outs, _ = emulate_ring_forward_fp8([q for q, _ in qq], k8, v8, [s for _, s in qq], kd, vd, layout=layout,
                                       causal=causal, hopwise=hopwise, sinks=sinks)
    refs, _ = gdc._ref_ring(qf, kf, vf, layout, causal, None, 0.0, None, sinks=sinks)
    o16, _ = emulate_ring_forward([t.bfloat16() for t in qf], [t.bfloat16() for t in kf], [t.bfloat16() for t in vf],
                                  layout=layout, causal=causal, hopwise=hopwise, sinks=sinks)
    torch.cuda.synchronize()

    def rel(xs):
        num = sum((x.float() - r).pow(2).sum() for x, r in zip(xs, refs))
        return (num / sum(r.pow(2).sum() for r in refs)).sqrt().item()

    return rel(outs), rel(o16)


FP8 = {
    "near": dict(kind="near"),
    "above": dict(kind="above"),
    "mix_gqa_b2": dict(kind="mix", b=2, h=6, hk=2),
    "below_ring2_hop": dict(kind="below", world=2, n=1024, hopwise=True),
    "mix_ring4_striped": dict(kind="mix", world=4, n=512, layout="striped", h=3),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FP8))
def test_fp8_forward_with_sinks(name):
    """Bounds of tests/test_fp8_prefill.py: relative RMS error <= 5e-2 and <= 13x the bf16 kernel's."""
    e8, e16 = _fp8_sink_case(**FP8[name])
    print(f"[fp8 sinks {name}] rel rms fp8 {e8:.3e} bf16 {e16:.3e} ratio {e8 / e16:.2f}")
    assert e8 <= 5e-2 and e8 <= 13.0 * e16


@pytest.mark.gpu
@pytest.mark.parametrize("tensor_core", [True, False])
@pytest.mark.parametrize("cache", ["bf16", "fp8"])
@pytest.mark.parametrize("n", [1, 300, 4099])
def test_tree_decode_kernel_with_sinks(tensor_core, cache, n):
    from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc

    old = dict(tdc.CONFIG)
    tdc.CONFIG["tensor_core"] = "on" if tensor_core else "off"
    try:
        torch.manual_seed(n)
        b, h, hk, d = 3, 8, 2, 128
        q = torch.randn(b, h, 1, d, device="cuda", dtype=torch.bfloat16)
        k = torch.randn(b, hk, n, d, device="cuda", dtype=torch.bfloat16)
        v = torch.randn(b, hk, n, d, device="cuda", dtype=torch.bfloat16)
        sinks = gdc.make_sinks("mix", [q.transpose(1, 2)], [k.transpose(1, 2)])
        kw = {}
        if cache == "fp8":
            k8, v8 = k.float().to(torch.float8_e4m3fn), v.float().to(torch.float8_e4m3fn)
            k, v = k8.float(), v8.float()
            kw = dict(k_scale=torch.ones(b * hk, device="cuda"), v_scale=torch.ones(b * hk, device="cuda"))
            out = tdc.tree_decode_cuda(q, k8, v8, dim_v=d, sinks=sinks, **kw)
        else:
            out = tdc.tree_decode_cuda(q, k, v, dim_v=d, sinks=sinks)
        torch.cuda.synchronize()

        def dense(dt):
            return attention_with_positions(q.transpose(1, 2).to(dt), k.transpose(1, 2).to(dt),
                                            v.transpose(1, 2).to(dt), sinks=sinks.to(dt)).transpose(1, 2)

        res = gdc.noise_bound(out, dense(torch.float32), dense(torch.bfloat16), gdc.CAP_OUT)
        _report(f"decode tc={tensor_core} {cache} n={n}", {"out": res})
        assert res["ok"], res
    finally:
        tdc.CONFIG.update(old)


def _real_ring_worker(rank, world, layout, backward, memory):
    from ring_attention_pytorch_b200.ops import ring_cuda

    ring_cuda.CONFIG["backward"] = backward
    ring_cuda.CONFIG["memory"] = memory
    torch.manual_seed(0)
    b, n, h, hk, d = 1, 640, 4, 2, 128
    dev = torch.device("cuda", rank)
    pm = make_position_map(layout, world, n)
    qs = [torch.randn(b, n, h, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    ks = [torch.randn(b, n, hk, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    vs = [torch.randn(b, n, hk, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    gs = [torch.randn(b, n, h, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    sinks = torch.tensor([-1.0, 1.0, 3.0, 6.0], device=dev, requires_grad=True)
    q, k, v = (t[rank].clone().requires_grad_() for t in (qs, ks, vs))
    out = ring_cuda.ring_flash_attn_cuda(q, k, v, None, True, 1024, True, layout == "striped", None, world,
                                         layout=layout, sinks=sinks)
    dq, dk, dv, ds = torch.autograd.grad(out, (q, k, v, sinks), gs[rank])
    _, _, ref = gdc._ref_ring(qs, ks, vs, layout, True, None, 0.0, None, dos=gs, sinks=sinks.detach())
    outs, _ = gdc._ref_ring(qs, ks, vs, layout, True, None, 0.0, None, sinks=sinks.detach())
    assert (out.float() - outs[rank]).abs().max() < 3e-2
    for got, want in zip((dq, dk, dv, ds), ref[rank]):
        assert (got.float() - want).abs().max() / want.abs().max() < 3e-2
    dist.barrier()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("layout,backward,memory", [("striped", "fused", "gather"), ("zigzag", "fused", "ring"),
                                                    ("plain", "two_kernel", "gather")])
def test_real_ring_with_sinks(world, layout, backward, memory):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    run_distributed(_real_ring_worker, world, layout, backward, memory, backend="nccl", timeout=600.0)


def _real_decode_worker(rank, world, n):
    from ring_attention_pytorch_b200.ops.tree_decode import tree_attn_decode

    torch.manual_seed(0)
    dev = torch.device("cuda", rank)
    q = torch.randn(2, 8, 1, 128, device=dev, dtype=torch.bfloat16)
    k = torch.randn(2, 4, n, 128, device=dev, dtype=torch.bfloat16)
    v = torch.randn(2, 4, n, 128, device=dev, dtype=torch.bfloat16)
    sinks = torch.linspace(-2.0, 6.0, 8, device=dev)
    out = tree_attn_decode(q, k, v, sinks=sinks)
    ref = _decode_ref(q, k, v, sinks)
    assert (out.double() - ref).abs().max() < 2e-2
    dist.barrier()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("n", [4099, 1])
def test_real_tree_decode_with_sinks(world, n):
    """The P2P merge, or the NVLS merge where the NVSwitch offers multicast; n = 1 leaves ranks without keys."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    run_distributed(_real_decode_worker, world, n, backend="nccl", timeout=600.0)
