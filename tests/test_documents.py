"""Document masking for packed sequences (``document_ids``): interval builder, portable op, gloo rings, modules and
the sm_90a kernels.

A document is a maximal run of equal ids in global position order; a query sees only keys of its own run, on top of
the causal rule, the look-back window and the key mask.
"""
import os
import random
import sys

import pytest
import torch
import torch.distributed as dist

from dist_utils import run_distributed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

LAYOUTS = ("plain", "striped", "zigzag")


def _brute_spans(ids):
    """[total] global ids -> [total, 2] run intervals, by scanning left and right from every position."""
    total = len(ids)
    out = []
    for p in range(total):
        s = p
        while s > 0 and ids[s - 1] == ids[p]:
            s -= 1
        e = p + 1
        while e < total and ids[e] == ids[p]:
            e += 1
        out.append((s, e))
    return torch.tensor(out)


def _random_ids(rng, b, total):
    rows = []
    for _ in range(b):
        vocab = rng.choice([1, 2, 3, 50])
        run = rng.choice([1, 2, 5, 40])
        row, cur = [], rng.randrange(vocab)
        while len(row) < total:
            row += [cur] * rng.randint(1, run)
            cur = rng.randrange(vocab)
        rows.append(row[:total])
    return torch.tensor(rows)


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("world", range(1, 9))
def test_interval_builder_matches_brute_force(layout, world):
    from ring_attention_pytorch_b200.parallel.documents import document_spans
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    rng = random.Random(world * 10 + LAYOUTS.index(layout))
    for trial in range(6):
        n = 2 * rng.randint(1, 12)
        b = rng.randint(1, 3)
        ids = _random_ids(rng, b, world * n)
        pm = make_position_map(layout, world, n)
        shards = torch.stack([ids[:, pm.positions(r)] for r in range(world)])
        spans = document_spans(shards, pm)
        assert spans.dtype == torch.int32 and spans.shape == (world, b, n, 2)
        for bi in range(b):
            want = _brute_spans(ids[bi].tolist())
            for r in range(world):
                assert torch.equal(spans[r, bi].long(), want[pm.positions(r)]), (trial, r, bi)


def _split_reference(q, k, v, g, ids, **kw):
    """Run every document of a [1, n] row through ring_flash_attn on its own; returns (out, dq, dk, dv)."""
    from ring_attention_pytorch_b200 import ring_flash_attn

    outs, dqs, dks, dvs = [], [], [], []
    bounds = [0] + [i for i in range(1, ids.shape[1]) if ids[0, i] != ids[0, i - 1]] + [ids.shape[1]]
    for s, e in zip(bounds[:-1], bounds[1:]):
        qs, ks, vs = (t[:, s:e].detach().clone().requires_grad_() for t in (q, k, v))
        o = ring_flash_attn(qs, ks, vs, **kw)
        dq, dk, dv = torch.autograd.grad(o, (qs, ks, vs), g[:, s:e])
        outs.append(o)
        dqs.append(dq)
        dks.append(dk)
        dvs.append(dv)
    return [torch.cat(t, 1) for t in (outs, dqs, dks, dvs)]


@pytest.mark.parametrize("causal,window,hk,softclamp", [(True, None, 4, False), (False, None, 4, False),
                                                          (True, 6, 2, False), (False, None, 1, True),
                                                          (True, None, 2, True)])
def test_portable_packed_equals_separate_documents(causal, window, hk, softclamp):
    from ring_attention_pytorch_b200 import ring_flash_attn

    torch.manual_seed(0)
    n, h, d = 40, 4, 8
    ids = torch.tensor([[0] * 7 + [1] + [2] * 13 + [0] * 9 + [5] * 10])  # a reused id and a length-1 document
    q, k, v, g = torch.randn(1, n, h, d), torch.randn(1, n, hk, d), torch.randn(1, n, hk, d), torch.randn(1, n, h, d)
    kw = dict(causal=causal, bucket_size=8, max_lookback_seq_len=window, softclamp_qk_sim=softclamp,
              softclamp_value=5.0)
    qp, kp, vp = (t.clone().requires_grad_() for t in (q, k, v))
    out = ring_flash_attn(qp, kp, vp, document_ids=ids, **kw)
    got = (out, *torch.autograd.grad(out, (qp, kp, vp), g))
    want = _split_reference(q, k, v, g, ids, **kw)
    for a, b in zip(got, want):
        assert torch.allclose(a, b, atol=2e-5), (a - b).abs().max()


def test_portable_one_document_equals_none():
    from ring_attention_pytorch_b200 import ring_flash_attn

    torch.manual_seed(1)
    q, k, v, g = (torch.randn(2, 33, 2, 8) for _ in range(4))
    for causal in (False, True):
        res = []
        for ids in (None, torch.full((2, 33), 7)):
            qp, kp, vp = (t.clone().requires_grad_() for t in (q, k, v))
            o = ring_flash_attn(qp, kp, vp, causal=causal, bucket_size=8, document_ids=ids)
            res.append((o, *torch.autograd.grad(o, (qp, kp, vp), g)))
        for a, b in zip(*res):
            assert torch.equal(a, b)


def test_fully_masked_document_gives_zeros_not_nan():
    from ring_attention_pytorch_b200 import ring_flash_attn

    q, k, v = (torch.randn(1, 12, 2, 8) for _ in range(3))
    ids = torch.tensor([[0] * 4 + [1] * 4 + [2] * 4])
    mask = ids != 1
    out = ring_flash_attn(q, k, v, mask, False, document_ids=ids)
    assert torch.isfinite(out).all() and out[:, 4:8].abs().max() == 0


def test_cross_attention_with_documents_raises():
    from ring_attention_pytorch_b200 import ring_flash_attn

    q, k = torch.randn(1, 8, 2, 8), torch.randn(1, 12, 2, 8)
    with pytest.raises(ValueError, match="self-attention"):
        ring_flash_attn(q, k, k, document_ids=torch.zeros(1, 8, dtype=torch.long))


# ------------------------------------------------------------------------------------------------
# gloo rings
# ------------------------------------------------------------------------------------------------
def _ring_doc_worker(rank, world, layout):
    from ring_attention_pytorch_b200 import ring_flash_attn
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.parallel.documents import document_runs
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    torch.manual_seed(0)
    b, n, h, hk, d = 2, 12, 4, 2, 8
    pm = make_position_map(layout, world, n)
    ids = torch.stack([torch.tensor(sorted(random.Random(s).choices(range(6), k=world * n))) for s in range(b)])
    ids[1, ::5] = 9  # length-1 documents and a reused id
    runs = document_runs(ids)  # [b, total] labels in global order
    for causal, window in ((False, None), (True, None), (True, 7)):
        qs = [torch.randn(b, n, h, d) for _ in range(world)]
        ks = [torch.randn(b, n, hk, d) for _ in range(world)]
        vs = [torch.randn(b, n, hk, d) for _ in range(world)]
        gs = [torch.randn(b, n, h, d) for _ in range(world)]
        q, k, v = (t[rank].clone().requires_grad_() for t in (qs, ks, vs))
        out = ring_flash_attn(q, k, v, None, causal, 4, True, layout == "striped", window, world, layout=layout,
                              document_ids=ids[:, pm.positions(rank)])
        dq, dk, dv = torch.autograd.grad(out, (q, k, v), gs[rank])

        qf = [t.clone().requires_grad_() for t in qs]
        kf = [t.clone().requires_grad_() for t in ks]
        vf = [t.clone().requires_grad_() for t in vs]
        k_pos = torch.cat([pm.positions(r) for r in range(world)])
        loss, outs = 0, []
        for r in range(world):
            o = attention_with_positions(qf[r], torch.cat(kf, 1), torch.cat(vf, 1), pm.positions(r), k_pos,
                                         causal=causal, window=window, q_doc=runs[:, pm.positions(r)],
                                         k_doc=runs[:, k_pos])
            outs.append(o)
            loss = loss + (o * gs[r]).sum()
        loss.backward()
        assert torch.allclose(out, outs[rank], atol=2e-5), (causal, (out - outs[rank]).abs().max())
        for got, ref in ((dq, qf[rank].grad), (dk, kf[rank].grad), (dv, vf[rank].grad)):
            assert torch.allclose(got, ref, atol=5e-5), (causal, (got - ref).abs().max())


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("world", [2, 4])
def test_gloo_ring_documents_match_oracle(world, layout):
    run_distributed(_ring_doc_worker, world, layout)


def _transformer_doc_worker(rank, world, striped):
    from math import ceil

    from ring_attention_pytorch_b200 import RingTransformer
    from ring_attention_pytorch_b200.models.ring_attention import _pad_tokens, stripe

    torch.manual_seed(0)
    seq_len = 31  # needs padding to a multiple of ring_seq_size * world
    ring_seq_size = ceil(seq_len / world)
    kw = dict(num_tokens=64, dim=16, depth=2, causal=True, dim_head=8, heads=4, num_grouped_query_heads=2,
              bucket_size=ring_seq_size, use_cuda_kernel=False)
    ring = RingTransformer(ring_attn=True, striped_ring_attn=striped, ring_seq_size=ring_seq_size, **kw)
    flash = RingTransformer(ring_attn=False, **kw)
    flash.load_state_dict(ring.state_dict())
    torch.manual_seed(100 + rank)
    tokens = torch.randint(0, 64, (2, seq_len))
    ids = torch.tensor([[0] * 9 + [1] * 3 + [0] * 11 + [4] * 8, [2] * 1 + [3] * 20 + [5] * 10])
    g = torch.randn(2, seq_len, 64)
    lr = ring(tokens, document_ids=ids)
    lf = flash(tokens, document_ids=ids)
    assert not torch.allclose(lf, flash(tokens), atol=1e-3), "documents must change the result"
    assert torch.allclose(lr, lf, atol=5e-5), (lr - lf).abs().max()
    (lr * g).sum().backward()
    (lf * g).sum().backward()
    for (name, pr), (_, pf) in zip(ring.named_parameters(), flash.named_parameters()):
        gr, gf = pr.grad.clone(), pf.grad.clone()
        dist.all_reduce(gr)
        dist.all_reduce(gf)
        assert torch.allclose(gr, gf, atol=5e-4), (name, (gr - gf).abs().max())

    # return_loss shifts the ids with the input; the ring loss is the mean over this rank's valid labels
    loss_r = ring(tokens, return_loss=True, document_ids=ids)
    loss_f = flash(tokens, return_loss=True, document_ids=ids)
    valid = _pad_tokens(torch.ones(1, seq_len - 1, dtype=torch.bool), ring_seq_size, False)
    if striped:
        valid = stripe(valid, ring_seq_size)
    count = torch.tensor(float(valid[0, rank * ring_seq_size:(rank + 1) * ring_seq_size].sum()))
    num = loss_r.detach() * count
    dist.all_reduce(num)
    dist.all_reduce(count)
    ref = loss_f.detach().clone()
    dist.all_reduce(ref)
    assert torch.allclose(num / count, ref / world, atol=1e-5), (num / count, ref / world)


@pytest.mark.parametrize("striped", [False, True])
def test_ring_transformer_documents_match_unsharded(striped):
    run_distributed(_transformer_doc_worker, 4, striped)


# ================================================================================================
# GPU: the sm_90a kernels
# ================================================================================================
def _cases():
    import gpu_dev_check

    return gpu_dev_check


DOC_FWD_CASES = {
    "d128_causal_ragged": dict(n=1000, h=2, causal=True, docs="ragged"),
    "d128_noncausal_tiny": dict(n=512, h=2, docs="tiny"),
    "d64_causal_len1": dict(n=777, d=64, h=4, causal=True, docs="len1"),
    "d64_noncausal_ragged": dict(n=640, d=64, h=2, docs="ragged", b=2),
    "window_ragged": dict(n=1024, h=2, causal=True, window=200, docs="ragged"),
    "gqa_causal_reuse": dict(n=512, h=8, hk=2, causal=True, docs="reuse"),
    "kmask_masked_doc": dict(n=384, h=2, kmask=True, b=2, docs="masked"),
    "softclamp_tiny": dict(n=384, h=2, softclamp=20.0, causal=True, docs="tiny"),
    "fp16_causal_ragged": dict(n=512, h=2, causal=True, dtype="fp16", docs="ragged"),
    "span_one_rank": dict(n=300, h=2, causal=True, docs="span"),
    "ring1_plain_len1": dict(world=1, n=256, h=2, causal=True, docs="len1"),
    "ring2_plain_ragged": dict(world=2, n=256, h=2, docs="ragged"),
    "ring2_zigzag_causal_span": dict(world=2, n=384, h=2, layout="zigzag", causal=True, docs="span"),
    "ring4_striped_causal_gqa_tiny": dict(world=4, n=384, h=4, hk=2, layout="striped", causal=True, docs="tiny"),
    "ring4_zigzag_causal_ragged": dict(world=4, n=512, h=2, layout="zigzag", causal=True, docs="ragged"),
    "ring4_plain_window_span": dict(world=4, n=256, h=2, causal=True, window=300, docs="span"),
    "ring4_plain_kmask_masked": dict(world=4, n=200, h=2, kmask=True, docs="masked"),
    "ring8_striped_causal_ragged": dict(world=8, n=512, h=4, hk=2, layout="striped", causal=True, docs="ragged"),
    "ring8_zigzag_causal_len1": dict(world=8, n=256, h=2, layout="zigzag", causal=True, docs="len1"),
    "ring8_plain_noncausal_span": dict(world=8, n=128, h=2, docs="span"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DOC_FWD_CASES))
def test_kernel_forward_documents(name):
    res = _cases().case_fwd(**DOC_FWD_CASES[name])
    assert res["ok"], res


DOC_BWD_CASES = dict(DOC_FWD_CASES)
DOC_BWD_CASES["two_kernel_d128_causal_ragged"] = dict(n=1000, causal=True, h=4, fused=False, docs="ragged")
DOC_BWD_CASES["two_kernel_gqa_tiny"] = dict(n=512, h=8, hk=2, causal=True, fused=False, docs="tiny")
DOC_BWD_CASES["two_kernel_ring4_striped_span"] = dict(world=4, n=384, h=4, hk=2, layout="striped", causal=True,
                                                      fused=False, docs="span")
DOC_BWD_CASES["two_kernel_ring2_kmask_masked"] = dict(world=2, n=256, h=2, kmask=True, fused=False, docs="masked")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DOC_BWD_CASES))
def test_kernel_backward_documents(name):
    res = _cases().case_bwd(**DOC_BWD_CASES[name])
    assert res["ok"], res


DOC_HOP_CASES = {k: dict(v, hopwise=True) for k, v in DOC_FWD_CASES.items() if k.startswith("ring") and "ring1" not in k}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DOC_HOP_CASES))
def test_kernel_hopwise_documents(name):
    res = _cases().case_fwd(**DOC_HOP_CASES[name])
    assert res["ok"], res
    if DOC_HOP_CASES[name].get("d", 128) == 128:
        res = _cases().case_bwd(**DOC_HOP_CASES[name])
        assert res["ok"], res


@pytest.mark.gpu
@pytest.mark.parametrize("d,fused", [(128, True), (128, False), (64, False)])
def test_kernel_one_document_equals_none(d, fused):
    """The document instantiations with one document reproduce the default kernels: the forward and the deterministic
    two-kernel backward bit for bit, the one-pass backward (fp32 reductions in no fixed order) within tolerance."""
    from ring_attention_pytorch_b200.ops.fused import emulate_ring_backward, emulate_ring_forward

    torch.manual_seed(0)
    b, n, h, hk = 2, 700, 4, 2
    q = torch.randn(b, n, h, d, device="cuda", dtype=torch.bfloat16)
    k, v = (torch.randn(b, n, hk, d, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    do = torch.randn(b, n, h, d, device="cuda", dtype=torch.bfloat16)
    one = [torch.zeros(b, n, dtype=torch.long, device="cuda")]
    for causal in (False, True):
        res = []
        for ids in (None, one):
            outs, lses = emulate_ring_forward([q], [k], [v], causal=causal, document_ids=ids)
            grads = emulate_ring_backward([q], [k], [v], outs, lses, [do], causal=causal, fused=fused,
                                          document_ids=ids)
            res.append((outs[0], lses[0], *grads[0]))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
        for a, b_ in zip(res[0][2:], res[1][2:]):
            if fused:
                assert (a.float() - b_.float()).abs().max() <= 1e-2 * b_.float().abs().max()
            else:
                assert torch.equal(a, b_)


@pytest.mark.gpu
def test_op_documents_causal_matches_oracle_and_skips_work():
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda
    from ring_attention_pytorch_b200.parallel.documents import document_runs

    torch.manual_seed(0)
    b, n, h, d = 1, 1500, 4, 128
    q, k, v, g = (torch.randn(b, n, h, d, device="cuda", dtype=torch.bfloat16) for _ in range(4))
    ids = _cases().make_document_ids("ragged", b, n)
    qp, kp, vp = (t.clone().requires_grad_() for t in (q, k, v))
    out = ring_flash_attn_cuda(qp, kp, vp, None, True, document_ids=ids)
    got = (out, *torch.autograd.grad(out, (qp, kp, vp), g))
    qf, kf, vf = (t.float().requires_grad_() for t in (q, k, v))
    runs = document_runs(ids)
    ref = attention_with_positions(qf, kf, vf, causal=True, q_doc=runs, k_doc=runs)
    want = (ref, *torch.autograd.grad(ref, (qf, kf, vf), g.float()))
    for a, w in zip(got, want):
        assert (a.float() - w).abs().max() / w.abs().max() < 3e-2
    with pytest.raises(ValueError, match="self-attention"):
        ring_flash_attn_cuda(q[:, :100], k, v, None, True, document_ids=ids[:, :100])


@pytest.mark.gpu
def test_transformer_kernel_documents_match_regular_attention():
    from ring_attention_pytorch_b200 import RingTransformer

    torch.manual_seed(0)
    kw = dict(num_tokens=128, dim=128, depth=2, causal=True, dim_head=64, heads=4, num_grouped_query_heads=2,
              bucket_size=64, ring_attn=False)
    fused = RingTransformer(use_cuda_kernel=True, **kw).cuda()
    dense = RingTransformer(use_cuda_kernel=False, force_regular_attn=True, **kw).cuda()
    dense.load_state_dict(fused.state_dict())
    tokens = torch.randint(0, 128, (2, 300), device="cuda")
    ids = _cases().make_document_ids("ragged", 2, 300)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        lf = fused(tokens, document_ids=ids)
        ld = dense(tokens, document_ids=ids)
        loss_f = fused(tokens, return_loss=True, document_ids=ids)
        loss_d = dense(tokens, return_loss=True, document_ids=ids)
    assert (lf.float() - ld.float()).abs().max() < 5e-2
    assert abs(loss_f.item() - loss_d.item()) < 1e-2
    loss_f.backward()
    loss_d.backward()
    gf, gd = fused.token_emb.weight.grad, dense.token_emb.weight.grad
    assert (gf - gd).abs().max() / gd.abs().max() < 5e-2


def _real_ring_doc_worker(rank, world, layout, backward, memory):
    from ring_attention_pytorch_b200.ops import ring_cuda

    ring_cuda.CONFIG["backward"] = backward
    ring_cuda.CONFIG["memory"] = memory

    import gpu_dev_check
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda
    from ring_attention_pytorch_b200.parallel.documents import document_runs
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    torch.manual_seed(0)
    b, n, h, hk, d = 1, 640, 4, 2, 128
    dev = torch.device("cuda", rank)
    pm = make_position_map(layout, world, n)
    ids = gpu_dev_check.make_document_ids("ragged", b, world * n, device=dev)
    runs = document_runs(ids)
    qs = [torch.randn(b, n, h, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    ks = [torch.randn(b, n, hk, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    vs = [torch.randn(b, n, hk, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    gs = [torch.randn(b, n, h, d, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    q, k, v = (t[rank].clone().requires_grad_() for t in (qs, ks, vs))
    out = ring_flash_attn_cuda(q, k, v, None, True, 1024, True, layout == "striped", None, world, layout=layout,
                               document_ids=ids[:, pm.positions(rank, dev)])
    dq, dk, dv = torch.autograd.grad(out, (q, k, v), gs[rank])
    torch.cuda.synchronize()
    qf = [t.float().requires_grad_() for t in qs]
    kf = [t.float().requires_grad_() for t in ks]
    vf = [t.float().requires_grad_() for t in vs]
    k_pos = torch.cat([pm.positions(r, dev) for r in range(world)])
    loss, outs = 0, []
    for r in range(world):
        o = attention_with_positions(qf[r], torch.cat(kf, 1), torch.cat(vf, 1), pm.positions(r, dev), k_pos,
                                     causal=True, q_doc=runs[:, pm.positions(r, dev)], k_doc=runs[:, k_pos])
        outs.append(o)
        loss = loss + (o * gs[r].float()).sum()
    loss.backward()
    assert (out.float() - outs[rank]).abs().max() < 3e-2
    for got, ref in ((dq, qf[rank].grad), (dk, kf[rank].grad), (dv, vf[rank].grad)):
        assert (got.float() - ref).abs().max() / ref.abs().max() < 3e-2
    dist.barrier()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("layout,backward,memory", [("striped", "fused", "gather"), ("zigzag", "fused", "ring"),
                                                    ("plain", "two_kernel", "gather")])
def test_real_ring_documents(world, layout, backward, memory):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    run_distributed(_real_ring_doc_worker, world, layout, backward, memory, backend="nccl", timeout=600.0)
