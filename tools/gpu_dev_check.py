"""GPU bring-up checks, each case in its own subprocess with a timeout so a trap or hang in one kernel
cannot take the rest of the run down.

    python tools/gpu_dev_check.py [--only fwd,ring,perf] [--timeout 120] [--log FILE]

Writes a log (default: dev_check.log in the temporary directory) and prints a summary.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


# ----------------------------------------------------------------------------------------------
# individual cases (run in a child process: `python tools/gpu_dev_check.py --case NAME`)
# ----------------------------------------------------------------------------------------------
def make_document_ids(kind, b, total, seed=0, device="cuda"):
    """Global [b, total] document ids of a packed row (``docs=`` option of the cases).

    one    : a single document
    len1   : documents of length 1 to 4, many of length 1
    ragged : lengths 1..300, not multiples of the 64 / 128 tiles
    tiny   : lengths 1..16, many documents inside one tile
    span   : one document covering everything but 5 tokens at each end (spans every rank of a ring)
    reuse  : ids alternate between 0 and 1, so separate runs share an id
    masked : like ragged; with ``kmask`` every key of document 1 is masked (its rows see nothing when non-causal)
    """
    import torch

    g = torch.Generator().manual_seed(seed)
    if kind == "one":
        return torch.zeros(b, total, dtype=torch.int64, device=device)
    if kind == "span":
        ids = torch.ones(total, dtype=torch.int64)
        ids[:5], ids[total - 5:] = 0, 2
        return ids.expand(b, total).contiguous().to(device)
    if kind == "reuse":
        return ((torch.arange(total) // 37) % 2).expand(b, total).contiguous().to(device)
    hi = {"len1": 4, "ragged": 300, "tiny": 16, "masked": 300}[kind]
    rows = []
    for _ in range(b):
        lens = torch.randint(1, hi + 1, (total,), generator=g)
        if kind == "len1":
            lens = torch.where(torch.rand(total, generator=g) < 0.5, torch.ones_like(lens), lens)
        starts = torch.zeros(total, dtype=torch.int64)
        starts[lens.cumsum(0)[lens.cumsum(0) < total]] = 1
        rows.append(starts.cumsum(0))
    return torch.stack(rows).to(device)


def _shard_ids(ids, layout, world):
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    n = ids.shape[1] // world
    pm = make_position_map(layout, world, n)
    return [ids[:, pm.positions(r, ids.device)] for r in range(world)]


def _doc_labels(doc_ids, layout, n):
    """Per-rank document ids -> per-rank run labels for the oracle (start of each token's document)."""
    import torch
    from ring_attention_pytorch_b200.parallel.documents import document_spans
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    spans = document_spans(torch.stack(doc_ids), make_position_map(layout, len(doc_ids), n))
    return [spans[r, ..., 0] for r in range(len(doc_ids))]


def _ref_ring(qs, ks, vs, layout, causal, window, softclamp, key_masks, doc_ids=None, dos=None, dtype=None,
              sinks=None):
    """The oracle over the whole emulated ring: per-rank (outs, lses), and with ``dos`` also per-rank (dq, dk, dv)
    through autograd.  ``dtype`` (default fp32) is the precision the oracle computes in.  ``sinks`` ([h] attention
    sinks): with ``dos`` every rank's tuple gains that rank's own sink gradient (its rows only), as the kernels give."""
    import torch
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    dtype = dtype or torch.float32
    world = len(qs)
    n = qs[0].shape[1]
    pm = make_position_map(layout, world, n)
    grad = dos is not None
    qf = [q.to(dtype).requires_grad_(grad) for q in qs]
    kf = [k.to(dtype).requires_grad_(grad) for k in ks]
    vf = [v.to(dtype).requires_grad_(grad) for v in vs]
    k_all, v_all = torch.cat(kf, 1), torch.cat(vf, 1)
    k_pos = torch.cat([pm.positions(r, qs[0].device) for r in range(world)])
    km = None if key_masks is None else torch.cat(list(key_masks), 1)
    labels = _doc_labels(doc_ids, layout, n) if doc_ids is not None else None
    sf = None if sinks is None else sinks.detach().to(dtype).clone().requires_grad_(grad)
    outs, lses, dsinks = [], [], []
    loss = 0.0
    with torch.enable_grad():
        for r in range(world):
            o, lse = attention_with_positions(qf[r], k_all, v_all, pm.positions(r, qs[0].device), k_pos,
                                              causal=causal, window=window, key_mask=km, softclamp_value=softclamp,
                                              return_lse=True, q_doc=None if labels is None else labels[r],
                                              k_doc=None if labels is None else torch.cat(labels, 1), sinks=sf)
            outs.append(o.detach())
            lses.append(lse.detach())
            if grad:
                loss_r = (o * dos[r].to(dtype)).sum()
                if sf is not None:
                    dsinks.append(torch.autograd.grad(loss_r, sf, retain_graph=True)[0])
                loss = loss + loss_r
        if not grad:
            return outs, lses
        loss.backward()
    grads = [(qf[r].grad, kf[r].grad, vf[r].grad) for r in range(world)]
    if sf is not None:
        grads = [(*g, ds) for g, ds in zip(grads, dsinks)]
    return outs, lses, grads


# ----------------------------------------------------------------------------------------------
# error rule of every kernel-vs-oracle comparison
# ----------------------------------------------------------------------------------------------
# A fixed absolute bound does not follow the case: at a small |out| it lets a kernel be wrong by many times its own
# rounding error, at a large one it fails a correct kernel.  The bound here is the rounding noise of the operation
# itself: the fp32 oracle run in the input dtype (bf16 / fp16 logits, softmax, products and gradients) is a second,
# low-precision implementation of the op, and its distance from the fp32 oracle is what rounding alone costs at this
# case.  A kernel result must satisfy, over all ranks of the case,
#     max|got - ref|  <= ERR_C * max|lowp - ref|  + ERR_EPS * u * max|ref|
#     rms(got - ref)  <= ERR_C * rms(lowp - ref)  + ERR_EPS * u * rms(ref)
# with u the machine epsilon of the input dtype (2^-7 for bf16, 2^-10 for fp16).  The RMS half keeps an error
# confined to a few rows from hiding behind the maximum of the others.  ERR_C = 2 as in FlashAttention's tests.  The
# ERR_EPS term is half a rounding step of the result, which no kernel writing bf16 / fp16 can beat; it keeps the
# bound positive where the low-precision oracle happens to be exact (rows that see no key, one-hot rows).  Both were
# set once from the CPU emulation in tests/test_kernel_numerics.py (an emulation of the kernel's algorithm with P
# rounded to bf16 stays below the bound in every input regime, and every mutant exceeds it at least 3x) and are not
# tuned per case.  Entries where the oracle is not finite (lse = +inf of a row with no key) must be equal.
ERR_C = 2.0
ERR_EPS = 0.5
# The low-precision oracle rounds its logits, softmax statistics and lse to the input dtype, which the kernels never
# do (they keep S, the running maximum, l and lse in fp32), so on its own its noise can exceed the fixed bounds the
# cases used before.  The maximum bound is therefore also capped at those: |out| error 3e-2, |lse| error 2e-2, and
# 3e-2 of max|ref| for dq, dk and dv.  The rule is never looser than the fixed bounds and is tighter wherever the
# oracle's own rounding is small.
CAP_OUT, CAP_LSE, CAP_GRAD_REL = 3e-2, 2e-2, 3e-2


def noise_bound(got, ref, lowp, cap=None):
    """The error rule above on lists of per-rank tensors (or single tensors).  Returns a dict with the kernel error,
    the low-precision oracle's error, the bounds and ``ratio`` = the larger of error / bound for max and RMS.
    ``cap``: the maximum bound never exceeds ``cap`` (absolute) -- see CAP_OUT below."""
    import torch

    def flat(ts):
        ts = ts if isinstance(ts, (list, tuple)) else [ts]
        return torch.cat([t.detach().float().reshape(-1) for t in ts])

    ulp = torch.finfo((lowp[0] if isinstance(lowp, (list, tuple)) else lowp).dtype).eps
    got, ref, lowp = flat(got), flat(ref), flat(lowp)
    fin = torch.isfinite(ref)
    nonfinite_ok = bool(torch.equal(got[~fin], ref[~fin]))
    g, r, lo = got[fin], ref[fin], lowp[fin]
    nan = not bool(torch.isfinite(g).all())
    if r.numel() == 0:
        return {"err": 0.0, "lowp_err": 0.0, "bound": 0.0, "ratio": 0.0, "nan": nan, "ok": nonfinite_ok and not nan}
    err, lerr = (g - r).abs().max().item(), (lo - r).abs().max().item()
    rms, lrms = (g - r).pow(2).mean().sqrt().item(), (lo - r).pow(2).mean().sqrt().item()
    bound = ERR_C * lerr + ERR_EPS * ulp * r.abs().max().item()
    if cap is not None:
        bound = min(bound, cap)
    rbound = ERR_C * lrms + ERR_EPS * ulp * r.pow(2).mean().sqrt().item()

    def frac(a, b):
        return 0.0 if a == 0 else (a / b if b > 0 else float("inf"))

    ratio = max(frac(err, bound), frac(rms, rbound))
    if nan:
        ratio = float("inf")
    return {"err": err, "lowp_err": lerr, "bound": bound, "rms": rms, "rms_bound": rbound, "ratio": ratio, "nan": nan,
            "ok": ratio <= 1.0 and nonfinite_ok and not nan}


# ----------------------------------------------------------------------------------------------
# input regimes (``regime=`` option of the cases): inputs that reach what N(0, 1) data never does
# ----------------------------------------------------------------------------------------------
LAZY_TILE, LAZY_THRESHOLD = 128, 8.0  # the forward kernel's key tile and lazy-maximum threshold (log2 units)


def visit_order(pm, rank, causal, window):
    """Global key indices (into the rank-concatenated K of an emulated ring) in the order the forward kernel walks
    them for a query of ``rank``: hops in ``ring_hop_owners`` order, 128-key tiles ascending inside each hop.  The
    single launch and the hop-wise launches walk the same order.  Returns a list of index tensors, one per tile."""
    import torch
    from ring_attention_pytorch_b200.parallel.layout import ring_hop_owners

    tiles = []
    for owner in ring_hop_owners(pm, rank, causal, window):
        for t0 in range(0, pm.n, LAZY_TILE):
            tiles.append(owner * pm.n + torch.arange(t0, min(t0 + LAZY_TILE, pm.n)))
    return tiles


def _visible(q_pos, k_pos, causal, window):
    import torch

    vis = torch.ones(len(q_pos), len(k_pos), dtype=torch.bool, device=q_pos.device)
    if causal:
        rel = q_pos[:, None] - k_pos[None, :]
        vis = rel >= 0
        if window:
            vis = vis & (rel <= window)
    return vis


def replay_lazy_max(qs, ks, layout, causal, window, scale=None, softclamp=0.0, mass_share=0.1):
    """Replay the forward kernel's lazy running maximum (tile 128, threshold 2^8) on a case's own inputs.

    Returns the share of (batch, head, row) rows of the whole ring for which the maximum is raised after the first
    visited tile with a nonzero rescale factor while the tiles visited before that carry at least ``mass_share`` of
    the row's softmax mass, and the largest such rise (log2 units)."""
    import math

    import torch
    from ring_attention_pytorch_b200.ops.oracle import expand_kv_heads
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    world, n, h, d = len(qs), qs[0].shape[1], qs[0].shape[2], qs[0].shape[3]
    scale = d ** -0.5 if scale is None else scale
    pm = make_position_map(layout, world, n)
    k_all = expand_kv_heads(torch.cat([k.float() for k in ks], 1), h)
    k_pos = torch.cat([pm.positions(r, qs[0].device) for r in range(world)])
    hit, rows, top = 0, 0, 0.0
    for r in range(world):
        s = torch.einsum("bihd,bjhd->bhij", qs[r].float(), k_all) * scale
        if softclamp:
            s = (s / softclamp).tanh() * softclamp
        s = s * (1.0 / math.log(2.0))
        s = s.masked_fill(~_visible(pm.positions(r, s.device), k_pos, causal, window), -math.inf)
        total = torch.logsumexp(s * math.log(2.0), -1)
        m_used = torch.full(s.shape[:-1], -math.inf, device=s.device)
        seen = torch.full_like(m_used, -math.inf)  # log of the mass of the tiles visited so far
        ok = torch.zeros_like(m_used, dtype=torch.bool)
        for idx in visit_order(pm, r, causal, window):
            st = s[..., idx.to(s.device)]
            cmax = st.amax(-1)
            rise = (cmax > m_used + LAZY_THRESHOLD) & torch.isfinite(m_used)
            share = (seen - total).exp()
            ok |= rise & (share >= mass_share)
            top = max(top, (cmax - m_used)[rise].max().item() if rise.any() else 0.0)
            m_used = torch.where(cmax > m_used + LAZY_THRESHOLD, cmax, m_used)
            seen = torch.logaddexp(seen, torch.logsumexp(st * math.log(2.0), -1))
        hit += int(ok.sum())
        rows += ok.numel()
    return {"rescaled_share": hit / rows, "max_rise_log2": top}


def make_case_inputs(regime, world, b, n, h, hk, d, dt, layout="plain", causal=False, window=None, softclamp=0.0,
                     seed=0, grad=False, device="cuda"):
    """Per-rank (qs, ks, vs, dos) of a case; ``dos`` is None unless ``grad``.

    regime None : N(0, 1) q, k, v (and dout)
    late_spike  : logits ~N(0, 0.01) except one key per row, in the last tile the kernel visits for that row (never
                  the first), 6.6 to 7.2 nats above the rest: the running maximum rises by about 9 to 10.4 log2 units
                  (6.6 to 7.2 nats, less the first tile's own maximum) while
                  the tiles visited before still carry a share of the mass, so the rescale of O and l matters.
                  The spike keys get orthogonal directions, so each row spikes on its own key only.
    sinkD       : key 0 (global position 0) sits D nats above every row's other logits; V has a per-channel mean
                  offset, as real values do, so dropped probability mass shows in the output
    peaky       : q scaled by 8: nearly one-hot rows
    softclamp_sat: logits of 1 to 2 times the softclamp value, where tanh saturates
    """
    import math

    import torch
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    torch.manual_seed(seed)
    if regime is None:
        qs = [torch.randn(b, n, h, d, device=device, dtype=dt) for _ in range(world)]
        ks = [torch.randn(b, n, hk, d, device=device, dtype=dt) for _ in range(world)]
        vs = [torch.randn(b, n, hk, d, device=device, dtype=dt) for _ in range(world)]
        dos = [torch.randn(b, n, h, d, device=device, dtype=dt) for _ in range(world)] if grad else None
        return qs, ks, vs, dos
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(b, world * n, h, d, generator=g)
    k = torch.randn(b, world * n, hk, d, generator=g)
    v = torch.randn(b, world * n, hk, d, generator=g)
    do = torch.randn(b, world * n, h, d, generator=g) if grad else None
    pm = make_position_map(layout, world, n)
    k_pos = torch.cat([pm.positions(r) for r in range(world)])
    if regime == "peaky":
        q = q * 8.0
    elif regime == "softclamp_sat":
        assert softclamp > 0
        q = q * 1.5 * softclamp
    elif regime.startswith("sink"):
        delta = float(regime[4:])
        u = torch.nn.functional.normalize(torch.randn(hk, d, generator=g), dim=-1)
        uq = u.repeat(h // hk, 1)  # query head j reads kv head j % hk
        q = q - (q * uq).sum(-1, keepdim=True) * uq + math.sqrt(d) * uq
        k = k - (k * u).sum(-1, keepdim=True) * u
        k0 = int((k_pos == 0).nonzero())
        k[:, k0] += delta * u
        v = v + (1.0 + 0.5 * torch.randn(hk, d, generator=g))
    elif regime == "late_spike":
        spikes = {}  # spike key -> direction index
        rows = []    # (rank, row, spike key)
        for r in range(world):
            vis = _visible(pm.positions(r), k_pos, causal, window)
            tiles = [t for t in visit_order(pm, r, causal, window)]
            for i in range(n):
                seen = [t[vis[i, t]] for t in tiles if vis[i, t].any()]
                if len(seen) >= 2:
                    key = int(seen[-1][0])
                    spikes.setdefault(key, len(spikes))
                    rows.append((r, i, key))
        assert len(spikes) <= d, (len(spikes), d)
        basis = torch.linalg.qr(torch.randn(d, d, generator=g))[0][:, :len(spikes)]  # orthonormal columns
        q = 0.1 * (q - q @ basis @ basis.T)
        k = k - k @ basis @ basis.T
        for key, a in spikes.items():
            k[:, key] += math.sqrt(d) * basis[:, a]
        t = 6.6 + 0.6 * torch.rand(b, world * n, h, generator=g)
        for r, i, key in rows:
            q[:, r * n + i] += t[:, r * n + i, :, None] * basis[:, spikes[key]]
    else:
        raise ValueError(f"unknown regime {regime!r}")

    def shards(x):
        return None if x is None else [x[:, r * n:(r + 1) * n].to(device=device, dtype=dt) for r in range(world)]

    return shards(q), shards(k), shards(v), shards(do)


def make_sinks(kind, qs, ks, softclamp=0.0):
    """fp32 ``[h]`` attention sinks of a case (``sinks=`` option), placed against the case's own logits (natural log,
    after scale and softclamp):

    below : 10 nats below the head's median row maximum
    near  : at the head's median row maximum
    above : 10 nats above every logit of the head
    mix   : the heads cycle through below, near and above
    """
    import torch
    from ring_attention_pytorch_b200.ops.oracle import expand_kv_heads

    h, d = qs[0].shape[2], qs[0].shape[3]
    k_all = expand_kv_heads(torch.cat([k.float() for k in ks], 1), h)
    row_max, top = [], torch.full((h,), -float("inf"), device=qs[0].device)
    for q in qs:
        s = torch.einsum("bihd,bjhd->bhij", q.float(), k_all) * d ** -0.5
        if softclamp:
            s = (s / softclamp).tanh() * softclamp
        m = s.amax(-1)
        row_max.append(m.transpose(0, 1).reshape(h, -1))
        top = torch.maximum(top, m.amax(dim=(0, 2)))
    med = torch.cat(row_max, 1).median(1).values
    choice = {"below": med - 10.0, "near": med, "above": top + 10.0}
    if kind == "mix":
        return torch.stack([choice[("below", "near", "above")[i % 3]][i] for i in range(h)]).contiguous()
    return choice[kind].contiguous()


def decode_reference(q, k, v, sinks=None, dtype=None, batch_chunk=8):
    """The oracle of tree decode: ``q [b, h, 1, d]`` against ``k, v [b, hk, n, d]`` (already dequantised; None or
    n = 0 for an empty shard) with ``attention_with_positions``, computed in ``dtype`` (default fp32) and returned as
    ``[b, h, 1, d]`` in that dtype.  It runs ``batch_chunk`` sequences at a time, so the grouped-query expansion of K
    and V is never built for the whole batch at once (a batch-256, 8192-key cache would need 68 GB of it in fp32)."""
    import torch
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions

    dtype = dtype or torch.float32
    b, h, _, d = q.shape
    if k is None or k.shape[2] == 0:
        return torch.zeros(b, h, 1, v.shape[-1] if v is not None else d, device=q.device, dtype=dtype)
    sk = None if sinks is None else sinks.to(dtype)
    outs = []
    for i in range(0, b, batch_chunk):
        qc, kc, vc = (t[i:i + batch_chunk].transpose(1, 2).to(dtype) for t in (q, k, v))
        outs.append(attention_with_positions(qc, kc, vc, sinks=sk).transpose(1, 2))
    return torch.cat(outs)


def _case_docs(docs, b, n, world, layout, kmask, seed):
    """(per-rank document ids, per-rank key masks) of a case."""
    import torch

    kms = [torch.rand(b, n, device="cuda") > 0.3 for _ in range(world)] if kmask else None
    if docs is None:
        return None, kms
    ids = make_document_ids(docs, b, world * n, seed)
    doc_ids = _shard_ids(ids, layout, world)
    if kmask and docs == "masked":
        kms = [m & (d != 1) for m, d in zip(kms, doc_ids)]
    return doc_ids, kms


def _case_inputs(regime, world, b, n, h, hk, d, dtype, layout, causal, window, softclamp, kmask, docs, seed, grad):
    """Inputs of case_fwd / case_bwd: (qs, ks, vs, dos, doc_ids, key_masks, info).  ``regime="empty_rows"`` is N(0, 1)
    data whose batch 0 has every key masked; ``info`` holds the lazy-maximum replay of ``late_spike``."""
    import torch

    dt = torch.bfloat16 if dtype == "bf16" else torch.float16
    empty = regime == "empty_rows"
    qs, ks, vs, dos = make_case_inputs(None if empty else regime, world, b, n, h, hk, d, dt, layout, causal, window,
                                       softclamp, seed, grad)
    doc_ids, kms = _case_docs(docs, b, n, world, layout, kmask or empty, seed)
    if empty:
        for m in kms:
            m[0] = False
    info = {}
    if regime == "late_spike":
        info = replay_lazy_max(qs, ks, layout, causal, window, softclamp=softclamp)
    return qs, ks, vs, dos, doc_ids, kms, info


def _empty_rows(qs, ks, vs, layout, causal, window, softclamp, kms, doc_ids, rlses, sk):
    """Per-rank [b, h, n] masks of the rows that see no key (with sinks their lse is finite: ask a sink-free oracle)."""
    import torch

    if sk is not None:
        qs, ks, vs = ([t.detach() for t in ts] for ts in (qs, ks, vs))
        rlses = _ref_ring(qs, ks, vs, layout, causal, window, softclamp, kms, doc_ids)[1]
    return [torch.isinf(l) for l in rlses]


def case_fwd(world=1, b=1, n=256, h=2, hk=None, d=128, layout="plain", causal=False, window=None, softclamp=0.0,
             kmask=False, dtype="bf16", seed=0, hopwise=False, docs=None, regime=None, sinks=None):
    import torch
    from ring_attention_pytorch_b200.ops.fused import emulate_ring_forward

    hk = hk or h
    qs, ks, vs, _, doc_ids, kms, info = _case_inputs(regime, world, b, n, h, hk, d, dtype, layout, causal, window,
                                                     softclamp, kmask, docs, seed, False)
    sk = None if sinks is None else make_sinks(sinks, qs, ks, softclamp)
    outs, lses = emulate_ring_forward(qs, ks, vs, layout=layout, causal=causal, window=window, softclamp=softclamp,
                                      key_masks=kms, hopwise=hopwise, document_ids=doc_ids, sinks=sk)
    torch.cuda.synchronize()
    routs, rlses = _ref_ring(qs, ks, vs, layout, causal, window, softclamp, kms, doc_ids, sinks=sk)
    louts, llses = _ref_ring(qs, ks, vs, layout, causal, window, softclamp, kms, doc_ids, dtype=qs[0].dtype, sinks=sk)
    res = {"out": noise_bound(outs, routs, louts, CAP_OUT), "lse": noise_bound(lses, rlses, llses, CAP_LSE), **info}
    # rows that see no key: exactly zero output (the rule above only bounds them by its epsilon); with sinks their
    # lse is the sink's
    empty = _empty_rows(qs, ks, vs, layout, causal, window, softclamp, kms, doc_ids, rlses, sk)
    res["empty_rows_exact"] = all(bool((o.float()[e.transpose(1, 2)] == 0).all()) for o, e in zip(outs, empty))
    if sk is not None:
        res["empty_rows_lse_is_sink"] = all(
            bool(((l - sk[None, :, None]).abs()[e] <= 1e-5 * (1 + sk.abs().max())).all()) for l, e in zip(lses, empty))
        res["empty_rows_exact"] = res["empty_rows_exact"] and res["empty_rows_lse_is_sink"]
    res["ok"] = res["out"]["ok"] and res["lse"]["ok"] and res["empty_rows_exact"]
    return res


def case_bwd(world=1, b=1, n=256, h=2, hk=None, d=128, layout="plain", causal=False, window=None, softclamp=0.0,
             kmask=False, dtype="bf16", seed=0, fused=None, hopwise=False, docs=None, regime=None, sinks=None):
    """With ``sinks`` the result also holds ``dsinks`` (every rank's sink gradient against the oracle's) and
    ``dsinks_deterministic`` (a second backward gives bitwise the same sink gradients)."""
    import torch
    from ring_attention_pytorch_b200.ops.fused import emulate_ring_backward, emulate_ring_forward

    hk = hk or h
    qs, ks, vs, dos, doc_ids, kms, info = _case_inputs(regime, world, b, n, h, hk, d, dtype, layout, causal, window,
                                                       softclamp, kmask, docs, seed, True)
    sk = None if sinks is None else make_sinks(sinks, qs, ks, softclamp)
    outs, lses = emulate_ring_forward(qs, ks, vs, layout=layout, causal=causal, window=window, softclamp=softclamp,
                                      key_masks=kms, hopwise=hopwise, document_ids=doc_ids, sinks=sk)

    def backward():
        return emulate_ring_backward(qs, ks, vs, outs, lses, dos, layout=layout, causal=causal, window=window,
                                     softclamp=softclamp, key_masks=kms, fused=fused, hopwise=hopwise,
                                     document_ids=doc_ids, sinks=sk)

    grads = backward()
    again = backward() if sk is not None else None
    torch.cuda.synchronize()
    _, rlses, ref = _ref_ring(qs, ks, vs, layout, causal, window, softclamp, kms, doc_ids, dos=dos, sinks=sk)
    _, _, lowp = _ref_ring(qs, ks, vs, layout, causal, window, softclamp, kms, doc_ids, dos=dos, dtype=qs[0].dtype,
                           sinks=sk)
    names = ("dq", "dk", "dv") if sk is None else ("dq", "dk", "dv", "dsinks")
    res = {name: noise_bound([g[i] for g in grads], [x[i] for x in ref], [x[i] for x in lowp],
                             CAP_GRAD_REL * max(x[i].abs().max().item() for x in ref))
           for i, name in enumerate(names)}
    res.update(info)
    if sk is not None:
        res["dsinks_deterministic"] = all(bool(torch.equal(g[3], a[3])) for g, a in zip(grads, again))
    # exact zeros: dq of rows that see no key, dk / dv of masked keys (no query sees them)
    empty = _empty_rows(qs, ks, vs, layout, causal, window, softclamp, kms, doc_ids, rlses, sk)
    exact = all(bool((g[0].float()[e.transpose(1, 2)] == 0).all()) for g, e in zip(grads, empty))
    if kms is not None:
        exact = exact and all(bool((g[i].float()[~m] == 0).all()) for g, m in zip(grads, kms) for i in (1, 2))
    res["empty_rows_exact"] = exact
    ok = all(res[k2]["ok"] for k2 in names) and exact and res.get("dsinks_deterministic", True)
    res["ok"] = ok
    if not ok:
        # localise: per rank / tensor / head / 128-row tile error (nan -> 999)
        detail = {}
        for r in range(world):
            for name, got, want in (("dq", grads[r][0], ref[r][0]), ("dk", grads[r][1], ref[r][1]),
                                    ("dv", grads[r][2], ref[r][2])):
                e = torch.nan_to_num((got.float() - want).abs(), nan=999.0)
                nt = (n + 127) // 128
                pad = nt * 128 - n
                e = torch.nn.functional.pad(e, (0, 0, 0, 0, 0, pad))
                tile = e.view(b, nt, 128, e.shape[2], d).amax(dim=(2, 4))  # [b, tile, head]
                detail[f"r{r}_{name}"] = [[round(x, 3) for x in row] for row in tile[0].tolist()]
        res["detail_b0_tile_by_head"] = detail
    return res


def case_perf_bwd_fused(n=16384, h=16, causal=True, iters=5, b=1, hk=None):
    """The one-kernel backward (prep + kernel + dQ convert), timed like case_perf_bwd."""
    import torch
    from ring_attention_pytorch_b200.ops import _ext
    from ring_attention_pytorch_b200.ops.fused import (alloc_kv_buffer, alloc_qdo_buffer, alloc_stat_buffer,
                                                       fused_attn_bwd_ring, fused_attn_fwd)
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    ops = _ext.ops()
    hk = hk or h
    d = 128
    dt = torch.bfloat16
    q = torch.randn(b, n, h, d, device="cuda", dtype=dt)
    k = torch.randn(b, n, hk, d, device="cuda", dtype=dt)
    v = torch.randn(b, n, hk, d, device="cuda", dtype=dt)
    do = torch.randn(b, n, h, d, device="cuda", dtype=dt)
    pm = make_position_map("plain", 1, n)
    kv = alloc_kv_buffer(1, b, hk, n, d, dt, "cuda")
    qdo = alloc_qdo_buffer(1, b, h, n, d, dt, "cuda")
    stat = alloc_stat_buffer(1, b, h, n, "cuda")
    ops.pack_kv(k, v, kv[0])
    ready = torch.zeros(1, dtype=torch.int32, device="cuda")
    o, lse = fused_attn_fwd(q, kv, [0], ready, None, kv_heads=hk, rank=0, pm=pm, causal=causal, window=None,
                            scale=d ** -0.5)
    dq = torch.empty_like(q)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]

    def run(timed=False):
        if timed:
            ev[0].record()
        ops.bwd_prep(q, o, do, lse, qdo, stat, 0)
        if timed:
            ev[1].record()
        acc = torch.zeros(b * h, stat.shape[-1], d, dtype=torch.float32, device="cuda")
        if timed:
            ev[2].record()
        _, dk, dv = fused_attn_bwd_ring(qdo[0], stat[0], kv, None, batch=b, heads=h, kv_heads=hk, rank=0, pm=pm,
                                        causal=causal, window=None, scale=d ** -0.5, dq_acc=acc)
        if timed:
            ev[3].record()
        ops.acc_convert(acc, dq, d ** -0.5)
        if timed:
            ev[4].record()
        return dq, dk, dv

    for _ in range(2):
        run()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = sorted(times)[len(times) // 2]
    flops = 2.5 * 4.0 * b * h * n * n * d * (0.5 if causal else 1.0)
    run(timed=True)
    torch.cuda.synchronize()
    return {"ms": ms, "tflops_5gemm": flops / ms / 1e9, "ms_prep": ev[0].elapsed_time(ev[1]),
            "ms_zero": ev[1].elapsed_time(ev[2]), "ms_kernel": ev[2].elapsed_time(ev[3]),
            "ms_convert": ev[3].elapsed_time(ev[4]), "tflops_kernel_only": flops / ev[2].elapsed_time(ev[3]) / 1e9,
            "ok": True}


def case_perf_bwd(n=16384, h=16, d=128, causal=True, iters=5, b=1, hk=None):
    import torch
    from ring_attention_pytorch_b200.ops import _ext
    from ring_attention_pytorch_b200.ops.fused import (alloc_kv_buffer, alloc_qdo_buffer, alloc_stat_buffer,
                                                       fused_attn_bwd, fused_attn_fwd)
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    ops = _ext.ops()
    hk = hk or h
    dt = torch.bfloat16
    q = torch.randn(b, n, h, d, device="cuda", dtype=dt)
    k = torch.randn(b, n, hk, d, device="cuda", dtype=dt)
    v = torch.randn(b, n, hk, d, device="cuda", dtype=dt)
    do = torch.randn(b, n, h, d, device="cuda", dtype=dt)
    pm = make_position_map("plain", 1, n)
    kv = alloc_kv_buffer(1, b, hk, n, d, dt, "cuda")
    qdo = alloc_qdo_buffer(1, b, h, n, d, dt, "cuda")
    stat = alloc_stat_buffer(1, b, h, n, "cuda")
    ops.pack_kv(k, v, kv[0])
    ready = torch.zeros(1, dtype=torch.int32, device="cuda")
    o, lse = fused_attn_fwd(q, kv, [0], ready, None, kv_heads=hk, rank=0, pm=pm, causal=causal, window=None,
                            scale=d ** -0.5)

    def run():
        ops.bwd_prep(q, o, do, lse, qdo, stat, 0)
        return fused_attn_bwd(qdo, kv, stat, None, batch=b, heads=h, kv_heads=hk, rank=0, pm=pm, causal=causal,
                              window=None, scale=d ** -0.5)

    for _ in range(2):
        run()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = sorted(times)[len(times) // 2]
    flops = 2.5 * 4.0 * b * h * n * n * d * (0.5 if causal else 1.0)
    res = {"ms": ms, "tflops_5gemm_equiv": flops / ms / 1e9, "tflops_executed_7gemm": flops * 1.4 / ms / 1e9}
    # per-kernel split
    e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    common = (None, b, h, hk, 0, causal, 0, d ** -0.5, 0.0, pm.stride, pm.seg_len, pm.base0, pm.base1, 0)
    e[0].record()
    ops.bwd_prep(q, o, do, lse, qdo, stat, 0)
    e[1].record()
    ops.attn_bwd_dq(qdo, kv, stat, None, 0, *common, [0])
    e[2].record()
    ops.attn_bwd_dkdv(qdo, kv, stat, None, 0, *common, [0])
    e[3].record()
    torch.cuda.synchronize()
    res["ms_prep"], res["ms_dq"], res["ms_dkdv"] = e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), e[2].elapsed_time(e[3])
    try:
        from flash_attn import flash_attn_func

        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        out = flash_attn_func(qq, kk, vv, causal=causal)
        out.backward(do, retain_graph=True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            out.backward(do, retain_graph=True)
        e1.record()
        torch.cuda.synchronize()
        res["flash_attn2_bwd_tflops"] = flops / (e0.elapsed_time(e1) / 3) / 1e9
    except Exception as ex:  # noqa: BLE001
        res["flash_attn2_bwd_tflops"] = f"n/a: {type(ex).__name__}"
    res["ok"] = True
    return res


def case_perf_decode(batch=256, h=32, hk=8, n=8192, d=128, fp8=False, iters=20, tensor_core="auto"):
    import torch
    from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc
    from ring_attention_pytorch_b200.ops.tree_decode_cuda import tree_decode_cuda

    tdc.CONFIG["tensor_core"] = tensor_core

    q = torch.randn(batch, h, 1, d, device="cuda", dtype=torch.bfloat16)
    k = torch.randn(batch, hk, n, d, device="cuda", dtype=torch.bfloat16)
    v = torch.randn(batch, hk, n, d, device="cuda", dtype=torch.bfloat16)
    ks = vs = None
    if fp8:
        k, v = k.to(torch.float8_e4m3fn), v.to(torch.float8_e4m3fn)
        ks = torch.ones(batch * hk, device="cuda")
        vs = torch.ones(batch * hk, device="cuda")
    for _ in range(3):
        out = tree_decode_cuda(q, k, v, dim_v=d, k_scale=ks, v_scale=vs)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = tree_decode_cuda(q, k, v, dim_v=d, k_scale=ks, v_scale=vs)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    kv_bytes = 2 * k.numel() * k.element_size()
    # correctness spot check on a slice
    kx = k[:2].float().repeat(1, h // hk, 1, 1)
    vx = v[:2].float().repeat(1, h // hk, 1, 1)
    sim = torch.einsum("bhid,bhjd->bhij", q[:2].float(), kx) * d ** -0.5
    ref = torch.einsum("bhij,bhjd->bhid", sim.softmax(-1), vx)
    err = (out[:2].float() - ref).abs().max().item()
    return {"ms": ms, "kv_gb_per_s": kv_bytes / ms / 1e6, "hbm_frac_of_datasheet_3350": kv_bytes / ms / 1e6 / 3350.0, "err": err,
            "tensor_core": tensor_core, "launches_per_step": 1, "ok": err < 3e-2}


def case_perf_hop(world=4, n=16384, h=8, hk=None, d=128, layout="striped", causal=True, iters=3):
    """Cost of the hop-at-a-time schedule (memory="ring") against the single-launch schedule for one emulated rank:
    same K/V slots (already local: no transfer in either arm), forward and one-kernel backward."""
    import torch
    from ring_attention_pytorch_b200.ops import _ext
    from ring_attention_pytorch_b200.ops.fused import (alloc_fwd_carry, alloc_kv_buffer, alloc_qdo_buffer,
                                                       alloc_stat_buffer, fused_attn_bwd_ring, fused_attn_fwd,
                                                       fused_attn_fwd_hop, pad128)
    from ring_attention_pytorch_b200.parallel.layout import make_position_map, ring_hop_owners

    ops = _ext.ops()
    hk = hk or h
    dt = torch.bfloat16
    b, rank = 1, world - 1
    q = torch.randn(b, n, h, d, device="cuda", dtype=dt)
    do = torch.randn(b, n, h, d, device="cuda", dtype=dt)
    buf = alloc_kv_buffer(world, b, hk, n, d, dt, "cuda")
    for o_ in range(world):
        ops.pack_kv(torch.randn(b, n, hk, d, device="cuda", dtype=dt), torch.randn(b, n, hk, d, device="cuda", dtype=dt),
                    buf[o_])
    pm = make_position_map(layout, world, n)
    hops = ring_hop_owners(pm, rank, causal, None)
    ready = torch.zeros(world, dtype=torch.int32, device="cuda")
    peers = [0] * world  # every slot is local: the fetchers copy slot -> slot (same bytes a real ring pulls)
    kw = dict(kv_heads=hk, rank=rank, pm=pm, causal=causal, window=None, scale=d ** -0.5)
    carry_o, carry_ml = alloc_fwd_carry(q)
    accs = [torch.zeros(2, b * hk, pad128(n), d, dtype=torch.float32, device="cuda") for _ in range(world)]
    ptrs = [a.data_ptr() for a in accs]
    state = {}

    def fwd_single():
        state["o"], state["lse"] = fused_attn_fwd(q, buf, [buf[o_].data_ptr() if o_ != rank else 0 for o_ in range(world)],
                                                  ready, None, **kw)

    def fwd_hop():
        for s_, owner in enumerate(hops):
            state["o"], state["lse"] = fused_attn_fwd_hop(q, buf[owner], owner, world, carry_o, carry_ml, None,
                                                          carry_in=s_ > 0, carry_out=s_ + 1 < len(hops), **kw)

    def prep():
        qdo = alloc_qdo_buffer(1, b, h, n, d, dt, "cuda")
        stat = alloc_stat_buffer(1, b, h, n, "cuda")
        ops.bwd_prep(q, state["o"], do, state["lse"], qdo, stat, 0)
        return qdo, stat

    def bwd_single():
        fused_attn_bwd_ring(state["qdo"][0], state["stat"][0], buf, None, batch=b, heads=h, dq_acc=state["dq"],
                            dkv_acc_ptrs=ptrs, nk_pad=pad128(n), **kw)

    def bwd_hop():
        for owner in hops:
            fused_attn_bwd_ring(state["qdo"][0], state["stat"][0], buf[owner:owner + 1], None, batch=b, heads=h,
                                dq_acc=state["dq"], dkv_acc_ptrs=ptrs, nk_pad=pad128(n), hop_owner=[owner], world=world,
                                slot_owner=owner, **kw)

    def timeit(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return sorted(ts)[len(ts) // 2]

    res = {"hops": len(hops)}
    res["fwd_single_ms"] = timeit(fwd_single)
    o_ref = state["o"].clone()
    res["fwd_hop_ms"] = timeit(fwd_hop)
    res["fwd_max_diff"] = (state["o"].float() - o_ref.float()).abs().max().item()
    state["qdo"], state["stat"] = prep()
    state["dq"] = torch.zeros(b * h, state["stat"].shape[-1], d, dtype=torch.float32, device="cuda")
    res["bwd_single_ms"] = timeit(bwd_single)
    res["bwd_hop_ms"] = timeit(bwd_hop)
    flops = 4.0 * b * h * n * (n * world) * d * (0.5 if causal else 1.0)
    res["fwd_single_tflops"] = flops / res["fwd_single_ms"] / 1e9
    res["fwd_hop_tflops"] = flops / res["fwd_hop_ms"] / 1e9
    res["bwd_single_tflops"] = 2.5 * flops / res["bwd_single_ms"] / 1e9
    res["bwd_hop_tflops"] = 2.5 * flops / res["bwd_hop_ms"] / 1e9
    res["ok"] = res["fwd_max_diff"] < 2e-2
    return res


def case_perf(n=16384, h=16, d=128, causal=True, iters=5, b=1, hk=None):
    import torch
    from ring_attention_pytorch_b200.ops import _ext
    from ring_attention_pytorch_b200.ops.fused import alloc_kv_buffer, fused_attn_fwd
    from ring_attention_pytorch_b200.parallel.layout import make_position_map

    ops = _ext.ops()
    hk = hk or h
    dt = torch.bfloat16
    q = torch.randn(b, n, h, d, device="cuda", dtype=dt)
    k = torch.randn(b, n, hk, d, device="cuda", dtype=dt)
    v = torch.randn(b, n, hk, d, device="cuda", dtype=dt)
    pm = make_position_map("plain", 1, n)
    buf = alloc_kv_buffer(1, b, hk, n, d, dt, "cuda")
    ops.pack_kv(k, v, buf[0])
    ready = torch.zeros(1, dtype=torch.int32, device="cuda")

    def run():
        return fused_attn_fwd(q, buf, [0], ready, None, kv_heads=hk, rank=0, pm=pm, causal=causal, window=None,
                              scale=d ** -0.5)

    for _ in range(2):
        run()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = sorted(times)[len(times) // 2]
    flops = 4.0 * b * h * n * n * d * (0.5 if causal else 1.0)
    res = {"ms": ms, "tflops": flops / ms / 1e9}
    try:
        from flash_attn import flash_attn_func

        for _ in range(2):
            flash_attn_func(q, k, v, causal=causal)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            flash_attn_func(q, k, v, causal=causal)
        e1.record()
        torch.cuda.synchronize()
        res["flash_attn2_tflops"] = flops / (e0.elapsed_time(e1) / 3) / 1e9
    except Exception as e:  # noqa: BLE001
        res["flash_attn2_tflops"] = f"n/a: {type(e).__name__}"
    res["ok"] = True
    return res


CASES = {
    # single-rank forward
    "fwd_d128_n256": lambda: case_fwd(),
    "fwd_d128_n128_h1": lambda: case_fwd(n=128, h=1),
    "fwd_d128_causal_n512": lambda: case_fwd(n=512, causal=True),
    "fwd_d128_n300_tail": lambda: case_fwd(n=300, b=2),
    "fwd_d128_causal_n1000": lambda: case_fwd(n=1000, causal=True, h=4),
    "fwd_d64_n512": lambda: case_fwd(n=512, d=64, h=4),
    "fwd_d64_causal_n777": lambda: case_fwd(n=777, d=64, h=4, causal=True),
    "fwd_gqa_causal": lambda: case_fwd(n=512, h=8, hk=2, causal=True),
    "fwd_kmask": lambda: case_fwd(n=384, h=2, kmask=True, b=2),
    "fwd_softclamp": lambda: case_fwd(n=384, h=2, softclamp=20.0),
    "fwd_window": lambda: case_fwd(n=1024, h=2, causal=True, window=200),
    "fwd_fp16": lambda: case_fwd(n=512, h=2, causal=True, dtype="fp16"),
    "fwd_many_items": lambda: case_fwd(n=2048, h=16, b=2, causal=True),
    # emulated rings (W ranks on one GPU)
    "ring2_plain": lambda: case_fwd(world=2, n=256, h=2),
    "ring2_plain_causal": lambda: case_fwd(world=2, n=256, h=2, causal=True),
    "ring4_striped_causal": lambda: case_fwd(world=4, n=384, h=4, hk=2, layout="striped", causal=True),
    "ring4_zigzag_causal": lambda: case_fwd(world=4, n=512, h=2, layout="zigzag", causal=True),
    "ring4_plain_window": lambda: case_fwd(world=4, n=256, h=2, causal=True, window=300),
    "ring3_kmask": lambda: case_fwd(world=3, n=200, h=2, kmask=True),
    "ring8_striped_causal_big": lambda: case_fwd(world=8, n=1024, h=8, hk=2, layout="striped", causal=True),
    # backward, single rank
    "bwd_d128_n256": lambda: case_bwd(),
    "bwd_d128_n128_h1": lambda: case_bwd(n=128, h=1),
    "bwd_d128_n64_h1": lambda: case_bwd(n=64, h=1),
    "bwd_d128_causal_n512": lambda: case_bwd(n=512, causal=True),
    "bwd_d128_n300_tail": lambda: case_bwd(n=300, b=2),
    "bwd_d128_causal_n1000": lambda: case_bwd(n=1000, causal=True, h=4),
    "bwd_d64_n512": lambda: case_bwd(n=512, d=64, h=4),
    "bwd_d64_causal_n777": lambda: case_bwd(n=777, d=64, h=4, causal=True),
    "bwd_gqa_causal": lambda: case_bwd(n=512, h=8, hk=2, causal=True),
    "bwd_kmask": lambda: case_bwd(n=384, h=2, kmask=True, b=2),
    "bwd_softclamp": lambda: case_bwd(n=384, h=2, softclamp=20.0),
    "bwd_window": lambda: case_bwd(n=1024, h=2, causal=True, window=200),
    "bwd_fp16": lambda: case_bwd(n=512, h=2, causal=True, dtype="fp16"),
    "bwd_many_items": lambda: case_bwd(n=2048, h=16, b=2, causal=True),
    # backward, emulated rings
    "rbwd2_plain_h1": lambda: case_bwd(world=2, n=128, h=1),
    "rbwd3_plain": lambda: case_bwd(world=3, n=128, h=1),
    "rbwd3_plain_causal": lambda: case_bwd(world=3, n=128, h=1, causal=True),
    "rbwd4_plain_causal": lambda: case_bwd(world=4, n=256, h=2, causal=True),
    "rbwd2_plain": lambda: case_bwd(world=2, n=256, h=2),
    "rbwd2_plain_causal": lambda: case_bwd(world=2, n=256, h=2, causal=True),
    "rbwd4_striped_causal": lambda: case_bwd(world=4, n=384, h=4, hk=2, layout="striped", causal=True),
    "rbwd4_zigzag_causal": lambda: case_bwd(world=4, n=512, h=2, layout="zigzag", causal=True),
    "rbwd4_plain_window": lambda: case_bwd(world=4, n=256, h=2, causal=True, window=300),
    "rbwd3_kmask": lambda: case_bwd(world=3, n=200, h=2, kmask=True),
    # the two-kernel backward at head dim 128 (the default there is the one-kernel backward)
    "bwd2k_d128_causal_n1000": lambda: case_bwd(n=1000, causal=True, h=4, fused=False),
    "bwd2k_gqa_causal": lambda: case_bwd(n=512, h=8, hk=2, causal=True, fused=False),
    "bwd2k_ring4_striped_causal": lambda: case_bwd(world=4, n=384, h=4, hk=2, layout="striped", causal=True, fused=False),
    # performance
    "perffz_causal_16k": lambda: case_perf_bwd_fused(),
    "perffz_full_8k": lambda: case_perf_bwd_fused(n=8192, causal=False),
    "perffz_causal_64k_h8": lambda: case_perf_bwd_fused(n=65536, h=8, iters=3),
    "perffz_gqa_causal_32k": lambda: case_perf_bwd_fused(n=32768, h=16, hk=4, iters=3),
    "perfbwd_causal_16k": lambda: case_perf_bwd(),
    "perfbwd_full_8k": lambda: case_perf_bwd(n=8192, causal=False),
    "perfbwd_causal_64k_h8": lambda: case_perf_bwd(n=65536, h=8, iters=3),
    "dec_small_tc": lambda: case_perf_decode(batch=2, h=8, hk=2, n=512, iters=1),
    "dec_small_tc_fp8": lambda: case_perf_decode(batch=2, h=8, hk=2, n=512, iters=1, fp8=True),
    "dec_small_cudacore": lambda: case_perf_decode(batch=2, h=8, hk=2, n=512, iters=1, tensor_core=False),
    "perfdec_bf16": lambda: case_perf_decode(),
    "perfdec_fp8": lambda: case_perf_decode(fp8=True),
    "perfdec_mha_b32": lambda: case_perf_decode(batch=32, h=32, hk=32, n=8192),
    "perfdec_cudacore_bf16": lambda: case_perf_decode(tensor_core=False),
    "perfdec_cudacore_fp8": lambda: case_perf_decode(fp8=True, tensor_core=False),
    "perfdec_g16_bf16": lambda: case_perf_decode(batch=64, h=64, hk=4, n=16384),
    "perfhop_w4_striped_16k": lambda: case_perf_hop(),
    "perfhop_w8_striped_8k_h16": lambda: case_perf_hop(world=8, n=8192, h=16),
    "perf_causal_16k": lambda: case_perf(),
    "perf_full_8k": lambda: case_perf(n=8192, causal=False),
    "perf_causal_64k_h8": lambda: case_perf(n=65536, h=8, iters=3),
    "perf_d64_causal_16k": lambda: case_perf(d=64, h=32),
}

GROUPS = {
    "fwd": [c for c in CASES if c.startswith("fwd")],
    "ring": [c for c in CASES if c.startswith("ring")],
    "bwd": [c for c in CASES if c.startswith("bwd")],
    "rbwd": [c for c in CASES if c.startswith("rbwd")],
    "bwd2k": [c for c in CASES if c.startswith("bwd2k")],
    "perffz": [c for c in CASES if c.startswith("perffz")],
    "perfbwd": [c for c in CASES if c.startswith("perfbwd")],
    "perfdec": [c for c in CASES if c.startswith("perfdec")],
    "perf": [c for c in CASES if c.startswith("perf_")],
    "perfhop": [c for c in CASES if c.startswith("perfhop")],
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case")
    ap.add_argument("--only", default="fwd,ring,perf")
    ap.add_argument("--timeout", type=int, default=150)
    ap.add_argument("--log", default=os.path.join(tempfile.gettempdir(), "dev_check.log"))
    ap.add_argument("--max-fail", type=int, default=0, help="stop after this many failed cases (0: never)")
    args = ap.parse_args()

    if args.case:
        res = CASES[args.case]()
        print("RESULT " + json.dumps(res))
        return

    os.makedirs(os.path.dirname(args.log), exist_ok=True)
    names = []
    for g in args.only.split(","):
        names += GROUPS.get(g, [g] if g in CASES else [])
    summary = []
    nfail = 0
    with open(args.log, "a") as log:
        log.write(f"\n==== dev check {time.strftime('%F %T')} only={args.only}\n")
        for name in names:
            t0 = time.time()
            try:
                proc = subprocess.run([sys.executable, os.path.abspath(__file__), "--case", name], capture_output=True,
                                      text=True, timeout=args.timeout)
                out = proc.stdout + proc.stderr
                line = [l for l in proc.stdout.splitlines() if l.startswith("RESULT ")]
                status = line[-1][7:] if line else f"FAILED rc={proc.returncode}"
            except subprocess.TimeoutExpired as e:
                out = (e.stdout or b"").decode() if isinstance(e.stdout, bytes) else (e.stdout or "")
                out += (e.stderr or b"").decode() if isinstance(e.stderr, bytes) else (e.stderr or "")
                status = "TIMEOUT"
            dt = time.time() - t0
            msg = f"{name:32s} {dt:6.1f}s  {status}"
            print(msg, flush=True)
            summary.append(msg)
            log.write(msg + "\n")
            if not status.startswith("{") or '"ok": false' in status:
                log.write("---- output tail\n" + out[-3000:] + "\n----\n")
                nfail += 1
            log.flush()
            if args.max_fail and nfail >= args.max_fail:
                print(f"stopping after {nfail} failed cases", flush=True)
                break


if __name__ == "__main__":
    main()
