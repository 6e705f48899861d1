"""Numerics of the attention kernels on inputs that N(0, 1) data never produces, under the noise-scaled error rule.

Every comparison uses ``gpu_dev_check.noise_bound``: the kernel's distance from the fp32 oracle must stay within
``ERR_C`` times the distance of the same oracle run in the input dtype, plus half a rounding step of the result (see
the comment at the rule), in both the maximum and the RMS.  The input regimes (``gpu_dev_check.make_case_inputs``) reach the paths that random data leaves cold:

- ``late_spike``: a row's running maximum rises by 9 to 10 log2 units after its first tile, so the forward's lazy
  maximum rescales O and l (and the carried O of the hop-wise and fp8 paths);
- ``sink6`` / ``sink10``: one early key 6 or 10 nats above the rest and V with a nonzero channel mean, the shape of
  attention sinks in long-context prefill;
- ``peaky``: q scaled by 8, nearly one-hot rows (exp2 near the maximum, the lse the backward reads);
- ``softclamp_sat``: logits at 1 to 2 times the softclamp value, where tanh saturates;
- ``empty_rows``: rows that see no key (out = 0, lse = +inf, zero gradients, no NaN).

The CPU half proves the rule can fail: a torch emulation of the kernel's algorithm (128-key tiles, lazy maximum,
P rounded to bf16) passes it in every regime, and each of a set of plausible kernel mistakes, applied to the same
emulation, exceeds the bound at least 3x in a regime that exposes it.
"""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import gpu_dev_check as gdc  # noqa: E402

REL_RMS_TOL, BF16_RATIO_TOL = 5e-2, 13.0  # the fp8 forward's bounds (tests/test_fp8_prefill.py)


# ================================================================================================
# CPU: a torch model of the kernels' arithmetic, and mutants of it
# ================================================================================================
def _round(x, dtype):
    return x.to(dtype).float()


def emulate_kernel(q, k, v, do=None, *, causal=False, window=None, key_mask=None, softclamp=0.0, doc_ids=None,
                   p_rule="bf16", mutant=None):
    """The forward kernel's algorithm on one rank (keys walked in 128-key tiles, ascending), and the backward's.

    q [b, i, h, d], k / v [b, j, hk, d] (values representable in bf16).  S in fp32; the running maximum is raised only
    when a tile beats it by more than 2^8, and only then are O and l rescaled.  ``p_rule``:
      bf16      : P rounded to bf16 for P V, l summed from the unrounded P (the bf16 kernel)
      e4m3      : P rounded to e4m3 for P V, l summed from the unrounded P (the fp8 kernel before the fix)
      e4m3_tile : each tile's P taken against its own maximum - 8 (floored 40 log2 units below the running maximum),
                  rounded to e4m3, and l summed from the rounded P; O and l rescaled every tile (the fp8 kernel)
    ``mutant``: window_plus1 / window_minus1, no_tanh_grad, no_rescale, gqa_div, drop_tail_key, doc_end_plus1.
    Returns out (bf16 values), lse, and with ``do`` the bf16 gradients (dq, dk, dv).
    """
    b, i, h, d = q.shape
    j, hk = k.shape[1], k.shape[2]
    g = h // hk
    scale = d ** -0.5
    heads = torch.arange(h) // g if mutant == "gqa_div" else torch.arange(h) % hk
    kx, vx = k[:, :, heads].float(), v[:, :, heads].float()
    s = torch.einsum("bihd,bjhd->bhij", q.float(), kx) * scale
    th = None
    if softclamp:
        th = torch.tanh(s / softclamp)
        s = th * softclamp
    pos = torch.arange(j)
    q_pos = torch.arange(i) + (j - i)
    vis = torch.ones(b, 1, i, j, dtype=torch.bool)
    if causal:
        rel = q_pos[:, None] - pos[None, :]
        vv = rel >= 0
        if window:
            w = window + {"window_plus1": 1, "window_minus1": -1}.get(mutant, 0)
            vv = vv & (rel <= w)
        vis = vis & vv
    if key_mask is not None:
        vis = vis & key_mask[:, None, None, :]
    if doc_ids is not None:
        from ring_attention_pytorch_b200.parallel.documents import document_spans
        from ring_attention_pytorch_b200.parallel.layout import make_position_map

        sp = document_spans(doc_ids[None], make_position_map("plain", 1, j))[0]  # [b, n, 2] = [start, end)
        end = sp[..., 1] + (1 if mutant == "doc_end_plus1" else 0)
        vis = vis & ((sp[:, None, :, 0, None] <= pos) & (pos < end[:, None, :, None]))
    if mutant == "drop_tail_key" and j % gdc.LAZY_TILE:
        vis = vis.clone()
        vis[..., j - 1] = False
    s2 = torch.where(vis, s * (1 / math.log(2.0)), torch.tensor(-math.inf))

    m = torch.full((b, h, i, 1), -math.inf)
    l = torch.zeros(b, h, i, 1)
    o = torch.zeros(b, h, i, d)
    m_run = m.clone()
    for t0 in range(0, j, gdc.LAZY_TILE):
        st = s2[..., t0:t0 + gdc.LAZY_TILE]
        vt = vx[:, t0:t0 + gdc.LAZY_TILE].permute(0, 2, 1, 3)
        cmax = st.amax(-1, keepdim=True)
        if p_rule == "e4m3_tile":
            m_run = torch.maximum(m_run, cmax)
            new = torch.maximum(cmax, m_run - 32.0) - 8.0
            new = torch.where(torch.isfinite(cmax), new, m)  # a tile the row sees nothing of leaves it alone
            factor = torch.where(torch.isfinite(m), torch.exp2(m - new), torch.zeros_like(m))
            m = new
        else:
            raise_ = cmax > m + gdc.LAZY_THRESHOLD
            new = torch.where(raise_, torch.maximum(m, cmax), m)
            factor = torch.where(raise_ & torch.isfinite(m), torch.exp2(m - new), torch.where(raise_, 0.0, 1.0))
            if mutant == "no_rescale":
                factor = torch.where(torch.isfinite(m), torch.ones_like(factor), factor)
            m = new
        l, o = l * factor, o * factor
        p = torch.exp2(st - torch.where(torch.isfinite(m), m, torch.zeros_like(m)))
        if p_rule == "bf16":
            pn, pl = _round(p, torch.bfloat16), p
        else:
            pn = _round(p, torch.float8_e4m3fn)
            pl = pn if p_rule == "e4m3_tile" else p
        l = l + pl.sum(-1, keepdim=True)
        o = o + pn @ vt
    empty = l == 0
    out = torch.where(empty, torch.zeros_like(o), o / l.clamp_min(1e-30))
    lse = torch.where(empty, torch.tensor(math.inf), (torch.where(torch.isfinite(m), m, 0.0) + torch.log2(l)) * math.log(2.0))
    out = _round(out.permute(0, 2, 1, 3), torch.bfloat16)
    lse = lse.squeeze(-1)
    if do is None:
        return out, lse, None
    # backward: P recomputed from lse in fp32, P and dS rounded to bf16 for their products
    p = torch.where(vis, torch.exp(s - torch.where(torch.isfinite(lse), lse, 0.0)[..., None]), torch.tensor(0.0))
    dof = do.float().permute(0, 2, 1, 3)
    dv = _round(p, torch.bfloat16).transpose(-1, -2) @ dof
    dp = dof @ vx.permute(0, 2, 3, 1)
    delta = (dof * out.permute(0, 2, 1, 3)).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    if softclamp and mutant != "no_tanh_grad":
        ds = ds * (1 - th * th)
    ds = _round(ds, torch.bfloat16)
    dq = ds @ kx.permute(0, 2, 1, 3) * scale
    dk = ds.transpose(-1, -2) @ q.float().permute(0, 2, 1, 3) * scale
    # query head x read kv head heads[x]: sum its gradient there
    dkk = torch.zeros(b, hk, j, d).index_add_(1, heads, dk)
    dvv = torch.zeros(b, hk, j, d).index_add_(1, heads, dv)
    grads = tuple(_round(t.permute(0, 2, 1, 3), torch.bfloat16) for t in (dq, dkk, dvv))
    return out, lse, grads


def _oracle(q, k, v, do, dtype, *, causal, window, key_mask, softclamp, doc_ids):
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.parallel.documents import document_runs

    runs = None if doc_ids is None else document_runs(doc_ids)
    qf, kf, vf = (t.to(dtype).requires_grad_(do is not None) for t in (q, k, v))
    o, lse = attention_with_positions(qf, kf, vf, causal=causal, window=window, key_mask=key_mask,
                                      softclamp_value=softclamp, return_lse=True, q_doc=runs, k_doc=runs)
    if do is None:
        return o, lse, None
    (o * do.to(dtype)).sum().backward()
    return o.detach(), lse.detach(), (qf.grad, kf.grad, vf.grad)


# (regime, case options) of the CPU checks; single rank, bf16
CPU_CASES = {
    "randn_window": (None, dict(n=300, h=2, causal=True, window=127)),
    "late_spike": ("late_spike", dict(n=300, h=2)),
    "late_spike_causal": ("late_spike", dict(n=384, h=2, causal=True)),
    "sink6": ("sink6", dict(n=512, h=2, causal=True)),
    # forward only: with a 10-nat sink the backward's D = rowsum(dO * O), taken from the bf16 output as in every
    # FlashAttention backward, cancels against dP of the sink key; the bf16 oracle does not share that rounding
    # (emulated dq / dk RMS 1.6x its bound), so this is a property of the algorithm, not a kernel mistake
    "sink10": ("sink10", dict(n=512, h=2, causal=True, fwd_only=True)),
    "peaky_gqa": ("peaky", dict(n=257, h=8, hk=2)),
    "softclamp_sat20": ("softclamp_sat", dict(n=200, h=2, softclamp=20.0)),
    "softclamp_sat50": ("softclamp_sat", dict(n=200, h=2, softclamp=50.0, causal=True)),
    "empty_rows": ("empty_rows", dict(n=129, h=2, b=2)),
    "docs": ("docs", dict(n=300, h=2)),
}


def _cpu_case(name):
    regime, kw = CPU_CASES[name]
    kw = dict(kw)
    b, n, h = kw.pop("b", 1), kw.pop("n"), kw.pop("h")
    hk = kw.pop("hk", h)
    d = 64
    gen = None if regime in ("empty_rows", "docs") else regime
    qs, ks, vs, dos = gdc.make_case_inputs(gen, 1, b, n, h, hk, d, torch.bfloat16, "plain", kw.get("causal", False),
                                           kw.get("window"), kw.get("softclamp", 0.0), seed=1, grad=True, device="cpu")
    opts = dict(causal=kw.get("causal", False), window=kw.get("window"), softclamp=kw.get("softclamp", 0.0),
                key_mask=None, doc_ids=None)
    if kw.get("fwd_only"):
        dos = [None]
    if regime == "empty_rows":
        opts["key_mask"] = torch.rand(b, n, generator=torch.Generator().manual_seed(2)) > 0.3
        opts["key_mask"][0] = False
    if regime == "docs":
        opts["doc_ids"] = gdc.make_document_ids("tiny", b, n, seed=3, device="cpu")
    return (qs[0], ks[0], vs[0], dos[0]), opts


def _rule(got, ref, lowp):
    """The rule over out, lse and (when given) the three gradients: worst ratio and the per-tensor results."""
    names = ("out", "lse", "dq", "dk", "dv")
    res = {nm: gdc.noise_bound(gg, rr, ll) for nm, gg, rr, ll in
           zip(names, (got[0], got[1], *(got[2] or ())), (ref[0], ref[1], *(ref[2] or ())),
               (lowp[0], lowp[1], *(lowp[2] or ())))}
    worst = max(r["ratio"] if r["ok"] or r["ratio"] > 1 else float("inf") for r in res.values())
    return worst, res


def _reference(args, opts):
    q, k, v, do = args
    ref = _oracle(q, k, v, do, torch.float32, **opts)
    lowp = _oracle(q, k, v, do, torch.bfloat16, **opts)
    return ref, lowp


@pytest.mark.parametrize("name", list(CPU_CASES))
def test_rule_accepts_the_kernel_algorithm(name):
    args, opts = _cpu_case(name)
    ref, lowp = _reference(args, opts)
    got = emulate_kernel(*args, **opts)
    worst, res = _rule(got, ref, lowp)
    print(f"[accept] {name}: worst error/bound {worst:.3f}")
    assert worst <= 1.0, res


def test_late_spike_regime_reaches_the_rescale():
    """The late_spike inputs raise the running maximum after the first tile, with a nonzero rescale factor, on most
    rows, in every path's visit order; N(0, 1) inputs never do."""
    for world, layout, causal in ((1, "plain", False), (1, "plain", True), (2, "plain", True), (4, "striped", True),
                                  (4, "zigzag", True), (3, "plain", False)):
        qs, ks, _, _ = gdc.make_case_inputs("late_spike", world, 1, 256, 2, 2, 64, torch.bfloat16, layout, causal,
                                            None, seed=0, device="cpu")
        rep = gdc.replay_lazy_max(qs, ks, layout, causal, None)
        assert rep["rescaled_share"] >= 0.3, (world, layout, causal, rep)
        assert 9.0 <= rep["max_rise_log2"] <= 12.0, rep
        qs, ks, _, _ = gdc.make_case_inputs(None, world, 1, 256, 2, 2, 64, torch.bfloat16, layout, causal, None,
                                            seed=0, device="cpu")
        assert gdc.replay_lazy_max(qs, ks, layout, causal, None)["rescaled_share"] == 0.0


# (mutant, CPU case that exposes it, p_rule)
MUTANTS = [
    ("window_plus1", "randn_window", "bf16"),
    ("window_minus1", "randn_window", "bf16"),
    ("no_tanh_grad", "softclamp_sat20", "bf16"),
    ("no_tanh_grad", "softclamp_sat50", "bf16"),
    ("no_rescale", "late_spike", "bf16"),
    ("no_rescale", "late_spike_causal", "bf16"),
    ("gqa_div", "peaky_gqa", "bf16"),
    ("drop_tail_key", "peaky_gqa", "bf16"),
    ("drop_tail_key", "empty_rows", "bf16"),
    ("doc_end_plus1", "docs", "bf16"),
    (None, "sink6", "e4m3"),
    (None, "sink10", "e4m3"),
]


@pytest.mark.parametrize("mutant,case,p_rule", MUTANTS)
def test_rule_rejects_kernel_mistakes(mutant, case, p_rule):
    args, opts = _cpu_case(case)
    ref, lowp = _reference(args, opts)
    got = emulate_kernel(*args, **opts, p_rule=p_rule, mutant=mutant)
    worst, res = _rule(got, ref, lowp)
    print(f"[reject] {mutant or p_rule} on {case}: worst error/bound {worst:.2f}")
    assert worst >= 3.0, res


@pytest.mark.parametrize("regime", ["sink6", "sink10", "late_spike", "peaky"])
def test_fp8_tile_reference_keeps_sink_mass(regime):
    """The last 64 queries of an 8192-key causal prefill.  With each tile's P taken against that tile's own maximum
    and l summed from the rounded P, e4m3 P stays within the fp8 forward's bounds; with the running maximum and l
    summed from the unrounded P (the rule before the fix), the sink inputs lose the tail's mass from P V only.

    This checks the choice of P, not the kernel's arithmetic: the emulation adds each tile's P V to O in fp32, which
    the kernel does too (each tile's e4m3 product goes into zeroed registers), but it does not model the reduced
    precision of the MMA inside one tile.  The GPU cases below check the kernel itself on the same regimes."""
    n, rows = 8192, 64
    qs, ks, vs, _ = gdc.make_case_inputs(regime, 1, 1, n, 1, 1, 64, torch.bfloat16, "plain", True, None, seed=5,
                                         device="cpu")
    q, k, v = qs[0][:, -rows:], ks[0], vs[0]
    ref = _oracle(q, k, v, None, torch.float32, causal=True, window=None, key_mask=None, softclamp=0.0,
                  doc_ids=None)[0]

    def rel(x):
        return ((x - ref).norm() / ref.norm()).item()

    e16 = rel(emulate_kernel(q, k, v, causal=True)[0])
    fixed = rel(emulate_kernel(q, k, v, causal=True, p_rule="e4m3_tile")[0])
    old = rel(emulate_kernel(q, k, v, causal=True, p_rule="e4m3")[0])
    print(f"[fp8 emulation] {regime}: rel rms bf16 P {e16:.2e}, e4m3 tile reference {fixed:.2e}, "
          f"e4m3 running maximum {old:.2e}")
    assert fixed <= REL_RMS_TOL and fixed <= BF16_RATIO_TOL * e16
    if regime.startswith("sink"):
        assert old > REL_RMS_TOL


# ================================================================================================
# GPU: the kernels under the rule, per regime and path
# ================================================================================================
def _report(name, res):
    for key, r in res.items():
        if isinstance(r, dict) and "bound" in r:
            print(f"[{name}] {key}: err {r['err']:.3e} lowp {r['lowp_err']:.3e} bound {r['bound']:.3e} "
                  f"ratio {r['ratio']:.3f}")


FWD = {
    # late_spike: the lazy maximum's rescale, in the single launch, the hop-wise launches and every ring rank
    "spike_n257": dict(n=257, h=2, regime="late_spike"),
    "spike_causal_gqa": dict(n=384, h=8, hk=2, causal=True, regime="late_spike"),
    "spike_ring2_causal": dict(world=2, n=256, h=2, causal=True, regime="late_spike"),
    "spike_ring4_striped": dict(world=4, n=256, h=2, layout="striped", causal=True, regime="late_spike"),
    "spike_ring4_zigzag_fp16": dict(world=4, n=256, h=2, layout="zigzag", causal=True, dtype="fp16",
                                    regime="late_spike"),
    "spike_ring3_plain_d64": dict(world=3, n=129, h=2, d=64, regime="late_spike"),
    # sinks
    "sink6_causal_n1000": dict(n=1000, h=2, causal=True, regime="sink6"),
    "sink10_d64_fp16": dict(n=513, h=4, d=64, causal=True, dtype="fp16", regime="sink10"),
    "sink10_ring4_striped": dict(world=4, n=256, h=4, hk=1, layout="striped", causal=True, regime="sink10"),
    # nearly one-hot rows at the tile edges
    "peaky_n1": dict(n=1, h=2, regime="peaky"),
    "peaky_n63_d64": dict(n=63, h=2, d=64, regime="peaky"),
    "peaky_n64_fp16": dict(n=64, h=2, dtype="fp16", regime="peaky"),
    "peaky_n65_gqa_hk1": dict(n=65, h=8, hk=1, b=3, regime="peaky"),
    "peaky_n127_causal": dict(n=127, h=4, hk=1, causal=True, regime="peaky"),
    "peaky_n128_gqa4": dict(n=128, h=4, hk=1, b=3, causal=True, regime="peaky"),
    "peaky_n129_d64_gqa8": dict(n=129, h=8, hk=1, d=64, regime="peaky"),
    "peaky_ring2_zigzag": dict(world=2, n=128, h=2, layout="zigzag", causal=True, regime="peaky"),
    # windows at the tile edges
    "window1": dict(n=257, h=2, causal=True, window=1, regime="peaky"),
    "window127": dict(n=257, h=2, causal=True, window=127),
    "window128_d64": dict(n=257, h=2, d=64, causal=True, window=128, regime="sink6"),
    "window_ge_n": dict(n=300, h=2, causal=True, window=300, regime="late_spike"),
    # saturated softclamp
    "softclamp20_sat": dict(n=257, h=2, softclamp=20.0, regime="softclamp_sat"),
    "softclamp50_sat_causal": dict(n=300, h=2, softclamp=50.0, causal=True, regime="softclamp_sat"),
    "softclamp20_sat_d64_fp16": dict(n=129, h=2, d=64, softclamp=20.0, dtype="fp16", regime="softclamp_sat"),
    # rows that see no key
    "empty_kmask_batch": dict(n=200, h=2, b=2, regime="empty_rows"),
    "empty_kmask_batch_ring3": dict(world=3, n=128, h=2, b=2, regime="empty_rows"),
    "empty_docs_masked": dict(n=384, h=2, b=2, kmask=True, docs="masked"),
}
HOP = {k: dict(v) for k, v in FWD.items() if v.get("world", 1) > 1}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FWD))
def test_forward_regimes(name):
    res = gdc.case_fwd(**FWD[name])
    _report(name, res)
    if FWD[name].get("regime") == "late_spike":
        assert res["rescaled_share"] >= 0.3, res
    assert res["ok"], res


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(HOP))
def test_hopwise_forward_regimes(name):
    res = gdc.case_fwd(hopwise=True, **HOP[name])
    _report(name, res)
    assert res["ok"], res


BWD = {
    "spike_causal": dict(n=384, h=2, causal=True, regime="late_spike"),
    "sink6_causal_gqa": dict(n=512, h=8, hk=2, causal=True, regime="sink6"),
    "peaky_n65_hk1_b3": dict(n=65, h=8, hk=1, b=3, regime="peaky"),
    "peaky_n129_d64": dict(n=129, h=4, d=64, causal=True, regime="peaky"),
    "peaky_n1": dict(n=1, h=2, regime="peaky"),
    "window1_peaky": dict(n=257, h=2, causal=True, window=1, regime="peaky"),
    "window128": dict(n=257, h=2, causal=True, window=128, regime="sink6"),
    "softclamp20_sat": dict(n=257, h=2, softclamp=20.0, regime="softclamp_sat"),
    "softclamp50_sat_causal": dict(n=300, h=2, softclamp=50.0, causal=True, regime="softclamp_sat"),
    "softclamp20_sat_two_kernel": dict(n=257, h=2, softclamp=20.0, regime="softclamp_sat", fused=False),
    "softclamp50_sat_two_kernel_causal": dict(n=300, h=2, softclamp=50.0, causal=True, regime="softclamp_sat",
                                              fused=False),
    "softclamp20_sat_d64_fp16": dict(n=129, h=2, d=64, softclamp=20.0, dtype="fp16", regime="softclamp_sat"),
    "peaky_two_kernel_gqa8": dict(n=127, h=8, hk=1, causal=True, regime="peaky", fused=False),
    "sink6_fp16_two_kernel": dict(n=300, h=2, causal=True, dtype="fp16", regime="sink6", fused=False),
    "empty_kmask_batch": dict(n=200, h=2, b=2, regime="empty_rows"),
    "empty_kmask_batch_two_kernel": dict(n=200, h=2, b=2, regime="empty_rows", fused=False),
    "empty_docs_masked": dict(n=384, h=2, b=2, kmask=True, docs="masked"),
    "ring2_spike_hop": dict(world=2, n=256, h=2, causal=True, regime="late_spike", hopwise=True),
    "ring4_striped_sink6": dict(world=4, n=256, h=4, hk=1, layout="striped", causal=True, regime="sink6"),
    "ring4_zigzag_softclamp_sat_hop": dict(world=4, n=128, h=2, layout="zigzag", causal=True, softclamp=50.0,
                                           regime="softclamp_sat", hopwise=True),
    "ring3_empty": dict(world=3, n=128, h=2, b=2, regime="empty_rows"),
    "ring4_striped_peaky_two_kernel": dict(world=4, n=128, h=4, hk=2, layout="striped", causal=True, regime="peaky",
                                           fused=False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BWD))
def test_backward_regimes(name):
    res = gdc.case_bwd(**BWD[name])
    _report(name, res)
    assert res["ok"], res


@pytest.mark.gpu
@pytest.mark.parametrize("n_q,n_k,causal", [(70, 333, True), (70, 333, False), (300, 129, True), (300, 129, False)])
def test_bf16_cross_attention(n_q, n_k, causal):
    """bf16 cross-attention through the op, forward and backward.  With n_q > n_k under causal the first
    n_q - n_k query rows see no key: their output and gradients are zero."""
    from ring_attention_pytorch_b200.ops.oracle import attention_with_positions
    from ring_attention_pytorch_b200.ops.ring_cuda import ring_flash_attn_cuda

    torch.manual_seed(0)
    b, h, hk, d = 2, 4, 2, 128
    q = torch.randn(b, n_q, h, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(b, n_k, hk, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(b, n_k, hk, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    do = torch.randn(b, n_q, h, d, device="cuda", dtype=torch.bfloat16)
    out = ring_flash_attn_cuda(q, k, v, None, causal)
    got = (out, *torch.autograd.grad(out, (q, k, v), do))

    def oracle(dtype):
        qf, kf, vf = (t.detach().to(dtype).requires_grad_() for t in (q, k, v))
        o = attention_with_positions(qf, kf, vf, causal=causal)
        return (o.detach(), *torch.autograd.grad(o, (qf, kf, vf), do.to(dtype)))

    ref, lowp = oracle(torch.float32), oracle(torch.bfloat16)
    for name, g_, r_, l_ in zip(("out", "dq", "dk", "dv"), got, ref, lowp):
        res = gdc.noise_bound(g_, r_, l_)
        _report(f"cross {n_q}x{n_k} causal={causal}", {name: res})
        assert res["ok"], (name, res)
    if causal and n_q > n_k:
        dead = n_q - n_k
        assert (out[:, :dead] == 0).all() and (got[1][:, :dead] == 0).all()


def _fp8_case(regime, world=1, b=1, n=1024, h=2, hk=None, layout="plain", causal=True, hopwise=False, seed=0):
    """fp8 forward on a regime's inputs: relative RMS against the fp32 oracle on the dequantised inputs, and the bf16
    kernel's on the same inputs."""
    from ring_attention_pytorch_b200 import quantize_fp8
    from ring_attention_pytorch_b200.ops.fused import emulate_ring_forward, emulate_ring_forward_fp8

    hk = hk or h
    d = 128
    qs, ks, vs, _ = gdc.make_case_inputs(regime, world, b, n, h, hk, d, torch.float32, layout, causal, None, seed=seed)
    kq, kd = quantize_fp8(torch.cat(ks, 1), 1)
    vq, vd = quantize_fp8(torch.cat(vs, 1), 1)
    qq = [quantize_fp8(q, 1) for q in qs]
    k8, v8 = list(kq.split(n, 1)), list(vq.split(n, 1))
    outs, _ = emulate_ring_forward_fp8([q for q, _ in qq], k8, v8, [s for _, s in qq], kd, vd, layout=layout,
                                       causal=causal, hopwise=hopwise)

    def deq(t8, ds):
        return t8.float() * ds[:, None, :, None]

    qf = [deq(q, s) for q, s in qq]
    kf, vf = [deq(t, kd) for t in k8], [deq(t, vd) for t in v8]
    refs, _ = gdc._ref_ring(qf, kf, vf, layout, causal, None, 0.0, None)
    o16, _ = emulate_ring_forward([t.bfloat16() for t in qf], [t.bfloat16() for t in kf], [t.bfloat16() for t in vf],
                                  layout=layout, causal=causal, hopwise=hopwise)
    torch.cuda.synchronize()

    def rel(xs):
        num = sum((x.float() - r).pow(2).sum() for x, r in zip(xs, refs))
        return (num / sum(r.pow(2).sum() for r in refs)).sqrt().item()

    return rel(outs), rel(o16)


FP8 = {
    "sink6": dict(regime="sink6", n=4096),
    "sink10": dict(regime="sink10", n=4096),
    "sink10_gqa_b2": dict(regime="sink10", n=2048, b=2, h=8, hk=2),
    "sink10_ring2_hop": dict(regime="sink10", world=2, n=1024, hopwise=True),
    "sink6_ring4_striped_hop": dict(regime="sink6", world=4, n=512, layout="striped", hopwise=True),
    "late_spike": dict(regime="late_spike", n=384),
    "late_spike_ring2_hop": dict(regime="late_spike", world=2, n=256, hopwise=True),
    "peaky": dict(regime="peaky", n=1000, causal=False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FP8))
def test_fp8_forward_regimes(name):
    err8, err16 = _fp8_case(**FP8[name])
    print(f"[fp8 {name}] rel rms fp8 {err8:.3e}, bf16 {err16:.3e}, ratio {err8 / err16:.2f}")
    assert err8 <= REL_RMS_TOL, (err8, err16)
    assert err8 <= BF16_RATIO_TOL * err16, (err8, err16)
