"""The tree-decode kernels (``csrc/tree_decode_tc_sm90.cu``, ``csrc/tree_decode_sm90.cu`` and the split merge they share)
under the noise-scaled error rule, across head groups, split layouts, cache formats and cache views.

Every comparison uses ``gpu_dev_check.noise_bound`` with ``CAP_OUT`` on the maximum: the kernel's distance from the
fp32 oracle on the dequantised cache must stay within ``ERR_C`` times the distance of the same oracle run in the
cache's 16-bit type (bf16 for an fp8 cache), plus half a rounding step of the result, in both the maximum and the RMS.

The CPU half is a torch model of the kernels' algorithm (``emulate_decode``): tile-aligned key splits, an online
softmax per split over 64-key tiles, the per-block dequantisation scales, the merge of the splits and the sink.  It
passes the rule on every case, and each of a set of plausible kernel mistakes, applied to the same model, exceeds the
bound at least 3x on a case that exposes it.

The GPU half runs one table of cases (``CASES``) on both kernels and a few dedicated tests: the batch-256 shape of the
README, caches read in place through views, the cached buffers shared by calls of different shapes, empty shards and
bitwise reproducibility.  Each case names its kernel; a fixture restores ``tree_decode_cuda.CONFIG`` afterwards.
"""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import gpu_dev_check as gdc  # noqa: E402

from ring_attention_pytorch_b200.ops import tree_decode_cuda as tdc  # noqa: E402

TILE = 64  # keys per tile, in both kernels
LOG2E = 1.0 / math.log(2.0)
NOMINAL_RESIDENT = 132  # the CPU half's stand-in for the device's resident-CTA count (one CTA per H100 SM)
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


def split_layout(n, splits):
    """(per, non-empty splits) of the kernels' tile-aligned key splits: split s covers [s per, min(n, s per + per))."""
    per = ((n + splits - 1) // splits + TILE - 1) // TILE * TILE
    return per, ((n + per - 1) // per if n > 0 else 0)


def spike_position(regime, n, splits):
    """The key that a ``spike_*`` regime raises 10 nats above the rest (None for the other regimes)."""
    if regime not in ("spike_last_split", "spike_first_split"):
        return None
    per, live = split_layout(n, splits)
    first = 0 if regime == "spike_first_split" else (live - 1) * per
    return min(n - 1, first + 17)


# ================================================================================================
# inputs
# ================================================================================================
def make_inputs(regime, b, h, hk, n, d, *, spike_key=None, seed=0, device="cuda"):
    """fp32 ``q [b, h, 1, d]`` and ``k, v [b, hk, n, d]`` of an input regime.

    None      : N(0, 1)
    peaky     : ``make_case_inputs("peaky")``, q scaled by 8: nearly one-hot rows
    sink10    : ``make_case_inputs("sink10")``: key 0 sits 10 nats above the rest and V has a channel mean
    ramp      : N(0, 1), with the amplitude of K rising from 0.5 to 4 and that of V falling from 1 to 0.1 along the
                keys, so that neighbouring scale blocks of an fp8 cache get different scales
    spike_last_split / spike_first_split: the sink10 inputs with the 10-nat key moved to ``spike_key`` (keys and values
                roll together, which leaves the attention output unchanged): in the last non-empty split the merge
                has to scale the earlier splits down by 2^-14; in split 0 the later splits carry almost nothing
    The query is the last row of ``make_case_inputs``' sequence."""
    if regime is None:
        gen = torch.Generator(device).manual_seed(seed)
        q = torch.randn(b, h, 1, d, device=device, generator=gen)
        k = torch.randn(b, hk, n, d, device=device, generator=gen)
        v = torch.randn(b, hk, n, d, device=device, generator=gen)
        return q, k, v
    if regime == "ramp":
        q, k, v = make_inputs(None, b, h, hk, n, d, seed=seed, device=device)
        at = torch.linspace(0.0, 1.0, n, device=device)[None, None, :, None]
        return q, k * (0.5 + 3.5 * at), v * (1.0 - 0.9 * at)
    base = "sink10" if regime.startswith("spike") else regime
    qs, ks, vs, _ = gdc.make_case_inputs(base, 1, b, n, h, hk, d, torch.float32, seed=seed, device=device)
    q = qs[0][:, -1:].permute(0, 2, 1, 3).contiguous()
    k, v = (t[0].permute(0, 2, 1, 3).contiguous() for t in (ks, vs))
    if spike_key:
        k, v = k.roll(spike_key, 2), v.roll(spike_key, 2)
    return q, k, v


def make_cache(kind, q, k, v, seed=0):
    """The cache of a case from fp32 data.  Returns a dict: ``q`` (fp32, adjusted for ``fp8``), ``k`` / ``v`` as
    the kernel takes them, ``kd`` / ``vd`` the dequantised fp32 values, ``k_scale`` / ``v_scale`` / ``block`` (the
    kernel's scale arguments) and ``lowp``, the 16-bit type of the low-precision oracle.

    bf16, fp16 : the data in that type
    fp8_amax   : e4m3 with one scale per (batch, kv head), amax / 448
    fp8        : the same, but each (batch, kv head) of K and of V is first multiplied by its own factor spread over
                 three decades (K: 10^-1.5 .. 10^1.5, V: 10^-3 .. 1); the queries are divided by their K head's factor,
                 so the logits keep their scale and a scale read from the wrong row changes them by up to 1000x
    fp8_bB     : e4m3 with one scale per B keys (``scale_block_keys = B``), each block of K multiplied by a factor in
                 [1/2, 2] and each block of V by one in [1/100, 1]
    V is scaled down only, so that the output stays within the unit scale ``CAP_OUT`` is set for."""
    b, hk, n, d = k.shape
    h = q.shape[1]
    dev = k.device
    if kind in ("bf16", "fp16"):
        dt = DTYPES[kind]
        kc, vc = k.to(dt), v.to(dt)
        return dict(q=q, k=kc, v=vc, kd=kc.float(), vd=vc.float(), k_scale=None, v_scale=None, block=0, lowp=dt)
    gen = torch.Generator().manual_seed(seed + 1)
    e4m3 = torch.float8_e4m3fn
    if kind in ("fp8", "fp8_amax"):
        if kind == "fp8":
            ak = (10 ** (3 * torch.rand(b, hk, generator=gen) - 1.5)).to(dev)
            av = (10 ** (-3 * torch.rand(b, hk, generator=gen))).to(dev)
            k, v = k * ak[:, :, None, None], v * av[:, :, None, None]
            q = q / ak.repeat(1, h // hk)[:, :, None, None]  # query head j reads kv head j % hk
        ks = k.abs().amax(dim=(2, 3)) / 448.0
        vs = v.abs().amax(dim=(2, 3)) / 448.0
        k8, v8 = (k / ks[:, :, None, None]).to(e4m3), (v / vs[:, :, None, None]).to(e4m3)
        return dict(q=q, k=k8, v=v8, kd=k8.float() * ks[:, :, None, None], vd=v8.float() * vs[:, :, None, None],
                    k_scale=ks.reshape(-1).contiguous(), v_scale=vs.reshape(-1).contiguous(), block=0,
                    lowp=torch.bfloat16)
    blk = int(kind[len("fp8_b"):])
    nb = (n + blk - 1) // blk
    pad = nb * blk - n

    def quant(t, amp):
        t = t * amp.to(dev).repeat_interleave(blk, -1)[..., :n, None]
        tp = torch.nn.functional.pad(t, (0, 0, 0, pad)).view(b, hk, nb, blk, d)
        sc = tp.abs().amax(dim=(3, 4)).clamp(min=1e-30) / 448.0
        t8 = (tp / sc[..., None, None]).to(e4m3).view(b, hk, nb * blk, d)[:, :, :n].contiguous()
        deq = t8.float() * sc.repeat_interleave(blk, -1)[..., :n, None]
        return t8, sc.reshape(b * hk, nb).contiguous(), deq

    k8, ks, kd = quant(k, 2 ** (2 * torch.rand(b, hk, nb, generator=gen) - 1))
    v8, vs, vd = quant(v, 10 ** (-2 * torch.rand(b, hk, nb, generator=gen)))
    return dict(q=q, k=k8, v=v8, kd=kd, vd=vd, k_scale=ks, v_scale=vs, block=blk, lowp=torch.bfloat16)


def _round(x, dtype):
    return x.to(dtype).float() if dtype is not None and dtype != torch.float32 else x


# ================================================================================================
# CPU: a torch model of the kernels' algorithm, and mutants of it
# ================================================================================================
def emulate_decode(q, k, v, *, splits, k_scale=None, v_scale=None, block=0, sinks=None, p_dtype=None, mutant=None):
    """One decode step of the kernels on one rank, in fp32.

    q [b, h, 1, d]; k, v [b, hk, n, d] the cache's stored values (e4m3 values for an fp8 cache); ``k_scale`` /
    ``v_scale`` the kernel's ``[b*hk]`` or ``[b*hk, n_blocks]`` scales with ``block`` keys per block (0: per head).
    ``p_dtype``: the 16-bit type of the tensor-core kernel's MMA operands (q, and P times the V block scale), or None
    for the CUDA-core kernel, which keeps both in fp32.  The keys are cut into ``splits`` tile-aligned splits; each runs
    an online softmax over 64-key tiles with the K scale on the logits and the V scale on P (the denominator sums the
    unscaled P).  The last split's CTA merges them with weights 2^(m_s - m), and the sink joins the final denominator
    once.  ``mutant``:
      gqa_div           : query head j reads kv head j // g instead of j % hk
      drop_split_tail   : the last tile of every split is dropped
      no_merge_rescale  : the splits are merged with weight 1
      split_scale_block : every tile uses the block scale of its split's first key
      scale_head_swap   : the scale row of (b, kv head) is read at kvh * batch + b instead of b * hk + kvh
      v_scale_in_l      : the denominator sums P times the V scale
      sink_per_split    : the sink joins every split's partial instead of the merged denominator
    Returns fp32 [b, h, 1, d]."""
    b, h, _, d = q.shape
    hk, n = k.shape[1], k.shape[2]
    g = h // hk
    heads = torch.arange(h) // g if mutant == "gqa_div" else torch.arange(h) % hk
    kx, vx = k.float()[:, heads], v.float()[:, heads]  # [b, h, n, d]
    qf = q.float()[:, :, 0] if p_dtype is None else _round(q.float()[:, :, 0], p_dtype)
    bidx = torch.arange(b)[:, None]
    rows = heads[None, :] * b + bidx if mutant == "scale_head_swap" else bidx * hk + heads[None, :]  # [b, h]

    def scale_at(sc, key):
        if sc is None:
            return torch.ones(b, h)
        return sc.float().reshape(b * hk, -1)[rows, key // block if block else 0]

    scale_log2 = d ** -0.5 * LOG2E
    sg = None if sinks is None else sinks.float()[None, :].expand(b, h) * LOG2E
    per, _ = split_layout(n, splits)
    parts = []
    for s in range(splits):
        k0, k1 = s * per, min(n, s * per + per)
        m = torch.full((b, h), -math.inf)
        l = torch.zeros(b, h)
        o = torch.zeros(b, h, d)
        tiles = list(range(k0, k1, TILE))
        if mutant == "drop_split_tail":
            tiles = tiles[:-1]
        for t0 in tiles:
            t1 = min(k1, t0 + TILE)
            at = k0 if mutant == "split_scale_block" else t0
            ks, vs = scale_at(k_scale, at), scale_at(v_scale, at)
            st = torch.einsum("bhd,bhjd->bhj", qf, kx[:, :, t0:t1]) * (ks * scale_log2)[..., None]
            m_new = torch.maximum(m, st.amax(-1))
            corr = torch.where(torch.isfinite(m), torch.exp2(m - m_new), torch.zeros_like(m))
            p = torch.exp2(st - m_new[..., None])
            pv = p * vs[..., None]
            l = l * corr + (pv if mutant == "v_scale_in_l" else p).sum(-1)
            pv = pv if p_dtype is None else _round(pv, p_dtype)
            o = o * corr[..., None] + torch.einsum("bhj,bhjd->bhd", pv, vx[:, :, t0:t1])
            m = m_new
        if mutant == "sink_per_split" and sg is not None:
            m_new = torch.maximum(m, sg)
            corr = torch.where(torch.isfinite(m), torch.exp2(m - m_new), torch.zeros_like(m))
            l, o, m = l * corr + torch.exp2(sg - m_new), o * corr[..., None], m_new
        parts.append((m, l, o))
    # the merge of the splits (one split: the unit normalises its own rows)
    mm = torch.stack([p_[0] for p_ in parts])
    top = mm.amax(0)
    top_eff = torch.where(torch.isfinite(top), top, torch.zeros_like(top))
    w = torch.where(torch.isfinite(mm), torch.exp2(mm - top_eff), torch.zeros_like(mm))
    if mutant == "no_merge_rescale":
        w = torch.isfinite(mm).float()
    ll = sum(wi * p_[1] for wi, p_ in zip(w, parts))
    oo = sum(wi[..., None] * p_[2] for wi, p_ in zip(w, parts))
    live = ll > 0
    out = torch.where(live[..., None], oo / ll.clamp_min(1e-30)[..., None], torch.zeros_like(oo))
    lse2 = torch.where(live, top_eff + torch.log2(ll.clamp_min(1e-30)), torch.full_like(ll, -math.inf))
    if sg is not None and mutant != "sink_per_split":
        # the cross-rank merge of one rank: the sink is one more term of the denominator, with a zero value
        mx = torch.maximum(lse2, sg)
        wr = torch.where(live, torch.exp2(lse2 - mx), torch.zeros_like(mx))
        out = out * (wr / (wr + torch.exp2(sg - mx)))[..., None]
    return out[:, :, None]


def _kv_kind(cache):
    return {"bf16": 0, "fp16": 1}.get(cache, 2)


def _groups(b, h, hk, tensor_core):
    g = h // hk
    gm = (8 if g <= 8 else 16) if tensor_core else 4
    return b * hk * ((g + gm - 1) // gm)


# CPU cases: the splits are those of a device with NOMINAL_RESIDENT co-resident CTAs
CPU_CASES = {
    "bf16_tc_gqa": dict(tc=True, b=2, h=8, hk=2, n=1000, d=128, cache="bf16"),
    "fp16_cc_d64_g3": dict(tc=False, b=2, h=6, hk=2, n=777, d=64, cache="fp16", q="fp16"),
    "fp32_q_cc": dict(tc=False, b=2, h=4, hk=2, n=300, d=64, cache="bf16", q="fp32"),
    "fp32_q_tc": dict(tc=True, b=2, h=4, hk=2, n=300, d=128, cache="fp16", q="fp32"),
    "fp8_head_tc": dict(tc=True, b=2, h=6, hk=3, n=700, d=128, cache="fp8"),
    "fp8_head_cc": dict(tc=False, b=2, h=6, hk=3, n=700, d=64, cache="fp8"),
    "fp8_blk64_tc": dict(tc=True, b=1, h=4, hk=2, n=1000, d=128, cache="fp8_b64"),
    "fp8_blk128_cc": dict(tc=False, b=2, h=4, hk=2, n=1000, d=64, cache="fp8_b128"),
    "fp8_blk256_tc": dict(tc=True, b=1, h=4, hk=1, n=1100, d=128, cache="fp8_b256"),
    "peaky_g5_tc": dict(tc=True, b=2, h=10, hk=2, n=500, d=128, cache="bf16", regime="peaky"),
    "sink10_cc": dict(tc=False, b=1, h=4, hk=2, n=900, d=64, cache="bf16", regime="sink10"),
    "spike_last_split_tc": dict(tc=True, b=1, h=4, hk=2, n=2000, d=128, cache="bf16", regime="spike_last_split"),
    "spike_first_split_cc": dict(tc=False, b=1, h=4, hk=2, n=2000, d=64, cache="bf16", regime="spike_first_split"),
    "sinks_mix_g3_cc": dict(tc=False, b=2, h=6, hk=2, n=1500, d=64, cache="bf16", sinks=True),
    "sinks_mix_g5_tc_fp8": dict(tc=True, b=1, h=10, hk=2, n=1500, d=128, cache="fp8", sinks=True),
    # nearly one-hot rows: a sink at the row maximum takes about half of the row's mass
    "sinks_mix_peaky_g3_tc": dict(tc=True, b=1, h=6, hk=2, n=2000, d=128, cache="bf16", regime="peaky", sinks=True),
    "sinks_mix_peaky_g3_cc": dict(tc=False, b=1, h=6, hk=2, n=2000, d=64, cache="bf16", regime="peaky", sinks=True),
    # 8 groups, 8449 keys: 33 splits of 320 keys, the last 6 of them empty
    "empty_splits_tc": dict(tc=True, b=1, h=8, hk=8, n=8449, d=128, cache="bf16"),
    # 264 groups: one split of 5 tiles per unit
    "one_split_cc": dict(tc=False, b=33, h=8, hk=8, n=300, d=64, cache="bf16"),
}


def _cpu_case(name):
    c = dict(CPU_CASES[name])
    b, h, hk, n, d = c["b"], c["h"], c["hk"], c["n"], c["d"]
    splits = tdc._choose_splits(n, _groups(b, h, hk, c["tc"]), NOMINAL_RESIDENT)
    regime = c.get("regime")
    q, k, v = make_inputs(regime, b, h, hk, n, d, spike_key=spike_position(regime, n, splits), seed=7, device="cpu")
    cc = make_cache(c["cache"], q, k, v, seed=7)
    qdt = DTYPES[c.get("q", "bf16")]
    cc["q"] = cc["q"].to(qdt)
    cc["sinks"] = gdc.make_sinks("mix", [cc["q"].transpose(1, 2)], [cc["kd"].transpose(1, 2)]) if c.get("sinks") else None
    cc["p_dtype"] = (torch.float16 if c["cache"] == "fp16" else torch.bfloat16) if c["tc"] else None
    return cc, splits, qdt


def _emulated_ratio(name, mutant=None):
    cc, splits, qdt = _cpu_case(name)
    got = emulate_decode(cc["q"], cc["k"], cc["v"], splits=splits, k_scale=cc["k_scale"], v_scale=cc["v_scale"],
                         block=cc["block"], sinks=cc["sinks"], p_dtype=cc["p_dtype"], mutant=mutant)
    ref = gdc.decode_reference(cc["q"], cc["kd"], cc["vd"], cc["sinks"])
    lowp = gdc.decode_reference(cc["q"], cc["kd"], cc["vd"], cc["sinks"], dtype=cc["lowp"])
    res = gdc.noise_bound(_round(got, qdt), ref, lowp, gdc.CAP_OUT)
    n = CPU_CASES[name]["n"]
    per, live = split_layout(n, splits)
    return res, splits, splits - live, per


def test_cpu_cases_reach_the_split_regimes():
    """The nominal splits of the CPU cases include a single split of more than 4 tiles, many splits, and empty
    trailing splits."""
    def layout(name):
        c = CPU_CASES[name]
        s = tdc._choose_splits(c["n"], _groups(c["b"], c["h"], c["hk"], c["tc"]), NOMINAL_RESIDENT)
        return (s, *split_layout(c["n"], s))

    s, per, live = layout("one_split_cc")
    assert s == 1 and per // TILE > 4
    s, per, live = layout("empty_splits_tc")
    assert (s, per, s - live) == (33, 320, 6)
    s, per, live = layout("spike_last_split_tc")
    assert s > 1 and live == s


@pytest.mark.parametrize("name", list(CPU_CASES))
def test_rule_accepts_the_decode_algorithm(name):
    res, splits, empty, per = _emulated_ratio(name)
    print(f"[decode accept] {name}: splits {splits} empty {empty} per {per}: err {res['err']:.3e} "
          f"lowp {res['lowp_err']:.3e} bound {res['bound']:.3e} ratio {res['ratio']:.3f}")
    assert res["ok"], res


# (mutant, CPU case that exposes it)
MUTANTS = [
    ("gqa_div", "peaky_g5_tc"),
    ("gqa_div", "fp16_cc_d64_g3"),
    ("drop_split_tail", "bf16_tc_gqa"),
    ("drop_split_tail", "empty_splits_tc"),
    ("no_merge_rescale", "spike_last_split_tc"),
    ("split_scale_block", "fp8_blk64_tc"),
    ("split_scale_block", "fp8_blk128_cc"),
    ("scale_head_swap", "fp8_head_tc"),
    ("scale_head_swap", "fp8_head_cc"),
    ("v_scale_in_l", "fp8_head_cc"),
    ("v_scale_in_l", "fp8_blk64_tc"),
    ("sink_per_split", "sinks_mix_peaky_g3_tc"),
    ("sink_per_split", "sinks_mix_peaky_g3_cc"),
]


@pytest.mark.parametrize("mutant,case", MUTANTS)
def test_rule_rejects_decode_mistakes(mutant, case):
    res, splits, _, _ = _emulated_ratio(case, mutant)
    print(f"[decode reject] {mutant} on {case}: ratio {res['ratio']:.2f}")
    assert res["ratio"] >= 3.0, res


# ================================================================================================
# GPU: one table of cases
# ================================================================================================
@pytest.fixture
def decode_config():
    """Every GPU test here sets ``CONFIG["tensor_core"]`` itself; this puts the module's configuration back."""
    old = dict(tdc.CONFIG)
    yield tdc.CONFIG
    tdc.CONFIG.clear()
    tdc.CONFIG.update(old)


def _row(kernel, d=128, b=2, h=8, hk=2, n=1000, cache="bf16", q="bf16", regime=None, sinks=False, split=None,
         entry=None):
    """kernel: "on" (the wgmma kernel, head dim 128) or "off" (the CUDA-core kernel).  split: None, or the split
    regime the case must reach -- "one" (one split of more than 4 tiles; the batch is raised until the groups fill the
    grid), "multi", or "empty" (at least one empty trailing split; the batch and n are searched for it).  entry
    "attn" calls ``tree_attn_decode(shard_kv_seq=False)`` instead of ``tree_decode_cuda``."""
    return dict(kernel=kernel, d=d, b=b, h=h, hk=hk, n=n, cache=cache, q=q, regime=regime, sinks=sinks, split=split,
                entry=entry)


KERNELS = (("tc", "on", 128), ("cc128", "off", 128), ("cc64", "off", 64))
CASES = {}
# kernels x caches; n = 1000 is not a multiple of any scale block
for kname, kern, dd in KERNELS:
    for cache in ("bf16", "fp16", "fp8", "fp8_b64", "fp8_b128", "fp8_b256"):
        CASES[f"{kname}_{cache}"] = _row(kern, dd, cache=cache, q="fp16" if cache == "fp16" else "bf16")
# queries: fp32 queries give an fp32 output; fp16 queries on a bf16 cache
for kname, kern, dd in KERNELS:
    for cache in ("bf16", "fp8_b128"):
        CASES[f"{kname}_q32_{cache}"] = _row(kern, dd, b=3, h=6, hk=2, n=513, cache=cache, q="fp32")
    CASES[f"{kname}_q16_bf16"] = _row(kern, dd, n=700, q="fp16")
# head groups; the last head chunk is partly full for g = 3, 5, 6, 7 (CUDA-core) and 3, 5-7, 9-15, 17+ (tensor-core)
for g, hk in ((1, 8), (3, 2), (5, 1), (7, 2), (9, 1), (16, 2), (17, 1), (32, 8)):
    for kname, kern, dd in KERNELS[:2]:
        CASES[f"{kname}_g{g}_hk{hk}"] = _row(kern, dd, h=g * hk, hk=hk, n=777)
    if g in (3, 5, 7):
        CASES[f"cc64_g{g}_hk{hk}"] = _row("off", 64, h=g * hk, hk=hk, n=777, cache="fp8_b64")
# n at the tile edges
for n in (1, 63, 64, 65, 255, 256, 257, 4099):
    for kname, kern, dd in KERNELS[:2]:
        CASES[f"{kname}_n{n}"] = _row(kern, dd, b=3, n=n)
    if n in (1, 63, 65, 4099):
        CASES[f"cc64_n{n}"] = _row("off", 64, b=3, n=n, cache="fp16", q="fp16")
# split regimes, searched against the device's resident-CTA count
for kname, kern, dd in KERNELS:
    CASES[f"{kname}_one_split"] = _row(kern, dd, b=1, h=32, hk=8, n=1000, split="one")
    CASES[f"{kname}_multi_split"] = _row(kern, dd, b=1, h=8, hk=2, n=4099, split="multi")
    CASES[f"{kname}_empty_splits"] = _row(kern, dd, b=1, h=8, hk=8, n=None, split="empty")
CASES["tc_one_split_fp8"] = _row("on", b=1, h=32, hk=8, n=1000, cache="fp8", split="one")
CASES["cc128_empty_splits_fp8_b128"] = _row("off", b=1, h=8, hk=8, n=None, cache="fp8_b128", split="empty")
# input regimes
for regime in ("peaky", "sink10", "spike_last_split", "spike_first_split"):
    for kname, kern, dd in KERNELS:
        CASES[f"{kname}_{regime}"] = _row(kern, dd, b=2, h=8, hk=2, n=2500, regime=regime, split="multi")
CASES["tc_spike_last_split_fp8_b128"] = _row("on", b=2, h=8, hk=2, n=2500, cache="fp8_b128", regime="spike_last_split",
                                             split="multi")
# sinks on a partly full head chunk
CASES["tc_sinks_g5"] = _row("on", h=10, hk=2, n=3000, sinks=True, split="multi")
CASES["tc_sinks_g9_fp8"] = _row("on", h=9, hk=1, n=3000, cache="fp8", sinks=True, split="multi")
CASES["cc128_sinks_g3"] = _row("off", h=6, hk=2, n=3000, sinks=True, split="multi")
CASES["cc64_sinks_g3_one_split"] = _row("off", 64, h=24, hk=8, n=1000, sinks=True, split="one")
# the shapes the earlier fixed-bound decode tests used
for b, h, hk, n, d, dt in ((2, 8, 8, 1000, 128, "bf16"), (3, 8, 2, 4097, 128, "bf16"), (2, 16, 2, 777, 64, "fp16"),
                           (1, 4, 4, 31, 128, "bf16"), (4, 32, 8, 8192, 128, "bf16"), (2, 40, 2, 3000, 128, "fp16")):
    for kname, kern, dd in KERNELS[:2] if d == 128 else KERNELS[2:]:
        CASES[f"{kname}_attn_b{b}_h{h}_hk{hk}_n{n}"] = _row(kern, dd, b=b, h=h, hk=hk, n=n, cache=dt, q=dt,
                                                             entry="attn")
for kname, kern, dd in KERNELS[:2]:
    CASES[f"{kname}_fp8_amax_b2_h16_hk4_n2048"] = _row(kern, b=2, h=16, hk=4, n=2048, cache="fp8_amax")
for regime in ("sink10", "peaky"):
    for kname, kern, dd in KERNELS[:2]:
        CASES[f"{kname}_{regime}_b3_h8_hk1_n1000"] = _row(kern, b=3, h=8, hk=1, n=1000, regime=regime)
    CASES[f"cc64_{regime}_b2_h16_hk2_n777"] = _row("off", 64, b=2, h=16, hk=2, n=777, cache="fp16", q="fp16",
                                                   regime=regime)


def _resolve(c):
    """(b, n, plan) of a case, with the batch or n searched for its split regime."""
    b, h, hk, n, d = c["b"], c["h"], c["hk"], c["n"], c["d"]
    kind = _kv_kind(c["cache"])
    if c["split"] == "one":
        p = tdc.decode_plan(b, h, hk, n, d, kind)
        b = max(b, -(-2 * p.resident // (p.groups // b)))  # enough groups to fill the grid twice: one split each
    elif c["split"] == "empty":
        p = tdc.decode_plan(b, h, hk, 1, d, kind)
        per_b = p.groups // b
        b = max(1, 2 * p.resident // (40 * per_b))  # about 40 splits' worth of groups
        want = -(-2 * p.resident // (b * per_b))
        for n in range(256 * want + 1, 256 * want + 8 * TILE * want):
            s = tdc._choose_splits(n, b * per_b, p.resident)
            if split_layout(n, s)[1] < s:
                break
    return b, n, tdc.decode_plan(b, h, hk, n, d, kind)


def _stats(plan, n):
    per, live = split_layout(n, plan.splits)
    return per, plan.splits - live, -(-min(per, n) // TILE)


def _run_decode(c, b, n, plan, seed=0):
    h, hk, d = c["h"], c["hk"], c["d"]
    q, k, v = make_inputs(c["regime"], b, h, hk, n, d, spike_key=spike_position(c["regime"], n, plan.splits),
                          seed=seed)
    cc = make_cache(c["cache"], q, k, v, seed=seed)
    qc = cc["q"].to(DTYPES[c["q"]])
    sinks = gdc.make_sinks("mix", [qc.transpose(1, 2)], [cc["kd"].transpose(1, 2)]) if c["sinks"] else None
    if c["entry"] == "attn":
        from ring_attention_pytorch_b200 import tree_attn_decode

        out = tree_attn_decode(qc, cc["k"], cc["v"], shard_kv_seq=False, sinks=sinks)
    else:
        out = tdc.tree_decode_cuda(qc, cc["k"], cc["v"], dim_v=d, k_scale=cc["k_scale"], v_scale=cc["v_scale"],
                                   scale_block_keys=cc["block"], sinks=sinks)
    assert out.shape == (b, h, 1, d) and out.dtype == qc.dtype
    ref = gdc.decode_reference(qc, cc["kd"], cc["vd"], sinks)
    lowp = gdc.decode_reference(qc, cc["kd"], cc["vd"], sinks, dtype=cc["lowp"])
    return gdc.noise_bound(out, ref, lowp, gdc.CAP_OUT), out


def _print(name, c, plan, n, res, b=None):
    per, empty, tiles = _stats(plan, n)
    print(f"[decode {name}] kernel {'tc' if plan.tensor_core else 'cuda-core'} d {c['d']} cache {c['cache']} "
          f"q {c['q']} b {b or c['b']} n {n} g {c['h'] // c['hk']} splits {plan.splits} empty {empty} "
          f"tiles/unit {tiles}: err {res['err']:.3e} lowp {res['lowp_err']:.3e} bound {res['bound']:.3e} "
          f"rms {res['rms']:.3e} rms bound {res['rms_bound']:.3e} ratio {res['ratio']:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_decode_case(name, decode_config):
    c = CASES[name]
    decode_config["tensor_core"] = c["kernel"]
    b, n, plan = _resolve(c)
    assert plan.tensor_core == (c["kernel"] == "on" and n >= 1)
    per, empty, tiles = _stats(plan, n)
    if c["split"] == "one":
        assert plan.splits == 1 and tiles > 4, (plan, n)
    elif c["split"] == "multi":
        assert plan.splits > 1, plan
    elif c["split"] == "empty":
        assert empty >= 1, (plan, n)
    res, _ = _run_decode(c, b, n, plan)
    _print(name, c, plan, n, res, b)
    assert res["ok"], res


# ================================================================================================
# GPU: dedicated tests
# ================================================================================================
@pytest.mark.gpu
def test_decode_block_scaled_fp8_kv(decode_config):
    """An fp8 cache with one scale per 128 keys of every (batch, kv head), on the ``ramp`` inputs: K and V drift
    along the keys, so each tile must take its own block's scale.  Both kernels, under the rule."""
    for kernel in ("on", "off"):
        decode_config["tensor_core"] = kernel
        c = _row(kernel, b=2, h=8, hk=2, n=1000, cache="fp8_b128", regime="ramp", split="multi")
        plan = tdc.decode_plan(c["b"], c["h"], c["hk"], c["n"], c["d"], _kv_kind(c["cache"]))
        assert plan.tensor_core == (kernel == "on") and plan.splits > 1, plan
        res, _ = _run_decode(c, c["b"], c["n"], plan)
        _print(f"block_scaled_{kernel}", c, plan, c["n"], res)
        assert res["ok"], (kernel, res)


@pytest.mark.gpu
@pytest.mark.parametrize("cache", ["bf16", "fp8_amax"])
def test_decode_readme_shape(cache, decode_config):
    """The README's decode workload -- batch 256, 32 query / 8 kv heads, 8192 keys, head dim 128 -- with every row
    under the rule.  The bf16 K / V take 8.6 GB; the data is made and dequantised 16 sequences at a time, and the test
    skips when the device has less than 24 GB free."""
    decode_config["tensor_core"] = "auto"
    b, h, hk, n, d, chunk = 256, 32, 8, 8192, 128, 16
    free, _ = torch.cuda.mem_get_info()
    if free < 24 * 2 ** 30:
        msg = f"needs 24 GB free for the batch-256 decode shape, {free / 2 ** 30:.1f} GB free"
        print(f"[decode readme {cache}] skipped: {msg}")
        pytest.skip(msg)
    gen = torch.Generator("cuda").manual_seed(0)
    q = torch.randn(b, h, 1, d, device="cuda", generator=gen, dtype=torch.bfloat16)
    k = torch.randn(b, hk, n, d, device="cuda", generator=gen, dtype=torch.bfloat16)
    v = torch.randn(b, hk, n, d, device="cuda", generator=gen, dtype=torch.bfloat16)
    kw = {}
    if cache == "fp8_amax":  # one scale per (batch, kv head), amax / 448
        ks, vs = (t.abs().amax(dim=(2, 3)).float() / 448.0 for t in (k, v))
        k8, v8 = (torch.empty(t.shape, device="cuda", dtype=torch.float8_e4m3fn) for t in (k, v))
        for i in range(0, b, chunk):
            k8[i:i + chunk] = (k[i:i + chunk].float() / ks[i:i + chunk, :, None, None]).to(torch.float8_e4m3fn)
            v8[i:i + chunk] = (v[i:i + chunk].float() / vs[i:i + chunk, :, None, None]).to(torch.float8_e4m3fn)
        k, v = k8, v8
        kw = dict(k_scale=ks.reshape(-1).contiguous(), v_scale=vs.reshape(-1).contiguous())
    plan = tdc.decode_plan(b, h, hk, n, d, _kv_kind(cache))
    out = tdc.tree_decode_cuda(q, k, v, dim_v=d, **kw)
    refs, lows = [], []
    for i in range(0, b, chunk):
        kd, vd = k[i:i + chunk].float(), v[i:i + chunk].float()
        if kw:
            kd = kd * kw["k_scale"].view(b, hk)[i:i + chunk, :, None, None]
            vd = vd * kw["v_scale"].view(b, hk)[i:i + chunk, :, None, None]
        refs.append(gdc.decode_reference(q[i:i + chunk], kd, vd))
        lows.append(gdc.decode_reference(q[i:i + chunk], kd, vd, dtype=torch.bfloat16))
    res = gdc.noise_bound(out, refs, lows, gdc.CAP_OUT)
    _print(f"readme {cache}", _row("auto", b=b, h=h, hk=hk, n=n, cache=cache), plan, n, res)
    assert plan.tensor_core and plan.splits == 1
    assert res["ok"], res


def _nan_fill(t):
    """Fill a cache with NaN (0x7F in e4m3)."""
    if t.dtype == torch.float8_e4m3fn:
        t.view(torch.uint8).fill_(0x7F)
    else:
        t.fill_(float("nan"))
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["on", "off"])
@pytest.mark.parametrize("cache", ["bf16", "fp8_b128"])
@pytest.mark.parametrize("b,hk", [(3, 2), (1, 4), (2, 1)])
def test_decode_reads_cache_views_in_place(kernel, cache, b, hk, decode_config):
    """k / v = a prefix ``cache[:, :, :n]`` or a chunk ``cache[:, :, s:s+n]`` (s > 0) of a larger buffer whose every
    other entry is NaN.  The tensor-core kernel reads the view in place (b = 1 or hk = 1: the wrapper copies it); a key
    read outside the view would put NaN in the output.  The result must be bitwise the one of the view's contiguous
    copy, and pass the rule.  The fp8 cache has scales for the whole capacity: the prefix passes them as they are,
    the chunk (s a multiple of the block) the contiguous slice from block s / 128 on."""
    decode_config["tensor_core"] = kernel
    h, d, cap = 4 * hk, 128, 2048
    q, k, v = make_inputs(None, b, h, hk, cap, d, seed=3)
    cc = make_cache(cache, q, k, v, seed=3)
    qc = cc["q"].to(torch.bfloat16)
    kfull, vfull = cc["k"], cc["v"]
    for s, n in ((0, 300), (0, 1025), (256, 777), (1024, 1000), (1280, 5)):
        kv = [_nan_fill(torch.empty_like(t)) for t in (kfull, vfull)]
        for t, src in zip(kv, (kfull, vfull)):
            t[:, :, s:s + n] = src[:, :, s:s + n]
        kview, vview = (t[:, :, s:s + n] for t in kv)
        assert tdc._is_cache_prefix(kview) == (b > 1 and hk > 1)
        kw = {}
        if cc["block"]:
            blk = cc["block"]
            kw = dict(k_scale=cc["k_scale"][:, s // blk:].contiguous(), v_scale=cc["v_scale"][:, s // blk:].contiguous(),
                      scale_block_keys=blk)
        got = tdc.tree_decode_cuda(qc, kview, vview, dim_v=d, **kw)
        want = tdc.tree_decode_cuda(qc, kview.contiguous(), vview.contiguous(), dim_v=d, **kw)
        assert torch.equal(got, want), (s, n)
        kd, vd = cc["kd"][:, :, s:s + n], cc["vd"][:, :, s:s + n]
        ref = gdc.decode_reference(qc, kd, vd)
        res = gdc.noise_bound(got, ref, gdc.decode_reference(qc, kd, vd, dtype=torch.bfloat16), gdc.CAP_OUT)
        print(f"[decode view {kernel} {cache} b {b} hk {hk} s {s} n {n}] err {res['err']:.3e} "
              f"bound {res['bound']:.3e} ratio {res['ratio']:.3f}")
        assert res["ok"], (s, n, res)


@pytest.mark.gpu
def test_decode_buffer_reuse_across_shapes_and_kernels(decode_config):
    """One sequence of calls that share the cached buffers (same b * h and head dim): kv heads, n, cache type and
    kernel change from call to call, so the self-resetting queue and group counters, the epoch and the two halves of
    the partial buffer carry over between both kernels.  Every call is checked against the oracle, and the first
    shape, repeated at the end, must give bitwise the same result."""
    b, h, d = 4, 16, 128
    calls = [("on", 4, 1000, "bf16"), ("off", 16, 65, "fp16"), ("on", 1, 4099, "fp8"), ("off", 2, 300, "bf16"),
             ("off", 8, 2048, "fp8_b64"), ("on", 16, 1, "fp16"), ("on", 2, 8449, "fp8_b256"), ("off", 4, 1000, "bf16"),
             ("on", 4, 1000, "bf16")]
    first = None
    for i, (kernel, hk, n, cache) in enumerate(calls):
        decode_config["tensor_core"] = kernel
        c = _row(kernel, d, b=b, h=h, hk=hk, n=n, cache=cache, q="fp16" if cache == "fp16" else "bf16")
        plan = tdc.decode_plan(b, h, hk, n, d, _kv_kind(cache))
        res, out = _run_decode(c, b, n, plan, seed=11 if (kernel, hk, n, cache) == calls[0] else i)
        _print(f"reuse {i}", c, plan, n, res)
        assert res["ok"], (i, res)
        if first is None:
            first = out.clone()
    assert torch.equal(out, first)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["on", "off"])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("with_sinks", [False, True])
def test_decode_empty_shard_is_zero(kernel, d, with_sinks, decode_config):
    """A rank that holds no keys (``k = None`` or n = 0) gives exactly zero: the sink has a zero value vector."""
    from ring_attention_pytorch_b200 import tree_attn_decode

    decode_config["tensor_core"] = kernel
    b, h, hk = 3, 8, 2
    q = torch.randn(b, h, 1, d, device="cuda", dtype=torch.bfloat16)
    sinks = torch.linspace(-3.0, 12.0, h, device="cuda") if with_sinks else None
    empty = torch.empty(b, hk, 0, d, device="cuda", dtype=torch.bfloat16)
    outs = [tdc.tree_decode_cuda(q, None, None, dim_v=d, sinks=sinks),
            tdc.tree_decode_cuda(q, empty, empty, dim_v=d, sinks=sinks),
            tree_attn_decode(q, None, None, shard_kv_seq=False, dim_v=d, sinks=sinks)]
    for out in outs:
        assert out.shape == (b, h, 1, d) and out.dtype == q.dtype
        assert torch.equal(out, torch.zeros_like(out))


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["on", "off"])
@pytest.mark.parametrize("cache", ["bf16", "fp8_b128"])
def test_decode_is_bitwise_reproducible(kernel, cache, decode_config):
    """Only the work queue uses atomics; every sum runs in a fixed order.  So two identical calls agree bitwise,
    whichever CTA took which unit."""
    decode_config["tensor_core"] = kernel
    b, h, hk, n, d = 2, 12, 2, 5000, 128
    q, k, v = make_inputs("sink10", b, h, hk, n, d, seed=5)
    cc = make_cache(cache, q, k, v, seed=5)
    qc = cc["q"].to(torch.bfloat16)
    sinks = torch.linspace(-2.0, 4.0, h, device="cuda")
    plan = tdc.decode_plan(b, h, hk, n, d, _kv_kind(cache))
    assert plan.splits > 1

    def call():
        return tdc.tree_decode_cuda(qc, cc["k"], cc["v"], dim_v=d, k_scale=cc["k_scale"], v_scale=cc["v_scale"],
                                    scale_block_keys=cc["block"], sinks=sinks)

    first = call().clone()
    for _ in range(3):
        assert torch.equal(call(), first)
