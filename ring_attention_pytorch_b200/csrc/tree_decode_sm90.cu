// Tree-attention decode for sm_90a: one query token per (batch, head) against a KV cache that is sharded along the
// sequence across the ranks of one NVSwitch box — ONE persistent cooperative kernel per rank and step:
//
//   phase 1  split-KV flash decoding over this rank's shard.  Work units (batch*kv_head, group chunk, split) are handed
//            out by an atomic queue to a grid of co-resident CTAs.  Bandwidth bound, so the inner loop is built around
//            16-byte loads that are issued one tile AHEAD of their use (K of tile t+1 is in flight during the softmax and
//            P V of tile t, V of tile t+1 during the scores of tile t+1) and the g query heads that share a KV head are
//            processed together so K and V are read from HBM exactly once.  KV may be bf16 / fp16 or fp8-e4m3 with
//            per-head or per-block dequantisation scales (serve path).  The CTA that finishes the LAST split of a group
//            merges the splits and publishes (out, lse) in this rank's symmetric (peer-mapped) partial buffer.
//   phase 2  grid barrier (all partials of this rank are published) -> one st.release.sys per peer on its signal pad,
//            then every CTA waits until all peers have signalled this rank's pad (the pad is local memory).
//   phase 3  cross-rank merge with the max-rescale identity, one warp per (batch, head) row:
//              * P2P: every rank reads every peer's row straight over NVLink (W rows of d+2 floats), or
//              * NVLS: multimem.ld_reduce through the multicast mapping of the partial buffers — the NVSwitch returns
//                max_r(lse_r) and then sum_r(w_r out_r), sum_r(w_r) in two in-switch reductions.
//
// Replaces the reference's Triton launch padded to a 128-row tile plus three latency-bound NCCL all-reduces (MAX lse,
// SUM den, SUM num; tree_attn_decoding.py:60-102).  All counters are self-resetting and the cross-rank epoch lives in
// device memory, so the launch is CUDA-graph capturable; the host wrapper allocates nothing per call.
#include <cooperative_groups.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "tree_decode_common.cuh"

namespace rab {
namespace {

constexpr int TD_THREADS = 128;
constexpr int TD_TILE = 64;     // keys per inner tile
constexpr int TD_MAX_G = 4;     // query heads per kv head handled by one CTA (larger groups use more units)

// ---- raw 16-byte (bf16 / fp16) or 8-byte (fp8) vectors of 8 elements -> fp32 ---------------------------------------
template <int KV_KIND>  // 0 bf16, 1 fp16, 2 fp8 e4m3
struct KvVec;
template <>
struct KvVec<0> {
  using Raw = uint4;
  static constexpr int kBytes = 16;
  __device__ static void cvt(const Raw& v, float* out) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      out[2 * i] = __uint_as_float(w[i] << 16);
      out[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
};
template <>
struct KvVec<1> {
  using Raw = uint4;
  static constexpr int kBytes = 16;
  __device__ static void cvt(const Raw& v, float* out) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      out[2 * i] = f.x;
      out[2 * i + 1] = f.y;
    }
  }
};
template <>
struct KvVec<2> {
  using Raw = uint2;
  static constexpr int kBytes = 8;
  __device__ static void cvt(const Raw& v, float* out) {
    const uint32_t w[2] = {v.x, v.y};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        // cvt.rn.f16x2.e4m3x2: two fp8 values per instruction, then one unpack per pair
        const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)((w[i] >> (16 * j)) & 0xffffu), __NV_E4M3);
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
        out[4 * i + 2 * j] = f.x;
        out[4 * i + 2 * j + 1] = f.y;
      }
    }
  }
};


// RANGED: per-sequence visible key ranges and softclamp (TreeDecodeParams).  Key loads are clamped into [lo, k1), so a
// masked key's probability of 0 always multiplies a visible (finite) value row.  MULTI (with RANGED): the 4 columns of a
// unit are (query head, token) pairs of a multi-token call; the unit streams the union of its tokens' key ranges and
// masks each column with its own token's range.  PAGED (with RANGED): K / V rows come from page pools, each (clamped)
// key's row addressed through block_table and the pool strides with 64-bit offsets; the clamp into [lo, k1) keeps every
// table read on a page that holds a visible key.
template <int D, int KV_KIND, bool RANGED, bool MULTI, bool PAGED>
__device__ __forceinline__ void td_decode_body(const TreeDecodeParams& p) {
  static_assert(RANGED || !MULTI, "a multi-token call takes the ranged body");
  static_assert(RANGED || !PAGED, "a paged call takes the ranged body");
  using Vec = KvVec<KV_KIND>;
  using Raw = typename Vec::Raw;
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int g_total = MULTI ? p.heads / p.kv_heads * p.tokens : p.heads / p.kv_heads;  // columns per kv head
  const int zchunks = (g_total + TD_MAX_G - 1) / TD_MAX_G;
  const int groups = p.batch * p.kv_heads * zchunks;       // units = groups x splits
  const int total_units = p.n > 0 ? groups * p.splits : 0;
  constexpr int row_stride = TdCall<D, MULTI>::row_stride;
  uint32_t* const ctr = p.counters;                         // [0] queue head, [1] barrier count, [2] barrier gen, [3] epoch
  TdCall<D, MULTI> cs;
  cs.init(p);
  float* const my_partial = cs.my_partial;

  __shared__ __align__(16) float s_s[2][TD_TILE][TD_MAX_G];  // scores, then probabilities (double buffered per tile)
  __shared__ float corr_s[2][TD_MAX_G];
  __shared__ float red_s[8][TD_MAX_G][D + 1];
  __shared__ int unit_s;
  __shared__ uint32_t last_s;

  constexpr int EPL = D / 8;                    // QK: 8 lanes per key, EPL elements per lane
  constexpr int KVEC = EPL / 8;                 // 16-byte (8-byte for fp8) vectors per lane and key: 2 (D=128) or 1
  constexpr int CHUNKS = D / 8;                 // PV: thread -> (key group, 8-column chunk)
  constexpr int KGROUPS = TD_THREADS / CHUNKS;  // 8 or 16
  constexpr int KPT = TD_TILE / KGROUPS;        // keys per thread per tile: 8 or 4
  const int sub = lane / 8, l8 = lane % 8;
  const int chunk = tid % CHUNKS, kgrp = tid / CHUNKS;
  const size_t eb = KV_KIND == 2 ? 1 : 2;

  // =========================================== phase 1: split-KV partials ============================================
  while (true) {
    if (tid == 0) unit_s = (int)atomicAdd(&ctr[0], 1u);
    __syncthreads();
    const int unit = unit_s;
    __syncthreads();
    if (unit >= total_units) break;
    const int split = unit % p.splits;
    const int grp = unit / p.splits;
    const int zc = grp % zchunks;
    const int bhk = grp / zchunks;
    const int b = bhk / p.kv_heads, kvh = bhk % p.kv_heads;
    const int g0 = zc * TD_MAX_G;
    const int g = min(TD_MAX_G, g_total - g0);
    const int per = ((p.n + p.splits - 1) / p.splits + TD_TILE - 1) / TD_TILE * TD_TILE;  // tile-aligned splits
    int k0 = split * per, k1 = min(p.n, k0 + per), lo = 0;
    if constexpr (RANGED) {
      const TdUnitRange r = td_unit_range<TD_TILE, MULTI>(p, b, split);
      k0 = r.k0;
      k1 = r.k1;
      lo = r.lo;
    }
    // the partial row of column gi: (b, query head, token)
    auto prow = [&](int gi) -> size_t {
      const int c = g0 + gi;
      return ((size_t)b * p.heads + (size_t)(c / p.tokens) * p.kv_heads + kvh) * p.tokens + c % p.tokens;
    };
    int clo[TD_MAX_G], chi[TD_MAX_G];  // multi-token: the keys each column's token sees (read by MULTI only)
    if constexpr (MULTI) {
#pragma unroll
      for (int gi = 0; gi < TD_MAX_G; ++gi) {
        const TdColRange cr = td_col_range(p, b, (g0 + gi) % p.tokens, lo, k1);
        clo[gi] = cr.lo;
        chi[gi] = gi < g ? cr.hi : cr.lo;
      }
    }
    const float clamp_inv = RANGED && p.softclamp_log2 > 0.f ? 1.f / p.softclamp_log2 : 0.f;

    const float* ksb = p.k_scale ? p.k_scale + (size_t)bhk * p.n_scale_blocks : nullptr;
    const float* vsb = p.v_scale ? p.v_scale + (size_t)bhk * p.n_scale_blocks : nullptr;
    const uint8_t* kbase = reinterpret_cast<const uint8_t*>(p.k) + (size_t)bhk * p.n * D * eb;
    const uint8_t* vbase = reinterpret_cast<const uint8_t*>(p.v) + (size_t)bhk * p.n * D * eb;
    // paged: the byte offset of key's row from kbase / vbase (the kv head's offset in the pools)
    if constexpr (PAGED) {
      kbase = reinterpret_cast<const uint8_t*>(p.k) + (size_t)kvh * p.head_stride * eb;
      vbase = reinterpret_cast<const uint8_t*>(p.v) + (size_t)kvh * p.head_stride * eb;
    }
    auto page_off = [&](int key) -> size_t {
      const int page = __ldg(p.block_table + (size_t)b * p.max_pages + key / p.page_size);
      return ((size_t)page * p.page_stride + (size_t)(key % p.page_size) * p.slot_stride) * eb;
    };

    float2 qr[TD_MAX_G][EPL / 2];  // packed pairs: two lanes of a pair per dot-product step
#pragma unroll
    for (int gi = 0; gi < TD_MAX_G; ++gi) {
      if (RANGED && k0 >= k1) break;  // an empty unit loads nothing
#pragma unroll
      for (int e = 0; e < EPL / 2; ++e) {
        // query head j uses kv head j % kv_heads  ->  heads {kvh, kvh + hk, ...}
        const size_t qi = MULTI ? prow(gi) * D + l8 * EPL + 2 * e
                                : ((size_t)b * p.heads + (size_t)(g0 + gi) * p.kv_heads + kvh) * D + l8 * EPL + 2 * e;
        qr[gi][e] = gi < g ? make_float2(load_q(p.q, p.q_kind, qi) * p.scale_log2, load_q(p.q, p.q_kind, qi + 1) * p.scale_log2)
                           : make_float2(0.f, 0.f);
      }
    }
    float2 acc[TD_MAX_G][4];
#pragma unroll
    for (int gi = 0; gi < TD_MAX_G; ++gi)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[gi][e] = make_float2(0.f, 0.f);
    float m_run = -INFINITY, l_run = 0.f;  // warp gi keeps the running stats of head gi (identical in all lanes)

    Raw kraw[4][KVEC], vraw[KPT];
    auto load_k = [&](int t0) {
#pragma unroll
      for (int step = 0; step < 4; ++step) {
        int key = min(t0 + warp * 16 + step * 4 + sub, k1 - 1);  // clamp: loads stay in bounds
        if constexpr (RANGED) key = max(key, lo);
        const uint8_t* row = PAGED ? kbase + page_off(key) + (size_t)l8 * EPL * eb
                                   : kbase + ((size_t)key * D + l8 * EPL) * eb;
#pragma unroll
        for (int c = 0; c < KVEC; ++c) kraw[step][c] = *reinterpret_cast<const Raw*>(row + c * Vec::kBytes);
      }
    };
    auto load_v = [&](int t0) {
#pragma unroll
      for (int i = 0; i < KPT; ++i) {
        int key = min(t0 + kgrp + i * KGROUPS, k1 - 1);
        if constexpr (RANGED) key = max(key, lo);
        vraw[i] = *reinterpret_cast<const Raw*>(PAGED ? vbase + page_off(key) + (size_t)chunk * 8 * eb
                                                       : vbase + ((size_t)key * D + chunk * 8) * eb);
      }
    };
    if (k0 < k1) {
      load_k(k0);
      load_v(k0);
    }
    uint32_t par = 0;
    for (int t0 = k0; t0 < k1; t0 += TD_TILE, par ^= 1u) {
      const float ks = ksb ? ksb[t0 / p.scale_block] : 1.f;
      const float vs = vsb ? vsb[t0 / p.scale_block] : 1.f;
      const bool more = t0 + TD_TILE < k1;
      // ---- scores: consumes kraw ---------------------------------------------------------------------------------
#pragma unroll
      for (int step = 0; step < 4; ++step) {
        float kf[EPL];
#pragma unroll
        for (int c = 0; c < KVEC; ++c) Vec::cvt(kraw[step][c], kf + 8 * c);
        const int kl = warp * 16 + step * 4 + sub;
        const bool live = (t0 + kl) < k1 && (!RANGED || t0 + kl >= lo);
        float part[TD_MAX_G];
#pragma unroll
        for (int gi = 0; gi < TD_MAX_G; ++gi) {
          float2 a2 = make_float2(0.f, 0.f);
#pragma unroll
          for (int e = 0; e < EPL / 2; ++e) a2 = ffma2(make_float2(kf[2 * e], kf[2 * e + 1]), qr[gi][e], a2);
          float a = a2.x + a2.y;
          a += __shfl_xor_sync(0xffffffffu, a, 1);
          a += __shfl_xor_sync(0xffffffffu, a, 2);
          a += __shfl_xor_sync(0xffffffffu, a, 4);
          if constexpr (MULTI) {
            float x = a * ks;
            if (p.softclamp_log2 > 0.f) x = fast_tanh(x * clamp_inv) * p.softclamp_log2;
            part[gi] = (t0 + kl >= clo[gi] && t0 + kl < chi[gi]) ? x : -INFINITY;
          } else if constexpr (RANGED) {
            float x = a * ks;
            if (p.softclamp_log2 > 0.f) x = fast_tanh(x * clamp_inv) * p.softclamp_log2;
            part[gi] = live ? x : -INFINITY;
          } else {
            part[gi] = live ? a * ks : -INFINITY;
          }
        }
        if (l8 == 0) *reinterpret_cast<float4*>(&s_s[par][kl][0]) = make_float4(part[0], part[1], part[2], part[3]);
      }
      if (more) load_k(t0 + TD_TILE);  // in flight during the softmax and P V of this tile
      __syncthreads();
      // ---- online softmax: warp gi owns head gi ----------------------------------------------------------------
      if (warp < g) {
        const int gi = warp;
        const float a = s_s[par][lane][gi], bb = s_s[par][lane + 32][gi];
        float mx = fmaxf(a, bb);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        const float m_prev = m_run, l_prev = l_run;
        const float m_new = fmaxf(m_prev, mx);
        const float m_eff = m_new == -INFINITY ? 0.f : m_new;
        const float pa = fast_exp2(a - m_eff), pb = fast_exp2(bb - m_eff);
        float sum = pa + pb;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const float corr = m_prev == -INFINITY ? 0.f : fast_exp2(m_prev - m_eff);
        s_s[par][lane][gi] = pa * vs;  // V block scale rides on the probabilities (the denominator uses the unscaled p)
        s_s[par][lane + 32][gi] = pb * vs;
        m_run = m_new;
        l_run = l_prev * corr + sum;
        if (lane == 0) corr_s[par][gi] = corr;
      } else if (warp < TD_MAX_G) {
        // unused head slots must read as zero probability in the float4 broadcast below
        s_s[par][lane][warp] = 0.f;
        s_s[par][lane + 32][warp] = 0.f;
        if (lane == 0) corr_s[par][warp] = 0.f;
      }
      __syncthreads();
      // ---- P V: consumes vraw ---------------------------------------------------------------------------------------
#pragma unroll
      for (int gi = 0; gi < TD_MAX_G; ++gi) {
        const float c = corr_s[par][gi];
        const float2 c2 = make_float2(c, c);
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[gi][e] = fmul2(acc[gi][e], c2);
      }
#pragma unroll
      for (int i = 0; i < KPT; ++i) {
        float vf[8];
        Vec::cvt(vraw[i], vf);
        const int kl = kgrp + i * KGROUPS;
        const float4 p4 = *reinterpret_cast<const float4*>(&s_s[par][kl][0]);  // 0 for keys beyond the shard
        const float pk[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
        for (int gi = 0; gi < TD_MAX_G; ++gi) {
          const float2 p2 = make_float2(pk[gi], pk[gi]);
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[gi][e] = ffma2(p2, make_float2(vf[2 * e], vf[2 * e + 1]), acc[gi][e]);
        }
      }
      if (more) load_v(t0 + TD_TILE);  // in flight during the scores and the softmax of the next tile
      // no barrier here: the next tile writes the OTHER s_s / corr_s buffer; this one is rewritten two tiles later,
      // behind the two barriers of the next tile
    }

    // ---- reduce the key groups, write the split result ----------------------------------------------------------------
    __syncthreads();
    for (int gi = 0; gi < g; ++gi) {
      if (kgrp < 8) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          red_s[kgrp][gi][chunk * 8 + 2 * e] = acc[gi][e].x;
          red_s[kgrp][gi][chunk * 8 + 2 * e + 1] = acc[gi][e].y;
        }
      }
    }
    __syncthreads();
    if (KGROUPS > 8) {  // D = 64: 16 key groups, fold the upper 8 onto the lower 8
      for (int gi = 0; gi < g; ++gi) {
        if (kgrp >= 8) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            atomicAdd(&red_s[kgrp - 8][gi][chunk * 8 + 2 * e], acc[gi][e].x);
            atomicAdd(&red_s[kgrp - 8][gi][chunk * 8 + 2 * e + 1], acc[gi][e].y);
          }
        }
      }
      __syncthreads();
    }
    if (p.splits == 1) {
      // the unit IS the group: normalise and publish (out, lse2, valid) for its g heads directly
      if (warp < g && lane == 0) {
        corr_s[0][warp] = l_run > 0.f ? 1.f / l_run : 0.f;
        const int head = (g0 + warp) * p.kv_heads + kvh;
        float* row = my_partial + (MULTI ? prow(warp) : (size_t)b * p.heads + head) * row_stride;
        row[D] = l_run > 0.f ? (m_run == -INFINITY ? 0.f : m_run) + log2f(l_run) : -INFINITY;
        row[D + 1] = l_run > 0.f ? 1.f : 0.f;
      }
      __syncthreads();
      for (int i = tid; i < g * D; i += TD_THREADS) {
        const int gi = i / D, c = i % D;
        float sacc = 0.f;
#pragma unroll
        for (int kg = 0; kg < 8; ++kg) sacc += red_s[kg][gi][c];
        const int head = (g0 + gi) * p.kv_heads + kvh;
        my_partial[(MULTI ? prow(gi) : (size_t)b * p.heads + head) * row_stride + c] = sacc * corr_s[0][gi];
      }
    } else {
      float* out = p.scratch + (((size_t)bhk * p.splits + split) * g_total + g0) * row_stride;
      for (int i = tid; i < g * D; i += TD_THREADS) {
        const int gi = i / D, c = i % D;
        float sacc = 0.f;
#pragma unroll
        for (int kg = 0; kg < 8; ++kg) sacc += red_s[kg][gi][c];
        out[gi * row_stride + c] = sacc;
      }
      if (warp < g && lane == 0) {
        out[warp * row_stride + D] = m_run;
        out[warp * row_stride + D + 1] = l_run;
      }
      // the CTA that completes the last split of the group merges the splits
      __threadfence();
      __syncthreads();
      if (tid == 0) {
        const uint32_t done = atomicAdd(&p.group_done[grp], 1u);
        last_s = (done == (uint32_t)p.splits - 1) ? 1u : 0u;
        if (last_s) p.group_done[grp] = 0;  // self-resetting
      }
      __syncthreads();
      if (last_s) {
        __threadfence();
        for (int gi = 0; gi < g; ++gi) {
          const float* base = p.scratch + ((size_t)bhk * p.splits * g_total + g0 + gi) * row_stride;
          const size_t stride = (size_t)g_total * row_stride;
          float m = -INFINITY;
          for (int s = 0; s < p.splits; ++s) m = fmaxf(m, __ldcg(&base[s * stride + D]));
          const float m_eff = m == -INFINITY ? 0.f : m;
          float l = 0.f;
          for (int s = 0; s < p.splits; ++s) {
            const float ms = __ldcg(&base[s * stride + D]);
            l += ms == -INFINITY ? 0.f : __ldcg(&base[s * stride + D + 1]) * fast_exp2(ms - m_eff);
          }
          const int head = (g0 + gi) * p.kv_heads + kvh;
          float* row = my_partial + (MULTI ? prow(gi) : (size_t)b * p.heads + head) * row_stride;
          for (int c = tid; c < D; c += TD_THREADS) {
            float a = 0.f;
            for (int s = 0; s < p.splits; ++s) {
              const float ms = __ldcg(&base[s * stride + D]);
              if (ms != -INFINITY) a += __ldcg(&base[s * stride + c]) * fast_exp2(ms - m_eff);
            }
            row[c] = l > 0.f ? a / l : 0.f;
          }
          if (tid == 0) {
            row[D] = l > 0.f ? m_eff + log2f(l) : -INFINITY;
            row[D + 1] = l > 0.f ? 1.f : 0.f;
          }
        }
      }
    }
    __syncthreads();
  }
  td_cross_rank_merge<D, MULTI>(p, cs, total_units);
}

template <int D, int KV_KIND, bool RANGED, bool MULTI = false>
__global__ void __launch_bounds__(TD_THREADS)
tree_decode_kernel(const __grid_constant__ TreeDecodeParams p) {
  td_decode_body<D, KV_KIND, RANGED, MULTI, false>(p);
}

// paged K / V (TreeDecodeParams::block_table): always the ranged body.  Two CTAs per SM: without the hint ptxas caps the
// head-dim-64 fp8 variant at 128 registers and spills.
template <int D, int KV_KIND, bool MULTI>
__global__ void __launch_bounds__(TD_THREADS, 2)
tree_decode_paged_kernel(const __grid_constant__ TreeDecodeParams p) {
  td_decode_body<D, KV_KIND, true, MULTI, true>(p);
}

template <bool MULTI>
const void* pick_td_paged(int d, int kv_kind) {
  if (d == 128) {
    if (kv_kind == 0) return (const void*)tree_decode_paged_kernel<128, 0, MULTI>;
    if (kv_kind == 1) return (const void*)tree_decode_paged_kernel<128, 1, MULTI>;
    return (const void*)tree_decode_paged_kernel<128, 2, MULTI>;
  }
  if (kv_kind == 0) return (const void*)tree_decode_paged_kernel<64, 0, MULTI>;
  if (kv_kind == 1) return (const void*)tree_decode_paged_kernel<64, 1, MULTI>;
  return (const void*)tree_decode_paged_kernel<64, 2, MULTI>;
}

template <bool RANGED, bool MULTI = false>
const void* pick_td(int d, int kv_kind) {
  if (d == 128) {
    if (kv_kind == 0) return (const void*)tree_decode_kernel<128, 0, RANGED, MULTI>;
    if (kv_kind == 1) return (const void*)tree_decode_kernel<128, 1, RANGED, MULTI>;
    return (const void*)tree_decode_kernel<128, 2, RANGED, MULTI>;
  }
  if (kv_kind == 0) return (const void*)tree_decode_kernel<64, 0, RANGED, MULTI>;
  if (kv_kind == 1) return (const void*)tree_decode_kernel<64, 1, RANGED, MULTI>;
  return (const void*)tree_decode_kernel<64, 2, RANGED, MULTI>;
}

}  // namespace

int tree_decode_max_ctas(int d, int kv_kind, int num_sms, bool ranged, bool multi, bool paged) {
  int per_sm = 0;
  const void* fn = paged ? (multi ? pick_td_paged<true>(d, kv_kind) : pick_td_paged<false>(d, kv_kind))
                 : multi ? pick_td<true, true>(d, kv_kind)
                         : (ranged ? pick_td<true>(d, kv_kind) : pick_td<false>(d, kv_kind));
  cuda_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, TD_THREADS, 0), "tree_decode occupancy");
  return per_sm * num_sms;
}

void launch_tree_decode(const TreeDecodeParams& p, int d, int grid, cudaStream_t stream, bool ranged) {
  const bool multi = p.tokens > 1;
  const void* fn = p.block_table != nullptr
                       ? (multi ? pick_td_paged<true>(d, p.kv_kind) : pick_td_paged<false>(d, p.kv_kind))
                   : multi ? pick_td<true, true>(d, p.kv_kind)
                           : (ranged ? pick_td<true>(d, p.kv_kind) : pick_td<false>(d, p.kv_kind));
  void* args[] = {(void*)&p};
  // cooperative: the grid barrier and the cross-rank waits need every CTA of the grid to be resident
  cuda_check(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(TD_THREADS), args, 0, stream), "tree_decode launch");
}

}  // namespace rab
