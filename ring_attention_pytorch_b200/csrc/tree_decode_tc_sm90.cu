// Tree-attention decode on the Hopper tensor cores (head dim 128, up to 16 query heads -- or 32 (query head, token)
// columns of a multi-token call -- per work unit).
//
// A decode step is bandwidth bound, but with grouped-query heads the CUDA-core split-KV kernel (tree_decode_sm90.cu)
// spends g FMAs per loaded element on its own dependency chains.  Here both products run as wgmma in the TRANSPOSED
// form, so that keys / head-dim entries are the 64 MMA rows and the (few) query heads are MMA columns:
//
//      S^T [64 keys x NH heads] = K_tile [64 x d] . Q^T [d x NH]        A = K tile (TMA, K-major), B = Q (smem)
//      O^T [d x NH]            += V_tile^T [d x 64] . P [64 x NH]       A = V tile read MN-major, B = P (smem)
//
// K / V tiles of 64 keys are streamed by TMA through a 4-stage mbarrier ring straight from the cache (any plane stride,
// so a growing cache is read in place).  bf16 / fp16 caches feed the MMA directly; an fp8-e4m3 cache is loaded at half
// the bytes and widened to bf16 in shared memory (wgmma takes fp8 operands K-major only, and V^T is MN-major).  The
// per-block dequantisation scales ride on the logits (K) and on the probabilities (V).  The online softmax runs in the
// accumulator registers: per head, a tile maximum over the warpgroup, then exp2 and the rescale of O^T.
//
// One warpgroup per CTA takes work units (batch*kv_head, head chunk, split) from the same atomic queue as the CUDA-core
// kernel, and phases 2 and 3 of the step (publish -> cross-rank signal -> merge over NVLink loads or NVLS multimem) are
// shared with it (tree_decode_common.cuh): the whole step is still ONE cooperative launch.
// Reference: tree_attn_decoding.py:60-102.
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <type_traits>

// no printf in the watchdogs: a function call would serialize this kernel's wgmma (see ptx.cuh)
#define RAB_WATCHDOG_PRINTF 0
#include "tree_decode_common.cuh"

namespace rab {
namespace {

constexpr int TC_THREADS = 128;
constexpr int TC_TILE = 64;  // keys per tile
constexpr int TC_D = 128;
constexpr int TC_NST = 4;
constexpr int TC_SUB = TC_TILE * 128;  // one 128-byte wide, 64-key swizzled sub-tile

template <bool KV8, int NH>
struct TcSmem {
  static constexpr int TILE_BYTES = KV8 ? TC_SUB : 2 * TC_SUB;
  alignas(1024) uint8_t k[TC_NST][TILE_BYTES];
  alignas(1024) uint8_t v[TC_NST][TILE_BYTES];
  alignas(1024) uint8_t kc[KV8 ? 2 * TC_SUB : 16];  // fp8 tiles widened to bf16
  alignas(1024) uint8_t vc[KV8 ? 2 * TC_SUB : 16];
  alignas(1024) uint8_t q[2][NH * 128];  // Q as B operand: [d half][head][64 d] (128B swizzle)
  alignas(1024) uint8_t p[NH * 128];     // P as B operand: [head][64 keys]
  float red[4][NH];
  float o[NH][TC_D + 1];
  float ml[2][NH];
  uint64_t full[TC_NST];
  int unit;
  uint32_t last;
};
// multi-token units: the visible keys [clo, chi) of each column (its token's range within the unit's [lo, k1))
template <bool KV8, int NH>
struct TcSmemMulti : TcSmem<KV8, NH> {
  int clo[NH], chi[NH];
};

template <bool F16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  return F16 ? pack_f16x2(a, b) : pack_bf16x2(a, b);
}

// one fp8 tile [64 keys][128 B, swizzled] -> bf16 [2][64 keys][128 B, swizzled]
__device__ __forceinline__ void widen_fp8_tile(const uint8_t* src, uint8_t* dst, int tid) {
#pragma unroll
  for (int i = 0; i < (TC_TILE * 8) / TC_THREADS; ++i) {
    const int idx = tid + i * TC_THREADS;
    const int row = idx / 8, pc = idx % 8;
    const int lc = pc ^ (row & 7);  // logical 16-element chunk: d = 16 lc .. 16 lc + 15
    const uint4 raw = *reinterpret_cast<const uint4*>(src + row * 128 + pc * 16);
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
    uint32_t out[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)((w[j] >> (16 * h)) & 0xffffu), __NV_E4M3);
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
        out[2 * j + h] = pack_bf16x2(f.x, f.y);
      }
    }
    uint8_t* sub = dst + (lc / 4) * TC_SUB + row * 128;
    const int c0 = 2 * (lc % 4);
    *reinterpret_cast<uint4*>(sub + ((c0 ^ (row & 7)) << 4)) = make_uint4(out[0], out[1], out[2], out[3]);
    *reinterpret_cast<uint4*>(sub + (((c0 + 1) ^ (row & 7)) << 4)) = make_uint4(out[4], out[5], out[6], out[7]);
  }
}

// KVK: 0 bf16, 1 fp16, 2 fp8-e4m3 cache.  NH: query heads per unit (MMA N).  RANGED: per-sequence visible key ranges
// and softclamp (TreeDecodeParams); V rows of invisible keys in a unit's boundary tiles are zeroed in shared memory,
// since a probability of 0 does not cancel a NaN value row inside the MMA.  MULTI (with RANGED): the columns are the
// (query head, token) pairs of a multi-token call; the unit streams the union of its tokens' key ranges and, in the
// tiles that cross some column's bounds, masks each (key, column) with that column's range.  PAGED (with RANGED): K / V
// come from page pools through 4-D tensor maps (d, page_size, hk, num_pages), one box of min(page_size, 64) keys per
// page run of a sub-tile; each box's first key is clamped into [lo, k1 - 1] before its page id is read, so only table
// entries of visible pages are dereferenced (the boxes that clamp away are masked like any key outside the range).
template <int KVK, int NH, bool RANGED, bool MULTI, bool PAGED>
__device__ __forceinline__ void tc_decode_body(const CUtensorMap& map_k, const CUtensorMap& map_v,
                                               const TreeDecodeParams& p) {
  static_assert(RANGED || !MULTI, "a multi-token call takes the ranged body");
  static_assert(RANGED || !PAGED, "a paged call takes the ranged body");
  constexpr bool KV8 = KVK == 2;
  constexpr bool F16 = KVK == 1;
  constexpr int D = TC_D;
  constexpr int NJ = NH / 8;  // n8 column blocks of the accumulators
  using Smem = std::conditional_t<MULTI, TcSmemMulti<KV8, NH>, TcSmem<KV8, NH>>;
  extern __shared__ uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int r_lo = warp * 16 + lane / 4;  // accumulator rows r_lo, r_lo + 8
  const int cq = 2 * (lane % 4);          // accumulator columns 8 j + cq (+1)
  const int g_total = MULTI ? p.heads / p.kv_heads * p.tokens : p.heads / p.kv_heads;  // columns per kv head
  const int zchunks = (g_total + NH - 1) / NH;
  const int groups = p.batch * p.kv_heads * zchunks;
  const int total_units = p.n > 0 ? groups * p.splits : 0;
  constexpr int row_stride = TdCall<D, MULTI>::row_stride;
  uint32_t* const ctr = p.counters;
  TdCall<D, MULTI> cs;
  cs.init(p);
  float* const my_partial = cs.my_partial;

  constexpr uint64_t kmaj = gmma_desc_static(16, 1024);
  constexpr uint64_t mnmaj = gmma_desc_static(TC_SUB, 1024);
  constexpr uint32_t TX = KV8 ? 2 * TC_SUB : 4 * TC_SUB;  // K + V bytes of one tile

  if (tid == 0) {
    for (int i = 0; i < TC_NST; ++i) mbar_init(&sm.full[i], 1);
    fence_mbar_init();
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
  }
  __syncthreads();

  uint32_t n_tile = 0;  // tiles consumed by this CTA so far (stage ring position)
  while (true) {
    if (tid == 0) sm.unit = (int)atomicAdd(&ctr[0], 1u);
    __syncthreads();
    const int unit = sm.unit;
    if (unit >= total_units) break;
    const int split = unit % p.splits;
    const int grp = unit / p.splits;
    const int zc = grp % zchunks;
    const int bhk = grp / zchunks;
    const int b = bhk / p.kv_heads, kvh = bhk % p.kv_heads;
    const int g0 = zc * NH;
    const int g = min(NH, g_total - g0);
    const int per = ((p.n + p.splits - 1) / p.splits + TC_TILE - 1) / TC_TILE * TC_TILE;  // tile-aligned splits
    int k0 = split * per, k1 = min(p.n, k0 + per), lo = 0;
    if constexpr (RANGED) {
      const TdUnitRange r = td_unit_range<TC_TILE, MULTI>(p, b, split);
      k0 = r.k0;
      k1 = r.k1;
      lo = r.lo;
    }
    const int ntiles = k0 < k1 ? (k1 - k0 + TC_TILE - 1) / TC_TILE : 0;
    // the partial row of column gi: (b, query head, token)
    auto prow = [&](int gi) -> size_t {
      if constexpr (MULTI) {
        const int c = g0 + gi;
        return ((size_t)b * p.heads + (size_t)(c / p.tokens) * p.kv_heads + kvh) * p.tokens + c % p.tokens;
      } else {
        return (size_t)b * p.heads + (size_t)(g0 + gi) * p.kv_heads + kvh;
      }
    };
    auto orow = [&](int gi) -> size_t {  // the same row, as the single-token epilogue has always computed it
      if constexpr (MULTI) {
        return prow(gi);
      } else {
        const int head = (g0 + gi) * p.kv_heads + kvh;
        return (size_t)b * p.heads + head;
      }
    };
    // multi-token: tiles inside [lo_in, hi_in) are visible to every token of the call and skip the per-column masks
    int lo_in = 0, hi_in = 0;
    if constexpr (MULTI) {
      lo_in = td_col_range(p, b, p.tokens - 1, lo, k1).lo;
      hi_in = td_col_range(p, b, 0, lo, k1).hi;
      if (tid < NH) {
        const TdColRange cr = td_col_range(p, b, (g0 + tid) % p.tokens, lo, k1);
        sm.clo[tid] = tid < g ? cr.lo : 0;
        sm.chi[tid] = tid < g ? cr.hi : 0;
      }
    }
    const float* ksb = p.k_scale ? p.k_scale + (size_t)bhk * p.n_scale_blocks : nullptr;
    const float* vsb = p.v_scale ? p.v_scale + (size_t)bhk * p.n_scale_blocks : nullptr;

    // paged: the (page, slot) of each box of the next tile to issue.  Thread 0 reads them one tile ahead of the issue,
    // so the table load is in flight during a tile of compute instead of in front of the TMA.
    const int box_keys = PAGED ? min(p.page_size, TC_TILE) : TC_TILE;
    const int nbox = TC_TILE / box_keys;
    int pg[4], sl[4];
    auto lookup = [&](int i) {
      const int* tbl = p.block_table + (size_t)b * p.max_pages;
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        if (x < nbox) {
          const int key = min(max(k0 + i * TC_TILE + x * box_keys, lo), k1 - 1);
          pg[x] = __ldg(tbl + key / p.page_size);
          sl[x] = (key % p.page_size) & ~(box_keys - 1);
        }
      }
    };
    auto issue = [&](int i) {  // tile i of this unit into stage (n_tile + i) % TC_NST
      const uint32_t st = (n_tile + i) % TC_NST;
      const int key0 = k0 + i * TC_TILE;
      mbar_expect_tx(&sm.full[st], TX);
      if constexpr (PAGED) {
#pragma unroll
        for (int s = 0; s < (KV8 ? 1 : 2); ++s) {
#pragma unroll
          for (int x = 0; x < 4; ++x) {
            if (x < nbox) {  // each box lands 1 KB aligned: the sub-tile's 128B swizzle pattern is unchanged
              const int off = s * TC_SUB + x * box_keys * 128;
              tma_load_4d(sm.k[st] + off, &map_k, &sm.full[st], s * 64, sl[x], kvh, pg[x]);
              tma_load_4d(sm.v[st] + off, &map_v, &sm.full[st], s * 64, sl[x], kvh, pg[x]);
            }
          }
        }
      } else if constexpr (KV8) {
        tma_load_3d(sm.k[st], &map_k, &sm.full[st], 0, key0, bhk);
        tma_load_3d(sm.v[st], &map_v, &sm.full[st], 0, key0, bhk);
      } else {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          tma_load_3d(sm.k[st] + s * TC_SUB, &map_k, &sm.full[st], s * 64, key0, bhk);
          tma_load_3d(sm.v[st] + s * TC_SUB, &map_v, &sm.full[st], s * 64, key0, bhk);
        }
      }
    };
    if (tid == 0) {
      for (int i = 0; i < min(TC_NST, ntiles); ++i) {
        if constexpr (PAGED) lookup(i);
        issue(i);
      }
      if constexpr (PAGED) {
        if (TC_NST < ntiles) lookup(TC_NST);
      }
    }

    // Q^T as the B operand (16 bit, zero for padded heads); the softmax scale is applied to the logits
    for (int i = tid; i < ((!RANGED || ntiles > 0) ? NH * D / 2 : 0); i += TC_THREADS) {
      const int gi = i / (D / 2), c = 2 * (i % (D / 2));
      float a = 0.f, bq = 0.f;
      if (gi < g) {
        const size_t qi = prow(gi) * D + c;
        a = load_q(p.q, p.q_kind, qi);
        bq = load_q(p.q, p.q_kind, qi + 1);
      }
      *reinterpret_cast<uint32_t*>(sm.q[c / 64] + sw128_off(gi, c % 64)) = pack2<F16>(a, bq);
    }
    fence_proxy_async_shared();
    __syncthreads();

    float o[2][NH / 2];
    float mr[2 * NJ], lp[2 * NJ];  // running max / partial sum of this thread's head columns 8 j + cq + e
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NH / 2; ++i) o[h][i] = 0.f;
#pragma unroll
    for (int c = 0; c < 2 * NJ; ++c) {
      mr[c] = -INFINITY;
      lp[c] = 0.f;
    }
    const float clamp_inv = RANGED && p.softclamp_log2 > 0.f ? 1.f / p.softclamp_log2 : 0.f;
    const uint64_t q_desc = gmma_desc(kmaj, sm.q[0]);
    const uint64_t p_desc = gmma_desc(kmaj, sm.p);

    for (int t = 0; t < ntiles; ++t) {
      const uint32_t st = (n_tile + t) % TC_NST, ph = ((n_tile + t) / TC_NST) & 1;
      const int t0 = k0 + t * TC_TILE;
      mbar_wait(&sm.full[st], ph, 1600);
      const uint8_t* kt = sm.k[st];
      const uint8_t* vt = sm.v[st];
      if constexpr (KV8) {
        widen_fp8_tile(sm.k[st], sm.kc, tid);
        widen_fp8_tile(sm.v[st], sm.vc, tid);
        fence_proxy_async_shared();
        named_bar_sync(1, TC_THREADS);
        kt = sm.kc;
        vt = sm.vc;
      }
      if constexpr (RANGED) {
        if (t0 < lo || t0 + TC_TILE > k1) {  // boundary tile: zero the V rows of the keys outside [lo, k1)
          uint8_t* vz = KV8 ? sm.vc : sm.v[st];
          for (int i = tid; i < TC_TILE * 16; i += TC_THREADS) {
            const int row = i / 16, c = i % 16, key = t0 + row;
            if (key < lo || key >= k1)
              *reinterpret_cast<uint4*>(vz + (c / 8) * TC_SUB + row * 128 + (c % 8) * 16) = make_uint4(0u, 0u, 0u, 0u);
          }
          fence_proxy_async_shared();  // ordered before the P V wgmma by the barrier after P is written
        }
      }
      // ---- S^T = K Q^T --------------------------------------------------------------------------------------------
      float s[NH / 2];
      const uint64_t k_desc = gmma_desc(kmaj, kt);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk)
        wgmma_ss<!F16, NH, 0, 0>(s, gmma_desc_add(k_desc, (kk / 4) * TC_SUB + (kk % 4) * 32),
                                 gmma_desc_add(q_desc, (kk / 4) * (NH * 128) + (kk % 4) * 32), kk > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);

      // ---- online softmax over the keys (rows), per head (column) ---------------------------------------------------
      const float ks = (ksb ? ksb[t0 / p.scale_block] : 1.f) * p.scale_log2;
      const float vs = vsb ? vsb[t0 / p.scale_block] : 1.f;
      float cmax[2 * NJ];
#pragma unroll
      for (int c = 0; c < 2 * NJ; ++c) cmax[c] = -INFINITY;
      const bool edge = MULTI && (t0 < lo_in || t0 + TC_TILE > hi_in);
#pragma unroll
      for (int i = 0; i < NH / 2; ++i) {
        const int key = t0 + r_lo + 8 * ((i >> 1) & 1);
        if constexpr (MULTI) {
          float x = s[i] * ks;
          if (p.softclamp_log2 > 0.f) x = fast_tanh(x * clamp_inv) * p.softclamp_log2;
          const int col = 8 * (i / 4) + cq + (i & 1);
          s[i] = !edge || (key >= sm.clo[col] && key < sm.chi[col]) ? x : -INFINITY;
        } else if constexpr (RANGED) {
          float x = s[i] * ks;
          if (p.softclamp_log2 > 0.f) x = fast_tanh(x * clamp_inv) * p.softclamp_log2;
          s[i] = (key >= lo && key < k1) ? x : -INFINITY;  // a select: a NaN logit of a masked key goes too
        } else {
          s[i] = key < k1 ? s[i] * ks : -INFINITY;
        }
        const int c = 2 * (i / 4) + (i & 1);
        cmax[c] = fmaxf(cmax[c], s[i]);
      }
#pragma unroll
      for (int c = 0; c < 2 * NJ; ++c) {
#pragma unroll
        for (int off = 4; off < 32; off <<= 1) cmax[c] = fmaxf(cmax[c], __shfl_xor_sync(0xffffffffu, cmax[c], off));
      }
      if (lane < 4) {
#pragma unroll
        for (int c = 0; c < 2 * NJ; ++c) sm.red[warp][8 * (c / 2) + cq + (c & 1)] = cmax[c];
      }
      named_bar_sync(1, TC_THREADS);
      float corr[2 * NJ], m_eff[2 * NJ];
#pragma unroll
      for (int c = 0; c < 2 * NJ; ++c) {
        const int col = 8 * (c / 2) + cq + (c & 1);
        const float tmax = fmaxf(fmaxf(sm.red[0][col], sm.red[1][col]), fmaxf(sm.red[2][col], sm.red[3][col]));
        const float m_new = fmaxf(mr[c], tmax);
        m_eff[c] = m_new == -INFINITY ? 0.f : m_new;
        corr[c] = mr[c] == -INFINITY ? 0.f : fast_exp2(mr[c] - m_eff[c]);
        mr[c] = m_new;
        lp[c] *= corr[c];
      }
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < NH / 2; ++i) o[h][i] *= corr[2 * (i / 4) + (i & 1)];
      // P (times the V block scale; the denominator uses the unscaled p) as the K-major B operand [head][key]
#pragma unroll
      for (int i = 0; i < NH / 2; i += 2) {
        const int c = 2 * (i / 4);
        const float p0 = fast_exp2(s[i] - m_eff[c]), p1 = fast_exp2(s[i + 1] - m_eff[c + 1]);
        lp[c] += p0;
        lp[c + 1] += p1;
        const int key = r_lo + 8 * ((i >> 1) & 1);
        const int col = 8 * (i / 4) + cq;
        const uint32_t w = pack2<F16>(p0 * vs, p1 * vs);
        *reinterpret_cast<uint16_t*>(sm.p + sw128_off(col, key)) = (uint16_t)(w & 0xffffu);
        *reinterpret_cast<uint16_t*>(sm.p + sw128_off(col + 1, key)) = (uint16_t)(w >> 16);
      }
      fence_proxy_async_shared();
      named_bar_sync(1, TC_THREADS);

      // ---- O^T += V^T P, one 64-row half of d at a time ---------------------------------------------------------------
      wgmma_fence();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint64_t v_desc = gmma_desc(mnmaj, vt + h * TC_SUB);
#pragma unroll
        for (int kk = 0; kk < TC_TILE / 16; ++kk)
          wgmma_ss<!F16, NH, 1, 0>(o[h], gmma_desc_add(v_desc, kk * 2048), gmma_desc_add(p_desc, kk * 32), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(o[0]);
      fence_regs(o[1]);
      named_bar_sync(1, TC_THREADS);  // every warp is done with stage st, the widened tiles and P
      if (tid == 0 && t + TC_NST < ntiles) {
        issue(t + TC_NST);
        if constexpr (PAGED) {
          if (t + TC_NST + 1 < ntiles) lookup(t + TC_NST + 1);
        }
      }
    }
    n_tile += ntiles;

    // ---- per-head totals, O^T -> shared memory ------------------------------------------------------------------------
#pragma unroll
    for (int c = 0; c < 2 * NJ; ++c) {
#pragma unroll
      for (int off = 4; off < 32; off <<= 1) lp[c] += __shfl_xor_sync(0xffffffffu, lp[c], off);
    }
    if (lane < 4) {
#pragma unroll
      for (int c = 0; c < 2 * NJ; ++c) sm.red[warp][8 * (c / 2) + cq + (c & 1)] = lp[c];
    }
    if (warp == 0 && lane < 4) {
#pragma unroll
      for (int c = 0; c < 2 * NJ; ++c) sm.ml[0][8 * (c / 2) + cq + (c & 1)] = mr[c];
    }
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NH / 2; ++i)
        sm.o[8 * (i / 4) + cq + (i & 1)][64 * h + r_lo + 8 * ((i >> 1) & 1)] = o[h][i];
    __syncthreads();
    if (tid < NH) sm.ml[1][tid] = sm.red[0][tid] + sm.red[1][tid] + sm.red[2][tid] + sm.red[3][tid];
    __syncthreads();

    if (p.splits == 1) {
      // the unit IS the group: normalise and publish (out, lse2, valid) for its g heads directly
      for (int i = tid; i < g * D; i += TC_THREADS) {
        const int gi = i / D, c = i % D;
        const float l = sm.ml[1][gi];
        my_partial[orow(gi) * row_stride + c] = l > 0.f ? sm.o[gi][c] / l : 0.f;
      }
      if (tid < g) {
        const float l = sm.ml[1][tid], m = sm.ml[0][tid];
        float* row = my_partial + orow(tid) * row_stride;
        row[D] = l > 0.f ? (m == -INFINITY ? 0.f : m) + log2f(l) : -INFINITY;
        row[D + 1] = l > 0.f ? 1.f : 0.f;
      }
    } else {
      float* out = p.scratch + (((size_t)bhk * p.splits + split) * g_total + g0) * row_stride;
      for (int i = tid; i < g * D; i += TC_THREADS) out[(i / D) * row_stride + i % D] = sm.o[i / D][i % D];
      if (tid < g) {
        out[tid * row_stride + D] = sm.ml[0][tid];
        out[tid * row_stride + D + 1] = sm.ml[1][tid];
      }
      // the CTA that completes the last split of the group merges the splits
      __threadfence();
      __syncthreads();
      if (tid == 0) {
        const uint32_t done = atomicAdd(&p.group_done[grp], 1u);
        sm.last = (done == (uint32_t)p.splits - 1) ? 1u : 0u;
        if (sm.last) p.group_done[grp] = 0;  // self-resetting
      }
      __syncthreads();
      if (sm.last) {
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
          float* row = my_partial + orow(gi) * row_stride;
          for (int c = tid; c < D; c += TC_THREADS) {
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

template <int KVK, int NH, bool RANGED, bool MULTI = false>
__global__ void __launch_bounds__(TC_THREADS, 1)
tree_decode_tc_kernel(const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                      const __grid_constant__ TreeDecodeParams p) {
  tc_decode_body<KVK, NH, RANGED, MULTI, false>(map_k, map_v, p);
}

// paged K / V (TreeDecodeParams::block_table): always the ranged body
template <int KVK, int NH, bool MULTI>
__global__ void __launch_bounds__(TC_THREADS, 1)
tree_decode_tc_paged_kernel(const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                            const __grid_constant__ TreeDecodeParams p) {
  tc_decode_body<KVK, NH, true, MULTI, true>(map_k, map_v, p);
}

template <int KVK, bool RANGED>
const void* tc_ptr_nh(bool small_group) {
  return small_group ? (const void*)tree_decode_tc_kernel<KVK, 8, RANGED>
                     : (const void*)tree_decode_tc_kernel<KVK, 16, RANGED>;
}
// multi-token calls: NH = 8, 16 or 32 columns per unit for g * tokens <= 8, <= 16, larger
int tc_multi_nh(int cols) { return cols <= 8 ? 8 : (cols <= 16 ? 16 : 32); }
template <int KVK>
const void* tc_ptr_multi(int nh) {
  if (nh == 8) return (const void*)tree_decode_tc_kernel<KVK, 8, true, true>;
  if (nh == 16) return (const void*)tree_decode_tc_kernel<KVK, 16, true, true>;
  return (const void*)tree_decode_tc_kernel<KVK, 32, true, true>;
}
const void* pick_tc_multi(int kv_kind, int nh) {
  if (kv_kind == 2) return tc_ptr_multi<2>(nh);
  return kv_kind == 1 ? tc_ptr_multi<1>(nh) : tc_ptr_multi<0>(nh);
}
template <bool KV8>
size_t tc_smem_multi(int nh) {
  if (nh == 8) return sizeof(TcSmemMulti<KV8, 8>) + 1024;
  if (nh == 16) return sizeof(TcSmemMulti<KV8, 16>) + 1024;
  return sizeof(TcSmemMulti<KV8, 32>) + 1024;
}
template <bool RANGED>
const void* pick_tc_r(int kv_kind, bool small_group) {
  if (kv_kind == 2) return tc_ptr_nh<2, RANGED>(small_group);
  return kv_kind == 1 ? tc_ptr_nh<1, RANGED>(small_group) : tc_ptr_nh<0, RANGED>(small_group);
}
const void* pick_tc(int kv_kind, bool small_group, bool ranged) {
  return ranged ? pick_tc_r<true>(kv_kind, small_group) : pick_tc_r<false>(kv_kind, small_group);
}
// paged calls: NH = 8 or 16 single-token (small_group), 8, 16 or 32 multi-token (tc_multi_nh)
template <int KVK>
const void* tc_ptr_paged(bool multi, int nh) {
  if (multi) {
    if (nh == 8) return (const void*)tree_decode_tc_paged_kernel<KVK, 8, true>;
    if (nh == 16) return (const void*)tree_decode_tc_paged_kernel<KVK, 16, true>;
    return (const void*)tree_decode_tc_paged_kernel<KVK, 32, true>;
  }
  return nh == 8 ? (const void*)tree_decode_tc_paged_kernel<KVK, 8, false>
                 : (const void*)tree_decode_tc_paged_kernel<KVK, 16, false>;
}
const void* pick_tc_paged(int kv_kind, bool multi, int nh) {
  if (kv_kind == 2) return tc_ptr_paged<2>(multi, nh);
  return kv_kind == 1 ? tc_ptr_paged<1>(multi, nh) : tc_ptr_paged<0>(multi, nh);
}
size_t tc_smem(int kv_kind, bool small_group) {
  size_t s;
  if (kv_kind == 2) s = small_group ? sizeof(TcSmem<true, 8>) : sizeof(TcSmem<true, 16>);
  else s = small_group ? sizeof(TcSmem<false, 8>) : sizeof(TcSmem<false, 16>);
  return s + 1024;
}

}  // namespace

int tree_decode_tc_max_ctas(int kv_kind, int num_sms, bool ranged, int cols, bool paged) {
  const bool small = false;  // the 16-head variant: the larger shared-memory footprint bounds residency
  // a multi-token or paged call plans with the residency of the variant it launches
  const int nh = tc_multi_nh(cols);
  const void* fn = paged ? pick_tc_paged(kv_kind, cols > 0, cols > 0 ? nh : 16)
                         : (cols > 0 ? pick_tc_multi(kv_kind, nh) : pick_tc(kv_kind, small, ranged));
  const size_t smem = cols > 0 ? (kv_kind == 2 ? tc_smem_multi<true>(nh) : tc_smem_multi<false>(nh))
                               : tc_smem(kv_kind, small);
  cuda_check(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "tree_decode_tc smem attr");
  int per_sm = 0;
  cuda_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, TC_THREADS, smem), "tree_decode_tc occupancy");
  return per_sm * num_sms;
}

void launch_tree_decode_tc(const CUtensorMap& map_k, const CUtensorMap& map_v, const TreeDecodeParams& p, int grid,
                           cudaStream_t stream, bool ranged) {
  const bool small = p.heads / p.kv_heads <= 8;
  const bool multi = p.tokens > 1;
  const int nh = tc_multi_nh(p.heads / p.kv_heads * p.tokens);
  const void* fn = p.block_table != nullptr ? pick_tc_paged(p.kv_kind, multi, multi ? nh : (small ? 8 : 16))
                   : (multi ? pick_tc_multi(p.kv_kind, nh) : pick_tc(p.kv_kind, small, ranged));
  const size_t smem = multi ? (p.kv_kind == 2 ? tc_smem_multi<true>(nh) : tc_smem_multi<false>(nh))
                            : tc_smem(p.kv_kind, small);
  cuda_check(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "tree_decode_tc smem attr");
  void* args[] = {(void*)&map_k, (void*)&map_v, (void*)&p};
  // cooperative: the grid barrier and the cross-rank waits need every CTA of the grid to be resident
  cuda_check(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(TC_THREADS), args, smem, stream), "tree_decode_tc launch");
}

}  // namespace rab
