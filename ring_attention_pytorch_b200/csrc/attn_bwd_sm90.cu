// Ring flash-attention backward for sm_90a (wgmma + TMA + mbarrier): two warp-specialised kernels.
//
//   attn_bwd_dq_kernel   (Q-stationary)  per 128-row query tile (64 rows per consumer warpgroup), for every visible
//        K/V tile, in two 64-key halves:  S = Q K^T, dP = dO V^T (shared-memory operands, registers out)
//        dS = P o (dP - delta)  ->  dQ += dS K (dS straight from registers, K read MN-major)
//   attn_bwd_dkv_kernel  (KV-stationary) per 128-key tile (64 keys per consumer warpgroup), for every query tile
//        (64 rows) that can see it:  S^T = K Q^T, dP^T = V dO^T  ->  P^T, dS^T in registers
//        dV += P^T dO, dK += dS^T Q (Q / dO read MN-major).
//        ONE_PASS (the ring backward of attn_bwd_ring): both warpgroups write their dS^T half into one shared
//        [128 keys][64 queries] tile; dK += dS^T Q reads it from there, and warpgroup w computes
//        dQ[64 q][64 w .. 64 w + 63] = dS K over all 128 keys, staged in shared memory and added into the fp32 dQ
//        accumulator with TMA tensor reductions.
//        dK / dV then go out either as 16 bit (single rank) or added into the K/V owner's fp32 accumulators (ring).
//
// Roles (384 threads, 1 CTA / SM, persistent): warps 0-3 / 4-7 consumer warpgroups (issue their own wgmma), warp 8
// TMA producer (it also walks the tile schedule and hands each streamed tile to the consumers), warps 9-11 idle.
// The softmax scale is folded into the dQ / dK epilogues.
//
// Inputs of the two-kernel pass are the *gathered* ring buffers (see kernels.h); remote slots are published through
// ready flags.
#include <cuda_fp16.h>

// no printf in the watchdogs: a function call would serialize the wgmma of these kernels (see ptx.cuh)
#define RAB_WATCHDOG_PRINTF 0
#include "attn_common.cuh"

namespace rab {
namespace {

constexpr int NTHREADS = 384;
constexpr int SUB128 = 128 * 128;  // 64-element-wide sub-tile, 128 rows
constexpr int SUB64 = 64 * 128;    // 64-element-wide sub-tile, 64 rows
constexpr uint64_t KMAJ = gmma_desc_static(16, 1024);

template <class P>
__device__ __forceinline__ void wait_owner_ready(const P& p, int owner, uint32_t& mask, int tag) {
  if ((mask >> owner) & 1u) return;
  if (p.ready != nullptr) {
    spin_until_ge_gpu(p.ready + owner, p.ready_target, tag);
    fence_proxy_async_global();
  }
  mask |= 1u << owner;
}

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

template <bool BF16>
__device__ __forceinline__ uint32_t pack16(float a, float b) {
  return BF16 ? pack_bf16x2(a, b) : pack_f16x2(a, b);
}

// =================================================================================================
// dQ kernel
// =================================================================================================
constexpr int DQ_NST = 2;

template <int D>
struct DqSmem {
  static constexpr int NSUB = D / 64;
  static constexpr int TILE = NSUB * SUB128;
  alignas(1024) uint8_t q[TILE];
  alignas(1024) uint8_t dout[TILE];
  alignas(1024) uint8_t k[DQ_NST][TILE];
  alignas(1024) uint8_t v[DQ_NST][TILE];
  uint64_t qdo_full, qdo_empty;
  uint64_t kv_full[DQ_NST], kv_empty[DQ_NST];
};

struct DqItem {
  int b, h, kvh, qt, row0;
  int qlo, qhi;
};

__device__ __forceinline__ int dq_num_items(const AttnBwdParams& p) {
  return p.batch * p.heads * ((p.n_q + 127) / 128);
}

__device__ __forceinline__ void dq_decode(const AttnBwdParams& p, int idx, DqItem& it) {
  const int bh = p.batch * p.heads;
  const int nqt = (p.n_q + 127) / 128;
  it.qt = nqt - 1 - idx / bh;
  const int r = idx % bh;
  it.b = r / p.heads;
  const int hh = r % p.heads;
  const int groups = p.heads / p.kv_heads;
  it.kvh = hh / groups;
  it.h = (hh % groups) * p.kv_heads + it.kvh;
  it.row0 = it.qt * 128;
  pos_range(p.pos, p.rank, it.row0, min(it.row0 + 128, p.n_q) - 1, it.qlo, it.qhi);
  it.qlo += p.q_pos_offset;
  it.qhi += p.q_pos_offset;
}

template <bool DOCS>
using DqScan = WarpTileScan<2, false, DOCS>;

template <bool DOCS>
__device__ __forceinline__ void dq_init_scan(DqScan<DOCS>& sc, const AttnBwdParams& p, const DqItem& it) {
  sc.pm = &p.pos;
  sc.hop_owner = p.hop_owner;
  sc.hop_count = p.hop_count;
  sc.groups = 1;
  sc.n_stream = p.n_k;
  sc.tile = 128;
  sc.stream_off = 0;
  sc.stat_off = 0;
  sc.mc = MaskCfg{p.causal, p.window, p.kmask_bits != nullptr};
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const int a = it.row0 + 64 * t;
    const bool valid = a < p.n_q;
    int lo = 0, hi = 0;
    if (valid) {
      pos_range(p.pos, p.rank, a, min(a + 64, p.n_q) - 1, lo, hi);
      lo += p.q_pos_offset;
      hi += p.q_pos_offset;
    }
    sc.st[t] = StatRange{lo, hi, valid, false};
    if constexpr (DOCS) {
      if (valid)
        sc.doc[t] = doc_range(doc_row_spans(p.doc_spans, p.batch, p.n_q, p.rank, it.b), a, min(a + 64, p.n_q) - 1,
                                 lane_id());
    }
  }
}

template <int D, bool DOCS>
__device__ __forceinline__ void dq_producer(DqSmem<D>& sm, const AttnBwdParams& p, const CUtensorMap* map_qd,
                                            const CUtensorMap* map_kv) {
  constexpr int NSUB = DqSmem<D>::NSUB;
  constexpr uint32_t TILE = DqSmem<D>::TILE;
  const int lane = lane_id();
  uint32_t n_item = 0, n_tile = 0;
  uint32_t ready_mask = 1u << p.rank;
  const int total = dq_num_items(p);
  for (int idx = blockIdx.x; idx < total; idx += gridDim.x, ++n_item) {
    DqItem it;
    dq_decode(p, idx, it);
    if (lane == 0) {
      mbar_wait(&sm.qdo_empty, (n_item & 1) ^ 1, 500);
      mbar_expect_tx(&sm.qdo_full, 2 * TILE);
#pragma unroll
      for (int s = 0; s < NSUB; ++s) {
        tma_load_4d(sm.q + s * SUB128, map_qd, &sm.qdo_full, s * 64, it.row0, it.b * p.heads + it.h, p.rank * 2);
        tma_load_4d(sm.dout + s * SUB128, map_qd, &sm.qdo_full, s * 64, it.row0, it.b * p.heads + it.h,
                    p.rank * 2 + 1);
      }
    }
    DqScan<DOCS> scan;
    dq_init_scan<DOCS>(scan, p, it);
    ScanTile t;
    while (scan.next(lane, t)) {
      if (lane == 0) {
        wait_owner_ready(p, t.owner, ready_mask, 501);
        const uint32_t st = n_tile % DQ_NST, ph = (n_tile / DQ_NST) & 1;
        mbar_wait(&sm.kv_empty[st], ph ^ 1, 510 + st);
        mbar_expect_tx(&sm.kv_full[st], 2 * TILE);
#pragma unroll
        for (int s = 0; s < NSUB; ++s) {
          tma_load_4d(sm.k[st] + s * SUB128, map_kv, &sm.kv_full[st], s * 64, t.idx * 128,
                      it.b * p.kv_heads + it.kvh, t.owner * 2);
          tma_load_4d(sm.v[st] + s * SUB128, map_kv, &sm.kv_full[st], s * 64, t.idx * 128,
                      it.b * p.kv_heads + it.kvh, t.owner * 2 + 1);
        }
      }
      n_tile++;
      __syncwarp();
    }
  }
}

// Thread layout as in the forward: rows r_lo and r_lo + 8 of the warpgroup's 64 query rows, column pairs 8 j + cq.
template <int D, bool BF16, bool DOCS>
__device__ __forceinline__ void dq_consumer(DqSmem<D>& sm, const AttnBwdParams& p, const int W) {
  constexpr uint64_t mnmaj = gmma_desc_static(SUB128, 1024);  // K as the MN-major B of dQ += dS K
  const int wg_tid = threadIdx.x - 128 * W;
  const int lane = lane_id();
  const int r_lo = (wg_tid / 32) * 16 + lane / 4;
  const int cq = 2 * (lane % 4);
  uint32_t n_item = 0, n_tile = 0;

  const bool clamp = p.softclamp > 0.f;
  const float mul = clamp ? 1.f : p.scale * kLog2e;
  const float pre = clamp ? p.scale / p.softclamp : 0.f;
  const float post = clamp ? p.softclamp * kLog2e : 0.f;

  const int total = dq_num_items(p);
  for (int idx = blockIdx.x; idx < total; idx += gridDim.x, ++n_item) {
    DqItem it;
    dq_decode(p, idx, it);
    int grow[2], pos_q[2];
    bool row_ok[2];
    float lse2[2], delta[2];
    const size_t stat_row = ((size_t)(p.rank * 2) * p.batch * p.heads + (size_t)it.b * p.heads + it.h) * p.n_pad;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      grow[h] = it.row0 + 64 * W + r_lo + 8 * h;
      row_ok[h] = grow[h] < p.n_q;
      pos_q[h] = pos_of(p.pos, p.rank, min(grow[h], p.n_q - 1)) + p.q_pos_offset;
      lse2[h] = row_ok[h] ? p.stat[stat_row + grow[h]] : INFINITY;
      delta[h] = row_ok[h] ? p.stat[stat_row + (size_t)p.batch * p.heads * p.n_pad + grow[h]] : 0.f;
    }
    int2 span[2];  // document interval of each of this thread's query rows
    if constexpr (DOCS) {
      const int2* rows = doc_row_spans(p.doc_spans, p.batch, p.n_q, p.rank, it.b);
#pragma unroll
      for (int h = 0; h < 2; ++h) span[h] = rows[min(grow[h], p.n_q - 1)];
    }

    mbar_wait(&sm.qdo_full, n_item & 1, 600 + W);
    const uint64_t q_desc = gmma_desc(KMAJ, sm.q + W * SUB64);
    const uint64_t do_desc = gmma_desc(KMAJ, sm.dout + W * SUB64);

    float dq[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) dq[i] = 0.f;

    DqScan<DOCS> scan;
    dq_init_scan<DOCS>(scan, p, it);
    ScanTile t;
    while (scan.next(lane, t)) {
      const uint32_t st = n_tile % DQ_NST, ph = (n_tile / DQ_NST) & 1;
      n_tile++;
      const bool need = W ? t.need[1] : t.need[0];
      const bool part = W ? t.part[1] : t.part[0];
      mbar_wait(&sm.kv_full[st], ph, 610 + W);
      if (need) {
        const int c0 = t.idx * 128;
        const int split = p.pos.seg_len - c0;
        const int a0 = p.pos.base0[t.owner] + p.pos.stride * c0;
        const int a1 = p.pos.base1[t.owner] + p.pos.stride * (c0 - p.pos.seg_len);
        const int ncols = p.n_k - c0;
        uint32_t mb[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
        if (part && p.kmask_bits != nullptr) {
          const uint32_t* w = p.kmask_bits + ((size_t)t.owner * p.batch + it.b) * p.kmask_words + (size_t)t.idx * 4;
#pragma unroll
          for (int i = 0; i < 4; ++i) mb[i] = w[i];
        }
#pragma unroll 1
        for (int half = 0; half < 2; ++half) {
          const uint64_t k_desc = gmma_desc(KMAJ, sm.k[st] + half * SUB64);
          const uint64_t v_desc = gmma_desc(KMAJ, sm.v[st] + half * SUB64);
          float s[32], dp[32];
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < D / 16; ++kk) {
            const uint32_t off_a = (kk / 4) * SUB128 + (kk % 4) * 32;
            const uint32_t off_b = (kk / 4) * SUB128 + (kk % 4) * 32;
            wgmma_ss<BF16, 64, 0, 0>(s, gmma_desc_add(q_desc, off_a), gmma_desc_add(k_desc, off_b), kk > 0 ? 1u : 0u);
          }
#pragma unroll
          for (int kk = 0; kk < D / 16; ++kk) {
            const uint32_t off = (kk / 4) * SUB128 + (kk % 4) * 32;
            wgmma_ss<BF16, 64, 0, 0>(dp, gmma_desc_add(do_desc, off), gmma_desc_add(v_desc, off), kk > 0 ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs(s);
          fence_regs(dp);
          uint32_t da[16];
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            float ds2[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int h = (i >> 1) & 1;
              const int col = half * 64 + 8 * (i / 4) + cq + e;
              const float sv = s[i + e];
              float pj, chain = 1.f;
              if (clamp) {
                const float th = fast_tanh(sv * pre);
                pj = fast_exp2(fmaf(th, post, -lse2[h]));
                chain = 1.f - th * th;
              } else {
                pj = fast_exp2(fmaf(sv, mul, -lse2[h]));
              }
              if (part) {
                const int pk = (col < split ? a0 : a1) + p.pos.stride * col;
                bool keep = (col < ncols) && ((mb[half * 2 + (i / 16)] >> (col & 31)) & 1u);  // col / 32
                if (p.causal) {
                  keep = keep && (pk <= pos_q[h]);
                  if (p.window > 0) keep = keep && (pos_q[h] - pk <= p.window);
                }
                if constexpr (DOCS) keep = keep && (span[h].x <= pk) && (pk < span[h].y);
                if (!keep) pj = 0.f;
              }
              ds2[e] = pj * (dp[i + e] - delta[h]) * chain;
            }
            da[i / 2] = pack16<BF16>(ds2[0], ds2[1]);
          }
          const uint64_t kb_desc = gmma_desc(mnmaj, sm.k[st] + half * SUB64);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const uint32_t a4[4] = {da[4 * kk], da[4 * kk + 1], da[4 * kk + 2], da[4 * kk + 3]};
            wgmma_rs<BF16, D, 1>(dq, a4, gmma_desc_add(kb_desc, kk * 2048), 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs(dq);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.kv_empty[st]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.qdo_empty);

#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!row_ok[h]) continue;
      uint16_t* drow = reinterpret_cast<uint16_t*>(p.dq) + (((size_t)it.b * p.n_q + grow[h]) * p.heads + it.h) * D;
#pragma unroll
      for (int j = 0; j < D / 8; ++j)
        *reinterpret_cast<uint32_t*>(drow + 8 * j + cq) =
            pack16<BF16>(dq[4 * j + 2 * h] * p.scale, dq[4 * j + 2 * h + 1] * p.scale);
    }
  }
}

template <int D, bool BF16, bool DOCS>
__global__ void __launch_bounds__(NTHREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap map_qd, const __grid_constant__ CUtensorMap map_kv,
                   const __grid_constant__ AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  DqSmem<D>& sm = *reinterpret_cast<DqSmem<D>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x / 32;
  if (threadIdx.x == 0) {
    mbar_init(&sm.qdo_full, 1);
    mbar_init(&sm.qdo_empty, 8);
    for (int i = 0; i < DQ_NST; ++i) {
      mbar_init(&sm.kv_full[i], 1);
      mbar_init(&sm.kv_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (warp == 8) dq_producer<D, DOCS>(sm, p, &map_qd, &map_kv);
  } else {
    setmaxnreg_inc<232>();
    dq_consumer<D, BF16, DOCS>(sm, p, warp < 4 ? 0 : 1);
  }
}

// =================================================================================================
// KV-stationary kernel (dK / dV, and dQ in the one-pass ring backward)
// =================================================================================================
constexpr int QST = 3;

// What the producer hands the consumers with each Q / dO stage (written before its arrive on qd_full).
struct DkvTileRec {
  int idx;    // query tile index; -1 marks the end of the item (the stage then carries no data)
  int rep;    // query head inside the GQA group
  int owner;  // ring rank of the queries
  int part;   // the tile pair needs per-element masking
};

template <int D>
struct DkvSmem {
  static constexpr int NSUB = D / 64;
  static constexpr int KV_TILE = NSUB * SUB128;  // 128 keys
  static constexpr int Q_TILE = NSUB * SUB64;    // 64 queries
  alignas(1024) uint8_t k[KV_TILE];
  alignas(1024) uint8_t v[KV_TILE];
  alignas(1024) uint8_t q[QST][Q_TILE];
  alignas(1024) uint8_t dout[QST][Q_TILE];
  // one-pass mode: dS^T [128 keys][64 queries] (warpgroup w writes keys 64 w ..), double buffered so that a
  // warpgroup can write the next tile's half while the other one's dQ wgmma still reads this one
  alignas(1024) uint8_t ds[2][SUB128];
  // one-pass mode: dQ [64 q][64 d] of warpgroup w as two [64 q][32 d] boxes (128B swizzle), source of the tensor reduce
  alignas(1024) float dq_stage[2][64 * 64];
  alignas(16) float lse2[QST][64];
  alignas(16) float delta[QST][64];
  DkvTileRec rec[QST];
  uint64_t kv_full, kv_empty;
  uint64_t qd_full[QST], qd_empty[QST];
};
static_assert(sizeof(DkvSmem<128>) + 1024 <= 227 * 1024, "DkvSmem exceeds the opt-in shared memory of an SM");

struct DkvItem {
  int owner, b, kvh, key0;  // owner: ring rank whose keys the item holds
  int klo, khi;
  bool k_tail;
};

template <bool ONE_PASS, class P>
__device__ __forceinline__ int dkv_num_items(const P& p) {
  return (ONE_PASS ? p.hop_count : 1) * p.batch * p.kv_heads * ((p.n_k + 127) / 128);
}

// Two-kernel pass: this rank's key tiles, heaviest (earliest) first.  One-pass ring backward: hop-major (the K/V of
// later hops arrive later), then (batch, kv head), then key tile; waves of gridDim items alternate direction so that
// the static round-robin assignment balances the triangular work.
template <bool ONE_PASS, class P>
__device__ __forceinline__ void dkv_decode(const P& p, int L, DkvItem& it) {
  const int nkt = (p.n_k + 127) / 128;
  const int bhk = p.batch * p.kv_heads;
  int kt, bkv;
  if constexpr (ONE_PASS) {
    const int G = gridDim.x;
    const int total = dkv_num_items<true>(p);
    const int wave = L / G, ln = L % G;
    int Lp = L;
    if ((wave & 1) && (wave + 1) * G <= total) Lp = wave * G + (G - 1 - ln);
    kt = Lp % nkt;
    const int r = Lp / nkt;
    bkv = r % bhk;
    it.owner = p.hop_owner[r / bhk];
  } else {
    kt = L / bhk;
    bkv = L % bhk;
    it.owner = p.rank;
  }
  it.b = bkv / p.kv_heads;
  it.kvh = bkv % p.kv_heads;
  it.key0 = kt * 128;
  pos_range(p.pos, it.owner, it.key0, min(it.key0 + 128, p.n_k) - 1, it.klo, it.khi);
  it.k_tail = (it.key0 + 128) > p.n_k;
}

template <bool DOCS>
using DkvScan = WarpTileScan<1, true, DOCS>;

// streamed side = query tiles of 64 rows (one-pass: the local queries only); rep = query head inside the GQA group
template <bool ONE_PASS, bool DOCS, class P>
__device__ __forceinline__ void dkv_init_scan(DkvScan<DOCS>& sc, const P& p, const DkvItem& it) {
  sc.pm = &p.pos;
  if constexpr (ONE_PASS) {
    sc.hop_owner = p.self_owner;
    sc.hop_count = 1;
  } else {
    sc.hop_owner = p.hop_owner;
    sc.hop_count = p.hop_count;
  }
  sc.groups = p.heads / p.kv_heads;
  sc.n_stream = p.n_q;
  sc.tile = 64;
  sc.stream_off = p.q_pos_offset;
  sc.stat_off = 0;
  sc.mc = MaskCfg{p.causal, p.window, p.kmask_bits != nullptr};
  sc.st[0] = StatRange{it.klo, it.khi, true, it.k_tail};
  if constexpr (DOCS)
    sc.doc[0] = doc_range(doc_row_spans(p.doc_spans, p.batch, p.n_k, it.owner, it.b), it.key0,
                             min(it.key0 + 128, p.n_k) - 1, lane_id());
}

template <int D, bool ONE_PASS, bool DOCS, class P>
__device__ __forceinline__ void dkv_producer(DkvSmem<D>& sm, const P& p, const CUtensorMap* map_qd64,
                                             const CUtensorMap* map_kv) {
  constexpr int NSUB = DkvSmem<D>::NSUB;
  constexpr uint32_t KV_TILE = DkvSmem<D>::KV_TILE, Q_TILE = DkvSmem<D>::Q_TILE;
  const int lane = lane_id();
  uint32_t n_item = 0, n_tile = 0;
  uint32_t ready_mask = 1u << p.rank;
  const int total = dkv_num_items<ONE_PASS>(p);
  const size_t stat_half = (size_t)p.batch * p.heads * p.n_pad;
  for (int idx = blockIdx.x; idx < total; idx += gridDim.x, ++n_item) {
    DkvItem it;
    dkv_decode<ONE_PASS>(p, idx, it);
    if (lane == 0) {
      if (ONE_PASS) wait_owner_ready(p, it.owner, ready_mask, 801);
      mbar_wait(&sm.kv_empty, (n_item & 1) ^ 1, 800);
      mbar_expect_tx(&sm.kv_full, 2 * KV_TILE);
#pragma unroll
      for (int s = 0; s < NSUB; ++s) {
        tma_load_4d(sm.k + s * SUB128, map_kv, &sm.kv_full, s * 64, it.key0, it.b * p.kv_heads + it.kvh,
                    it.owner * 2);
        tma_load_4d(sm.v + s * SUB128, map_kv, &sm.kv_full, s * 64, it.key0, it.b * p.kv_heads + it.kvh,
                    it.owner * 2 + 1);
      }
    }
    DkvScan<DOCS> scan;
    dkv_init_scan<ONE_PASS, DOCS>(scan, p, it);
    ScanTile t;
    bool more = true;
    while (more) {
      more = scan.next(lane, t);
      if (lane == 0 && !more) {  // end of the item: an empty stage whose record tells the consumers to move on
        const uint32_t st = n_tile % QST, ph = (n_tile / QST) & 1;
        mbar_wait(&sm.qd_empty[st], ph ^ 1, 810 + st);
        sm.rec[st] = DkvTileRec{-1, 0, 0, 0};
        mbar_arrive(&sm.qd_full[st]);
      }
      if (lane == 0 && more) {
        if (!ONE_PASS) wait_owner_ready(p, t.owner, ready_mask, 802);
        const uint32_t st = n_tile % QST, ph = (n_tile / QST) & 1;
        const int bh = it.b * p.heads + t.rep * p.kv_heads + it.kvh;
        const int slot = ONE_PASS ? 0 : t.owner * 2;  // the one-pass kernel reads the local [2][b*h][n_q][d] Q / dO
        mbar_wait(&sm.qd_empty[st], ph ^ 1, 810 + st);
        sm.rec[st] = DkvTileRec{t.idx, t.rep, t.owner, t.part[0] ? 1 : 0};
        mbar_expect_tx(&sm.qd_full[st], 2 * Q_TILE + 2 * 64 * 4);
#pragma unroll
        for (int s = 0; s < NSUB; ++s) {
          tma_load_4d(sm.q[st] + s * SUB64, map_qd64, &sm.qd_full[st], s * 64, t.idx * 64, bh, slot);
          tma_load_4d(sm.dout[st] + s * SUB64, map_qd64, &sm.qd_full[st], s * 64, t.idx * 64, bh, slot + 1);
        }
        const size_t stat_slot = ONE_PASS ? 0 : (size_t)(t.owner * 2) * p.batch * p.heads;
        const float* srow = p.stat + (stat_slot + bh) * p.n_pad + (size_t)t.idx * 64;
        bulk_load_1d(sm.lse2[st], srow, 64 * 4, &sm.qd_full[st]);
        bulk_load_1d(sm.delta[st], srow + stat_half, 64 * 4, &sm.qd_full[st]);
      }
      n_tile++;
      __syncwarp();
    }
  }
}

// Thread layout: rows (keys) r_lo and r_lo + 8 of the warpgroup's 64 keys, query columns 8 j + cq (+1).
template <int D, bool BF16, bool ONE_PASS, bool DOCS, class P>
__device__ __forceinline__ void dkv_consumer(DkvSmem<D>& sm, const P& p, const CUtensorMap* map_dq, const int W) {
  constexpr uint64_t qmn = gmma_desc_static(SUB64, 1024);   // Q / dO as MN-major B (K = queries, N = d)
  constexpr uint64_t kmn = gmma_desc_static(SUB128, 1024);  // K as MN-major B of dQ = dS K (K = keys, N = d)
  constexpr uint64_t dsmn = gmma_desc_static(SUB64, 1024);  // dS^T [key][q] as MN-major A of dQ = dS K
  const int wg_tid = threadIdx.x - 128 * W;
  const int wg_warp = wg_tid / 32;
  const int lane = lane_id();
  const int r_lo = wg_warp * 16 + lane / 4;
  const int cq = 2 * (lane % 4);
  uint32_t n_item = 0, n_tile = 0;
  uint32_t n_ds = 0;  // tiles computed so far: selects the dS^T buffer (one-pass mode)

  const bool clamp = p.softclamp > 0.f;
  const float mul = clamp ? 1.f : p.scale * kLog2e;
  const float pre = clamp ? p.scale / p.softclamp : 0.f;
  const float post = clamp ? p.softclamp * kLog2e : 0.f;

  const int total = dkv_num_items<ONE_PASS>(p);
  for (int idx = blockIdx.x; idx < total; idx += gridDim.x, ++n_item) {
    DkvItem it;
    dkv_decode<ONE_PASS>(p, idx, it);
    int key[2], pos_k[2];
    bool key_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      key[h] = it.key0 + 64 * W + r_lo + 8 * h;
      key_ok[h] = key[h] < p.n_k;
      pos_k[h] = pos_of(p.pos, it.owner, min(key[h], p.n_k - 1));
      if (key_ok[h] && p.kmask_bits != nullptr) {
        const uint32_t wbits = p.kmask_bits[((size_t)it.owner * p.batch + it.b) * p.kmask_words + (key[h] >> 5)];
        key_ok[h] = (wbits >> (key[h] & 31)) & 1u;
      }
    }
    int2 span[2];  // document interval of each of this thread's keys
    if constexpr (DOCS) {
      const int2* rows = doc_row_spans(p.doc_spans, p.batch, p.n_k, it.owner, it.b);
#pragma unroll
      for (int h = 0; h < 2; ++h) span[h] = rows[min(key[h], p.n_k - 1)];
    }

    mbar_wait(&sm.kv_full, n_item & 1, 900 + W);
    const uint64_t k_desc = gmma_desc(KMAJ, sm.k + W * SUB64);
    const uint64_t v_desc = gmma_desc(KMAJ, sm.v + W * SUB64);

    float dk[D / 2], dv[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) dk[i] = dv[i] = 0.f;

    bool any = false;
    while (true) {
      const uint32_t st = n_tile % QST, ph = (n_tile / QST) & 1;
      n_tile++;
      mbar_wait(&sm.qd_full[st], ph, 910 + W);
      const DkvTileRec t = sm.rec[st];
      if (t.idx < 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.qd_empty[st]);
        break;
      }
      any = true;
      float s[32], dp[32];
      const uint64_t q_desc = gmma_desc(KMAJ, sm.q[st]);
      const uint64_t do_desc = gmma_desc(KMAJ, sm.dout[st]);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t off_a = (kk / 4) * SUB128 + (kk % 4) * 32, off_b = (kk / 4) * SUB64 + (kk % 4) * 32;
        wgmma_ss<BF16, 64, 0, 0>(s, gmma_desc_add(k_desc, off_a), gmma_desc_add(q_desc, off_b), kk > 0 ? 1u : 0u);
      }
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t off_a = (kk / 4) * SUB128 + (kk % 4) * 32, off_b = (kk / 4) * SUB64 + (kk % 4) * 32;
        wgmma_ss<BF16, 64, 0, 0>(dp, gmma_desc_add(v_desc, off_a), gmma_desc_add(do_desc, off_b), kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      fence_regs(dp);

      // P^T = exp2(S^T * c - lse[col]); dS^T = P^T o (dP^T - delta[col]) [* (1 - tanh^2) with softclamp]
      const int c0 = t.idx * 64;
      const int split = p.pos.seg_len - c0;
      const int a0 = p.pos.base0[t.owner] + p.pos.stride * c0 + p.q_pos_offset;
      const int a1 = p.pos.base1[t.owner] + p.pos.stride * (c0 - p.pos.seg_len) + p.q_pos_offset;
      const int ncols = p.n_q - c0;
      const bool part = t.part != 0;
      uint32_t pa[16], da[16];
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int h = (i >> 1) & 1;
        const int col0 = 8 * (i / 4) + cq;
        const float2 lv = *reinterpret_cast<const float2*>(&sm.lse2[st][col0]);
        const float2 dl = *reinterpret_cast<const float2*>(&sm.delta[st][col0]);
        float pp[2], dd[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = col0 + e;
          const float sv = s[i + e];
          const float ls = e ? lv.y : lv.x, de = e ? dl.y : dl.x;
          float pj, chain = 1.f;
          if (clamp) {
            const float th = fast_tanh(sv * pre);
            pj = fast_exp2(fmaf(th, post, -ls));
            chain = 1.f - th * th;
          } else {
            pj = fast_exp2(fmaf(sv, mul, -ls));
          }
          if (part) {
            const int pq = (col < split ? a0 : a1) + p.pos.stride * col;
            bool keep = key_ok[h] && (col < ncols);
            if (p.causal) {
              keep = keep && (pos_k[h] <= pq);
              if (p.window > 0) keep = keep && (pq - pos_k[h] <= p.window);
            }
            if constexpr (DOCS) keep = keep && (span[h].x <= pq) && (pq < span[h].y);
            if (!keep) pj = 0.f;
          }
          pp[e] = pj;
          dd[e] = pj * (dp[i + e] - de) * chain;
        }
        pa[i / 2] = pack16<BF16>(pp[0], pp[1]);
        da[i / 2] = pack16<BF16>(dd[0], dd[1]);
      }
      const uint64_t qb_desc = gmma_desc(qmn, sm.q[st]);
      const uint64_t dob_desc = gmma_desc(qmn, sm.dout[st]);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t a4[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
        wgmma_rs<BF16, D, 1>(dv, a4, gmma_desc_add(dob_desc, kk * 2048), 1u);
      }
      if constexpr (ONE_PASS) {
        wgmma_commit();
        // dS^T -> this warpgroup's 64 key rows of the shared [128 keys][64 queries] tile (128B swizzle): the K-major A
        // of dK += dS^T Q and, read MN-major, the A of dQ = dS K.
        uint8_t* ds = sm.ds[n_ds & 1];
        ++n_ds;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int row = 64 * W + r_lo + 8 * (i & 1);
          const int col = 8 * (i / 2) + cq;
          *reinterpret_cast<uint32_t*>(ds + sw128_off(row, col)) = da[i];
        }
        fence_proxy_async_shared();
        // the previous tile's bulk reduce has finished reading the staging buffer before anyone passes the barrier
        if (wg_tid == 0) bulk_wait_read<0>();
        named_bar_sync(1, 256);  // both halves of dS^T are in place
        const uint64_t dsk_desc = gmma_desc(KMAJ, ds + W * SUB64);
        const uint64_t dsq_desc = gmma_desc(dsmn, ds);
        const uint64_t kb_desc = gmma_desc(kmn, sm.k + W * SUB128);
        float dq[32];
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_ss<BF16, D, 0, 1>(dk, gmma_desc_add(dsk_desc, kk * 32), gmma_desc_add(qb_desc, kk * 2048), 1u);
        // dQ[64 q][64 W ..] = dS[q][128 keys] K[128 keys][64 W ..]
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
          wgmma_ss<BF16, 64, 1, 1>(dq, gmma_desc_add(dsq_desc, kk * 2048), gmma_desc_add(kb_desc, kk * 2048),
                                   kk > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dv);
        fence_regs(dk);
        fence_regs(dq);
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.qd_empty[st]);

        // stage dQ in the layout of map_dq's 128B-swizzled [64 rows][32 fp32] box, then two tensor reductions add it
        // into dq_acc (rows past n_q carry exact zeros and stay inside n_pad, a multiple of 64)
        float* stage = sm.dq_stage[W];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = r_lo + 8 * h;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int chunk = 2 * (j % 4) + cq / 4;  // 16-byte chunk of the 128-byte box row
            *reinterpret_cast<float2*>(stage + (j / 4) * 2048 + row * 32 + ((chunk ^ (row & 7)) * 4) + cq % 4) =
                make_float2(dq[4 * j + 2 * h], dq[4 * j + 2 * h + 1]);
          }
        }
        fence_proxy_async_shared();
        named_bar_sync(2 + W, 128);
        if (wg_tid == 0) {
          const int bh = it.b * p.heads + t.rep * p.kv_heads + it.kvh;
          tma_reduce_add_2d(map_dq, stage, 64 * W, bh * p.n_pad + c0);
          tma_reduce_add_2d(map_dq, stage + 2048, 64 * W + 32, bh * p.n_pad + c0);
          bulk_commit();
        }
      } else {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint32_t a4[4] = {da[4 * kk], da[4 * kk + 1], da[4 * kk + 2], da[4 * kk + 3]};
          wgmma_rs<BF16, D, 1>(dk, a4, gmma_desc_add(qb_desc, kk * 2048), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dv);
        fence_regs(dk);
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.qd_empty[st]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.kv_empty);
    // the item's dQ reductions are complete before the CTA can exit (and its shared memory go away)
    if (ONE_PASS && wg_tid == 0) bulk_wait<0>();

    // epilogue: dK carries the folded softmax scale
    bool ring = false;
    if constexpr (ONE_PASS) ring = p.ring_reduce != 0;
    if (ring) {
      if constexpr (ONE_PASS) {
        if (any) {
          // added into the owner's fp32 [2][b*hk][nk_pad][d] accumulators (peer-mapped in a ring)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const size_t row = ((size_t)it.b * p.kv_heads + it.kvh) * p.nk_pad + key[h];
            float* dkr = p.dkv_acc[it.owner] + row * D;
            float* dvr = p.dkv_acc[it.owner] + ((size_t)p.batch * p.kv_heads * p.nk_pad + row) * D;
#pragma unroll
            for (int j = 0; j < D / 8; ++j) {
              red_add_v2(dkr + 8 * j + cq, dk[4 * j + 2 * h] * p.scale, dk[4 * j + 2 * h + 1] * p.scale);
              red_add_v2(dvr + 8 * j + cq, dv[4 * j + 2 * h], dv[4 * j + 2 * h + 1]);
            }
          }
        }
      }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (key[h] >= p.n_k) continue;
        const size_t off = (((size_t)it.b * p.n_k + key[h]) * p.kv_heads + it.kvh) * D;
        uint16_t* dkr = reinterpret_cast<uint16_t*>(p.dk) + off;
        uint16_t* dvr = reinterpret_cast<uint16_t*>(p.dv) + off;
#pragma unroll
        for (int j = 0; j < D / 8; ++j) {
          *reinterpret_cast<uint32_t*>(dkr + 8 * j + cq) =
              pack16<BF16>(dk[4 * j + 2 * h] * p.scale, dk[4 * j + 2 * h + 1] * p.scale);
          *reinterpret_cast<uint32_t*>(dvr + 8 * j + cq) = pack16<BF16>(dv[4 * j + 2 * h], dv[4 * j + 2 * h + 1]);
        }
      }
    }
  }
}

template <int D, bool BF16, bool ONE_PASS, bool DOCS, class P>
__global__ void __launch_bounds__(NTHREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap map_qd64, const __grid_constant__ CUtensorMap map_kv,
                    const __grid_constant__ CUtensorMap map_dq, const __grid_constant__ P p) {
  extern __shared__ uint8_t smem_raw[];
  DkvSmem<D>& sm = *reinterpret_cast<DkvSmem<D>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x / 32;
  if (threadIdx.x == 0) {
    mbar_init(&sm.kv_full, 1);
    mbar_init(&sm.kv_empty, 8);
    for (int i = 0; i < QST; ++i) {
      mbar_init(&sm.qd_full[i], 1);
      mbar_init(&sm.qd_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  // one-pass: the asynchronous consumer schedule spills less at 240 registers than at 232 (232 against 380 bytes of
  // spill stores, CUDA 12.9); the producer warp's own spills at 24 stay off the consumers' path
  if (warp >= 8) {
    setmaxnreg_dec<ONE_PASS ? 24 : 40>();
    if (warp == 8) dkv_producer<D, ONE_PASS, DOCS>(sm, p, &map_qd64, &map_kv);
  } else {
    setmaxnreg_inc<ONE_PASS ? 240 : 232>();
    dkv_consumer<D, BF16, ONE_PASS, DOCS>(sm, p, &map_dq, warp < 4 ? 0 : 1);
  }
}

template <bool BF16>
__global__ void bwd_prep_kernel(const uint16_t* __restrict__ q, const uint16_t* __restrict__ o,
                                const uint16_t* __restrict__ dout, const float* __restrict__ lse,
                                uint16_t* __restrict__ qdo_slot, float* __restrict__ stat_slot, int batch, int n,
                                int heads, int d, int n_pad) {
  const int vec_per_row = d / 8;  // 8 or 16 lanes per row
  const long long rows = (long long)batch * n * heads;
  const long long gid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long row = gid / vec_per_row;
  const int c = gid % vec_per_row;
  float part = 0.f;
  long long out_row = 0;
  int hh = 0, i = 0, b = 0;
  const bool active = row < rows;
  if (active) {
    hh = row % heads;
    i = (row / heads) % n;
    b = row / ((long long)heads * n);
    out_row = ((long long)b * heads + hh) * n + i;
    const uint4 qv = reinterpret_cast<const uint4*>(q + row * d)[c];
    const uint4 ov = reinterpret_cast<const uint4*>(o + row * d)[c];
    const uint4 dv = reinterpret_cast<const uint4*>(dout + row * d)[c];
    reinterpret_cast<uint4*>(qdo_slot + out_row * d)[c] = qv;
    reinterpret_cast<uint4*>(qdo_slot + (rows + out_row) * d)[c] = dv;
    const uint32_t ow[4] = {ov.x, ov.y, ov.z, ov.w}, dw[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float o0, o1, d0, d1;
      if (BF16) {
        o0 = __uint_as_float(ow[e] << 16); o1 = __uint_as_float(ow[e] & 0xffff0000u);
        d0 = __uint_as_float(dw[e] << 16); d1 = __uint_as_float(dw[e] & 0xffff0000u);
      } else {
        const __half2 oh = *reinterpret_cast<const __half2*>(&ow[e]);
        const __half2 dh = *reinterpret_cast<const __half2*>(&dw[e]);
        o0 = __low2float(oh); o1 = __high2float(oh);
        d0 = __low2float(dh); d1 = __high2float(dh);
      }
      part += o0 * d0 + o1 * d1;
    }
  }
  for (int off = vec_per_row / 2; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
  if (active && c == 0) {
    const long long srow = ((long long)b * heads + hh) * n_pad + i;
    const float l = lse[((long long)b * heads + hh) * n + i];
    stat_slot[srow] = l * kLog2e;  // +inf stays +inf
    stat_slot[(long long)batch * heads * n_pad + srow] = part;
  }
}

// Attention-sink gradient of this rank's rows, from the stat slot bwd_prep has just written (lse*log2e, delta):
//   dsinks[h] = -sum_{b,i} exp(sinks[h] - lse[b,h,i]) * delta[b,h,i]
// One CTA per head, a fixed row-to-thread assignment and a fixed reduction tree: no atomics, so the result is bitwise
// reproducible.  Rows that see no key have delta = 0 (and, without a sink, lse = +inf), so they add 0.
constexpr int SINK_GRAD_THREADS = 256;
__global__ void __launch_bounds__(SINK_GRAD_THREADS)
sink_grad_kernel(const float* __restrict__ stat_slot, const float* __restrict__ sinks, float* __restrict__ dsinks,
                 int batch, int n, int heads, int n_pad) {
  const int h = blockIdx.x;
  const float s2 = sinks[h] * kLog2e;
  float acc = 0.f;
  for (int b = 0; b < batch; ++b) {
    const float* lse2 = stat_slot + ((long long)b * heads + h) * n_pad;
    const float* delta = lse2 + (long long)batch * heads * n_pad;
    for (int i = threadIdx.x; i < n; i += SINK_GRAD_THREADS) acc += exp2f(s2 - lse2[i]) * delta[i];
  }
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  __shared__ float part[SINK_GRAD_THREADS / 32];
  if (lane_id() == 0) part[threadIdx.x / 32] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float total = 0.f;
    for (int w = 0; w < SINK_GRAD_THREADS / 32; ++w) total += part[w];
    dsinks[h] = -total;
  }
}

// fp32 accumulator [rows_outer][n_pad][d] -> 16 bit [b][n][h][d] (rows_outer = b * h), scaled.  One thread = 8 elements.
template <bool BF16>
__global__ void acc_convert_kernel(const float* __restrict__ acc, uint16_t* __restrict__ out, int batch, int heads,
                                   int n, int n_pad, int d, float scale) {
  const int vec_per_row = d / 8;
  const long long total = (long long)batch * n * heads * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = i % vec_per_row;
    long long r = i / vec_per_row;
    const int h = r % heads;
    r /= heads;
    const int row = r % n;
    const int b = r / n;
    const float4* src =
        reinterpret_cast<const float4*>(acc + (((long long)b * heads + h) * n_pad + row) * d + c * 8);
    const float4 a = src[0], bq = src[1];
    uint4 w;
    if (BF16) {
      w.x = pack_bf16x2(a.x * scale, a.y * scale);
      w.y = pack_bf16x2(a.z * scale, a.w * scale);
      w.z = pack_bf16x2(bq.x * scale, bq.y * scale);
      w.w = pack_bf16x2(bq.z * scale, bq.w * scale);
    } else {
      w.x = pack_f16x2(a.x * scale, a.y * scale);
      w.y = pack_f16x2(a.z * scale, a.w * scale);
      w.z = pack_f16x2(bq.x * scale, bq.y * scale);
      w.w = pack_f16x2(bq.z * scale, bq.w * scale);
    }
    reinterpret_cast<uint4*>(out)[i] = w;
  }
}


}  // namespace

template <int D>
void launch_attn_bwd_dq(const CUtensorMap& map_qd, const CUtensorMap& map_kv, const AttnBwdParams& p, int num_sms,
                        cudaStream_t stream) {
  using Kern = void (*)(const CUtensorMap, const CUtensorMap, const AttnBwdParams);
  Kern kern = p.doc_spans != nullptr
                  ? (p.is_bf16 ? attn_bwd_dq_kernel<D, true, true> : attn_bwd_dq_kernel<D, false, true>)
                  : (p.is_bf16 ? attn_bwd_dq_kernel<D, true, false> : attn_bwd_dq_kernel<D, false, false>);
  const size_t smem = sizeof(DqSmem<D>) + 1024;
  cuda_check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "bwd_dq smem attr");
  const int items = p.batch * p.heads * ((p.n_q + 127) / 128);
  const int grid = items < num_sms ? items : num_sms;
  void* args[] = {(void*)&map_qd, (void*)&map_kv, (void*)&p};
  cuda_check(cudaLaunchKernel((void*)kern, dim3(grid), dim3(NTHREADS), args, smem, stream), "bwd_dq launch");
}

template <int D>
void launch_attn_bwd_dkdv(const CUtensorMap& map_qd64, const CUtensorMap& map_kv, const AttnBwdParams& p,
                          int num_sms, cudaStream_t stream) {
  using Kern = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const AttnBwdParams);
  Kern kern = p.doc_spans != nullptr ? (p.is_bf16 ? attn_bwd_dkv_kernel<D, true, false, true, AttnBwdParams>
                                                   : attn_bwd_dkv_kernel<D, false, false, true, AttnBwdParams>)
                                     : (p.is_bf16 ? attn_bwd_dkv_kernel<D, true, false, false, AttnBwdParams>
                                                   : attn_bwd_dkv_kernel<D, false, false, false, AttnBwdParams>);
  const size_t smem = sizeof(DkvSmem<D>) + 1024;
  cuda_check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
             "bwd_dkdv smem attr");
  const int items = p.batch * p.kv_heads * ((p.n_k + 127) / 128);
  const int grid = items < num_sms ? items : num_sms;
  void* args[] = {(void*)&map_qd64, (void*)&map_kv, (void*)&map_kv /* map_dq: one-pass form only */, (void*)&p};
  cuda_check(cudaLaunchKernel((void*)kern, dim3(grid), dim3(NTHREADS), args, smem, stream), "bwd_dkdv launch");
}

void launch_attn_bwd_fused(const CUtensorMap& map_qd64, const CUtensorMap& map_kv, const CUtensorMap& map_dq,
                           const AttnBwdFusedParams& p, int num_sms, cudaStream_t stream) {
  using Kern = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const AttnBwdFusedParams);
  Kern kern = p.doc_spans != nullptr ? (p.is_bf16 ? attn_bwd_dkv_kernel<128, true, true, true, AttnBwdFusedParams>
                                                   : attn_bwd_dkv_kernel<128, false, true, true, AttnBwdFusedParams>)
                                     : (p.is_bf16 ? attn_bwd_dkv_kernel<128, true, true, false, AttnBwdFusedParams>
                                                   : attn_bwd_dkv_kernel<128, false, true, false, AttnBwdFusedParams>);
  const size_t smem = sizeof(DkvSmem<128>) + 1024;
  cuda_check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "bwd_fused smem attr");
  const int items = p.hop_count * p.batch * p.kv_heads * ((p.n_k + 127) / 128);
  const int grid = items < num_sms ? items : num_sms;
  void* args[] = {(void*)&map_qd64, (void*)&map_kv, (void*)&map_dq, (void*)&p};
  cuda_check(cudaLaunchKernel((void*)kern, dim3(grid), dim3(NTHREADS), args, smem, stream), "bwd_fused launch");
}

size_t attn_bwd_fused_smem_bytes() { return sizeof(DkvSmem<128>) + 1024; }

void launch_bwd_prep(const void* q, const void* o, const void* dout, const float* lse, void* qdo_slot,
                     float* stat_slot, int batch, int n, int heads, int d, int n_pad, int is_bf16,
                     cudaStream_t stream, const float* sinks, float* dsinks) {
  const long long threads_total = (long long)batch * n * heads * (d / 8);
  if (threads_total == 0) {
    if (sinks != nullptr) cuda_check(cudaMemsetAsync(dsinks, 0, sizeof(float) * heads, stream), "dsinks memset");
    return;
  }
  const int threads = 256;
  const long long blocks = (threads_total + threads - 1) / threads;
  auto kern = is_bf16 ? bwd_prep_kernel<true> : bwd_prep_kernel<false>;
  kern<<<(unsigned)blocks, threads, 0, stream>>>(
      reinterpret_cast<const uint16_t*>(q), reinterpret_cast<const uint16_t*>(o),
      reinterpret_cast<const uint16_t*>(dout), lse, reinterpret_cast<uint16_t*>(qdo_slot), stat_slot, batch, n, heads,
      d, n_pad);
  cuda_check(cudaGetLastError(), "bwd_prep launch");
  if (sinks != nullptr) {
    sink_grad_kernel<<<heads, SINK_GRAD_THREADS, 0, stream>>>(stat_slot, sinks, dsinks, batch, n, heads, n_pad);
    cuda_check(cudaGetLastError(), "sink_grad launch");
  }
}

void launch_acc_convert(const float* acc, void* out, int batch, int heads, int n, int n_pad, int d, float scale,
                        int is_bf16, cudaStream_t stream) {
  const long long vecs = (long long)batch * n * heads * (d / 8);
  if (vecs == 0) return;
  const int threads = 256;
  long long blocks = (vecs + threads - 1) / threads;
  if (blocks > 132 * 32) blocks = 132 * 32;
  auto kern = is_bf16 ? acc_convert_kernel<true> : acc_convert_kernel<false>;
  kern<<<(int)blocks, threads, 0, stream>>>(acc, reinterpret_cast<uint16_t*>(out), batch, heads, n, n_pad, d, scale);
  cuda_check(cudaGetLastError(), "acc_convert launch");
}

template void launch_attn_bwd_dq<64>(const CUtensorMap&, const CUtensorMap&, const AttnBwdParams&, int, cudaStream_t);
template void launch_attn_bwd_dq<128>(const CUtensorMap&, const CUtensorMap&, const AttnBwdParams&, int, cudaStream_t);
template void launch_attn_bwd_dkdv<64>(const CUtensorMap&, const CUtensorMap&, const AttnBwdParams&, int, cudaStream_t);
template void launch_attn_bwd_dkdv<128>(const CUtensorMap&, const CUtensorMap&, const AttnBwdParams&, int, cudaStream_t);

}  // namespace rab
