// Fused ring flash-attention forward for sm_90a (wgmma + TMA + mbarrier).
//
// One persistent, warp-specialised CTA per SM (384 threads):
//   warps 0-3   consumer WG 0 : query rows [0, 64) of the item's 128-row Q tile
//   warps 4-7   consumer WG 1 : query rows [64, 128)
//               each consumer issues its own wgmma: S = Q K^T (both operands from shared memory, S in registers),
//               online softmax in registers, O += P V (P straight from the S registers as the A operand, V read
//               MN-major from shared memory).  O, the running maximum and the running sum stay in registers across
//               every hop of the ring, so nothing is re-normalised or round-tripped through HBM between hops.
//   warp 8      TMA producer  : Q tiles and K/V tiles (128B-swizzled tensor-map boxes) -> shared memory
//   warp 10     ring fetcher  : pulls the other ring ranks' K/V slots over NVLink with bulk-TMA copies
//                               (peer global -> smem -> local global) and publishes per-owner ready counters
//   warps 9, 11 idle (keep the producer warpgroup whole for setmaxnreg)
//
// The ring itself is only a schedule: ring rank r visits owners hop_owner[0..hop_count) (itself first).
// K/V of owner o live in slot o of a symmetric [world][2][b*hk][n][d] buffer.  Slot r is written locally
// by pack_kv; the other slots are filled inside this kernel by the fetcher warps of all CTAs (each moves
// 1/gridDim of every slot), overlapping the NVLink transfer with the MMAs of earlier hops.  Layout (plain / striped /
// zig-zag), causal + sliding-window masking, key padding and packed documents are position functions evaluated
// in-kernel; fully masked tiles are never loaded.
//
// attn_fwd_fp8_kernel is the same body on e4m3 operands (head dim 128, forward only, see consumer_role): K and V^T
// slots written by pack_kv_fp8, both attention matmuls as e4m3 wgmma, bf16 output.
#include <cstdlib>
#include <stdexcept>

#include "attn_common.cuh"

namespace rab {
namespace {

constexpr int BM = 64;   // query rows per consumer warpgroup (wgmma M); an item is 2 * BM rows
constexpr int BN = 128;  // keys per K/V tile
constexpr int NSLOT = 4;
constexpr int FETCH_PIECE = 16384;
constexpr int NTHREADS = 384;
constexpr int SUB_BYTES = 128 * 128;  // one 64-element-wide, 128-row swizzled sub-tile

template <int D>
struct FwdSmem {
  static constexpr int NSUB = D / 64;
  static constexpr int TILE_BYTES = NSUB * SUB_BYTES;
  alignas(1024) uint8_t q[2][TILE_BYTES];
  alignas(1024) uint8_t kv[NSLOT][TILE_BYTES];
  alignas(1024) uint8_t fetch[2][FETCH_PIECE];
  uint64_t q_full[2], q_empty[2];
  uint64_t kv_full[NSLOT], kv_empty[NSLOT];
  uint64_t fetch_full[2];
};

struct Item {
  int b, h, kvh, qp;
  int row0[2];
  bool tvalid[2];
  int qlo[2], qhi[2];
};

__device__ __forceinline__ int num_items(const AttnFwdParams& p) {
  const int nqp = (p.n_q + 2 * BM - 1) / (2 * BM);
  return p.batch * p.heads * nqp;
}

// Work items are ordered heaviest-first (largest q index first under causal masking) and, inside one
// q-pair, so that query heads sharing a KV head are adjacent (L2 reuse of the K/V tiles).
__device__ __forceinline__ void decode_item(const AttnFwdParams& p, int idx, Item& it) {
  const int bh = p.batch * p.heads;
  const int nqp = (p.n_q + 2 * BM - 1) / (2 * BM);
  it.qp = nqp - 1 - idx / bh;
  const int r = idx % bh;
  it.b = r / p.heads;
  const int hh = r % p.heads;
  const int groups = p.heads / p.kv_heads;
  it.kvh = hh / groups;
  it.h = (hh % groups) * p.kv_heads + it.kvh;  // reference mapping: query head j uses kv head j % kv_heads
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    it.row0[t] = it.qp * 2 * BM + t * BM;
    it.tvalid[t] = it.row0[t] < p.n_q;
    if (it.tvalid[t]) {
      pos_range(p.pos, p.rank, it.row0[t], min(it.row0[t] + BM, p.n_q) - 1, it.qlo[t], it.qhi[t]);
      it.qlo[t] += p.q_pos_offset;
      it.qhi[t] += p.q_pos_offset;
    } else {
      it.qlo[t] = it.qhi[t] = 0;
    }
  }
}

template <bool DOCS>
using FwdScan = WarpTileScan<2, false, DOCS>;

template <bool DOCS>
__device__ __forceinline__ void init_scan(FwdScan<DOCS>& sc, const AttnFwdParams& p, const Item& it) {
  sc.pm = &p.pos;
  sc.hop_owner = p.hop_owner;
  sc.hop_count = p.hop_count;
  sc.groups = 1;
  sc.n_stream = p.n_k;
  sc.tile = BN;
  sc.stream_off = 0;
  sc.stat_off = 0;
  sc.mc = MaskCfg{p.causal, p.window, p.kmask_bits != nullptr};
#pragma unroll
  for (int t = 0; t < 2; ++t) sc.st[t] = StatRange{it.qlo[t], it.qhi[t], it.tvalid[t], false};
  if constexpr (DOCS) {
    const int2* rows = doc_row_spans(p.doc_spans, p.batch, p.n_q, p.rank, it.b);
#pragma unroll
    for (int t = 0; t < 2; ++t)
      if (it.tvalid[t]) sc.doc[t] = doc_range(rows, it.row0[t], min(it.row0[t] + BM, p.n_q) - 1, lane_id());
  }
}

// ------------------------------------------------------------------------------------------------
// warp 8: TMA producer (all 32 lanes scan tiles, lane 0 issues)
// ------------------------------------------------------------------------------------------------
// FP8: Q, K and V^T tiles are one 128-byte-wide sub-tile each (e4m3), so every tile is one box of SUB_BYTES.
template <int D, bool DOCS, bool FP8 = false>
__device__ __forceinline__ void producer_role(FwdSmem<D>& sm, const AttnFwdParams& p, const CUtensorMap* map_q,
                                              const CUtensorMap* map_kv) {
  constexpr int NSUB = FP8 ? 1 : FwdSmem<D>::NSUB;
  constexpr uint32_t TILE_BYTES = FP8 ? SUB_BYTES : FwdSmem<D>::TILE_BYTES;
  const int lane = lane_id();
  uint32_t n_slot = 0;
  uint32_t items = 0;
  uint32_t ready_mask = p.all_ready ? 0xffffffffu : (1u << p.rank);
  const int total = num_items(p);
  for (int idx = blockIdx.x; idx < total; idx += gridDim.x) {
    Item it;
    decode_item(p, idx, it);
    if (lane == 0) {  // both warpgroups' rows in one 128-row box per 64-wide sub-tile
      const uint32_t buf = items & 1;
      mbar_wait(&sm.q_empty[buf], ((items >> 1) & 1) ^ 1, 100 + buf);
      mbar_expect_tx(&sm.q_full[buf], TILE_BYTES);
#pragma unroll
      for (int s = 0; s < NSUB; ++s)
        tma_load_4d(sm.q[buf] + s * SUB_BYTES, map_q, &sm.q_full[buf], s * 64, it.h, it.row0[0], it.b);
    }
    items++;
    FwdScan<DOCS> scan;
    init_scan<DOCS>(scan, p, it);
    ScanTile ti;
    while (scan.next(lane, ti)) {
      if (!((ready_mask >> ti.owner) & 1u)) {
        if (lane == 0) {
          spin_until_ge_gpu(&p.ready[ti.owner], gridDim.x, 110);
          fence_proxy_async_global();
        }
        ready_mask |= 1u << ti.owner;
      }
      if (lane == 0) {
#pragma unroll
        for (int which = 0; which < 2; ++which) {
          const uint32_t n = n_slot + which;
          const uint32_t slot = n % NSLOT, ph = (n / NSLOT) & 1;
          mbar_wait(&sm.kv_empty[slot], ph ^ 1, 120 + slot);
          mbar_expect_tx(&sm.kv_full[slot], TILE_BYTES);
#pragma unroll
          for (int s = 0; s < NSUB; ++s)
            tma_load_4d(sm.kv[slot] + s * SUB_BYTES, map_kv, &sm.kv_full[slot], s * 64, ti.idx * BN,
                        it.b * p.kv_heads + it.kvh, ti.owner * 2 + which);
        }
      }
      n_slot += 2;
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// warp 10: ring fetcher (peer K/V slot -> local slot, 1/gridDim of every slot per CTA)
// ------------------------------------------------------------------------------------------------
template <int D>
__device__ __forceinline__ void fetch_role(FwdSmem<D>& sm, const AttnFwdParams& p) {
  uint32_t fcount = 0;
  const unsigned long long npieces = (p.slot_bytes + FETCH_PIECE - 1) / FETCH_PIECE;
  const unsigned long long t_begin = global_timer_ns();
  for (int s = 1; s < p.hop_count; ++s) {
    const int o = p.hop_owner[s];
    const uint8_t* src = p.kv_peer[o];  // owner o's own slot (peer-mapped staging)
    uint8_t* dst = p.kv_local + (unsigned long long)o * p.slot_bytes;
    auto piece_bytes = [&](unsigned long long pc) -> uint32_t {
      const unsigned long long rem = p.slot_bytes - pc * FETCH_PIECE;
      return rem < (unsigned long long)FETCH_PIECE ? (uint32_t)rem : (uint32_t)FETCH_PIECE;
    };
    unsigned long long pc = blockIdx.x;
    if (pc < npieces) {
      // software pipeline: load(i+1) is in flight while load(i) is drained to local memory
      bulk_wait_read<0>();
      {
        const uint32_t buf = fcount & 1;
        const uint32_t bytes = piece_bytes(pc);
        mbar_expect_tx(&sm.fetch_full[buf], bytes);
        bulk_load_1d(sm.fetch[buf], src + pc * FETCH_PIECE, bytes, &sm.fetch_full[buf]);
      }
      while (pc < npieces) {
        const unsigned long long pn = pc + gridDim.x;
        if (pn < npieces) {
          bulk_wait_read<0>();  // the store that last read the other buffer has drained it
          const uint32_t buf = (fcount + 1) & 1;
          const uint32_t bytes = piece_bytes(pn);
          mbar_expect_tx(&sm.fetch_full[buf], bytes);
          bulk_load_1d(sm.fetch[buf], src + pn * FETCH_PIECE, bytes, &sm.fetch_full[buf]);
        }
        const uint32_t buf = fcount & 1;
        mbar_wait(&sm.fetch_full[buf], (fcount >> 1) & 1, 300 + buf);
        bulk_store_1d(dst + pc * FETCH_PIECE, sm.fetch[buf], piece_bytes(pc));
        bulk_commit();
        fcount++;
        pc = pn;
      }
      bulk_wait<0>();  // all stores of this owner's slot are complete
    }
    fence_proxy_async_global();
    __threadfence();
    red_release_gpu_add(&p.ready[o], 1u);
  }
  if (p.fetch_times != nullptr && p.hop_count > 1) {  // bench.py: ring K/V GB/s over the fetch-active window
    p.fetch_times[2 * blockIdx.x] = t_begin;
    p.fetch_times[2 * blockIdx.x + 1] = global_timer_ns();
  }
}

// ------------------------------------------------------------------------------------------------
// warps 0-7: consumer warpgroups (S = Q K^T, online softmax, O += P V, epilogue)
//
// Thread t of warpgroup w owns rows 16 (t / 32) + (t % 32) / 4 and +8 of the warpgroup's 64 rows (wgmma accumulator
// layout, see ptx.cuh); a row is spread over 4 lanes, so row maxima and sums take two shuffles.  The running maximum
// is lazy: it is only raised when a tile exceeds it by more than 2^8, and only then are l and O rescaled.
// Every consumer walks the whole tile sequence of the item (also tiles its rows do not need, and items whose second
// tile lies beyond n_q) so that each K/V stage is released by both warpgroups exactly once, in order.
// ------------------------------------------------------------------------------------------------
//
// FP8 (e4m3 Q, K, V^T; BF16 output): S = Q K^T and O += P V^T run as m64n128k32 e4m3 wgmma, 4 k-steps each.  P goes
// from the S registers into the A operand as e4m3 in register order; the V^T tile's key order (v8_key_of_slot) makes
// that product right.  The lazy maximum is not used here: against a maximum that is only raised, every key more than
// about 7 nats below it falls under e4m3's smallest value (2^-9), and with an attention sink that is most of a long
// row's tail.  Instead each tile's P is taken against that tile's own maximum minus 8 (so P <= 2^8 = 256, inside
// e4m3's range of 448); the tile maximum used is floored 2^32 below the running maximum, so the reference is never
// more than 2^40 below it and O and l stay far inside fp32.  O and l are rescaled to the new reference every tile.
// l sums the e4m3-rounded P, the same values P V multiplies.  Each tile's P V is accumulated into zeroed registers and
// added to O in fp32: the e4m3 MMA accumulates at reduced precision, and with O as its accumulator a tile that is
// small against O loses its low bits.  A carried hop state is handed over against the running maximum.  q_descale * k_descale is folded into the logit scale of
// each item, v_descale into the epilogue; the carried O of the hop mode stays unscaled (v_descale is the same for
// every owner).
// ------------------------------------------------------------------------------------------------
//
// SINK (a separate instantiation, selected by a non-null p.sinks): the row's learned sink logit sigma_h is its initial
// softmax state, m = sigma_h * log2(e), l = 1, O = 0, in every launch that does not carry a state in (the single launch,
// and hop 0 of the hop-wise mode), so it is counted exactly once per row; the carry and the epilogue are unchanged.  A
// row that sees no key ends with out = 0 and lse = sigma_h.  FP8: the running maximum starts at sigma_h too, so P <= 2^8
// and a reference at most 2^40 below max(sigma_h, key maxima) still hold.  Only a row whose every key weighs less than
// 2^-32 of the sink meets the floor: its keys are then taken against sigma_h - 40 log2 units and those below 2^-49 of
// the sink round to zero in e4m3.
// ------------------------------------------------------------------------------------------------
template <int D, bool BF16, bool DOCS, bool FP8 = false, bool SINK = false>
__device__ __forceinline__ void consumer_role(FwdSmem<D>& sm, const AttnFwdParams& p, const int t) {
  constexpr int NO = D / 2;  // O accumulator registers per thread
  // K-major operands (Q, K): 8-row groups 1024 B apart.  MN-major V (B of P V): d sub-tiles SUB_BYTES apart.
  constexpr uint64_t kmaj = gmma_desc_static(16, 1024);
  constexpr uint64_t vmaj = gmma_desc_static(SUB_BYTES, 1024);
  constexpr uint32_t TILE_BYTES = FwdSmem<D>::TILE_BYTES;
  const int wg_tid = threadIdx.x - 128 * t;
  const int lane = lane_id();
  const int warp_in_wg = wg_tid / 32;
  const int r_lo = warp_in_wg * 16 + lane / 4;  // this thread's rows: r_lo, r_lo + 8
  const int cq = 2 * (lane % 4);                // first of this thread's column pairs

  const bool clamp = p.softclamp > 0.f;
  const float mul = clamp ? 1.f : p.scale * kLog2e;
  const float pre = clamp ? p.scale / p.softclamp : 0.f;
  const float post = clamp ? p.softclamp * kLog2e : 0.f;

  uint32_t n_kv = 0;
  uint32_t items = 0;
  const int total = num_items(p);
  for (int idx = blockIdx.x; idx < total; idx += gridDim.x) {
    Item it;
    decode_item(p, idx, it);
    float mul_it = mul, pre_it = pre, v_scale = 1.f;
    if constexpr (FP8) {
      const float qk = p.q_descale[it.b * p.heads + it.h] * p.k_descale[it.b * p.kv_heads + it.kvh];
      if (clamp) pre_it *= qk;
      else mul_it *= qk;
      v_scale = p.v_descale[it.b * p.kv_heads + it.kvh];
    }
    const uint32_t buf = items & 1;
    mbar_wait(&sm.q_full[buf], (items >> 1) & 1, 400 + t);
    items++;
    const bool tvalid = t ? it.tvalid[1] : it.tvalid[0];
    const int row0 = t ? it.row0[1] : it.row0[0];
    int grow[2];
    bool row_ok[2];
    int pos_q[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      grow[h] = row0 + r_lo + 8 * h;
      row_ok[h] = tvalid && grow[h] < p.n_q;
      pos_q[h] = pos_of(p.pos, p.rank, min(grow[h], p.n_q - 1)) + p.q_pos_offset;
    }
    int2 span[2];  // document interval of each of this thread's rows
    if constexpr (DOCS) {
      const int2* rows = doc_row_spans(p.doc_spans, p.batch, p.n_q, p.rank, it.b);
#pragma unroll
      for (int h = 0; h < 2; ++h) span[h] = rows[min(grow[h], p.n_q - 1)];
    }

    float o[NO];
    float m_used[2] = {-INFINITY, -INFINITY};  // the reference of O and l (FP8: of the last tile)
    float m_run[2] = {-INFINITY, -INFINITY};   // FP8: the running maximum
    float l[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < NO; ++i) o[i] = 0.f;
    if (p.carry_in && tvalid) {
      // hop-at-a-time mode: O / m / l of this row continue from the previous hop's launch
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!row_ok[h]) continue;
        const size_t mlrow = ((size_t)it.b * p.heads + it.h) * p.n_q + grow[h];
        m_used[h] = p.carry_ml[mlrow];
        if constexpr (FP8) m_run[h] = m_used[h];
        l[h] = (lane % 4 == 0) ? p.carry_ml[(size_t)p.batch * p.heads * p.n_q + mlrow] : 0.f;
        const float* crow = p.carry_o + (((size_t)it.b * p.n_q + grow[h]) * p.heads + it.h) * D;
#pragma unroll
        for (int j = 0; j < D / 8; ++j) {
          const float2 x = *reinterpret_cast<const float2*>(crow + 8 * j + cq);
          o[4 * j + 2 * h] = x.x;
          o[4 * j + 2 * h + 1] = x.y;
        }
      }
    }
    if constexpr (SINK) {
      if (!p.carry_in) {
        const float sg = p.sinks[it.h] * kLog2e;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          m_used[h] = sg;
          if constexpr (FP8) m_run[h] = sg;
          l[h] = (lane % 4 == 0) ? 1.f : 0.f;  // l is summed over the row's 4 lanes at the end
        }
      }
    }

    const uint64_t q_desc = gmma_desc(kmaj, sm.q[buf] + t * BM * 128);
    FwdScan<DOCS> scan;
    init_scan<DOCS>(scan, p, it);
    ScanTile ti;
    while (scan.next(lane, ti)) {
      const bool need = t ? ti.need[1] : ti.need[0];
      const bool part = t ? ti.part[1] : ti.part[0];
      const uint32_t ks = (2 * n_kv) % NSLOT, kph = ((2 * n_kv) / NSLOT) & 1;
      const uint32_t vs = (2 * n_kv + 1) % NSLOT, vph = ((2 * n_kv + 1) / NSLOT) & 1;
      n_kv++;
      float s[64];
      mbar_wait(&sm.kv_full[ks], kph, 410 + t);
      if (need) {
        const uint64_t k_desc = gmma_desc(kmaj, sm.kv[ks]);
        wgmma_fence();
        if constexpr (FP8) {
#pragma unroll
          for (int kk = 0; kk < D / 32; ++kk)
            wgmma_e4m3_ss_n128(s, gmma_desc_add(q_desc, kk * 32), gmma_desc_add(k_desc, kk * 32), kk > 0 ? 1u : 0u);
        } else {
#pragma unroll
          for (int kk = 0; kk < D / 16; ++kk) {
            const uint32_t off = (kk / 4) * SUB_BYTES + (kk % 4) * 32;
            wgmma_ss<BF16, 128, 0, 0>(s, gmma_desc_add(q_desc, off), gmma_desc_add(k_desc, off), kk > 0 ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.kv_empty[ks]);

      uint32_t pa[32];
      float o_fac[2] = {1.f, 1.f};  // FP8: rescale of O to this tile's reference
      if (need) {
        if (clamp) {
#pragma unroll
          for (int i = 0; i < 64; ++i) s[i] = fast_tanh(s[i] * pre_it) * post;
        }
        if (part) {
          const int c0 = ti.idx * BN;
          const int split = p.pos.seg_len - c0;
          const int a0 = p.pos.base0[ti.owner] + p.pos.stride * c0;
          const int a1 = p.pos.base1[ti.owner] + p.pos.stride * (c0 - p.pos.seg_len);
          const int ncols = p.n_k - c0;
          uint32_t mb[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
          if (p.kmask_bits != nullptr) {
            const uint32_t* w = p.kmask_bits + ((size_t)ti.owner * p.batch + it.b) * p.kmask_words + (size_t)ti.idx * 4;
#pragma unroll
            for (int i = 0; i < 4; ++i) mb[i] = w[i];
          }
#pragma unroll
          for (int i = 0; i < 64; ++i) {
            const int col = 8 * (i / 4) + cq + (i & 1);
            const int h = (i >> 1) & 1;
            const int pk = (col < split ? a0 : a1) + p.pos.stride * col;
            bool keep = (col < ncols) && ((mb[i / 16] >> (col & 31)) & 1u);  // col / 32 == i / 16
            if (p.causal) {
              keep = keep && (pk <= pos_q[h]);
              if (p.window > 0) keep = keep && (pos_q[h] - pk <= p.window);
            }
            if constexpr (DOCS) keep = keep && (span[h].x <= pk) && (pk < span[h].y);
            if (!keep) s[i] = -INFINITY;
          }
        }
        float cmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 64; ++i) cmax[(i >> 1) & 1] = fmaxf(cmax[(i >> 1) & 1], s[i]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          cmax[h] = fmaxf(cmax[h], __shfl_xor_sync(0xffffffffu, cmax[h], 1));
          cmax[h] = fmaxf(cmax[h], __shfl_xor_sync(0xffffffffu, cmax[h], 2));
          cmax[h] *= mul_it;
        }
        float m_eff[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if constexpr (FP8) {
            // P of this tile against the tile's own maximum minus 8 (P <= 2^8); that reference is never taken more
            // than 2^40 below the running maximum (tile maxima are floored 2^32 below it), so O and l stay far inside
            // fp32.  l follows the new reference here, O when this tile's P V is added (o_fac)
            if (cmax[h] != -INFINITY) {
              m_run[h] = fmaxf(m_run[h], cmax[h]);
              const float ref = fmaxf(cmax[h], m_run[h] - 32.f) - 8.f;
              o_fac[h] = (m_used[h] == -INFINITY) ? 0.f : fast_exp2(m_used[h] - ref);
              l[h] *= o_fac[h];
              m_used[h] = ref;
            }
          } else if (cmax[h] > m_used[h] + 8.f) {  // raise the running max (rare): rescale l and O
            const float m_new = fmaxf(m_used[h], cmax[h]);
            const float factor = (m_used[h] == -INFINITY) ? 0.f : fast_exp2(m_used[h] - m_new);
            l[h] *= factor;
#pragma unroll
            for (int j = 0; j < D / 8; ++j) {
              o[4 * j + 2 * h] *= factor;
              o[4 * j + 2 * h + 1] *= factor;
            }
            m_used[h] = m_new;
          }
          m_eff[h] = (m_used[h] == -INFINITY) ? 0.f : m_used[h];
        }
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
          const int h = (i >> 1) & 1;
          const float e0 = fast_exp2(fmaf(s[i], mul_it, -m_eff[h]));
          const float e1 = fast_exp2(fmaf(s[i + 1], mul_it, -m_eff[h]));
          if constexpr (FP8) {
            s[i] = e0;
            s[i + 1] = e1;
          } else {
            l[h] += e0 + e1;
            pa[i / 2] = BF16 ? pack_bf16x2(e0, e1) : pack_f16x2(e0, e1);
          }
        }
        if constexpr (FP8) {
          // A operand of k-step g = S columns [32 g, 32 g + 32) in register order (see v8_key_of_slot); even words
          // hold row r_lo, odd words row r_lo + 8.  l sums the rounded P that P V multiplies.
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const float* x = s + 16 * g;
            pa[4 * g + 0] = pack_e4m3x4(x[0], x[1], x[4], x[5]);
            pa[4 * g + 1] = pack_e4m3x4(x[2], x[3], x[6], x[7]);
            pa[4 * g + 2] = pack_e4m3x4(x[8], x[9], x[12], x[13]);
            pa[4 * g + 3] = pack_e4m3x4(x[10], x[11], x[14], x[15]);
          }
#pragma unroll
          for (int w = 0; w < 16; ++w) l[w & 1] += sum_e4m3x4(pa[w]);
        }
      }

      mbar_wait(&sm.kv_full[vs], vph, 420 + t);
      if (need) {
        wgmma_fence();
        if constexpr (FP8) {
          // The e4m3 MMA adds its products into the accumulator at reduced precision, so with O as the accumulator
          // a tile that is small against O (the tail of a row behind an attention sink) loses its low bits, tile
          // after tile.  This tile's P V goes into zeroed registers and is added to O in fp32, one half of the
          // head dim at a time (d rows 64..127 of the V^T tile start 64 * 128 bytes in) to bound register use.
          const uint64_t vt_desc = gmma_desc(kmaj, sm.kv[vs]);  // V^T: d rows, key slots K-major
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            float acc[NO / 2];
#pragma unroll
            for (int kk = 0; kk < BN / 32; ++kk) {
              const uint32_t a4[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
              wgmma_e4m3_rs_n64(acc, a4, gmma_desc_add(vt_desc, half * 64 * 128 + kk * 32), kk > 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(acc);
#pragma unroll
            for (int i = 0; i < NO / 2; ++i) {
              float& oi = o[half * (NO / 2) + i];
              oi = fmaf(oi, o_fac[(i >> 1) & 1], acc[i]);
            }
          }
        } else {
          const uint64_t v_desc = gmma_desc(vmaj, sm.kv[vs]);
#pragma unroll
          for (int kk = 0; kk < BN / 16; ++kk) {
            const uint32_t a4[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
            wgmma_rs<BF16, D, 1>(o, a4, gmma_desc_add(v_desc, kk * 2048), 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs(o);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.kv_empty[vs]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.q_empty[buf]);
    if (!tvalid) continue;

#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    }
    if (p.carry_out) {
      // hand the un-normalised state to the next hop's launch
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!row_ok[h]) continue;
        if constexpr (FP8) {
          // carry O and l against the running maximum, the reference the next launch starts from
          if (m_used[h] != -INFINITY) {
            const float factor = fast_exp2(m_used[h] - m_run[h]);
            l[h] *= factor;
#pragma unroll
            for (int j = 0; j < D / 8; ++j) {
              o[4 * j + 2 * h] *= factor;
              o[4 * j + 2 * h + 1] *= factor;
            }
            m_used[h] = m_run[h];
          }
        }
        float* crow = p.carry_o + (((size_t)it.b * p.n_q + grow[h]) * p.heads + it.h) * D;
#pragma unroll
        for (int j = 0; j < D / 8; ++j)
          *reinterpret_cast<float2*>(crow + 8 * j + cq) = make_float2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
        if (lane % 4 == 0) {
          const size_t mlrow = ((size_t)it.b * p.heads + it.h) * p.n_q + grow[h];
          p.carry_ml[mlrow] = m_used[h];
          p.carry_ml[(size_t)p.batch * p.heads * p.n_q + mlrow] = l[h];
        }
      }
      continue;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!row_ok[h]) continue;
      float inv = l[h] > 0.f ? 1.f / l[h] : 0.f;
      if constexpr (FP8) inv *= v_scale;
      uint16_t* orow = reinterpret_cast<uint16_t*>(p.o) + (((size_t)it.b * p.n_q + grow[h]) * p.heads + it.h) * D;
#pragma unroll
      for (int j = 0; j < D / 8; ++j) {
        const float a = o[4 * j + 2 * h] * inv, bq = o[4 * j + 2 * h + 1] * inv;
        *reinterpret_cast<uint32_t*>(orow + 8 * j + cq) = BF16 ? pack_bf16x2(a, bq) : pack_f16x2(a, bq);
      }
      if (lane % 4 == 0) {
        const float m_eff = (m_used[h] == -INFINITY) ? 0.f : m_used[h];
        p.lse[((size_t)it.b * p.heads + it.h) * p.n_q + grow[h]] = l[h] > 0.f ? (m_eff + log2f(l[h])) * kLn2 : INFINITY;
      }
    }
  }
}

template <int D, bool BF16, bool DOCS, bool FP8, bool SINK = false>
__device__ __forceinline__ void attn_fwd_body(const CUtensorMap& map_q, const CUtensorMap& map_kv,
                                              const AttnFwdParams& p) {
  extern __shared__ uint8_t smem_raw[];
  FwdSmem<D>& sm =
      *reinterpret_cast<FwdSmem<D>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x / 32;

  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) {
      mbar_init(&sm.q_full[i], 1);
      mbar_init(&sm.q_empty[i], 8);  // lane 0 of each consumer warp
      mbar_init(&sm.fetch_full[i], 1);
    }
    for (int i = 0; i < NSLOT; ++i) {
      mbar_init(&sm.kv_full[i], 1);
      mbar_init(&sm.kv_empty[i], 8);
    }
    fence_mbar_init();
  }
  if (warp == 8 && lane_id() == 0) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_kv);
  }
  __syncthreads();

  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (warp == 8) {
      producer_role<D, DOCS, FP8>(sm, p, &map_q, &map_kv);
    } else if (warp == 10) {
      if (lane_id() == 0) fetch_role<D>(sm, p);
    }
  } else {
    setmaxnreg_inc<232>();
    consumer_role<D, BF16, DOCS, FP8, SINK>(sm, p, warp < 4 ? 0 : 1);
  }
}

template <int D, bool BF16, bool DOCS>
__global__ void __launch_bounds__(NTHREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                const __grid_constant__ AttnFwdParams p) {
  attn_fwd_body<D, BF16, DOCS, false>(map_q, map_kv, p);
}

// e4m3 operands, head dim 128, bf16 output
template <bool DOCS>
__global__ void __launch_bounds__(NTHREADS, 1)
attn_fwd_fp8_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                    const __grid_constant__ AttnFwdParams p) {
  attn_fwd_body<128, true, DOCS, true>(map_q, map_kv, p);
}

// attention sinks: the same bodies with the sink as initial softmax state (the kernels above keep their code)
template <int D, bool BF16, bool DOCS, bool FP8>
__global__ void __launch_bounds__(NTHREADS, 1)
attn_fwd_sink_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                     const __grid_constant__ AttnFwdParams p) {
  attn_fwd_body<D, BF16, DOCS, FP8, true>(map_q, map_kv, p);
}

}  // namespace

size_t attn_fwd_smem_bytes(int head_dim) {
  return (head_dim == 128 ? sizeof(FwdSmem<128>) : sizeof(FwdSmem<64>)) + 1024;
}

template <int D>
void launch_attn_fwd(const CUtensorMap& map_q, const CUtensorMap& map_kv, const AttnFwdParams& p, int num_sms,
                     cudaStream_t stream) {
  using Kern = void (*)(const CUtensorMap, const CUtensorMap, const AttnFwdParams);
  // documents are a separate instantiation: the default kernels keep their code unchanged
  Kern kern = p.doc_spans != nullptr ? (p.is_bf16 ? attn_fwd_kernel<D, true, true> : attn_fwd_kernel<D, false, true>)
                                     : (p.is_bf16 ? attn_fwd_kernel<D, true, false> : attn_fwd_kernel<D, false, false>);
  if (p.is_fp8) {
    if (D != 128) throw std::runtime_error("[ring_attention_b200] the fp8 forward needs head dim 128");
    kern = p.doc_spans != nullptr ? attn_fwd_fp8_kernel<true> : attn_fwd_fp8_kernel<false>;
  }
  if (p.sinks != nullptr) {
    if (p.is_fp8) {
      kern = p.doc_spans != nullptr ? attn_fwd_sink_kernel<128, true, true, true>
                                    : attn_fwd_sink_kernel<128, true, false, true>;
    } else if (p.doc_spans != nullptr) {
      kern = p.is_bf16 ? attn_fwd_sink_kernel<D, true, true, false> : attn_fwd_sink_kernel<D, false, true, false>;
    } else {
      kern = p.is_bf16 ? attn_fwd_sink_kernel<D, true, false, false> : attn_fwd_sink_kernel<D, false, false, false>;
    }
  }
  const size_t smem = sizeof(FwdSmem<D>) + 1024;
  cuda_check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
             "attn_fwd smem attribute");
  const int items = p.batch * p.heads * ((p.n_q + 2 * BM - 1) / (2 * BM));
  void* args[] = {(void*)&map_q, (void*)&map_kv, (void*)&p};
  if (p.hop_count > 1) {
    // every CTA owns a share of the NVLink fetch and other CTAs spin on it: all CTAs must be co-resident
    cuda_check(cudaLaunchCooperativeKernel((void*)kern, dim3(num_sms), dim3(NTHREADS), args, smem, stream),
               "attn_fwd cooperative launch");
  } else {
    const int grid = items < num_sms ? items : num_sms;
    cuda_check(cudaLaunchKernel((void*)kern, dim3(grid), dim3(NTHREADS), args, smem, stream), "attn_fwd launch");
  }
}

template void launch_attn_fwd<64>(const CUtensorMap&, const CUtensorMap&, const AttnFwdParams&, int, cudaStream_t);
template void launch_attn_fwd<128>(const CUtensorMap&, const CUtensorMap&, const AttnFwdParams&, int, cudaStream_t);

}  // namespace rab
