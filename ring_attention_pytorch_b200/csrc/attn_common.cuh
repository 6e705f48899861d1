// Shared device-side helpers for the attention kernels: position maps, tile classification and the
// deterministic per-work-item KV tile schedule that every warp role replays independently.
#pragma once
#include <climits>

#include "kernels.h"
#include "ptx.cuh"

namespace rab {

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// position of local index i on ring rank r
__device__ __forceinline__ int pos_of(const PosMap& pm, int r, int i) {
  return i < pm.seg_len ? pm.base0[r] + pm.stride * i : pm.base1[r] + pm.stride * (i - pm.seg_len);
}

// [lo, hi] position range covered by local indices a..b (inclusive) on ring rank r
__device__ __forceinline__ void pos_range(const PosMap& pm, int r, int a, int b, int& lo, int& hi) {
  if (b < pm.seg_len) {
    lo = pm.base0[r] + pm.stride * a;
    hi = pm.base0[r] + pm.stride * b;
  } else if (a >= pm.seg_len) {
    lo = pm.base1[r] + pm.stride * (a - pm.seg_len);
    hi = pm.base1[r] + pm.stride * (b - pm.seg_len);
  } else {
    const int lo0 = pm.base0[r] + pm.stride * a, hi0 = pm.base0[r] + pm.stride * (pm.seg_len - 1);
    const int lo1 = pm.base1[r], hi1 = pm.base1[r] + pm.stride * (b - pm.seg_len);
    lo = min(lo0, lo1);
    hi = max(hi0, hi1);
  }
}

// ------------------------------------------------------------------------------------------------
// fp8 (e4m3) forward: key order of the V^T operand.
//
// Inside each 32-key group, lane quad q (= lane % 4) holds the fp32 S accumulator columns {2q, 2q+1, 8+2q, 9+2q, 16+2q,
// 17+2q, 24+2q, 25+2q} of its rows, while the e4m3 A operand of m64nNk32 wants columns {4q..4q+3, 16+4q..16+4q+3}.
// Rather than shuffling P between lanes, the consumer feeds its S values in register order as A columns, and the
// V^T tile stores at key slot kappa the key v8_key_of_slot(kappa), so that sum_kappa P_A[kappa] V^T[kappa] is
// sum_key P[key] V[key].  ops/ring_fp8.py mirrors this map for the tests.
// ------------------------------------------------------------------------------------------------
__host__ __device__ constexpr int v8_key_of_slot(int kappa) {
  return (kappa & ~31) + 16 * ((kappa >> 4) & 1) + 8 * ((kappa >> 1) & 1) + 2 * ((kappa >> 2) & 3) + (kappa & 1);
}

// Mask parameters shared by forward and backward kernels.
struct MaskCfg {
  int causal;
  int window;
  int has_kmask;
};

// need: at least one (q, k) pair of the tile pair may be visible.  partial: per-element masking required.
__device__ __forceinline__ void classify_tile(const MaskCfg& mc, int qlo, int qhi, int klo, int khi, bool k_tail,
                                              bool& need, bool& partial) {
  need = true;
  partial = k_tail || mc.has_kmask;
  if (mc.causal) {
    if (klo > qhi) {
      need = false;
    } else if (khi > qlo) {
      partial = true;
    }
    if (mc.window > 0) {
      if (qlo - khi > mc.window) {
        need = false;
      } else if (qhi - klo > mc.window) {
        partial = true;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Document masking (packed sequences).  spans: int32 [world][batch][n][2], the half-open interval
// [start, end) of global positions of the document holding local token i of ring rank r (built by
// parallel/documents.py).  q and k share a document iff pos(k) lies in q's interval iff pos(q) lies in
// k's, so a kernel only needs the intervals of its stationary rows.
// ------------------------------------------------------------------------------------------------
struct DocRange {
  int min_s, max_s;  // min / max document start over the stationary tile's rows
  int min_e, max_e;  // min / max document end
};

__device__ __forceinline__ const int2* doc_row_spans(const int* spans, int batch, int n, int r, int b) {
  return reinterpret_cast<const int2*>(spans) + ((size_t)r * batch + b) * n;
}

// Summary of the intervals of rows [a, last] (inclusive).  All 32 lanes call it convergently.
__device__ __forceinline__ DocRange doc_range(const int2* rows, int a, int last, int lane) {
  int mn_s = INT_MAX, mx_s = INT_MIN, mn_e = INT_MAX, mx_e = INT_MIN;
  for (int i = a + lane; i <= last; i += 32) {
    const int2 s = rows[i];
    mn_s = min(mn_s, s.x);
    mx_s = max(mx_s, s.x);
    mn_e = min(mn_e, s.y);
    mx_e = max(mx_e, s.y);
  }
  return DocRange{__reduce_min_sync(0xffffffffu, mn_s), __reduce_max_sync(0xffffffffu, mx_s),
                  __reduce_min_sync(0xffffffffu, mn_e), __reduce_max_sync(0xffffffffu, mx_e)};
}

// Streamed positions [lo, hi] against the stationary rows' intervals: skip when no row's document can reach the
// range, per-element masking unless every row's document covers all of it.
__device__ __forceinline__ void classify_doc(const DocRange& d, int lo, int hi, bool& need, bool& partial) {
  if (hi < d.min_s || lo >= d.max_e) {
    need = false;
  } else if (!(d.max_s <= lo && hi < d.min_e)) {
    partial = true;
  }
}

// ------------------------------------------------------------------------------------------------
// Warp-cooperative tile scanner.
//
// Every warp role (TMA producer, MMA issuer, softmax warps) replays the same deterministic sequence of
// streamed tiles.  Classifying tiles one at a time on a single thread puts ~100 dependent instructions
// between two MMA issues; here the 32 lanes of a warp classify 32 tiles at once and publish the
// result as ballot masks, so advancing to the next visible tile is a find-first-set.
//
// Sequence order: repeat `groups` times { for hop s in [0, hop_count) { tiles ascending } }.
// All 32 lanes must call next() convergently; the scanner state is warp-uniform.
// DOCS: the stationary tiles also carry a DocRange (doc[i]) and streamed tiles are classified against it.
// ------------------------------------------------------------------------------------------------
struct StatRange {
  int lo, hi;   // position range of the stationary tile
  bool valid;   // false: the stationary tile does not exist (e.g. second Q tile beyond n_q)
  bool tail;    // the stationary tile is ragged (forces per-element masking)
};

// Document summaries of the stationary tiles; empty (and so absent from the default scanners) without documents.
template <int NSTAT, bool DOCS>
struct ScanDocs {
  DocRange doc[NSTAT];
};
template <int NSTAT>
struct ScanDocs<NSTAT, false> {};

struct ScanTile {
  int rep;       // group repetition index
  int owner;     // ring rank that owns the streamed tile
  int idx;       // tile index inside the owner's shard
  bool need[2];
  bool part[2];
};

template <int NSTAT, bool STREAM_IS_Q, bool DOCS = false>
struct WarpTileScan : ScanDocs<NSTAT, DOCS> {
  const PosMap* pm;
  const int* hop_owner;
  int hop_count, groups;
  int n_stream, tile, stream_off, stat_off;
  MaskCfg mc;
  StatRange st[NSTAT];
  // iteration state (warp-uniform)
  int rep = 0, s = 0, base = 0;
  uint32_t need[NSTAT], part[NSTAT], any = 0;
  bool primed = false;

  __device__ __forceinline__ void load_chunk(int lane) {
    const int o = hop_owner[s];
    const int t = base + lane;
    const int nt = (n_stream + tile - 1) / tile;
    bool nd[NSTAT], pt[NSTAT];
#pragma unroll
    for (int i = 0; i < NSTAT; ++i) nd[i] = pt[i] = false;
    if (t < nt) {
      const int a = t * tile, b = min(a + tile, n_stream) - 1;
      int lo, hi;
      pos_range(*pm, o, a, b, lo, hi);
      lo += stream_off;
      hi += stream_off;
      const bool tail = (a + tile) > n_stream;
#pragma unroll
      for (int i = 0; i < NSTAT; ++i) {
        if (st[i].valid) {
          if (STREAM_IS_Q) {
            classify_tile(mc, lo, hi, st[i].lo + stat_off, st[i].hi + stat_off, tail || st[i].tail, nd[i], pt[i]);
          } else {
            classify_tile(mc, st[i].lo + stat_off, st[i].hi + stat_off, lo, hi, tail || st[i].tail, nd[i], pt[i]);
          }
          if constexpr (DOCS) classify_doc(this->doc[i], lo, hi, nd[i], pt[i]);
        }
      }
    }
    any = 0;
#pragma unroll
    for (int i = 0; i < NSTAT; ++i) {
      need[i] = __ballot_sync(0xffffffffu, nd[i]);
      part[i] = __ballot_sync(0xffffffffu, pt[i]);
      any |= need[i];
    }
  }

  // Number of tiles next() will hand out.  Call on a freshly initialised scanner only (state is reset afterwards).
  __device__ __forceinline__ uint32_t count(int lane) {
    const int nt = (n_stream + tile - 1) / tile;
    uint32_t c = 0;
    for (s = 0; s < hop_count; ++s) {
      for (base = 0; base < nt; base += 32) {
        load_chunk(lane);
        c += __popc(any);
      }
    }
    s = 0;
    base = 0;
    any = 0;
    rep = 0;
    primed = false;
    return c * (uint32_t)groups;
  }

  __device__ __forceinline__ bool next(int lane, ScanTile& t) {
    const int nt = (n_stream + tile - 1) / tile;
    while (true) {
      if (!primed) {
        if (rep >= groups) return false;
        load_chunk(lane);
        primed = true;
      }
      if (any) {
        const int bit = __ffs(any) - 1;
        any &= any - 1;
        t.rep = rep;
        t.owner = hop_owner[s];
        t.idx = base + bit;
#pragma unroll
        for (int i = 0; i < NSTAT; ++i) {
          t.need[i] = (need[i] >> bit) & 1u;
          t.part[i] = (part[i] >> bit) & 1u;
        }
        return true;
      }
      primed = false;
      base += 32;
      if (base >= nt) {
        base = 0;
        if (++s >= hop_count) {
          s = 0;
          ++rep;
        }
      }
    }
  }
};

}  // namespace rab
