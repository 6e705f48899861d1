// Shared device-side helpers for the attention kernels: position maps, tile classification and the
// deterministic per-work-item KV tile schedule that every warp role replays independently.
#pragma once
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
// Warp-cooperative tile scanner.
//
// Every warp role (TMA producer, MMA issuer, softmax warps) replays the same deterministic sequence of
// streamed tiles.  Classifying tiles one at a time on a single thread puts ~100 dependent instructions
// between two MMA issues; here the 32 lanes of a warp classify 32 tiles at once and publish the
// result as ballot masks, so advancing to the next visible tile is a find-first-set.
//
// Sequence order: repeat `groups` times { for hop s in [0, hop_count) { tiles ascending } }.
// All 32 lanes must call next() convergently; the scanner state is warp-uniform.
// ------------------------------------------------------------------------------------------------
struct StatRange {
  int lo, hi;   // position range of the stationary tile
  bool valid;   // false: the stationary tile does not exist (e.g. second Q tile beyond n_q)
  bool tail;    // the stationary tile is ragged (forces per-element masking)
};

struct ScanTile {
  int rep;       // group repetition index
  int owner;     // ring rank that owns the streamed tile
  int idx;       // tile index inside the owner's shard
  bool need[2];
  bool part[2];
};

template <int NSTAT, bool STREAM_IS_Q>
struct WarpTileScan {
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
