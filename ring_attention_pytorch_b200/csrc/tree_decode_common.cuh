// Shared pieces of the tree-decode kernels (the CUDA-core split-KV kernel): query loads, the
// multimem (NVLS) wrappers, the grid barrier, and the cross-rank part of a decode step (publish -> signal -> merge).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "kernels.h"
#include "ptx.cuh"

namespace rab {

__device__ __forceinline__ float load_q(const void* q, int kind, size_t idx) {
  if (kind == 0) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(q)[idx]);
  if (kind == 1) return __half2float(reinterpret_cast<const __half*>(q)[idx]);
  return reinterpret_cast<const float*>(q)[idx];
}

// Ranged decode: the keys unit (b, split) covers, [k0, k1), and the first visible key lo (keys in [k0, lo) are masked).
// Tiles start at lo rounded down to a multiple of TILE, so they stay aligned with the scale blocks of an fp8 cache.
// MULTI: the union of the visible ranges of the p.tokens query tokens (lo from the first token, hi from the last).
struct TdUnitRange {
  int lo, k0, k1;
};
__device__ __forceinline__ long long td_floor_div(long long a, long long b) {  // b > 0, any sign of a
  return a >= 0 ? a / b : -((-a + b - 1) / b);
}
template <int TILE, bool MULTI = false>
__device__ __forceinline__ TdUnitRange td_unit_range(const TreeDecodeParams& p, int b, int split) {
  long long lo = 0, hi = p.n;
  if (p.cache_seqlens != nullptr) hi = min(hi, (long long)p.cache_seqlens[b]);
  long long span = p.n;  // the most keys (with tile slack) one sequence's visible range can touch
  if (p.q_pos != nullptr) {
    const long long rel = (long long)p.q_pos[b] - p.kv_pos_offset;  // negative: every key here lies after the query
    const long long last = MULTI ? (long long)p.tokens - 1 : 0;        // the last token sits at q_pos + last
    hi = min(hi, td_floor_div(rel + last, p.kv_pos_stride) + 1);      // P(j) <= q_pos (+ last)
    if (p.window > 0) {
      lo = max(lo, -td_floor_div((long long)p.window - rel, p.kv_pos_stride));  // q_pos - P(j) <= window
      span = min(span, ((long long)p.window + last) / p.kv_pos_stride + TILE);
    }
  }
  lo = min(lo, (long long)p.n);
  const long long per = ((span + p.splits - 1) / p.splits + TILE - 1) / TILE * TILE;
  TdUnitRange r;
  r.lo = (int)lo;
  r.k0 = (int)min((lo & ~(long long)(TILE - 1)) + split * per, (long long)p.n);
  r.k1 = lo < hi ? (int)max(min(hi, (long long)r.k0 + per), (long long)r.k0) : r.k0;
  return r;
}

// Multi-token decode: the keys of [lo, k1) (a unit's range) that token t sees, [clo, chi) (empty when chi <= clo).
struct TdColRange {
  int lo, hi;
};
__device__ __forceinline__ TdColRange td_col_range(const TreeDecodeParams& p, int b, int t, int lo, int k1) {
  long long clo = lo, chi = k1;
  if (p.q_pos != nullptr) {
    const long long rel = (long long)p.q_pos[b] + t - p.kv_pos_offset;
    chi = min(chi, td_floor_div(rel, p.kv_pos_stride) + 1);
    if (p.window > 0) clo = max(clo, -td_floor_div((long long)p.window - rel, p.kv_pos_stride));
  }
  TdColRange r;
  r.lo = (int)min(clo, (long long)k1);
  r.hi = (int)max(chi, (long long)lo);
  return r;
}

// order-preserving map fp32 -> int32 (so that an integer max is the float max); used for the in-switch max
__device__ __forceinline__ int float_to_ordered(float f) {
  const int i = __float_as_int(f);
  return i ^ ((i >> 31) & 0x7fffffff);
}
__device__ __forceinline__ float ordered_to_float(int i) { return __int_as_float(i ^ ((i >> 31) & 0x7fffffff)); }

__device__ __forceinline__ float4 multimem_add_f32x4(const float* mc_addr) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(mc_addr)
               : "memory");
  return r;
}
__device__ __forceinline__ float multimem_add_f32(const float* mc_addr) {
  float r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.f32 %0, [%1];" : "=f"(r) : "l"(mc_addr) : "memory");
  return r;
}
__device__ __forceinline__ int multimem_max_s32(const int* mc_addr) {
  int r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.max.s32 %0, [%1];" : "=r"(r) : "l"(mc_addr) : "memory");
  return r;
}

// sense-reversing grid barrier on two words of device memory (all CTAs are co-resident: cooperative launch)
__device__ __forceinline__ void grid_barrier(uint32_t* count, uint32_t* gen) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t my_gen = ld_acquire_gpu(gen);
    __threadfence();
    if (atomicAdd(count, 1u) == gridDim.x - 1) {
      *count = 0;
      __threadfence();
      red_release_gpu_add(gen, 1u);
    } else {
      const long long t0 = clock64();
      while (ld_acquire_gpu(gen) == my_gen) {
        if (clock64() - t0 > RAB_WATCHDOG_CYCLES) watchdog_trap(1700);
      }
    }
  }
  __syncthreads();
}

// State every thread derives from the launch parameters: which half of the double-buffered symmetric buffers this call
// uses and the epoch it signals with.  MULTI: rows are (batch, head, token), b * h * tokens of them.
template <int D, bool MULTI = false>
struct TdCall {
  static constexpr int row_stride = D + 4;  // (out[D], lse2, valid, pad, pad): rows stay 16-byte aligned
  uint32_t base;
  size_t half_off, aux_off;
  float* my_partial;
  float* my_aux;
  __device__ __forceinline__ void init(const TreeDecodeParams& p) {
    // The cross-rank epoch lives in device memory (graph replays advance it).  Calls alternate between two halves of the
    // symmetric buffers: a half is rewritten two calls later, after every peer has signalled a round it can only reach
    // once its reads of that half are complete.
    base = ld_acquire_gpu(&p.counters[3]);  // block 0 advances it behind the last grid barrier
    const bool nvls_cfg = p.mc_partial != nullptr && p.world > 1;
    const uint32_t call = nvls_cfg ? (base >> 1) : base;
    if constexpr (MULTI) {
      half_off = (size_t)(call & 1u) * (size_t)p.batch * p.heads * p.tokens * row_stride;
      aux_off = (size_t)(call & 1u) * (size_t)p.batch * p.heads * p.tokens * 2;
    } else {
      half_off = (size_t)(call & 1u) * (size_t)p.batch * p.heads * row_stride;
      aux_off = (size_t)(call & 1u) * (size_t)p.batch * p.heads * 2;
    }
    my_partial = p.partial_local + half_off;
    my_aux = p.aux_local + aux_off;
  }
};

// Phases 2 and 3 of a decode step; every thread of every CTA of the (cooperative) grid calls it after its last unit.
template <int D, bool MULTI = false>
__device__ __forceinline__ void td_cross_rank_merge(const TreeDecodeParams& p, const TdCall<D, MULTI>& cs,
                                                    int total_units) {
  constexpr int row_stride = TdCall<D, MULTI>::row_stride;
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int nthreads = blockDim.x;
  uint32_t* const ctr = p.counters;
  const uint32_t base = cs.base;
  const size_t half_off = cs.half_off, aux_off = cs.aux_off;
  float* const my_partial = cs.my_partial;
  float* const my_aux = cs.my_aux;
  if (total_units == 0) {  // this rank holds no keys: publish empty rows
    for (int i = blockIdx.x * nthreads + tid; i < (MULTI ? p.batch * p.heads * p.tokens : p.batch * p.heads);
         i += gridDim.x * nthreads) {
      my_partial[(size_t)i * row_stride + D] = -INFINITY;
      my_partial[(size_t)i * row_stride + D + 1] = 0.f;
    }
  }

  // ====================================== phase 2: everyone's partials are visible ====================================
  __threadfence();
  grid_barrier(&ctr[1], &ctr[2]);
  const int rows = MULTI ? p.batch * p.heads * p.tokens : p.batch * p.heads;
  const int gwarp = blockIdx.x * (nthreads / 32) + warp, nwarps = gridDim.x * (nthreads / 32);
  const bool nvls = p.mc_partial != nullptr && p.world > 1;
  int* const my_ord = reinterpret_cast<int*>(my_aux);  // [rows] order-preserving integer image of this rank's lse
  float* const my_w = my_aux + rows;                    // [rows] weight of this rank (NVLS path)
  if (nvls) {
    for (int bh = gwarp * 32 + lane; bh < rows; bh += nwarps * 32)
      my_ord[bh] = float_to_ordered(my_partial[(size_t)bh * row_stride + D]);
    __threadfence();
    grid_barrier(&ctr[1], &ctr[2]);
  }
  // One signal round: block 0 tells every peer "my rows of this epoch are complete", then every CTA waits until all
  // peers have said the same on THIS rank's pad (local memory: polling it costs no NVLink traffic).
  auto signal_round = [&](int round, uint32_t epoch) {
    if (p.world <= 1) return;
    if (blockIdx.x == 0 && tid < p.world && tid != p.rank) {
      __threadfence_system();
      st_release_sys(p.pads[tid] + round * kMaxWorld + p.rank, epoch);
    }
    if (tid < p.world && tid != p.rank) {
      const uint32_t* mine = p.pads[p.rank] + round * kMaxWorld + tid;
      const long long t0 = clock64();
      while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) {
        if (clock64() - t0 > 8 * RAB_WATCHDOG_CYCLES) watchdog_trap(1710 + round);
      }
    }
    __syncthreads();
  };
  signal_round(0, base + 1);

  // ================================================ phase 3: merge ====================================================
  auto store_row = [&](int bh, int c, float4 o) {
    if (p.out_kind == 2) {
      reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + (size_t)bh * D)[c] = o;
    } else {
      uint2 w;
      w.x = p.out_kind == 1 ? pack_bf16x2(o.x, o.y) : pack_f16x2(o.x, o.y);
      w.y = p.out_kind == 1 ? pack_bf16x2(o.z, o.w) : pack_f16x2(o.z, o.w);
      reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(p.out) + (size_t)bh * D)[c] = w;
    }
  };
  const bool own = lane * 4 < D;  // one warp per row; lane c owns columns [4c, 4c + 4)
  // attention sink of row bh in log2 units: one more term of the merged denominator, with a zero value vector
  auto sink2 = [&](int bh) { return p.sinks[(MULTI ? bh / p.tokens : bh) % p.heads] * 1.4426950408889634f; };
  if (!nvls) {
    // P2P: every rank reads every peer's row straight over NVLink
    for (int bh = gwarp; bh < rows; bh += nwarps) {
      float lse[kMaxWorld];
      float mx = -INFINITY;
#pragma unroll 1
      for (int r = 0; r < p.world; ++r) {
        lse[r] = (p.partials[r] + half_off)[(size_t)bh * row_stride + D];
        mx = fmaxf(mx, lse[r]);
      }
      const float sg = p.sinks != nullptr ? sink2(bh) : -INFINITY;
      mx = fmaxf(mx, sg);
      const float m_eff = mx == -INFINITY ? 0.f : mx;
      float den = p.sinks != nullptr ? fast_exp2(sg - m_eff) : 0.f;
      float4 num = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
      for (int r = 0; r < p.world; ++r) {
        if (lse[r] == -INFINITY) continue;
        const float wgt = fast_exp2(lse[r] - m_eff);
        den += wgt;
        if (own) {
          const float4 x = reinterpret_cast<const float4*>(p.partials[r] + half_off + (size_t)bh * row_stride)[lane];
          num.x += wgt * x.x; num.y += wgt * x.y; num.z += wgt * x.z; num.w += wgt * x.w;
        }
      }
      if (own) {
        const float inv = 1.f / fmaxf(den, p.eps);
        store_row(bh, lane, make_float4(num.x * inv, num.y * inv, num.z * inv, num.w * inv));
      }
    }
  } else {
    // NVLS: the switch returns M = max_r lse_r (integer max of the order-preserving image); every rank rescales ITS
    // rows in place by w_r = 2^(lse_r - M) and publishes w_r; after a second signal round the switch returns
    // sum_r w_r out_r and sum_r w_r.  With sinks every rank raises M to max(M, sink) first, and rank 0 publishes
    // w_0 + 2^(sink - M), so the summed denominator holds the sink exactly once.
    const int* mc_ord = reinterpret_cast<const int*>(p.mc_aux + aux_off);
    for (int bh = gwarp; bh < rows; bh += nwarps) {
      float M = ordered_to_float(multimem_max_s32(mc_ord + bh));
      const float sg = p.sinks != nullptr ? sink2(bh) : -INFINITY;
      M = fmaxf(M, sg);
      const float m_eff = M == -INFINITY ? 0.f : M;
      float* row = my_partial + (size_t)bh * row_stride;
      const float l = row[D];
      const float wgt = l == -INFINITY ? 0.f : fast_exp2(l - m_eff);
      if (own) {
        float4 x = reinterpret_cast<float4*>(row)[lane];
        x.x *= wgt; x.y *= wgt; x.z *= wgt; x.w *= wgt;
        reinterpret_cast<float4*>(row)[lane] = x;
      }
      if (lane == 0) my_w[bh] = (p.sinks != nullptr && p.rank == 0) ? wgt + fast_exp2(sg - m_eff) : wgt;
    }
    __threadfence();
    grid_barrier(&ctr[1], &ctr[2]);
    signal_round(1, base + 2);
    const float* mc_w = p.mc_aux + aux_off + rows;
    const float* mc_rows = p.mc_partial + half_off;
    for (int bh = gwarp; bh < rows; bh += nwarps) {
      const float den = multimem_add_f32(mc_w + bh);
      if (own) {
        const float4 num = multimem_add_f32x4(mc_rows + (size_t)bh * row_stride + lane * 4);
        const float inv = 1.f / fmaxf(den, p.eps);
        store_row(bh, lane, make_float4(num.x * inv, num.y * inv, num.z * inv, num.w * inv));
      }
    }
  }
  // every CTA is done with the queue and has used `base`: reset / advance them for the next launch (graph replay safe)
  grid_barrier(&ctr[1], &ctr[2]);
  if (blockIdx.x == 0 && tid == 0) {
    ctr[0] = 0;
    ctr[3] = base + (nvls ? 2u : 1u);
  }
}

}  // namespace rab
