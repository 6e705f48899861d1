// Memory-bound helper kernels: K/V packing into the symmetric ring slot, the cross-device barrier on
// peer-mapped signal pads, and small conversion kernels used by the backward pass.
#include <cuda_fp16.h>

#include "attn_common.cuh"
#include "kernels.h"
#include "ptx.cuh"

namespace rab {
namespace {

// k, v: [b, n, hk, d] (strided, unit stride on d) -> slot: [2][b*hk][n][d] contiguous 16-bit.
// One thread moves 16 bytes.
__global__ void pack_kv_kernel(const uint16_t* __restrict__ k, const uint16_t* __restrict__ v,
                               uint16_t* __restrict__ slot, int batch, int n, int kv_heads, int d, long long k_sb,
                               long long k_sn, long long k_sh, long long v_sb, long long v_sn, long long v_sh,
                               int which) {
  const int vec_per_row = d / 8;
  const long long per_tensor = (long long)batch * kv_heads * n * vec_per_row;
  const long long lo = (which & 1) ? 0 : per_tensor, hi = (which & 2) ? 2 * per_tensor : per_tensor;
  for (long long i = lo + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < hi;
       i += (long long)gridDim.x * blockDim.x) {
    const int which = i >= per_tensor;
    long long r = which ? i - per_tensor : i;
    const int c = r % vec_per_row;
    r /= vec_per_row;
    const int row = r % n;
    r /= n;
    const int h = r % kv_heads;
    const int b = r / kv_heads;
    const uint16_t* src = which ? v + b * v_sb + row * v_sn + h * v_sh : k + b * k_sb + row * k_sn + h * k_sh;
    const uint4 val = *reinterpret_cast<const uint4*>(src + c * 8);
    reinterpret_cast<uint4*>(slot)[i] = val;
  }
}

// fp8 slot for the e4m3 forward (layout in kernels.h).  One block per (128-key tile, b*hk): K rows are copied through,
// V goes through shared memory and leaves transposed, in the key-slot order of v8_key_of_slot.  Keys past n are zero:
// e4m3 has NaN encodings and P = 0 times NaN would still poison O.
__global__ void pack_kv_fp8_kernel(const uint8_t* __restrict__ k, const uint8_t* __restrict__ v,
                                   uint8_t* __restrict__ slot, int batch, int n, int kv_heads, int n_pad,
                                   long long k_sb, long long k_sn, long long k_sh, long long v_sb, long long v_sn,
                                   long long v_sh) {
  __shared__ __align__(16) uint8_t vt[128][128 + 16];
  const int tile = blockIdx.x, bh = blockIdx.y;
  const int b = bh / kv_heads, h = bh % kv_heads;
  const size_t tile_off = ((size_t)bh * n_pad + (size_t)tile * 128) * 128;
  uint8_t* kdst = slot + tile_off;
  uint8_t* vdst = slot + (size_t)batch * kv_heads * n_pad * 128 + tile_off;
  for (int i = threadIdx.x; i < 128 * 8; i += blockDim.x) {
    const int r = i / 8, c = i % 8;
    const long long key = (long long)tile * 128 + r;
    uint4 kx = make_uint4(0, 0, 0, 0), vx = kx;
    if (key < n) {
      kx = *reinterpret_cast<const uint4*>(k + b * k_sb + key * k_sn + h * k_sh + c * 16);
      vx = *reinterpret_cast<const uint4*>(v + b * v_sb + key * v_sn + h * v_sh + c * 16);
    }
    reinterpret_cast<uint4*>(kdst)[i] = kx;
    *reinterpret_cast<uint4*>(&vt[r][c * 16]) = vx;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 128 * 8; i += blockDim.x) {
    const int dr = i % 128, c = i / 128;  // key slots [16 c, 16 c + 16) of V^T row dr
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t x = 0;
#pragma unroll
      for (int e = 0; e < 4; ++e) x |= uint32_t(vt[v8_key_of_slot(16 * c + 4 * j + e)][dr]) << (8 * e);
      w[j] = x;
    }
    reinterpret_cast<uint4*>(vdst + dr * 128)[c] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// Rotary position embedding fused with the layout change / head-dim padding that precedes the attention kernels.
// x: [b, n, h, d] 16 bit (arbitrary batch / seq / head strides, unit stride on d); angles: fp32 [n, >= d/2], row stride
// `astride` (the reference's rotary tensor is cat(freqs, freqs): only the first half is read).  Convention of
// reference ring_attention.py:160-172 (rotate_half): pairs (j, j + d/2):
//     out[j]       = x[j] cos a_j - sign * x[j + d/2] sin a_j
//     out[j + d/2] = x[j + d/2] cos a_j + sign * x[j] sin a_j          sign = +1 forward, -1 inverse (gradients)
// One thread owns a (batch, token, 8-column chunk pair) and walks the heads, so sincosf runs once per token and
// frequency instead of once per head.  Output element (b, row, head, col) lives at ob*b + on*row + oh*head + col:
// [b, n, h, d_pad] token-major for Q, the K half of the head-major gather slot for K.
template <bool BF16>
__global__ void rotary_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ out,
                              const float* __restrict__ angles, int astride, int batch, int n, int heads, int d,
                              long long sb, long long sn, long long sh, long long ob, long long on, long long oh,
                              float sign) {
  const int pairs = d / 16;
  const long long total = (long long)batch * n * pairs;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = i % pairs;
    const int row = (i / pairs) % n;
    const int b = i / ((long long)pairs * n);
    float cs[8], sn_[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      sincosf(angles[(long long)row * astride + c * 8 + j], &sn_[j], &cs[j]);
      sn_[j] *= sign;
    }
    const uint16_t* src = x + b * sb + row * sn;
    uint16_t* dst = out + b * ob + row * on;
    for (int hh = 0; hh < heads; ++hh) {
      const uint4 lo = *reinterpret_cast<const uint4*>(src + hh * sh + c * 8);
      const uint4 hi = *reinterpret_cast<const uint4*>(src + hh * sh + d / 2 + c * 8);
      const uint32_t lw[4] = {lo.x, lo.y, lo.z, lo.w}, hw[4] = {hi.x, hi.y, hi.z, hi.w};
      uint32_t ol[4], oh_[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float a0, a1, b0, b1;
        if (BF16) {
          a0 = __uint_as_float(lw[e] << 16); a1 = __uint_as_float(lw[e] & 0xffff0000u);
          b0 = __uint_as_float(hw[e] << 16); b1 = __uint_as_float(hw[e] & 0xffff0000u);
        } else {
          const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&lw[e]));
          const float2 fb = __half22float2(*reinterpret_cast<const __half2*>(&hw[e]));
          a0 = fa.x; a1 = fa.y; b0 = fb.x; b1 = fb.y;
        }
        const float r0 = a0 * cs[2 * e] - b0 * sn_[2 * e], r1 = a1 * cs[2 * e + 1] - b1 * sn_[2 * e + 1];
        const float t0 = b0 * cs[2 * e] + a0 * sn_[2 * e], t1 = b1 * cs[2 * e + 1] + a1 * sn_[2 * e + 1];
        ol[e] = BF16 ? pack_bf16x2(r0, r1) : pack_f16x2(r0, r1);
        oh_[e] = BF16 ? pack_bf16x2(t0, t1) : pack_f16x2(t0, t1);
      }
      *reinterpret_cast<uint4*>(dst + hh * oh + c * 8) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
      *reinterpret_cast<uint4*>(dst + hh * oh + d / 2 + c * 8) = make_uint4(oh_[0], oh_[1], oh_[2], oh_[3]);
    }
  }
}

__global__ void device_barrier_kernel(const __grid_constant__ BarrierParams p) {
  const int peer = threadIdx.x;
  if (peer >= p.world) return;
  if (peer != p.rank) {
    __threadfence_system();
    st_release_sys(p.pads[peer] + p.rank, p.epoch);
    const uint32_t* mine = p.pads[p.rank] + peer;
    const long long t0 = clock64();
    while ((int32_t)(ld_acquire_sys(mine) - p.epoch) < 0) {
      __nanosleep(100);
      // ranks may reach their first barrier seconds apart (lazy module loading, allocator warm-up): be generous
      if (clock64() - t0 > 8 * RAB_WATCHDOG_CYCLES) {
        printf("[rab] device barrier watchdog: rank %d waiting for %d epoch %u (have %u)\n", p.rank, peer, p.epoch,
               ld_acquire_sys(mine));
        __trap();
      }
    }
  }
}

}  // namespace

void launch_pack_kv(const void* k, const void* v, void* slot, int batch, int n, int kv_heads, int d, long long k_sb,
                    long long k_sn, long long k_sh, long long v_sb, long long v_sn, long long v_sh, int which,
                    cudaStream_t stream) {
  const long long vecs = ((which & 1) + ((which >> 1) & 1)) * (long long)batch * kv_heads * n * (d / 8);
  if (vecs == 0) return;
  const int threads = 256;
  long long blocks = (vecs + threads - 1) / threads;
  if (blocks > 132 * 16) blocks = 132 * 16;
  pack_kv_kernel<<<(int)blocks, threads, 0, stream>>>(
      reinterpret_cast<const uint16_t*>(k), reinterpret_cast<const uint16_t*>(v), reinterpret_cast<uint16_t*>(slot),
      batch, n, kv_heads, d, k_sb, k_sn, k_sh, v_sb, v_sn, v_sh, which);
  cuda_check(cudaGetLastError(), "pack_kv launch");
}

void launch_pack_kv_fp8(const void* k, const void* v, void* slot, int batch, int n, int kv_heads, long long k_sb,
                        long long k_sn, long long k_sh, long long v_sb, long long v_sn, long long v_sh,
                        cudaStream_t stream) {
  const int n_pad = (n + 127) / 128 * 128;
  if (n_pad == 0 || batch * kv_heads == 0) return;
  pack_kv_fp8_kernel<<<dim3(n_pad / 128, batch * kv_heads), 256, 0, stream>>>(
      reinterpret_cast<const uint8_t*>(k), reinterpret_cast<const uint8_t*>(v), reinterpret_cast<uint8_t*>(slot), batch,
      n, kv_heads, n_pad, k_sb, k_sn, k_sh, v_sb, v_sn, v_sh);
  cuda_check(cudaGetLastError(), "pack_kv_fp8 launch");
}

void launch_rotary(const void* x, void* out, const float* angles, int astride, int batch, int n, int heads, int d,
                   long long sb, long long sn, long long sh, long long ob, long long on, long long oh, float sign,
                   int is_bf16, cudaStream_t stream) {
  const long long total = (long long)batch * n * (d / 16);
  if (total == 0) return;
  const int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  if (blocks > 132 * 16) blocks = 132 * 16;
  auto kern = is_bf16 ? rotary_kernel<true> : rotary_kernel<false>;
  kern<<<(int)blocks, threads, 0, stream>>>(reinterpret_cast<const uint16_t*>(x), reinterpret_cast<uint16_t*>(out), angles,
                                            astride, batch, n, heads, d, sb, sn, sh, ob, on, oh, sign);
  cuda_check(cudaGetLastError(), "rotary launch");
}

void launch_device_barrier(const BarrierParams& p, cudaStream_t stream) {
  device_barrier_kernel<<<1, 32, 0, stream>>>(p);
  cuda_check(cudaGetLastError(), "device_barrier launch");
}

}  // namespace rab
