// torch.ops.rab.* bindings.  Only this file sees torch headers.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/torch.h>

#include <vector>

#include "kernels.h"
#include "symm.h"

namespace {

using torch::Tensor;

int sm_count() {
  static int n = [] {
    int dev = 0, v = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v;
  }();
  return n;
}

// bench.py hook: when set, the next forward launches record the activity window of their in-kernel K/V fetchers
unsigned long long* g_fetch_times = nullptr;
int64_t g_fetch_times_rows = 0;

void set_fetch_timing(const c10::optional<Tensor>& t) {
  if (!t.has_value()) {
    g_fetch_times = nullptr;
    g_fetch_times_rows = 0;
    return;
  }
  TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kLong && t->is_contiguous() && t->dim() == 2 && t->size(1) == 2);
  g_fetch_times = reinterpret_cast<unsigned long long*>(t->data_ptr<int64_t>());
  g_fetch_times_rows = t->size(0);
}

void check_16bit(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.scalar_type() == at::kBFloat16 || t.scalar_type() == at::kHalf, name, " must be bf16 or fp16");
}

// ---------------------------------------------------------------------------------------------
// fused ring attention forward
// ---------------------------------------------------------------------------------------------
void fill_posmap(rab::PosMap& pm, int64_t stride, int64_t seg_len, at::IntArrayRef base0, at::IntArrayRef base1,
                 int world) {
  pm.stride = (int)stride;
  pm.seg_len = (int)seg_len;
  TORCH_CHECK((int)base0.size() == world && (int)base1.size() == world, "position map needs one base per rank");
  for (int i = 0; i < rab::kMaxWorld; ++i) {
    pm.base0[i] = i < world ? (int)base0[i] : 0;
    pm.base1[i] = i < world ? (int)base1[i] : 0;
  }
}

// Document intervals int32 [world, b, n, 2] (parallel/documents.py), or null: document masking off.
const int* doc_spans_ptr(const c10::optional<Tensor>& spans, int world, int batch, int n_q, int n_k,
                         int64_t q_pos_offset) {
  if (!spans.has_value()) return nullptr;
  const Tensor& t = *spans;
  TORCH_CHECK(n_q == n_k && q_pos_offset == 0, "document masking needs self-attention (n_q == n_k)");
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kInt && t.is_contiguous() && t.dim() == 4 && t.size(0) == world &&
                  t.size(1) == batch && t.size(2) == n_k && t.size(3) == 2,
              "doc_spans must be contiguous int32 [world, b, n, 2]");
  return t.data_ptr<int>();
}

// Hop mode (memory = "ring"): kv_buf holds ONE owner's slot ([1, 2, b*hk, n_k, d]); the launch visits that owner only
// and carries the online-softmax state (un-normalised O, running max / sum) in fp32 buffers between launches.
struct FwdHop {
  int owner = -1;        // -1: single-launch mode
  int world = 0;
  float* carry_o = nullptr;
  float* carry_ml = nullptr;
  bool carry_in = false, carry_out = false;
};

// fp8 forward (attn_fwd_fp8 / attn_fwd_hop_fp8): e4m3 q, uint8 K/V slots of pack_kv_fp8 ([.., 2, b*hk, n_pad, 128]), the
// true key count and the fp32 descales.
struct FwdFp8 {
  int64_t n_k = 0;
  const Tensor* q_descale = nullptr;
  const Tensor* k_descale = nullptr;
  const Tensor* v_descale = nullptr;
};

const float* descale_ptr(const Tensor& t, int64_t numel, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous() && t.numel() == numel, name,
              " must be a contiguous fp32 CUDA tensor of ", numel, " elements");
  return t.data_ptr<float>();
}

// Attention sinks fp32 [heads] (natural-log logits, by query head), or null: no sink.
const float* sinks_ptr(const c10::optional<Tensor>& sinks, int64_t heads, const Tensor& like) {
  if (!sinks.has_value()) return nullptr;
  const Tensor& t = *sinks;
  TORCH_CHECK(t.is_cuda() && t.device() == like.device() && t.scalar_type() == at::kFloat && t.is_contiguous() &&
                  t.dim() == 1 && t.size(0) == heads,
              "sinks must be a contiguous fp32 CUDA tensor [", heads, "] on the device of q");
  return t.data_ptr<float>();
}

std::tuple<Tensor, Tensor> attn_fwd_impl(const Tensor& q, const Tensor& kv_buf, at::IntArrayRef peer_ptrs,
                                         const c10::optional<Tensor>& ready_opt,
                                         const c10::optional<Tensor>& kmask_bits, int64_t kv_heads, int64_t rank,
                                         bool causal, int64_t window, double scale, double softclamp,
                                         int64_t pos_stride, int64_t seg_len, at::IntArrayRef base0,
                                         at::IntArrayRef base1, int64_t q_pos_offset, at::IntArrayRef hop_owner,
                                         const FwdHop& hop, const c10::optional<Tensor>& doc_spans,
                                         const c10::optional<Tensor>& sinks, const FwdFp8* fp8 = nullptr) {
  if (fp8 != nullptr) {
    TORCH_CHECK(q.is_cuda() && q.scalar_type() == at::kFloat8_e4m3fn, "q must be a float8_e4m3fn CUDA tensor");
    TORCH_CHECK(kv_buf.is_cuda() && kv_buf.scalar_type() == at::kByte, "kv_buf must be the uint8 slot of pack_kv_fp8");
  } else {
    check_16bit(q, "q");
    check_16bit(kv_buf, "kv_buf");
    TORCH_CHECK(kv_buf.scalar_type() == q.scalar_type());
  }
  const bool hop_mode = hop.owner >= 0;
  TORCH_CHECK(q.dim() == 4 && q.is_contiguous(), "q must be contiguous [b, n, h, d]");
  TORCH_CHECK(kv_buf.dim() == 5 && kv_buf.is_contiguous(), "kv_buf must be contiguous [world, 2, b*hk, n_k, d]");
  const int b = q.size(0), n_q = q.size(1), h = q.size(2), d = q.size(3);
  const int world = hop_mode ? hop.world : (int)kv_buf.size(0);
  const int n_k = fp8 != nullptr ? (int)fp8->n_k : (int)kv_buf.size(3);
  TORCH_CHECK(kv_buf.size(1) == 2 && kv_buf.size(2) == b * kv_heads && kv_buf.size(4) == d);
  if (fp8 != nullptr) {
    TORCH_CHECK(d == 128, "the fp8 forward needs head dim 128");
    TORCH_CHECK(n_k > 0 && kv_buf.size(3) == (n_k + 127) / 128 * 128, "fp8 kv_buf needs round_up(n_k, 128) key rows");
  }
  TORCH_CHECK(d == 64 || d == 128, "head dim must be 64 or 128");
  TORCH_CHECK(h % kv_heads == 0);
  TORCH_CHECK(world <= rab::kMaxWorld);
  if (hop_mode) {
    TORCH_CHECK(kv_buf.size(0) == 1 && hop.owner < world && hop_owner.size() == 1 && hop_owner[0] == hop.owner);
  } else {
    TORCH_CHECK((int)peer_ptrs.size() == world && ready_opt.has_value());
    TORCH_CHECK(ready_opt->is_cuda() && ready_opt->scalar_type() == at::kInt && ready_opt->numel() >= world);
    TORCH_CHECK(hop_owner.size() >= 1 && (int)hop_owner.size() <= world && hop_owner[0] == rank);
  }
  c10::cuda::CUDAGuard guard(q.device());
  auto stream = at::cuda::getCurrentCUDAStream();

  Tensor o = fp8 != nullptr ? torch::empty(q.sizes(), q.options().dtype(at::kBFloat16)) : torch::empty_like(q);
  Tensor lse = torch::empty({b, h, n_q}, q.options().dtype(at::kFloat));

  rab::AttnFwdParams p;
  std::memset(&p, 0, sizeof(p));
  p.batch = b; p.heads = h; p.kv_heads = (int)kv_heads;
  p.n_q = n_q; p.n_k = n_k; p.world = world; p.rank = (int)rank;
  p.causal = causal; p.window = (int)window;
  p.is_bf16 = q.scalar_type() == at::kBFloat16;
  p.scale = (float)scale; p.softclamp = (float)softclamp;
  fill_posmap(p.pos, pos_stride, seg_len, base0, base1, world);
  p.q_pos_offset = (int)q_pos_offset;
  p.hop_count = (int)hop_owner.size();
  for (int i = 0; i < p.hop_count; ++i) p.hop_owner[i] = (int)hop_owner[i];
  p.o = o.data_ptr();
  p.lse = lse.data_ptr<float>();
  if (kmask_bits.has_value()) {
    const Tensor& km = *kmask_bits;
    TORCH_CHECK(km.is_cuda() && km.scalar_type() == at::kInt && km.is_contiguous() && km.dim() == 3);
    TORCH_CHECK(km.size(0) == world && km.size(1) == b && km.size(2) % 4 == 0 && km.size(2) * 32 >= n_k);
    p.kmask_bits = reinterpret_cast<const uint32_t*>(km.data_ptr<int>());
    p.kmask_words = km.size(2);
  }
  p.doc_spans = doc_spans_ptr(doc_spans, world, b, n_q, n_k, q_pos_offset);
  p.sinks = sinks_ptr(sinks, h, q);
  p.slot_bytes = 2ull * b * kv_heads * kv_buf.size(3) * d * kv_buf.element_size();
  if (fp8 != nullptr) {
    p.is_fp8 = 1;
    p.is_bf16 = 1;  // output type
    p.q_descale = descale_ptr(*fp8->q_descale, (int64_t)b * h, "q_descale");
    p.k_descale = descale_ptr(*fp8->k_descale, (int64_t)b * kv_heads, "k_descale");
    p.v_descale = descale_ptr(*fp8->v_descale, (int64_t)b * kv_heads, "v_descale");
  }
  // the kernels address owner o's K / V at slot o of the buffer; in hop mode the one slot we were given IS slot
  // `owner`, so the base is shifted down by owner slots (only that slot is ever dereferenced)
  uint8_t* kv_base = reinterpret_cast<uint8_t*>(kv_buf.data_ptr()) - (hop_mode ? hop.owner * p.slot_bytes : 0);
  p.kv_local = kv_base;
  if (hop_mode) {
    p.all_ready = 1;
    p.carry_o = hop.carry_o;
    p.carry_ml = hop.carry_ml;
    p.carry_in = hop.carry_in;
    p.carry_out = hop.carry_out;
  } else {
    for (int i = 0; i < world; ++i)
      p.kv_peer[i] = peer_ptrs[i] ? reinterpret_cast<const uint8_t*>(peer_ptrs[i]) : p.kv_local + i * p.slot_bytes;
    p.ready = reinterpret_cast<uint32_t*>(ready_opt->data_ptr<int>());
    rab::cuda_check(cudaMemsetAsync(p.ready, 0, sizeof(uint32_t) * world, stream), "ready memset");
    p.fetch_times = (g_fetch_times != nullptr && g_fetch_times_rows >= sm_count()) ? g_fetch_times : nullptr;
  }

  if (fp8 != nullptr) {
    // Q: [b, n, h, 128] bytes -> dims (d, h, n, b), box (128, 1, 128, 1).  K and V^T tiles are both 128 rows of 128
    // bytes: dims (128, n_pad, b*hk, 2*world), box (128, 128, 1, 1), K / V^T of tile i at rows [128 i, 128 i + 128)
    const int n_pad = kv_buf.size(3);
    uint64_t qdims[4] = {(uint64_t)d, (uint64_t)h, (uint64_t)n_q, (uint64_t)b};
    uint64_t qstr[3] = {(uint64_t)d, (uint64_t)h * d, (uint64_t)n_q * h * d};
    uint32_t qbox[4] = {128, 1, 128, 1};
    CUtensorMap map_q = rab::make_tmap_u8(q.data_ptr(), 4, qdims, qstr, qbox, rab::TmapSwizzle::B128);
    uint64_t kdims[4] = {(uint64_t)d, (uint64_t)n_pad, (uint64_t)b * kv_heads, (uint64_t)2 * world};
    uint64_t kstr[3] = {(uint64_t)d, (uint64_t)n_pad * d, (uint64_t)b * kv_heads * n_pad * d};
    uint32_t kbox[4] = {128, 128, 1, 1};
    CUtensorMap map_kv = rab::make_tmap_u8(kv_base, 4, kdims, kstr, kbox, rab::TmapSwizzle::B128);
    rab::launch_attn_fwd<128>(map_q, map_kv, p, sm_count(), stream);
    return {o, lse};
  }
  // Q: [b, n, h, d] -> dims (d, h, n, b), box (64, 1, 128, 1)
  uint64_t qdims[4] = {(uint64_t)d, (uint64_t)h, (uint64_t)n_q, (uint64_t)b};
  uint64_t qstr[3] = {(uint64_t)d * 2, (uint64_t)h * d * 2, (uint64_t)n_q * h * d * 2};
  uint32_t qbox[4] = {64, 1, 128, 1};
  CUtensorMap map_q = rab::make_tmap_bf16(q.data_ptr(), 4, qdims, qstr, qbox, rab::TmapSwizzle::B128);
  // KV: [world, 2, b*hk, n_k, d] -> dims (d, n_k, b*hk, 2*world), box (64, 128, 1, 1)
  uint64_t kdims[4] = {(uint64_t)d, (uint64_t)n_k, (uint64_t)b * kv_heads, (uint64_t)2 * world};
  uint64_t kstr[3] = {(uint64_t)d * 2, (uint64_t)n_k * d * 2, (uint64_t)b * kv_heads * n_k * d * 2};
  uint32_t kbox[4] = {64, 128, 1, 1};
  CUtensorMap map_kv = rab::make_tmap_bf16(kv_base, 4, kdims, kstr, kbox, rab::TmapSwizzle::B128);

  if (d == 128) {
    rab::launch_attn_fwd<128>(map_q, map_kv, p, sm_count(), stream);
  } else {
    rab::launch_attn_fwd<64>(map_q, map_kv, p, sm_count(), stream);
  }
  return {o, lse};
}

std::tuple<Tensor, Tensor> attn_fwd(const Tensor& q, const Tensor& kv_buf, at::IntArrayRef peer_ptrs,
                                    const Tensor& ready, const c10::optional<Tensor>& kmask_bits,
                                    int64_t kv_heads, int64_t rank, bool causal, int64_t window, double scale,
                                    double softclamp, int64_t pos_stride, int64_t seg_len, at::IntArrayRef base0,
                                    at::IntArrayRef base1, int64_t q_pos_offset, at::IntArrayRef hop_owner,
                                    const c10::optional<Tensor>& doc_spans, const c10::optional<Tensor>& sinks) {
  return attn_fwd_impl(q, kv_buf, peer_ptrs, ready, kmask_bits, kv_heads, rank, causal, window, scale, softclamp,
                       pos_stride, seg_len, base0, base1, q_pos_offset, hop_owner, FwdHop{}, doc_spans, sinks);
}

// One ring hop of the forward: q against owner `owner`'s K / V slot.  carry_o fp32 [b, n_q, h, d] and carry_ml fp32
// [2, b*h, n_q] hold the online-softmax state between hops; the launch with carry_out = false writes the final O / lse.
std::tuple<Tensor, Tensor> attn_fwd_hop_impl(const Tensor& q, const Tensor& kv_slot, int64_t owner, int64_t world,
                                             Tensor carry_o, Tensor carry_ml, bool carry_in, bool carry_out,
                                             const c10::optional<Tensor>& kmask_bits, int64_t kv_heads, int64_t rank,
                                             bool causal, int64_t window, double scale, double softclamp,
                                             int64_t pos_stride, int64_t seg_len, at::IntArrayRef base0,
                                             at::IntArrayRef base1, int64_t q_pos_offset,
                                             const c10::optional<Tensor>& doc_spans,
                                             const c10::optional<Tensor>& sinks, const FwdFp8* fp8) {
  TORCH_CHECK(q.dim() == 4);
  const int64_t b = q.size(0), n_q = q.size(1), h = q.size(2), d = q.size(3);
  TORCH_CHECK(carry_o.is_cuda() && carry_o.scalar_type() == at::kFloat && carry_o.is_contiguous() &&
              carry_o.numel() == b * n_q * h * d, "carry_o must be fp32 [b, n_q, h, d]");
  TORCH_CHECK(carry_ml.is_cuda() && carry_ml.scalar_type() == at::kFloat && carry_ml.is_contiguous() &&
              carry_ml.numel() == 2 * b * h * n_q, "carry_ml must be fp32 [2, b*h, n_q]");
  TORCH_CHECK(owner >= 0 && owner < world);
  FwdHop hop;
  hop.owner = (int)owner;
  hop.world = (int)world;
  hop.carry_o = carry_o.data_ptr<float>();
  hop.carry_ml = carry_ml.data_ptr<float>();
  hop.carry_in = carry_in;
  hop.carry_out = carry_out;
  const int64_t owners[1] = {owner};
  return attn_fwd_impl(q, kv_slot, {}, c10::nullopt, kmask_bits, kv_heads, rank, causal, window, scale, softclamp,
                       pos_stride, seg_len, base0, base1, q_pos_offset, at::IntArrayRef(owners, 1), hop, doc_spans, sinks,
                       fp8);
}

std::tuple<Tensor, Tensor> attn_fwd_hop(const Tensor& q, const Tensor& kv_slot, int64_t owner, int64_t world,
                                        Tensor carry_o, Tensor carry_ml, bool carry_in, bool carry_out,
                                        const c10::optional<Tensor>& kmask_bits, int64_t kv_heads, int64_t rank,
                                        bool causal, int64_t window, double scale, double softclamp,
                                        int64_t pos_stride, int64_t seg_len, at::IntArrayRef base0,
                                        at::IntArrayRef base1, int64_t q_pos_offset,
                                        const c10::optional<Tensor>& doc_spans, const c10::optional<Tensor>& sinks) {
  return attn_fwd_hop_impl(q, kv_slot, owner, world, carry_o, carry_ml, carry_in, carry_out, kmask_bits, kv_heads, rank,
                           causal, window, scale, softclamp, pos_stride, seg_len, base0, base1, q_pos_offset, doc_spans,
                           sinks, nullptr);
}

// fp8 forward (head dim 128): q e4m3 [b, n_q, h, 128], kv_buf the uint8 [world, 2, b*hk, n_pad, 128] gather of
// pack_kv_fp8 slots with n_k true keys per owner, descales fp32 [b*h] / [b*hk].  Returns bf16 o and fp32 lse.
std::tuple<Tensor, Tensor> attn_fwd_fp8(const Tensor& q, const Tensor& kv_buf, int64_t n_k, const Tensor& q_descale,
                                        const Tensor& k_descale, const Tensor& v_descale, at::IntArrayRef peer_ptrs,
                                        const Tensor& ready, const c10::optional<Tensor>& kmask_bits,
                                        int64_t kv_heads, int64_t rank, bool causal, int64_t window, double scale,
                                        double softclamp, int64_t pos_stride, int64_t seg_len, at::IntArrayRef base0,
                                        at::IntArrayRef base1, int64_t q_pos_offset, at::IntArrayRef hop_owner,
                                        const c10::optional<Tensor>& doc_spans, const c10::optional<Tensor>& sinks) {
  const FwdFp8 fp8{n_k, &q_descale, &k_descale, &v_descale};
  return attn_fwd_impl(q, kv_buf, peer_ptrs, ready, kmask_bits, kv_heads, rank, causal, window, scale, softclamp,
                       pos_stride, seg_len, base0, base1, q_pos_offset, hop_owner, FwdHop{}, doc_spans, sinks, &fp8);
}

std::tuple<Tensor, Tensor> attn_fwd_hop_fp8(const Tensor& q, const Tensor& kv_slot, int64_t n_k,
                                            const Tensor& q_descale, const Tensor& k_descale, const Tensor& v_descale,
                                            int64_t owner, int64_t world, Tensor carry_o, Tensor carry_ml,
                                            bool carry_in, bool carry_out, const c10::optional<Tensor>& kmask_bits,
                                            int64_t kv_heads, int64_t rank, bool causal, int64_t window, double scale,
                                            double softclamp, int64_t pos_stride, int64_t seg_len,
                                            at::IntArrayRef base0, at::IntArrayRef base1, int64_t q_pos_offset,
                                            const c10::optional<Tensor>& doc_spans,
                                            const c10::optional<Tensor>& sinks) {
  const FwdFp8 fp8{n_k, &q_descale, &k_descale, &v_descale};
  return attn_fwd_hop_impl(q, kv_slot, owner, world, carry_o, carry_ml, carry_in, carry_out, kmask_bits, kv_heads, rank,
                           causal, window, scale, softclamp, pos_stride, seg_len, base0, base1, q_pos_offset, doc_spans,
                           sinks, &fp8);
}


// ---------------------------------------------------------------------------------------------
// fused ring attention backward
// ---------------------------------------------------------------------------------------------
// sinks fp32 [h] (optional): also writes dsinks fp32 [h], the sink gradient of this rank's rows
void bwd_prep(const Tensor& q, const Tensor& o, const Tensor& dout, const Tensor& lse, Tensor qdo_buf,
              Tensor stat_buf, int64_t rank, const c10::optional<Tensor>& sinks, const c10::optional<Tensor>& dsinks) {
  check_16bit(q, "q");
  TORCH_CHECK(q.is_contiguous() && o.is_contiguous() && dout.is_contiguous() && lse.is_contiguous());
  TORCH_CHECK(o.scalar_type() == q.scalar_type() && dout.scalar_type() == q.scalar_type());
  TORCH_CHECK(lse.scalar_type() == at::kFloat && stat_buf.scalar_type() == at::kFloat);
  const int b = q.size(0), n = q.size(1), h = q.size(2), d = q.size(3);
  TORCH_CHECK(qdo_buf.dim() == 5 && qdo_buf.is_contiguous() && qdo_buf.size(1) == 2 && qdo_buf.size(2) == b * h &&
              qdo_buf.size(3) == n && qdo_buf.size(4) == d && qdo_buf.scalar_type() == q.scalar_type());
  TORCH_CHECK(stat_buf.dim() == 4 && stat_buf.is_contiguous() && stat_buf.size(1) == 2 && stat_buf.size(2) == b * h);
  const int n_pad = stat_buf.size(3);
  TORCH_CHECK(n_pad >= n && n_pad % 64 == 0);
  const float* sk = sinks_ptr(sinks, h, q);
  float* dsk = nullptr;
  if (sk != nullptr) {
    TORCH_CHECK(dsinks.has_value() && dsinks->is_cuda() && dsinks->scalar_type() == at::kFloat &&
                    dsinks->is_contiguous() && dsinks->numel() == h,
                "dsinks must be a contiguous fp32 CUDA tensor of ", h, " elements");
    dsk = dsinks->data_ptr<float>();
  }
  c10::cuda::CUDAGuard guard(q.device());
  rab::launch_bwd_prep(q.data_ptr(), o.data_ptr(), dout.data_ptr(), lse.data_ptr<float>(),
                       qdo_buf[rank].data_ptr(), stat_buf[rank].data_ptr<float>(), b, n, h, d, n_pad,
                       q.scalar_type() == at::kBFloat16, at::cuda::getCurrentCUDAStream(), sk, dsk);
}

struct BwdSetup {
  rab::AttnBwdParams p;
  CUtensorMap map_qd128, map_qd64, map_kv;
};

BwdSetup make_bwd_setup(const Tensor& qdo_buf, const Tensor& kv_buf, const Tensor& stat_buf,
                        const c10::optional<Tensor>& ready, int64_t ready_target,
                        const c10::optional<Tensor>& kmask_bits, int64_t batch, int64_t heads, int64_t kv_heads,
                        int64_t rank, bool causal, int64_t window, double scale, double softclamp, int64_t pos_stride,
                        int64_t seg_len, at::IntArrayRef base0, at::IntArrayRef base1, int64_t q_pos_offset,
                        at::IntArrayRef hop_owner, const c10::optional<Tensor>& doc_spans) {
  check_16bit(qdo_buf, "qdo_buf");
  check_16bit(kv_buf, "kv_buf");
  TORCH_CHECK(qdo_buf.is_contiguous() && kv_buf.is_contiguous() && stat_buf.is_contiguous());
  TORCH_CHECK(qdo_buf.dim() == 5 && kv_buf.dim() == 5 && stat_buf.dim() == 4);
  const int world = kv_buf.size(0), n_k = kv_buf.size(3), d = kv_buf.size(4);
  const int n_q = qdo_buf.size(3);
  TORCH_CHECK(qdo_buf.size(0) == world && qdo_buf.size(2) == batch * heads && qdo_buf.size(4) == d);
  TORCH_CHECK(kv_buf.size(2) == batch * kv_heads && stat_buf.size(0) == world && stat_buf.size(2) == batch * heads);
  TORCH_CHECK(d == 64 || d == 128);
  TORCH_CHECK(hop_owner.size() >= 1 && (int)hop_owner.size() <= world && hop_owner[0] == rank);
  BwdSetup s;
  rab::AttnBwdParams& p = s.p;
  std::memset(&p, 0, sizeof(p));
  p.batch = (int)batch; p.heads = (int)heads; p.kv_heads = (int)kv_heads;
  p.n_q = n_q; p.n_k = n_k; p.n_pad = stat_buf.size(3);
  p.world = world; p.rank = (int)rank;
  p.causal = causal; p.window = (int)window;
  p.is_bf16 = kv_buf.scalar_type() == at::kBFloat16;
  p.scale = (float)scale; p.softclamp = (float)softclamp;
  fill_posmap(p.pos, pos_stride, seg_len, base0, base1, world);
  p.q_pos_offset = (int)q_pos_offset;
  p.hop_count = (int)hop_owner.size();
  for (int i = 0; i < p.hop_count; ++i) p.hop_owner[i] = (int)hop_owner[i];
  p.stat = stat_buf.data_ptr<float>();
  if (kmask_bits.has_value()) {
    const Tensor& km = *kmask_bits;
    TORCH_CHECK(km.is_cuda() && km.scalar_type() == at::kInt && km.is_contiguous() && km.dim() == 3);
    TORCH_CHECK(km.size(0) == world && km.size(1) == batch && km.size(2) % 4 == 0 && km.size(2) * 32 >= n_k);
    p.kmask_bits = reinterpret_cast<const uint32_t*>(km.data_ptr<int>());
    p.kmask_words = km.size(2);
  }
  if (ready.has_value()) {
    TORCH_CHECK(ready->is_cuda() && ready->scalar_type() == at::kInt && ready->numel() >= world);
    p.ready = reinterpret_cast<const uint32_t*>(ready->data_ptr<int>());
    p.ready_target = (uint32_t)ready_target;
  }
  p.doc_spans = doc_spans_ptr(doc_spans, world, (int)batch, n_q, n_k, q_pos_offset);
  uint64_t qdims[4] = {(uint64_t)d, (uint64_t)n_q, (uint64_t)batch * heads, (uint64_t)2 * world};
  uint64_t qstr[3] = {(uint64_t)d * 2, (uint64_t)n_q * d * 2, (uint64_t)batch * heads * n_q * d * 2};
  uint32_t qbox128[4] = {64, 128, 1, 1};
  uint32_t qbox64[4] = {64, 64, 1, 1};
  s.map_qd128 = rab::make_tmap_bf16(qdo_buf.data_ptr(), 4, qdims, qstr, qbox128, rab::TmapSwizzle::B128);
  s.map_qd64 = rab::make_tmap_bf16(qdo_buf.data_ptr(), 4, qdims, qstr, qbox64, rab::TmapSwizzle::B128);
  uint64_t kdims[4] = {(uint64_t)d, (uint64_t)n_k, (uint64_t)batch * kv_heads, (uint64_t)2 * world};
  uint64_t kstr[3] = {(uint64_t)d * 2, (uint64_t)n_k * d * 2, (uint64_t)batch * kv_heads * n_k * d * 2};
  uint32_t kbox[4] = {64, 128, 1, 1};
  s.map_kv = rab::make_tmap_bf16(kv_buf.data_ptr(), 4, kdims, kstr, kbox, rab::TmapSwizzle::B128);
  return s;
}

Tensor attn_bwd_dq(const Tensor& qdo_buf, const Tensor& kv_buf, const Tensor& stat_buf,
                   const c10::optional<Tensor>& ready, int64_t ready_target, const c10::optional<Tensor>& kmask_bits,
                   int64_t batch, int64_t heads, int64_t kv_heads, int64_t rank, bool causal, int64_t window,
                   double scale, double softclamp, int64_t pos_stride, int64_t seg_len, at::IntArrayRef base0,
                   at::IntArrayRef base1, int64_t q_pos_offset, at::IntArrayRef hop_owner,
                   const c10::optional<Tensor>& doc_spans) {
  c10::cuda::CUDAGuard guard(kv_buf.device());
  BwdSetup s = make_bwd_setup(qdo_buf, kv_buf, stat_buf, ready, ready_target, kmask_bits, batch, heads, kv_heads, rank,
                              causal, window, scale, softclamp, pos_stride, seg_len, base0, base1, q_pos_offset,
                              hop_owner, doc_spans);
  const int d = kv_buf.size(4);
  Tensor dq = torch::empty({batch, s.p.n_q, heads, d}, kv_buf.options());
  s.p.dq = dq.data_ptr();
  auto stream = at::cuda::getCurrentCUDAStream();
  if (d == 128) {
    rab::launch_attn_bwd_dq<128>(s.map_qd128, s.map_kv, s.p, sm_count(), stream);
  } else {
    rab::launch_attn_bwd_dq<64>(s.map_qd128, s.map_kv, s.p, sm_count(), stream);
  }
  return dq;
}

std::tuple<Tensor, Tensor> attn_bwd_dkdv(const Tensor& qdo_buf, const Tensor& kv_buf, const Tensor& stat_buf,
                                         const c10::optional<Tensor>& ready, int64_t ready_target,
                                         const c10::optional<Tensor>& kmask_bits, int64_t batch, int64_t heads,
                                         int64_t kv_heads, int64_t rank, bool causal, int64_t window, double scale,
                                         double softclamp, int64_t pos_stride, int64_t seg_len, at::IntArrayRef base0,
                                         at::IntArrayRef base1, int64_t q_pos_offset, at::IntArrayRef hop_owner,
                                         const c10::optional<Tensor>& doc_spans) {
  c10::cuda::CUDAGuard guard(kv_buf.device());
  BwdSetup s = make_bwd_setup(qdo_buf, kv_buf, stat_buf, ready, ready_target, kmask_bits, batch, heads, kv_heads, rank,
                              causal, window, scale, softclamp, pos_stride, seg_len, base0, base1, q_pos_offset,
                              hop_owner, doc_spans);
  const int d = kv_buf.size(4);
  Tensor dk = torch::empty({batch, s.p.n_k, kv_heads, d}, kv_buf.options());
  Tensor dv = torch::empty({batch, s.p.n_k, kv_heads, d}, kv_buf.options());
  s.p.dk = dk.data_ptr();
  s.p.dv = dv.data_ptr();
  auto stream = at::cuda::getCurrentCUDAStream();
  if (d == 128) {
    rab::launch_attn_bwd_dkdv<128>(s.map_qd64, s.map_kv, s.p, sm_count(), stream);
  } else {
    rab::launch_attn_bwd_dkdv<64>(s.map_qd64, s.map_kv, s.p, sm_count(), stream);
  }
  return {dk, dv};
}

// One-kernel (5-GEMM) ring backward, head dim 128 (attn_bwd_sm90.cu, KV-stationary kernel in its one-pass form).
//   qdo [2][b*h][n_q][d] 16 bit and stat [2][b*h][n_pad] fp32: this rank's bwd_prep output
//   kv_buf [world][2][b*hk][n_k][d]: the K/V gather (slot o valid once ready[o] >= ready_target; no flags: all valid)
//   dq_acc fp32 [b*h][n_pad][d], zeroed by the caller: dQ (unscaled) is ADDED into it
//   dkv_acc_ptrs: empty -> dK, dV are returned as 16 bit [b, n_k, hk, d] (single rank);
//                 else one pointer per ring rank to that rank's zeroed fp32 [2][b*hk][nk_pad][d] accumulator (peer
//                 mapped): the kernel adds its dK / dV tiles into the owner's accumulator and returns empty tensors
std::tuple<Tensor, Tensor> attn_bwd_ring(const Tensor& qdo, const Tensor& kv_buf, const Tensor& stat, Tensor dq_acc,
                                         const c10::optional<Tensor>& ready, int64_t ready_target,
                                         const c10::optional<Tensor>& kmask_bits, int64_t batch, int64_t heads,
                                         int64_t kv_heads, int64_t rank, bool causal, int64_t window, double scale,
                                         double softclamp, int64_t pos_stride, int64_t seg_len, at::IntArrayRef base0,
                                         at::IntArrayRef base1, int64_t q_pos_offset, at::IntArrayRef hop_owner,
                                         at::IntArrayRef dkv_acc_ptrs, int64_t nk_pad, int64_t world_size,
                                         int64_t slot_owner, const c10::optional<Tensor>& doc_spans) {
  // slot_owner >= 0 (memory = "ring"): kv_buf is ONE owner's slot [1, 2, b*hk, n_k, d] of a `world_size` ring and
  // hop_owner == [slot_owner]; dq_acc and the dK / dV accumulators keep adding up across the per-hop launches
  check_16bit(qdo, "qdo");
  check_16bit(kv_buf, "kv_buf");
  TORCH_CHECK(qdo.is_contiguous() && kv_buf.is_contiguous() && stat.is_contiguous() && dq_acc.is_contiguous());
  TORCH_CHECK(kv_buf.dim() == 5 && qdo.dim() == 4 && stat.dim() == 3 && dq_acc.dim() == 3);
  const bool hop_mode = slot_owner >= 0;
  const int world = hop_mode ? (int)world_size : (int)kv_buf.size(0), n_k = kv_buf.size(3), d = kv_buf.size(4);
  const int n_q = qdo.size(2), n_pad = stat.size(2);
  TORCH_CHECK(d == 128, "attn_bwd_ring: head dim 128 only");
  TORCH_CHECK(qdo.size(0) == 2 && qdo.size(1) == batch * heads && qdo.size(3) == d);
  TORCH_CHECK(stat.size(0) == 2 && stat.size(1) == batch * heads && stat.scalar_type() == at::kFloat);
  TORCH_CHECK(n_pad % 64 == 0 && n_pad >= n_q);
  TORCH_CHECK(dq_acc.scalar_type() == at::kFloat && dq_acc.size(0) == batch * heads && dq_acc.size(1) == n_pad &&
              dq_acc.size(2) == d);
  TORCH_CHECK(kv_buf.size(1) == 2 && kv_buf.size(2) == batch * kv_heads && heads % kv_heads == 0);
  TORCH_CHECK(world <= rab::kMaxWorld && hop_owner.size() >= 1 && (int)hop_owner.size() <= world);
  if (hop_mode) {
    TORCH_CHECK(kv_buf.size(0) == 1 && slot_owner < world && hop_owner.size() == 1 && hop_owner[0] == slot_owner);
  } else {
    TORCH_CHECK(hop_owner[0] == rank);
  }
  c10::cuda::CUDAGuard guard(kv_buf.device());
  auto stream = at::cuda::getCurrentCUDAStream();

  rab::AttnBwdFusedParams p;
  std::memset(&p, 0, sizeof(p));
  p.batch = (int)batch; p.heads = (int)heads; p.kv_heads = (int)kv_heads;
  p.n_q = n_q; p.n_k = n_k; p.n_pad = n_pad; p.nk_pad = (int)nk_pad;
  p.world = world; p.rank = (int)rank;
  p.causal = causal; p.window = (int)window;
  p.is_bf16 = kv_buf.scalar_type() == at::kBFloat16;
  p.scale = (float)scale; p.softclamp = (float)softclamp;
  fill_posmap(p.pos, pos_stride, seg_len, base0, base1, world);
  p.q_pos_offset = (int)q_pos_offset;
  p.hop_count = (int)hop_owner.size();
  for (int i = 0; i < p.hop_count; ++i) p.hop_owner[i] = (int)hop_owner[i];
  p.self_owner[0] = (int)rank;
  p.stat = stat.data_ptr<float>();
  if (kmask_bits.has_value()) {
    const Tensor& km = *kmask_bits;
    TORCH_CHECK(km.is_cuda() && km.scalar_type() == at::kInt && km.is_contiguous() && km.dim() == 3);
    TORCH_CHECK(km.size(0) == world && km.size(1) == batch && km.size(2) % 4 == 0 && km.size(2) * 32 >= n_k);
    p.kmask_bits = reinterpret_cast<const uint32_t*>(km.data_ptr<int>());
    p.kmask_words = km.size(2);
  }
  if (ready.has_value()) {
    TORCH_CHECK(ready->is_cuda() && ready->scalar_type() == at::kInt && ready->numel() >= world);
    p.ready = reinterpret_cast<const uint32_t*>(ready->data_ptr<int>());
    p.ready_target = (uint32_t)ready_target;
  }
  p.doc_spans = doc_spans_ptr(doc_spans, world, (int)batch, n_q, n_k, q_pos_offset);
  // local Q / dO: dims (d, n_q, b*h, 2), box (64, 64, 1, 1)
  uint64_t qdims[4] = {(uint64_t)d, (uint64_t)n_q, (uint64_t)batch * heads, 2};
  uint64_t qstr[3] = {(uint64_t)d * 2, (uint64_t)n_q * d * 2, (uint64_t)batch * heads * n_q * d * 2};
  uint32_t qbox64[4] = {64, 64, 1, 1};
  CUtensorMap map_qd64 = rab::make_tmap_bf16(qdo.data_ptr(), 4, qdims, qstr, qbox64, rab::TmapSwizzle::B128);
  uint64_t kdims[4] = {(uint64_t)d, (uint64_t)n_k, (uint64_t)batch * kv_heads, (uint64_t)2 * world};
  uint64_t kstr[3] = {(uint64_t)d * 2, (uint64_t)n_k * d * 2, (uint64_t)batch * kv_heads * n_k * d * 2};
  uint32_t kbox[4] = {64, 128, 1, 1};
  const uint8_t* kv_base = reinterpret_cast<const uint8_t*>(kv_buf.data_ptr()) -
                           (hop_mode ? (size_t)slot_owner * kstr[2] * 2 : 0);  // see attn_fwd_impl
  CUtensorMap map_kv = rab::make_tmap_bf16(kv_base, 4, kdims, kstr, kbox, rab::TmapSwizzle::B128);
  p.dq_acc = dq_acc.data_ptr<float>();
  // dq_acc as rows (b*h*n_pad) of d fp32: one 64-query x 32-column box per tensor reduction
  uint64_t ddims[2] = {(uint64_t)d, (uint64_t)batch * heads * n_pad};
  uint64_t dstr[1] = {(uint64_t)d * 4};
  uint32_t dbox[2] = {32, 64};
  CUtensorMap map_dq = rab::make_tmap_f32(p.dq_acc, 2, ddims, dstr, dbox, rab::TmapSwizzle::B128);

  Tensor dk, dv;
  if (dkv_acc_ptrs.empty()) {
    dk = torch::empty({batch, n_k, kv_heads, d}, kv_buf.options());
    dv = torch::empty({batch, n_k, kv_heads, d}, kv_buf.options());
    p.dk = dk.data_ptr();
    p.dv = dv.data_ptr();
    p.ring_reduce = 0;
  } else {
    TORCH_CHECK((int)dkv_acc_ptrs.size() == world && nk_pad % 128 == 0 && nk_pad >= n_k);
    dk = torch::empty({0}, kv_buf.options());
    dv = torch::empty({0}, kv_buf.options());
    p.ring_reduce = 1;
    for (int o = 0; o < world; ++o) p.dkv_acc[o] = reinterpret_cast<float*>(dkv_acc_ptrs[o]);
  }
  rab::launch_attn_bwd_fused(map_qd64, map_kv, map_dq, p, sm_count(), stream);
  return {dk, dv};
}

// acc fp32 [b*h][n_pad][d] -> out 16 bit [b][n][h][d] * scale
void acc_convert(const Tensor& acc, Tensor out, double scale) {
  TORCH_CHECK(acc.is_cuda() && acc.scalar_type() == at::kFloat && acc.is_contiguous() && acc.dim() == 3);
  check_16bit(out, "out");
  TORCH_CHECK(out.is_contiguous() && out.dim() == 4);
  const int b = out.size(0), n = out.size(1), h = out.size(2), d = out.size(3);
  TORCH_CHECK(acc.size(0) == b * h && acc.size(1) >= n && acc.size(2) == d && d % 8 == 0);
  c10::cuda::CUDAGuard guard(acc.device());
  rab::launch_acc_convert(acc.data_ptr<float>(), out.data_ptr(), b, h, n, (int)acc.size(1), d, (float)scale,
                          out.scalar_type() == at::kBFloat16, at::cuda::getCurrentCUDAStream());
}

// ---------------------------------------------------------------------------------------------
// tree-attention decode: ONE persistent cooperative kernel (split-KV partials, in-kernel merge of the splits, publish,
// cross-rank signal, merge over NVLink loads or NVLS multimem reductions).  Every buffer is owned by the caller
// (ops/tree_decode_cuda.py caches them), so the call allocates nothing and can be captured in a CUDA graph.
// ---------------------------------------------------------------------------------------------
// cols > 0: a multi-token call with g * tokens (query head, token) columns per kv head
// paged: the residency of the paged instantiation a call with a block table launches
int64_t tree_decode_max_ctas(int64_t d, int64_t kv_kind, bool tensor_core, bool ranged, int64_t cols, bool paged) {
  if (tensor_core) return rab::tree_decode_tc_max_ctas((int)kv_kind, sm_count(), ranged, (int)cols, paged);
  return rab::tree_decode_max_ctas((int)d, (int)kv_kind, sm_count(), ranged, cols > 0, paged);
}

// int32 [b] on q's device (ranged decode: per-sequence cache lengths / query positions), or null
const int* seq_vector_ptr(const c10::optional<Tensor>& t, int64_t b, const Tensor& q, const char* name) {
  if (!t.has_value()) return nullptr;
  TORCH_CHECK(t->device() == q.device() && t->scalar_type() == at::kInt && t->dim() == 1 && t->size(0) == b &&
                  t->is_contiguous(),
              name, " must be a contiguous int32 [batch] tensor on q's device");
  return t->data_ptr<int>();
}

void tree_decode(const Tensor& q, const c10::optional<Tensor>& k, const c10::optional<Tensor>& v,
                 const c10::optional<Tensor>& k_scale, const c10::optional<Tensor>& v_scale, Tensor scratch,
                 Tensor group_done, Tensor counters, at::IntArrayRef partial_ptrs, int64_t aux_local_ptr,
                 at::IntArrayRef pad_ptrs, int64_t mc_partial_ptr, int64_t mc_aux_ptr, int64_t rank, Tensor out,
                 int64_t kv_heads, int64_t splits, double scale, int64_t scale_block_keys, double eps, int64_t grid,
                 bool tensor_core, const c10::optional<Tensor>& sinks, const c10::optional<Tensor>& cache_seqlens,
                 const c10::optional<Tensor>& q_pos, int64_t window, int64_t kv_pos_offset, int64_t kv_pos_stride,
                 double softclamp, const c10::optional<Tensor>& block_table) {
  TORCH_CHECK(q.is_cuda() && q.is_contiguous() && (q.dim() == 3 || q.dim() == 4),
              "q must be contiguous [b, h, d] or [b, h, tokens, d]");
  const int b = q.size(0), h = q.size(1), d = q.size(-1);
  const int tokens = q.dim() == 4 ? (int)q.size(2) : 1;
  TORCH_CHECK(tokens >= 1, "q needs at least one token");
  TORCH_CHECK(d == 64 || d == 128, "tree decode supports head dim 64 or 128");
  rab::TreeDecodeParams p;
  std::memset(&p, 0, sizeof(p));
  p.q = q.data_ptr();
  p.q_kind = q.scalar_type() == at::kBFloat16 ? 0 : (q.scalar_type() == at::kHalf ? 1 : 2);
  TORCH_CHECK(p.q_kind != 2 || q.scalar_type() == at::kFloat, "q must be bf16, fp16 or fp32");
  int n = 0;
  int64_t kv_plane_stride = 0;  // elements between consecutive (batch, kv head) planes
  const bool paged = block_table.has_value();
  TORCH_CHECK(!paged || k.has_value(), "block_table needs the k / v page pools");
  if (paged) {
    // page pools [num_pages, hk, page_size, d]: any page / head / slot strides (HND, or NHD seen as HND), unit d stride
    TORCH_CHECK(v.has_value() && k->dim() == 4 && k->sizes() == v->sizes() && k->strides() == v->strides() &&
                    k->scalar_type() == v->scalar_type(),
                "k / v page pools must share shape, dtype and strides");
    TORCH_CHECK(k->size(0) >= 1 && k->size(1) == kv_heads && k->size(3) == d && k->stride(3) == 1,
                "page pools must be [num_pages, hk, page_size, d] with unit d stride");
    const int64_t ps = k->size(2);
    TORCH_CHECK(ps == 16 || ps == 32 || (ps > 0 && ps % 64 == 0), "page_size must be 16, 32 or a multiple of 64");
    const Tensor& t = *block_table;
    TORCH_CHECK(t.device() == q.device() && t.scalar_type() == at::kInt && t.dim() == 2 && t.size(0) == b &&
                    t.size(1) >= 1 && t.is_contiguous(),
                "block_table must be a contiguous int32 [batch, max_pages] tensor on q's device");
    TORCH_CHECK(t.size(1) * ps < ((int64_t)1 << 31), "max_pages * page_size must be below 2^31");
    const int64_t eb = k->element_size();
    for (int i = 0; i < 3; ++i) TORCH_CHECK((k->stride(i) * eb) % 16 == 0, "pool strides must be multiples of 16 bytes");
    TORCH_CHECK(reinterpret_cast<uintptr_t>(k->data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(v->data_ptr()) % 16 == 0,
                "page pools must be 16-byte aligned");
    n = (int)(t.size(1) * ps);
    p.block_table = t.data_ptr<int>();
    p.max_pages = (int)t.size(1);
    p.page_size = (int)ps;
    p.page_stride = k->stride(0);
    p.head_stride = k->stride(1);
    p.slot_stride = k->stride(2);
    if (k->scalar_type() == at::kBFloat16) p.kv_kind = 0;
    else if (k->scalar_type() == at::kHalf) p.kv_kind = 1;
    else if (k->scalar_type() == at::kFloat8_e4m3fn) p.kv_kind = 2;
    else TORCH_CHECK(false, "k/v must be bf16, fp16 or float8_e4m3fn");
    p.k = k->data_ptr();
    p.v = v->data_ptr();
  } else if (k.has_value()) {
    TORCH_CHECK(v.has_value() && k->dim() == 4 && k->sizes() == v->sizes());
    TORCH_CHECK(k->is_contiguous() ? v->is_contiguous() : k->strides() == v->strides(), "k and v must share a layout");
    TORCH_CHECK(k->size(0) == b && k->size(1) == kv_heads && k->size(3) == d);
    n = k->size(2);
    // a growing cache passes the filled prefix [b, hk, :n, d] of a [b, hk, capacity, d] buffer: rows stay dense, the
    // (batch, head) planes keep the buffer's stride.  Only the tensor-core kernel takes that (it sees K / V through
    // tensor maps); the CUDA-core kernel needs dense planes.
    const bool rows_dense = k->stride(3) == 1 && k->stride(2) == d && k->stride(0) == kv_heads * k->stride(1) &&
                            k->stride(1) >= (int64_t)n * d;
    TORCH_CHECK(k->is_contiguous() || (tensor_core && rows_dense),
                "k / v must be contiguous [b, hk, n, d] (or, for the tensor-core kernel, a prefix view of a [b, hk, "
                "capacity, d] buffer)");
    kv_plane_stride = k->is_contiguous() ? (int64_t)n * d : k->stride(1);  // strides of size-1 dims are arbitrary
    if (k->scalar_type() == at::kBFloat16) p.kv_kind = 0;
    else if (k->scalar_type() == at::kHalf) p.kv_kind = 1;
    else if (k->scalar_type() == at::kFloat8_e4m3fn) p.kv_kind = 2;
    else TORCH_CHECK(false, "k/v must be bf16, fp16 or float8_e4m3fn");
    TORCH_CHECK(v->scalar_type() == k->scalar_type());
    p.k = k->data_ptr();
    p.v = v->data_ptr();
  }
  p.n_scale_blocks = 1;
  p.scale_block = 1 << 30;  // per-head scales: the whole shard is one block
  if (k_scale.has_value()) {
    TORCH_CHECK(v_scale.has_value() && k_scale->sizes() == v_scale->sizes(), "k_scale and v_scale come together");
    TORCH_CHECK(k_scale->scalar_type() == at::kFloat && v_scale->scalar_type() == at::kFloat);
    TORCH_CHECK(k_scale->is_contiguous() && v_scale->is_contiguous() && k_scale->numel() % (b * kv_heads) == 0);
    p.n_scale_blocks = k_scale->numel() / (b * kv_heads);
    p.k_scale = k_scale->data_ptr<float>();
    p.v_scale = v_scale->data_ptr<float>();
    if (p.n_scale_blocks > 1) {
      TORCH_CHECK(scale_block_keys > 0 && scale_block_keys % 64 == 0, "scale_block_keys must be a multiple of 64");
      TORCH_CHECK((int64_t)p.n_scale_blocks * scale_block_keys >= n, "not enough scale blocks for the shard");
      p.scale_block = (int)scale_block_keys;
    }
  }
  p.batch = b; p.heads = h; p.kv_heads = (int)kv_heads; p.n = n; p.splits = (int)splits;
  TORCH_CHECK(h % kv_heads == 0 && splits >= 1);
  p.scale_log2 = (float)(scale * 1.4426950408889634);
  const int g = h / (int)kv_heads * tokens;  // columns per kv head
  TORCH_CHECK(scratch.scalar_type() == at::kFloat && scratch.is_contiguous() &&
              scratch.numel() >= (int64_t)b * kv_heads * splits * g * (d + 4));
  TORCH_CHECK(group_done.scalar_type() == at::kInt && group_done.numel() >= (int64_t)b * kv_heads * ((g + 3) / 4));
  p.tokens = tokens;
  TORCH_CHECK(counters.scalar_type() == at::kInt && counters.numel() >= 4);
  p.scratch = scratch.data_ptr<float>();
  p.group_done = reinterpret_cast<uint32_t*>(group_done.data_ptr<int>());
  p.counters = reinterpret_cast<uint32_t*>(counters.data_ptr<int>());
  p.world = (int)partial_ptrs.size();
  p.rank = (int)rank;
  TORCH_CHECK(p.world >= 1 && p.world <= rab::kMaxWorld && p.rank < p.world && (int)pad_ptrs.size() == p.world);
  for (int i = 0; i < p.world; ++i) {
    p.partials[i] = reinterpret_cast<const float*>(partial_ptrs[i]);
    p.pads[i] = reinterpret_cast<uint32_t*>(pad_ptrs[i]);
  }
  p.partial_local = const_cast<float*>(p.partials[p.rank]);
  p.aux_local = reinterpret_cast<float*>(aux_local_ptr);
  p.mc_partial = reinterpret_cast<const float*>(mc_partial_ptr);
  p.mc_aux = reinterpret_cast<const float*>(mc_aux_ptr);
  TORCH_CHECK(out.is_cuda() && out.is_contiguous() && out.numel() == (int64_t)b * h * tokens * d);
  p.out = out.data_ptr();
  p.out_kind = out.scalar_type() == at::kBFloat16 ? 1 : (out.scalar_type() == at::kHalf ? 0 : 2);
  TORCH_CHECK(p.out_kind != 2 || out.scalar_type() == at::kFloat);
  p.eps = (float)eps;
  p.sinks = sinks_ptr(sinks, h, q);
  p.cache_seqlens = seq_vector_ptr(cache_seqlens, b, q, "cache_seqlens");
  p.q_pos = seq_vector_ptr(q_pos, b, q, "q_pos");
  TORCH_CHECK(window >= 0 && window <= INT32_MAX && (window == 0 || p.q_pos != nullptr),
              "window must be >= 0 and needs q_pos");
  TORCH_CHECK(kv_pos_offset >= 0 && kv_pos_offset <= INT32_MAX && kv_pos_stride >= 1 && kv_pos_stride <= INT32_MAX,
              "kv_pos needs offset >= 0 and stride >= 1");
  TORCH_CHECK(softclamp >= 0.0, "softclamp must be >= 0");
  p.window = (int)window;
  p.kv_pos_offset = (int)kv_pos_offset;
  p.kv_pos_stride = (int)kv_pos_stride;
  p.softclamp_log2 = (float)(softclamp * 1.4426950408889634);
  TORCH_CHECK(!paged || p.cache_seqlens != nullptr, "a paged call needs cache_seqlens");
  // a multi-token or paged call always takes the ranged body (its kernels derive per-token / per-sequence key ranges)
  const bool ranged = p.cache_seqlens != nullptr || p.q_pos != nullptr || softclamp > 0.0 || tokens > 1 || paged;
  c10::cuda::CUDAGuard guard(q.device());
  if (tensor_core && paged) {
    TORCH_CHECK(d == 128, "the tensor-core decode kernel needs head dim 128");
    // the pools as (d, page_size, hk, num_pages); box = one 128-byte wide sub-tile of min(page_size, 64) keys of a page
    const uint64_t eb = p.kv_kind == 2 ? 1 : 2;
    uint64_t dims[4] = {(uint64_t)d, (uint64_t)p.page_size, (uint64_t)kv_heads, (uint64_t)k->size(0)};
    uint64_t strides[3] = {(uint64_t)p.slot_stride * eb, (uint64_t)p.head_stride * eb, (uint64_t)p.page_stride * eb};
    uint32_t box[4] = {(uint32_t)(128 / eb), (uint32_t)std::min(p.page_size, 64), 1, 1};
    auto mk = [&](const void* base) {
      if (p.kv_kind == 2) return rab::make_tmap_u8(base, 4, dims, strides, box, rab::TmapSwizzle::B128);
      if (p.kv_kind == 1) return rab::make_tmap_f16(base, 4, dims, strides, box, rab::TmapSwizzle::B128);
      return rab::make_tmap_bf16(base, 4, dims, strides, box, rab::TmapSwizzle::B128);
    };
    CUtensorMap map_k = mk(p.k), map_v = mk(p.v);
    rab::launch_tree_decode_tc(map_k, map_v, p, (int)grid, at::cuda::getCurrentCUDAStream(), ranged);
  } else if (tensor_core) {
    TORCH_CHECK(d == 128 && n > 0, "the tensor-core decode kernel needs head dim 128 and a non-empty shard");
    // K, V [b*hk, n, d] with any plane stride (a growing cache is read in place) -> dims (d, n, b*hk);
    // box = one 128-byte wide, 64-key sub-tile
    const uint64_t eb = p.kv_kind == 2 ? 1 : 2;
    uint64_t dims[3] = {(uint64_t)d, (uint64_t)n, (uint64_t)b * kv_heads};
    uint64_t strides[2] = {(uint64_t)d * eb, (uint64_t)kv_plane_stride * eb};
    TORCH_CHECK(strides[1] % 16 == 0, "k / v plane stride must be a multiple of 16 bytes");
    uint32_t box[3] = {(uint32_t)(128 / eb), 64, 1};
    auto mk = [&](const void* base) {
      if (p.kv_kind == 2) return rab::make_tmap_u8(base, 3, dims, strides, box, rab::TmapSwizzle::B128);
      if (p.kv_kind == 1) return rab::make_tmap_f16(base, 3, dims, strides, box, rab::TmapSwizzle::B128);
      return rab::make_tmap_bf16(base, 3, dims, strides, box, rab::TmapSwizzle::B128);
    };
    CUtensorMap map_k = mk(p.k), map_v = mk(p.v);
    rab::launch_tree_decode_tc(map_k, map_v, p, (int)grid, at::cuda::getCurrentCUDAStream(), ranged);
  } else {
    rab::launch_tree_decode(p, d, (int)grid, at::cuda::getCurrentCUDAStream(), ranged);
  }
}

void pack_kv(const Tensor& k, const Tensor& v, Tensor slot, int64_t which) {
  check_16bit(k, "k");
  check_16bit(v, "v");
  TORCH_CHECK(k.dim() == 4 && v.dim() == 4 && k.sizes() == v.sizes());
  TORCH_CHECK(k.stride(3) == 1 && v.stride(3) == 1, "k/v need unit stride on the head dim");
  const int b = k.size(0), n = k.size(1), hk = k.size(2), d = k.size(3);
  TORCH_CHECK(d % 8 == 0);
  for (int i = 0; i < 3; ++i)
    TORCH_CHECK(k.stride(i) % 8 == 0 && v.stride(i) % 8 == 0, "k/v strides must be multiples of 8 elements");
  TORCH_CHECK(slot.is_contiguous() && slot.numel() == 2ll * b * n * hk * d && slot.scalar_type() == k.scalar_type());
  c10::cuda::CUDAGuard guard(k.device());
  TORCH_CHECK(which >= 1 && which <= 3, "which: 1 = K half, 2 = V half, 3 = both");
  rab::launch_pack_kv(k.data_ptr(), v.data_ptr(), slot.data_ptr(), b, n, hk, d, k.stride(0), k.stride(1), k.stride(2),
                      v.stride(0), v.stride(1), v.stride(2), (int)which, at::cuda::getCurrentCUDAStream());
}

// k, v [b, n, hk, 128] e4m3 (unit stride on d) -> slot uint8 [2, b*hk, n_pad, 128] (layout in kernels.h)
void pack_kv_fp8(const Tensor& k, const Tensor& v, Tensor slot) {
  TORCH_CHECK(k.is_cuda() && k.scalar_type() == at::kFloat8_e4m3fn && v.scalar_type() == at::kFloat8_e4m3fn,
              "k / v must be float8_e4m3fn CUDA tensors");
  TORCH_CHECK(k.dim() == 4 && k.sizes() == v.sizes() && k.size(3) == 128, "k / v must be [b, n, hk, 128]");
  TORCH_CHECK(k.stride(3) == 1 && v.stride(3) == 1, "k/v need unit stride on the head dim");
  for (int i = 0; i < 3; ++i)
    TORCH_CHECK(k.stride(i) % 16 == 0 && v.stride(i) % 16 == 0, "k/v strides must be multiples of 16 elements");
  const int b = k.size(0), n = k.size(1), hk = k.size(2);
  const int64_t n_pad = (n + 127) / 128 * 128;
  TORCH_CHECK(slot.is_cuda() && slot.scalar_type() == at::kByte && slot.is_contiguous() &&
                  slot.numel() == 2 * (int64_t)b * hk * n_pad * 128,
              "slot must be contiguous uint8 [2, b*hk, n_pad, 128]");
  c10::cuda::CUDAGuard guard(k.device());
  rab::launch_pack_kv_fp8(k.data_ptr(), v.data_ptr(), slot.data_ptr(), b, n, hk, k.stride(0), k.stride(1), k.stride(2),
                          v.stride(0), v.stride(1), v.stride(2), at::cuda::getCurrentCUDAStream());
}

// x [b, n, h, d] 16 bit (unit stride on d) -> out, rotated by angles [n, >= d/2] fp32 (sign -1: inverse rotation).
//   head_major = false: out [b, n, h, d_out] (d_out >= d: the caller pre-zeroes the padding columns)
//   head_major = true : out [b*h, n, d_out]  (one half of a K/V gather slot)
void rotary(const Tensor& x, const Tensor& angles, Tensor out, bool head_major, double sign) {
  check_16bit(x, "x");
  TORCH_CHECK(x.dim() == 4 && x.stride(3) == 1 && out.is_contiguous() && out.scalar_type() == x.scalar_type());
  const int b = x.size(0), n = x.size(1), h = x.size(2), d = x.size(3);
  TORCH_CHECK(d % 16 == 0, "rotary kernel needs head dim % 16 == 0");
  TORCH_CHECK(angles.is_cuda() && angles.scalar_type() == at::kFloat && angles.dim() == 2 && angles.size(0) == n &&
              angles.size(1) >= d / 2 && angles.stride(1) == 1);
  for (int i = 0; i < 3; ++i) TORCH_CHECK(x.stride(i) % 8 == 0, "x strides must be multiples of 8 elements");
  const int d_out = out.size(-1);
  TORCH_CHECK(d_out >= d && d_out % 8 == 0 && out.numel() == (int64_t)b * n * h * d_out);
  long long ob, on, oh;
  if (head_major) { ob = (long long)h * n * d_out; oh = (long long)n * d_out; on = d_out; }
  else { ob = (long long)n * h * d_out; on = (long long)h * d_out; oh = d_out; }
  c10::cuda::CUDAGuard guard(x.device());
  rab::launch_rotary(x.data_ptr(), out.data_ptr(), angles.data_ptr<float>(), (int)angles.stride(0), b, n, h, d,
                     x.stride(0), x.stride(1), x.stride(2), ob, on, oh, (float)sign,
                     x.scalar_type() == at::kBFloat16, at::cuda::getCurrentCUDAStream());
}

void device_barrier(at::IntArrayRef pad_ptrs, int64_t rank, int64_t epoch) {
  rab::BarrierParams p;
  std::memset(&p, 0, sizeof(p));
  p.world = (int)pad_ptrs.size();
  TORCH_CHECK(p.world <= rab::kMaxWorld);
  p.rank = (int)rank;
  p.epoch = (uint32_t)epoch;
  for (int i = 0; i < p.world; ++i) p.pads[i] = reinterpret_cast<uint32_t*>(pad_ptrs[i]);
  rab::launch_device_barrier(p, at::cuda::getCurrentCUDAStream());
}

// ---------------------------------------------------------------------------------------------
// symmetric memory
// ---------------------------------------------------------------------------------------------
std::tuple<Tensor, Tensor> symm_alloc(int64_t bytes) {
  Tensor handle = torch::empty({rab::kIpcHandleBytes}, torch::dtype(torch::kUInt8));
  void* base = rab::symm_alloc((size_t)bytes, handle.data_ptr<uint8_t>());
  int dev = 0;
  cudaGetDevice(&dev);
  Tensor t = torch::from_blob(
      base, {bytes}, [base](void*) { rab::symm_free(base); },
      torch::TensorOptions().dtype(torch::kUInt8).device(torch::kCUDA, dev));
  return {t, handle};
}

void peer_copy(Tensor dst, int64_t src_ptr, int64_t nbytes) {
  TORCH_CHECK(dst.is_cuda() && dst.is_contiguous() && (int64_t)dst.nbytes() >= nbytes);
  c10::cuda::CUDAGuard guard(dst.device());
  rab::cuda_check(cudaMemcpyAsync(dst.data_ptr(), reinterpret_cast<const void*>(src_ptr), (size_t)nbytes,
                                  cudaMemcpyDeviceToDevice, at::cuda::getCurrentCUDAStream()),
                  "peer_copy");
}

// Stream-ordered 32-bit flag write (cuStreamWriteValue32): a memory operation of the stream itself, no kernel and no
// copy-engine job.  The backward uses it to publish "K/V slot o has landed" from the side stream while its persistent
// kernel owns every SM (a flag written by a kernel could never be scheduled next to it).
void stream_write_u32(Tensor flags, int64_t index, int64_t value) {
  TORCH_CHECK(flags.is_cuda() && flags.scalar_type() == at::kInt && flags.is_contiguous() && index >= 0 &&
              index < flags.numel());
  c10::cuda::CUDAGuard guard(flags.device());
  rab::stream_write_value32(flags.data_ptr<int>() + index, (uint32_t)value, at::cuda::getCurrentCUDAStream());
}

int64_t symm_open(const Tensor& handle) {
  TORCH_CHECK(!handle.is_cuda() && handle.scalar_type() == torch::kUInt8 && handle.numel() == rab::kIpcHandleBytes);
  return reinterpret_cast<int64_t>(rab::symm_open(handle.contiguous().data_ptr<uint8_t>()));
}

void symm_close(int64_t ptr) { rab::symm_close(reinterpret_cast<void*>(ptr)); }

}  // namespace

TORCH_LIBRARY(rab, m) {
  m.def("attn_fwd(Tensor q, Tensor kv_buf, int[] peer_ptrs, Tensor ready, Tensor? kmask_bits, int kv_heads, int rank, "
        "bool causal, int window, float scale, float softclamp, int pos_stride, int seg_len, int[] base0, int[] "
        "base1, int q_pos_offset, int[] hop_owner, Tensor? doc_spans=None, Tensor? sinks=None) -> (Tensor, Tensor)");
  m.def("pack_kv(Tensor k, Tensor v, Tensor(a!) slot, int which=3) -> ()");
  m.def("rotary(Tensor x, Tensor angles, Tensor(a!) out, bool head_major, float sign) -> ()");
  m.def("tree_decode(Tensor q, Tensor? k, Tensor? v, Tensor? k_scale, Tensor? v_scale, Tensor(a!) scratch, Tensor(b!) "
        "group_done, Tensor(c!) counters, int[] partial_ptrs, int aux_local_ptr, int[] pad_ptrs, int mc_partial_ptr, int "
        "mc_aux_ptr, int rank, Tensor(d!) out, int kv_heads, int splits, float scale, int scale_block_keys, float eps, "
        "int grid, bool tensor_core, Tensor? sinks=None, Tensor? cache_seqlens=None, Tensor? q_pos=None, int window=0, "
        "int kv_pos_offset=0, int kv_pos_stride=1, float softclamp=0.0, Tensor? block_table=None) -> ()");
  m.def("tree_decode_max_ctas(int d, int kv_kind, bool tensor_core, bool ranged=False, int cols=0, bool paged=False) "
        "-> int");
  m.def("bwd_prep(Tensor q, Tensor o, Tensor dout, Tensor lse, Tensor(a!) qdo_buf, Tensor(b!) stat_buf, int rank, "
        "Tensor? sinks=None, Tensor(c!)? dsinks=None) -> ()");
  m.def("attn_bwd_dq(Tensor qdo_buf, Tensor kv_buf, Tensor stat_buf, Tensor? ready, int ready_target, Tensor? "
        "kmask_bits, int batch, int heads, int kv_heads, int rank, bool causal, int window, float scale, float "
        "softclamp, int pos_stride, int seg_len, int[] base0, int[] base1, int q_pos_offset, int[] hop_owner, Tensor? "
        "doc_spans=None) -> Tensor");
  m.def("attn_bwd_dkdv(Tensor qdo_buf, Tensor kv_buf, Tensor stat_buf, Tensor? ready, int ready_target, Tensor? "
        "kmask_bits, int batch, int heads, int kv_heads, int rank, bool causal, int window, float scale, float "
        "softclamp, int pos_stride, int seg_len, int[] base0, int[] base1, int q_pos_offset, int[] hop_owner, Tensor? "
        "doc_spans=None) -> (Tensor, Tensor)");
  m.def("attn_bwd_ring(Tensor qdo, Tensor kv_buf, Tensor stat, Tensor(a!) dq_acc, Tensor? ready, int ready_target, "
        "Tensor? kmask_bits, int batch, int heads, int kv_heads, int rank, bool causal, int window, float scale, float "
        "softclamp, int pos_stride, int seg_len, int[] base0, int[] base1, int q_pos_offset, int[] hop_owner, int[] "
        "dkv_acc_ptrs, int nk_pad, int world_size=0, int slot_owner=-1, Tensor? doc_spans=None) -> (Tensor, Tensor)");
  m.def("attn_fwd_hop(Tensor q, Tensor kv_slot, int owner, int world, Tensor(a!) carry_o, Tensor(b!) carry_ml, bool "
        "carry_in, bool carry_out, Tensor? kmask_bits, int kv_heads, int rank, bool causal, int window, float scale, "
        "float softclamp, int pos_stride, int seg_len, int[] base0, int[] base1, int q_pos_offset, Tensor? doc_spans=None, "
        "Tensor? sinks=None) -> (Tensor, Tensor)");
  m.def("attn_fwd_fp8(Tensor q, Tensor kv_buf, int n_k, Tensor q_descale, Tensor k_descale, Tensor v_descale, int[] "
        "peer_ptrs, Tensor ready, Tensor? kmask_bits, int kv_heads, int rank, bool causal, int window, float scale, "
        "float softclamp, int pos_stride, int seg_len, int[] base0, int[] base1, int q_pos_offset, int[] hop_owner, "
        "Tensor? doc_spans=None, Tensor? sinks=None) -> (Tensor, Tensor)");
  m.def("attn_fwd_hop_fp8(Tensor q, Tensor kv_slot, int n_k, Tensor q_descale, Tensor k_descale, Tensor v_descale, int "
        "owner, int world, Tensor(a!) carry_o, Tensor(b!) carry_ml, bool carry_in, bool carry_out, Tensor? kmask_bits, "
        "int kv_heads, int rank, bool causal, int window, float scale, float softclamp, int pos_stride, int seg_len, "
        "int[] base0, int[] base1, int q_pos_offset, Tensor? doc_spans=None, Tensor? sinks=None) -> (Tensor, Tensor)");
  m.def("pack_kv_fp8(Tensor k, Tensor v, Tensor(a!) slot) -> ()");
  m.def("acc_convert(Tensor acc, Tensor(a!) out, float scale) -> ()");
  m.def("set_fetch_timing(Tensor? times) -> ()");
  m.def("device_barrier(int[] pad_ptrs, int rank, int epoch) -> ()");
  m.def("peer_copy(Tensor(a!) dst, int src_ptr, int nbytes) -> ()");
  m.def("stream_write_u32(Tensor(a!) flags, int index, int value) -> ()");
  m.def("symm_alloc(int bytes) -> (Tensor, Tensor)");
  m.def("symm_open(Tensor handle) -> int");
  m.def("symm_close(int ptr) -> ()");
}

TORCH_LIBRARY_IMPL(rab, CUDA, m) {
  m.impl("attn_fwd", &attn_fwd);
  m.impl("attn_fwd_hop", &attn_fwd_hop);
  m.impl("pack_kv", &pack_kv);
  m.impl("attn_fwd_fp8", &attn_fwd_fp8);
  m.impl("attn_fwd_hop_fp8", &attn_fwd_hop_fp8);
  m.impl("pack_kv_fp8", &pack_kv_fp8);
  m.impl("rotary", &rotary);
  m.impl("tree_decode", &tree_decode);
  m.impl("bwd_prep", &bwd_prep);
  m.impl("attn_bwd_dq", &attn_bwd_dq);
  m.impl("attn_bwd_dkdv", &attn_bwd_dkdv);
  m.impl("attn_bwd_ring", &attn_bwd_ring);
  m.impl("acc_convert", &acc_convert);
}

TORCH_LIBRARY_IMPL(rab, CompositeExplicitAutograd, m) {
  m.impl("set_fetch_timing", &set_fetch_timing);
  m.impl("device_barrier", &device_barrier);
  m.impl("peer_copy", &peer_copy);
  m.impl("stream_write_u32", &stream_write_u32);
  m.impl("tree_decode_max_ctas", &tree_decode_max_ctas);
  m.impl("symm_alloc", &symm_alloc);
  m.impl("symm_open", &symm_open);
  m.impl("symm_close", &symm_close);
}
