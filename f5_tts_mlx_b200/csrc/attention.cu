// Host launcher + C-ABI entry for the wgmma flash-attention forward (attention_sm90.cuh).
#include "attention_sm90.cuh"
#include "host_common.h"

static int attention_impl(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch, int32_t frames,
                          int32_t heads, int32_t head_dim, const int32_t* kv_len, int out_fp8, void* stream_,
                          float* scale_out = nullptr);

extern "C" int f5_attention_fwd(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out,
                                int32_t batch, int32_t frames, int32_t heads, int32_t head_dim,
                                const int32_t* kv_len, void* stream_) {
  return attention_impl(qkv, ld_qkv, out, ld_out, batch, frames, heads, head_dim, kv_len, 0, stream_);
}
// the same attention with an e4m3 output (ld_out in bytes): FP8 mode, the out-projection's A operand
extern "C" int f5_attention_fwd_e4m3(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out,
                                     int32_t batch, int32_t frames, int32_t heads, int32_t head_dim,
                                     const int32_t* kv_len, void* stream_) {
  return attention_impl(qkv, ld_qkv, out, ld_out, batch, frames, heads, head_dim, kv_len, 1, stream_);
}
// block-scaled e4m3 output: each (row, head) with its own power-of-two scale, scale_out fp32 [heads][batch * frames]
extern "C" int f5_attention_fwd_e4m3_scaled(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out,
                                            int32_t batch, int32_t frames, int32_t heads, int32_t head_dim,
                                            const int32_t* kv_len, float* scale_out, void* stream_) {
  F5_REQUIRE(scale_out != nullptr, "f5_attention_fwd_e4m3_scaled: null scale_out");
  return attention_impl(qkv, ld_qkv, out, ld_out, batch, frames, heads, head_dim, kv_len, 1, stream_, scale_out);
}

static int attention_impl(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch, int32_t frames,
                          int32_t heads, int32_t head_dim, const int32_t* kv_len, int out_fp8, void* stream_,
                          float* scale_out) {
  using namespace f5;
  if (int e = device_check()) return e;
  F5_REQUIRE(qkv && out, "f5_attention_fwd: null pointer");
  F5_REQUIRE(head_dim == 64, "f5_attention_fwd: head_dim %d unsupported (only 64)", head_dim);
  F5_REQUIRE(batch > 0 && frames > 0 && heads > 0, "f5_attention_fwd: bad shape");
  F5_REQUIRE(ld_qkv % 8 == 0 && ld_qkv >= 3 * heads * 64, "f5_attention_fwd: bad ld_qkv");
  F5_REQUIRE(ld_out % (out_fp8 ? 16 : 8) == 0 && ld_out >= heads * 64, "f5_attention_fwd: bad ld_out");
  CUtensorMap tm;
  uint64_t dims[3] = {(uint64_t)3 * heads * 64, (uint64_t)frames, (uint64_t)batch};
  uint64_t str[2] = {(uint64_t)ld_qkv * 2, (uint64_t)ld_qkv * 2 * (uint64_t)frames};
  uint32_t box[3] = {64, 128, 1};
  if (int e = make_tmap_bf16(&tm, qkv, 3, dims, str, box)) return e;
  AttnParams p;
  p.B = batch; p.N = frames; p.H = heads;
  p.kv_len = kv_len;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ldo = (int)ld_out;
  p.out_fp8 = out_fp8;
  p.scale_out = scale_out;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ProfScope ps(PROF_ATTN, 4.0 * batch * heads * (double)frames * frames * 64.0,
               2.0 * batch * (double)frames * heads * 64.0 * 4.0);
  p.prof = ps.slot;
  auto launch = [&](auto kern, SmemAttrOnce& once, dim3 grid, int threads, int smem) -> int {
    F5_CHECK_CUDA(ensure_dyn_smem(once, kern, smem));
    F5_CHECK_CUDA(launch_kernel(kern, grid, dim3(threads), smem, stream, tm, p));
    F5_CHECK_CUDA(cudaGetLastError());
    return 0;
  };
  const dim3 grid(cdiv(frames, 128), heads, batch);
  static SmemAttrOnce o4, o8, o8s;
  if (scale_out != nullptr) return launch(attn_fwd_kernel<true, true>, o8s, grid, 384, AttnSmem::kTotal);
  if (out_fp8) return launch(attn_fwd_kernel<true>, o8, grid, 384, AttnSmem::kTotal);
  return launch(attn_fwd_kernel<false>, o4, grid, 384, AttnSmem::kTotal);
}
