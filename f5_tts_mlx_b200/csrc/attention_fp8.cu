// Host launchers + C-ABI entries of the FP8 attention (attention_fp8_sm90.cuh): the quantise pass and the attention.
#include "attention_fp8_sm90.cuh"
#include "host_common.h"

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int f5_qkv_quant_e4m3_masked(const void* qkv, int64_t ld_qkv, void* qk8, int64_t ld_qk8, void* vt8,
                                        int64_t vt_ld, float* qkv_scale, int32_t batch, int32_t frames, int32_t heads,
                                        const int32_t* kv_len, void* stream_) {
  using namespace f5;
  if (int e = device_check()) return e;
  ProfScope ps(PROF_OTHER, 0.0, (double)batch * frames * heads * 64.0 * (2.0 * 3 + 3) + 12.0 * batch * frames * heads);
  F5_REQUIRE(qkv && qk8 && vt8 && qkv_scale, "f5_qkv_quant_e4m3: null pointer");
  F5_REQUIRE(batch > 0 && frames > 0 && heads > 0, "f5_qkv_quant_e4m3: bad shape");
  F5_REQUIRE(aligned16(qkv) && aligned16(qk8) && aligned16(vt8), "f5_qkv_quant_e4m3: pointers must be 16-byte aligned");
  F5_REQUIRE(ld_qkv % 8 == 0 && ld_qkv >= 3 * heads * 64, "f5_qkv_quant_e4m3: bad ld_qkv");
  F5_REQUIRE(ld_qk8 % 16 == 0 && ld_qk8 >= 2 * heads * 64, "f5_qkv_quant_e4m3: bad ld_qk8");
  F5_REQUIRE(vt_ld % 16 == 0 && vt_ld >= (int64_t)cdiv(frames, 128) * 128,
             "f5_qkv_quant_e4m3: vt_ld %lld must be a multiple of 16 and >= roundup(frames, 128)", (long long)vt_ld);
  QkvQuantParams p;
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv);
  p.ld_qkv = ld_qkv;
  p.qk8 = reinterpret_cast<uint8_t*>(qk8);
  p.ld_qk8 = ld_qk8;
  p.vt8 = reinterpret_cast<uint8_t*>(vt8);
  p.vt_ld = vt_ld;
  p.scale = qkv_scale;
  p.B = batch; p.N = frames; p.H = heads;
  p.kv_len = kv_len;
  p.prof = ps.slot;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  F5_CHECK_CUDA(launch_kernel(qkv_quant_e4m3_kernel, dim3(cdiv(frames, 128), heads, batch), dim3(256), 0, stream, p));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// the ABI 2.001 entry: every key below frames is valid
extern "C" int f5_qkv_quant_e4m3(const void* qkv, int64_t ld_qkv, void* qk8, int64_t ld_qk8, void* vt8, int64_t vt_ld,
                                 float* qkv_scale, int32_t batch, int32_t frames, int32_t heads, void* stream) {
  return f5_qkv_quant_e4m3_masked(qkv, ld_qkv, qk8, ld_qk8, vt8, vt_ld, qkv_scale, batch, frames, heads, nullptr, stream);
}

extern "C" int f5_attention_fwd_fp8(const void* qk8, int64_t ld_qk8, const void* vt8, int64_t vt_ld,
                                    const float* qkv_scale, void* out, int64_t ld_out, int32_t batch, int32_t frames,
                                    int32_t heads, int32_t head_dim, const int32_t* kv_len, float* scale_out,
                                    void* stream_) {
  using namespace f5;
  if (int e = device_check()) return e;
  F5_REQUIRE(qk8 && vt8 && qkv_scale && out && scale_out, "f5_attention_fwd_fp8: null pointer");
  F5_REQUIRE(head_dim == 64, "f5_attention_fwd_fp8: head_dim %d unsupported (only 64)", head_dim);
  F5_REQUIRE(batch > 0 && frames > 0 && heads > 0, "f5_attention_fwd_fp8: bad shape");
  F5_REQUIRE(ld_qk8 % 16 == 0 && ld_qk8 >= 2 * heads * 64, "f5_attention_fwd_fp8: bad ld_qk8");
  F5_REQUIRE(vt_ld % 16 == 0 && vt_ld >= (int64_t)cdiv(frames, 128) * 128, "f5_attention_fwd_fp8: bad vt_ld");
  F5_REQUIRE(ld_out % 16 == 0 && ld_out >= heads * 64, "f5_attention_fwd_fp8: bad ld_out");
  CUtensorMap tqk, tvt;
  {
    uint64_t dims[3] = {(uint64_t)2 * heads * 64, (uint64_t)frames, (uint64_t)batch};
    uint64_t str[2] = {(uint64_t)ld_qk8, (uint64_t)ld_qk8 * (uint64_t)frames};
    uint32_t box[3] = {64, 128, 1};
    if (int e = make_tmap_u8_sw64(&tqk, qk8, 3, dims, str, box)) return e;
  }
  {
    uint64_t dims[3] = {(uint64_t)cdiv(frames, 128) * 128, (uint64_t)heads * 64, (uint64_t)batch};
    uint64_t str[2] = {(uint64_t)vt_ld, (uint64_t)vt_ld * heads * 64};
    uint32_t box[3] = {128, 64, 1};
    if (int e = make_tmap_u8(&tvt, vt8, 3, dims, str, box)) return e;
  }
  Fp8AttnParams p;
  p.B = batch; p.N = frames; p.H = heads;
  p.kv_len = kv_len;
  p.scale = qkv_scale;
  p.out = reinterpret_cast<uint8_t*>(out);
  p.ldo = (int)ld_out;
  p.scale_out = scale_out;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ProfScope ps(PROF_ATTN, 4.0 * batch * heads * (double)frames * frames * 64.0,
               (double)batch * frames * heads * 64.0 * 4.0);
  p.prof = ps.slot;
  static SmemAttrOnce once;
  F5_CHECK_CUDA(ensure_dyn_smem(once, attn_fp8_kernel, Fp8AttnSmem::kTotal));
  F5_CHECK_CUDA(launch_kernel(attn_fp8_kernel, dim3(cdiv(frames, 128), heads, batch), dim3(384), Fp8AttnSmem::kTotal,
                              stream, tqk, tvt, p));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}
