// Host launchers + C-ABI entries for the HBM-bound kernels (elementwise.cuh).
#include <string.h>

#include "elementwise.cuh"
#include "host_common.h"
#include "launch.h"

namespace f5 {

template <bool OUT_F32>
static int launch_ln_any(const float* x, void* yo, int rows, int dim, int rows_per_batch,
                         const float* scale, const float* shift, long long mod_batch_stride,
                         int add_one, cudaStream_t st) {
  F5_REQUIRE(x && yo && scale && shift, "ln_modulate: null pointer");
  F5_REQUIRE(rows > 0, "ln_modulate: rows=%d", rows);
  const int blocks = cdiv(rows * 32, 256);
  ProfScope ps(PROF_LN, 0.0, (double)rows * dim * (OUT_F32 ? 8.0 : 6.0));
  switch (dim) {
#define F5_LN_CASE(DD)                                                                         \
  case DD:                                                                                     \
    F5_CHECK_CUDA(launch_kernel(ln_mod_kernel<DD, OUT_F32>, dim3(blocks), dim3(256), 0, st, x, yo, rows, rows_per_batch, scale,     \
                                                       shift, mod_batch_stride, add_one));      \
    break;
    F5_LN_CASE(256) F5_LN_CASE(512) F5_LN_CASE(768) F5_LN_CASE(1024) F5_LN_CASE(1536) F5_LN_CASE(2048)
#undef F5_LN_CASE
    default:
      return set_error(F5_ERR_INVALID, "ln_modulate: unsupported dim %d", dim);
  }
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_ln_modulate(const float* x, void* y, int rows, int dim, int rows_per_batch,
                       const float* scale, const float* shift, long long mod_batch_stride,
                       int add_one, cudaStream_t st) {
  return launch_ln_any<false>(x, y, rows, dim, rows_per_batch, scale, shift, mod_batch_stride,
                              add_one, st);
}

// affine LayerNorm with fp32 output (Vocos backbone.norm: the result is the residual stream)
int launch_ln_f32(const float* x, float* y, int rows, int dim, const float* w, const float* b,
                  cudaStream_t st) {
  return launch_ln_any<true>(x, y, rows, dim, 0, w, b, 0, 0, st);
}

int launch_ln_tab_prep(const float* mod, void* prep_bf16, int T, int L, int D, int NM, cudaStream_t st) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  F5_REQUIRE(mod && prep_bf16 && T > 0 && L > 0, "ln_tab_prep: bad arguments");
  F5_CHECK_CUDA(launch_kernel(ln_tab_prep_kernel, dim3(T, 2 * L + 1), dim3(256), 0, st, mod,
                              reinterpret_cast<__nv_bfloat16*>(prep_bf16), T, L, D, NM));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_dwconv7_ln(const float* x, void* y, int B, int N, int C, const float* wt,
                      const float* wb, const float* ln_w, const float* ln_b, cudaStream_t st) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  F5_REQUIRE(x && y && wt && wb && ln_w && ln_b, "dwconv7_ln: null pointer");
  const int blocks = cdiv(B * N * 32, 256);
  __nv_bfloat16* yo = reinterpret_cast<__nv_bfloat16*>(y);
  switch (C) {
    case 256: F5_CHECK_CUDA(launch_kernel(dwconv7_ln_kernel<256>, dim3(blocks), dim3(256), 0, st, x, yo, B, N, wt, wb, ln_w, ln_b)); break;
    case 512: F5_CHECK_CUDA(launch_kernel(dwconv7_ln_kernel<512>, dim3(blocks), dim3(256), 0, st, x, yo, B, N, wt, wb, ln_w, ln_b)); break;
    case 1024: F5_CHECK_CUDA(launch_kernel(dwconv7_ln_kernel<1024>, dim3(blocks), dim3(256), 0, st, x, yo, B, N, wt, wb, ln_w, ln_b)); break;
    default: return set_error(F5_ERR_INVALID, "dwconv7_ln: unsupported channels %d", C);
  }
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_grn(const void* h, void* y, float* nx_scratch, const float* gamma, const float* beta,
               int B, int N, int C, cudaStream_t st, const int* valid_len) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  F5_REQUIRE(h && y && nx_scratch && gamma && beta, "grn: null pointer");
  F5_REQUIRE(C % 4 == 0, "grn: C %% 4");
  const int nblk = cdiv(N, kGrnRowsPerBlock);
  F5_CHECK_CUDA(launch_kernel(grn_sumsq_kernel, dim3(nblk, B), dim3(256), 0, st,
                              reinterpret_cast<const __nv_bfloat16*>(h), nx_scratch, N, C, nblk, valid_len));
  F5_CHECK_CUDA(launch_kernel(grn_finalize_kernel, dim3(B), dim3(256), 0, st, nx_scratch, C, nblk));
  const long long total4 = (long long)B * N * C / 4;
  F5_CHECK_CUDA(launch_kernel(grn_apply_kernel, dim3((unsigned)((total4 + 255) / 256)), dim3(256), 0, st,
                              reinterpret_cast<const __nv_bfloat16*>(h),
                              reinterpret_cast<__nv_bfloat16*>(y), (const float*)nx_scratch,
                              (long long)(1 + nblk) * C, gamma, beta, N, C, total4));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_text_embed_gather(const int* text, int B, int nt, int N, int C, const float* emb,
                             const float* pos_table, int max_pos, float* x, int Bout,
                             int drop_from, cudaStream_t st, int mask_padding, const int* valid_len) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  F5_REQUIRE(text && emb && x, "text_embed_gather: null pointer");
  F5_REQUIRE(pos_table || max_pos == 0, "text_embed_gather: max_pos %d without a position table", max_pos);
  F5_REQUIRE(C % 4 == 0, "text_embed_gather: C %% 4");
  F5_CHECK_CUDA(launch_kernel(text_embed_gather_kernel, dim3(dim3(N, Bout)), dim3(128), 0, st, text, B, nt, N, C, emb, pos_table,
                                                          max_pos, x, drop_from, mask_padding, valid_len));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_time_mlp(const float* tvals, int T, int D, const float* w0, const float* b0,
                    const float* w2, const float* b2, float* t_emb, void* silu_bf16,
                    cudaStream_t st) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  F5_REQUIRE(tvals && w0 && b0 && w2 && b2 && silu_bf16, "time_mlp: null pointer");
  F5_CHECK_CUDA(launch_kernel(time_mlp_kernel, dim3(T, cdiv(D, kTimeMlpCols)), dim3(256), (256 + D) * sizeof(float), st, 
      tvals, D, w0, b0, w2, b2, t_emb, reinterpret_cast<__nv_bfloat16*>(silu_bf16)));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_ode_update(const OdeUpdateParams& p, cudaStream_t st) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  const long long tot = (long long)p.rows * p.d;
  F5_CHECK_CUDA(launch_kernel(cfg_ode_update_kernel, dim3((unsigned)((tot + 255) / 256)), dim3(256), 0, st, p));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_cast_pad_bf16(const float* src, int d, void* dst, int ld, int rows,
                         long long copy_row_offset, cudaStream_t st) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  const long long tot = (long long)rows * ld;
  F5_CHECK_CUDA(launch_kernel(cast_pad_bf16_kernel, dim3((unsigned)((tot + 255) / 256)), dim3(256), 0, st, 
      src, d, reinterpret_cast<__nv_bfloat16*>(dst), ld, rows, copy_row_offset));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_concat_cond_text(const float* cond, int dc, int Bc, int N, const float* text, int dt,
                            void* dst, int ld, int rows, int drop_from_row, cudaStream_t st,
                            const int* cond_len) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  const long long tot = (long long)rows * ld;
  F5_CHECK_CUDA(launch_kernel(concat_cond_text_kernel, dim3((unsigned)((tot + 255) / 256)), dim3(256), 0, st, 
      cond, dc, Bc, N, text, dt, reinterpret_cast<__nv_bfloat16*>(dst), ld, rows, drop_from_row, cond_len));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_duration_head(const float* x, int B, int N, int D, const int* len, const float* norm_w,
                         const float* pred_w, float* out, cudaStream_t st) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  F5_REQUIRE(x && len && norm_w && pred_w && out, "duration_head: null pointer");
  switch (D) {
    case 256: F5_CHECK_CUDA(launch_kernel(duration_head_kernel<256>, dim3(B), dim3(256), 0, st, x, N, len, norm_w, pred_w, out)); break;
    case 512: F5_CHECK_CUDA(launch_kernel(duration_head_kernel<512>, dim3(B), dim3(256), 0, st, x, N, len, norm_w, pred_w, out)); break;
    case 1024: F5_CHECK_CUDA(launch_kernel(duration_head_kernel<1024>, dim3(B), dim3(256), 0, st, x, N, len, norm_w, pred_w, out)); break;
    default: return set_error(F5_ERR_INVALID, "duration_head: unsupported dim %d", D);
  }
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------
// UNetT time token (unett.py: x = cat([t[:, None], x], dim=1)): xe fp32 [BU, N, D] -> x fp32 [BU, N + 1, D] with t_emb
// [D] at row 0 of each utterance, its bf16 copy (row stride ld2) and the per-64-column (sum, sum of squares) of every
// row, the statistics the GEMM epilogue's producer side writes.  One block per output row, one warp per 64-column unit
// (two columns per lane).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
unett_time_pack_kernel(const float* __restrict__ xe, const float* __restrict__ t_emb, float* __restrict__ x,
                       __nv_bfloat16* __restrict__ xb, long long ld2, float2* __restrict__ ln_stats, int N, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.x, bu = blockIdx.y;     // n: row inside the utterance, 0 = the time token
  const size_t row = (size_t)bu * (N + 1) + n;
  const float* src = n == 0 ? t_emb : xe + ((size_t)bu * N + n - 1) * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int u = warp; u < D / 64; u += blockDim.x >> 5) {
    const int c = u * 64 + 2 * lane;
    const float2 v = *reinterpret_cast<const float2*>(src + c);
    *reinterpret_cast<float2*>(x + row * D + c) = v;
    *reinterpret_cast<uint32_t*>(xb + row * ld2 + c) = pack_bf16x2(v.x, v.y);
    const float s1 = warp_sum(v.x + v.y), s2 = warp_sum(fmaf(v.x, v.x, v.y * v.y));
    if (lane == 0) ln_stats[row * (D / 64) + u] = make_float2(s1, s2);
  }
}

int launch_unett_time_pack(const float* xe, const float* t_emb, float* x, void* x_bf16, long long ld_bf16,
                           float* ln_stats, int BU, int N, int D, cudaStream_t st) {
  ProfScope ps(PROF_OTHER, 0.0, 0.0);
  F5_REQUIRE(xe && t_emb && x && x_bf16 && ln_stats, "unett_time_pack: null pointer");
  F5_REQUIRE(BU > 0 && N > 0 && D > 0 && D % 64 == 0 && ld_bf16 >= D && ld_bf16 % 2 == 0,
             "unett_time_pack: bad shape BU=%d N=%d D=%d ld=%lld", BU, N, D, ld_bf16);
  F5_CHECK_CUDA(launch_kernel(unett_time_pack_kernel, dim3(N + 1, BU), dim3(128), 0, st, xe, t_emb, x,
                              reinterpret_cast<__nv_bfloat16*>(x_bf16), ld_bf16, reinterpret_cast<float2*>(ln_stats), N, D));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace f5

extern "C" {

int f5_ln_modulate(const float* x, void* y_bf16, int32_t rows, int32_t dim, int32_t rows_per_batch,
                   const float* scale, const float* shift, int64_t mod_batch_stride,
                   int32_t add_one, void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_ln_modulate(x, y_bf16, rows, dim, rows_per_batch, scale, shift,
                                mod_batch_stride, add_one, (cudaStream_t)stream);
}

int f5_dwconv7_ln(const float* x, void* y_bf16, int32_t batch, int32_t frames, int32_t channels,
                  const float* w_tap_major, const float* bias, const float* ln_w, const float* ln_b,
                  void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_dwconv7_ln(x, y_bf16, batch, frames, channels, w_tap_major, bias, ln_w, ln_b,
                               (cudaStream_t)stream);
}

int f5_grn(const void* h_bf16, void* y_bf16, float* nx_scratch, const float* gamma,
           const float* beta, int32_t batch, int32_t frames, int32_t channels, void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_grn(h_bf16, y_bf16, nx_scratch, gamma, beta, batch, frames, channels,
                        (cudaStream_t)stream);
}

// ---- kernel test entries: each runs one launcher of the DiT / UNetT / duration / Vocos paths alone ----

int f5_ln_affine_f32(const float* x, float* y, int32_t rows, int32_t dim, const float* w, const float* b,
                     void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_ln_f32(x, y, rows, dim, w, b, (cudaStream_t)stream);
}

int f5_ln_tab_prep(const float* mod, void* prep_bf16, int32_t times, int32_t depth, int32_t dim,
                   int32_t mod_cols, void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_ln_tab_prep(mod, prep_bf16, times, depth, dim, mod_cols, (cudaStream_t)stream);
}

int f5_text_embed(const int32_t* text, int32_t batch, int32_t text_cols, int32_t frames, int32_t channels,
                  const float* emb, const float* pos_table, int32_t max_pos, float* x, int32_t batch_out,
                  int32_t drop_from, int32_t mask_padding, const int32_t* valid_len, void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_text_embed_gather(text, batch, text_cols, frames, channels, emb, pos_table, max_pos, x,
                                      batch_out, drop_from, (cudaStream_t)stream, mask_padding, valid_len);
}

int f5_time_mlp(const float* tvals, int32_t times, int32_t dim, const float* w0, const float* b0,
                const float* w2, const float* b2, float* t_emb, void* silu_bf16, void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_time_mlp(tvals, times, dim, w0, b0, w2, b2, t_emb, silu_bf16, (cudaStream_t)stream);
}

int f5_ode_update(const float* v, int32_t ldv, int64_t null_row_offset, float cfg_strength,
                  const float* y_base, float* y_out, float a, float* k_acc, float acc_w, int32_t acc_init,
                  int32_t use_acc, void* y_bf16, int32_t ld_bf16, int64_t bf16_copy_row_offset, int32_t rows,
                  int32_t d, void* stream) {
  if (int e = f5::device_check()) return e;
  F5_REQUIRE(v && rows > 0 && d > 0 && ldv >= d, "ode_update: bad arguments");
  F5_REQUIRE(!y_out || y_base, "ode_update: y_out needs y_base");
  F5_REQUIRE(!y_bf16 || ld_bf16 >= d, "ode_update: ld_bf16 < d");
  f5::OdeUpdateParams p;
  memset(&p, 0, sizeof(p));
  p.v = v; p.ldv = ldv; p.null_row_offset = null_row_offset; p.cfg_strength = cfg_strength;
  p.y_base = y_base; p.y_out = y_out; p.a = a;
  p.k_acc = k_acc; p.acc_w = acc_w; p.acc_init = acc_init; p.use_acc = use_acc;
  p.y_bf16 = reinterpret_cast<__nv_bfloat16*>(y_bf16); p.ld_bf16 = ld_bf16;
  p.bf16_copy_row_offset = bf16_copy_row_offset;
  p.rows = rows; p.d = d;
  return f5::launch_ode_update(p, (cudaStream_t)stream);
}

int f5_cast_pad_bf16(const float* src, int32_t d, void* dst, int32_t ld, int32_t rows, int64_t copy_row_offset,
                     void* stream) {
  if (int e = f5::device_check()) return e;
  F5_REQUIRE(src && dst && rows > 0 && ld >= d, "cast_pad_bf16: bad arguments");
  return f5::launch_cast_pad_bf16(src, d, dst, ld, rows, copy_row_offset, (cudaStream_t)stream);
}

int f5_concat_cond_text(const float* cond, int32_t dc, int32_t batch_cond, int32_t frames, const float* text,
                        int32_t dt, void* dst, int32_t ld, int32_t rows, int32_t drop_from_row,
                        const int32_t* cond_len, void* stream) {
  if (int e = f5::device_check()) return e;
  F5_REQUIRE(cond && text && dst && rows > 0 && ld >= dc + dt, "concat_cond_text: bad arguments");
  return f5::launch_concat_cond_text(cond, dc, batch_cond, frames, text, dt, dst, ld, rows, drop_from_row,
                                     (cudaStream_t)stream, cond_len);
}

int f5_duration_head(const float* x, int32_t batch, int32_t frames, int32_t dim, const int32_t* len,
                     const float* norm_w, const float* pred_w, float* out, void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_duration_head(x, batch, frames, dim, len, norm_w, pred_w, out, (cudaStream_t)stream);
}

int f5_grn_valid(const void* h_bf16, void* y_bf16, float* nx_scratch, const float* gamma, const float* beta,
                 int32_t batch, int32_t frames, int32_t channels, const int32_t* valid_len, void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_grn(h_bf16, y_bf16, nx_scratch, gamma, beta, batch, frames, channels,
                        (cudaStream_t)stream, valid_len);
}

int f5_unett_time_pack(const float* xe, const float* t_emb, float* x, void* x_bf16, int64_t ld_bf16, float* ln_stats,
                       int32_t batch, int32_t frames, int32_t dim, void* stream) {
  if (int e = f5::device_check()) return e;
  return f5::launch_unett_time_pack(xe, t_emb, x, x_bf16, ld_bf16, ln_stats, batch, frames, dim, (cudaStream_t)stream);
}

}  // extern "C"
