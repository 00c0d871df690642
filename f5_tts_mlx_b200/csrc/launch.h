// Internal launcher prototypes shared between translation units (not part of the C ABI).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/f5_b200.h"

namespace f5 {
struct OdeUpdateParams {
  const float* v; int ldv; long long null_row_offset; float cfg_strength;
  const float* y_base; float* y_out; float a;
  float* k_acc; float acc_w; int acc_init; int use_acc;
  __nv_bfloat16* y_bf16; int ld_bf16; long long bf16_copy_row_offset;
  int rows; int d;
  // UNetT: v holds v_frames + 1 rows per utterance, the time row first, so state row r reads v row r + r / v_frames + 1
  // (null_row_offset counts v rows); 0 = one v row per state row (the DiT)
  int v_frames;
};


int launch_ln_modulate(const float* x, void* y, int rows, int dim, int rows_per_batch,
                       const float* scale, const float* shift, long long mod_batch_stride,
                       int add_one, cudaStream_t st);
int launch_ln_f32(const float* x, float* y, int rows, int dim, const float* w, const float* b,
                  cudaStream_t st);
int launch_dwconv7_ln(const float* x, void* y, int B, int N, int C, const float* wt,
                      const float* wb, const float* ln_w, const float* ln_b, cudaStream_t st);
int launch_grn(const void* h, void* y, float* nx_scratch, const float* gamma, const float* beta,
               int B, int N, int C, cudaStream_t st, const int* valid_len = nullptr);
int launch_text_embed_gather(const int* text, int B, int nt, int N, int C, const float* emb,
                             const float* pos_table, int max_pos, float* x, int Bout,
                             int drop_from, cudaStream_t st, int mask_padding = 1,
                             const int* valid_len = nullptr);
int launch_time_mlp(const float* tvals, int T, int D, const float* w0, const float* b0,
                    const float* w2, const float* b2, float* t_emb, void* silu_bf16,
                    cudaStream_t st);
int launch_ode_update(const OdeUpdateParams& p, cudaStream_t st);
int launch_cast_pad_bf16(const float* src, int d, void* dst, int ld, int rows,
                         long long copy_row_offset, cudaStream_t st);
int launch_concat_cond_text(const float* cond, int dc, int Bc, int N, const float* text, int dt,
                            void* dst, int ld, int rows, int drop_from_row, cudaStream_t st,
                            const int* cond_len = nullptr);
int launch_ln_tab_prep(const float* mod, void* prep_bf16, int T, int L, int D, int NM, cudaStream_t st);
int launch_duration_head(const float* x, int B, int N, int D, const int* len, const float* norm_w,
                         const float* pred_w, float* out, cudaStream_t st);
// the UNetT time token: x [BU, N + 1, D] = [t_emb | xe] per utterance, its bf16 copy (row stride ld_bf16) and the
// per-64-column row statistics (f5_unett_time_pack)
int launch_unett_time_pack(const float* xe, const float* t_emb, float* x, void* x_bf16, long long ld_bf16,
                           float* ln_stats, int BU, int N, int D, cudaStream_t st);

// ---- host-side stages shared by the DiT (dit.cu, where they are defined), the UNetT and the duration predictor ----
// f5_gemm_args of out = A·W^T with every optional field off; w_static as f5_gemm_args.w_static
f5_gemm_args gemm_args(const void* a, int64_t lda, const void* w, int64_t ldw, int m, int n, int k, void* out,
                       int64_t ldo, bool out_bf16, bool w_static);
// one grouped k=31 conv of ConvPositionEmbedding (dit.py:33-38), Mish(conv(a) + bias), over `batches` utterances of
// N frames; the caller adds the second conv's residual
f5_gemm_args conv_pos_args(const void* a, const void* w, const float* bias, void* out, bool out_bf16, int D, int N,
                           int batches, bool w_static);
// TextEmbedding (dit.py:196-229) on f5_dit_* or f5_duration_* weights and buffers: the gather of `batch_out`
// utterances into b->text_x (text-dropped from drop_from on), then each ConvNeXtV2 block: dwconv7 + LayerNorm,
// pwconv1 + exact GELU, GRN (over valid_len frames, NULL = all) and pwconv2 + residual, whose rows at or beyond
// row_len are written as zeros (row_len NULL: none)
template <typename Weights, typename Buffers>
int text_embedding(const Weights* w, const Buffers* b, int batch_out, int drop_from, int mask_padding,
                   const int* valid_len, const int* row_len, bool w_static, cudaStream_t st);
// the dim / heads / mel_dim rules of a backbone, refused with messages beginning `who: `
int check_dims(const char* who, int dim, int heads, int mel_dim);
// The rest take f5_dit_* or f5_unett_* weights and buffers.
// The hoisted part of InputEmbedding.proj (dit.py:248-249): [cond | text] · W[:, mel:]^T + b into b->hoist, from
// b->cond and the text embedding in b->text_x (audio condition dropped from batch on with CFG, or by drop_flags bit 0)
template <typename Weights, typename Buffers>
int input_embed_hoist(const Weights* w, const Buffers* b, cudaStream_t st);
// InputEmbedding (dit.py:249-251) on the ODE state in b->y_bf16: launches x·Wx + hoist into b->h (bf16 copy in
// b->a_bf16) and ConvPositionEmbedding's first conv into b->c_bf16, and sets *conv2 to its second conv, fp32 into
// `out` with residual b->h, for the caller to finish and launch
template <typename Weights, typename Buffers>
int input_embedding(const Weights* w, const Buffers* b, void* out, cudaStream_t st, f5_gemm_args* conv2);
// The fixed-grid solve of f5_ode_sample (Euler, midpoint, RK4) with `forward` as the flow field.  `u` holds the
// caller's v, v_frames and null_row_offset; the argument checks' messages begin `who: `.
template <typename Weights, typename Buffers>
int ode_sample(int (*forward)(const Weights*, const Buffers*, int32_t, void*), const Weights* w, const Buffers* b,
               OdeUpdateParams u, const char* who, const float* t, int steps, int method, float cfg_strength, float* y,
               float* trajectory, float* scratch, cudaStream_t st);
}  // namespace f5
