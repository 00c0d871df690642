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
}  // namespace f5
