// DurationPredictor forward (duration.py:97-253, inference branch) as a stream-ordered sequence of
// the same sm_90a kernels the DiT uses: TextEmbedding (mask_padding=False, 2 ConvNeXtV2 blocks),
// DurationInputEmbedding (Linear on [mel | text] + ConvPositionEmbedding), `depth` DurationBlocks
// (plain LayerNorm -> attention (no mask, duration.py:245) -> residual -> LayerNorm -> FF -> residual),
// RMSNorm + masked mean + Linear(dim->1) + Softplus.  Runs once per sample() when duration=None
// (cfm.py:253-262, 307-308).
#include "host_common.h"
#include "launch.h"

using namespace f5;

extern "C" int f5_duration_forward(const f5_duration_weights* w, const f5_duration_buffers* b,
                                   void* stream_) {
  if (int e = device_check()) return e;
  F5_REQUIRE(w && b, "f5_duration_forward: null pointer");
  // the grouped conv's dim/16-channel groups must tile its 64-channel blocks (check_common in dit.cu)
  F5_REQUIRE(w->dim % 128 == 0 && 64 % (w->dim / 16) == 0 && w->dim == w->heads * 64,
             "f5_duration_forward: dim %d heads %d", w->dim, w->heads);
  F5_REQUIRE(b->batch > 0 && b->frames > 0, "f5_duration_forward: bad shape");
  cudaStream_t st = (cudaStream_t)stream_;
  const int D = w->dim, N = b->frames, B = b->batch, R = B * N, F = w->ff_inner;
  const int C = w->text_dim;

  // TextEmbedding with mask_padding=False: no row is zeroed, every ConvNeXt block sees all N rows
  if (int e = text_embedding(w, b, B, B, /*mask_padding=*/0, nullptr, nullptr, false, st)) return e;
  // DurationInputEmbedding: Linear([mel (zeroed beyond lens) | text_embed]) then + conv_pos_embed
  if (int e = launch_concat_cond_text(b->inp, w->mel_dim, B, N, b->text_x, C, b->ct_bf16, w->ct_ld, R, R, st,
                                      b->lens))
    return e;
  {
    f5_gemm_args g = gemm_args(b->ct_bf16, w->ct_ld, w->in_w, w->ct_ld, R, D, w->ct_ld, b->h, D, false, false);
    g.bias = w->in_b; g.out2_bf16 = b->a_bf16; g.ldo2 = D;
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  for (int j = 0; j < 2; ++j) {
    f5_gemm_args g = conv_pos_args(j == 0 ? b->a_bf16 : b->c_bf16, w->conv_w[j], w->conv_b[j],
                                   j == 0 ? b->c_bf16 : (void*)b->x, j == 0, D, N, B, false);
    if (j == 1) { g.resid = b->h; g.ldr = D; }
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  for (int l = 0; l < w->depth; ++l) {
    const f5_dit_block_weights& bw = w->blocks[l];
    // nn.LayerNorm(affine=False): scale = 0 (+1), shift = 0
    if (int e = launch_ln_modulate(b->x, b->a_bf16, R, D, 0, w->zeros, w->zeros, 0, 1, st)) return e;
    {
      f5_gemm_args g = gemm_args(b->a_bf16, D, bw.qkv_w, D, R, 3 * D, D, b->qkv_bf16, 3 * D, true, false);
      g.bias = bw.qkv_b; g.rows_per_batch = N; g.num_batches = B;
      g.rope = b->rope; g.rope_cols = 2 * D; g.q_scale = 0.125f; g.q_cols = D;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    if (int e = f5_attention_fwd(b->qkv_bf16, 3 * D, b->c_bf16, D, B, N, w->heads, 64, nullptr, st)) return e;
    {
      f5_gemm_args g = gemm_args(b->c_bf16, D, bw.out_w, D, R, D, D, b->x, D, false, false);
      g.bias = bw.out_b; g.resid = b->x; g.ldr = D;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    if (int e = launch_ln_modulate(b->x, b->a_bf16, R, D, 0, w->zeros, w->zeros, 0, 1, st)) return e;
    {
      f5_gemm_args g = gemm_args(b->a_bf16, D, bw.ff1_w, D, R, F, D, b->ff_bf16, F, true, false);
      g.bias = bw.ff1_b; g.act = F5_ACT_GELU_TANH;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    {
      f5_gemm_args g = gemm_args(b->ff_bf16, F, bw.ff2_w, F, R, D, F, b->x, D, false, false);
      g.bias = bw.ff2_b; g.resid = b->x; g.ldr = D;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
  }
  return launch_duration_head(b->x, B, N, D, b->lens, w->norm_w, w->pred_w, b->out, st);
}
