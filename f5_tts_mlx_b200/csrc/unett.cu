// UNetT forward (upstream F5-TTS E2TTS_Base) and its ODE loop as a stream-ordered sequence of the sm_90a kernels in
// this directory (C-ABI: f5_unett_precompute / f5_unett_forward / f5_unett_ode_sample; see include/f5_b200.h).  Like
// dit.cu it holds no kernels; the time-token pack, the one kernel only this backbone needs, is in elementwise.cu.
//
// Row layout: the frames of an utterance are R = BU * N rows up to the end of the input embedding; the time token then
// makes every utterance N + 1 rows (R1 = BU * (N + 1)), the time row first.  Each RMSNorm is folded: its gain into the
// consuming weight at pack time, its row scale sqrt(D) / max(||x||, 1e-12) into the consuming GEMM's epilogue
// (f5_gemm_args.ln_rms) from the (sum, sum of squares) statistics the producing GEMM writes next to a bf16 copy of x.
#include "host_common.h"
#include "launch.h"

namespace f5 {
namespace {

int check_unett(const f5_unett_weights* w, const f5_unett_buffers* b) {
  F5_REQUIRE(w && b, "unett: null weights/buffers");
  if (int e = check_dims("unett", w->dim, w->heads, w->mel_dim)) return e;
  F5_REQUIRE(w->depth > 0 && w->depth % 2 == 0, "unett: depth %d must be even and positive", w->depth);
  F5_REQUIRE(w->text_dim % 4 == 0 && w->ct_ld % 64 == 0 && w->ct_ld >= w->mel_dim + w->text_dim,
             "unett: text_dim %d / ct_ld %d", w->text_dim, w->ct_ld);
  F5_REQUIRE(w->ff_inner % 64 == 0, "unett: ff_inner %d", w->ff_inner);
  F5_REQUIRE(w->rope_heads >= 0 && w->rope_heads <= w->heads, "unett: rope_heads %d not in [0, heads %d]",
             w->rope_heads, w->heads);
  F5_REQUIRE(w->blocks && w->skip_w && w->proj_w, "unett: no blocks / skip_w / proj_w");
  for (int l = 0; l < w->depth; ++l) {
    const f5_dit_block_weights& k = w->blocks[l];
    F5_REQUIRE(k.qkv_w && k.out_w && k.ff1_w && k.ff2_w, "unett: blocks[%d] has a NULL weight", l);
    F5_REQUIRE(!(k.qkv_w8 || k.ff1_w8 || k.out_w8 || k.ff2_w8 || k.qkv_ws || k.ff1_ws || k.out_ws || k.ff2_ws),
               "unett: blocks[%d] has FP8 weights: this backbone runs in bf16 only", l);
  }
  F5_REQUIRE(b->batch > 0 && b->frames > 0 && b->n_times > 0, "unett: bad buffer shape");
  F5_REQUIRE(!b->valid_len == !b->valid_len1, "unett: valid_len and valid_len1 are bound together or not at all");
  F5_REQUIRE(b->x && b->a_bf16 && b->c_bf16 && b->qkv_bf16 && b->ff_bf16 && b->ln_stats && b->skip && b->v && b->h &&
                 b->y_bf16 && b->hoist && b->t_emb && b->rope,
             "unett: a NULL buffer");
  return 0;
}

// out = A·W^T, W a model weight
f5_gemm_args weight_gemm(const void* a, int64_t lda, const void* w, int m, int n, int k, void* out, int64_t ldo,
                         bool out_bf16, const void* prefetch, int64_t prefetch_bytes) {
  f5_gemm_args g = gemm_args(a, lda, w, k, m, n, k, out, ldo, out_bf16, true);
  g.prefetch = prefetch; g.prefetch_bytes = prefetch_bytes;
  return g;
}

// producer of the residual stream x: a bf16 copy of it to out2 (row stride ld2) and, when a norm consumes it next, the
// row statistics
void producer(f5_gemm_args& g, void* out2, int64_t ld2, float* ln_stats) {
  g.out2_bf16 = out2; g.ldo2 = ld2; g.ln_stats = ln_stats;
}

// consumer of RMSNorm(x), the norm's gain folded into the weight
void rms_consumer(f5_gemm_args& g, const float* ln_stats) {
  g.ln_rms = 1; g.ln_in_stats = ln_stats;
}

}  // namespace
}  // namespace f5

using namespace f5;

extern "C" int f5_unett_precompute(const f5_unett_weights* w, const f5_unett_buffers* b, void* stream_) {
  if (int e = device_check()) return e;
  if (int e = check_unett(w, b)) return e;
  F5_REQUIRE(w->text_emb && b->text && b->cond && b->tvals && b->text_x && b->ct_bf16 && b->silu_t,
             "unett_precompute: a NULL input or buffer");
  cudaStream_t st = (cudaStream_t)stream_;
  const int D = w->dim, N = b->frames, B = b->batch;
  const int BU = (b->cfg ? 2 : 1) * B;
  // TextEmbedding with conv_layers = 0 and mask_padding = False: the embedding gather alone, filler rows embed[0];
  // bucket rows (>= valid_len) zero.  CFG: the second half text-dropped.
  const int drop_from = b->cfg ? B : ((b->drop_flags & 2) ? 0 : BU);
  if (int e = launch_text_embed_gather(b->text, B, b->text_len_max, N, w->text_dim, w->text_emb, nullptr, 0, b->text_x,
                                       BU, drop_from, st, 0, b->valid_len))
    return e;
  // hoisted part of InputEmbedding.proj: [cond | text] · W[:, mel:]^T + b
  if (int e = input_embed_hoist(w, b, st)) return e;
  // TimestepEmbedding of every evaluation time: the time tokens
  return launch_time_mlp(b->tvals, b->n_times, D, w->time_w0, w->time_b0, w->time_w2, w->time_b2, b->t_emb, b->silu_t,
                         st);
}

extern "C" int f5_unett_forward(const f5_unett_weights* w, const f5_unett_buffers* b, int32_t ti, void* stream_) {
  if (int e = device_check()) return e;
  if (int e = check_unett(w, b)) return e;
  F5_REQUIRE(ti >= 0 && ti < b->n_times, "unett_forward: time_index %d out of [0,%d)", ti, b->n_times);
  cudaStream_t st = (cudaStream_t)stream_;
  const int D = w->dim, N = b->frames, N1 = N + 1, F = w->ff_inner, H = w->depth / 2;
  const int BU = (b->cfg ? 2 : 1) * b->batch;
  const int R1 = BU * N1;
  const bool prefetch = R1 <= 16384;   // as the DiT: weights prefetched into L2 while they are comparable to activations
  __nv_bfloat16* skip = reinterpret_cast<__nv_bfloat16*>(b->skip);
  auto slot = [&](int j) { return skip + (size_t)j * R1 * 2 * D; };
  const __nv_bfloat16* skip_w = reinterpret_cast<const __nv_bfloat16*>(w->skip_w);
  auto skip_weight = [&](int l) { return skip_w + (size_t)(l - H) * D * 2 * D; };
  const int32_t* kv_len = b->seq_len1 ? b->seq_len1 : b->valid_len1;

  // ---- InputEmbedding: x·Wx + hoist, then + ConvPositionEmbedding (the DiT's, on R rows) ----
  {
    f5_gemm_args g;
    if (int e = input_embedding(w, b, b->h, st, &g)) return e;
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  // ---- time token at row 0: x [BU, N + 1, D], its bf16 copy in the right half of skip slot 0 (layer 0's push and its
  // QKV operand), and the statistics of attn_norm ----
  if (int e = launch_unett_time_pack(b->h, b->t_emb + (size_t)ti * D, b->x, slot(0) + D, 2 * D, b->ln_stats, BU, N, D,
                                     st))
    return e;

  for (int l = 0; l < w->depth; ++l) {
    const f5_dit_block_weights& bw = w->blocks[l];
    // the bf16 x this layer's QKV reads: the pushed copy in slot l (first half), skip_proj's output (second half)
    const void* xa = b->a_bf16;
    int64_t lda = D;
    if (l < H) {
      xa = slot(l) + D; lda = 2 * D;
    } else {
      // x = skip_proj([x | skip]): slot depth-1-l holds x (left, written by the previous FF2) and the skip (right)
      f5_gemm_args g = weight_gemm(slot(w->depth - 1 - l), 2 * D, skip_weight(l), R1, D, 2 * D, b->x, D, false,
                                   prefetch ? bw.qkv_w : nullptr, prefetch ? (int64_t)6 * D * D : 0);
      producer(g, b->a_bf16, D, b->ln_stats);
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    {  // attn(RMSNorm(x)): QKV with the rotation of the leading rope_heads heads, q scaled by 1/8
      f5_gemm_args g = weight_gemm(xa, lda, bw.qkv_w, R1, 3 * D, D, b->qkv_bf16, 3 * D, true,
                                   prefetch ? bw.out_w : nullptr, prefetch ? (int64_t)2 * D * D : 0);
      g.bias = bw.qkv_b;
      rms_consumer(g, b->ln_stats);
      g.rows_per_batch = N1; g.num_batches = BU;
      g.rope = b->rope; g.rope_cols = 2 * D; g.q_scale = 0.125f; g.q_cols = D;
      if (w->rope_heads) { g.rope_cols = 64 * w->rope_heads; g.rope_col2 = D; }
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    if (int e = f5_attention_fwd(b->qkv_bf16, 3 * D, b->c_bf16, D, BU, N1, w->heads, 64, kv_len, st)) return e;
    {  // x += to_out(attention), padded rows' output masked to 0; then ff_norm's operand
      f5_gemm_args g = weight_gemm(b->c_bf16, D, bw.out_w, R1, D, D, b->x, D, false,
                                   prefetch ? bw.ff1_w : nullptr, prefetch ? (int64_t)2 * F * D : 0);
      g.bias = bw.out_b;
      g.rows_per_batch = N1; g.num_batches = BU; g.row_len = b->seq_len1;
      g.resid = b->x; g.ldr = D;
      producer(g, b->a_bf16, D, b->ln_stats);
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    {  // ff(RMSNorm(x)) first Linear + GELU(tanh)
      f5_gemm_args g = weight_gemm(b->a_bf16, D, bw.ff1_w, R1, F, D, b->ff_bf16, F, true,
                                   prefetch ? bw.ff2_w : nullptr, prefetch ? (int64_t)2 * D * F : 0);
      g.bias = bw.ff1_b; g.act = F5_ACT_GELU_TANH;
      rms_consumer(g, b->ln_stats);
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    {  // x += second Linear; the bf16 copy goes where the next layer reads it
      const int nx = l + 1;
      const void* pf = nullptr;
      int64_t pf_bytes = 0;
      if (prefetch && nx < w->depth) {
        pf = nx < H ? w->blocks[nx].qkv_w : (const void*)skip_weight(nx);
        pf_bytes = nx < H ? (int64_t)6 * D * D : (int64_t)4 * D * D;
      }
      f5_gemm_args g = weight_gemm(b->ff_bf16, F, bw.ff2_w, R1, D, F, b->x, D, false, pf, pf_bytes);
      g.bias = bw.ff2_b;
      g.resid = b->x; g.ldr = D;
      if (nx < H) producer(g, slot(nx) + D, 2 * D, b->ln_stats);                // push, and the QKV operand
      else if (nx < w->depth) producer(g, slot(w->depth - 1 - nx), 2 * D, nullptr);   // x beside its skip
      else producer(g, b->a_bf16, D, b->ln_stats);                              // norm_out's operand
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
  }

  // ---- proj_out(RMSNorm_out(x)) over all N + 1 rows; the solver skips the time rows ----
  f5_gemm_args g = weight_gemm(b->a_bf16, D, w->proj_w, R1, w->mel_dim, D, b->v, w->mel_dim, false, nullptr, 0);
  g.bias = w->proj_b;
  rms_consumer(g, b->ln_stats);
  return f5_gemm_bf16(&g, st);
}

extern "C" int f5_unett_ode_sample(const f5_unett_weights* w, const f5_unett_buffers* b, const float* t, int32_t steps,
                                   int32_t method, float cfg_strength, float* y, float* trajectory, float* scratch,
                                   void* stream_) {
  if (int e = device_check()) return e;
  if (int e = check_unett(w, b)) return e;
  // v: frames + 1 rows per utterance (time row first); the null (CFG) rows start after batch of them
  OdeUpdateParams u = {};
  u.v = b->v; u.v_frames = b->frames;
  u.null_row_offset = b->cfg ? (long long)b->batch * (b->frames + 1) : 0;
  return ode_sample(f5_unett_forward, w, b, u, "unett_ode_sample", t, steps, method, cfg_strength, y, trajectory,
                    scratch, (cudaStream_t)stream_);
}
