// DiT forward and the ODE loop of F5TTS.sample as a stream-ordered sequence of the sm_90a kernels
// in this directory (C-ABI: f5_dit_precompute / f5_dit_forward / f5_ode_sample).
//
// What the reference recomputes on every forward but depends only on (text, cond, t) is hoisted:
//   * TextEmbedding (dit.py:390)                      -> once per sample, per CFG branch
//   * cond·Wc + text·Wt + b of InputEmbedding.proj    -> once per sample (dit.py:249)
//   * TimestepEmbedding + all 23 AdaLN linears         -> one GEMM over all time points (dit.py:389,267,286)
// and the two unbatched CFG passes (cfm.py:342-363) run as one forward over a doubled batch.
#include <stdlib.h>
#include <string.h>

#include "host_common.h"
#include "launch.h"

extern "C" int f5_attention_fwd(const void*, int64_t, void*, int64_t, int32_t, int32_t, int32_t,
                                int32_t, const int32_t*, void*);
extern "C" int f5_attention_fwd_e4m3(const void*, int64_t, void*, int64_t, int32_t, int32_t, int32_t,
                                     int32_t, const int32_t*, void*);

namespace f5 {

static f5_gemm_args gemm_base(const void* a, int64_t lda, const void* w, int64_t ldw, int m, int n,
                              int k, void* out, int64_t ldo, bool out_bf16) {
  f5_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.a = a; g.lda = lda; g.w = w; g.ldw = ldw;
  g.m = m; g.n = n; g.k = k;
  g.num_batches = 1;
  g.conv_taps = 1;
  g.out = out; g.ldo = ldo; g.out_bf16 = out_bf16 ? 1 : 0;
  g.q_scale = 1.f;
  g.w_static = 1;   // every W on this path is a model weight
  return g;
}

static int check_common(const f5_dit_weights* w, const f5_dit_buffers* b) {
  F5_REQUIRE(w && b, "dit: null weights/buffers");
  F5_REQUIRE(w->dim % 128 == 0 && w->dim >= 256 && w->dim <= 1024,
             "dit: dim %d unsupported (128 | dim, 256..1024: the grouped conv packs 16 groups of <= 64 channels)", w->dim);
  F5_REQUIRE(w->dim == w->heads * 64, "dit: dim %d != heads %d * 64", w->dim, w->heads);
  F5_REQUIRE(w->mel_dim % 4 == 0 && w->mel_dim <= 128, "dit: mel_dim %d", w->mel_dim);
  F5_REQUIRE(w->blocks && w->depth > 0, "dit: no blocks");
  F5_REQUIRE(b->batch > 0 && b->frames > 0 && b->n_times > 0, "dit: bad buffer shape");
  return 0;
}

// Tuning aid: F5_TUNE="qkv=2:192,out=1:128,ff1=1:128,ff2=1:64" overrides (variant:tile_n) of the block's GEMMs so the
// kernel-variant space can be measured in situ (bench.py) without rebuilding; unset = the launcher's own heuristics.
struct GemmTune { int variant, tile_n; };
static GemmTune tune_of(const char* key) {
  GemmTune t = {0, 0};
  const char* env = getenv("F5_TUNE");
  if (!env) return t;
  const char* p = strstr(env, key);
  if (!p) return t;
  p += strlen(key);
  if (*p != '=') return t;
  t.variant = atoi(p + 1);
  const char* c = strchr(p, ':');
  const char* comma = strchr(p, ',');
  if (c && (!comma || c < comma)) t.tile_n = atoi(c + 1);
  return t;
}

static long long ln_tab_ld(const f5_dit_weights* w) {
  return (long long)w->depth * (3 * w->dim + w->ff_inner) + 128;
}
// F5_LN_FUSED=0 keeps the separate LayerNorm+modulate launches even when the fused-AdaLN buffers are present
static bool ln_fused(const f5_dit_buffers* b) {
  static int env = -1;
  if (env < 0) { const char* v = getenv("F5_LN_FUSED"); env = (v && v[0] == '0') ? 0 : 1; }
  return env && b->ln_stats && b->ln_tab && b->ln_prep;
}

}  // namespace f5

using namespace f5;

extern "C" int64_t f5_dit_ln_tab_ld(const f5_dit_weights* w) { return w ? ln_tab_ld(w) : 0; }

extern "C" int f5_dit_precompute(const f5_dit_weights* w, const f5_dit_buffers* b, void* stream_) {
  if (int e = device_check()) return e;
  if (int e = check_common(w, b)) return e;
  cudaStream_t st = (cudaStream_t)stream_;
  const int D = w->dim, N = b->frames, B = b->batch;
  const int BU = (b->cfg ? 2 : 1) * B;  // row-utterances
  const int R = BU * N;
  const int C = w->text_dim, Ci = w->text_inner;

  // ---- TextEmbedding (dit.py:196-229) for the cond rows and, with CFG, the text-dropped rows ----
  if (int e = launch_text_embed_gather(b->text, B, b->text_len_max, N, C, w->text_emb, w->text_pos,
                                       w->text_max_pos, b->text_x, BU,
                                       b->cfg ? B : ((b->drop_flags & 2) ? 0 : BU), st))
    return e;
  for (int l = 0; l < w->conv_layers; ++l) {
    const f5_convnext_weights& cw = w->text_blocks[l];
    if (int e = launch_dwconv7_ln(b->text_x, b->text_a, BU, N, C, cw.dw_w, cw.dw_b, cw.ln_w, cw.ln_b, st))
      return e;
    {  // pwconv1 + exact GELU (convnext_v2.py:50-51)
      f5_gemm_args g = gemm_base(b->text_a, C, cw.pw1_w, C, R, Ci, C, b->text_h, Ci, true);
      g.bias = cw.pw1_b; g.act = F5_ACT_GELU_ERF;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    if (int e = launch_grn(b->text_h, b->text_g, b->grn_nx, cw.grn_gamma, cw.grn_beta, BU, N, Ci, st, b->valid_len))
      return e;
    {  // pwconv2 + residual, then the re-mask of dit.py:225 (masked rows have a zero residual)
      f5_gemm_args g = gemm_base(b->text_g, Ci, cw.pw2_w, Ci, R, C, Ci, b->text_x, C, false);
      g.bias = cw.pw2_b; g.resid = b->text_x; g.ldr = C;
      g.rows_per_batch = N; g.num_batches = BU; g.row_len = b->text_len;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
  }

  // ---- hoisted part of InputEmbedding.proj (dit.py:248-249): [cond | text] · W[:,100:]^T + b ----
  if (int e = launch_concat_cond_text(b->cond, w->mel_dim, B, N, b->text_x, C, b->ct_bf16, w->ct_ld,
                                      R, b->cfg ? B * N : ((b->drop_flags & 1) ? 0 : R), st))
    return e;
  {
    f5_gemm_args g = gemm_base(b->ct_bf16, w->ct_ld, w->in_ct_w, w->ct_ld, R, D, w->ct_ld, b->hoist, D, false);
    g.bias = w->in_b;
    if (b->valid_len) { g.rows_per_batch = N; g.num_batches = BU; g.row_len = b->valid_len; }   // bucket rows stay 0
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }

  // ---- TimestepEmbedding for every evaluation time, then ALL AdaLN linears as one GEMM ----
  if (int e = launch_time_mlp(b->tvals, b->n_times, D, w->time_w0, w->time_b0, w->time_w2,
                              w->time_b2, nullptr, b->silu_t, st))
    return e;
  {
    const int NM = w->depth * 6 * D + 2 * D;
    f5_gemm_args g = gemm_base(b->silu_t, D, w->mod_w, D, b->n_times, NM, D, b->mod_table, NM, false);
    g.bias = w->mod_b;
    g.tile_n = 128;
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  // ---- fused AdaLN: c1 = (1 + scale) W^T and c2 = shift W^T of every consuming Linear, for all times ----
  if (ln_fused(b)) {
    const int NM = w->depth * 6 * D + 2 * D, T = b->n_times, F = w->ff_inner;
    const long long ld = ln_tab_ld(w);
    if (int e = launch_ln_tab_prep(b->mod_table, b->ln_prep, T, w->depth, D, NM, st)) return e;
    const __nv_bfloat16* prep = reinterpret_cast<const __nv_bfloat16*>(b->ln_prep);
    for (int site = 0; site <= 2 * w->depth; ++site) {
      const int l = site >> 1;
      const void* wt; int n; long long off;
      if (site == 2 * w->depth) { wt = w->proj_w; n = w->mel_dim; off = (long long)w->depth * (3 * D + F); }
      else if (site & 1) { wt = w->blocks[l].ff1_w; n = F; off = (long long)l * (3 * D + F) + 3 * D; }
      else { wt = w->blocks[l].qkv_w; n = 3 * D; off = (long long)l * (3 * D + F); }
      f5_gemm_args g = gemm_base(prep + (size_t)site * 4 * T * D, D, wt, D, 4 * T, n, D, b->ln_tab + off, ld, false);
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
  }
  return 0;
}

extern "C" int f5_dit_forward(const f5_dit_weights* w, const f5_dit_buffers* b, int32_t ti,
                              void* stream_) {
  if (int e = device_check()) return e;
  if (int e = check_common(w, b)) return e;
  F5_REQUIRE(ti >= 0 && ti < b->n_times, "dit_forward: time_index %d out of [0,%d)", ti, b->n_times);
  cudaStream_t st = (cudaStream_t)stream_;
  const int D = w->dim, N = b->frames, F = w->ff_inner;
  const int BU = (b->cfg ? 2 : 1) * b->batch;
  const int R = BU * N;
  const int NM = w->depth * 6 * D + 2 * D;
  const float* mod = b->mod_table + (size_t)ti * NM;
  // weight prefetch chain: worthwhile while a GEMM's weights are comparable to its activations
  // (small batch); at large batch the activations evict them anyway and HBM is busy
  static int pf_env = -1;
  if (pf_env < 0) { const char* v = getenv("F5_PREFETCH"); pf_env = (v && v[0] == '0') ? 0 : 1; }
  const bool prefetch = pf_env && R <= 16384;
  const bool fused = ln_fused(b);
  // FP8 mode of the QKV / FF1 GEMMs: e4m3 operand written by the producing epilogue, e4m3 weights (per-tensor scale)
  const bool fp8 = fused && b->a_fp8 != nullptr && w->blocks[0].qkv_w8 != nullptr && w->blocks[0].ff1_w8 != nullptr;
  // ... and of the out-projection / FF2 (A = attention output / GELU output, written as e4m3 by their producers into the
  // first half of the bf16 buffers); F5_FP8_LEVEL=1 keeps those two in bf16 (A/B measurements)
  static int fp8_level = -1;
  if (fp8_level < 0) { const char* v = getenv("F5_FP8_LEVEL"); fp8_level = (v && v[0] == '1') ? 1 : 2; }
  const bool fp8b = fp8 && fp8_level >= 2 && w->blocks[0].out_w8 != nullptr && w->blocks[0].ff2_w8 != nullptr;
  static const GemmTune t_qkv = tune_of("qkv"), t_out = tune_of("out"), t_ff1 = tune_of("ff1"), t_ff2 = tune_of("ff2");
  const long long tab_ld = ln_tab_ld(w);
  const float* tab = fused ? b->ln_tab + (size_t)4 * ti * tab_ld : nullptr;   // this time's 4 operand rows

  // ---- InputEmbedding (dit.py:249-251): x·Wx + hoist, then + ConvPositionEmbedding ----
  {
    f5_gemm_args g = gemm_base(b->y_bf16, 128, w->in_x_w, 128, R, D, 128, b->h, D, false);
    g.resid = b->hoist; g.ldr = D;
    g.out2_bf16 = b->a_bf16; g.ldo2 = D;
    // bucket rows (>= valid_len): x·Wx masked to 0 + hoist (0 there) = 0 — the conv below sees the reference's zero padding
    if (b->valid_len) { g.rows_per_batch = N; g.num_batches = BU; g.row_len = b->valid_len; }
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  {
    f5_gemm_args g = gemm_base(b->a_bf16, D, w->conv_w[0], 31 * 64, R, D, 64, b->c_bf16, D, true);
    g.bias = w->conv_b[0]; g.act = F5_ACT_MISH;
    g.rows_per_batch = N; g.num_batches = BU; g.batched_tiles = 1;
    g.conv_taps = 31; g.conv_pad = 15; g.conv_grouped = 1;
    g.row_len = b->valid_len;      // NULL, or: the second conv's input is zero on bucket rows too
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  {
    f5_gemm_args g = gemm_base(b->c_bf16, D, w->conv_w[1], 31 * 64, R, D, 64, b->x, D, false);
    g.bias = w->conv_b[1]; g.act = F5_ACT_MISH;
    g.rows_per_batch = N; g.num_batches = BU; g.batched_tiles = 1;
    g.conv_taps = 31; g.conv_pad = 15; g.conv_grouped = 1;
    g.resid = b->h; g.ldr = D;
    if (fused) {   // the stream's first producer: operand + statistics for block 0's attn_norm
      g.ln_scale = (w->depth > 0 ? mod + D : mod + (size_t)w->depth * 6 * D); g.ln_stats = b->ln_stats;
      g.out2_bf16 = fp8 ? b->a_fp8 : b->a_bf16; g.ldo2 = D; g.out2_fp8 = fp8 ? 1 : 0;
    }
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }

  // ---- transformer blocks (dit.py:311-325) ----
  for (int l = 0; l < w->depth; ++l) {
    const f5_dit_block_weights& bw = w->blocks[l];
    const float* m = mod + (size_t)l * 6 * D;  // shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp
    if (!fused)
      if (int e = launch_ln_modulate(b->x, b->a_bf16, R, D, 0, m + D, m, 0, 1, st)) return e;
    {
      f5_gemm_args g = gemm_base(b->a_bf16, D, bw.qkv_w, D, R, 3 * D, D, b->qkv_bf16, 3 * D, true);
      g.bias = bw.qkv_b;
      if (fused) { g.ln_in_stats = b->ln_stats; g.ln_tab = tab + (size_t)l * (3 * D + F); g.ln_tab_ld = tab_ld; }
      if (fp8) { g.a = b->a_fp8; g.w = bw.qkv_w8; g.ab_fp8 = 1; g.acc_scale = bw.qkv_s8; }
      g.variant = t_qkv.variant; g.tile_n = t_qkv.tile_n;
      g.rows_per_batch = N; g.num_batches = BU;
      g.rope = b->rope; g.rope_cols = 2 * D; g.q_scale = 0.125f; g.q_cols = D;
      // weight prefetch chain (L2): while QKV runs, pull in out_w and ff1_w (contiguous in the pack)
      if (prefetch) { g.prefetch = bw.out_w; g.prefetch_bytes = (int64_t)2 * D * D; }
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    if (int e = (fp8b ? f5_attention_fwd_e4m3 : f5_attention_fwd)(b->qkv_bf16, 3 * D, b->c_bf16, D, BU, N, w->heads, 64,
                                                                  b->seq_len ? b->seq_len : b->valid_len, st))
      return e;
    {
      f5_gemm_args g = gemm_base(b->c_bf16, D, bw.out_w, D, R, D, D, b->x, D, false);
      g.bias = bw.out_b;
      g.rows_per_batch = N; g.num_batches = BU; g.row_len = b->seq_len;
      g.gate = m + 2 * D; g.gate_ld = 0;
      g.resid = b->x; g.ldr = D;
      if (prefetch) { g.prefetch = bw.ff1_w; g.prefetch_bytes = (int64_t)2 * F * D; }
      if (fused) {   // ff_norm
        g.ln_scale = m + 4 * D; g.ln_stats = b->ln_stats;
        g.out2_bf16 = fp8 ? b->a_fp8 : b->a_bf16; g.ldo2 = D; g.out2_fp8 = fp8 ? 1 : 0;
      }
      if (fp8b) { g.w = bw.out_w8; g.ab_fp8 = 1; g.acc_scale = bw.out_s8; }     // A = c_bf16's bytes, e4m3 [R, D]
      g.variant = t_out.variant; g.tile_n = t_out.tile_n;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    if (!fused)
      if (int e = launch_ln_modulate(b->x, b->a_bf16, R, D, 0, m + 4 * D, m + 3 * D, 0, 1, st)) return e;
    {
      f5_gemm_args g = gemm_base(b->a_bf16, D, bw.ff1_w, D, R, F, D, b->ff_bf16, F, true);
      g.bias = bw.ff1_b; g.act = F5_ACT_GELU_TANH;
      if (fused) { g.ln_in_stats = b->ln_stats; g.ln_tab = tab + (size_t)l * (3 * D + F) + 3 * D; g.ln_tab_ld = tab_ld; }
      if (fp8) { g.a = b->a_fp8; g.w = bw.ff1_w8; g.ab_fp8 = 1; g.acc_scale = bw.ff1_s8; }
      if (fp8b) g.out_fp8 = 1;                                                   // ff_bf16's bytes as e4m3 [R, F]
      g.variant = t_ff1.variant; g.tile_n = t_ff1.tile_n;
      if (prefetch) { g.prefetch = bw.ff2_w; g.prefetch_bytes = (int64_t)2 * D * F; }
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    {
      f5_gemm_args g = gemm_base(b->ff_bf16, F, bw.ff2_w, F, R, D, F, b->x, D, false);
      g.bias = bw.ff2_b;
      g.rows_per_batch = N; g.num_batches = BU;
      g.gate = m + 5 * D; g.gate_ld = 0;
      g.resid = b->x; g.ldr = D;
      if (prefetch && l + 1 < w->depth) {
        g.prefetch = w->blocks[l + 1].qkv_w; g.prefetch_bytes = (int64_t)2 * 3 * D * D;
      }
      if (fused) {   // next block's attn_norm scale, or norm_out's (scale first, dit.py:287)
        g.ln_scale = (l + 1 < w->depth) ? mod + (size_t)(l + 1) * 6 * D + D : mod + (size_t)w->depth * 6 * D;
        g.ln_stats = b->ln_stats; g.out2_bf16 = b->a_bf16; g.ldo2 = D;
        if (fp8 && l + 1 < w->depth) { g.out2_bf16 = b->a_fp8; g.out2_fp8 = 1; }   // proj_out (after the last block) stays bf16
      }
      if (fp8b) { g.w = bw.ff2_w8; g.ab_fp8 = 1; g.acc_scale = bw.ff2_s8; }
      g.variant = t_ff2.variant; g.tile_n = t_ff2.tile_n;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
  }

  // ---- AdaLayerNormZero_Final (scale first, dit.py:287) + proj_out (dit.py:398-399) ----
  {
    const float* mf = mod + (size_t)w->depth * 6 * D;
    if (!fused)
      if (int e = launch_ln_modulate(b->x, b->a_bf16, R, D, 0, mf, mf + D, 0, 1, st)) return e;
    f5_gemm_args g = gemm_base(b->a_bf16, D, w->proj_w, D, R, w->mel_dim, D, b->v, w->mel_dim, false);
    g.bias = w->proj_b;
    if (fused) { g.ln_in_stats = b->ln_stats; g.ln_tab = tab + (size_t)w->depth * (3 * D + F); g.ln_tab_ld = tab_ld; }
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  return 0;
}

// Evaluation times in the order the solvers call fn (cfm.py:50-59, 76-89, 106-120), computed in
// fp32 exactly as the reference does (t_current + 0.5 * dt etc.).
extern "C" int f5_ode_eval_times(const float* t, int32_t steps, int32_t method, float* out,
                                 int32_t cap) {
  F5_REQUIRE(t && steps >= 2, "ode_eval_times: need >= 2 grid points");
  F5_REQUIRE(method >= 0 && method <= 2, "ode_eval_times: unknown method %d", method);
  const int per = method == 0 ? 1 : (method == 1 ? 2 : 4);
  const int n = (steps - 1) * per;
  if (out == nullptr) return n;
  F5_REQUIRE(cap >= n, "ode_eval_times: capacity %d < %d", cap, n);
  int k = 0;
  for (int i = 0; i + 1 < steps; ++i) {
    const float tc = t[i];
    const float dt = t[i + 1] - tc;
    out[k++] = tc;
    if (method == 1) {
      out[k++] = tc + 0.5f * dt;
    } else if (method == 2) {
      out[k++] = tc + 0.5f * dt;
      out[k++] = tc + 0.5f * dt;
      out[k++] = tc + dt;
    }
  }
  return n;
}

extern "C" int f5_ode_sample(const f5_dit_weights* w, const f5_dit_buffers* b, const float* t,
                             int32_t steps, int32_t method, float cfg_strength, float* y,
                             float* trajectory, float* scratch, void* stream_) {
  if (int e = device_check()) return e;
  if (int e = check_common(w, b)) return e;
  F5_REQUIRE(t && steps >= 2 && y, "ode_sample: bad arguments");
  F5_REQUIRE(method >= 0 && method <= 2, "ode_sample: unknown method %d", method);
  F5_REQUIRE((cfg_strength >= 1e-5f) == (b->cfg != 0),
             "ode_sample: buffers built with cfg=%d but cfg_strength=%g", b->cfg, cfg_strength);
  const int per = method == 0 ? 1 : (method == 1 ? 2 : 4);
  F5_REQUIRE(b->n_times == (steps - 1) * per, "ode_sample: n_times %d != %d", b->n_times,
             (steps - 1) * per);
  F5_REQUIRE(method == 0 || scratch, "ode_sample: scratch required for midpoint/rk4");
  cudaStream_t st = (cudaStream_t)stream_;
  const int BN = b->batch * b->frames, d = w->mel_dim;
  const size_t state = (size_t)BN * d;
  const long long dup = b->cfg ? BN : 0;

  // A operand of the first x-projection: bf16(y0), both CFG halves
  const float* y_cur = trajectory ? trajectory : y;
  if (int e = launch_cast_pad_bf16(y_cur, d, b->y_bf16, 128, BN, dup, st)) return e;

  OdeUpdateParams u;
  memset(&u, 0, sizeof(u));
  u.v = b->v; u.ldv = d; u.null_row_offset = dup; u.cfg_strength = cfg_strength;
  u.y_bf16 = reinterpret_cast<__nv_bfloat16*>(b->y_bf16); u.ld_bf16 = 128;
  u.bf16_copy_row_offset = dup;
  u.rows = BN; u.d = d;
  float* y_tmp = scratch;
  float* k_acc = scratch ? scratch + state : nullptr;

  int ti = 0;
  for (int i = 0; i + 1 < steps; ++i) {
    const float dt = t[i + 1] - t[i];
    float* y_next = trajectory ? trajectory + (size_t)(i + 1) * state : y;
    u.y_base = y_cur;
    if (method == 0) {
      if (int e = f5_dit_forward(w, b, ti++, st)) return e;
      u.y_out = y_next; u.a = dt; u.k_acc = nullptr; u.use_acc = 0;
      if (int e = launch_ode_update(u, st)) return e;
    } else if (method == 1) {
      if (int e = f5_dit_forward(w, b, ti++, st)) return e;
      u.y_out = y_tmp; u.a = 0.5f * dt; u.k_acc = nullptr; u.use_acc = 0;
      if (int e = launch_ode_update(u, st)) return e;
      if (int e = f5_dit_forward(w, b, ti++, st)) return e;
      u.y_out = y_next; u.a = dt;
      if (int e = launch_ode_update(u, st)) return e;
    } else {
      const float as[4] = {0.5f * dt, 0.5f * dt, dt, dt / 6.f};
      const float ws[4] = {1.f, 2.f, 2.f, 1.f};
      for (int s = 0; s < 4; ++s) {
        if (int e = f5_dit_forward(w, b, ti++, st)) return e;
        u.k_acc = k_acc; u.acc_w = ws[s]; u.acc_init = (s == 0); u.use_acc = (s == 3);
        u.y_out = (s == 3) ? y_next : y_tmp; u.a = as[s];
        if (int e = launch_ode_update(u, st)) return e;
      }
    }
    y_cur = y_next;
  }
  return 0;
}
