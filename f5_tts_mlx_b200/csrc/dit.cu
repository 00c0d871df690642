// DiT forward and the ODE loop of F5TTS.sample as a stream-ordered sequence of the sm_90a kernels
// in this directory (C-ABI: f5_dit_precompute / f5_dit_forward / f5_ode_sample).
//
// What the reference recomputes on every forward but depends only on (text, cond, t) is hoisted:
//   * TextEmbedding (dit.py:390)                      -> once per sample, per CFG branch
//   * cond·Wc + text·Wt + b of InputEmbedding.proj    -> once per sample (dit.py:249)
//   * TimestepEmbedding + all 23 AdaLN linears         -> one GEMM over all time points (dit.py:389,267,286)
// and the two unbatched CFG passes (cfm.py:342-363) run as one forward over a doubled batch.
#include <string.h>

#include <initializer_list>

#include "host_common.h"
#include "launch.h"

namespace f5 {

f5_gemm_args gemm_args(const void* a, int64_t lda, const void* w, int64_t ldw, int m, int n, int k, void* out,
                       int64_t ldo, bool out_bf16, bool w_static) {
  f5_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.a = a; g.lda = lda; g.w = w; g.ldw = ldw;
  g.m = m; g.n = n; g.k = k;
  g.num_batches = 1;
  g.conv_taps = 1;
  g.out = out; g.ldo = ldo; g.out_bf16 = out_bf16 ? 1 : 0;
  g.q_scale = 1.f;
  g.w_static = w_static ? 1 : 0;
  return g;
}

f5_gemm_args conv_pos_args(const void* a, const void* w, const float* bias, void* out, bool out_bf16, int D, int N,
                           int batches, bool w_static) {
  f5_gemm_args g = gemm_args(a, D, w, 31 * 64, batches * N, D, 64, out, D, out_bf16, w_static);
  g.bias = bias; g.act = F5_ACT_MISH;
  g.rows_per_batch = N; g.num_batches = batches; g.batched_tiles = 1;
  g.conv_taps = 31; g.conv_pad = 15; g.conv_grouped = 1;
  return g;
}

template <typename Weights, typename Buffers>
int text_embedding(const Weights* w, const Buffers* b, int batch_out, int drop_from, int mask_padding,
                   const int* valid_len, const int* row_len, bool w_static, cudaStream_t st) {
  const int N = b->frames, R = batch_out * N, C = w->text_dim, Ci = w->text_inner;
  if (int e = launch_text_embed_gather(b->text, b->batch, b->text_len_max, N, C, w->text_emb, w->text_pos,
                                       w->text_max_pos, b->text_x, batch_out, drop_from, st, mask_padding, valid_len))
    return e;
  for (int l = 0; l < w->conv_layers; ++l) {
    const f5_convnext_weights& cw = w->text_blocks[l];
    if (int e = launch_dwconv7_ln(b->text_x, b->text_a, batch_out, N, C, cw.dw_w, cw.dw_b, cw.ln_w, cw.ln_b, st))
      return e;
    {  // pwconv1 + exact GELU (convnext_v2.py:50-51)
      f5_gemm_args g = gemm_args(b->text_a, C, cw.pw1_w, C, R, Ci, C, b->text_h, Ci, true, w_static);
      g.bias = cw.pw1_b; g.act = F5_ACT_GELU_ERF;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    if (int e = launch_grn(b->text_h, b->text_g, b->grn_nx, cw.grn_gamma, cw.grn_beta, batch_out, N, Ci, st,
                           valid_len))
      return e;
    {  // pwconv2 + residual, then the re-mask of dit.py:225 (masked rows have a zero residual)
      f5_gemm_args g = gemm_args(b->text_g, Ci, cw.pw2_w, Ci, R, C, Ci, b->text_x, C, false, w_static);
      g.bias = cw.pw2_b; g.resid = b->text_x; g.ldr = C;
      if (row_len) { g.rows_per_batch = N; g.num_batches = batch_out; g.row_len = row_len; }
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
  }
  return 0;
}
template int text_embedding(const f5_dit_weights*, const f5_dit_buffers*, int, int, int, const int*, const int*, bool,
                            cudaStream_t);
template int text_embedding(const f5_duration_weights*, const f5_duration_buffers*, int, int, int, const int*,
                            const int*, bool, cudaStream_t);

// What f5_dit_forward runs, chosen by the buffers the caller binds (see f5_dit_buffers in include/f5_b200.h)
struct DitMode {
  bool fused;   // AdaLN LayerNorm folded into the GEMM epilogues (ln_stats / ln_tab / ln_prep)
  bool fp8;     // the four block GEMMs on e4m3 operands (a_fp8)
  bool blk8;    // ... with block scales (a_fp8_scale / attn_scale / ff_scale)
  bool attn8;   // ... and the attention on e4m3 Q, K, V (qk_fp8 / vt_fp8 / qkv_scale)
};

struct NamedPtr { const char* name; const void* p; };
// 0 when every pointer of `ptrs` is set, else F5_ERR_INVALID naming the NULL ones (of blocks[block] when block >= 0)
static int need_all(const char* mode, int block, std::initializer_list<NamedPtr> ptrs) {
  char missing[128] = "";
  for (const NamedPtr& n : ptrs) {
    const size_t len = strlen(missing);
    if (n.p == nullptr) snprintf(missing + len, sizeof(missing) - len, "%s%s", len ? ", " : "", n.name);
  }
  if (missing[0] == 0) return 0;
  if (block < 0) return set_error(F5_ERR_INVALID, "dit: %s needs %s", mode, missing);
  return set_error(F5_ERR_INVALID, "dit: %s needs %s of blocks[%d]", mode, missing, block);
}

// A partly bound mode is an error rather than a quiet fall-back to another mode.
static int check_mode(const f5_dit_weights* w, const f5_dit_buffers* b, DitMode& m) {
  m.fused = b->ln_stats || b->ln_tab || b->ln_prep;
  m.blk8 = b->a_fp8_scale || b->attn_scale || b->ff_scale;
  m.fp8 = b->a_fp8 || m.blk8;
  if (m.fused)
    if (int e = need_all("fused AdaLN", -1, {{"ln_stats", b->ln_stats}, {"ln_tab", b->ln_tab}, {"ln_prep", b->ln_prep}}))
      return e;
  if (m.fp8) {
    F5_REQUIRE(m.fused, "dit: FP8 needs the fused AdaLN buffers ln_stats, ln_tab and ln_prep");
    if (int e = need_all("FP8", -1, {{"a_fp8", b->a_fp8}})) return e;
  }
  if (m.blk8)
    if (int e = need_all("block-scaled FP8", -1, {{"a_fp8_scale", b->a_fp8_scale}, {"attn_scale", b->attn_scale},
                                                  {"ff_scale", b->ff_scale}}))
      return e;
  m.attn8 = b->qk_fp8 || b->vt_fp8 || b->qkv_scale;
  if (m.attn8) {
    if (int e = need_all("FP8 attention", -1, {{"qk_fp8", b->qk_fp8}, {"vt_fp8", b->vt_fp8}, {"qkv_scale", b->qkv_scale}}))
      return e;
    F5_REQUIRE(m.blk8, "dit: FP8 attention needs the block-scaled FP8 mode (a_fp8_scale, attn_scale and ff_scale)");
  }
  for (int l = 0; m.fp8 && l < w->depth; ++l) {
    const f5_dit_block_weights& bw = w->blocks[l];
    if (int e = need_all("FP8", l, {{"qkv_w8", bw.qkv_w8}, {"ff1_w8", bw.ff1_w8}, {"out_w8", bw.out_w8},
                                    {"ff2_w8", bw.ff2_w8}}))
      return e;
    // per-channel scales without the block-scale buffers would run the per-tensor mode on per-channel weights
    F5_REQUIRE(m.blk8 || !(bw.qkv_ws || bw.ff1_ws || bw.out_ws || bw.ff2_ws),
               "dit: blocks[%d] has per-channel weight scales (*_ws): block-scaled FP8 needs a_fp8_scale, attn_scale "
               "and ff_scale", l);
    if (m.blk8)
      if (int e = need_all("block-scaled FP8", l, {{"qkv_ws", bw.qkv_ws}, {"ff1_ws", bw.ff1_ws}, {"out_ws", bw.out_ws},
                                                   {"ff2_ws", bw.ff2_ws}}))
        return e;
  }
  return 0;
}

static int check_common(const f5_dit_weights* w, const f5_dit_buffers* b, DitMode& mode) {
  F5_REQUIRE(w && b, "dit: null weights/buffers");
  // the implicit grouped conv reads 64-channel blocks, so each of its 16 groups (dim/16 channels) must lie inside one
  // block: dim/16 divides 64, which within 256..1024 leaves 256, 512 and 1024
  F5_REQUIRE(w->dim % 128 == 0 && w->dim >= 256 && w->dim <= 1024 && 64 % (w->dim / 16) == 0,
             "dit: dim %d unsupported (256, 512 or 1024: the conv's dim/16-channel groups must tile 64-channel blocks)",
             w->dim);
  F5_REQUIRE(w->dim == w->heads * 64, "dit: dim %d != heads %d * 64", w->dim, w->heads);
  F5_REQUIRE(w->mel_dim % 4 == 0 && w->mel_dim <= 128, "dit: mel_dim %d", w->mel_dim);
  F5_REQUIRE(w->blocks && w->depth > 0, "dit: no blocks");
  F5_REQUIRE(b->batch > 0 && b->frames > 0 && b->n_times > 0, "dit: bad buffer shape");
  return check_mode(w, b, mode);
}

static long long ln_tab_ld(const f5_dit_weights* w) {
  return (long long)w->depth * (3 * w->dim + w->ff_inner) + 128;
}

// What one of a block's four GEMMs reads in the current mode
struct GemmOperands {
  const void* a;
  const void* w;             // the bf16 weight, or its e4m3 copy
  int ab_fp8;
  float acc_scale;           // per-tensor FP8: the weight's scale; block-scaled: 1; bf16: unused (0)
  const float* a_scale;      // block-scaled FP8: A's per-(row, 64-column unit) scales
  const float* w_scale;      // block-scaled FP8: the weight's per-channel scales
  const void* prefetch;      // weights of the next GEMM to pull into L2, or NULL
  int64_t prefetch_bytes;
};
struct BlockOperands { GemmOperands qkv, out, ff1, ff2; };

// FP8 mode: the QKV / FF1 operand is written as e4m3 by the producing epilogue, the out-projection / FF2 operand
// (attention output / GELU output) by its producer into the first half of the bf16 buffer.  Block-scaled FP8
// (DESIGN.md section 8) adds per-channel weight scales and per-(row, 64-column unit) activation scales.
static BlockOperands block_operands(const f5_dit_weights* w, const f5_dit_buffers* b, const DitMode& m, int l,
                                    bool prefetch) {
  const f5_dit_block_weights& k = w->blocks[l];
  auto pick = [&](const void* a16, const void* a8, const void* w16, const void* w8, float s8, const float* ws,
                  const float* a_scale) {
    GemmOperands o = {};
    o.a = m.fp8 ? a8 : a16;
    o.w = m.fp8 ? w8 : w16;
    o.ab_fp8 = m.fp8 ? 1 : 0;
    o.acc_scale = m.blk8 ? 1.f : m.fp8 ? s8 : 0.f;
    if (m.blk8) { o.a_scale = a_scale; o.w_scale = ws; }
    return o;
  };
  BlockOperands o = {pick(b->a_bf16, b->a_fp8, k.qkv_w, k.qkv_w8, k.qkv_s8, k.qkv_ws, b->a_fp8_scale),
                     pick(b->c_bf16, b->c_bf16, k.out_w, k.out_w8, k.out_s8, k.out_ws, b->attn_scale),
                     pick(b->a_bf16, b->a_fp8, k.ff1_w, k.ff1_w8, k.ff1_s8, k.ff1_ws, b->a_fp8_scale),
                     pick(b->ff_bf16, b->ff_bf16, k.ff2_w, k.ff2_w8, k.ff2_s8, k.ff2_ws, b->ff_scale)};
  // weight prefetch chain (L2): each GEMM pulls in the next one's weights, FF2 the next block's QKV weights.
  // The per-tensor FP8 mode prefetches the bf16 copies, which it does not read.
  auto fetch = [&](GemmOperands& g, const void* w16, const void* w8, int64_t elems) {
    if (!prefetch) return;
    g.prefetch = m.blk8 ? w8 : w16;
    g.prefetch_bytes = m.blk8 ? elems : 2 * elems;
  };
  const int64_t D = w->dim, F = w->ff_inner;
  fetch(o.qkv, k.out_w, k.out_w8, D * D);
  fetch(o.out, k.ff1_w, k.ff1_w8, F * D);
  fetch(o.ff1, k.ff2_w, k.ff2_w8, D * F);
  if (l + 1 < w->depth) fetch(o.ff2, w->blocks[l + 1].qkv_w, w->blocks[l + 1].qkv_w8, 3 * D * D);
  return o;
}

// A [m, k] and W [n, k] dense
static f5_gemm_args block_gemm(const GemmOperands& o, int m, int n, int k, void* out, int64_t ldo, bool out_bf16) {
  f5_gemm_args g = gemm_args(o.a, k, o.w, k, m, n, k, out, ldo, out_bf16, true);
  g.ab_fp8 = o.ab_fp8; g.acc_scale = o.acc_scale;
  if (o.a_scale) { g.a_scale = o.a_scale; g.a_scale_ld = m; }
  g.w_scale = o.w_scale;
  g.prefetch = o.prefetch; g.prefetch_bytes = o.prefetch_bytes;
  return g;
}

// Fused AdaLN, producer side: the GEMM writing the residual stream also writes the next LayerNorm's operand
// x * (1 + ln_scale), as e4m3 (with its block scales in the block-scaled mode) when the next GEMM reads e4m3
static void ln_producer(f5_gemm_args& g, const DitMode& m, const f5_dit_buffers* b, int D, const float* ln_scale,
                        bool e4m3) {
  if (!m.fused) return;
  g.ln_scale = ln_scale; g.ln_stats = b->ln_stats;
  g.out2_bf16 = e4m3 ? b->a_fp8 : b->a_bf16; g.ldo2 = D; g.out2_fp8 = e4m3 ? 1 : 0;
  if (e4m3 && m.blk8) g.out2_scale = b->a_fp8_scale;
}

// Fused AdaLN, consumer side: the GEMM normalises its A operand with the producer's statistics and the c1 / c2 rows of
// time ti, from ln_tab column `col` on
static void ln_consumer(f5_gemm_args& g, const DitMode& m, const f5_dit_weights* w, const f5_dit_buffers* b, int ti,
                        long long col) {
  if (!m.fused) return;
  g.ln_in_stats = b->ln_stats; g.ln_tab = b->ln_tab + (size_t)4 * ti * ln_tab_ld(w) + col; g.ln_tab_ld = ln_tab_ld(w);
}

// attention of b->qkv_bf16 into b->c_bf16: bf16 output, or e4m3 for the FP8 modes' out-projection
static int attention(const f5_dit_weights* w, const f5_dit_buffers* b, const DitMode& m, int BU, cudaStream_t st) {
  const int D = w->dim, N = b->frames;
  const int32_t* kv_len = b->seq_len ? b->seq_len : b->valid_len;   // the pass and the attention mask alike
  if (m.attn8) {
    const int64_t vt_ld = (int64_t)cdiv(N, 128) * 128;
    if (int e = f5_qkv_quant_e4m3_masked(b->qkv_bf16, 3 * D, b->qk_fp8, 2 * D, b->vt_fp8, vt_ld, b->qkv_scale, BU, N,
                                         w->heads, kv_len, st))
      return e;
    return f5_attention_fwd_fp8(b->qk_fp8, 2 * D, b->vt_fp8, vt_ld, b->qkv_scale, b->c_bf16, D, BU, N, w->heads, 64,
                                kv_len, b->attn_scale, st);
  }
  if (m.blk8)
    return f5_attention_fwd_e4m3_scaled(b->qkv_bf16, 3 * D, b->c_bf16, D, BU, N, w->heads, 64, kv_len, b->attn_scale,
                                        st);
  return (m.fp8 ? f5_attention_fwd_e4m3 : f5_attention_fwd)(b->qkv_bf16, 3 * D, b->c_bf16, D, BU, N, w->heads, 64,
                                                            kv_len, st);
}

}  // namespace f5

using namespace f5;

extern "C" int64_t f5_dit_ln_tab_ld(const f5_dit_weights* w) { return w ? ln_tab_ld(w) : 0; }

extern "C" int f5_dit_precompute(const f5_dit_weights* w, const f5_dit_buffers* b, void* stream_) {
  if (int e = device_check()) return e;
  DitMode mode;
  if (int e = check_common(w, b, mode)) return e;
  cudaStream_t st = (cudaStream_t)stream_;
  const int D = w->dim, N = b->frames, B = b->batch;
  const int BU = (b->cfg ? 2 : 1) * B;  // row-utterances
  const int R = BU * N;
  const int C = w->text_dim;

  // ---- TextEmbedding (dit.py:196-229) for the cond rows and, with CFG, the text-dropped rows ----
  if (int e = text_embedding(w, b, BU, b->cfg ? B : ((b->drop_flags & 2) ? 0 : BU), 1, b->valid_len, b->text_len,
                             true, st))
    return e;

  // ---- hoisted part of InputEmbedding.proj (dit.py:248-249): [cond | text] · W[:,100:]^T + b ----
  if (int e = launch_concat_cond_text(b->cond, w->mel_dim, B, N, b->text_x, C, b->ct_bf16, w->ct_ld,
                                      R, b->cfg ? B * N : ((b->drop_flags & 1) ? 0 : R), st))
    return e;
  {
    f5_gemm_args g = gemm_args(b->ct_bf16, w->ct_ld, w->in_ct_w, w->ct_ld, R, D, w->ct_ld, b->hoist, D, false, true);
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
    f5_gemm_args g = gemm_args(b->silu_t, D, w->mod_w, D, b->n_times, NM, D, b->mod_table, NM, false, true);
    g.bias = w->mod_b;
    g.tile_n = 128;
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  // ---- fused AdaLN: c1 = (1 + scale) W^T and c2 = shift W^T of every consuming Linear, for all times ----
  if (mode.fused) {
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
      f5_gemm_args g =
          gemm_args(prep + (size_t)site * 4 * T * D, D, wt, D, 4 * T, n, D, b->ln_tab + off, ld, false, true);
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
  }
  return 0;
}

extern "C" int f5_dit_forward(const f5_dit_weights* w, const f5_dit_buffers* b, int32_t ti,
                              void* stream_) {
  if (int e = device_check()) return e;
  DitMode mode;
  if (int e = check_common(w, b, mode)) return e;
  F5_REQUIRE(ti >= 0 && ti < b->n_times, "dit_forward: time_index %d out of [0,%d)", ti, b->n_times);
  cudaStream_t st = (cudaStream_t)stream_;
  const int D = w->dim, N = b->frames, F = w->ff_inner;
  const int BU = (b->cfg ? 2 : 1) * b->batch;
  const int R = BU * N;
  const int NM = w->depth * 6 * D + 2 * D;
  const float* mod = b->mod_table + (size_t)ti * NM;
  // weight prefetch chain: worthwhile while a GEMM's weights are comparable to its activations
  // (small batch); at large batch the activations evict them anyway and HBM is busy
  const bool prefetch = R <= 16384;

  // ---- InputEmbedding (dit.py:249-251): x·Wx + hoist, then + ConvPositionEmbedding ----
  {
    f5_gemm_args g = gemm_args(b->y_bf16, 128, w->in_x_w, 128, R, D, 128, b->h, D, false, true);
    g.resid = b->hoist; g.ldr = D;
    g.out2_bf16 = b->a_bf16; g.ldo2 = D;
    // bucket rows (>= valid_len): x·Wx masked to 0 + hoist (0 there) = 0 — the conv below sees the reference's zero padding
    if (b->valid_len) { g.rows_per_batch = N; g.num_batches = BU; g.row_len = b->valid_len; }
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  {
    f5_gemm_args g = conv_pos_args(b->a_bf16, w->conv_w[0], w->conv_b[0], b->c_bf16, true, D, N, BU, true);
    g.row_len = b->valid_len;      // NULL, or: the second conv's input is zero on bucket rows too
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  {
    f5_gemm_args g = conv_pos_args(b->c_bf16, w->conv_w[1], w->conv_b[1], b->x, false, D, N, BU, true);
    g.resid = b->h; g.ldr = D;
    ln_producer(g, mode, b, D, mod + D, mode.fp8);   // the stream's first producer: block 0's attn_norm
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }

  // ---- transformer blocks (dit.py:311-325) ----
  for (int l = 0; l < w->depth; ++l) {
    const f5_dit_block_weights& bw = w->blocks[l];
    const BlockOperands op = block_operands(w, b, mode, l, prefetch);
    const float* m = mod + (size_t)l * 6 * D;  // shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp
    const bool last = l + 1 == w->depth;
    if (!mode.fused)
      if (int e = launch_ln_modulate(b->x, b->a_bf16, R, D, 0, m + D, m, 0, 1, st)) return e;
    {
      f5_gemm_args g = block_gemm(op.qkv, R, 3 * D, D, b->qkv_bf16, 3 * D, true);
      g.bias = bw.qkv_b;
      ln_consumer(g, mode, w, b, ti, (long long)l * (3 * D + F));
      g.rows_per_batch = N; g.num_batches = BU;
      g.rope = b->rope; g.rope_cols = 2 * D; g.q_scale = 0.125f; g.q_cols = D;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    if (int e = attention(w, b, mode, BU, st)) return e;
    {
      f5_gemm_args g = block_gemm(op.out, R, D, D, b->x, D, false);
      g.bias = bw.out_b;
      g.rows_per_batch = N; g.num_batches = BU; g.row_len = b->seq_len;
      g.gate = m + 2 * D;
      g.resid = b->x; g.ldr = D;
      ln_producer(g, mode, b, D, m + 4 * D, mode.fp8);   // ff_norm
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    if (!mode.fused)
      if (int e = launch_ln_modulate(b->x, b->a_bf16, R, D, 0, m + 4 * D, m + 3 * D, 0, 1, st)) return e;
    {
      f5_gemm_args g = block_gemm(op.ff1, R, F, D, b->ff_bf16, F, true);
      g.bias = bw.ff1_b; g.act = F5_ACT_GELU_TANH;
      ln_consumer(g, mode, w, b, ti, (long long)l * (3 * D + F) + 3 * D);
      g.out_fp8 = mode.fp8 ? 1 : 0;   // FP8: ff_bf16's bytes as e4m3 [R, F], FF2's operand
      g.out_scale = mode.blk8 ? b->ff_scale : nullptr;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    {
      f5_gemm_args g = block_gemm(op.ff2, R, D, F, b->x, D, false);
      g.bias = bw.ff2_b;
      g.rows_per_batch = N; g.num_batches = BU;
      g.gate = m + 5 * D;
      g.resid = b->x; g.ldr = D;
      // next block's attn_norm scale, or norm_out's (scale first, dit.py:287); proj_out's operand stays bf16
      ln_producer(g, mode, b, D, last ? mod + (size_t)w->depth * 6 * D : m + 6 * D + D, mode.fp8 && !last);
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
  }

  // ---- AdaLayerNormZero_Final (scale first, dit.py:287) + proj_out (dit.py:398-399) ----
  {
    const float* mf = mod + (size_t)w->depth * 6 * D;
    if (!mode.fused)
      if (int e = launch_ln_modulate(b->x, b->a_bf16, R, D, 0, mf, mf + D, 0, 1, st)) return e;
    f5_gemm_args g = gemm_args(b->a_bf16, D, w->proj_w, D, R, w->mel_dim, D, b->v, w->mel_dim, false, true);
    g.bias = w->proj_b;
    ln_consumer(g, mode, w, b, ti, (long long)w->depth * (3 * D + F));
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
  DitMode mode;
  if (int e = check_common(w, b, mode)) return e;
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
