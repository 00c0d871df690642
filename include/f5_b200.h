/*
 * f5_b200.h — C ABI of libf5b200.so, the H100 (sm_90a) implementation of the f5-tts-mlx hot path.
 *
 * The reference (lucasnewman/f5-tts-mlx) has no FFI/plugin boundary: it is pure Python on MLX, and
 * its "operators" are the mlx.nn / mx.fast calls inside f5_tts_mlx/{cfm,dit,convnext_v2,rope,audio}.py.
 * Each entry point below replaces one of those call sites (cited as file:line of the reference) and
 * is what a binding for that call site would bind.  Conventions:
 *
 *   - every function returns 0 on success or a negative F5_ERR_* code; f5_last_error() returns a
 *     thread-local message for the last failure on the calling thread;
 *   - the caller owns every buffer (weights, activations, workspace); nothing is allocated, no
 *     host synchronisation happens, every launch is ordered on `stream` (a cudaStream_t passed as
 *     void*), so a sequence of calls can be captured into a CUDA graph;
 *   - all pointers are DEVICE pointers unless the parameter name starts with `h_`;
 *   - activations are channels-last (rows = batch*frames, row-major), bf16 operands for the tensor
 *     cores ("bf16" below = __nv_bfloat16 bits), fp32 for the residual stream, statistics, softmax
 *     and ODE state.  Linear weights are (out_features, in_features) row-major bf16, exactly the
 *     reference's nn.Linear.weight layout.
 *   - there is NO CPU fallback: if no sm_90 device is present every compute entry point fails with
 *     F5_ERR_NO_DEVICE.
 */
#ifndef F5_H100_H_
#define F5_H100_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define F5_OK 0
#define F5_ERR_INVALID (-1)   /* bad argument (shape/alignment/null)            */
#define F5_ERR_CUDA (-2)      /* a CUDA runtime / driver call failed             */
#define F5_ERR_NO_DEVICE (-3) /* no sm_90 GPU: this library has no CPU path     */

const char* f5_last_error(void);
/* library/ABI version (major*1000+minor) and the device check used by every entry point */
int f5_abi_version(void);
int f5_device_check(void);
/* number of kernels this library has launched in this process (bench.py "gpu_launches") */
long long f5_launch_count(void);
/* sizeof() of the ABI structs in declaration order: f5_gemm_args, f5_convnext_weights,
 * f5_dit_block_weights, f5_dit_weights, f5_dit_buffers, f5_vocos_block_weights, f5_vocos_weights,
 * f5_vocos_buffers, f5_duration_weights, f5_duration_buffers — lets a binding check its layout at
 * load time.  Returns the count (10). */
int f5_struct_sizes(int32_t* out, int32_t n);
/* In-situ kernel timing inside a captured CUDA graph (bench.py's roofline): install a device buffer of max_slots x 2
 * uint64; from then on the i-th launched kernel of the tensor-core families (GEMM, attention) gets slot i and writes
 * [i][0] = min over its CTAs of %globaltimer after the dependency wait, [i][1] = max over CTAs at exit (the caller
 * presets the columns to UINT64_MAX / 0 before each replay).  f5_prof_graph_meta returns the family of every slot
 * handed out since the install (0 GEMM, 1 attention, 2 LayerNorm+modulate, 3 everything else) and its algorithmic
 * flops / bytes; slots = NULL uninstalls. */
int f5_prof_graph_begin(void* slots, int32_t max_slots);
int f5_prof_graph_meta(int32_t* kinds, double* flops, double* bytes, int32_t cap);

/* ------------------------------------------------------------------------------------------ *
 * Dense / implicit-conv GEMM on wgmma tensor cores:  out = epilogue(A · W^T)
 * Replaces every nn.Linear / nn.Conv1d on the path (dit.py:33-38,77,94-99,136-143,170,249,267,
 * 286,399; convnext_v2.py:35-44) together with the elementwise ops the reference applies to its
 * result (bias, GELU/Mish, RoPE rope.py:94-107, "* mask" dit.py:172-173, AdaLN gate + residual
 * dit.py:319,323).
 * ------------------------------------------------------------------------------------------ */
enum { F5_ACT_NONE = 0, F5_ACT_GELU_TANH = 1, F5_ACT_GELU_ERF = 2, F5_ACT_MISH = 3 };

typedef struct f5_gemm_args {
  /* operands */
  const void* a;      /* bf16 [rows, lda]; rows = M (flat) or num_batches*rows_per_batch        */
  int64_t lda;        /* elements, multiple of 8                                                */
  const void* w;      /* bf16 [N, ldw] (out_features major)                                     */
  int64_t ldw;        /* elements, multiple of 8                                                */
  int32_t m, n, k;    /* k: reduction length per tap                                            */
  /* row -> (utterance, frame) mapping */
  int32_t rows_per_batch; /* frames per utterance; 0: single utterance of m rows               */
  int32_t num_batches;    /* >=1                                                                */
  int32_t batched_tiles;  /* 1: tiles never straddle utterances (required for conv_taps > 1)    */
  /* implicit 1-D convolution over frames (conv_taps = 1: plain GEMM).  W is then
   * [N, conv_taps * k_pad] with k_pad = round_up(k, 64), tap-major.                            */
  int32_t conv_taps;
  int32_t conv_pad;
  int32_t conv_grouped;   /* 1: block-diagonal groups of 64 channels (k must be 64)             */
  /* epilogue */
  int32_t act;            /* F5_ACT_*                                                            */
  int32_t out_bf16;       /* 1: bf16 output, 0: fp32                                            */
  const float* bias;      /* [n] or NULL                                                        */
  void* out;              /* [rows, ldo]                                                        */
  int64_t ldo;
  const float* resid;     /* fp32 [rows, ldr] or NULL; may alias out                            */
  int64_t ldr;
  const float* gate;      /* fp32 [n], shared by all utterances, or NULL: out = v * gate + resid */
  const int32_t* row_len; /* [num_batches] valid frames (rows beyond are written as 0) or NULL  */
  const float* rope;      /* fp32 [rows_per_batch, 32, 2] (cos,sin) or NULL                     */
  int32_t rope_cols;      /* columns [0, rope_cols) are rotated in adjacent pairs               */
  float q_scale;          /* columns [0, q_cols) are multiplied by q_scale after the rotation   */
  int32_t q_cols;
  int32_t tile_n;         /* 0 = auto, else 64 | 128                                             */
  void* out2_bf16;        /* optional second copy of the result as bf16 [rows, ldo2], or NULL    */
  int64_t ldo2;
  int32_t w_static;       /* nonzero: `w` is never written by work that precedes this call on the stream
                             (model weights): the kernel may start fetching it before its programmatic
                             dependency on the preceding kernel has resolved                           */
  /* RMSNorm consumer mode (ABI 2.006; the field occupies what was padding after w_static, so sizeof and every other
   * offset are unchanged): nonzero makes the GEMM consume RMSNorm(x) = x * sqrt(k) / max(||x||_2, 1e-12) * g through
   * the linearity of the Linear, with g folded into `w` at pack time (w = W diag(g)):
   *     out = acc * sqrt(k) / max(sqrt(sum_col x^2), 1e-12) + bias,
   * the row's sum of squares taken from `ln_in_stats` ([rows][k / 64][2], as the fused-AdaLN producer writes them: a
   * producer with out2_bf16 and ln_stats but no ln_scale writes a plain bf16 copy of x).  Needs ln_in_stats, no ln_tab,
   * no second output, a plain bf16 GEMM with k % 128 == 0.  An all-zero row gives bias (0 * finite).  0 = off. */
  int32_t ln_rms;
  const void* prefetch;   /* NULL, or device memory (weights of a later GEMM) to pull into L2       */
  int64_t prefetch_bytes;
  /* Fused AdaLayerNormZero (dit.py:262-271, 281-290; call sites dit.py:313,321,397) by linearity of the Linear that
   * consumes the normalised activations:
   *     Linear(LN(x) * (1 + s) + b) = rstd * ((x * (1 + s)) W^T - mean * c1) + c2,   c1 = (1 + s) W^T,  c2 = b W^T.
   * Producer side (the GEMM whose fp32 `out` is the residual stream x): with `ln_scale` = s of the NEXT AdaLN,
   * out2_bf16 receives bf16(out * (1 + s[col])) and ln_stats[row][col / 64] the (sum, sum of squares) of each
   * 64-column unit of the finished row (requires out_bf16 == 0, n % 64 == 0).
   * Consumer side (`a` is such an out2 matrix): with `ln_in_stats` = that statistics array ([rows][k / 64][2]) the
   * epilogue computes rstd * (acc - mean * c1[col]) + c2[col] + bias[col] before the activation; ln_tab holds 4 rows
   * of ln_tab_ld floats — c1_hi, c1_lo, c2_hi, c2_lo (the table GEMM runs on a bf16 hi/lo split of (1 + s) and b,
   * f5_dit_precompute) — already offset to this GEMM's column 0.  A GEMM is producer or consumer, not both. */
  const float* ln_scale;
  float* ln_stats;
  const float* ln_in_stats;
  const float* ln_tab;
  int64_t ln_tab_ld;
  /* FP8 mode (the H100 analogue of the reference's quantised `--q` checkpoints, cfm.py:451-452,510-515): with ab_fp8
   * both `a` and `w` hold e4m3 bytes (lda / ldw in elements = bytes, multiples of 16; k a multiple of 128) and the
   * accumulator is multiplied by acc_scale (the weight tensor's quantisation scale, > 0) before bias / LN terms;
   * with out2_fp8 the second output out2_bf16 is written as e4m3 bytes (ldo2 in bytes) — the A operand of the next
   * FP8-mode GEMM.  Both 0 = bf16 everywhere. */
  int32_t ab_fp8;
  int32_t out2_fp8;
  float acc_scale;
  int32_t out_fp8;        /* with out_bf16 = 1: `out` is written as e4m3 bytes instead (ldo in bytes, multiple of 16) */
  /* Block-scaled FP8 (ABI 1.101; any of the four pointers non-NULL selects it).  Every scale is a power of two s, the
   * smallest with amax <= 448 s (not below 2^-126; 1 for amax = 0), so that x ~= s * e4m3 is exact to scale.
   * a_scale: fp32 [k/64][a_scale_ld] (a_scale_ld >= rows), the scale of `a` (ab_fp8) per (row, 64-column unit);
   * w_scale: fp32 [n], the per-output-channel scale of `w` (the accumulator term is multiplied by acc_scale * w_scale);
   * out_scale / out2_scale: fp32 [n/64][rows], written with the block-scaled e4m3 `out` (out_fp8) / `out2` (out2_fp8):
   * each (row, 64-column unit) is quantised with its own scale (n % 64 == 0).  Built for the epilogues of the DiT's
   * block-scaled mode only (RoPE QKV, residual fp32 + out2, GELU e4m3 out, Mish fp32 + out2). */
  const float* a_scale;
  int64_t a_scale_ld;
  const float* w_scale;
  float* out_scale;
  float* out2_scale;
  /* Second rotated column range (ABI 2.004): nonzero rotates [rope_col2, rope_col2 + rope_cols) as well as
   * [0, rope_cols) — the leading heads of q and of k when the QKV GEMM rotates only the first heads (F5TTS_Base v0:
   * rope_cols = 64 * rope_heads, rope_col2 = D).  A multiple of 64, >= rope_cols, with rope_col2 + rope_cols <= n and a
   * rope table set.  0 = [0, rope_cols) alone. */
  int32_t rope_col2;
  /* Dilated implicit convolution (ABI 2.005): with conv_taps > 1, tap t of output frame m reads input frame
   * m + t * conv_dilation - conv_pad (zero outside the utterance) — nn.Conv1d(dilation=conv_dilation,
   * padding=conv_pad).  0 or 1 = adjacent frames.  The field occupies what was the struct's tail padding: sizeof is
   * unchanged, so a zero-initialised 2.004 struct keeps its meaning. */
  int32_t conv_dilation;
} f5_gemm_args;

int f5_gemm_bf16(const f5_gemm_args* args, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * Flash-attention forward (non-causal, key-padding mask, head_dim 64) — replaces
 * mx.fast.scaled_dot_product_attention + head split/merge at dit.py:141-143,161-167.
 * qkv: bf16 [batch*frames, ld_qkv] = [q | k | v], each heads*64 wide, q pre-scaled by 1/sqrt(64)
 * and q,k already rotated (f5_gemm_bf16 epilogue).  out: bf16 [batch*frames, ld_out].
 * kv_len: int32 [batch] valid keys per utterance or NULL.
 * ------------------------------------------------------------------------------------------ */
int f5_attention_fwd(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch,
                     int32_t frames, int32_t heads, int32_t head_dim, const int32_t* kv_len,
                     void* stream);
/* the same with an e4m3 output (ld_out in bytes): the A operand of the FP8-mode out-projection */
int f5_attention_fwd_e4m3(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch,
                          int32_t frames, int32_t heads, int32_t head_dim, const int32_t* kv_len,
                          void* stream);
/* block-scaled e4m3 output: each (row, head) of O is quantised with its own power-of-two scale (see f5_gemm_args.a_scale),
 * written to scale_out fp32 [heads][batch*frames] — the a_scale of the block-scaled out-projection */
int f5_attention_fwd_e4m3_scaled(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch,
                                 int32_t frames, int32_t heads, int32_t head_dim, const int32_t* kv_len,
                                 float* scale_out, void* stream);
/* FP8 attention of the block-scaled FP8 mode (ABI 2.001): e4m3 Q·K^T and P·V with power-of-two scales, one per
 * (row, head) of Q and one per (utterance, head, 128-key tile) of K and of V.
 * f5_qkv_quant_e4m3    : qkv bf16 [batch*frames, ld_qkv] as above -> qk8 e4m3 [batch*frames, ld_qk8] = [q | k]
 *                        (ld_qk8 bytes, multiple of 16), vt8 e4m3 [batch][heads*64][vt_ld] = V transposed with keys
 *                        contiguous, in the order of weights.fp8_vt_key_order() within every 32 keys, zero for keys
 *                        in [frames, roundup(frames, 128)) (vt_ld bytes, multiple of 16, >= roundup(frames, 128)), and
 *                        qkv_scale fp32 [3*heads][batch*frames]: q head h -> unit h, k head h -> heads + h, v head h ->
 *                        2*heads + h (the scale rule of f5_gemm_args.a_scale, applied to the bf16 values; every k and v row holds
 *                        the scale of its 128-key tile).  Every key below frames is valid.
 * f5_qkv_quant_e4m3_masked (ABI 2.002): the same with kv_len int32 [batch] (NULL = frames), the valid keys as
 *                        f5_attention_fwd_fp8 takes them: keys at or beyond kv_len[b] do not enter their tile's k or v
 *                        amax and get zero K and V codes; a tile without a valid key has scale 1.  Pass the
 *                        attention's kv_len, so that masked keys cannot move the valid keys' scales.
 * f5_attention_fwd_fp8 : attention on those operands; out / scale_out as f5_attention_fwd_e4m3_scaled.
 * Pointers 16-byte aligned. */
int f5_qkv_quant_e4m3(const void* qkv, int64_t ld_qkv, void* qk8, int64_t ld_qk8, void* vt8, int64_t vt_ld,
                      float* qkv_scale, int32_t batch, int32_t frames, int32_t heads, void* stream);
int f5_qkv_quant_e4m3_masked(const void* qkv, int64_t ld_qkv, void* qk8, int64_t ld_qk8, void* vt8, int64_t vt_ld,
                             float* qkv_scale, int32_t batch, int32_t frames, int32_t heads, const int32_t* kv_len,
                             void* stream);
int f5_attention_fwd_fp8(const void* qk8, int64_t ld_qk8, const void* vt8, int64_t vt_ld, const float* qkv_scale,
                         void* out, int64_t ld_out, int32_t batch, int32_t frames, int32_t heads, int32_t head_dim,
                         const int32_t* kv_len, float* scale_out, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * HBM-bound pieces.
 * f5_ln_modulate : nn.LayerNorm(affine=False, eps=1e-6)(x) * (add_one + scale[b]) + shift[b]
 *                  (AdaLayerNormZero dit.py:270,289,321; with add_one=0 and mod_batch_stride=0 it
 *                  is the affine nn.LayerNorm of convnext_v2.py:38).  x fp32 -> y bf16.
 * f5_dwconv7_ln  : depthwise Conv1d(k=7,pad=3)+bias then affine LayerNorm (convnext_v2.py:35-38,
 *                  48-49).  x fp32 [batch, frames, C]; w_tap_major fp32 [7, C]; y bf16.
 * f5_grn         : GRN over the frame axis (convnext_v2.py:15-18). h,y bf16 [batch, frames, C];
 *                  nx_scratch fp32 [batch, 1 + ceil(frames/32), C] (deterministic two-stage
 *                  reduction: slot 0 receives Nx, the rest per-32-frame partial sums).
 * ------------------------------------------------------------------------------------------ */
int f5_ln_modulate(const float* x, void* y_bf16, int32_t rows, int32_t dim, int32_t rows_per_batch,
                   const float* scale, const float* shift, int64_t mod_batch_stride,
                   int32_t add_one, void* stream);
int f5_dwconv7_ln(const float* x, void* y_bf16, int32_t batch, int32_t frames, int32_t channels,
                  const float* w_tap_major, const float* bias, const float* ln_w, const float* ln_b,
                  void* stream);
int f5_grn(const void* h_bf16, void* y_bf16, float* nx_scratch, const float* gamma,
           const float* beta, int32_t batch, int32_t frames, int32_t channels, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * Kernel test entries: each runs one kernel that the model paths otherwise reach only inside
 * f5_dit_precompute / f5_ode_sample / f5_duration_forward / f5_vocos_decode, with the same arguments.
 * f5_ln_affine_f32    : affine LayerNorm with fp32 output (the Vocos backbone norm).
 * f5_ln_tab_prep      : the fused-AdaLN operand rows hi/lo(1 + scale), hi/lo(shift) of every LN site.
 *                       mod fp32 [times, mod_cols]; prep bf16 [2 depth + 1][4 times][dim].
 * f5_text_embed       : TextEmbedding's gather (ids + 1, CFG drop from row drop_from, embedding +
 *                       position table, masked rows 0).  x fp32 [batch_out, frames, channels];
 *                       valid_len int32 [batch_out] or NULL: rows beyond it are written as zeros.
 * f5_time_mlp         : TimestepEmbedding; t_emb fp32 [times, dim] (or NULL), silu_bf16 [times, dim].
 * f5_ode_update       : CFG combine + explicit-solver stage update (see f5_ode_sample).
 * f5_cast_pad_bf16    : fp32 [rows, d] -> bf16 [rows, ld], zero columns d..ld, optional row copy.
 * f5_concat_cond_text : [cond | text | 0] as bf16 [rows, ld]; cond_len int32 [batch_cond] or NULL.
 * f5_duration_head    : RMSNorm, masked mean over len[b] frames, Linear(dim -> 1), Softplus.
 * f5_grn_valid        : f5_grn with valid_len int32 [batch] (frames beyond it excluded from the norm).
 * ------------------------------------------------------------------------------------------ */
int f5_ln_affine_f32(const float* x, float* y, int32_t rows, int32_t dim, const float* w, const float* b,
                     void* stream);
int f5_ln_tab_prep(const float* mod, void* prep_bf16, int32_t times, int32_t depth, int32_t dim,
                   int32_t mod_cols, void* stream);
int f5_text_embed(const int32_t* text, int32_t batch, int32_t text_cols, int32_t frames, int32_t channels,
                  const float* emb, const float* pos_table, int32_t max_pos, float* x, int32_t batch_out,
                  int32_t drop_from, int32_t mask_padding, const int32_t* valid_len, void* stream);
int f5_time_mlp(const float* tvals, int32_t times, int32_t dim, const float* w0, const float* b0,
                const float* w2, const float* b2, float* t_emb, void* silu_bf16, void* stream);
int f5_ode_update(const float* v, int32_t ldv, int64_t null_row_offset, float cfg_strength,
                  const float* y_base, float* y_out, float a, float* k_acc, float acc_w, int32_t acc_init,
                  int32_t use_acc, void* y_bf16, int32_t ld_bf16, int64_t bf16_copy_row_offset, int32_t rows,
                  int32_t d, void* stream);
int f5_cast_pad_bf16(const float* src, int32_t d, void* dst, int32_t ld, int32_t rows, int64_t copy_row_offset,
                     void* stream);
int f5_concat_cond_text(const float* cond, int32_t dc, int32_t batch_cond, int32_t frames, const float* text,
                        int32_t dt, void* dst, int32_t ld, int32_t rows, int32_t drop_from_row,
                        const int32_t* cond_len, void* stream);
int f5_duration_head(const float* x, int32_t batch, int32_t frames, int32_t dim, const int32_t* len,
                     const float* norm_w, const float* pred_w, float* out, void* stream);
int f5_grn_valid(const void* h_bf16, void* y_bf16, float* nx_scratch, const float* gamma, const float* beta,
                 int32_t batch, int32_t frames, int32_t channels, const int32_t* valid_len, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * DiT (dit.py:331-401) and the ODE loop of F5TTS.sample (cfm.py:340-393).
 *
 * Weight layout ("packed"): what f5_tts_mlx_b200.weights.pack_dit() produces from the MLX
 * parameter tree: Linear weights bf16 (out,in); q/k/v fused row-wise into one
 * [3D, D] matrix; the per-block AdaLN linears (dit.py:263,282) concatenated row-wise into one
 * [depth*6D + 2D, D] matrix so the modulation vectors of ALL ODE time points are one GEMM; the
 * grouped k=31 convs (dit.py:33-38) as [D, 31*64] tap-major block-diagonal-by-64; the input
 * projection (dit.py:239) split by source: columns of x (padded to 128) and of [cond|text]
 * (padded to a multiple of 64).
 * ------------------------------------------------------------------------------------------ */
typedef struct f5_convnext_weights {
  const float* dw_w;   /* fp32 [7, C] tap-major (MLX (C,7,1) transposed) */
  const float* dw_b;   /* [C] */
  const float* ln_w;   /* [C] */
  const float* ln_b;
  const void* pw1_w;   /* bf16 [Ci, C] */
  const float* pw1_b;
  const float* grn_gamma; /* [Ci] */
  const float* grn_beta;
  const void* pw2_w;   /* bf16 [C, Ci] */
  const float* pw2_b;
} f5_convnext_weights;

typedef struct f5_dit_block_weights {
  const void* qkv_w;  const float* qkv_b;   /* bf16 [3D, D], fp32 [3D]   (dit.py:119-121) */
  const void* out_w;  const float* out_b;   /* [D, D]                     (dit.py:124)     */
  const void* ff1_w;  const float* ff1_b;   /* [F, D]                     (dit.py:94-95)   */
  const void* ff2_w;  const float* ff2_b;   /* [D, F]                     (dit.py:96)      */
  /* FP8 mode (optional, NULL = bf16 only): e4m3 copies of the four block weights, ONE scale per tensor
   * (w ~= scale * e4m3); used by f5_dit_forward when f5_dit_buffers.a_fp8 is set (see f5_gemm_args.ab_fp8), which then
   * needs all four in every block.  All four block GEMMs run in FP8: the attention and FF1 write e4m3 for the
   * out-projection and FF2. */
  const void* qkv_w8; const void* ff1_w8; const void* out_w8; const void* ff2_w8;
  float qkv_s8, ff1_s8, out_s8, ff2_s8;
  /* Block-scaled FP8 mode (ABI 1.101, optional): fp32 per-output-channel scales of the *_w8 weights (w[o] ~= s[o] *
   * e4m3, *_s8 = 1).  With these and f5_dit_buffers.a_fp8 / a_fp8_scale / attn_scale / ff_scale all set, the four block
   * GEMMs run on block-scaled e4m3 operands (see f5_gemm_args.a_scale).  In FP8 mode they need the block-scale buffers:
   * all four in every block, or none. */
  const float* qkv_ws; const float* ff1_ws; const float* out_ws; const float* ff2_ws;
} f5_dit_block_weights;

typedef struct f5_dit_weights {
  int32_t dim, depth, heads, ff_inner, mel_dim, text_dim, text_inner, conv_layers;
  int32_t text_rows;     /* rows of the embedding table (text_num_embeds + 1) */
  int32_t text_max_pos;  /* 4096 (dit.py:190) */
  int32_t ct_ld;         /* padded width of [cond|text] (multiple of 64) */
  int32_t reserved;
  const float* time_w0; const float* time_b0;   /* fp32 [D,256],[D]   (dit.py:77) */
  const float* time_w2; const float* time_b2;   /* fp32 [D,D],[D] */
  const float* text_emb;                        /* fp32 [text_rows, text_dim] */
  const float* text_pos;                        /* fp32 [text_max_pos, text_dim] (rope.py:63-73) */
  const f5_convnext_weights* text_blocks;       /* HOST array [conv_layers] */
  const void* in_x_w;                           /* bf16 [D, 128] */
  const void* in_ct_w;                          /* bf16 [D, ct_ld] */
  const float* in_b;                            /* fp32 [D] */
  const void* conv_w[2]; const float* conv_b[2];/* bf16 [D, 31*64], fp32 [D] */
  const void* mod_w; const float* mod_b;        /* bf16 [depth*6D+2D, D], fp32 */
  const f5_dit_block_weights* blocks;           /* HOST array [depth] */
  const void* proj_w; const float* proj_b;      /* bf16 [mel_dim, D], fp32 [mel_dim] */
  /* Model version (ABI 2.004; zero = the v1 DiT that from_pretrained builds, cfm.py:459-469):
   * text_unmasked 1: TextEmbedding(mask_padding=False) (dit.py:182-229) — filler tokens (id 0) and the rows past the
   *   text keep the filler embedding + position table and the ConvNeXt blocks run on them without re-zeroing;
   * rope_heads 1..heads: rotary embedding on the first rope_heads heads of q and of k only (upstream's pe_attn_head;
   *   F5TTS_Base v0 rotates the first 64 columns of the un-split q and k projections = head 0); 0 = every head. */
  int32_t text_unmasked;
  int32_t rope_heads;
} f5_dit_weights;

/* Caller-allocated device buffers for one sampling session of `batch` utterances padded to
 * `frames`.  rows = (cfg ? 2 : 1) * batch * frames: with classifier-free guidance the
 * conditional and unconditional passes of cfm.py:342-363 run as ONE forward over a doubled batch
 * (cond rows first). */
typedef struct f5_dit_buffers {
  int32_t batch, frames, cfg, n_times;
  int32_t text_len_max;       /* nt: columns of `text` */
  int32_t drop_flags;         /* only when cfg == 0: bit0 drop_audio_cond, bit1 drop_text (dit.py:380-381) */
  /* inputs */
  const int32_t* text;        /* int32 [batch, nt], pad -1 */
  const int32_t* text_len;    /* int32 [rows/frames]: valid tokens (<= frames) per row-utterance */
  const int32_t* seq_len;     /* int32 [rows/frames] valid frames, or NULL when mask is None */
  const float* cond;          /* fp32 [batch, frames, mel_dim] step_cond (cfm.py:331) */
  const float* tvals;         /* fp32 [n_times] DiT evaluation times, in evaluation order */
  const float* rope;          /* fp32 [frames, 32, 2] cos/sin of n*theta_i (rope.py:38-53) */
  /* precomputed by f5_dit_precompute */
  float* hoist;               /* fp32 [rows, D]: cond·Wc + text·Wt + b (dit.py:249, step-invariant) */
  float* mod_table;           /* fp32 [n_times, depth*6D+2D] */
  /* scratch */
  float* text_x;              /* fp32 [rows, text_dim] */
  void* text_a;               /* bf16 [rows, text_dim] */
  void* text_h;               /* bf16 [rows, text_inner] */
  void* text_g;               /* bf16 [rows, text_inner] */
  float* grn_nx;              /* fp32 [rows/frames, 1 + ceil(frames/32), text_inner] (f5_grn scratch) */
  void* ct_bf16;              /* bf16 [rows, ct_ld] */
  void* silu_t;               /* bf16 [n_times, D] */
  void* y_bf16;               /* bf16 [rows, 128]: current ODE state, A operand of the x-projection */
  float* x;                   /* fp32 [rows, D] residual stream */
  float* h;                   /* fp32 [rows, D] */
  void* a_bf16;               /* bf16 [rows, D] */
  void* c_bf16;               /* bf16 [rows, D] */
  void* qkv_bf16;             /* bf16 [rows, 3D] */
  void* ff_bf16;              /* bf16 [rows, ff_inner] */
  float* v;                   /* fp32 [rows, mel_dim]: DiT output (flow prediction) */
  /* Fused AdaLN (see f5_gemm_args.ln_*): all three set selects it, all three NULL keeps the separate
   * f5_ln_modulate launches; anything else is F5_ERR_INVALID.  ln_tab_ld = depth*(3D + ff_inner) + 128
   * (f5_dit_ln_tab_ld). */
  float* ln_stats;            /* fp32 [rows, D/64, 2]: per-row (sum, sum of squares) per 64 columns of the residual stream */
  float* ln_tab;              /* fp32 [4*n_times, ln_tab_ld]: c1/c2 operand rows per time, columns = per block [qkv 3D | ff1 F], then proj_out */
  void* ln_prep;              /* bf16 [2*depth+1, 4*n_times, D]: operand rows of the table GEMMs */
  /* Frame bucketing (plan reuse across utterances of different length): the buffers are sized for `frames` rows per
   * utterance but only the first valid_len[u] (= the reference's N, cfm.py:319) exist; rows beyond are kept exactly
   * zero where the reference's zero padding would be seen (the k=31 ConvPositionEmbedding input, dit.py:45) and are
   * masked as attention keys, so rows < N equal the unpadded computation.  NULL = all `frames` rows are real. */
  const int32_t* valid_len;   /* int32 [rows/frames], every entry the same N <= frames, or NULL */
  /* FP8 mode: e4m3 [rows, D] — the AdaLN-modulated operand of the QKV / FF1 GEMMs (written by the producing GEMM's
   * epilogue instead of a_bf16); requires the fused AdaLN buffers and all four blocks[i].*_w8.  NULL = bf16. */
  void* a_fp8;
  /* Block-scaled FP8 mode (ABI 1.101): per (row, 64-column unit) scales, unit-major — fp32 [D/64][rows] of a_fp8, fp32
   * [heads][rows] of the attention output (e4m3 in c_bf16), fp32 [ff_inner/64][rows] of the FF1 output (e4m3 in
   * ff_bf16).  All three set selects the mode and requires a_fp8 and all four blocks[i].*_ws; all three NULL =
   * per-tensor FP8 (or bf16). */
  float* a_fp8_scale;
  float* attn_scale;
  float* ff_scale;
  /* FP8 attention (ABI 2.001, see f5_attention_fwd_fp8): e4m3 [rows, 2D] Q | K, e4m3 [rows/frames][D][roundup(frames,
   * 128)] V^T and fp32 [3*heads][rows] scales.  All three set selects it inside the block-scaled FP8 mode (which it
   * requires); all three NULL keeps the bf16 attention with a block-scaled e4m3 output. */
  void* qk_fp8;
  void* vt_fp8;
  float* qkv_scale;
} f5_dit_buffers;

/* step-invariant work, once per sample(): text embedding (dit.py:196-229), hoisted conditioning
 * projection, TimestepEmbedding + every AdaLN linear for all n_times (dit.py:73-82,267,286). */
int f5_dit_precompute(const f5_dit_weights* w, const f5_dit_buffers* b, void* stream);
/* row length (floats) of f5_dit_buffers.ln_tab for this model */
int64_t f5_dit_ln_tab_ld(const f5_dit_weights* w);
/* one DiT evaluation (dit.py:374-401) at tvals[time_index] on the state in b->y_bf16 -> b->v */
int f5_dit_forward(const f5_dit_weights* w, const f5_dit_buffers* b, int32_t time_index, void* stream);

/* Fixed-grid explicit ODE solve (cfm.py:38-122, 340-393).  t_grid: HOST fp32 [steps] (the sway-
 * warped grid, `steps` grid points = steps-1 intervals).  method: 0 euler, 1 midpoint, 2 rk4.
 * b->tvals / n_times must hold the evaluation times in the order the solver visits them (see
 * f5_ode_eval_times).  y: fp32 [batch*frames, mel_dim] initial noise, overwritten by the final
 * state unless `trajectory` (fp32 [steps, batch*frames, mel_dim]) is given, in which case
 * trajectory[0] must hold y0 and every state is stored (cfm.py:61).  scratch: fp32
 * [2, batch*frames, mel_dim]. */
int f5_ode_eval_times(const float* h_t_grid, int32_t steps, int32_t method, float* h_out, int32_t cap);
int f5_ode_sample(const f5_dit_weights* w, const f5_dit_buffers* b, const float* h_t_grid,
                  int32_t steps, int32_t method, float cfg_strength, float* y, float* trajectory,
                  float* scratch, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * UNetT (ABI 2.006): the flat UNet-Transformer backbone of upstream F5-TTS's E2TTS_Base (f5_tts/model/backbones/unett.py,
 * skip_connect_type "concat", qk_norm None, conv_layers 0, text_mask_padding False).  Per utterance of N frames:
 *   t = TimestepEmbedding(time); x = InputEmbedding(x, cond, TextEmbedding(text)) (the DiT's, with a plain embedding
 *   gather: no position table, no ConvNeXt); x = [t | x], N + 1 rows, the time token at row 0 (RoPE positions 0..N);
 *   for layer i < depth/2: push x; for i >= depth/2: x = skip_proj_i([x | pop()]) (no residual);
 *   x += attn(RMSNorm(x)); x += ff(RMSNorm(x)); v = proj_out(RMSNorm_out(x)[1:]).
 * RMSNorm is x * sqrt(D) / max(||x||, 1e-12) * g; each g is folded into the consuming weight (f5_gemm_args.ln_rms).
 * Skip slots: bf16 [depth/2][rows, 2D]; slot j's right half is x at the start of layer j (written by the GEMM that
 * produced it, and read by that layer's QKV with lda = 2D), its left half x at the start of layer depth - 1 - j (written
 * by the FF2 before it), so skip_proj is one GEMM with k = 2D over the slot.  bf16 + fp32 only (no FP8 modes).
 * ------------------------------------------------------------------------------------------ */
typedef struct f5_unett_weights {
  int32_t dim, depth, heads, ff_inner, mel_dim, text_dim;
  int32_t text_rows;      /* rows of the embedding table (text_num_embeds + 1) */
  int32_t ct_ld;          /* padded width of [cond|text] (multiple of 64) */
  int32_t rope_heads;     /* rotary embedding on the first rope_heads heads of q and k (E2TTS_Base: 1); 0 = all */
  int32_t reserved;
  const float* time_w0; const float* time_b0;   /* fp32 [D,256],[D] */
  const float* time_w2; const float* time_b2;   /* fp32 [D,D],[D] */
  const float* text_emb;                        /* fp32 [text_rows, text_dim] */
  const void* in_x_w;                           /* bf16 [D, 128] */
  const void* in_ct_w;                          /* bf16 [D, ct_ld] */
  const float* in_b;                            /* fp32 [D] */
  const void* conv_w[2]; const float* conv_b[2];/* bf16 [D, 31*64], fp32 [D] */
  /* HOST array [depth]: qkv_w = bf16([Wq; Wk; Wv] diag(attn_norm.g)), ff1_w = bf16(W1 diag(ff_norm.g)), out_w / ff2_w
   * as in the DiT; every FP8 field NULL */
  const f5_dit_block_weights* blocks;
  const void* skip_w;                           /* bf16 [depth/2][D, 2D]: skip_proj of layer depth/2 + i at i */
  const void* proj_w; const float* proj_b;      /* bf16(W diag(norm_out.g)) [mel_dim, D], fp32 [mel_dim] */
} f5_unett_weights;

/* Device buffers of one sampling session; R = (cfg ? 2 : 1) * batch * frames rows of frames, R1 = R + (cfg ? 2 : 1) *
 * batch rows with the time token.  The skip slots cost depth/2 * R1 * 2D * 2 bytes. */
typedef struct f5_unett_buffers {
  int32_t batch, frames, cfg, n_times;
  int32_t text_len_max;       /* nt: columns of `text` */
  int32_t drop_flags;         /* only when cfg == 0: bit0 drop_audio_cond, bit1 drop_text */
  /* inputs */
  const int32_t* text;        /* int32 [batch, nt], pad -1 */
  const int32_t* seq_len1;    /* int32 [R / frames]: valid frames + 1 (the time row), or NULL when mask is None */
  const int32_t* valid_len;   /* int32 [R / frames]: frame bucketing as f5_dit_buffers.valid_len, or NULL */
  const int32_t* valid_len1;  /* int32 [R / frames]: valid_len + 1; set exactly when valid_len is */
  const float* cond;          /* fp32 [batch, frames, mel_dim] */
  const float* tvals;         /* fp32 [n_times] */
  const float* rope;          /* fp32 [frames + 1, 32, 2] */
  /* precomputed by f5_unett_precompute */
  float* hoist;               /* fp32 [R, D] */
  float* t_emb;               /* fp32 [n_times, D] */
  /* scratch */
  float* text_x;              /* fp32 [R, text_dim] */
  void* ct_bf16;              /* bf16 [R, ct_ld] */
  void* silu_t;               /* bf16 [n_times, D] */
  void* y_bf16;               /* bf16 [R, 128]: current ODE state */
  float* h;                   /* fp32 [R, D]: input embedding */
  float* x;                   /* fp32 [R1, D] residual stream */
  void* a_bf16;               /* bf16 [R1, D] */
  void* c_bf16;               /* bf16 [R1, D] */
  void* qkv_bf16;             /* bf16 [R1, 3D] */
  void* ff_bf16;              /* bf16 [R1, ff_inner] */
  float* ln_stats;            /* fp32 [R1, D/64, 2] */
  void* skip;                 /* bf16 [depth/2, R1, 2D] */
  float* v;                   /* fp32 [R1, mel_dim]: output rows, the time rows included */
} f5_unett_buffers;

/* text embedding, hoisted [cond | text] projection, TimestepEmbedding of every evaluation time */
int f5_unett_precompute(const f5_unett_weights* w, const f5_unett_buffers* b, void* stream);
/* one UNetT evaluation at tvals[time_index] on the state in b->y_bf16 -> b->v */
int f5_unett_forward(const f5_unett_weights* w, const f5_unett_buffers* b, int32_t time_index, void* stream);
/* f5_ode_sample on this backbone: the solver update reads v past each utterance's time row */
int f5_unett_ode_sample(const f5_unett_weights* w, const f5_unett_buffers* b, const float* h_t_grid, int32_t steps,
                        int32_t method, float cfg_strength, float* y, float* trajectory, float* scratch, void* stream);
/* Kernel test entry: the time-token pack.  xe fp32 [batch, frames, D] (the input embedding), t_emb fp32 [D] ->
 * x fp32 [batch, frames + 1, D] with t_emb at row 0 of each utterance, x_bf16 = bf16(x) [batch * (frames + 1), ld_bf16],
 * ln_stats fp32 [batch * (frames + 1), D / 64, 2] (sum, sum of squares per 64 columns). */
int f5_unett_time_pack(const float* xe, const float* t_emb, float* x, void* x_bf16, int64_t ld_bf16, float* ln_stats,
                       int32_t batch, int32_t frames, int32_t dim, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * DurationPredictor (duration.py:97-253, inference branch; call site cfm.py:253-262,307-308): runs
 * once per sample() when duration=None.  mel fp32 [batch, frames, mel_dim] (frames >= text columns;
 * rows beyond lens[b] are treated as zero, duration.py:241-243) + text ids -> seconds fp32 [batch].
 * Reuses f5_convnext_weights / f5_dit_block_weights.  zeros: fp32 [dim] of zeros (the shift/scale
 * of the non-affine LayerNorms).  in_w: bf16 [dim, ct_ld] = proj.weight over [mel | text], padded.
 * ------------------------------------------------------------------------------------------ */
typedef struct f5_duration_weights {
  int32_t dim, depth, heads, ff_inner, mel_dim, text_dim, text_inner, conv_layers;
  int32_t text_rows, text_max_pos, ct_ld, reserved;
  const float* text_emb; const float* text_pos;
  const f5_convnext_weights* text_blocks;       /* HOST array [conv_layers] */
  const void* in_w; const float* in_b;
  const void* conv_w[2]; const float* conv_b[2];
  const f5_dit_block_weights* blocks;           /* HOST array [depth] */
  const float* zeros;
  const float* norm_w;                          /* RMSNorm weight [dim] */
  const float* pred_w;                          /* to_pred Linear(dim -> 1) weight [dim] */
} f5_duration_weights;

typedef struct f5_duration_buffers {
  int32_t batch, frames, text_len_max, reserved;
  const int32_t* text;        /* int32 [batch, text_len_max], pad -1 */
  const int32_t* lens;        /* int32 [batch] valid frames */
  const float* inp;           /* fp32 [batch, frames, mel_dim] */
  const float* rope;          /* fp32 [frames, 32, 2] */
  float* text_x; void* text_a; void* text_h; void* text_g; float* grn_nx; void* ct_bf16;
  float* x; float* h; void* a_bf16; void* c_bf16; void* qkv_bf16; void* ff_bf16;
  float* out;                 /* fp32 [batch] seconds */
} f5_duration_buffers;

int f5_duration_forward(const f5_duration_weights* w, const f5_duration_buffers* b, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * Log-mel front-end — replaces log_mel_spectrogram / MelSpec (audio.py:162-230): zero-padded
 * centred frames (n_fft 1024), periodic Hann, real FFT, magnitude, HTK filterbank, log(max(.,1e-5)),
 * LAST FRAME DROPPED (audio.py:203) => frames = samples / hop.
 * audio fp32 [batch, samples]; window fp32 [1024]; filters_t fp32 [513, n_mels] (filterbank
 * transposed); out fp32 [batch, frames, n_mels].
 * ------------------------------------------------------------------------------------------ */
int f5_mel_forward(const float* audio, int32_t batch, int32_t samples, const float* window,
                   const float* filters_t, int32_t n_mels, int32_t hop, float* out, int32_t frames,
                   void* stream);

/* BigVGAN's mel (ABI 2.005; upstream F5-TTS get_bigvgan_mel_spectrogram, the front-end of F5TTS_Base_bigvgan):
 * frames of the REFLECT-padded signal (pad (1024 - hop) / 2 = 384 on each side), non-centred, periodic Hann, real FFT,
 * magnitude sqrt(re^2 + im^2 + 1e-9), filters_t (Slaney filterbank, transposed), log(max(., 1e-5)).
 * frames must equal (samples + 2 pad - 1024) / hop + 1, and samples > pad (reflect padding needs them). */
int f5_mel_forward_bigvgan(const float* audio, int32_t batch, int32_t samples, const float* window,
                           const float* filters_t, int32_t n_mels, int32_t hop, float* out, int32_t frames,
                           void* stream);

/* ------------------------------------------------------------------------------------------ *
 * Sample-rate conversion (ABI 2.003) — torchaudio.functional.resample at its defaults (sinc_interp_hann,
 * lowpass_filter_width 6, rolloff 0.99), the resampler upstream F5-TTS puts in front of the mel front-end for
 * reference clips that are not 24 kHz.  With g = gcd(orig, new), O = orig / g, N = new / g:
 *
 *     base = min(O, N) * 0.99;   w = ceil(6 * O / base);   taps = 2 * w + O
 *     for phase p in [0, N), tap k in [0, taps):
 *         t = clamp(((k - w) / O - p / N) * base, -6, 6)
 *         h[p][k] = (t == 0 ? 1 : sin(pi t) / (pi t)) * cos(pi t / 12)^2 * base / O
 *     out_samples = ceil(N * samples / O)
 *     y[j] = sum_{k ascending} h[j % N][k] * x[(j / N) * O + k - w]        (x = 0 outside [0, samples))
 *
 * f5_resample_table : HOST function: returns N * taps, and writes h row-major [N][taps] to h_table when h_table is
 *                     non-NULL and cap >= N * taps (computed in double, rounded once to fp32).  orig == new is the
 *                     identity and returns 0.  F5_ERR_INVALID for a non-positive rate or a table of more than 65536
 *                     entries (every pair of 8, 11.025, 16, 22.05, 32, 44.1, 48, 88.2, 96 kHz with 24 kHz fits).
 * f5_resample       : x fp32 [batch, samples] -> out fp32 [batch, out_samples] with the table above (device memory);
 *                     out_samples must equal ceil(N * samples / O).  Each output is one fp32 fused multiply-add chain
 *                     in ascending k: bitwise reproducible, rows independent.  orig == new copies x to out (table
 *                     may be NULL).  F5_ERR_INVALID also when one tile's input window exceeds shared memory
 *                     (decimation by more than about 200:1).  x and out 4-byte aligned.
 * ------------------------------------------------------------------------------------------ */
int f5_resample_table(int32_t orig_freq, int32_t new_freq, float* h_table, int64_t cap);
int f5_resample(const float* x, int32_t batch, int64_t samples, int32_t orig_freq, int32_t new_freq,
                const float* table, float* out, int64_t out_samples, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * Vocos vocoder — replaces vocos_mlx.Vocos.decode (third-party; call sites cfm.py:399-400,446,
 * 471): Conv1d(100->512,k7) LN 8x[dwconv7 LN Linear GELU Linear gamma* +res] LN Linear(512->1026)
 * -> (log-mag, phase) -> ISTFT(n_fft 1024, hop 256).
 * f5_istft: h fp32 [batch*frames, ldh] = [log-mag 513 | phase 513 | pad]; per-frame inverse real
 * FFT, windowed overlap-add, divided by the window envelope (norm_sq 0: sum w — vocos-mlx;
 * 1: sum w^2 — torch.istft), `trim` leading samples dropped.  out fp32 [batch, out_len].
 * ------------------------------------------------------------------------------------------ */
typedef struct f5_vocos_block_weights {
  const float* dw_w; const float* dw_b;      /* fp32 [7, D] tap-major, [D] */
  const float* ln_w; const float* ln_b;
  const void* pw1_w; const float* pw1_b;     /* bf16 [Ci, D] */
  const void* pw2_w; const float* pw2_b;     /* bf16 [D, Ci] */
  const float* gamma;                        /* fp32 [D] layer scale */
} f5_vocos_block_weights;

typedef struct f5_vocos_weights {
  int32_t n_mels, dim, inner, num_layers;
  int32_t head_ld;        /* padded width of the head output (1028) */
  int32_t hop, istft_norm_sq, istft_trim;
  const void* embed_w; const float* embed_b;     /* bf16 [D, 7*128] tap-major, fp32 [D] */
  const float* norm_w; const float* norm_b;
  const f5_vocos_block_weights* blocks;          /* HOST array [num_layers] */
  const float* final_w; const float* final_b;
  const void* head_w; const float* head_b;       /* bf16 [head_ld, D], fp32 [head_ld] */
  const float* window;                           /* fp32 [1024] periodic Hann */
} f5_vocos_weights;

typedef struct f5_vocos_buffers {
  int32_t batch, frames, out_len, reserved;
  void* mel_bf16;      /* bf16 [R, 128]   R = batch*frames */
  float* h;            /* fp32 [R, D] */
  float* x;            /* fp32 [R, D] */
  void* a_bf16;        /* bf16 [R, D] */
  void* i_bf16;        /* bf16 [R, inner] */
  float* head;         /* fp32 [R, head_ld] */
  float* frames_f32;   /* fp32 [R, 1024] */
} f5_vocos_buffers;

int f5_istft(const float* h, int64_t ldh, int32_t batch, int32_t frames, const float* window,
             int32_t hop, int32_t norm_sq, int32_t trim, float* frames_scratch, float* out,
             int32_t out_len, void* stream);
int f5_vocos_decode(const f5_vocos_weights* w, const f5_vocos_buffers* b, const float* mel,
                    float* wave, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * BigVGAN v2 vocoder (ABI 2.005; NVIDIA's bigvgan_v2_24khz_100band_256x, upstream F5-TTS --vocoder_name bigvgan), resblock
 * "1" (AMPBlock1) with Snake / SnakeBeta.  Channels-last throughout: an utterance of T frames and C channels is
 * [T, C] row-major, utterances one after another.
 *
 *   conv_pre   Conv1d(num_mels, C0, 7, pad 3): implicit GEMM over the bf16 mel padded to 128 columns, bf16 out
 *   ups[i]     ConvTranspose1d(C_i, C_i / 2, k_i, stride u_i, pad (k_i - u_i) / 2) as a POLYPHASE implicit conv: output
 *              frame n u + q only reads input frames n - up_pad .. n - up_pad + up_taps - 1, so with the weights packed
 *              as up_w[(q, c_out)][tap][c_in] the GEMM's [T, u C_out] fp32 output is exactly [u T, C_out]
 *   resblocks  x_j = AMPBlock1_j(x) for j < num_kernels, then x = (x_0 + ... + x_{nk-1}) / nk (fp32 sum in j order,
 *              one IEEE division; bf16 when it feeds the next ups GEMM, fp32 before activation_post)
 *              AMPBlock1: for m < 3: t = act(x) [bf16]; t = conv1_m(t) [fp32, dilation d_m]; t = act(t) [bf16];
 *                         x = conv2_m(t) + x [fp32, the GEMM epilogue's residual]
 *   act_post   anti-aliased activation, fp32 out
 *   conv_post  Conv1d(C_last, 1, 7, pad 3, bias optional) on the CUDA cores, then tanh (use_tanh_at_final) or
 *              clamp(-1, 1)
 *
 * Anti-aliased activation (Activation1d): per channel, with replicate padding at each utterance's two edges,
 *     u[m] = 2 sum_j h_up[j] xp[(m + 15 - j) / 2]    (j with m + 15 - j even; xp = x padded by 5 frames each side)
 *     a[m] = u[m] + sin(alpha u[m])^2 / (beta + 1e-9)                   (Snake: beta = alpha)
 *     z[n] = sum_j h_down[j] ap[2 n + j]                (ap = a padded by 5 / 6 samples: replicates the ACTIVATED signal)
 * in one pass: the 2T-long intermediate stays in shared memory.  sin is the accurate sinf.
 * ------------------------------------------------------------------------------------------ */
#define F5_BIGVGAN_MAX_UPS 8
#define F5_BIGVGAN_MAX_KERNELS 4

typedef struct f5_bigvgan_act {
  const float* alpha;    /* fp32 [C], already exp() of the stored value when snake_logscale */
  const float* beta;     /* fp32 [C] (SnakeBeta), or NULL (Snake: the divisor is alpha) */
  const float* h_up;     /* fp32 [12] upsample.filter */
  const float* h_down;   /* fp32 [12] downsample.lowpass.filter */
} f5_bigvgan_act;

typedef struct f5_bigvgan_amp_weights {
  int32_t kernel;                 /* k of every conv of the block */
  int32_t dilation[3];
  const void* conv1_w[3];         /* bf16 [C, k * round_up(C, 64)] tap-major: w[o][t * kp + i] = conv.weight[o, i, t] */
  const float* conv1_b[3];        /* fp32 [C] */
  const void* conv2_w[3];
  const float* conv2_b[3];
  f5_bigvgan_act act[6];          /* activations[0..5]: act[2m] before conv1_m, act[2m + 1] before conv2_m */
} f5_bigvgan_amp_weights;

typedef struct f5_bigvgan_weights {
  int32_t num_mels;               /* <= 128 */
  int32_t num_upsamples;          /* <= F5_BIGVGAN_MAX_UPS */
  int32_t num_kernels;            /* resblocks per stage, <= F5_BIGVGAN_MAX_KERNELS */
  int32_t channels0;              /* upsample_initial_channel C0; stage i has C0 >> (i + 1) channels */
  int32_t use_tanh_at_final;
  int32_t reserved[3];
  int32_t up_rate[F5_BIGVGAN_MAX_UPS];
  int32_t up_taps[F5_BIGVGAN_MAX_UPS];   /* taps of the polyphase packing */
  int32_t up_pad[F5_BIGVGAN_MAX_UPS];
  const void* conv_pre_w;         /* bf16 [C0, 7 * 128] tap-major, mel channels padded to 128 */
  const float* conv_pre_b;        /* fp32 [C0] */
  const void* up_w[F5_BIGVGAN_MAX_UPS];   /* bf16 [u C_out, up_taps * round_up(C_in, 64)] */
  const float* up_b[F5_BIGVGAN_MAX_UPS];  /* fp32 [u C_out]: bias[c_out] repeated per phase */
  const f5_bigvgan_amp_weights* blocks;   /* HOST array [num_upsamples * num_kernels], resblocks.{n} order */
  f5_bigvgan_act act_post;
  const float* conv_post_w;       /* fp32 [7, C_last] tap-major */
  const float* conv_post_b;       /* fp32 [1], or NULL (use_bias_at_final = false) */
} f5_bigvgan_weights;

/* stage_elems = max(frames * C0, max_i T_i C_i) with T_i = frames * u_0 ... u_i: the per-utterance size of the scratch */
typedef struct f5_bigvgan_buffers {
  int32_t batch, frames, reserved[2];
  int64_t stage_elems;
  void* mel_bf16;       /* bf16 [batch * frames, 128] */
  void* a_bf16;         /* bf16 [batch * stage_elems]: GEMM operands */
  float* x_up;          /* fp32 [batch * stage_elems]: output of the stage's ups GEMM */
  float* t;             /* fp32 [batch * stage_elems]: conv1 outputs, the activation_post output */
  float* xk;            /* fp32 [num_kernels][batch * stage_elems]: the resblocks' residual streams */
} f5_bigvgan_buffers;

/* mel fp32 [batch, frames, num_mels] -> wave fp32 [batch, frames * prod(up_rate)] */
int f5_bigvgan_decode(const f5_bigvgan_weights* w, const f5_bigvgan_buffers* b, const float* mel, float* wave,
                      void* stream);
/* Kernel test entry: the anti-aliased activation on x fp32 [batch, rows_per_batch, channels]; utterance u has lens[u]
 * frames (int32 device [batch], or NULL = rows_per_batch), rows at or beyond it are not written.  act is a HOST pointer
 * to device tables.  out: bf16 (out_bf16 = 1) or fp32, the same layout. */
int f5_bigvgan_act_forward(const float* x, int32_t batch, int32_t rows_per_batch, int32_t channels,
                           const int32_t* lens, const f5_bigvgan_act* act, int32_t out_bf16, void* out, void* stream);
/* Kernel test entry (ABI 2.007): the resblock mean out[i] = (xk[i] + xk[stride + i] + ... ) / nk over nk fp32 streams
 * stride elements apart, i < n, summed in stream order in fp32 with one IEEE division; out bf16 (out_bf16 = 1) or fp32
 * [n]. */
int f5_bigvgan_resblock_mean(const float* xk, int64_t stride, int32_t nk, int64_t n, int32_t out_bf16, void* out,
                             void* stream);
/* Kernel test entry (ABI 2.007): conv_post, Conv1d(channels, 1, 7, padding=3) over x fp32 [batch, frames, channels]
 * with zero padding inside each utterance, w fp32 [7, channels] tap-major, bias fp32 [1] or NULL, then tanh (use_tanh)
 * or a clamp to [-1, 1]; out fp32 [batch, frames]. */
int f5_bigvgan_conv_post(const float* x, int32_t batch, int32_t frames, int32_t channels, const float* w,
                         const float* bias, int32_t use_tanh, float* out, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * Host utilities for hosts that are not Python (the package's weights.PackedDiT / dit.DitSession / parallel.py do
 * the same from Python): sizing + packing + binding of the weight buffer, sizing + carving of the session workspace,
 * and the ONE collective of the multi-GPU path.
 *
 * f5_pack_weights    : what F5TTS.from_pretrained + load_weights amount to for the DiT (cfm.py:455-517 after the key
 *                      conversion): `get(user, mlx_name, &numel)` returns the fp32 HOST tensor of an MLX-named parameter
 *                      ("transformer.transformer_blocks.3.attn.to_q.weight", MLX layouts) or NULL; host_out receives
 *                      f5_packed_weights_bytes() bytes in the layout every kernel expects (copy it to the device,
 *                      then f5_bind_packed_weights on the device copy).
 * f5_bind_workspace  : carves f5_dit_buffers out of one 256-byte-aligned device block of f5_workspace_bytes(), zeroes
 *                      it and uploads the RoPE table; the caller then fills text / text_len / seq_len / cond / tvals.
 * f5_nccl_broadcast_weights : ncclBroadcast of the packed buffer from `root` ("a single NCCL broadcast of
 *                      weights at load, no per-step collective"); `nccl_comm` is an initialised ncclComm_t; the NCCL
 *                      symbol is taken from the library already loaded in the process (or libnccl.so.2).
 * ------------------------------------------------------------------------------------------ */
typedef struct f5_dit_dims {
  int32_t dim, depth, heads, ff_inner, mel_dim, text_dim, conv_layers, text_num_embeds;
  /* ABI 2.004: copied into f5_dit_weights by f5_bind_packed_weights (see there); 0, 0 = v1, 1, 1 = F5TTS_Base (v0).
   * The packed layout does not depend on them. */
  int32_t text_unmasked, rope_heads;
} f5_dit_dims;
typedef struct f5_dit_shape {
  int32_t batch, frames, cfg, n_times, text_len_max;
  int32_t masked;        /* allocate seq_len (batch > 1, cfm.py:333-336)            */
  int32_t fused_adaln;   /* allocate ln_stats / ln_tab / ln_prep                    */
  int32_t bucketed;      /* allocate valid_len (frames is a bucket size)            */
} f5_dit_shape;
typedef const float* (*f5_tensor_lookup)(void* user, const char* mlx_name, int64_t* numel);

int64_t f5_packed_weights_bytes(const f5_dit_dims* d);
int f5_pack_weights(const f5_dit_dims* d, f5_tensor_lookup get, void* user, void* host_out);
int f5_bind_packed_weights(const f5_dit_dims* d, const void* device_base, f5_dit_weights* out,
                           f5_convnext_weights* text_blocks /* [conv_layers] */,
                           f5_dit_block_weights* blocks /* [depth] */);
int64_t f5_workspace_bytes(const f5_dit_dims* d, const f5_dit_shape* s);
int f5_bind_workspace(const f5_dit_dims* d, const f5_dit_shape* s, void* device_base, f5_dit_buffers* out, void* stream);
int f5_nccl_broadcast_weights(void* device_buf, int64_t bytes, int32_t root, void* nccl_comm, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* F5_H100_H_ */
