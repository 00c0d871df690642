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
/* optional per-kernel-family device timing: enable, run, then read
 * out[kinds][4] = {milliseconds, algorithmic flops, bytes, launches}; kinds: 0 GEMM, 1 attention,
 * 2 LayerNorm+modulate, 3 everything else. */
/* sizeof() of the ABI structs in declaration order: f5_gemm_args, f5_convnext_weights,
 * f5_dit_block_weights, f5_dit_weights, f5_dit_buffers, f5_vocos_block_weights, f5_vocos_weights,
 * f5_vocos_buffers, f5_duration_weights, f5_duration_buffers — lets a binding check its layout at
 * load time.  Returns the count (10). */
int f5_struct_sizes(int32_t* out, int32_t n);
int f5_prof_enable(int on);
int f5_prof_summary(double* out, int kinds);
/* In-situ kernel timing inside a captured CUDA graph (bench.py's roofline): install a device buffer of max_slots x 2
 * uint64; from then on the i-th launched kernel of the tensor-core families (GEMM, attention) gets slot i and writes
 * [i][0] = min over its CTAs of %globaltimer after the dependency wait, [i][1] = max over CTAs at exit (the caller
 * presets the columns to UINT64_MAX / 0 before each replay).  f5_prof_graph_meta returns the family (kinds as above)
 * and the algorithmic flops / bytes of every slot handed out since the install; slots = NULL uninstalls. */
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
  const float* gate;      /* fp32 [num_batches, gate_ld] or NULL                                */
  int64_t gate_ld;
  const int32_t* row_len; /* [num_batches] valid frames (rows beyond are written as 0) or NULL  */
  const float* rope;      /* fp32 [rows_per_batch, 32, 2] (cos,sin) or NULL                     */
  int32_t rope_cols;      /* columns [0, rope_cols) are rotated in adjacent pairs               */
  float q_scale;          /* columns [0, q_cols) are multiplied by q_scale after the rotation   */
  int32_t q_cols;
  int32_t tile_n;         /* 0 = auto, else 64 | 128 (192 | 256 are accepted and run as 128)     */
  void* out2_bf16;        /* optional second copy of the result as bf16 [rows, ldo2], or NULL    */
  int64_t ldo2;
  int32_t variant;        /* 0 | 1 | 2, kept for ABI compatibility: sm_90 has one 128xBN kernel   */
  int32_t w_static;       /* nonzero: `w` is never written by work that precedes this call on the stream
                             (model weights): the kernel may start fetching it before its programmatic
                             dependency on the preceding kernel has resolved                           */
  void* debug_ts;         /* NULL, or uint64 [ctas, 10]: per-CTA phase timestamps (globaltimer ns)  */
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
} f5_gemm_args;

int f5_gemm_bf16(const f5_gemm_args* args, void* stream);
/* debug aid: the next `max_calls` f5_gemm_bf16 calls without their own debug_ts write their per-CTA
 * timestamps to base + i * stride_bytes (i = call index); pass NULL to stop. */
int f5_debug_gemm_ts(void* base, int64_t stride_bytes, int32_t max_calls);

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
/* kept for ABI compatibility: accepts any `base` and returns 0; the attention kernel records no timeline */
int f5_debug_attention_ts(void* base);

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
  /* FP8 mode (optional, NULL = bf16 only): e4m3 copies of the QKV / FF1 weights, ONE scale per tensor
   * (w ~= scale * e4m3); used by f5_dit_forward when f5_dit_buffers.a_fp8 is set (see f5_gemm_args.ab_fp8).  With
   * out_w8 / ff2_w8 also the out-projection (attention writes e4m3) and FF2 (FF1 writes e4m3) run in FP8. */
  const void* qkv_w8; const void* ff1_w8; const void* out_w8; const void* ff2_w8;
  float qkv_s8, ff1_s8, out_s8, ff2_s8;
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
  /* Fused AdaLN (see f5_gemm_args.ln_*): all three non-NULL selects it, any NULL keeps the separate
   * f5_ln_modulate launches.  ln_tab_ld = depth*(3D + ff_inner) + 128 (f5_dit_ln_tab_ld). */
  float* ln_stats;            /* fp32 [rows, D/64, 2]: per-row (sum, sum of squares) per 64 columns of the residual stream */
  float* ln_tab;              /* fp32 [4*n_times, ln_tab_ld]: c1/c2 operand rows per time, columns = per block [qkv 3D | ff1 F], then proj_out */
  void* ln_prep;              /* bf16 [2*depth+1, 4*n_times, D]: operand rows of the table GEMMs */
  /* Frame bucketing (plan reuse across utterances of different length): the buffers are sized for `frames` rows per
   * utterance but only the first valid_len[u] (= the reference's N, cfm.py:319) exist; rows beyond are kept exactly
   * zero where the reference's zero padding would be seen (the k=31 ConvPositionEmbedding input, dit.py:45) and are
   * masked as attention keys, so rows < N equal the unpadded computation.  NULL = all `frames` rows are real. */
  const int32_t* valid_len;   /* int32 [rows/frames], every entry the same N <= frames, or NULL */
  /* FP8 mode: e4m3 [rows, D] — the AdaLN-modulated operand of the QKV / FF1 GEMMs (written by the producing GEMM's
   * epilogue instead of a_bf16); requires the fused AdaLN buffers and blocks[i].qkv_w8 / ff1_w8.  NULL = bf16. */
  void* a_fp8;
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
