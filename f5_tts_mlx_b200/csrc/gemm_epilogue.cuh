// Fused GEMM epilogue of the wgmma GEMM (gemm_sm90.cuh): one thread owns one output row and 32 consecutive
// accumulator columns, read from the fp32 accumulator tile the consumer warpgroup left in shared memory.
#pragma once
#include "ptx.cuh"

namespace f5 {

enum GemmAct { ACT_NONE = 0, ACT_GELU_TANH = 1, ACT_GELU_ERF = 2, ACT_MISH = 3 };

struct GemmParams {
  int M, N, K;             // logical problem (flat mode: M rows; batched mode: see below)
  // row mapping
  int rows_per_batch;      // frames per utterance (row -> batch = row / rows_per_batch); 0 = M
  int tiles_per_batch;     // >0: M tiles never straddle utterances (batched / conv mode)
  int num_batches;
  // implicit-conv mode
  int conv_taps;           // 1 = plain GEMM
  int conv_pad;            // frames of left padding (k//2)
  int k_per_tap;           // K elements per tap (multiple of 64)
  int conv_grouped;        // 1: A channel base = output column base (block-diagonal groups of 64)
  // epilogue
  const float* bias;       // [N] or null
  void* out;               // bf16 or f32, row-major, ldo elements
  int ldo;
  const float* resid;      // f32 [rows, ldr] or null (may alias out)
  int ldr;
  const float* gate;       // f32 [N], shared by all utterances, or null
  const int* row_len;      // [num_batches] valid frames per utterance, or null
  const float2* rope;      // [rows_per_batch, 32] (cos, sin), or null
  int rope_cols;           // columns [0, rope_cols) are rotated ...
  int rope_col2;           // ... and [rope_col2, rope_col2 + rope_cols) (0: the same range again)
  float q_scale;
  int q_cols;
  __nv_bfloat16* out2;     // optional bf16 copy of the result
  int ldo2;
  unsigned long long* prof;  // in-graph timing slot (ptx.cuh prof_stamp_*), or null
  int w_static;            // B operand may be fetched before the PDL wait (weights)
  const char* pf_ptr;      // weights of a LATER GEMM to pull into L2 while this one runs, or null
  long long pf_bytes;
  // ---- fused AdaLayerNormZero (dit.py:270,289,321), by linearity of the consuming Linear ----
  //   Linear(LN(x) (1+s) + b) = rstd * ( (x (1+s)) W^T - mean * c1 ) + c2,  c1 = (1+s) W^T,  c2 = b W^T + bias
  // producer side (this GEMM writes the fp32 residual stream x): out2 <- bf16(x * (1 + ln_scale[col])) through the
  // staged store path, ln_stats[row][col/64] <- (sum, sum of squares) of each 64-column unit of the row
  const float* ln_scale;   // [N] scale vector of the NEXT AdaLN, or null
  float2* ln_stats;        // [rows][N/64]
  // consumer side (A is such an out2 matrix): the epilogue finishes the LayerNorm
  const float2* ln_in_stats;  // [rows][K/64] or null
  int ln_in_units;            // K/64
  const float* ln_tab;        // 4 rows of ln_tab_ld floats: c1_hi, c1_lo, c2_hi, c2_lo (bf16-split operand rows of
  long long ln_tab_ld;        //   the table GEMM), already offset to this GEMM's column 0
  // ---- FP8 mode of the block GEMMs (DESIGN.md section 8) ----
  int ab8;                 // A and W are e4m3 bytes: 128-element k-blocks, e4m3 wgmma
  float acc_scale;         // multiplies the accumulator (the weight tensor's quantisation scale); 1 otherwise
  int out2_fp8;            // the second output is e4m3 (1 byte per element) instead of bf16
  int out_fp8;             // the primary output is e4m3 (bf16-output instantiations only): 32-byte rows per chunk
  // ---- block-scaled FP8 (SCALED instantiations only; DESIGN.md section 8): power-of-two scales, x ~= s * e4m3 ----
  const float* a_scale;    // [K/64][a_scale_ld]: scale of A per (row, 64-column unit), or null (A unscaled)
  long long a_scale_ld;
  const float* w_scale;    // [N]: per-output-channel weight scale (multiplies acc_scale), or null
  float* out_scale;        // [N/64][M]: with out_fp8, `out` is quantised per (row, 64-column unit) and the scales written
  float* out2_scale;       // [N/64][M]: the same for out2 (out2_fp8)
  int conv_dilation;       // implicit-conv mode: frames between taps (0 or 1: adjacent frames)
  // RMSNorm consumer (f5_gemm_args.ln_rms): the row scale is sqrt(K) / max(||x||, 1e-12) from ln_in_stats, no mean
  // term and no ln_tab (the norm's gain is folded into W)
  int ln_rms;
  // BN = 128, no RoPE: the CTA's last tile is drained by both consumer warpgroups, one 64-column unit each; 0
  // drains it on its owner alone, bit for bit the same outputs (f5_gemm_test_tail_split)
  int tail_split;
};

// Each CTA touches its 1/num_ctas slice of [pf_ptr, pf_ptr + pf_bytes) with L2 prefetches (one warp,
// 128 B per lane per iteration).  At batch 1 the 0.67 GB of weights stream from HBM once per DiT
// evaluation and every GEMM would otherwise start cold, so the next GEMMs' weights are fetched ahead of time.
__device__ __forceinline__ void prefetch_slice_l2(const GemmParams& p, int cta, int num_ctas, int lane) {
  if (p.pf_ptr == nullptr) return;
  const long long per = (((p.pf_bytes + num_ctas - 1) / num_ctas) + 127) & ~127LL;
  const long long lo = (long long)cta * per;
  const long long hi = lo + per < p.pf_bytes ? lo + per : p.pf_bytes;
  for (long long o = lo + (long long)lane * 128; o < hi; o += 32 * 128)
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p.pf_ptr + o));
}

// ---------------------------------------------------------------------------------------------
// Epilogue, organised for memory-level parallelism (a load -> use chain per operand and chunk leaves the
// epilogue latency-bound):
//   * bias and gate of the tile's columns are staged in shared memory once (epi_stage_cols);
//   * the RoPE cos/sin of the thread's row (32 pairs = one head) are loaded into registers BEFORE the
//     accumulator is awaited (epi_load_rope), as is the residual of the first chunk; the residual of
//     chunk c+1 is requested before chunk c is processed (double buffer);
//   * activations use the MUFU approximations (tanh.approx / ex2.approx / lg2.approx).
// One thread owns one output row; a chunk is 32 consecutive accumulator columns.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_tanh_fast(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * fmaf(k1 * x * x, x, x);
  return 0.5f * x * (1.f + tanh_approx(u));
}
__device__ __forceinline__ float mish_fast(float x) {
  // x * tanh(softplus(x)), softplus = log(1 + e^x) (= x beyond 15)
  const float sp = x > 15.f ? x : __logf(1.f + __expf(x));
  return x * tanh_approx(sp);
}

// stage bias[n0..n0+BN) and gate[n0..n0+BN) (1 when there is no gate) into shared memory; called by the 128 epilogue
// threads, `et` = 0..127
// aux_s: c1 of the fused-LN consumer mode, or the second output's scale 1 + ln_scale (1 when there is none) — a GEMM is
// never both.  In consumer mode bias_s holds c2 + bias.
// ws_s (SCALED instantiations): acc_scale * w_scale[col], the factor of the accumulator term.
template <int BN, bool SC = false>
__device__ __forceinline__ void epi_stage_cols(const GemmParams& p, int n0, int et, float* bias_s,
                                               float* gate_s, float* aux_s, float* ws_s = nullptr) {
#pragma unroll
  for (int i = et; i < BN; i += 128) {
    const int col = n0 + i;
    const bool ok = col < p.N;
    if constexpr (SC) ws_s[i] = (p.w_scale != nullptr && ok) ? p.acc_scale * p.w_scale[col] : p.acc_scale;
    float b = (p.bias != nullptr && ok) ? p.bias[col] : 0.f;
    float x = (p.ln_scale != nullptr && ok) ? 1.f + p.ln_scale[col] : 1.f;
    if (p.ln_in_stats != nullptr && ok && !p.ln_rms) {
      const float* t = p.ln_tab + col;
      x = t[0] + t[p.ln_tab_ld];
      b += t[2 * p.ln_tab_ld] + t[3 * p.ln_tab_ld];
    }
    bias_s[i] = b;
    gate_s[i] = (p.gate != nullptr && ok) ? p.gate[col] : 1.f;
    aux_s[i] = x;
  }
}

// consumer side of the fused LN: the row's (sum, sum of squares) per 64-column unit, added in a fixed order
// (deterministic), -> (mean * rstd, rstd); eps as nn.LayerNorm(eps=1e-6) (dit.py:262,281).  Without the mode the
// pair is (0, 1), which makes the epilogue's rstd * acc - mu_r * c1 + bias the plain acc + bias.
__device__ __forceinline__ void epi_load_ln_row(const GemmParams& p, int row, bool row_ok, float& mu_r, float& rstd) {
  mu_r = 0.f; rstd = 1.f;
  if (p.ln_in_stats == nullptr || !row_ok) return;
  const float4* st = reinterpret_cast<const float4*>(p.ln_in_stats + (size_t)row * p.ln_in_units);
  float s1 = 0.f, s2 = 0.f;
  for (int u = 0; u < p.ln_in_units; u += 2) {
    const float4 v = st[u >> 1];
    s1 += v.x; s2 += v.y;
    s1 += v.z; s2 += v.w;
  }
  const float inv_k = 1.f / (64.f * p.ln_in_units);
  if (p.ln_rms) {   // RMSNorm: sqrt(K) / max(||x||, 1e-12) = rsqrt(max(sum x^2, 1e-24) / K), finite for an all-zero row
    rstd = rsqrtf(fmaxf(s2, 1e-24f) * inv_k);
    return;
  }
  const float mean = s1 * inv_k;
  rstd = rsqrtf(fmaxf(s2 * inv_k - mean * mean, 0.f) + 1e-6f);
  mu_r = mean * rstd;
}

template <bool ROPE>
__device__ __forceinline__ void epi_load_rope(const GemmParams& p, int pos, float2 (&cs)[ROPE ? 32 : 1]) {
  if (ROPE) {
    const float4* rp = reinterpret_cast<const float4*>(p.rope + (size_t)pos * 32);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float4 v = rp[j];
      cs[2 * j] = make_float2(v.x, v.y);
      cs[2 * j + 1] = make_float2(v.z, v.w);
    }
  }
}

__device__ __forceinline__ void epi_load_resid(const GemmParams& p, int row, int col0, bool row_ok,
                                               float4 (&r)[8]) {
  if (p.resid != nullptr && row_ok && col0 < p.N) {
    const float4* rr = reinterpret_cast<const float4*>(p.resid + (size_t)row * p.ldr + col0);
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = (col0 + 4 * j < p.N) ? rr[j] : make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// Stores: a thread owns a ROW, so direct 16-byte stores would land in 32 different rows per warp instruction
// (half-sector writes 4 KB apart).  So every chunk (128 rows x 32 columns) is written to shared memory in the
// layout of a swizzled TMA box (fp32: 128-byte rows, SWIZZLE_128B; bf16: 64-byte rows, SWIZZLE_64B — the XOR patterns
// below are exactly those) and ONE thread hands it to the TMA unit (cp.async.bulk.tensor store), which also clips
// rows / columns outside the matrix.  The fp32 accumulator tile is itself BN / 32 such fp32 boxes (16 KB each), so an
// fp32 chunk is written back in place over the accumulator values its thread has just read (its own row) and stored
// from there; bf16 / e4m3 chunks, and the second output, go to two alternating 8 KB staging buffers.  Per chunk one
// named barrier (128 threads).
struct EpiStage {
  uint8_t* acc;            // the tile's fp32 accumulator boxes: BN / 32 x (128 rows x 128 bytes, SWIZZLE_128B), 1024-aligned
  uint8_t* stg;            // 2 x 8 KB staging of the bf16 / e4m3 output, or of the second output (1024-aligned)
  int et;                  // epilogue thread 0..127 of the warpgroup; thread 0 issues the TMA stores
  int r;                   // this thread's row inside the tile
  int bar_id;              // named barrier of the epilogue warpgroup
  const CUtensorMap* map_out;   // (cols, rows per utterance, utterances) of `out` / `out2`
  const CUtensorMap* map_out2;
  int c1, c2;              // tensor-map coordinates of tile row 0: row inside the utterance, utterance
  int out_fp8;             // primary output as e4m3 (GemmParams::out_fp8)
  float mu_r, rstd;        // fused-LN consumer mode: this thread's row statistics ((0, 1) otherwise)
};

// this thread's row of a 128 x 32 fp32 box (SWIZZLE_128B: 16-byte piece j of row r at (j ^ (r & 7)) * 16)
__device__ __forceinline__ void epi_stage_f32(uint8_t* buf, int r, const float (&v)[32]) {
  uint8_t* mine = buf + r * 128;
  const int sw = r & 7;
#pragma unroll
  for (int j = 0; j < 8; ++j)
    *reinterpret_cast<float4*>(mine + ((j ^ sw) * 16)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
}

// chunk `ch` (columns [32 ch, 32 ch + 32) of the tile) of `out`, with its second output `w2` (bf16, 4 x uint4 per row,
// or e4m3 when `w2_fp8`: 32-byte rows, SWIZZLE_32B = 16-byte piece index ^ bit 7 of the row offset) or nullptr
template <bool OUT_BF16>
__device__ __forceinline__ void epi_store_tma(const float (&v)[32], const EpiStage& st, int ch, int col0,
                                              const uint4* w2 = nullptr, bool w2_fp8 = false) {
  uint8_t* box = st.acc + ch * 16384;
  uint8_t* buf = st.stg + (ch & 1) * 8192;
  if (OUT_BF16 && st.out_fp8) {
    uint8_t* mine = buf + st.r * 32;           // e4m3: 32-byte rows, SWIZZLE_32B
    const int sw = (st.r >> 2) & 1;
#pragma unroll
    for (int j = 0; j < 2; ++j)
      *reinterpret_cast<uint4*>(mine + ((j ^ sw) * 16)) =
          make_uint4(pack_e4m3x4(v[16 * j], v[16 * j + 1], v[16 * j + 2], v[16 * j + 3]),
                     pack_e4m3x4(v[16 * j + 4], v[16 * j + 5], v[16 * j + 6], v[16 * j + 7]),
                     pack_e4m3x4(v[16 * j + 8], v[16 * j + 9], v[16 * j + 10], v[16 * j + 11]),
                     pack_e4m3x4(v[16 * j + 12], v[16 * j + 13], v[16 * j + 14], v[16 * j + 15]));
  } else if (OUT_BF16) {
    uint8_t* mine = buf + st.r * 64;
    const int sw = (st.r >> 1) & 3;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<uint4*>(mine + ((j ^ sw) * 16)) =
          make_uint4(pack_bf16x2(v[8 * j], v[8 * j + 1]), pack_bf16x2(v[8 * j + 2], v[8 * j + 3]),
                     pack_bf16x2(v[8 * j + 4], v[8 * j + 5]), pack_bf16x2(v[8 * j + 6], v[8 * j + 7]));
  } else {
    epi_stage_f32(box, st.r, v);
  }
  if (w2 != nullptr) {   // fp32 `out` only: the staging buffers are free for the second output
    if (w2_fp8) {
      uint8_t* mine2 = buf + st.r * 32;
      const int sw2 = (st.r >> 2) & 1;
#pragma unroll
      for (int j = 0; j < 2; ++j) *reinterpret_cast<uint4*>(mine2 + ((j ^ sw2) * 16)) = w2[j];
    } else {
      uint8_t* mine2 = buf + st.r * 64;
      const int sw2 = (st.r >> 1) & 3;
#pragma unroll
      for (int j = 0; j < 4; ++j) *reinterpret_cast<uint4*>(mine2 + ((j ^ sw2) * 16)) = w2[j];
    }
  }
  fence_proxy_async_smem();                           // generic-proxy writes -> visible to the TMA unit
  // the OTHER staging buffer is rewritten by the next chunk: every store issued so far must have read its source
  // (the previous chunk's store was issued a whole chunk of work ago)
  if (st.et == 0) tma_store_wait_read<0>();
  asm volatile("bar.sync %0, 128;" ::"r"(st.bar_id) : "memory");
  if (st.et == 0) {
    tma_store_3d(st.map_out, OUT_BF16 ? buf : box, col0, st.c1, st.c2);
    if (w2 != nullptr) tma_store_3d(st.map_out2, buf, col0, st.c1, st.c2);
    tma_store_commit();
  }
}

// Block-scaled e4m3 output of one 64-column unit (the unit's scale needs both chunks, so it is quantised and stored once
// chunk B is done).  Chunk A is not held in registers: its fp32 values wait in chunk A's accumulator box (its thread's
// own row), written there by HALF 0 — as the in-place fp32 `out` store of the producer form, or, for the e4m3 primary
// output, by this thread alone (no barrier) — and are read back by the same thread in HALF 1.

// e4m3 codes of 32 values x = v * aux (aux = null: x = v), quantised as x * inv (inv = 1 / scale, exact)
__device__ __forceinline__ void epi_quant32(const float (&v)[32], const float* aux, float inv, uint4 (&q)[2]) {
  uint32_t w[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) x[k] = (aux != nullptr ? v[4 * i + k] * aux[4 * i + k] : v[4 * i + k]) * inv;
    w[i] = pack_e4m3x4(x[0], x[1], x[2], x[3]);
  }
  q[0] = make_uint4(w[0], w[1], w[2], w[3]);
  q[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// the same for chunk A, read back from this thread's row of its fp32 box
__device__ __forceinline__ void epi_quant32_staged(const uint8_t* buf, int r, const float* aux, float inv, uint4 (&q)[2]) {
  const uint8_t* mine = buf + r * 128;
  const int sw = r & 7;
  uint32_t w[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 a = *reinterpret_cast<const float4*>(mine + ((i ^ sw) * 16));
    float x[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) x[k] = (aux != nullptr ? x[k] * aux[4 * i + k] : x[k]) * inv;
    w[i] = pack_e4m3x4(x[0], x[1], x[2], x[3]);
  }
  q[0] = make_uint4(w[0], w[1], w[2], w[3]);
  q[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// HALF 1 of a block-scaled unit (chunks chA, chA + 1): the unit's scale from the running amax (NaN propagates), written
// to scale[colA / 64][row] (rows past the matrix write none); then the e4m3 chunks A (colA) and B (colA + 32) are staged
// as 32-byte rows (SWIZZLE_32B), 4 KB each, in the unit's 8 KB staging buffer (units alternate between the two, so a
// unit never rewrites the buffer the previous unit's store may still read) — of `out` (OUT_BF16: the e4m3 primary
// output) or of out2 (with the fp32 chunk B of `out` written in place in its box) — and stored.  Each staged piece is
// written as soon as it is formed, so that few values are live at once.
template <bool OUT_BF16>
__device__ __forceinline__ void epi_finish_unit8(const float (&v)[32], const float* aux, float amax, float* scale,
                                                 int M, int colA, int row, bool row_ok, const EpiStage& st, int chA) {
  float inv;
  const float s = e4m3_block_scale(amax, inv);
  if (row_ok) scale[(size_t)(colA >> 6) * M + row] = s;
  uint8_t* q8 = st.stg + ((chA >> 1) & 1) * 8192;
  const int sw = (st.r >> 2) & 1;
  {
    uint4 q[2];
    epi_quant32(v, aux, inv, q);
#pragma unroll
    for (int j = 0; j < 2; ++j) *reinterpret_cast<uint4*>(q8 + 4096 + st.r * 32 + ((j ^ sw) * 16)) = q[j];
  }
  uint8_t* box_b = st.acc + (chA + 1) * 16384;
  if constexpr (!OUT_BF16) epi_stage_f32(box_b, st.r, v);
  {
    uint4 q[2];
    epi_quant32_staged(st.acc + chA * 16384, st.r, aux != nullptr ? aux - 32 : nullptr, inv, q);
#pragma unroll
    for (int j = 0; j < 2; ++j) *reinterpret_cast<uint4*>(q8 + st.r * 32 + ((j ^ sw) * 16)) = q[j];
  }
  fence_proxy_async_smem();
  if (st.et == 0) tma_store_wait_read<0>();
  asm volatile("bar.sync %0, 128;" ::"r"(st.bar_id) : "memory");
  if (st.et == 0) {
    if constexpr (!OUT_BF16) tma_store_3d(st.map_out, box_b, colA + 32, st.c1, st.c2);
    const CUtensorMap* m8 = OUT_BF16 ? st.map_out : st.map_out2;
    tma_store_3d(m8, q8, colA, st.c1, st.c2);
    tma_store_3d(m8, q8 + 4096, colA + 32, st.c1, st.c2);
    tma_store_commit();
  }
}

// HALF: which 32-column half of a 64-column head this chunk is (static RoPE register indexing); `ch`: the chunk's index
// in the tile (its accumulator box)
// `unit_acc`: running (sum, sum of squares) of this thread's row over the 64-column unit (HALF 0 starts it, HALF 1
// completes and stores it) — fused-LN producer mode only.
// SC (block-scaled instantiations): the accumulator term is multiplied by ws_s[col] (acc_scale * w_scale); a block-scaled
// e4m3 output carries the running amax of its 64-column unit from chunk A to chunk B in `unit_amax`.
template <int ACT, bool OUT_BF16, bool ROPE, int HALF, bool SC = false>
__device__ __forceinline__ void epi_apply(const uint32_t (&acc)[32], const float4 (&res)[8],
                                          const float* bias_s, const float* gate_s, const float* aux_s,
                                          const float2 (&cs)[ROPE ? 32 : 1], const GemmParams& p,
                                          int col0, int ch, int row, bool row_ok, bool row_valid,
                                          const EpiStage& st, float2& unit_acc, const float* ws_s = nullptr,
                                          float* unit_amax = nullptr) {
  float v[32];
  // rstd * acc - (mean * rstd) * c1 + (c2 + bias): the fused-LN consumer; (mu_r, rstd) = (0, 1) otherwise.
  // acc_scale (the e4m3 weight tensor's scale in FP8 mode, else 1) belongs to the accumulator term only.
  if constexpr (SC) {
    // rstd * w_s[col] * acc - mu_r * c1 + c2 for the fused-LN consumer, and acc * w_s[col] + bias otherwise: with
    // (mu_r, rstd) = (0, 1) the same expression (rstd * w_s = w_s and -0 * aux + bias = bias exactly; aux is 1 + s or 1)
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      const float4 bb = *reinterpret_cast<const float4*>(bias_s + j);
      const float4 cc = *reinterpret_cast<const float4*>(aux_s + j);
      const float4 ww = *reinterpret_cast<const float4*>(ws_s + j);
      v[j] = fmaf(__uint_as_float(acc[j]), st.rstd * ww.x, fmaf(-st.mu_r, cc.x, bb.x));
      v[j + 1] = fmaf(__uint_as_float(acc[j + 1]), st.rstd * ww.y, fmaf(-st.mu_r, cc.y, bb.y));
      v[j + 2] = fmaf(__uint_as_float(acc[j + 2]), st.rstd * ww.z, fmaf(-st.mu_r, cc.z, bb.z));
      v[j + 3] = fmaf(__uint_as_float(acc[j + 3]), st.rstd * ww.w, fmaf(-st.mu_r, cc.w, bb.w));
    }
  } else if (p.ln_in_stats != nullptr) {   // uniform: only a fused-LN consumer pays for the mean term
    const float ra = st.rstd * p.acc_scale;
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      const float4 bb = *reinterpret_cast<const float4*>(bias_s + j);
      const float4 cc = *reinterpret_cast<const float4*>(aux_s + j);
      v[j] = fmaf(__uint_as_float(acc[j]), ra, fmaf(-st.mu_r, cc.x, bb.x));
      v[j + 1] = fmaf(__uint_as_float(acc[j + 1]), ra, fmaf(-st.mu_r, cc.y, bb.y));
      v[j + 2] = fmaf(__uint_as_float(acc[j + 2]), ra, fmaf(-st.mu_r, cc.z, bb.z));
      v[j + 3] = fmaf(__uint_as_float(acc[j + 3]), ra, fmaf(-st.mu_r, cc.w, bb.w));
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      const float4 bb = *reinterpret_cast<const float4*>(bias_s + j);
      v[j] = fmaf(__uint_as_float(acc[j]), p.acc_scale, bb.x);
      v[j + 1] = fmaf(__uint_as_float(acc[j + 1]), p.acc_scale, bb.y);
      v[j + 2] = fmaf(__uint_as_float(acc[j + 2]), p.acc_scale, bb.z);
      v[j + 3] = fmaf(__uint_as_float(acc[j + 3]), p.acc_scale, bb.w);
    }
  }
  if (ACT == ACT_GELU_TANH) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = gelu_tanh_fast(v[j]);
  } else if (ACT == ACT_GELU_ERF) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = gelu_erf_f(v[j]);
  } else if (ACT == ACT_MISH) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = mish_fast(v[j]);
  }
  if (ROPE) {
    // uniform per chunk (heads are 64 columns, so whole chunks); rope_col2 = 0 repeats the first range
    if (col0 < p.rope_cols || (unsigned)(col0 - p.rope_col2) < (unsigned)p.rope_cols) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 c = cs[HALF * 16 + j];
        const float a = v[2 * j], b = v[2 * j + 1];
        v[2 * j] = a * c.x - b * c.y;
        v[2 * j + 1] = b * c.x + a * c.y;
      }
    }
    if (col0 < p.q_cols) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] *= p.q_scale;
    }
  }
  if (p.row_len != nullptr) {     // uniform: GEMMs without a row mask skip the 32 predicated moves
    if (!row_valid) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = 0.f;
    }
  }
  // residual + gate * v as one FMA per element; without a gate gate_s is 1, and fmaf(v, 1, r) rounds exactly as v + r
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 gg = *reinterpret_cast<const float4*>(gate_s + 4 * j);
    v[4 * j] = fmaf(v[4 * j], gg.x, res[j].x); v[4 * j + 1] = fmaf(v[4 * j + 1], gg.y, res[j].y);
    v[4 * j + 2] = fmaf(v[4 * j + 2], gg.z, res[j].z); v[4 * j + 3] = fmaf(v[4 * j + 3], gg.w, res[j].w);
  }
  if constexpr (!OUT_BF16) {
    if (p.out2 != nullptr) {
      // second output: bf16(v * aux) — the fused-LN operand x * (1 + s) of the GEMM that consumes LN(x) (aux = 1 when
      // no ln_scale is given: a plain bf16 copy); with ln_stats also the unit statistics of the finished row
      if (p.ln_stats != nullptr) {
        // four partial sums each: a 32-long dependent add chain costs more than the rest of the chunk's arithmetic
        float s1[4] = {HALF == 0 ? 0.f : unit_acc.x, 0.f, 0.f, 0.f}, s2[4] = {HALF == 0 ? 0.f : unit_acc.y, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
#pragma unroll
          for (int i = 0; i < 4; ++i) { s1[i] += v[j + i]; s2[i] = fmaf(v[j + i], v[j + i], s2[i]); }
        }
        unit_acc = make_float2((s1[0] + s1[1]) + (s1[2] + s1[3]), (s2[0] + s2[1]) + (s2[2] + s2[3]));
        if (HALF == 1 && row_ok && col0 < p.N) p.ln_stats[(size_t)row * (p.N >> 6) + (col0 >> 6)] = unit_acc;
      }
      if constexpr (SC) {
        if (p.out2_fp8 && p.out2_scale != nullptr) {   // block-scaled e4m3 operand x (1 + s): one scale per unit
          float amax = HALF == 0 ? 0.f : *unit_amax;
#pragma unroll
          for (int j = 0; j < 32; ++j) amax = fmax_nan(amax, fabsf(v[j] * aux_s[j]));
          if (HALF == 0) {
            *unit_amax = amax;
            epi_store_tma<OUT_BF16>(v, st, ch, col0);    // the fp32 chunk A leaves now (and stays in its box)
          } else {
            epi_finish_unit8<OUT_BF16>(v, aux_s, amax, p.out2_scale, p.M, col0 - 32, row, row_ok, st, ch - 1);
          }
          return;
        }
      }
      uint4 w2[4];
      if (p.out2_fp8) {      // e4m3 operand of an FP8-mode consumer: 32 bytes per row and chunk
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          uint32_t q[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float4 sc = *reinterpret_cast<const float4*>(aux_s + 16 * j + 4 * i);
            q[i] = pack_e4m3x4(v[16 * j + 4 * i] * sc.x, v[16 * j + 4 * i + 1] * sc.y, v[16 * j + 4 * i + 2] * sc.z,
                               v[16 * j + 4 * i + 3] * sc.w);
          }
          w2[j] = make_uint4(q[0], q[1], q[2], q[3]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float4 s0 = *reinterpret_cast<const float4*>(aux_s + 8 * j);
          const float4 s1 = *reinterpret_cast<const float4*>(aux_s + 8 * j + 4);
          w2[j] = make_uint4(pack_bf16x2(v[8 * j] * s0.x, v[8 * j + 1] * s0.y), pack_bf16x2(v[8 * j + 2] * s0.z, v[8 * j + 3] * s0.w),
                             pack_bf16x2(v[8 * j + 4] * s1.x, v[8 * j + 5] * s1.y), pack_bf16x2(v[8 * j + 6] * s1.z, v[8 * j + 7] * s1.w));
        }
      }
      epi_store_tma<OUT_BF16>(v, st, ch, col0, w2, p.out2_fp8 != 0);
      return;
    }
  }
  if constexpr (SC && OUT_BF16) {
    if (st.out_fp8 && p.out_scale != nullptr) {   // block-scaled e4m3 output (FF1's GELU output)
      float amax = HALF == 0 ? 0.f : *unit_amax;
#pragma unroll
      for (int j = 0; j < 32; ++j) amax = fmax_nan(amax, fabsf(v[j]));
      if (HALF == 0) {
        *unit_amax = amax;
        epi_stage_f32(st.acc + ch * 16384, st.r, v);   // chunk A waits in its own row of its fp32 box
      } else {
        epi_finish_unit8<OUT_BF16>(v, nullptr, amax, p.out_scale, p.M, col0 - 32, row, row_ok, st, ch - 1);
      }
      return;
    }
  }
  epi_store_tma<OUT_BF16>(v, st, ch, col0);   // all 128 threads of the warpgroup take part (barrier inside)
}

// the 32 fp32 accumulator columns of this thread's row in a 128 x 32 box (SWIZZLE_128B, as epi_stage_f32 writes them)
__device__ __forceinline__ void acc_ld32(const uint8_t* box, int r, uint32_t (&acc)[32]) {
  const uint8_t* mine = box + r * 128;
  const int sw = r & 7;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 v = *reinterpret_cast<const float4*>(mine + ((j ^ sw) * 16));
    acc[4 * j] = __float_as_uint(v.x); acc[4 * j + 1] = __float_as_uint(v.y);
    acc[4 * j + 2] = __float_as_uint(v.z); acc[4 * j + 3] = __float_as_uint(v.w);
  }
}

// Drains the 64-column units [cc0, cc0 + ncc) of an accumulator tile of BN columns (st.acc: its BN / 32 fp32 boxes;
// this thread's row st.r).  `res0` holds the residual of unit cc0's first 32 columns (loaded here instead in the RoPE
// and block-scaled forms).
template <int BN, int ACT, bool OUT_BF16, bool ROPE, bool SC = false>
__device__ __forceinline__ void epi_drain_tile(const float* bias_s, const float* gate_s, const float* aux_s,
                                               const float2 (&cs)[ROPE ? 32 : 1], float4 (&res0)[8], const GemmParams& p,
                                               int n0, int cc0, int ncc, int row, bool row_ok, bool row_valid,
                                               const EpiStage& st, const float* ws_s = nullptr) {
  float4 res1[8];
  float2 unit_acc = make_float2(0.f, 0.f);
  float unit_amax = 0.f;
#pragma unroll 1
  for (int cc = cc0; cc < cc0 + ncc; ++cc) {
    const int colA = n0 + cc * 64, colB = colA + 32;
    uint32_t acc[32];
    // chunk A (first half of the head): request chunk B's residual, then drain A.  A later unit's first residual is
    // requested here too, not under the previous chunk B.  The RoPE and block-scaled epilogues hold more registers
    // (the head's cos / sin, the unit's amax): they request chunk B's residual after chunk A (RoPE GEMMs get none).
    constexpr bool kLateB = ROPE || SC;
    if (kLateB || cc > cc0) epi_load_resid(p, row, colA, row_ok, res0);
    if constexpr (!kLateB) epi_load_resid(p, row, colB, row_ok, res1);
    acc_ld32(st.acc + (2 * cc) * 16384, st.r, acc);
    if (colA < p.N)   // uniform per CTA
      epi_apply<ACT, OUT_BF16, ROPE, 0, SC>(acc, res0, bias_s + cc * 64, gate_s + cc * 64, aux_s + cc * 64, cs, p, colA,
                                            2 * cc, row, row_ok, row_valid, st, unit_acc, SC ? ws_s + cc * 64 : nullptr,
                                            &unit_amax);
    // chunk B
    if constexpr (kLateB) epi_load_resid(p, row, colB, row_ok, res1);
    acc_ld32(st.acc + (2 * cc + 1) * 16384, st.r, acc);
    if (colB < p.N)
      epi_apply<ACT, OUT_BF16, ROPE, 1, SC>(acc, res1, bias_s + cc * 64 + 32, gate_s + cc * 64 + 32, aux_s + cc * 64 + 32, cs,
                                            p, colB, 2 * cc + 1, row, row_ok, row_valid, st, unit_acc,
                                            SC ? ws_s + cc * 64 + 32 : nullptr, &unit_amax);
  }
}

}  // namespace f5
