// HBM-bound kernels of the DiT path (sm_90a).  All are coalesced / 128-bit vectorised, one warp
// per frame row where a row reduction is needed, fp32 arithmetic, bf16 only as the tensor-core
// operand they hand to the next GEMM.
#pragma once
#include "ptx.cuh"
#include "launch.h"

namespace f5 {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------
// LayerNorm (eps 1e-6, biased variance, two-pass in registers) followed by
//   MODULATE: y = ln(x) * (1 + scale[b]) + shift[b]      (AdaLayerNormZero, dit.py:270,289,321)
//   AFFINE  : y = ln(x) * w + b                           (nn.LayerNorm, convnext_v2.py:38,49)
// x: fp32 [rows, D]; y: bf16 [rows, D].  One warp per row; D = 128 * VEC_ITERS.
// ---------------------------------------------------------------------------------------------
template <int D, bool OUT_F32>
__global__ void __launch_bounds__(256)
ln_mod_kernel(const float* __restrict__ x, void* __restrict__ y, int rows,
              int rows_per_batch, const float* __restrict__ scale, const float* __restrict__ shift,
              long long mod_batch_stride, int add_one) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int IT = D / 128;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)warp * D);
  // the modulation vectors do not depend on x: request them together with the row, so that their L2 round
  // trip overlaps the row's instead of following the two reductions
  const int b_idx = rows_per_batch > 0 ? warp / rows_per_batch : 0;
  const float4* sc = reinterpret_cast<const float4*>(scale + (size_t)b_idx * mod_batch_stride);
  const float4* sh = reinterpret_cast<const float4*>(shift + (size_t)b_idx * mod_batch_stride);
  float4 v[IT], g[IT], h[IT];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < IT; ++i) v[i] = xr[i * 32 + lane];
#pragma unroll
  for (int i = 0; i < IT; ++i) {
    g[i] = sc[i * 32 + lane];
    h[i] = sh[i * 32 + lane];
  }
#pragma unroll
  for (int i = 0; i < IT; ++i) s += v[i].x + v[i].y + v[i].z + v[i].w;
  const float mean = warp_sum(s) * (1.f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < IT; ++i) {
    float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += a * a + b * b + c * c + d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + 1e-6f);
  const float one = add_one ? 1.f : 0.f;
#pragma unroll
  for (int i = 0; i < IT; ++i) {
    float a = (v[i].x - mean) * rstd * (one + g[i].x) + h[i].x;
    float b = (v[i].y - mean) * rstd * (one + g[i].y) + h[i].y;
    float c = (v[i].z - mean) * rstd * (one + g[i].z) + h[i].z;
    float d = (v[i].w - mean) * rstd * (one + g[i].w) + h[i].w;
    if (OUT_F32)
      reinterpret_cast<float4*>(reinterpret_cast<float*>(y) + (size_t)warp * D)[i * 32 + lane] =
          make_float4(a, b, c, d);
    else
      reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(y) + (size_t)warp * D)[i * 32 + lane] =
          make_uint2(pack_bf16x2(a, b), pack_bf16x2(c, d));
  }
}

// ---------------------------------------------------------------------------------------------
// Operand rows of the fused-AdaLN table GEMMs (f5_dit_precompute): for LN site s (2l: attn_norm of block l, 2l+1:
// its ff_norm, 2L: norm_out) and evaluation time t, the four bf16 rows hi(1+scale), lo(1+scale), hi(shift),
// lo(shift) with hi = bf16(v), lo = bf16(v - hi) — the GEMM against the consuming Linear's weight then yields
// c1 = (1+scale) W^T and c2 = shift W^T to ~16 bits from bf16 tensor-core operands.
// mod: fp32 [T, NM] (per block: shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp; then norm_out's
// scale, shift — dit.py:268,287); prep: bf16 [2L+1][4T][D].
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ln_tab_prep_kernel(const float* __restrict__ mod, __nv_bfloat16* __restrict__ prep, int T, int L, int D, int NM) {
  pdl_launch_dependents();
  pdl_wait();
  const int site = blockIdx.y, t = blockIdx.x;
  long long off_scale, off_shift;
  if (site < 2 * L) {
    const long long base = (long long)(site >> 1) * 6 * D + ((site & 1) ? 3 * D : 0);
    off_shift = base; off_scale = base + D;
  } else {
    off_scale = (long long)L * 6 * D; off_shift = off_scale + D;
  }
  const float* m = mod + (size_t)t * NM;
  __nv_bfloat16* o = prep + ((size_t)site * 4 * T + 4 * t) * D;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    const float a = 1.f + m[off_scale + c], b = m[off_shift + c];
    const __nv_bfloat16 ah = __float2bfloat16(a), bh = __float2bfloat16(b);
    o[c] = ah;
    o[D + c] = __float2bfloat16(a - __bfloat162float(ah));
    o[2 * D + c] = bh;
    o[3 * D + c] = __float2bfloat16(b - __bfloat162float(bh));
  }
}

// ---------------------------------------------------------------------------------------------
// Depthwise Conv1d(k=7, pad 3, groups=C, +bias) over frames, then affine LayerNorm(eps 1e-6):
// the first half of ConvNeXtV2Block (convnext_v2.py:35-38,48-49) and of a Vocos ConvNeXt block.
// x: fp32 [B, N, C] channels-last; wt: fp32 [7, C] (tap-major); y: bf16 [B*N, C].
// One warp per (b, n); each lane owns C/32 channels as float4 groups.
// ---------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256)
dwconv7_ln_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int B, int N,
                  const float* __restrict__ wt, const float* __restrict__ wb,
                  const float* __restrict__ ln_w, const float* __restrict__ ln_b) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int IT = C / 128;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= B * N) return;
  const int b = warp / N, n = warp - b * N;
  float4 acc[IT];
#pragma unroll
  for (int i = 0; i < IT; ++i) acc[i] = reinterpret_cast<const float4*>(wb)[i * 32 + lane];
#pragma unroll
  for (int t = 0; t < 7; ++t) {
    const int nn = n + t - 3;
    if (nn < 0 || nn >= N) continue;
    const float4* xr = reinterpret_cast<const float4*>(x + ((size_t)b * N + nn) * C);
    const float4* wr = reinterpret_cast<const float4*>(wt + (size_t)t * C);
#pragma unroll
    for (int i = 0; i < IT; ++i) {
      const float4 xv = xr[i * 32 + lane];
      const float4 wv = wr[i * 32 + lane];
      acc[i].x += xv.x * wv.x; acc[i].y += xv.y * wv.y;
      acc[i].z += xv.z * wv.z; acc[i].w += xv.w * wv.w;
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < IT; ++i) s += acc[i].x + acc[i].y + acc[i].z + acc[i].w;
  const float mean = warp_sum(s) * (1.f / C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < IT; ++i) {
    float a = acc[i].x - mean, bb = acc[i].y - mean, c = acc[i].z - mean, d = acc[i].w - mean;
    q += a * a + bb * bb + c * c + d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.f / C) + 1e-6f);
  uint2* yo = reinterpret_cast<uint2*>(y + (size_t)warp * C);
#pragma unroll
  for (int i = 0; i < IT; ++i) {
    const float4 g = reinterpret_cast<const float4*>(ln_w)[i * 32 + lane];
    const float4 h = reinterpret_cast<const float4*>(ln_b)[i * 32 + lane];
    float a = (acc[i].x - mean) * rstd * g.x + h.x;
    float bb = (acc[i].y - mean) * rstd * g.y + h.y;
    float c = (acc[i].z - mean) * rstd * g.z + h.z;
    float d = (acc[i].w - mean) * rstd * g.w + h.w;
    yo[i * 32 + lane] = make_uint2(pack_bf16x2(a, bb), pack_bf16x2(c, d));
  }
}

// ---------------------------------------------------------------------------------------------
// GRN (convnext_v2.py:15-18): Gx[b,c] = ||x[b,:,c]||_2 over ALL N frames (padded ones included),
// Nx = Gx / (mean_c Gx + 1e-6), y = gamma * (x * Nx) + beta + x.
// Three tiny kernels, DETERMINISTIC (no atomics: with fp32 atomics the summation order changes run
// to run, and the 1-ulp noise is amplified to ~1e-3 by the bf16 roundings downstream, which broke
// bitwise reproducibility of sample()): per-32-frame partial sums of squares -> fixed-order
// reduction + per-utterance normalisation -> apply.
// h: bf16 [B, N, C]; scratch: fp32 [B, 1 + ceil(N/32), C] (slot 0 = Nx, slots 1.. = partials).
// ---------------------------------------------------------------------------------------------
constexpr int kGrnRowsPerBlock = 32;

__global__ void __launch_bounds__(256)
grn_sumsq_kernel(const __nv_bfloat16* __restrict__ h, float* __restrict__ scratch, int N, int C,
                 int nblk, const int* __restrict__ valid_len) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const int r0 = blockIdx.x * kGrnRowsPerBlock;
  // frame bucketing: rows >= valid_len[b] do not exist in the reference's (b, N, C) tensor — they must not enter the norm
  const int nv = valid_len != nullptr ? min(N, valid_len[b]) : N;
  const int r1 = min(nv, r0 + kGrnRowsPerBlock);
  float* part = scratch + ((size_t)b * (1 + nblk) + 1 + blockIdx.x) * C;
  for (int c4 = threadIdx.x * 4; c4 < C; c4 += blockDim.x * 4) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int r = r0; r < r1; ++r) {
      const uint2 u = *reinterpret_cast<const uint2*>(h + ((size_t)b * N + r) * C + c4);
      const __nv_bfloat162 p0 = *reinterpret_cast<const __nv_bfloat162*>(&u.x);
      const __nv_bfloat162 p1 = *reinterpret_cast<const __nv_bfloat162*>(&u.y);
      const float2 f0 = __bfloat1622float2(p0), f1 = __bfloat1622float2(p1);
      a0 += f0.x * f0.x; a1 += f0.y * f0.y; a2 += f1.x * f1.x; a3 += f1.y * f1.y;
    }
    *reinterpret_cast<float4*>(part + c4) = make_float4(a0, a1, a2, a3);
  }
}

// slot 0 of the utterance's scratch <- Nx[c]
__global__ void __launch_bounds__(256)
grn_finalize_kernel(float* __restrict__ scratch, int C, int nblk) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8];
  float* base = scratch + (size_t)blockIdx.x * (1 + nblk) * C;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float q = 0.f;
    for (int k = 0; k < nblk; ++k) q += base[(size_t)(1 + k) * C + c];
    const float gx = sqrtf(q);
    base[c] = gx;
    s += gx;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
  const float denom = tot / C + 1e-6f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) base[c] = base[c] / denom;
}

__global__ void __launch_bounds__(256)
grn_apply_kernel(const __nv_bfloat16* __restrict__ h, __nv_bfloat16* __restrict__ y,
                 const float* __restrict__ nx, long long nx_batch_stride,
                 const float* __restrict__ gamma, const float* __restrict__ beta, int N, int C,
                 long long total4) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= total4) return;
  const long long e = i4 * 4;
  const int c = (int)(e % C);
  const int b = (int)(e / ((long long)N * C));
  const uint2 u = *reinterpret_cast<const uint2*>(h + e);
  const float2 f0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
  const float2 f1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  const float4 n4 = *reinterpret_cast<const float4*>(nx + (size_t)b * nx_batch_stride + c);
  const float4 g = *reinterpret_cast<const float4*>(gamma + c);
  const float4 bt = *reinterpret_cast<const float4*>(beta + c);
  const float a0 = g.x * (f0.x * n4.x) + bt.x + f0.x;
  const float a1 = g.y * (f0.y * n4.y) + bt.y + f0.y;
  const float a2 = g.z * (f1.x * n4.z) + bt.z + f1.x;
  const float a3 = g.w * (f1.y * n4.w) + bt.w + f1.y;
  *reinterpret_cast<uint2*>(y + e) = make_uint2(pack_bf16x2(a0, a1), pack_bf16x2(a2, a3));
}

// ---------------------------------------------------------------------------------------------
// TextEmbedding front (dit.py:196-222): ids+1, truncate/pad to N with 0, text_mask = (id == 0)
// computed BEFORE the CFG drop, drop -> id 0, Embedding gather, + sinusoid table row
// min(n, 4095) (rope.py:76-84; pos_table NULL: none), masked rows -> 0.  text: int32 [B, nt] (pad -1).
// Output x: fp32 [Bout, N, C].  Utterance bo reads text row (bo % B); rows bo >= drop_from are the
// CFG "uncond" copies (ids dropped to 0, mask still from the real text).  valid_len (frame bucketing,
// may be NULL): rows n >= valid_len[bo] do not exist in the reference, whose text is truncated to the
// real N — they are written as zeros, so the first dwconv7 sees zero padding there.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
text_embed_gather_kernel(const int* __restrict__ text, int B, int nt, int N, int C,
                         const float* __restrict__ emb, const float* __restrict__ pos_table,
                         int max_pos, float* __restrict__ x, int drop_from, int mask_padding,
                         const int* __restrict__ valid_len) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.x, bo = blockIdx.y;
  const int b = bo % B;
  int id = 0;
  if (n < nt) id = text[(size_t)b * nt + n] + 1;
  const bool beyond = valid_len != nullptr && n >= valid_len[bo];
  const bool masked = beyond || (mask_padding && (id == 0));   // DurationTransformer: mask_padding=False (duration.py:118-120)
  if (bo >= drop_from) id = 0;
  const int p = n < max_pos ? n : max_pos - 1;
  const float4* er = reinterpret_cast<const float4*>(emb + (size_t)id * C);
  const float4* pr = pos_table != nullptr ? reinterpret_cast<const float4*>(pos_table + (size_t)p * C) : nullptr;
  float4* xo = reinterpret_cast<float4*>(x + ((size_t)bo * N + n) * C);
  for (int i = threadIdx.x; i < C / 4; i += blockDim.x) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!masked) {
      const float4 e = er[i];
      if (pr != nullptr) {
        const float4 q = pr[i];
        v = make_float4(e.x + q.x, e.y + q.y, e.z + q.z, e.w + q.w);
      } else {   // no position table (UNetT, conv_layers = 0): the embedding row alone
        v = e;
      }
    }
    xo[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// TimestepEmbedding (dit.py:56-82) for T time values at once, fp32 weights:
//   e = 1000 t exp(-i ln(1e4)/127), [sin e | cos e] (256) -> Linear(256->D) -> SiLU -> Linear(D->D)
// Outputs t_emb fp32 [T, D] (optional) and silu(t_emb) as bf16 [T, D], the A operand of the
// AdaLN modulation-table GEMM (dit.py:267,286 apply SiLU to t before their Linear).
// Grid (T, D/64): every block recomputes the cheap first layer (256 x D MACs) for its time value and
// then produces 64 features of the second layer; one warp per output feature, coalesced weight rows.
// ---------------------------------------------------------------------------------------------
constexpr int kTimeMlpCols = 64;
__global__ void __launch_bounds__(256)
time_mlp_kernel(const float* __restrict__ tvals, int D, const float* __restrict__ w0,
                const float* __restrict__ b0, const float* __restrict__ w2,
                const float* __restrict__ b2, float* __restrict__ t_emb,
                __nv_bfloat16* __restrict__ silu_bf16) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float sm[];
  float* h0 = sm;         // 256
  float* h1 = sm + 256;   // D
  const int ti = blockIdx.x;
  const int o0 = blockIdx.y * kTimeMlpCols;
  const float t = tvals[ti];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  if (threadIdx.x < 128) {
    const float f = expf((float)threadIdx.x * -(9.210340371976184f / 127.f));
    const float e = 1000.f * t * f;
    h0[threadIdx.x] = sinf(e);
    h0[threadIdx.x + 128] = cosf(e);
  }
  __syncthreads();
  for (int o = warp; o < D; o += nw) {
    const float* wr = w0 + (size_t)o * 256;
    float s = 0.f;
#pragma unroll
    for (int k = lane; k < 256; k += 32) s += wr[k] * h0[k];
    s = warp_sum(s);
    if (lane == 0) h1[o] = silu_f(s + b0[o]);
  }
  __syncthreads();
  for (int o = o0 + warp; o < min(D, o0 + kTimeMlpCols); o += nw) {
    const float* wr = w2 + (size_t)o * D;
    float s = 0.f;
    for (int k = lane; k < D; k += 32) s += wr[k] * h1[k];
    s = warp_sum(s);
    if (lane == 0) {
      const float v = s + b2[o];
      if (t_emb) t_emb[(size_t)ti * D + o] = v;
      silu_bf16[(size_t)ti * D + o] = __float2bfloat16(silu_f(v));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// CFG combine + explicit-solver stage update (cfm.py:364, 56, 82, 86, 117):
//   k      = pred + (pred - null) * cfg           (pred rows [0,BN), null rows [BN,2BN) of v)
//   acc    = (acc_init ? 0 : acc) + acc_w * k      (rk4: k1 + 2k2 + 2k3 + k4; optional)
//   y_out  = y_base + a * (use_acc ? acc : k)      (a = dt, dt/2, dt/6 ...)
// and refreshes the bf16 A operand of the next input-projection GEMM (both CFG halves, 128-col
// padded rows).  v: fp32 [rows_v, ldv]; y: fp32 [rows, d].
// ---------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) cfg_ode_update_kernel(const OdeUpdateParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)p.rows * p.d) return;
  const int r = (int)(i / p.d), c = (int)(i - (long long)r * p.d);
  const size_t vr = p.v_frames > 0 ? (size_t)r + r / p.v_frames + 1 : (size_t)r;
  float k = p.v[vr * p.ldv + c];
  if (p.null_row_offset > 0) {
    const float nu = p.v[(vr + p.null_row_offset) * p.ldv + c];
    k = k + (k - nu) * p.cfg_strength;
  }
  float upd = k;
  if (p.k_acc) {
    const float acc = (p.acc_init ? 0.f : p.k_acc[i]) + p.acc_w * k;
    p.k_acc[i] = acc;
    if (p.use_acc) upd = acc;
  }
  if (p.y_out) {
    const float yn = p.y_base[i] + p.a * upd;
    p.y_out[i] = yn;
    if (p.y_bf16) {
      const __nv_bfloat16 hb = __float2bfloat16(yn);
      p.y_bf16[(size_t)r * p.ld_bf16 + c] = hb;
      if (p.bf16_copy_row_offset > 0)
        p.y_bf16[(size_t)(r + p.bf16_copy_row_offset) * p.ld_bf16 + c] = hb;
    }
  }
}

// fp32 [rows, d] -> bf16 [rows, ld] (zero padded columns), optionally duplicated at a row offset
__global__ void __launch_bounds__(256)
cast_pad_bf16_kernel(const float* __restrict__ src, int d, __nv_bfloat16* __restrict__ dst, int ld,
                     int rows, long long copy_row_offset) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * ld) return;
  const int r = (int)(i / ld), c = (int)(i - (long long)r * ld);
  const __nv_bfloat16 v = c < d ? __float2bfloat16(src[(size_t)r * d + c]) : __float2bfloat16(0.f);
  dst[i] = v;
  if (copy_row_offset > 0) dst[i + copy_row_offset * ld] = v;
}

// A operand of the hoisted conditioning GEMM (dit.py:249): [cond | text_embed | 0] as bf16
// [rows, ld].  cond: fp32 [Bc, N, dc] (utterance b = (row / N) % Bc); rows >= drop_from_row get
// cond = 0 (drop_audio_cond, dit.py:248).  text: fp32 [rows, dt].
__global__ void __launch_bounds__(256)
concat_cond_text_kernel(const float* __restrict__ cond, int dc, int Bc, int N,
                        const float* __restrict__ text, int dt, __nv_bfloat16* __restrict__ dst,
                        int ld, int rows, int drop_from_row, const int* __restrict__ cond_len) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * ld) return;
  const int r = (int)(i / ld), c = (int)(i - (long long)r * ld);
  float v = 0.f;
  if (c < dc) {
    if (r < drop_from_row) {
      const int b = (r / N) % Bc, n = r % N;
      // DurationPredictor zeroes the mel beyond each utterance's length (duration.py:241-243)
      if (cond_len == nullptr || n < cond_len[b]) v = cond[((size_t)b * N + n) * dc + c];
    }
  } else if (c < dc + dt) {
    v = text[(size_t)r * dt + (c - dc)];
  }
  dst[i] = __float2bfloat16(v);
}

// ---------------------------------------------------------------------------------------------
// DurationPredictor head (duration.py:129,187-189,246-247): nn.RMSNorm(dim) (eps 1e-5, weight),
// masked mean over the frames n < len[b], Linear(dim -> 1, no bias), Softplus -> seconds.
// One block per utterance, deterministic (fixed row partition per warp, fixed-order reduction).
// ---------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(256)
duration_head_kernel(const float* __restrict__ x, int N, const int* __restrict__ len,
                     const float* __restrict__ norm_w, const float* __restrict__ pred_w,
                     float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int IT = D / 128;
  __shared__ float4 part[8][D / 4];
  __shared__ float red[8];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = min(max(len[b], 0), N);
  float4 acc[IT];
#pragma unroll
  for (int i = 0; i < IT; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int n = warp; n < L; n += 8) {
    const float4* xr = reinterpret_cast<const float4*>(x + ((size_t)b * N + n) * D);
    float4 v[IT];
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < IT; ++i) {
      v[i] = xr[i * 32 + lane];
      q += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
    }
    const float r = rsqrtf(warp_sum(q) * (1.f / D) + 1e-5f);
#pragma unroll
    for (int i = 0; i < IT; ++i) {
      acc[i].x += v[i].x * r; acc[i].y += v[i].y * r; acc[i].z += v[i].z * r; acc[i].w += v[i].w * r;
    }
  }
#pragma unroll
  for (int i = 0; i < IT; ++i) part[warp][i * 32 + lane] = acc[i];
  __syncthreads();
  float s = 0.f;
  const float inv_len = 1.f / (float)max(L, 1);
  for (int c = threadIdx.x; c < D; c += 256) {
    float m = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) m += reinterpret_cast<const float*>(part[w])[c];
    s += m * inv_len * norm_w[c] * pred_w[c];
  }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    out[b] = t > 20.f ? t : log1pf(expf(t));   // Softplus
  }
}

}  // namespace f5
