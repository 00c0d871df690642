// Log-mel front-end (audio.py:115-210) and the Vocos back-end (vocos_mlx.Vocos.decode, call site
// cfm.py:399-400) for sm_90a.  FFTs are warp-level (fft.cuh): one warp = one frame.
#include <string.h>

#include "fft.cuh"
#include "launch.h"
#include "host_common.h"

namespace f5 {

// ---------------------------------------------------------------------------------------------
// K1  mel front-end: frame f = samples [f*hop - 512, f*hop + 512) of the zero-padded signal
// (audio.py:143-158), * periodic Hann, 1024-pt real FFT, |.|, @ filters^T, log(max(., 1e-5)).
// filt_t: fp32 [513, n_mels] (transposed filterbank -> coalesced across mel bins).
// ---------------------------------------------------------------------------------------------
constexpr int kMelWarps = 4;

__global__ void __launch_bounds__(kMelWarps * 32)
mel_kernel(const float* __restrict__ audio, int T, const float* __restrict__ window,
           const float* __restrict__ filt_t, int n_mels, int hop, float* __restrict__ out,
           int frames) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float2 Zs[kMelWarps][512];
  __shared__ float mags[kMelWarps][516];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * kMelWarps + warp;
  const int b = blockIdx.y;
  if (f >= frames) return;
  const float* x = audio + (size_t)b * T;
  const long long s0 = (long long)f * hop - 512;

  // z[n] = x[2n] + i x[2n+1], n = 32 r + lane
  float2 a[16];
#pragma unroll
  for (int r = 0; r < 16; ++r) {
    const int n = 32 * r + lane;
    const long long i0 = s0 + 2 * n;
    const float x0 = (i0 >= 0 && i0 < T) ? x[i0] : 0.f;
    const float x1 = (i0 + 1 >= 0 && i0 + 1 < T) ? x[i0 + 1] : 0.f;
    const float2 w = reinterpret_cast<const float2*>(window)[n];
    a[r] = make_float2(x0 * w.x, x1 * w.y);
  }
  fft512_warp(a, lane);
  const int kbase = 16 * bitrev5(lane);
#pragma unroll
  for (int r = 0; r < 16; ++r) Zs[warp][r + kbase] = a[r];
  __syncwarp();
  // split: X[k] = (Z[k] + conj Z[512-k])/2 - i W_1024^k (Z[k] - conj Z[512-k])/2, k = 0..512
  for (int k = lane; k <= 512; k += 32) {
    const float2 zk = Zs[warp][k & 511];
    const float2 zc = cconj(Zs[warp][(512 - k) & 511]);
    const float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
    const float2 d = make_float2(0.5f * (zk.x - zc.x), 0.5f * (zk.y - zc.y));
    const float2 wd = cmul(twiddle(k, 1024), d);          // W^k * d
    const float re = e.x + wd.y, im = e.y - wd.x;         // e - i * wd
    mags[warp][k] = sqrtf(re * re + im * im);
  }
  __syncwarp();
  for (int m = lane; m < n_mels; m += 32) {
    float acc = 0.f;
    for (int k = 0; k <= 512; ++k) acc = fmaf(mags[warp][k], filt_t[(size_t)k * n_mels + m], acc);
    out[((size_t)b * frames + f) * n_mels + m] = logf(fmaxf(acc, 1e-5f));
  }
}

// ---------------------------------------------------------------------------------------------
// K10a  ISTFT head, per frame: h = [log-mag(513) | phase(513)] -> S = min(exp(.),1e2) e^{i phase}
// -> irfft(1024) (imaginary parts of DC / Nyquist ignored, as pocketfft c2r) -> * window.
// frames_out: fp32 [rows, 1024].
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 vocos_bin(const float* __restrict__ hrow, int k) {
  const float mg = fminf(expf(hrow[k]), 100.f);
  float s, c;
  sincosf(hrow[513 + k], &s, &c);
  float2 v = make_float2(mg * c, mg * s);
  if (k == 0 || k == 512) v.y = 0.f;
  return v;
}

__global__ void __launch_bounds__(kMelWarps * 32)
istft_frames_kernel(const float* __restrict__ h, int ldh, const float* __restrict__ window,
                    float* __restrict__ frames_out, int rows) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float2 Zs[kMelWarps][512];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * kMelWarps + warp;
  if (f >= rows) return;
  const float* hrow = h + (size_t)f * ldh;
  float2 a[16];
#pragma unroll
  for (int r = 0; r < 16; ++r) {
    const int k = 32 * r + lane;                     // 0..511
    const float2 xk = vocos_bin(hrow, k);
    const float2 xc = cconj(vocos_bin(hrow, 512 - k));
    const float2 e = make_float2(0.5f * (xk.x + xc.x), 0.5f * (xk.y + xc.y));
    const float2 d = make_float2(0.5f * (xk.x - xc.x), 0.5f * (xk.y - xc.y));
    const float2 o = cmul(d, cconj(twiddle(k, 1024)));   // * exp(+2 pi i k / 1024)
    // Z = E + i O ; feed conj(Z) to the forward FFT
    a[r] = make_float2(e.x - o.y, -(e.y + o.x));
  }
  fft512_warp(a, lane);
  const int nbase = 16 * bitrev5(lane);
#pragma unroll
  for (int r = 0; r < 16; ++r) {
    const int n = r + nbase;
    const float2 w = reinterpret_cast<const float2*>(window)[n];
    // z = conj(result) / 512 ; x[2n] = Re z, x[2n+1] = Im z
    Zs[warp][n] = make_float2(a[r].x * (1.f / 512.f) * w.x, -a[r].y * (1.f / 512.f) * w.y);
  }
  __syncwarp();
  float2* fo = reinterpret_cast<float2*>(frames_out + (size_t)f * 1024);
  for (int i = lane; i < 512; i += 32) fo[i] = Zs[warp][i];
}

// K10b  overlap-add + envelope normalisation (gather form: <= 4 frames per output sample).
// norm_sq: 0 -> divide by sum of window (vocos-mlx per-frame OLA), 1 -> by sum of window^2.
__global__ void __launch_bounds__(256)
istft_ola_kernel(const float* __restrict__ frames, const float* __restrict__ window, int n_frames,
                 int hop, int norm_sq, int trim, float* __restrict__ out, int out_len) {
  pdl_launch_dependents();
  pdl_wait();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (j >= out_len) return;
  const int t = j + trim;
  int f_hi = t / hop;
  if (f_hi > n_frames - 1) f_hi = n_frames - 1;
  int f_lo = (t - 1023 + hop - 1) / hop;
  if (t - 1023 <= 0) f_lo = 0;
  const float* fr = frames + (size_t)b * n_frames * 1024;
  float acc = 0.f, env = 0.f;
  for (int f = f_lo; f <= f_hi; ++f) {
    const int i = t - f * hop;
    acc += fr[(size_t)f * 1024 + i];
    const float w = window[i];
    env += norm_sq ? w * w : w;
  }
  out[(size_t)b * out_len + j] = env > 1e-11f ? acc / env : acc;
}

}  // namespace f5

using namespace f5;

extern "C" {

int f5_mel_forward(const float* audio, int32_t batch, int32_t samples, const float* window,
                   const float* filters, int32_t n_mels, int32_t hop, float* out, int32_t frames,
                   void* stream) {
  if (int e = device_check()) return e;
  F5_REQUIRE(audio && window && filters && out, "f5_mel_forward: null pointer");
  F5_REQUIRE(batch > 0 && samples > 0 && frames > 0 && n_mels > 0, "f5_mel_forward: bad shape");
  F5_REQUIRE(frames <= samples / hop, "f5_mel_forward: frames %d > samples/hop %d", frames,
             samples / hop);
  ProfScope ps(PROF_OTHER, 0.0, 4.0 * batch * (double)samples + 4.0 * batch * (double)frames * n_mels,
               (cudaStream_t)stream);
  F5_CHECK_CUDA(launch_kernel(mel_kernel, dim3(dim3(cdiv(frames, kMelWarps), batch)), dim3(kMelWarps * 32), 0, (cudaStream_t)stream, 
      audio, samples, window, filters, n_mels, hop, out, frames));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int f5_istft(const float* h, int64_t ldh, int32_t batch, int32_t frames, const float* window,
             int32_t hop, int32_t norm_sq, int32_t trim, float* frames_scratch, float* out,
             int32_t out_len, void* stream) {
  if (int e = device_check()) return e;
  F5_REQUIRE(h && window && frames_scratch && out, "f5_istft: null pointer");
  F5_REQUIRE(ldh >= 1026, "f5_istft: ldh %lld < 1026", (long long)ldh);
  const int rows = batch * frames;
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps(PROF_OTHER, 0.0, 0.0, st);
  F5_CHECK_CUDA(launch_kernel(istft_frames_kernel, dim3(cdiv(rows, kMelWarps)), dim3(kMelWarps * 32), 0, st, h, (int)ldh, window,
                                                                       frames_scratch, rows));
  F5_CHECK_CUDA(launch_kernel(istft_ola_kernel, dim3(dim3(cdiv(out_len, 256), batch)), dim3(256), 0, st, frames_scratch, window, frames,
                                                                   hop, norm_sq, trim, out, out_len));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// Vocos.decode: mel fp32 [batch, frames, 100] -> waveform fp32 [batch, out_len]
int f5_vocos_decode(const f5_vocos_weights* w, const f5_vocos_buffers* b, const float* mel,
                    float* wave, void* stream) {
  if (int e = device_check()) return e;
  F5_REQUIRE(w && b && mel && wave, "f5_vocos_decode: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int B = b->batch, N = b->frames, R = B * N, D = w->dim, Ci = w->inner;
  F5_REQUIRE(w->n_mels <= 128 && D % 128 == 0, "f5_vocos_decode: unsupported dims");
  // embed: Conv1d(n_mels -> D, k=7, pad 3) as an implicit GEMM over the 128-padded mel rows
  if (int e = launch_cast_pad_bf16(mel, w->n_mels, b->mel_bf16, 128, R, 0, st)) return e;
  {
    f5_gemm_args g;
    memset(&g, 0, sizeof(g));
    g.a = b->mel_bf16; g.lda = 128; g.w = w->embed_w; g.ldw = 7 * 128;
    g.m = R; g.n = D; g.k = 128;
    g.rows_per_batch = N; g.num_batches = B; g.batched_tiles = 1;
    g.conv_taps = 7; g.conv_pad = 3;
    g.bias = w->embed_b; g.out = b->h; g.ldo = D; g.q_scale = 1.f;
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  if (int e = launch_ln_f32(b->h, b->x, R, D, w->norm_w, w->norm_b, st)) return e;
  for (int l = 0; l < w->num_layers; ++l) {
    const f5_vocos_block_weights& bw = w->blocks[l];
    if (int e = launch_dwconv7_ln(b->x, b->a_bf16, B, N, D, bw.dw_w, bw.dw_b, bw.ln_w, bw.ln_b, st))
      return e;
    {
      f5_gemm_args g;
      memset(&g, 0, sizeof(g));
      g.a = b->a_bf16; g.lda = D; g.w = bw.pw1_w; g.ldw = D; g.m = R; g.n = Ci; g.k = D;
      g.num_batches = 1; g.conv_taps = 1; g.act = F5_ACT_GELU_ERF; g.out_bf16 = 1;
      g.bias = bw.pw1_b; g.out = b->i_bf16; g.ldo = Ci; g.q_scale = 1.f;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
    {
      f5_gemm_args g;
      memset(&g, 0, sizeof(g));
      g.a = b->i_bf16; g.lda = Ci; g.w = bw.pw2_w; g.ldw = Ci; g.m = R; g.n = D; g.k = Ci;
      g.num_batches = 1; g.conv_taps = 1;
      g.bias = bw.pw2_b; g.out = b->x; g.ldo = D; g.q_scale = 1.f;
      g.gate = bw.gamma; g.gate_ld = 0;           // layer scale: per-channel gamma
      g.resid = b->x; g.ldr = D;
      if (int e = f5_gemm_bf16(&g, st)) return e;
    }
  }
  if (int e = launch_ln_modulate(b->x, b->a_bf16, R, D, 0, w->final_w, w->final_b, 0, 0, st)) return e;
  {
    f5_gemm_args g;
    memset(&g, 0, sizeof(g));
    g.a = b->a_bf16; g.lda = D; g.w = w->head_w; g.ldw = D; g.m = R; g.n = w->head_ld; g.k = D;
    g.num_batches = 1; g.conv_taps = 1;
    g.bias = w->head_b; g.out = b->head; g.ldo = w->head_ld; g.q_scale = 1.f;
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  return f5_istft(b->head, w->head_ld, B, N, w->window, w->hop, w->istft_norm_sq, w->istft_trim,
                  b->frames_f32, wave, b->out_len, st);
}

}  // extern "C"
