// BigVGAN v2 generator (bigvgan_v2_24khz_100band_256x, resblock "1") for sm_90a: the anti-aliased Snake / SnakeBeta
// activation, the resblock mean, conv_post, and f5_bigvgan_decode, which composes them with the implicit-conv GEMM
// (dilated AMP-block convolutions, transposed convolutions as polyphase convolutions).  See include/f5_b200.h.
#include <string.h>

#include <cuda_bf16.h>

#include "launch.h"
#include "host_common.h"
#include "ptx.cuh"

namespace f5 {

// ---------------------------------------------------------------------------------------------
// Anti-aliased activation: one block = 64 output frames x 32 channels of one utterance.  The x rows the block needs
// (replicate-clamped to the utterance) and the activated 2x-upsampled samples (index clamped to [0, 2T), i.e. the
// replicate padding of the ACTIVATED signal) are staged in shared memory; only z reaches HBM.
// ---------------------------------------------------------------------------------------------
constexpr int kActF = 64;                  // output frames per block
constexpr int kActRowsX = kActF + 12;      // x rows n0 - 6 .. n0 + kActF + 5
constexpr int kActRowsA = 2 * kActF + 10;  // activated samples m = 2 n0 - 5 .. 2 (n0 + kActF) + 4

template <bool OUT_BF16>
__global__ void __launch_bounds__(256)
bigvgan_act_kernel(const float* __restrict__ x, int rpb, int C, const int* __restrict__ lens, f5_bigvgan_act act,
                   void* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float xs[kActRowsX][32];
  __shared__ float as[kActRowsA][32];
  const int lane = threadIdx.x, wy = threadIdx.y;
  const int n0 = blockIdx.x * kActF, b = blockIdx.z;
  const int c = blockIdx.y * 32 + lane;
  const bool cok = c < C;
  const int T = lens != nullptr ? lens[b] : rpb;
  if (n0 >= T) return;
  const size_t base = (size_t)b * rpb * C;
  for (int r = wy; r < kActRowsX; r += 8) {
    const int i = min(max(n0 - 6 + r, 0), T - 1);
    xs[r][lane] = cok ? x[base + (size_t)i * C + c] : 0.f;
  }
  float hu[12], hd[12];
#pragma unroll
  for (int j = 0; j < 12; ++j) { hu[j] = act.h_up[j]; hd[j] = act.h_down[j]; }
  const float al = cok ? act.alpha[c] : 1.f;
  const float be = act.beta != nullptr ? (cok ? act.beta[c] : 1.f) : al;
  const float inv = 1.f / (be + 1e-9f);
  __syncthreads();
  const int m_lo = 2 * n0 - 5;
  for (int idx = wy; idx < kActRowsA; idx += 8) {
    const int m = min(max(m_lo + idx, 0), 2 * T - 1);
    // u[m] = 2 sum_j h_up[j] x[clamp((m + 5 - j) / 2)] over the six j with m + 5 - j even
    const int j0 = (m + 1) & 1;
    float acc = 0.f;
#pragma unroll
    for (int jj = 0; jj < 6; ++jj) {
      const int r = (m + 5 - j0 - 2 * jj) / 2 - (n0 - 6);   // exact: m + 5 - j is even
      acc = fmaf(j0 ? hu[2 * jj + 1] : hu[2 * jj], xs[r][lane], acc);
    }
    const float u = 2.f * acc;
    const float s = sinf(al * u);
    as[idx][lane] = fmaf(inv, s * s, u);
  }
  __syncthreads();
  if (!cok) return;
  for (int nn = wy; nn < kActF; nn += 8) {
    const int n = n0 + nn;
    if (n >= T) break;
    float z = 0.f;
#pragma unroll
    for (int j = 0; j < 12; ++j) z = fmaf(hd[j], as[2 * nn + j][lane], z);
    const size_t o = base + (size_t)n * C + c;
    if constexpr (OUT_BF16) reinterpret_cast<__nv_bfloat16*>(out)[o] = __float2bfloat16_rn(z);
    else reinterpret_cast<float*>(out)[o] = z;
  }
}

// x = (x_0 + ... + x_{nk-1}) / nk, summed in j order in fp32, one IEEE division
template <bool OUT_BF16>
__global__ void __launch_bounds__(256)
bigvgan_mean_kernel(const float* __restrict__ xk, long long stride, int nk, long long n, void* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  float s = xk[i];
  for (int k = 1; k < nk; ++k) s += xk[k * stride + i];
  s = s / (float)nk;
  if constexpr (OUT_BF16) reinterpret_cast<__nv_bfloat16*>(out)[i] = __float2bfloat16_rn(s);
  else reinterpret_cast<float*>(out)[i] = s;
}

// conv_post: Conv1d(C, 1, 7, padding=3) (zero padding inside each utterance) + optional bias, then tanh or clamp
__global__ void __launch_bounds__(256)
bigvgan_conv_post_kernel(const float* __restrict__ x, int T, int C, const float* __restrict__ w,
                         const float* __restrict__ bias, int use_tanh, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
  if (n >= T) return;
  float acc = 0.f;
  for (int t = 0; t < 7; ++t) {
    const int i = n + t - 3;
    if (i < 0 || i >= T) continue;
    const float* row = x + ((size_t)b * T + i) * C;
    const float* wt = w + t * C;
    for (int c = 0; c < C; ++c) acc = fmaf(wt[c], row[c], acc);
  }
  if (bias != nullptr) acc += bias[0];
  out[(size_t)b * T + n] = use_tanh ? tanhf(acc) : fminf(fmaxf(acc, -1.f), 1.f);
}

static int launch_bigvgan_act(const float* x, int batch, int rpb, int C, const int* lens, const f5_bigvgan_act& act,
                              bool out_bf16, void* out, cudaStream_t st) {
  ProfScope ps(PROF_OTHER, 0.0, (double)batch * rpb * C * (4.0 + (out_bf16 ? 2.0 : 4.0)));
  const dim3 grid(cdiv(rpb, kActF), cdiv(C, 32), batch), block(32, 8);
  if (out_bf16) F5_CHECK_CUDA(launch_kernel(bigvgan_act_kernel<true>, grid, block, 0, st, x, rpb, C, lens, act, out));
  else F5_CHECK_CUDA(launch_kernel(bigvgan_act_kernel<false>, grid, block, 0, st, x, rpb, C, lens, act, out));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// the resblock mean of n elements over nk streams stride apart (the decode and its test entry)
static int launch_bigvgan_mean(const float* xk, long long stride, int nk, long long n, bool out_bf16, void* out,
                               cudaStream_t st) {
  if (out_bf16)
    F5_CHECK_CUDA(launch_kernel(bigvgan_mean_kernel<true>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, xk,
                                stride, nk, n, out));
  else
    F5_CHECK_CUDA(launch_kernel(bigvgan_mean_kernel<false>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, xk,
                                stride, nk, n, out));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int launch_bigvgan_conv_post(const float* x, int batch, int T, int C, const float* w, const float* bias,
                                    int use_tanh, float* out, cudaStream_t st) {
  F5_CHECK_CUDA(launch_kernel(bigvgan_conv_post_kernel, dim3(cdiv(T, 256), batch), dim3(256), 0, st, x, T, C, w, bias,
                              use_tanh, out));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static bool act_ok(const f5_bigvgan_act& a) { return a.alpha && a.h_up && a.h_down; }

}  // namespace f5

using namespace f5;

extern "C" {

int f5_bigvgan_act_forward(const float* x, int32_t batch, int32_t rows_per_batch, int32_t channels,
                           const int32_t* lens, const f5_bigvgan_act* act, int32_t out_bf16, void* out, void* stream) {
  if (int e = device_check()) return e;
  F5_REQUIRE(x && act && out && act_ok(*act), "f5_bigvgan_act_forward: null pointer");
  F5_REQUIRE(batch > 0 && rows_per_batch > 0 && channels > 0 && batch <= 65535,
             "f5_bigvgan_act_forward: bad shape batch=%d rows=%d channels=%d", batch, rows_per_batch, channels);
  return launch_bigvgan_act(x, batch, rows_per_batch, channels, lens, *act, out_bf16 != 0, out, (cudaStream_t)stream);
}

int f5_bigvgan_decode(const f5_bigvgan_weights* w, const f5_bigvgan_buffers* b, const float* mel, float* wave,
                      void* stream) {
  if (int e = device_check()) return e;
  F5_REQUIRE(w && b && mel && wave && w->blocks, "f5_bigvgan_decode: null pointer");
  F5_REQUIRE(b->mel_bf16 && b->a_bf16 && b->x_up && b->t && b->xk, "f5_bigvgan_decode: null buffer");
  cudaStream_t st = (cudaStream_t)stream;
  const int B = b->batch, N = b->frames, NU = w->num_upsamples, NK = w->num_kernels;
  F5_REQUIRE(B > 0 && N > 0 && B <= 65535, "f5_bigvgan_decode: bad shape batch=%d frames=%d", B, N);
  F5_REQUIRE(w->num_mels > 0 && w->num_mels <= 128, "f5_bigvgan_decode: num_mels=%d not in [1, 128]", w->num_mels);
  F5_REQUIRE(NU >= 1 && NU <= F5_BIGVGAN_MAX_UPS && NK >= 1 && NK <= F5_BIGVGAN_MAX_KERNELS,
             "f5_bigvgan_decode: num_upsamples=%d num_kernels=%d", NU, NK);
  // shapes of every stage, checked before anything is launched
  {
    int64_t T = N, C = w->channels0, need = (int64_t)N * C;
    F5_REQUIRE(C % 8 == 0, "f5_bigvgan_decode: channels0=%d not a multiple of 8", w->channels0);
    for (int i = 0; i < NU; ++i) {
      F5_REQUIRE(w->up_rate[i] >= 1 && w->up_taps[i] >= 1 && w->up_pad[i] >= 0 && C % 16 == 0,
                 "f5_bigvgan_decode: stage %d: rate %d, taps %d, pad %d, %lld input channels", i, w->up_rate[i],
                 w->up_taps[i], w->up_pad[i], (long long)C);
      F5_REQUIRE(w->up_w[i] && w->up_b[i], "f5_bigvgan_decode: stage %d: null weights", i);
      T *= w->up_rate[i];
      C /= 2;
      need = need > T * C ? need : T * C;
      for (int j = 0; j < NK; ++j) {
        const f5_bigvgan_amp_weights& blk = w->blocks[i * NK + j];
        F5_REQUIRE(blk.kernel >= 1 && blk.kernel % 2 == 1, "f5_bigvgan_decode: resblock %d: kernel %d", i * NK + j,
                   blk.kernel);
        for (int m = 0; m < 3; ++m)
          F5_REQUIRE(blk.dilation[m] >= 1 && blk.conv1_w[m] && blk.conv1_b[m] && blk.conv2_w[m] && blk.conv2_b[m] &&
                         act_ok(blk.act[2 * m]) && act_ok(blk.act[2 * m + 1]),
                     "f5_bigvgan_decode: resblock %d: conv %d", i * NK + j, m);
      }
    }
    F5_REQUIRE(T * B <= INT32_MAX, "f5_bigvgan_decode: %lld output samples", (long long)(T * B));
    F5_REQUIRE(need <= b->stage_elems, "f5_bigvgan_decode: stage_elems %lld < %lld", (long long)b->stage_elems,
               (long long)need);
    F5_REQUIRE(act_ok(w->act_post) && w->conv_post_w && w->conv_pre_w && w->conv_pre_b,
               "f5_bigvgan_decode: null weights");
  }
  auto conv = [&](const void* a, int T, int Cin, const void* wt, int taps, int pad, int dil, const float* bias, int n,
                  void* out, bool out_bf16, const float* resid) -> int {
    f5_gemm_args g;
    memset(&g, 0, sizeof(g));
    g.a = a; g.lda = Cin; g.w = wt; g.ldw = (int64_t)taps * (cdiv(Cin, 64) * 64);
    g.m = B * T; g.n = n; g.k = Cin;
    g.rows_per_batch = T; g.num_batches = B; g.batched_tiles = 1;
    g.conv_taps = taps; g.conv_pad = pad; g.conv_dilation = dil;
    g.bias = bias; g.out = out; g.ldo = n; g.out_bf16 = out_bf16 ? 1 : 0; g.q_scale = 1.f;
    g.resid = resid; g.ldr = resid ? n : 0;
    g.w_static = 1;
    return f5_gemm_bf16(&g, st);
  };
  // conv_pre over the mel padded to 128 channels: bf16 out (the first ups GEMM's operand)
  if (int e = launch_cast_pad_bf16(mel, w->num_mels, b->mel_bf16, 128, B * N, 0, st)) return e;
  {
    f5_gemm_args g;
    memset(&g, 0, sizeof(g));
    g.a = b->mel_bf16; g.lda = 128; g.w = w->conv_pre_w; g.ldw = 7 * 128;
    g.m = B * N; g.n = w->channels0; g.k = 128;
    g.rows_per_batch = N; g.num_batches = B; g.batched_tiles = 1;
    g.conv_taps = 7; g.conv_pad = 3;
    g.bias = w->conv_pre_b; g.out = b->a_bf16; g.ldo = w->channels0; g.out_bf16 = 1; g.q_scale = 1.f;
    g.w_static = 1;
    if (int e = f5_gemm_bf16(&g, st)) return e;
  }
  const long long stride = (long long)B * b->stage_elems;
  int T = N, C = w->channels0;
  for (int i = 0; i < NU; ++i) {
    const int u = w->up_rate[i], Co = C / 2;
    if (int e = conv(b->a_bf16, T, C, w->up_w[i], w->up_taps[i], w->up_pad[i], 1, w->up_b[i], u * Co, b->x_up, false,
                     nullptr))
      return e;
    T *= u;
    C = Co;
    for (int j = 0; j < NK; ++j) {
      const f5_bigvgan_amp_weights& blk = w->blocks[i * NK + j];
      float* xj = b->xk + j * stride;
      const float* xin = b->x_up;
      const int k = blk.kernel;
      for (int m = 0; m < 3; ++m) {
        const int d = blk.dilation[m];
        if (int e = launch_bigvgan_act(xin, B, T, C, nullptr, blk.act[2 * m], true, b->a_bf16, st)) return e;
        if (int e = conv(b->a_bf16, T, C, blk.conv1_w[m], k, (k * d - d) / 2, d, blk.conv1_b[m], C, b->t, false,
                         nullptr))
          return e;
        if (int e = launch_bigvgan_act(b->t, B, T, C, nullptr, blk.act[2 * m + 1], true, b->a_bf16, st)) return e;
        if (int e = conv(b->a_bf16, T, C, blk.conv2_w[m], k, (k - 1) / 2, 1, blk.conv2_b[m], C, xj, false, xin))
          return e;
        xin = xj;
      }
    }
    const long long n = (long long)B * T * C;
    ProfScope ps(PROF_OTHER, 0.0, 4.0 * NK * n + (i + 1 < NU ? 2.0 : 4.0) * n);
    const bool last = i + 1 == NU;
    if (int e = launch_bigvgan_mean(b->xk, stride, NK, n, !last, last ? (void*)b->t : b->a_bf16, st)) return e;
  }
  if (int e = launch_bigvgan_act(b->t, B, T, C, nullptr, w->act_post, false, b->x_up, st)) return e;
  {
    ProfScope ps(PROF_OTHER, 14.0 * B * (double)T * C, 4.0 * B * (double)T * (C + 1));
    if (int e = launch_bigvgan_conv_post(b->x_up, B, T, C, w->conv_post_w, w->conv_post_b, w->use_tanh_at_final, wave,
                                         st))
      return e;
  }
  return 0;
}

int f5_bigvgan_resblock_mean(const float* xk, int64_t stride, int32_t nk, int64_t n, int32_t out_bf16, void* out,
                             void* stream) {
  if (int e = device_check()) return e;
  F5_REQUIRE(xk && out, "f5_bigvgan_resblock_mean: null pointer");
  F5_REQUIRE(nk >= 1 && n > 0 && (nk == 1 || stride >= n) && (n + 255) / 256 <= INT32_MAX,
             "f5_bigvgan_resblock_mean: bad shape nk=%d n=%lld stride=%lld", nk, (long long)n, (long long)stride);
  return launch_bigvgan_mean(xk, stride, nk, n, out_bf16 != 0, out, (cudaStream_t)stream);
}

int f5_bigvgan_conv_post(const float* x, int32_t batch, int32_t frames, int32_t channels, const float* w,
                         const float* bias, int32_t use_tanh, float* out, void* stream) {
  if (int e = device_check()) return e;
  F5_REQUIRE(x && w && out, "f5_bigvgan_conv_post: null pointer");
  F5_REQUIRE(batch > 0 && frames > 0 && channels > 0 && batch <= 65535,
             "f5_bigvgan_conv_post: bad shape batch=%d frames=%d channels=%d", batch, frames, channels);
  return launch_bigvgan_conv_post(x, batch, frames, channels, w, bias, use_tanh, out, (cudaStream_t)stream);
}

}  // extern "C"
