// Windowed-sinc sample-rate conversion for sm_90a: the definition of torchaudio.functional.resample at its defaults
// (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99), which is what upstream F5-TTS applies to reference clips
// that are not 24 kHz.  The polyphase table is host math (f5_resample_table, double, rounded once to fp32); the kernel
// is a gather: y[j] = sum_k h[j % N][k] * x[(j / N) * O + k - w], accumulated in fp32 in ascending k by one thread, so
// every output is bitwise reproducible and independent of the tiling and of the other rows.
#include <math.h>
#include <stdint.h>

#include "host_common.h"
#include "ptx.cuh"

namespace f5 {

constexpr int kResThreads = 256;
constexpr int64_t kResMaxTable = 1 << 16;      // N * taps entries (256 KB of fp32): every pair of common rates fits
// Tables up to this size are staged in shared memory next to the input window; larger ones (22.05 / 11.025 kHz
// pairs) are read through the read-only data cache, where a per-CTA copy would cost more L2 traffic than it saves.
constexpr int64_t kResSmemTable = 16 * 1024;   // entries (64 KB)
constexpr int kSm90SmemOptin = 227 * 1024;     // dynamic shared memory one CTA may opt in to on sm_90

struct ResampleGeom {
  int64_t O, N, w, taps;
  double base;
};

static int64_t gcd64(int64_t a, int64_t b) {
  while (b) { const int64_t t = a % b; a = b; b = t; }
  return a;
}

static ResampleGeom resample_geom(int32_t orig, int32_t new_freq) {
  ResampleGeom g;
  const int64_t d = gcd64(orig, new_freq);
  g.O = orig / d;
  g.N = new_freq / d;
  g.base = (double)(g.O < g.N ? g.O : g.N) * 0.99;
  g.w = (int64_t)ceil(6.0 * (double)g.O / g.base);
  g.taps = 2 * g.w + g.O;
  return g;
}

// Output tile of TJ samples of one row: it reads the input window [(j0 / N) * O - w, (j_last / N) * O - w + taps).
// The window is staged in shared memory with float4 loads aligned to the ROW-INDEPENDENT address of x (x_align_off =
// x's misalignment in floats), so `lead` = the window start's offset inside its first float4.
template <bool TABLE_SMEM>
__global__ void __launch_bounds__(kResThreads)
resample_kernel(const float* __restrict__ x, int64_t samples, const float* __restrict__ table, int64_t O, int64_t N,
                int64_t w, int32_t taps, float* __restrict__ out, int64_t out_samples, int32_t tile, int32_t x_align_off) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) float res_smem[];
  const int64_t row = blockIdx.y;
  const int64_t j0 = (int64_t)blockIdx.x * tile;
  const int64_t j_end = min(j0 + (int64_t)tile, out_samples);
  const int64_t q0 = j0 / N;
  const int64_t win = ((j_end - 1) / N - q0) * O + taps;
  const int64_t ntab = N * taps;

  float* tab_s = res_smem;
  float* win_s = res_smem + (TABLE_SMEM ? ((ntab + 3) & ~int64_t(3)) : 0);
  if (TABLE_SMEM) {
    for (int64_t i = threadIdx.x; i < ntab; i += kResThreads) tab_s[i] = __ldg(table + i);
  }

  // flat float index (from the aligned base of x) of the row's first sample and of the window's first sample
  const float* xa = x - x_align_off;
  const int64_t row0 = x_align_off + row * samples;
  const int64_t a = row0 + q0 * O - w;
  const int64_t c0 = a >> 2;                                 // floor, also for a < 0
  const int64_t c1 = (a + win - 1) >> 2;
  const int lead = (int)(a - 4 * c0);
  for (int64_t c = c0 + threadIdx.x; c <= c1; c += kResThreads) {
    const int64_t e0 = 4 * c;
    float4 v;
    if (e0 >= row0 && e0 + 4 <= row0 + samples) {
      v = __ldg(reinterpret_cast<const float4*>(xa) + c);
    } else {                                                 // straddles a row edge: per element, zero outside
      auto ld = [&](int64_t i) { return (i >= row0 && i < row0 + samples) ? __ldg(xa + i) : 0.f; };
      v = make_float4(ld(e0), ld(e0 + 1), ld(e0 + 2), ld(e0 + 3));
    }
    reinterpret_cast<float4*>(win_s)[c - c0] = v;
  }
  __syncthreads();

  const float* tab = TABLE_SMEM ? tab_s : table;
  float* orow = out + row * out_samples;
  for (int64_t j = j0 + threadIdx.x; j < j_end; j += kResThreads) {
    const int64_t q = j / N;
    const int64_t p = j - q * N;
    const float* h = tab + p * taps;
    const float* xs = win_s + lead + (q - q0) * O;
    float acc = 0.f;
    if (TABLE_SMEM) {
#pragma unroll 4
      for (int k = 0; k < taps; ++k) acc = fmaf(h[k], xs[k], acc);
    } else {
#pragma unroll 4
      for (int k = 0; k < taps; ++k) acc = fmaf(__ldg(h + k), xs[k], acc);
    }
    orow[j] = acc;
  }
}

}  // namespace f5

using namespace f5;

extern "C" {

int f5_resample_table(int32_t orig_freq, int32_t new_freq, float* h_table, int64_t cap) {
  F5_REQUIRE(orig_freq > 0 && new_freq > 0, "f5_resample_table: rates must be positive (%d -> %d)", orig_freq,
             new_freq);
  if (orig_freq == new_freq) return 0;                       // the identity has no filter
  const ResampleGeom g = resample_geom(orig_freq, new_freq);
  const int64_t n = g.N * g.taps;
  F5_REQUIRE(n <= kResMaxTable, "f5_resample_table: %d -> %d Hz needs a %lld x %lld table (> %lld entries)",
             orig_freq, new_freq, (long long)g.N, (long long)g.taps, (long long)kResMaxTable);
  if (h_table == nullptr || cap < n) return (int)n;
  const double pi = 3.14159265358979323846;
  for (int64_t p = 0; p < g.N; ++p) {
    for (int64_t k = 0; k < g.taps; ++k) {
      double t = ((double)(k - g.w) / (double)g.O - (double)p / (double)g.N) * g.base;
      t = t < -6.0 ? -6.0 : (t > 6.0 ? 6.0 : t);
      const double c = cos(pi * t / 12.0);
      const double s = t == 0.0 ? 1.0 : sin(pi * t) / (pi * t);
      h_table[p * g.taps + k] = (float)(s * c * c * g.base / (double)g.O);
    }
  }
  return (int)n;
}

int f5_resample(const float* x, int32_t batch, int64_t samples, int32_t orig_freq, int32_t new_freq,
                const float* table, float* out, int64_t out_samples, void* stream) {
  if (int e = device_check()) return e;
  F5_REQUIRE(orig_freq > 0 && new_freq > 0, "f5_resample: rates must be positive (%d -> %d)", orig_freq, new_freq);
  F5_REQUIRE(x && out, "f5_resample: null pointer");
  F5_REQUIRE(batch > 0 && batch <= 65535 && samples > 0, "f5_resample: bad shape (batch %d, samples %lld)", batch,
             (long long)samples);
  F5_REQUIRE(((uintptr_t)x & 3) == 0 && ((uintptr_t)out & 3) == 0, "f5_resample: x / out not 4-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (orig_freq == new_freq) {
    F5_REQUIRE(out_samples == samples, "f5_resample: out_samples %lld != samples %lld for equal rates",
               (long long)out_samples, (long long)samples);
    if (out != x) F5_CHECK_CUDA(cudaMemcpyAsync(out, x, (size_t)batch * samples * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  F5_REQUIRE(table, "f5_resample: null table");
  const ResampleGeom g = resample_geom(orig_freq, new_freq);
  const int64_t ntab = g.N * g.taps;
  F5_REQUIRE(ntab <= kResMaxTable, "f5_resample: %d -> %d Hz table of %lld entries exceeds %lld", orig_freq, new_freq,
             (long long)ntab, (long long)kResMaxTable);
  F5_REQUIRE(samples <= INT64_MAX / g.N, "f5_resample: samples %lld too large", (long long)samples);
  const int64_t want = (g.N * samples + g.O - 1) / g.O;
  F5_REQUIRE(out_samples == want, "f5_resample: out_samples %lld != ceil(%lld * %lld / %lld) = %lld",
             (long long)out_samples, (long long)g.N, (long long)samples, (long long)g.O, (long long)want);

  // outputs per CTA: 1024, fewer when a large decimation ratio makes the input window outgrow shared memory
  const int smem_optin = kSm90SmemOptin;
  const bool table_smem = ntab <= kResSmemTable;
  const int64_t tab_floats = table_smem ? ((ntab + 3) & ~int64_t(3)) : 0;
  int tile = 4 * kResThreads;
  auto smem_bytes = [&](int t) {
    const int64_t win = ((int64_t)(t - 1) / g.N + 1) * g.O + g.taps;   // widest window of a tile of t outputs
    return (tab_floats + 4 * ((win + 3) / 4 + 1)) * 4;                 // + one float4 for the misaligned start
  };
  while (tile > kResThreads && smem_bytes(tile) > smem_optin) tile /= 2;
  F5_REQUIRE(smem_bytes(tile) <= smem_optin,
             "f5_resample: %d -> %d Hz: the input window of %d outputs needs %lld bytes of shared memory (> %d)",
             orig_freq, new_freq, tile, (long long)smem_bytes(tile), smem_optin);
  const int64_t tiles = (out_samples + tile - 1) / tile;
  F5_REQUIRE(tiles <= INT32_MAX, "f5_resample: %lld output tiles", (long long)tiles);
  const int smem = (int)smem_bytes(tile);
  const int x_align_off = (int)(((uintptr_t)x & 15) / 4);

  ProfScope ps(PROF_OTHER, 2.0 * batch * (double)out_samples * g.taps,
               4.0 * batch * ((double)samples + (double)out_samples) + 4.0 * ntab);
  static SmemAttrOnce once_smem, once_ldg;
  if (table_smem) {
    F5_CHECK_CUDA(ensure_dyn_smem(once_smem, resample_kernel<true>, smem_optin));
    F5_CHECK_CUDA(launch_kernel(resample_kernel<true>, dim3((unsigned)tiles, batch), dim3(kResThreads), smem, st, x,
                                samples, table, g.O, g.N, g.w, (int)g.taps, out, out_samples, tile, x_align_off));
  } else {
    F5_CHECK_CUDA(ensure_dyn_smem(once_ldg, resample_kernel<false>, smem_optin));
    F5_CHECK_CUDA(launch_kernel(resample_kernel<false>, dim3((unsigned)tiles, batch), dim3(kResThreads), smem, st, x,
                                samples, table, g.O, g.N, g.w, (int)g.taps, out, out_samples, tile, x_align_off));
  }
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
