// Warp-level 512-point complex FFT (sm_90a): 16 points per lane in registers (radix-2 DIF,
// fully unrolled, compile-time twiddles) x 32 lanes via shuffle butterflies.  A 1024-point real
// FFT / inverse real FFT is one such transform plus an O(N) split step.
//
// Data distribution:  input  element n = 32*r + lane  lives in register r of `lane`
//                     output element k = r + 16*bitrev5(lane) lives in register r of `lane`
// (validated against numpy.fft in tests/test_fft_indexing.py with the same index algebra).
#pragma once
#include "ptx.cuh"

namespace f5 {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cconj(float2 a) { return make_float2(a.x, -a.y); }

// exp(-2*pi*i * num/den)
__device__ __forceinline__ float2 twiddle(int num, int den) {
  float s, c;
  sincospif(-2.f * (float)num / (float)den, &s, &c);
  return make_float2(c, s);
}

__device__ __forceinline__ int bitrev5(int l) { return (int)(__brev((unsigned)l) >> 27); }

// in-register 16-point forward FFT, natural order in and out
__device__ __forceinline__ void fft16(float2 (&a)[16]) {
  // W_16^j = exp(-2 pi i j / 16), j = 0..7
  constexpr float C[8] = {1.f, 0.9238795325112867f, 0.7071067811865476f, 0.3826834323650898f,
                          0.f, -0.3826834323650898f, -0.7071067811865476f, -0.9238795325112867f};
  constexpr float S[8] = {0.f, -0.3826834323650898f, -0.7071067811865476f, -0.9238795325112867f,
                          -1.f, -0.9238795325112867f, -0.7071067811865476f, -0.3826834323650898f};
#pragma unroll
  for (int half = 8; half >= 1; half >>= 1) {
#pragma unroll
    for (int blk = 0; blk < 16; blk += 2 * half) {
#pragma unroll
      for (int j = 0; j < half; ++j) {
        const int p = blk + j, q = p + half;
        const float2 u = a[p], v = a[q];
        a[p] = cadd(u, v);
        const float2 d = csub(u, v);
        const int tw = j * (8 / half);
        a[q] = make_float2(d.x * C[tw] - d.y * S[tw], d.x * S[tw] + d.y * C[tw]);
      }
    }
  }
  // DIF leaves bit-reversed order: swap (1,8) (2,4) (3,12) (5,10) (7,14) (11,13)
  float2 t;
  t = a[1]; a[1] = a[8]; a[8] = t;
  t = a[2]; a[2] = a[4]; a[4] = t;
  t = a[3]; a[3] = a[12]; a[12] = t;
  t = a[5]; a[5] = a[10]; a[10] = t;
  t = a[7]; a[7] = a[14]; a[14] = t;
  t = a[11]; a[11] = a[13]; a[13] = t;
}

// 512-point forward FFT across one warp (see the data distribution above)
__device__ __forceinline__ void fft512_warp(float2 (&a)[16], int lane) {
  fft16(a);
  // twiddle W_512^(lane * k1)
#pragma unroll
  for (int k1 = 1; k1 < 16; ++k1) a[k1] = cmul(a[k1], twiddle(lane * k1, 512));
  // radix-2 DIF over the lane index
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
    const bool upper = (lane & half) == 0;
    const float2 w = twiddle(lane & (half - 1), 2 * half);
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      float2 o;
      o.x = __shfl_xor_sync(0xffffffffu, a[r].x, half);
      o.y = __shfl_xor_sync(0xffffffffu, a[r].y, half);
      a[r] = upper ? cadd(a[r], o) : cmul(csub(o, a[r]), w);
    }
  }
}

}  // namespace f5
