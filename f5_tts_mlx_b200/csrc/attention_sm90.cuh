// Flash-attention forward for sm_90a (head_dim 64, non-causal, key-padding mask) on wgmma.
// Replaces mx.fast.scaled_dot_product_attention + the head split / merge (dit.py:141-143,161-167); the softmax scale
// is already folded into q by the QKV GEMM's epilogue.
//
//   warpgroup 0    TMA producer (one elected thread): the CTA's 128-query Q tile once, K/V 128-key tiles in
//                  2-stage rings
//   warpgroups 1-2 consumers, 64 query rows each (thread = 2 rows x 32 key columns of the accumulator fragment):
//                  S = Q K^T    wgmma m64n128k16, Q and K from shared memory (K-major)
//                  online softmax in registers (row max / sum over the 4 threads of a row: two shuffles)
//                  O += P V     wgmma m64n64k16, P from registers (the S fragment is the A fragment), V from shared
//                               memory as an MN-major B operand
#pragma once
#include "ptx.cuh"

namespace f5 {

struct AttnParams {
  int B, N, H;
  const int* kv_len;       // [B] valid keys per utterance, or null (= N)
  __nv_bfloat16* out;      // [B*N, H*64]
  int ldo;
  unsigned long long* prof;  // in-graph timing slot (ptx.cuh prof_stamp_*), or null
  int out_fp8;             // `out` receives e4m3 bytes (ldo in bytes) — the A operand of an FP8-mode out-projection
};

struct AttnSmem {
  static constexpr int kQ = 0;                        // 128 x 64 bf16
  static constexpr int kK = 16384;                    // 2 stages x (128 x 64 bf16)
  static constexpr int kV = kK + 2 * 16384;           // 2 stages
  static constexpr int kBar = kV + 2 * 16384;
  // q_full, k_full[2], k_empty[2], v_full[2], v_empty[2]
  static constexpr int kNumBars = 9;
  static constexpr int kTotal = kBar + kNumBars * 8 + 1024;   // + align slack
};

template <bool kOut8>     // e4m3 output (FP8 mode), its own instantiation
__global__ void __launch_bounds__(384, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tma_qkv, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // SWIZZLE_128B tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AttnSmem::kBar);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;    // [2]
  uint64_t* k_empty = bars + 3;   // [2]
  uint64_t* v_full = bars + 5;    // [2]
  uint64_t* v_empty = bars + 7;   // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 128;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int HD = p.H * 64;
  int kv_len = p.kv_len ? p.kv_len[b] : p.N;
  kv_len = min(max(kv_len, 1), p.N);
  const int num_kv = (kv_len + 127) >> 7;

  if (warp == 0 && F5_ELECT_LANE()) {
    tma_prefetch_desc(&tma_qkv);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 256);   // released by every consumer thread
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 256);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (threadIdx.x == 128) prof_stamp_begin(p.prof);   // a consumer thread, not the producer

  if (warp < 4) {
    // ===================== TMA producer =====================
    if (warp == 0 && F5_ELECT_LANE()) {
      mbar_expect_tx(q_full, 16384);
      tma_load_3d(smem + AttnSmem::kQ, &tma_qkv, q_full, h * 64, q0, b);
      for (int j = 0; j < num_kv; ++j) {
        const int s = j & 1;
        const uint32_t ph = (j >> 1) & 1;
        mbar_wait(&k_empty[s], ph ^ 1);
        mbar_expect_tx(&k_full[s], 16384);
        tma_load_3d(smem + AttnSmem::kK + s * 16384, &tma_qkv, &k_full[s], HD + h * 64, j * 128, b);
        mbar_wait(&v_empty[s], ph ^ 1);
        mbar_expect_tx(&v_full[s], 16384);
        tma_load_3d(smem + AttnSmem::kV + s * 16384, &tma_qkv, &v_full[s], 2 * HD + h * 64, j * 128, b);
      }
    }
  } else {
    // ===================== consumers =====================
    const int wg = (threadIdx.x >> 7) - 1;                       // query rows [64 wg, 64 wg + 64) of the tile
    const int rw = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);  // this thread's rows: rw and rw + 8 of the 64
    const uint32_t sQ = smem_u32(smem + AttnSmem::kQ) + wg * (64 * 128);
    constexpr float kLog2e = 1.4426950408889634f;
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    mbar_wait(q_full, 0);

    for (int j = 0; j < num_kv; ++j) {
      const int s = j & 1;
      const uint32_t ph = (j >> 1) & 1;
      // ---- S = Q K^T (64 x 128) ----
      float sv[64];
      mbar_wait(&k_full[s], ph);
      const uint32_t sK = smem_u32(smem + AttnSmem::kK + s * 16384);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_bf16_ss_n128(sv, gmma_desc_sw128(sQ + 32 * k, 16, 1024), gmma_desc_sw128(sK + 32 * k, 16, 1024), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(sv);
      mbar_arrive(&k_empty[s]);

      // ---- online softmax: sv[i] is (row rw + 8 ((i / 2) % 2), key 8 (i / 4) + 2 (lane % 4) + i % 2) ----
      const int kv0 = j * 128;
      if (kv0 + 128 > kv_len) {
#pragma unroll
        for (int i = 0; i < 64; ++i)
          if (kv0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= kv_len) sv[i] = -INFINITY;
      }
      float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
      for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sv[i]);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      }
      float sc[2], mb[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        sc[r] = ex2_approx((m_run[r] - mx[r]) * kLog2e);   // 0 on the first tile (m_run = -inf)
        m_run[r] = mx[r];
        mb[r] = mx[r] * kLog2e;
        l_run[r] *= sc[r];
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] *= sc[(i >> 1) & 1];
      uint32_t pa[8][4];   // P as the A fragments of the 8 K-steps (16 keys each) of the PV MMA
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int i = 8 * kk + 2 * m, r = m & 1;
          const float e0 = ex2_approx(fmaf(sv[i], kLog2e, -mb[r]));
          const float e1 = ex2_approx(fmaf(sv[i + 1], kLog2e, -mb[r]));
          l_run[r] += e0 + e1;
          pa[kk][m] = pack_bf16x2(e0, e1);
        }
      }

      // ---- O += P V (64 x 64) ----
      mbar_wait(&v_full[s], ph);
      const uint32_t sV = smem_u32(smem + AttnSmem::kV + s * 16384);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_bf16_rs_n64_tb(o, pa[kk], gmma_desc_sw128(sV + kk * 2048, 16384, 1024));
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(o);
      mbar_arrive(&v_empty[s]);
    }

    // ---- epilogue: O / l ----
    pdl_launch_dependents();
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const float inv[2] = {1.f / l_run[0], 1.f / l_run[1]};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int n = q0 + wg * 64 + rw + 8 * r;
      if (n >= p.N) continue;
      const size_t row = (size_t)b * p.N + n;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int col = h * 64 + 8 * c + 2 * (lane & 3);
        const float v0 = o[4 * c + 2 * r] * inv[r], v1 = o[4 * c + 2 * r + 1] * inv[r];
        if constexpr (kOut8) {
          uint16_t w;
          asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(w) : "f"(v1), "f"(v0));   // first source -> upper byte
          *reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(p.out) + row * p.ldo + col) = w;
        } else {
          *reinterpret_cast<uint32_t*>(p.out + row * p.ldo + col) = pack_bf16x2(v0, v1);
        }
      }
    }
  }

  __syncthreads();
  if (threadIdx.x == 0) prof_stamp_end(p.prof);
}

}  // namespace f5
