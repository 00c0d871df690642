// wgmma + TMA GEMM for sm_90a:  D[M,N] = epilogue( A[M,K] (bf16 or e4m3, K-major) · W[N,K]^T )
//
// One CTA computes one 128 x BN output tile with 384 threads (three warpgroups):
//   warpgroup 0   TMA producer (one elected thread of warp 0): A/B k-blocks -> 128B-swizzled smem ring; the first
//                 ring of weight tiles is requested before the PDL wait when the caller marks W as static
//   warpgroups 1-2 consumers: warpgroup g multiplies rows [64 g, 64 g + 64) of the tile (wgmma m64nBN, fp32
//                 accumulator in registers), keeping one MMA group in flight while the previous stage is released
// Pipeline: smem full/empty mbarriers (TMA <-> consumers).  After the main loop the consumers write their
// accumulators to an fp32 tile in shared memory and become the epilogue: one thread per output row, one group of
// 128 threads per BN / kGroups columns (gemm_epilogue.cuh).
//
// The same kernel runs the 1-D convolutions of the path as implicit GEMMs: the A operand is a
// 3-D tensor map (channels, frames, batch) and k-block kb reads the tile shifted by
// (tap - pad) frames; TMA zero-fills the out-of-range frames, which is exactly the conv's zero
// padding (reference: nn.Conv1d(padding=k//2), dit.py:33-38).
//
// Epilogue (all fp32, fused, per reference op):
//   v = acc + bias[col]                                   Linear bias        (dit.py:136-143 ...)
//   v = act(v)            none | GELU-tanh | GELU-erf | Mish   (dit.py:94-99, convnext_v2.py:41, dit.py:36)
//   RoPE on adjacent column pairs for col < rope_cols     (rope.py:87-107, dit.py:157-158)
//   v *= q_scale for col < q_cols                         softmax scale folded into q (dit.py:166)
//   v = row valid ? v : 0                                 "x * mask" (dit.py:172-173)
//   v *= gate[batch, col]                                 AdaLN-Zero gate (dit.py:319,323)
//   v += resid[row, col]                                  residual (fp32 stream)
//   store fp32 or bf16
#pragma once
#include <type_traits>

#include "ptx.cuh"
#include "gemm_epilogue.cuh"

namespace f5 {

template <int BN, int kStages>
struct GemmSmem {
  static constexpr int kABytes = 128 * 128;           // 128 rows x 128 bytes (64 bf16 / 128 e4m3)
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccOffset = kStages * kStageBytes;
  static constexpr int kAccLd = BN + 4;                // floats per accumulator row: conflict-free row-wise float4 reads
  static constexpr int kBarOffset = kAccOffset + 128 * kAccLd * 4;
  static constexpr int kColsOffset = (kBarOffset + 2 * kStages * 8 + 15) & ~15;   // bias_s[BN], gate_s[BN], aux_s[BN]
  static constexpr int kTotal = kColsOffset + 3 * BN * 4 + 1024;  // + align slack
  // epilogue store staging reuses the (idle) operand ring: fp32/bf16 chunks at [0, 64 KB) (32 KB per group), the
  // bf16 copy of the fused-LN producer mode at [64 KB, 96 KB) (16 KB per group, two alternating 8 KB buffers)
  static_assert(kStages * kStageBytes >= 98304, "operand ring too small for the epilogue staging");
  static_assert(kTotal <= 232448, "GEMM: shared memory over the 227 KB limit");
};

// Epilogue groups: 128 threads each (one per tile row); with 128-column tiles the two consumer warpgroups drain
// columns [0, 64) and [64, 128) side by side.
template <int BN>
struct GemmEpi {
  static constexpr int kGroups = BN >= 128 ? 2 : 1;
  static constexpr int kCols = BN / kGroups;          // columns per group
  static constexpr int kThreads = 384;
};

template <int BN, bool AB8>
__device__ __forceinline__ void gemm_wgmma(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (AB8) {
    if constexpr (BN == 128) wgmma_e4m3_ss_n128(acc, da, db, scale_d);
    else wgmma_e4m3_ss_n64(acc, da, db, scale_d);
  } else {
    if constexpr (BN == 128) wgmma_bf16_ss_n128(acc, da, db, scale_d);
    else wgmma_bf16_ss_n64(acc, da, db, scale_d);
  }
}

// FP8 = false instantiations have every e4m3 feature (ab8 / out_fp8 / out2_fp8 / acc_scale) folded away at compile
// time, so only the FP8 mode pays for the FP8 mode.  RESID = false instantiations (no residual input) drop the
// residual tiles from the epilogue's registers.
template <int BN, int kStages, int ACT, bool OUT_BF16, bool ROPE, bool FP8 = false, bool RESID = true>
__global__ void __launch_bounds__(384, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tma_a,
                    const __grid_constant__ CUtensorMap tma_b, const __grid_constant__ CUtensorMap tma_out,
                    const __grid_constant__ CUtensorMap tma_out2, const GemmParams p_arg) {
  GemmParams p = p_arg;
  if constexpr (!FP8) { p.ab8 = 0; p.out_fp8 = 0; p.out2_fp8 = 0; p.acc_scale = 1.f; }
  if constexpr (!RESID) p.resid = nullptr;
  using S = GemmSmem<BN, kStages>;
  using E = GemmEpi<BN>;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles must sit on 1024-byte boundaries
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOffset);
  uint64_t* empty_bar = full_bar + kStages;
  float* acc_s = reinterpret_cast<float*>(smem + S::kAccOffset);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // ---- tile coordinates ----
  const int n0 = blockIdx.x * BN;
  int batch = 0, m_in_batch0 = 0, row0;
  if (p.tiles_per_batch > 0) {
    batch = blockIdx.y / p.tiles_per_batch;
    m_in_batch0 = (blockIdx.y % p.tiles_per_batch) * 128;
    row0 = batch * p.rows_per_batch + m_in_batch0;
  } else {
    row0 = blockIdx.y * 128;
    m_in_batch0 = row0;
  }
  const int kbe = p.ab8 ? 128 : 64;      // elements per k-block: always 128 bytes per row (one swizzle span)
  const int kb_per_tap = (p.k_per_tap + kbe - 1) / kbe;
  const int num_kb = p.conv_taps * kb_per_tap;

  // ---- one-time setup (overlaps the predecessor kernel under PDL) ----
  const int cta_lin = blockIdx.y * gridDim.x + blockIdx.x;
  if (threadIdx.x == 0) ts_mark(p, cta_lin, 0);
  if (warp == 0 && F5_ELECT_LANE()) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    tma_prefetch_desc(&tma_out);
    if (p.out2 != nullptr) tma_prefetch_desc(&tma_out2);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 256);   // every consumer thread releases the stage it has read
    }
    fence_mbar_init();
  }
  if (warp == 1) prefetch_slice_l2(p, cta_lin, gridDim.x * gridDim.y, lane);
  __syncthreads();
  if (threadIdx.x == 0) ts_mark(p, cta_lin, 1);
  // weights do not depend on the predecessor kernel: the first ring of B tiles is requested BEFORE the PDL
  // wait, so their (possibly HBM) latency runs under the predecessor's tail
  const int early_b = p.w_static ? min(kStages, num_kb) : 0;
  if (warp == 0 && F5_ELECT_LANE()) {
    for (int kb = 0; kb < early_b; ++kb) {
      mbar_expect_tx(&full_bar[kb], S::kStageBytes);
      tma_load_2d(smem + kb * S::kStageBytes + S::kABytes, &tma_b, &full_bar[kb], kb * kbe, n0);
    }
  }
  pdl_wait();   // predecessor's outputs (our A operand / residual) are complete and visible
  if (threadIdx.x == 128) { ts_mark(p, cta_lin, 2); prof_stamp_begin(p.prof); }

  // Registers move from the producer warpgroup (one thread issues TMA) to the consumers, whose epilogue holds RoPE
  // tables and residual tiles next to the accumulator chunk: 128 x 40 + 256 x 232 = the 384 x 168 of the launch.
  if (warp < 4) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
    if (warp == 0 && F5_ELECT_LANE()) {
      auto produce = [&](auto ab8_tag) {
        constexpr int KBE = decltype(ab8_tag)::value ? 128 : 64;     // elements per k-block, compile-time in the loop
        // incremental stage / phase / tap bookkeeping: no division in the loop
        int s = 0, tap = 0, kc = 0;
        uint32_t ph = 1;
        uint8_t* sa = smem;
        const int a_col0 = p.conv_grouped ? n0 : 0;
        const int a_row0 = m_in_batch0 - p.conv_pad;
        const int a_b = p.tiles_per_batch > 0 ? batch : 0;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[s], ph);
          if (kb >= early_b) mbar_expect_tx(&full_bar[s], S::kStageBytes);
          tma_load_3d(sa, &tma_a, &full_bar[s], a_col0 + kc * KBE, a_row0 + tap, a_b);
          if (kb >= early_b) tma_load_2d(sa + S::kABytes, &tma_b, &full_bar[s], kb * KBE, n0);
          if (++s == kStages) { s = 0; ph ^= 1; sa = smem; } else { sa += S::kStageBytes; }
          if (++kc == kb_per_tap) { kc = 0; ++tap; }
        }
      };
      if (p.ab8) produce(std::true_type{});
      else produce(std::false_type{});
    }
  } else {
    // ===================== consumers: main loop =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
    const int wg = (threadIdx.x >> 7) - 1;          // 0: tile rows [0, 64), 1: [64, 128)
    const int et = threadIdx.x & 127;
    const int grp = wg;                             // epilogue group (columns [grp * kCols, (grp + 1) * kCols))
    constexpr int BNG = E::kCols;
    const int n0g = n0 + grp * BNG;
    float* bias_s = reinterpret_cast<float*>(smem + S::kColsOffset) + grp * BNG;
    float* gate_s = reinterpret_cast<float*>(smem + S::kColsOffset) + BN + grp * BNG;
    float* aux_s = reinterpret_cast<float*>(smem + S::kColsOffset) + 2 * BN + grp * BNG;
    if (grp < E::kGroups) epi_stage_cols<BNG>(p, n0g, et, bias_s, gate_s, aux_s);   // under the main loop's loads

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    auto mma_loop = [&](auto ab8_tag) {
      constexpr bool AB8 = decltype(ab8_tag)::value;
      const uint32_t ring = smem_u32(smem);
      int s = 0, s_prev = 0;
      uint32_t ph = 0;
      if constexpr (AB8) {
        // e4m3 wgmma accumulates with fewer mantissa bits than fp32: each k-block (128 products per output) goes to
        // a fresh partial accumulator that is added to the fp32 accumulator on the CUDA cores
        float part[BN / 2];
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&full_bar[s], ph);
          const uint32_t sa = ring + s * S::kStageBytes + wg * (64 * 128), sb = ring + s * S::kStageBytes + S::kABytes;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
            gemm_wgmma<BN, true>(part, gmma_desc_sw128(sa + 32 * k, 16, 1024), gmma_desc_sw128(sb + 32 * k, 16, 1024),
                                 k != 0);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_reg_fence(part);
          mbar_arrive(&empty_bar[s]);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
          if (++s == kStages) { s = 0; ph ^= 1; }
        }
      } else {
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&full_bar[s], ph);
          const uint32_t sa = ring + s * S::kStageBytes + wg * (64 * 128), sb = ring + s * S::kStageBytes + S::kABytes;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)    // 4 K-steps of 16 bf16 (32 bytes) per 128-byte k-block row
            gemm_wgmma<BN, false>(acc, gmma_desc_sw128(sa + 32 * k, 16, 1024), gmma_desc_sw128(sb + 32 * k, 16, 1024),
                                  (kb | k) != 0);
          wgmma_commit();
          // the previous k-block's MMAs have retired once at most this one is in flight: release its stage
          wgmma_wait<1>();
          if (kb > 0) mbar_arrive(&empty_bar[s_prev]);
          s_prev = s;
          if (++s == kStages) { s = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_reg_fence(acc);
      }
    };
    if (p.ab8) mma_loop(std::true_type{});
    else mma_loop(std::false_type{});

    // accumulator fragments -> fp32 tile in shared memory (row-major, kAccLd floats per row)
    {
      const int r = wg * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
      const int c = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<float2*>(acc_s + r * S::kAccLd + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(acc_s + (r + 8) * S::kAccLd + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    asm volatile("bar.sync 3, 256;" ::: "memory");   // accumulator tile and staged columns visible to both groups
    // PDL: the main loop is done — let the next kernel of the stream start its prologue under this epilogue; it
    // still waits (pdl_wait) for this grid to complete before touching memory
    pdl_launch_dependents();
    if (grp < E::kGroups) {
      // ===================== epilogue =====================
      if (et == 0 && grp == 0) ts_mark(p, cta_lin, 7);
      const int r_in_tile = et;
      const int m_in_batch = m_in_batch0 + r_in_tile;
      const int row = row0 + r_in_tile;
      bool row_ok;
      int b_idx, pos;
      if (p.tiles_per_batch > 0) {
        row_ok = m_in_batch < p.rows_per_batch;
        b_idx = batch;
        pos = m_in_batch;
      } else {
        row_ok = row < p.M;
        const int rpb = p.rows_per_batch > 0 ? p.rows_per_batch : p.M;
        b_idx = row / rpb;
        pos = row - b_idx * rpb;
      }
      if (!row_ok) { b_idx = 0; pos = 0; }
      bool row_valid = true;
      if (p.row_len != nullptr) row_valid = pos < p.row_len[b_idx];
      float ln_mu_r, ln_rstd;
      epi_load_ln_row(p, row, row_ok, ln_mu_r, ln_rstd);
      float2 cs[ROPE ? 32 : 1];
      epi_load_rope<ROPE>(p, pos, cs);
      float4 res0[8];
      epi_load_resid(p, row, n0g, row_ok, res0);
      // every MMA has retired, so the operand ring is idle: its first 32 KB per group stage the stores
      EpiStage stg;
      stg.buf = smem + grp * 32768;
      stg.et = et;
      stg.r = r_in_tile;
      stg.map_out = &tma_out;
      stg.map_out2 = &tma_out2;
      stg.c1 = m_in_batch0;
      stg.c2 = p.tiles_per_batch > 0 ? batch : 0;
      stg.bar_id = 1 + grp;
      stg.buf2 = smem + 65536 + grp * 16384;
      stg.buf2_par = 8192;
      stg.mu_r = ln_mu_r; stg.rstd = ln_rstd;
      stg.out_fp8 = p.out_fp8;
      epi_drain_tile<BNG, ACT, OUT_BF16, ROPE>(acc_s + r_in_tile * S::kAccLd + grp * BNG, bias_s, gate_s, aux_s, cs,
                                               res0, p, n0g, row, b_idx, row_ok, row_valid, stg);
      if (et == 0) tma_store_wait_read<0>();   // the staging buffers must outlive the TMA unit's reads; grid completion
                                               // makes the global writes visible to the dependent kernel
    }
  }

  __syncthreads();
  if (threadIdx.x == 0) { ts_mark(p, cta_lin, 9); prof_stamp_end(p.prof); }
}

}  // namespace f5
