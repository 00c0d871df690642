// wgmma + TMA GEMM for sm_90a:  D[M,N] = epilogue( A[M,K] (bf16 or e4m3, K-major) · W[N,K]^T )
//
// Persistent: min(tiles, SMs) CTAs of 384 threads (three warpgroups), one per SM; CTA c computes the 128 x BN output
// tiles t = c, c + G, c + 2G, ... (G = gridDim.x; tile t is column tile t % tiles_n of row tile t / tiles_n, so the
// tiles in flight at once are the first wave of the one-tile-per-CTA grid).
//   warpgroup 0   TMA producer (one elected thread of warp 0): streams the A/B k-blocks of the CTA's tiles, tile after
//                 tile, through one 128B-swizzled smem ring; the first ring of weight tiles is requested before the
//                 PDL wait when the caller marks W as static
//   warpgroups 1-2 consumers, ping-pong: local tile j of the CTA belongs to warpgroup j & 1, which multiplies all 128
//                 rows (two wgmma m64nBN accumulators in registers) and then runs the tile's epilogue — while the other
//                 warpgroup runs tile j + 1's MMAs
// Pipeline: smem full/empty mbarriers (TMA <-> the consumer warpgroup reading the stage), plus two hand-over mbarriers
// between the consumers: `mma_turn` (tile j's main loop is done: tile j + 1 may wait on the ring — the ring's phase
// bits only tell k-blocks apart in order) and `epi_free` (tile j's epilogue has finished with the accumulator tile and
// the staging: tile j + 1 may write them).  The accumulator tile is BN / 32 fp32 boxes of 128 rows x 32 columns in the
// layout of the epilogue's TMA stores; the epilogue is one thread per output row (gemm_epilogue.cuh).  The CTA's last
// tile has no next main loop to hide its epilogue under: at BN = 128 (RoPE epilogue excepted) its owner drains columns
// [0, 64) and the other consumer warpgroup, released by `tail_ready` once the accumulator boxes and staged columns are
// written, drains [64, 128) (the split drain).
//
// The same kernel runs the 1-D convolutions of the path as implicit GEMMs: the A operand is a
// 3-D tensor map (channels, frames, batch) and k-block kb reads the tile shifted by
// (tap * dilation - pad) frames; TMA zero-fills the out-of-range frames, which is exactly the conv's zero
// padding (reference: nn.Conv1d(padding=k//2), dit.py:33-38; dilation > 1: BigVGAN's AMP-block convolutions).
//
// Epilogue (all fp32, fused, per reference op):
//   v = acc + bias[col]                                   Linear bias        (dit.py:136-143 ...)
//   v = act(v)            none | GELU-tanh | GELU-erf | Mish   (dit.py:94-99, convnext_v2.py:41, dit.py:36)
//   RoPE on adjacent column pairs for col < rope_cols     (rope.py:87-107, dit.py:157-158)
//   v *= q_scale for col < q_cols                         softmax scale folded into q (dit.py:166)
//   v = row valid ? v : 0                                 "x * mask" (dit.py:172-173)
//   v = v * gate[col] + resid[row, col]                   AdaLN-Zero gate (dit.py:319,323), residual (fp32 stream)
//   store fp32 or bf16
#pragma once
#include <type_traits>

#include "ptx.cuh"
#include "gemm_epilogue.cuh"

namespace f5 {

template <int BN, int kStages, bool SCALED = false>
struct GemmSmem {
  static constexpr int kABytes = 128 * 128;           // 128 rows x 128 bytes (64 bf16 / 128 e4m3)
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // accumulator tile: BN / 32 fp32 boxes of 128 rows x 128 bytes (SWIZZLE_128B), the epilogue's fp32 TMA-store boxes
  static constexpr int kAccOffset = kStages * kStageBytes;
  static constexpr int kAccBytes = (BN / 32) * 16384;
  // staging of the bf16 / e4m3 outputs and of the second output: 2 x 8 KB
  static constexpr int kStgOffset = kAccOffset + kAccBytes;
  // full[kStages], empty[kStages], mma_turn, epi_free, tail_ready
  static constexpr int kBarOffset = kStgOffset + 16384;
  static constexpr int kColsOffset = (kBarOffset + (2 * kStages + 3) * 8 + 15) & ~15;   // bias_s[BN], gate_s[BN], aux_s[BN]
  // block-scaled instantiations also stage ws_s[BN] (the per-column weight scale)
  static constexpr int kTotal = kColsOffset + (SCALED ? 4 : 3) * BN * 4 + 1024;  // + align slack
  static_assert(kStageBytes % 1024 == 0, "SWIZZLE_128B tiles and boxes sit on 1024-byte boundaries");
  static_assert(kTotal <= 232448, "GEMM: shared memory over the 227 KB limit");
};

template <int BN>
struct GemmEpi {
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

// Output tile t of the grid-stride walk: column tile t % tiles_n, row tile t / tiles_n (flat rows, or tiles_per_batch
// row tiles per utterance in batched / conv mode).
struct GemmTile {
  int n0;             // first output column
  int batch;          // utterance (batched mode; 0 otherwise)
  int m_in_batch0;    // first row inside the utterance (flat mode: = row0)
  int row0;           // first row of the flat [M, ...] matrices
};
__device__ __forceinline__ GemmTile gemm_tile(const GemmParams& p, int t, int bn) {
  GemmTile g;
  const int tiles_n = (p.N + bn - 1) / bn;
  const int mt = t / tiles_n;
  g.n0 = (t - mt * tiles_n) * bn;
  if (p.tiles_per_batch > 0) {
    g.batch = mt / p.tiles_per_batch;
    g.m_in_batch0 = (mt - g.batch * p.tiles_per_batch) * 128;
    g.row0 = g.batch * p.rows_per_batch + g.m_in_batch0;
  } else {
    g.batch = 0;
    g.row0 = mt * 128;
    g.m_in_batch0 = g.row0;
  }
  return g;
}
__device__ __forceinline__ int gemm_tiles(const GemmParams& p, int bn) {
  return (p.N + bn - 1) / bn * (p.tiles_per_batch > 0 ? p.num_batches * p.tiles_per_batch : (p.M + 127) / 128);
}
// k-blocks per tile: always 128 bytes per row (one swizzle span), 64 bf16 or 128 e4m3 elements
__device__ __forceinline__ int gemm_num_kb(const GemmParams& p) {
  return p.conv_taps * (p.ab8 ? (p.k_per_tap + 127) >> 7 : (p.k_per_tap + 63) >> 6);
}

// Epilogue of the 64-column units [cc0, cc0 + ncc) of tile g, run by the 128 threads of consumer warpgroup wg (thread
// et drains tile row et) once the tile's owner has written the accumulator boxes and staged the columns.  The owner's
// threads meet at the warpgroup's named barrier; a helper's wait on tail_ready for the owner's writes.
template <int BN, int ACT, bool OUT_BF16, bool ROPE, bool SCALED>
__device__ __forceinline__ void gemm_epilogue_units(const GemmParams& p, const GemmTile& g, int cc0, int ncc, int wg,
                                                    int et, uint8_t* acc_tile, uint8_t* stg_buf, const float* bias_s,
                                                    const float* gate_s, const float* aux_s, const float* ws_s,
                                                    const CUtensorMap* tma_out, const CUtensorMap* tma_out2,
                                                    uint64_t* tail_ready, bool helper) {
  const int m_in_batch = g.m_in_batch0 + et;
  const int row = g.row0 + et;
  bool row_ok;
  int b_idx, pos;
  if (p.tiles_per_batch > 0) {
    row_ok = m_in_batch < p.rows_per_batch;
    b_idx = g.batch;
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
  if constexpr (!(ROPE || SCALED)) epi_load_resid(p, row, g.n0 + 64 * cc0, row_ok, res0);   // else in epi_drain_tile
  EpiStage stg;
  stg.acc = acc_tile;
  stg.stg = stg_buf;
  stg.et = et;
  stg.r = et;
  stg.map_out = tma_out;
  stg.map_out2 = tma_out2;
  stg.c1 = g.m_in_batch0;
  stg.c2 = g.batch;
  stg.bar_id = 1 + wg;
  stg.mu_r = ln_mu_r; stg.rstd = ln_rstd;
  stg.out_fp8 = p.out_fp8;
  // accumulator tile and staged columns visible
  if (helper) mbar_wait(tail_ready, 0);
  else asm volatile("bar.sync %0, 128;" ::"r"(stg.bar_id) : "memory");
  epi_drain_tile<BN, ACT, OUT_BF16, ROPE, SCALED>(bias_s, gate_s, aux_s, cs, res0, p, g.n0, cc0, ncc, row, row_ok,
                                                  row_valid, stg, ws_s);
  // the next tile may rewrite the accumulator tile and the staging once the TMA unit has read them (and the CTA
  // may exit); grid completion makes the global writes visible to the dependent kernel
  if (et == 0) tma_store_wait_read<0>();
}

// FP8 = false instantiations have every e4m3 feature (ab8 / out_fp8 / out2_fp8 / acc_scale) folded away at compile
// time, so only the FP8 mode pays for the FP8 mode.  RESID = false instantiations (no residual input) drop the
// residual tiles from the epilogue's registers.
// SCALED = true (block-scaled FP8, DESIGN.md section 8): A may carry a power-of-two scale per (row, 64-column unit), which
// the main loop applies when it promotes each unit's e4m3 wgmma partial; the epilogue multiplies the accumulator by a
// per-column weight scale and writes e4m3 outputs with one scale per (row, 64-column unit).
template <int BN, int kStages, int ACT, bool OUT_BF16, bool ROPE, bool FP8 = false, bool RESID = true, bool SCALED = false>
__global__ void __launch_bounds__(384, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tma_a,
                    const __grid_constant__ CUtensorMap tma_b, const __grid_constant__ CUtensorMap tma_out,
                    const __grid_constant__ CUtensorMap tma_out2, const GemmParams p_arg) {
  GemmParams p = p_arg;
  if constexpr (!FP8) { p.ab8 = 0; p.out_fp8 = 0; p.out2_fp8 = 0; p.acc_scale = 1.f; }
  if constexpr (!RESID) p.resid = nullptr;
  if constexpr (!SCALED) { p.a_scale = nullptr; p.w_scale = nullptr; p.out_scale = nullptr; p.out2_scale = nullptr; }
  using S = GemmSmem<BN, kStages, SCALED>;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles must sit on 1024-byte boundaries
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOffset);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* mma_turn = empty_bar + kStages;
  uint64_t* epi_free = mma_turn + 1;
  uint64_t* tail_ready = epi_free + 1;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // ---- one-time setup (overlaps the predecessor kernel under PDL) ----
  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    tma_prefetch_desc(&tma_out);
    if (p.out2 != nullptr) tma_prefetch_desc(&tma_out2);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 128);   // every thread of the consumer warpgroup that read the stage releases it
    }
    mbar_init(mma_turn, 128);
    mbar_init(epi_free, 128);
    mbar_init(tail_ready, 128);
    fence_mbar_init();
  }
  if (warp == 1) prefetch_slice_l2(p, blockIdx.x, gridDim.x, lane);
  __syncthreads();
  // weights do not depend on the predecessor kernel: the first ring of the first tile's B tiles is requested BEFORE
  // the PDL wait, so their (possibly HBM) latency runs under the predecessor's tail
  const int early_b = p.w_static ? min(kStages, gemm_num_kb(p)) : 0;
  if (warp == 0 && elect_one()) {
    const int n0 = gemm_tile(p, blockIdx.x, BN).n0;
    for (int kb = 0; kb < early_b; ++kb) {
      mbar_expect_tx(&full_bar[kb], S::kStageBytes);
      tma_load_2d(smem + kb * S::kStageBytes + S::kABytes, &tma_b, &full_bar[kb], kb * (p.ab8 ? 128 : 64), n0);
    }
  }
  pdl_wait();   // predecessor's outputs (our A operand / residual) are complete and visible
  if (threadIdx.x == 128) prof_stamp_begin(p.prof);

  // Registers move from the producer warpgroup (one thread issues TMA) to the consumers, which hold a whole tile's
  // accumulator (BN registers) in the main loop and RoPE tables and residual tiles in the epilogue:
  // 128 x 40 + 256 x 232 = the 384 x 168 of the launch.
  if (warp < 4) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
    if (warp == 0 && elect_one()) {
      auto produce = [&](auto ab8_tag) {
        constexpr int KBE = decltype(ab8_tag)::value ? 128 : 64;     // elements per k-block, compile-time in the loop
        // incremental stage / phase / tap bookkeeping: no division in the loop
        const int kb_per_tap = (p.k_per_tap + KBE - 1) / KBE, num_kb = p.conv_taps * kb_per_tap, tiles = gemm_tiles(p, BN);
        const int tap_step = p.conv_dilation > 1 ? p.conv_dilation : 1;
        int s = 0;
        uint32_t ph = 1;
        uint8_t* sa = smem;
        int early = p.w_static ? min(kStages, num_kb) : 0;   // the first tile's early weight tiles
        for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
          const GemmTile g = gemm_tile(p, t, BN);
          const int a_col0 = p.conv_grouped ? g.n0 : 0;
          // tap t reads frames m + t * conv_dilation - conv_pad (conv_dilation 0 or 1: m + t - conv_pad)
          int a_row = g.m_in_batch0 - p.conv_pad, kc = 0;
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&empty_bar[s], ph);
            if (kb >= early) mbar_expect_tx(&full_bar[s], S::kStageBytes);
            tma_load_3d(sa, &tma_a, &full_bar[s], a_col0 + kc * KBE, a_row, g.batch);
            if (kb >= early) tma_load_2d(sa + S::kABytes, &tma_b, &full_bar[s], kb * KBE, g.n0);
            if (++s == kStages) { s = 0; ph ^= 1; sa = smem; } else { sa += S::kStageBytes; }
            if (++kc == kb_per_tap) { kc = 0; a_row += tap_step; }
          }
          early = 0;
        }
      };
      if (p.ab8) produce(std::true_type{});
      else produce(std::false_type{});
    }
  } else {
    // ===================== consumers: ping-pong over the CTA's tiles =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
    const int wg = (threadIdx.x >> 7) - 1;          // local tiles j = wg, wg + 2, ...
    const int et = threadIdx.x & 127;               // epilogue: this thread's tile row
    const int wr = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);   // accumulator fragment rows wr, wr + 8 (+ 64 h)
    const uint32_t ring = smem_u32(smem);
    uint8_t* acc_tile = smem + S::kAccOffset;
    float* bias_s = reinterpret_cast<float*>(smem + S::kColsOffset);
    float* gate_s = bias_s + BN;
    float* aux_s = bias_s + 2 * BN;
    float* ws_s = SCALED ? bias_s + 3 * BN : nullptr;

    // local tile j waits for tile j - 1's hand-overs: phase j - 1 of mma_turn / epi_free, parity (j - 1) & 1 = wg ^ 1
    const uint32_t turn_par = (uint32_t)wg ^ 1u;
    // The RoPE epilogue (the QKV GEMM, 2-3 tiles per CTA at batch 1) measured slower with the split drain, so it keeps
    // the single-warpgroup drain (DESIGN.md section 7)
    constexpr bool kSplit = BN == 128 && !ROPE;
#pragma unroll 1
    for (int t = blockIdx.x + wg * gridDim.x;; t += 2 * gridDim.x) {
      // Split drain of the CTA's last tile (kSplit: BN = 128, two 64-column units): no further tile's MMAs hide its epilogue,
      // so its owner drains unit 0 and the other consumer warpgroup drains unit 1.  That helper is the warpgroup past
      // its own tiles when the last tile, t - G, is the other's: in a one-tile CTA the one that had no tile, else the
      // one whose own last epilogue has just ended.  A unit's fused-LN statistics, RoPE head and block scale stay with
      // one thread: every output bit is what one warpgroup computes alone.
      const bool past = t >= gemm_tiles(p, BN);   // this warpgroup has no tile left
      if (past && !(kSplit && p.tail_split && t - (int)gridDim.x < gemm_tiles(p, BN))) break;
      const bool help = kSplit && past;
      const bool first = t == (int)blockIdx.x;   // j == 0
      bool split = help;   // this warpgroup drains one unit of the tile
      GemmTile g;          // the tile whose epilogue it runs
      if (!help) {
        const int num_kb = gemm_num_kb(p);
        // the tile's first k-block in the CTA's stream: j * num_kb, j = local tile index (only t is carried across tiles)
        const int kb0 = (t - (int)blockIdx.x) / (int)gridDim.x * num_kb;
        int s = kb0 % kStages;
        uint32_t ph = (uint32_t)(kb0 / kStages) & 1u;
        if (!first) mbar_wait(mma_turn, turn_par);   // tile j - 1 has waited on all of its k-blocks

        float acc[2][BN / 2];   // rows [0, 64) and [64, 128) of the tile
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
        auto mma_loop = [&](auto ab8_tag) {
          constexpr bool AB8 = decltype(ab8_tag)::value;
          if constexpr (AB8) {
            // e4m3 wgmma accumulates with fewer mantissa bits than fp32: each k-block (128 products per output) goes to
            // a fresh partial accumulator that is added to the fp32 accumulator on the CUDA cores, one 64-row half at a time
            float part[BN / 2];
            for (int kb = 0; kb < num_kb; ++kb) {
              mbar_wait(&full_bar[s], ph);
              const uint32_t sa = ring + s * S::kStageBytes, sb = ring + s * S::kStageBytes + S::kABytes;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k)
                  gemm_wgmma<BN, true>(part, gmma_desc_sw128(sa + h * (64 * 128) + 32 * k, 16, 1024),
                                       gmma_desc_sw128(sb + 32 * k, 16, 1024), k != 0);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_reg_fence(part);
                if (h == 1) mbar_arrive(&empty_bar[s]);
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[h][i] += part[i];
              }
              if (++s == kStages) { s = 0; ph ^= 1; }
            }
          } else {
            int s_prev = 0;
            for (int kb = 0; kb < num_kb; ++kb) {
              mbar_wait(&full_bar[s], ph);
              const uint32_t sa = ring + s * S::kStageBytes, sb = ring + s * S::kStageBytes + S::kABytes;
              wgmma_fence();
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int k = 0; k < 4; ++k)    // 4 K-steps of 16 bf16 (32 bytes) per 128-byte k-block row
                  gemm_wgmma<BN, false>(acc[h], gmma_desc_sw128(sa + h * (64 * 128) + 32 * k, 16, 1024),
                                        gmma_desc_sw128(sb + 32 * k, 16, 1024), (kb | k) != 0);
              wgmma_commit();
              // the previous k-block's MMAs have retired once at most this one is in flight: release its stage
              wgmma_wait<1>();
              if (kb > 0) mbar_arrive(&empty_bar[s_prev]);
              s_prev = s;
              if (++s == kStages) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            wgmma_reg_fence(acc[0]);
            wgmma_reg_fence(acc[1]);
            mbar_arrive(&empty_bar[s_prev]);
          }
        };
        // Block-scaled A: each 128-byte e4m3 k-block holds two 64-element units with their own row scales.  A unit's two
        // k32 wgmmas go to a fresh partial that is promoted as acc = fma(part, s_a[row], acc), one 64-row half at a time.
        // The thread's fragment rows are wr and wr + 8 of each half (acc[h][i] belongs to row 64 h + wr + 8 ((i / 2) % 2));
        // their scales are loaded before the stage's wait, and only for rows that exist (TMA zero-fills A past the matrix
        // or the utterance, a plain load would not).
        auto mma_loop_scaled = [&]() {
          const GemmTile g = gemm_tile(p, t, BN);
          const int lim = p.tiles_per_batch > 0 ? p.rows_per_batch - g.m_in_batch0 : p.M - g.row0;   // rows that exist
          const float* sp = p.a_scale + g.row0 + wr;
          const size_t ld = (size_t)p.a_scale_ld;
          float part[BN / 2];
          for (int kb = 0; kb < num_kb; ++kb) {
            float sc[2][2][2];   // [unit][half][row]
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const float* su = sp + (size_t)(2 * kb + u) * ld;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                sc[u][h][0] = 64 * h + wr < lim ? su[64 * h] : 0.f;
                sc[u][h][1] = 64 * h + wr + 8 < lim ? su[64 * h + 8] : 0.f;
              }
            }
            mbar_wait(&full_bar[s], ph);
            const uint32_t sa = ring + s * S::kStageBytes, sb = ring + s * S::kStageBytes + S::kABytes;
#pragma unroll
            for (int u = 0; u < 2; ++u) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 2; ++k)
                  gemm_wgmma<BN, true>(part, gmma_desc_sw128(sa + h * (64 * 128) + 64 * u + 32 * k, 16, 1024),
                                       gmma_desc_sw128(sb + 64 * u + 32 * k, 16, 1024), k != 0);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_reg_fence(part);
                if (u == 1 && h == 1) mbar_arrive(&empty_bar[s]);
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[h][i] = fmaf(part[i], sc[u][h][(i >> 1) & 1], acc[h][i]);
              }
            }
            if (++s == kStages) { s = 0; ph ^= 1; }
          }
        };
        if constexpr (SCALED) {
          if (p.ab8 && p.a_scale != nullptr) mma_loop_scaled();
          else if (p.ab8) mma_loop(std::true_type{});
          else mma_loop(std::false_type{});
        } else {
          if (p.ab8) mma_loop(std::true_type{});
          else mma_loop(std::false_type{});
        }
        mbar_arrive(mma_turn);
        // PDL: the CTA's last main loop is done — let the next kernel of the stream start its prologue under this
        // epilogue; it still waits (pdl_wait) for this grid to complete before touching memory
        const bool last = t + (int)gridDim.x >= gemm_tiles(p, BN);
        if (last) pdl_launch_dependents();
        split = kSplit && p.tail_split && last;

        // ===================== epilogue =====================
        g = gemm_tile(p, t, BN);   // (not held in registers across the main loop)
        if (!first) mbar_wait(epi_free, turn_par);   // tile j - 1's epilogue is done with the shared tile
        // accumulator fragments -> the fp32 boxes (SWIZZLE_128B: 16-byte piece q of row r at (q ^ (r & 7)) * 16)
        {
          const int sw = wr & 7;   // = (wr + 8) & 7 = (wr + 64) & 7
          uint8_t* base = acc_tile + wr * 128 + (lane & 1) * 8;
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int q = 0; q < BN / 8; ++q) {   // columns 8 q + 2 (lane % 4) + {0, 1}
              uint8_t* pc = base + h * (64 * 128) + (q >> 2) * 16384 + (((2 * (q & 3) + ((lane >> 1) & 1)) ^ sw) << 4);
              *reinterpret_cast<float2*>(pc) = make_float2(acc[h][4 * q], acc[h][4 * q + 1]);
              *reinterpret_cast<float2*>(pc + 8 * 128) = make_float2(acc[h][4 * q + 2], acc[h][4 * q + 3]);
            }
        }
        epi_stage_cols<BN, SCALED>(p, g.n0, et, bias_s, gate_s, aux_s, ws_s);
        if (split) mbar_arrive(tail_ready);   // the helper may drain unit 1
      } else {
        g = gemm_tile(p, t - (int)gridDim.x, BN);   // the other warpgroup's tile, the CTA's last
      }
      // The helper stages its chunks in the first ring stage: the producer has issued, and the owner consumed, every
      // k-block of the CTA, so the ring is idle.
      gemm_epilogue_units<BN, ACT, OUT_BF16, ROPE, SCALED>(p, g, help ? 1 : 0, split ? 1 : BN / 64, wg, et, acc_tile,
                                                           help ? smem : smem + S::kStgOffset, bias_s, gate_s, aux_s,
                                                           ws_s, &tma_out, &tma_out2, tail_ready, help);
      // nothing waits on the last tile's epi_free phase; the CTA exits once both halves' TMA stores have read their
      // sources
      if (help) break;
      mbar_arrive(epi_free);
    }
  }

  __syncthreads();
  if (threadIdx.x == 0) prof_stamp_end(p.prof);
}

}  // namespace f5
