// FP8 attention of the block-scaled FP8 mode (DESIGN.md sections 5 and 8): e4m3 Q·K^T and P·V on wgmma.  Q has one
// power-of-two scale per (row, head); K and V have one per (utterance, head, 128-key tile), so that inside a key tile
// every score and every probability shares one scale and the softmax does no per-key scale work.  Two kernels:
//
//   qkv_quant_e4m3_kernel   the QKV GEMM's bf16 [q | k | v] -> e4m3 Q | K (row-major), e4m3 V^T per (utterance, head)
//                           with keys contiguous (the K-major B operand of P·V), and the scales [3H][rows]
//   attn_fp8_kernel         flash attention on those operands; same grid and roles as attn_fwd_kernel
//                           (attention_sm90.cuh): warpgroup 0 = TMA producer, warpgroups 1-2 = consumers of 64 query
//                           rows each:
//                             S = Q8 K8^T       wgmma m64n128k32 e4m3, both from shared memory (SWIZZLE_64B)
//                             log2 e * sq[row] * sk[tile] folded into the exponent (powers of two: exact)
//                             online softmax; l sums the fp32 p
//                             P~ = e4m3(2^8 p)
//                             O_t = P~ V8^T     wgmma m64n64k32 e4m3, P~ from registers, fresh accumulator per tile
//                             o = o * sc + sv[tile] * O_t
//                           and writes O / l as block-scaled e4m3 exactly like attn_fwd_kernel<true, true>.
//
// Key order of V^T.  The S accumulator holds, per row and per 32 keys, the keys {2l, 2l+1, 2l+8, 2l+9} and
// {16+2l, 17+2l, 24+2l, 25+2l} (l = lane % 4); the register A fragment of wgmma k32 e4m3 takes k = 4l .. 4l+3 and
// 16+4l .. 16+4l+3 (ptx.cuh wgmma_e4m3_rs_n64).  So V^T stores key fp8_vt_key(p) at position p of every 32-key
// group and the S fragment packs into the A fragment without a shuffle.  The host states the same order as
// weights.fp8_vt_key_order().
#pragma once
#include "ptx.cuh"

namespace f5 {

// position p (0..31) of a 32-key group of V^T holds key fp8_vt_key(p); fp8_vt_pos is its inverse
__host__ __device__ constexpr int fp8_vt_key(int p) {
  return (p & 16) + 2 * ((p >> 2) & 3) + ((p >> 1) & 1) * 8 + (p & 1);
}
__host__ __device__ constexpr int fp8_vt_pos(int k) {
  return (k & 16) + 4 * ((k >> 1) & 3) + 2 * ((k >> 3) & 1) + (k & 1);
}
__host__ __device__ constexpr bool fp8_vt_order_ok() {
  for (int p = 0; p < 32; ++p) {
    const int l = (p & 15) >> 2, i = p & 3;
    const int want = (p & 16) + (i == 0 ? 2 * l : i == 1 ? 2 * l + 1 : i == 2 ? 2 * l + 8 : 2 * l + 9);
    if (fp8_vt_key(p) != want || fp8_vt_pos(fp8_vt_key(p)) != p) return false;
  }
  return true;
}
static_assert(fp8_vt_order_ok(), "V^T key order: fp8_vt_key must be the fragment mapping and fp8_vt_pos its inverse");

struct QkvQuantParams {
  const __nv_bfloat16* qkv;  // [B*N, ld_qkv] = [q | k | v], each H*64 wide
  long long ld_qkv;          // elements
  uint8_t* qk8;              // e4m3 [B*N, ld_qk8] = [q | k]
  long long ld_qk8;          // bytes
  uint8_t* vt8;              // e4m3 [B][H*64][vt_ld]: V^T, keys in fp8_vt_key order per 32, zero beyond N
  long long vt_ld;           // bytes, >= roundup(N, 128)
  // [3H][B*N]: q head h -> unit h (the row's scale), k head h -> unit H + h, v head h -> 2H + h (for every key, the
  // scale of its 128-key tile)
  float* scale;
  int B, N, H;
  const int* kv_len;         // [B] valid keys per utterance, or null (= N): clamped as attn_fp8_kernel clamps it
  unsigned long long* prof;  // in-graph timing slot (ptx.cuh prof_stamp_*), or null
};

// grid (roundup(N, 128) / 128, H, B), 256 threads: one 128-key tile x (q, k, v) of one head; 8 threads per
// (row, unit), 12 (row, unit) tasks per thread.  The bf16 rows are read once and kept in registers while the tile's k
// and v amax is reduced through shared memory.  Keys at or beyond kv_len are read as zero: they do not move the tile's
// amax (a masked key must not set the scale of the valid keys beside it) and get zero K and V codes.
__global__ void __launch_bounds__(256) qkv_quant_e4m3_kernel(const QkvQuantParams p) {
  __shared__ uint32_t stage[64 * 33];   // V^T block [d][128 key positions], row pitch 132 B (2-way store conflicts)
  __shared__ uint32_t tile_amax[2];     // k, v: fp32 bits of a non-negative (or NaN) amax, ordered as unsigned
  pdl_launch_dependents();
  if (threadIdx.x < 2) tile_amax[threadIdx.x] = 0u;
  pdl_wait();
  if (threadIdx.x == 0) prof_stamp_begin(p.prof);
  const int tile = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int t8 = threadIdx.x & 7, lane = threadIdx.x & 31;
  const size_t R = (size_t)p.B * p.N;
  int kv_len = p.kv_len ? p.kv_len[b] : p.N;
  kv_len = min(max(kv_len, 1), p.N);
  uint8_t* st8 = reinterpret_cast<uint8_t*>(stage);
  // task it: unit u = it / 4 (0 q, 1 k, 2 v: uniform per iteration), key (it % 4) * 32 + threadIdx.x / 8
  uint4 raw[12];
#pragma unroll
  for (int it = 0; it < 12; ++it) {
    const int n = tile * 128 + (it & 3) * 32 + (threadIdx.x >> 3);
    const int col = (it >> 2) * p.H * 64 + h * 64 + 8 * t8;
    const int end = it < 4 ? p.N : kv_len;   // q: every row; k, v: the valid keys
    raw[it] = n < end ? *reinterpret_cast<const uint4*>(p.qkv + ((size_t)b * p.N + n) * p.ld_qkv + col)
                      : make_uint4(0u, 0u, 0u, 0u);
  }
  auto unpack = [](const uint4& r, float (&x)[8]) {
    const __nv_bfloat162* v2 = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(v2[i]);
      x[2 * i] = f.x; x[2 * i + 1] = f.y;
    }
  };
  // the tile's k and v amax: per thread, per warp (shuffles), per CTA (atomicMax on the bits: max.NaN order)
  __syncthreads();
#pragma unroll
  for (int u = 1; u < 3; ++u) {
    float amax = 0.f;
#pragma unroll
    for (int it = 4 * u; it < 4 * u + 4; ++it) {
      float x[8];
      unpack(raw[it], x);
#pragma unroll
      for (int i = 0; i < 8; ++i) amax = fmax_nan(amax, fabsf(x[i]));
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) amax = fmax_nan(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if (lane == 0) atomicMax(&tile_amax[u - 1], __float_as_uint(amax));
  }
  __syncthreads();
  float tinv[2], ts[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) ts[u] = e4m3_block_scale(__uint_as_float(tile_amax[u]), tinv[u]);
#pragma unroll
  for (int it = 0; it < 12; ++it) {
    const int u = it >> 2;
    const int key = (it & 3) * 32 + (threadIdx.x >> 3);
    const int n = tile * 128 + key;
    const bool valid = n < p.N;
    const size_t row = (size_t)b * p.N + n;
    float x[8];
    unpack(raw[it], x);
    float s, inv;
    if (u == 0) {   // q: the row's own scale
      float amax = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) amax = fmax_nan(amax, fabsf(x[i]));
      amax = fmax_nan(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
      amax = fmax_nan(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
      amax = fmax_nan(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
      s = e4m3_block_scale(amax, inv);
    } else {
      s = ts[u - 1]; inv = tinv[u - 1];
    }
    const uint32_t c0 = pack_e4m3x4(x[0] * inv, x[1] * inv, x[2] * inv, x[3] * inv);
    const uint32_t c1 = pack_e4m3x4(x[4] * inv, x[5] * inv, x[6] * inv, x[7] * inv);
    if (valid && t8 == 0) p.scale[(size_t)(u * p.H + h) * R + row] = s;
    if (u < 2) {
      if (valid) *reinterpret_cast<uint2*>(p.qk8 + row * p.ld_qk8 + u * p.H * 64 + h * 64 + 8 * t8) = make_uint2(c0, c1);
    } else {
      // padding keys (n >= N) and masked keys (n >= kv_len, read as zero) have zero codes: 0x7F is an e4m3 NaN, and
      // 0 * NaN would pass the mask
      const int pos = (key & ~31) + fp8_vt_pos(key & 31);
#pragma unroll
      for (int i = 0; i < 8; ++i) st8[(8 * t8 + i) * 132 + pos] = n < kv_len ? (uint8_t)(((i < 4 ? c0 : c1) >> (8 * (i & 3))) & 0xFF) : 0;
    }
  }
  __syncthreads();
  // one warp per V^T row of 128 bytes: coalesced 4-byte stores
  uint8_t* vt = p.vt8 + ((size_t)b * p.H * 64 + h * 64) * p.vt_ld + (size_t)tile * 128;
#pragma unroll 1
  for (int r = threadIdx.x >> 5; r < 64; r += 8)
    *reinterpret_cast<uint32_t*>(vt + (size_t)r * p.vt_ld + 4 * lane) = stage[r * 33 + lane];
  __syncthreads();
  if (threadIdx.x == 0) prof_stamp_end(p.prof);
}

struct Fp8AttnParams {
  int B, N, H;
  const int* kv_len;         // [B] valid keys per utterance, or null (= N)
  const float* scale;        // [3H][B*N] scales of Q (per row), K and V (per 128-key tile) (qkv_quant_e4m3_kernel)
  uint8_t* out;              // e4m3 [B*N, ldo bytes]
  int ldo;
  float* scale_out;          // [H][B*N] power-of-two scale per (row, head) of the output
  unsigned long long* prof;  // in-graph timing slot (ptx.cuh prof_stamp_*), or null
};

struct Fp8AttnSmem {
  static constexpr int kStages = 2;
  static constexpr int kQ = 0;                        // 128 x 64 B (SWIZZLE_64B)
  static constexpr int kK = 8192;                     // stages x (128 keys x 64 B, SWIZZLE_64B)
  static constexpr int kV = kK + kStages * 8192;      // stages x (64 d-rows x 128 keys, SWIZZLE_128B)
  static constexpr int kBar = kV + kStages * 8192;
  // q_full, k_full[S], k_empty[S], v_full[S], v_empty[S]
  static constexpr int kNumBars = 1 + 4 * kStages;
  static constexpr int kTotal = kBar + kNumBars * 8 + 1024;   // + align slack
};

__global__ void __launch_bounds__(384, 1)
attn_fp8_kernel(const __grid_constant__ CUtensorMap tma_qk, const __grid_constant__ CUtensorMap tma_vt,
                const Fp8AttnParams p) {
  using S = Fp8AttnSmem;
  constexpr int kS = S::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::kBar);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;
  uint64_t* k_empty = bars + 1 + kS;
  uint64_t* v_full = bars + 1 + 2 * kS;
  uint64_t* v_empty = bars + 1 + 3 * kS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 128;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int HD = p.H * 64;
  const size_t R = (size_t)p.B * p.N;

  if (warp == 0 && elect_one()) {
    tma_prefetch_desc(&tma_qk);
    tma_prefetch_desc(&tma_vt);
    mbar_init(q_full, 1);
    for (int i = 0; i < kS; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 256);   // released by every consumer thread
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 256);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (threadIdx.x == 128) prof_stamp_begin(p.prof);
  int kv_len = p.kv_len ? p.kv_len[b] : p.N;
  kv_len = min(max(kv_len, 1), p.N);
  const int num_kv = (kv_len + 127) >> 7;

  if (warp < 4) {
    // ===================== TMA producer =====================
    if (warp == 0 && elect_one()) {
      mbar_expect_tx(q_full, 8192);
      tma_load_3d(smem + S::kQ, &tma_qk, q_full, h * 64, q0, b);
      for (int j = 0; j < num_kv; ++j) {
        const int s = j % kS;
        const uint32_t ph = (j / kS) & 1;
        mbar_wait(&k_empty[s], ph ^ 1);
        mbar_expect_tx(&k_full[s], 8192);
        tma_load_3d(smem + S::kK + s * 8192, &tma_qk, &k_full[s], HD + h * 64, j * 128, b);
        mbar_wait(&v_empty[s], ph ^ 1);
        mbar_expect_tx(&v_full[s], 8192);
        tma_load_3d(smem + S::kV + s * 8192, &tma_vt, &v_full[s], j * 128, h * 64, b);
      }
    }
  } else {
    // ===================== consumers =====================
    const int wg = (threadIdx.x >> 7) - 1;
    const int rw = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);   // this thread's rows: rw and rw + 8 of the 64
    const int l4 = lane & 3;
    const uint32_t sQ = smem_u32(smem + S::kQ) + wg * (64 * 64);
    constexpr float kLog2e = 1.4426950408889634f;
    // log2 e * the row's q scale (a power of two); the running max m_run is kept in units of the q scale
    float fr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int n = q0 + wg * 64 + rw + 8 * r;
      fr[r] = kLog2e * (n < p.N ? p.scale[(size_t)h * R + (size_t)b * p.N + n] : 1.f);
    }
    // the k and v scales of key tile j sit at its first key; tile j + 1's are requested one tile ahead
    const float* ks = p.scale + (size_t)(p.H + h) * R + (size_t)b * p.N;
    const float* vs = p.scale + (size_t)(2 * p.H + h) * R + (size_t)b * p.N;
    float sk_next = ks[0], sv_next = vs[0];
    float o[32], ot[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { o[i] = 0.f; ot[i] = 0.f; }
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: 2^8 times the sum of p
    mbar_wait(q_full, 0);

    for (int j = 0; j < num_kv; ++j) {
      const int s = j % kS;
      const uint32_t ph = (j / kS) & 1;
      const float sk = sk_next, sv_t = sv_next;
      if (j + 1 < num_kv) { sk_next = ks[(j + 1) * 128]; sv_next = vs[(j + 1) * 128]; }
      // ---- S = Q8 K8^T (64 x 128 codes) ----
      float sv[64];
      mbar_wait(&k_full[s], ph);
      const uint32_t sK = smem_u32(smem + S::kK + s * 8192);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 2; ++k)
        wgmma_e4m3_ss_n128(sv, gmma_desc_sw64(sQ + 32 * k, 16, 512), gmma_desc_sw64(sK + 32 * k, 16, 512), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(sv);
      mbar_arrive(&k_empty[s]);

      // ---- online softmax: sv[i] is (row rw + 8 ((i / 2) % 2), key 8 (i / 4) + 2 (lane % 4) + i % 2), in units of
      // sq * sk ----
      const int kv0 = j * 128;
      if (kv0 + 128 > kv_len) {
#pragma unroll
        for (int i = 0; i < 64; ++i)
          if (kv0 + 8 * (i >> 2) + 2 * l4 + (i & 1) >= kv_len) sv[i] = -INFINITY;
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sv[i]);
      float sc[2], mb[2], fk[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float m_new = fmaxf(m_run[r], mx[r] * sk);   // exact: sk is a power of two
        sc[r] = ex2_approx((m_run[r] - m_new) * fr[r]);    // 0 on the first tile (m_run = -inf)
        m_run[r] = m_new;
        fk[r] = fr[r] * sk;
        mb[r] = m_new * fr[r] - 8.f;                        // e = 2^8 p
        l_run[r] *= sc[r];
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] *= sc[(i >> 1) & 1];
      // P~ = e4m3(2^8 p) as the A fragments of the 4 K-steps (32 keys each): register m of step g holds row
      // rw + 8 (m % 2) and the sv indices 16 g + 8 (m / 2) + 2 (m % 2) + {0, 1, 4, 5}
      uint32_t pa[4][4];
#pragma unroll
      for (int g = 0; g < 4; ++g) {
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int i = 16 * g + 8 * (m >> 1) + 2 * (m & 1), r = m & 1;
          const float e0 = ex2_approx(fmaf(sv[i], fk[r], -mb[r]));
          const float e1 = ex2_approx(fmaf(sv[i + 1], fk[r], -mb[r]));
          const float e2 = ex2_approx(fmaf(sv[i + 4], fk[r], -mb[r]));
          const float e3 = ex2_approx(fmaf(sv[i + 5], fk[r], -mb[r]));
          l_run[r] += (e0 + e1) + (e2 + e3);
          pa[g][m] = pack_e4m3x4(e0, e1, e2, e3);
        }
      }

      // ---- O_t = P~ V8^T (64 x 64) in a fresh accumulator, then o += sv_t 2^-8 ... (2^8 kept in l) ----
      mbar_wait(&v_full[s], ph);
      const uint32_t sV = smem_u32(smem + S::kV + s * 8192);
      wgmma_fence();
#pragma unroll
      for (int g = 0; g < 4; ++g) wgmma_e4m3_rs_n64(ot, pa[g], gmma_desc_sw128(sV + 32 * g, 16, 1024), g != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(ot);
      mbar_arrive(&v_empty[s]);
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = fmaf(sv_t, ot[i], o[i]);
    }

    // ---- epilogue: O / l as block-scaled e4m3, one power-of-two scale per (row, head) ----
    pdl_launch_dependents();
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const float inv[2] = {1.f / l_run[0], 1.f / l_run[1]};
    float qs[2], qinv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float amax = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        amax = fmax_nan(amax, fmax_nan(fabsf(o[4 * c + 2 * r] * inv[r]), fabsf(o[4 * c + 2 * r + 1] * inv[r])));
      amax = fmax_nan(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
      amax = fmax_nan(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
      qs[r] = e4m3_block_scale(amax, qinv[r]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int n = q0 + wg * 64 + rw + 8 * r;
      if (n >= p.N) continue;
      const size_t row = (size_t)b * p.N + n;
      if (l4 == 0) p.scale_out[(size_t)h * R + row] = qs[r];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int col = h * 64 + 8 * c + 2 * l4;
        const float v0 = o[4 * c + 2 * r] * inv[r] * qinv[r], v1 = o[4 * c + 2 * r + 1] * inv[r] * qinv[r];
        uint16_t w;
        asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(w) : "f"(v1), "f"(v0));   // first source -> upper byte
        *reinterpret_cast<uint16_t*>(p.out + row * p.ldo + col) = w;
      }
    }
  }

  __syncthreads();
  if (threadIdx.x == 0) prof_stamp_end(p.prof);
}

}  // namespace f5
