// Host launcher + C-ABI entry for the wgmma GEMM (see gemm_sm90.cuh and include/f5_b200.h).
#include <stdlib.h>

#include "gemm_sm90.cuh"
#include "host_common.h"

namespace f5 {

template <int BN, int kStages, int ACT, bool OUT_BF16, bool ROPE, bool FP8, bool RESID = true>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const CUtensorMap& to2,
                       const GemmParams& p, dim3 grid, cudaStream_t stream) {
  using S = GemmSmem<BN, kStages>;
  auto kern = gemm_bf16_tn_kernel<BN, kStages, ACT, OUT_BF16, ROPE, FP8, RESID>;
  static SmemAttrOnce once;  // per instantiation
  F5_CHECK_CUDA(ensure_dyn_smem(once, kern, S::kTotal));
  const double taps = p.conv_taps;
  ProfScope ps(PROF_GEMM, 2.0 * p.M * (double)p.N * (double)p.k_per_tap * taps,
               2.0 * ((double)p.M * p.k_per_tap + (double)p.N * p.k_per_tap * taps) +
                   (double)p.M * p.N * (OUT_BF16 ? 2.0 : 4.0),
               stream);
  GemmParams q = p;
  q.prof = ps.slot;
  F5_CHECK_CUDA(launch_kernel(kern, dim3(grid), dim3(GemmEpi<BN>::kThreads), S::kTotal, stream, ta, tb, to, to2, q));
  F5_CHECK_CUDA(cudaGetLastError());
  return 0;
}

template <int BN, int kStages>
static int dispatch_epi(int act, bool out_bf16, bool rope, const CUtensorMap& ta,
                        const CUtensorMap& tb, const CUtensorMap& to, const CUtensorMap& to2, const GemmParams& p,
                        dim3 grid, cudaStream_t stream) {
  const bool fp8 = p.ab8 || p.out_fp8 || p.out2_fp8;     // e4m3 features: separate instantiations (what the FP8 mode of the DiT uses)
  // residual-free GELU epilogue (FF1): no residual tiles in the epilogue's registers
  if (p.resid == nullptr && act == ACT_GELU_TANH && out_bf16 && !rope) {
    if (fp8) return launch_gemm<BN, kStages, ACT_GELU_TANH, true, false, true, false>(ta, tb, to, to2, p, grid, stream);
    return launch_gemm<BN, kStages, ACT_GELU_TANH, true, false, false, false>(ta, tb, to, to2, p, grid, stream);
  }
#define F5_CASE8(A, O, R) \
  if (fp8 && act == A && out_bf16 == O && rope == R) return launch_gemm<BN, kStages, A, O, R, true>(ta, tb, to, to2, p, grid, stream);
  F5_CASE8(ACT_NONE, true, true)
  F5_CASE8(ACT_NONE, true, false)
  F5_CASE8(ACT_NONE, false, false)
  F5_CASE8(ACT_GELU_TANH, true, false)
  F5_CASE8(ACT_MISH, false, false)
#undef F5_CASE8
  if (fp8) return set_error(F5_ERR_INVALID, "f5_gemm_bf16: FP8 features are not built for epilogue act=%d out_bf16=%d rope=%d", act, (int)out_bf16, (int)rope);
#define F5_CASE(A, O, R) \
  if (act == A && out_bf16 == O && rope == R) return launch_gemm<BN, kStages, A, O, R, false>(ta, tb, to, to2, p, grid, stream);
  F5_CASE(ACT_NONE, true, true)
  F5_CASE(ACT_NONE, true, false)
  F5_CASE(ACT_NONE, false, false)
  F5_CASE(ACT_GELU_TANH, true, false)
  F5_CASE(ACT_GELU_ERF, true, false)
  F5_CASE(ACT_MISH, true, false)
  F5_CASE(ACT_MISH, false, false)
#undef F5_CASE
  return set_error(F5_ERR_INVALID, "f5_gemm_bf16: unsupported epilogue act=%d out_bf16=%d rope=%d",
                   act, (int)out_bf16, (int)rope);
}

}  // namespace f5

// Debug aid: give successive f5_gemm_bf16 calls consecutive slices of a timestamp buffer, so the
// per-CTA phase timelines of every GEMM of a (graph-captured) step can be read back in situ.
static char* g_ts_base = nullptr;
static long long g_ts_stride = 0;
static int g_ts_max = 0, g_ts_idx = 0;
extern "C" int f5_debug_gemm_ts(void* base, int64_t stride_bytes, int32_t max_calls) {
  g_ts_base = reinterpret_cast<char*>(base);
  g_ts_stride = stride_bytes;
  g_ts_max = max_calls;
  g_ts_idx = 0;
  return 0;
}

extern "C" int f5_gemm_bf16(const f5_gemm_args* a_in, void* stream_) {
  using namespace f5;
  if (int e = device_check()) return e;
  F5_REQUIRE(a_in != nullptr, "f5_gemm_bf16: null args");
  f5_gemm_args a_copy = *a_in;
  if (g_ts_base && g_ts_idx < g_ts_max && a_copy.debug_ts == nullptr)
    a_copy.debug_ts = g_ts_base + (long long)(g_ts_idx++) * g_ts_stride;
  const f5_gemm_args* a = &a_copy;
  F5_REQUIRE(a != nullptr, "f5_gemm_bf16: null args");
  F5_REQUIRE(a->a && a->w && a->out, "f5_gemm_bf16: null operand pointer");
  F5_REQUIRE(a->m > 0 && a->n > 0 && a->k > 0, "f5_gemm_bf16: bad shape m=%d n=%d k=%d", a->m,
             a->n, a->k);
  F5_REQUIRE(a->lda % 8 == 0 && a->ldw % 8 == 0, "f5_gemm_bf16: lda/ldw must be multiples of 8");
  const bool ab8 = a->ab_fp8 != 0;
  if (ab8) {
    F5_REQUIRE(a->lda % 16 == 0 && a->ldw % 16 == 0 && a->k % 128 == 0 && a->acc_scale > 0.f,
               "f5_gemm_bf16: FP8 mode needs lda/ldw %% 16 == 0, k %% 128 == 0 and acc_scale > 0");
    F5_REQUIRE((a->conv_taps <= 1) && !a->conv_grouped, "f5_gemm_bf16: FP8 mode is for plain GEMMs");
  }
  const int esz = ab8 ? 1 : 2;       // operand element size
  const uint32_t kbox = ab8 ? 128 : 64;
  F5_REQUIRE(a->n % (a->out_bf16 ? 8 : 4) == 0, "f5_gemm_bf16: n=%d not vector aligned", a->n);
  F5_REQUIRE(a->ldo % (a->out_bf16 ? 8 : 4) == 0, "f5_gemm_bf16: ldo not vector aligned");
  const int taps = a->conv_taps > 0 ? a->conv_taps : 1;
  const int nb = a->num_batches > 0 ? a->num_batches : 1;
  const int rpb = a->rows_per_batch > 0 ? a->rows_per_batch : a->m;
  const bool batched = a->batched_tiles != 0;
  F5_REQUIRE(taps == 1 || batched, "f5_gemm_bf16: conv mode requires batched_tiles");
  F5_REQUIRE(!a->conv_grouped || a->k == 64, "f5_gemm_bf16: grouped conv needs k == 64");
  F5_REQUIRE((int64_t)nb * rpb == a->m, "f5_gemm_bf16: m=%d != num_batches*rows_per_batch=%d*%d",
             a->m, nb, rpb);
  if (a->rope) {
    F5_REQUIRE(a->rope_cols % 64 == 0 && a->q_cols % 32 == 0, "f5_gemm_bf16: rope_cols/q_cols");
    F5_REQUIRE(a->act == F5_ACT_NONE && a->out_bf16, "f5_gemm_bf16: rope epilogue is bf16/no-act");
  }
  if (a->ln_scale) {   // fused-LN producer mode
    F5_REQUIRE(!a->out_bf16 && a->out2_bf16 && a->ln_stats, "f5_gemm_bf16: ln_scale needs an fp32 out, out2_bf16 and ln_stats");
    F5_REQUIRE(a->n % 64 == 0 && !a->rope, "f5_gemm_bf16: ln_scale needs n %% 64 == 0");
  }
  if (a->ln_in_stats) {   // fused-LN consumer mode
    F5_REQUIRE(a->ln_tab && a->ln_tab_ld >= a->n && !a->out2_bf16 && taps == 1 && a->k % 128 == 0,
               "f5_gemm_bf16: ln_in_stats needs ln_tab (ld >= n), no second output, a plain GEMM with k %% 128 == 0");
  }
  if (a->resid) F5_REQUIRE(a->ldr % 4 == 0, "f5_gemm_bf16: ldr not multiple of 4");
  if (a->gate) F5_REQUIRE(a->gate_ld % 4 == 0, "f5_gemm_bf16: gate_ld not multiple of 4");

  // output tensor maps (TMA stores of the epilogue): (cols, rows per utterance, utterances) when tiles never straddle
  // utterances, else (cols, m, 1)
  CUtensorMap to, to2;
  {
    const uint64_t orows = batched ? (uint64_t)rpb : (uint64_t)a->m, obat = batched ? (uint64_t)nb : 1;
    F5_REQUIRE(!a->out_fp8 || (a->out_bf16 && a->ldo % 16 == 0), "f5_gemm_bf16: out_fp8 needs out_bf16 = 1 and ldo %% 16 == 0");
    if (int e = make_tmap_out(&to, a->out, a->out_fp8 ? 1 : (a->out_bf16 ? 2 : 4), (uint64_t)a->n, orows, obat, (uint64_t)a->ldo)) return e;
    if (a->out2_bf16) {
      F5_REQUIRE(!a->out_bf16, "f5_gemm_bf16: out2_bf16 needs an fp32 out");
      if (int e = make_tmap_out(&to2, a->out2_bf16, a->out2_fp8 ? 1 : 2, (uint64_t)a->n, orows, obat, (uint64_t)a->ldo2)) return e;
    } else {
      to2 = to;
    }
  }

  // tile width: 64 or 128 columns.  `variant` selects nothing on sm_90 (there is one kernel family); wider tile
  // requests (192, 256) get the widest tile there is.
  F5_REQUIRE(a->variant >= 0 && a->variant <= 2, "f5_gemm_bf16: variant must be 0, 1 or 2");
  F5_REQUIRE(a->tile_n == 0 || a->tile_n == 64 || a->tile_n == 128 || a->tile_n == 192 || a->tile_n == 256,
             "f5_gemm_bf16: tile_n must be 0, 64, 128, 192 or 256");
  int bn = a->tile_n > 128 ? 128 : a->tile_n;
  if (a->conv_grouped) bn = 64;
  if (bn == 0) {
    // fill the SMs: prefer 128-wide tiles unless that leaves most SMs idle
    const int mt = batched ? nb * cdiv(rpb, 128) : cdiv(a->m, 128);
    bn = (mt * cdiv(a->n, 128) >= (sm_count() * 13) / 16 || a->n <= 64) ? 128 : 64;
    if (a->n <= 64) bn = 64;
  }

  GemmParams p;
  p.M = a->m; p.N = a->n; p.K = a->k;
  p.rows_per_batch = rpb;
  p.tiles_per_batch = batched ? cdiv(rpb, 128) : 0;
  p.num_batches = nb;
  p.conv_taps = taps;
  p.conv_pad = a->conv_pad;
  p.k_per_tap = a->k;
  p.conv_grouped = a->conv_grouped;
  p.bias = a->bias;
  p.out = a->out; p.ldo = (int)a->ldo;
  p.resid = a->resid; p.ldr = (int)a->ldr;
  p.gate = a->gate; p.gate_ld = (int)a->gate_ld;
  p.row_len = a->row_len;
  p.rope = reinterpret_cast<const float2*>(a->rope);
  p.rope_cols = a->rope_cols;
  p.q_scale = a->q_scale;
  p.q_cols = a->q_cols;
  p.out2 = reinterpret_cast<__nv_bfloat16*>(a->out2_bf16);
  p.ldo2 = (int)a->ldo2;
  p.ts = reinterpret_cast<unsigned long long*>(a->debug_ts);
  p.w_static = a->w_static;
  p.pf_ptr = reinterpret_cast<const char*>(a->prefetch); p.pf_bytes = a->prefetch_bytes;
  p.ln_scale = a->ln_scale; p.ln_stats = reinterpret_cast<float2*>(a->ln_stats);
  p.ln_in_stats = reinterpret_cast<const float2*>(a->ln_in_stats); p.ln_in_units = a->k / 64;
  p.ln_tab = a->ln_tab; p.ln_tab_ld = a->ln_tab_ld;
  p.ab8 = ab8 ? 1 : 0; p.acc_scale = ab8 ? a->acc_scale : 1.f; p.out2_fp8 = a->out2_fp8; p.out_fp8 = a->out_fp8;
  if (a->out2_bf16) F5_REQUIRE(a->ldo2 % 8 == 0 && a->n % 8 == 0, "f5_gemm_bf16: out2 alignment");

  // A: (channels, frames, utterances); flat mode is one "utterance" of m rows
  CUtensorMap ta, tb;
  {
    const int kcols = a->conv_grouped ? a->n : a->k;  // grouped: channel axis spans all groups
    uint64_t dims[3] = {(uint64_t)kcols, (uint64_t)(batched ? rpb : a->m),
                        (uint64_t)(batched ? nb : 1)};
    uint64_t str[2] = {(uint64_t)a->lda * esz, (uint64_t)a->lda * esz * (uint64_t)rpb};
    uint32_t box[3] = {kbox, 128, 1};
    if (int e = (ab8 ? make_tmap_u8 : make_tmap_bf16)(&ta, a->a, 3, dims, str, box)) return e;
  }
  {
    const int kpad = cdiv(a->k, 64) * 64;
    uint64_t dims[2] = {(uint64_t)(taps == 1 ? a->k : taps * kpad), (uint64_t)a->n};
    uint64_t str[1] = {(uint64_t)a->ldw * esz};
    uint32_t box[2] = {kbox, (uint32_t)bn};
    if (int e = (ab8 ? make_tmap_u8 : make_tmap_bf16)(&tb, a->w, 2, dims, str, box)) return e;
  }
  dim3 grid(cdiv(a->n, bn), batched ? nb * cdiv(rpb, 128) : cdiv(a->m, 128), 1);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const bool rope = a->rope != nullptr;
  if (bn == 128) return dispatch_epi<128, 4>(a->act, a->out_bf16 != 0, rope, ta, tb, to, to2, p, grid, stream);
  return dispatch_epi<64, 6>(a->act, a->out_bf16 != 0, rope, ta, tb, to, to2, p, grid, stream);
}
