// Launch trace of the DiT, ODE sampler and duration predictor host code, without a GPU.
//
// csrc/dit.cu and csrc/duration.cu contain no kernels: they only decide which launchers run, in which order, with
// which arguments.  Linked against this file instead of the rest of the library, every launcher they call prints
// itself with all of its arguments, and main() runs f5_dit_precompute / f5_dit_forward / f5_ode_sample /
// f5_duration_forward over every mode and binding the forwards distinguish.  The output is the launch sequence those
// entry points issue, so two versions of the host code launch the same work exactly when their traces are equal
// (tests/test_host_launch_trace.py, tests/golden/make_launch_trace.py).
//
// Nothing is dereferenced on the device side, so each pointer field gets a slot of its own in an address range that
// is never touched; a pointer prints as its slot's name plus the byte offset into it (`b.ln_tab+0x1a0`), never as an
// address, and the trace is the same on every build.
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../f5_tts_mlx_b200/csrc/host_common.h"
#include "../../f5_tts_mlx_b200/csrc/launch.h"

namespace {

constexpr int kSlotBits = 36;   // 64 GiB per slot: more than any offset the host code adds to a pointer
std::vector<std::string> g_slots;

struct Slot {
  uintptr_t addr;
  template <typename T> operator T*() const { return reinterpret_cast<T*>(addr); }
};

Slot slot(const std::string& name) {
  g_slots.push_back(name);
  return Slot{(uintptr_t)g_slots.size() << kSlotBits};
}

std::string P(const void* p) {
  if (p == nullptr) return "NULL";
  const uintptr_t a = (uintptr_t)p, i = a >> kSlotBits, off = a & ((uintptr_t(1) << kSlotBits) - 1);
  if (i == 0 || i > g_slots.size()) return "<pointer outside the arena>";
  char buf[32] = "";
  if (off) snprintf(buf, sizeof(buf), "+0x%llx", (unsigned long long)off);
  return g_slots[i - 1] + buf;
}

// one line per call: name(arg=value, ...)
struct Line {
  std::string s;
  bool first = true;
  explicit Line(const char* fn) : s(fn) { s += '('; }
  Line& kv(const char* k, const std::string& v) {
    s += first ? "" : ", ";
    first = false;
    s += k; s += '='; s += v;
    return *this;
  }
  Line& p(const char* k, const void* v) { return kv(k, P(v)); }
  Line& i(const char* k, long long v) { return kv(k, std::to_string(v)); }
  Line& f(const char* k, float v) {
    char buf[32];
    snprintf(buf, sizeof(buf), "%.9g", v);
    return kv(k, buf);
  }
  int done() {
    printf("  %s)\n", s.c_str());
    return 0;
  }
};

}  // namespace

// ---------------- recording stubs of everything dit.o and duration.o link against ----------------
namespace f5 {

int set_error(int code, const char* fmt, ...) {
  char msg[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(msg, sizeof(msg), fmt, ap);
  va_end(ap);
  printf("  set_error(%d, \"%s\")\n", code, msg);
  return code;
}

int device_check() { return Line("device_check").done(); }

int launch_ln_modulate(const float* x, void* y, int rows, int dim, int rows_per_batch, const float* scale,
                       const float* shift, long long mod_batch_stride, int add_one, cudaStream_t st) {
  return Line("launch_ln_modulate").p("x", x).p("y", y).i("rows", rows).i("dim", dim)
      .i("rows_per_batch", rows_per_batch).p("scale", scale).p("shift", shift).i("mod_batch_stride", mod_batch_stride)
      .i("add_one", add_one).p("st", st).done();
}

int launch_dwconv7_ln(const float* x, void* y, int B, int N, int C, const float* wt, const float* wb, const float* ln_w,
                      const float* ln_b, cudaStream_t st) {
  return Line("launch_dwconv7_ln").p("x", x).p("y", y).i("B", B).i("N", N).i("C", C).p("wt", wt).p("wb", wb)
      .p("ln_w", ln_w).p("ln_b", ln_b).p("st", st).done();
}

int launch_grn(const void* h, void* y, float* nx_scratch, const float* gamma, const float* beta, int B, int N, int C,
               cudaStream_t st, const int* valid_len) {
  return Line("launch_grn").p("h", h).p("y", y).p("nx_scratch", nx_scratch).p("gamma", gamma).p("beta", beta)
      .i("B", B).i("N", N).i("C", C).p("st", st).p("valid_len", valid_len).done();
}

int launch_text_embed_gather(const int* text, int B, int nt, int N, int C, const float* emb, const float* pos_table,
                             int max_pos, float* x, int Bout, int drop_from, cudaStream_t st, int mask_padding,
                             const int* valid_len) {
  return Line("launch_text_embed_gather").p("text", text).i("B", B).i("nt", nt).i("N", N).i("C", C).p("emb", emb)
      .p("pos_table", pos_table).i("max_pos", max_pos).p("x", x).i("Bout", Bout).i("drop_from", drop_from)
      .p("st", st).i("mask_padding", mask_padding).p("valid_len", valid_len).done();
}

int launch_time_mlp(const float* tvals, int T, int D, const float* w0, const float* b0, const float* w2,
                    const float* b2, float* t_emb, void* silu_bf16, cudaStream_t st) {
  return Line("launch_time_mlp").p("tvals", tvals).i("T", T).i("D", D).p("w0", w0).p("b0", b0).p("w2", w2)
      .p("b2", b2).p("t_emb", t_emb).p("silu_bf16", silu_bf16).p("st", st).done();
}

int launch_ode_update(const OdeUpdateParams& u, cudaStream_t st) {
  return Line("launch_ode_update").p("v", u.v).i("ldv", u.ldv).i("null_row_offset", u.null_row_offset)
      .f("cfg_strength", u.cfg_strength).p("y_base", u.y_base).p("y_out", u.y_out).f("a", u.a).p("k_acc", u.k_acc)
      .f("acc_w", u.acc_w).i("acc_init", u.acc_init).i("use_acc", u.use_acc).p("y_bf16", u.y_bf16)
      .i("ld_bf16", u.ld_bf16).i("bf16_copy_row_offset", u.bf16_copy_row_offset).i("rows", u.rows).i("d", u.d)
      .p("st", st).done();
}

int launch_cast_pad_bf16(const float* src, int d, void* dst, int ld, int rows, long long copy_row_offset,
                         cudaStream_t st) {
  return Line("launch_cast_pad_bf16").p("src", src).i("d", d).p("dst", dst).i("ld", ld).i("rows", rows)
      .i("copy_row_offset", copy_row_offset).p("st", st).done();
}

int launch_concat_cond_text(const float* cond, int dc, int Bc, int N, const float* text, int dt, void* dst, int ld,
                            int rows, int drop_from_row, cudaStream_t st, const int* cond_len) {
  return Line("launch_concat_cond_text").p("cond", cond).i("dc", dc).i("Bc", Bc).i("N", N).p("text", text).i("dt", dt)
      .p("dst", dst).i("ld", ld).i("rows", rows).i("drop_from_row", drop_from_row).p("st", st).p("cond_len", cond_len)
      .done();
}

int launch_ln_tab_prep(const float* mod, void* prep_bf16, int T, int L, int D, int NM, cudaStream_t st) {
  return Line("launch_ln_tab_prep").p("mod", mod).p("prep_bf16", prep_bf16).i("T", T).i("L", L).i("D", D)
      .i("NM", NM).p("st", st).done();
}

int launch_duration_head(const float* x, int B, int N, int D, const int* len, const float* norm_w, const float* pred_w,
                         float* out, cudaStream_t st) {
  return Line("launch_duration_head").p("x", x).i("B", B).i("N", N).i("D", D).p("len", len).p("norm_w", norm_w)
      .p("pred_w", pred_w).p("out", out).p("st", st).done();
}

}  // namespace f5

// Every field of f5_gemm_args in declaration order.  A field that is zero (all bits) is left out: the host code
// builds the struct from a zeroed one, so the line still determines every field.
extern "C" int f5_gemm_bf16(const f5_gemm_args* g, void* st) {
  Line l("f5_gemm_bf16");
  auto p = [&](const char* k, const void* v) { if (v) l.p(k, v); };
  auto i = [&](const char* k, long long v) { if (v) l.i(k, v); };
  auto f = [&](const char* k, float v) { uint32_t bits; memcpy(&bits, &v, 4); if (bits) l.f(k, v); };
  p("a", g->a); i("lda", g->lda); p("w", g->w); i("ldw", g->ldw);
  i("m", g->m); i("n", g->n); i("k", g->k);
  i("rows_per_batch", g->rows_per_batch); i("num_batches", g->num_batches); i("batched_tiles", g->batched_tiles);
  i("conv_taps", g->conv_taps); i("conv_pad", g->conv_pad); i("conv_grouped", g->conv_grouped);
  i("act", g->act); i("out_bf16", g->out_bf16); p("bias", g->bias); p("out", g->out); i("ldo", g->ldo);
  p("resid", g->resid); i("ldr", g->ldr); p("gate", g->gate); p("row_len", g->row_len);
  p("rope", g->rope); i("rope_cols", g->rope_cols); f("q_scale", g->q_scale); i("q_cols", g->q_cols);
  i("tile_n", g->tile_n); p("out2_bf16", g->out2_bf16); i("ldo2", g->ldo2); i("w_static", g->w_static);
  p("prefetch", g->prefetch); i("prefetch_bytes", g->prefetch_bytes);
  p("ln_scale", g->ln_scale); p("ln_stats", g->ln_stats); p("ln_in_stats", g->ln_in_stats); p("ln_tab", g->ln_tab);
  i("ln_tab_ld", g->ln_tab_ld);
  i("ab_fp8", g->ab_fp8); i("out2_fp8", g->out2_fp8); f("acc_scale", g->acc_scale); i("out_fp8", g->out_fp8);
  p("a_scale", g->a_scale); i("a_scale_ld", g->a_scale_ld); p("w_scale", g->w_scale); p("out_scale", g->out_scale);
  p("out2_scale", g->out2_scale);
  return l.p("st", st).done();
}

extern "C" int f5_attention_fwd(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch,
                                int32_t frames, int32_t heads, int32_t head_dim, const int32_t* kv_len, void* st) {
  return Line("f5_attention_fwd").p("qkv", qkv).i("ld_qkv", ld_qkv).p("out", out).i("ld_out", ld_out)
      .i("batch", batch).i("frames", frames).i("heads", heads).i("head_dim", head_dim).p("kv_len", kv_len)
      .p("st", st).done();
}

extern "C" int f5_attention_fwd_e4m3(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch,
                                     int32_t frames, int32_t heads, int32_t head_dim, const int32_t* kv_len, void* st) {
  return Line("f5_attention_fwd_e4m3").p("qkv", qkv).i("ld_qkv", ld_qkv).p("out", out).i("ld_out", ld_out)
      .i("batch", batch).i("frames", frames).i("heads", heads).i("head_dim", head_dim).p("kv_len", kv_len)
      .p("st", st).done();
}

extern "C" int f5_attention_fwd_e4m3_scaled(const void* qkv, int64_t ld_qkv, void* out, int64_t ld_out, int32_t batch,
                                            int32_t frames, int32_t heads, int32_t head_dim, const int32_t* kv_len,
                                            float* scale_out, void* st) {
  return Line("f5_attention_fwd_e4m3_scaled").p("qkv", qkv).i("ld_qkv", ld_qkv).p("out", out).i("ld_out", ld_out)
      .i("batch", batch).i("frames", frames).i("heads", heads).i("head_dim", head_dim).p("kv_len", kv_len)
      .p("scale_out", scale_out).p("st", st).done();
}

extern "C" int f5_qkv_quant_e4m3_masked(const void* qkv, int64_t ld_qkv, void* qk8, int64_t ld_qk8, void* vt8,
                                        int64_t vt_ld, float* qkv_scale, int32_t batch, int32_t frames, int32_t heads,
                                        const int32_t* kv_len, void* st) {
  return Line("f5_qkv_quant_e4m3_masked").p("qkv", qkv).i("ld_qkv", ld_qkv).p("qk8", qk8).i("ld_qk8", ld_qk8)
      .p("vt8", vt8).i("vt_ld", vt_ld).p("qkv_scale", qkv_scale).i("batch", batch).i("frames", frames)
      .i("heads", heads).p("kv_len", kv_len).p("st", st).done();
}

extern "C" int f5_attention_fwd_fp8(const void* qk8, int64_t ld_qk8, const void* vt8, int64_t vt_ld,
                                    const float* qkv_scale, void* out, int64_t ld_out, int32_t batch, int32_t frames,
                                    int32_t heads, int32_t head_dim, const int32_t* kv_len, float* scale_out,
                                    void* st) {
  return Line("f5_attention_fwd_fp8").p("qk8", qk8).i("ld_qk8", ld_qk8).p("vt8", vt8).i("vt_ld", vt_ld)
      .p("qkv_scale", qkv_scale).p("out", out).i("ld_out", ld_out).i("batch", batch).i("frames", frames)
      .i("heads", heads).i("head_dim", head_dim).p("kv_len", kv_len).p("scale_out", scale_out).p("st", st).done();
}

// ---------------- the cases ----------------
namespace {

enum Mode { BF16, FUSED, FP8, BLK8, ATTN8, NMODES };
const char* kModeName[NMODES] = {"bf16", "fused-adaln", "fp8", "block-fp8", "block-fp8+fp8-attention"};

constexpr int kDim = 256, kHeads = 4, kDepth = 2, kFF = 512, kMel = 100, kText = 128, kTextInner = 256, kConv = 2;
constexpr int kBatch = 2;
// per utterance: 48 rows stay below the weight-prefetch cutoff of 16384 rows at either CFG setting, 8200 above it
constexpr int kFrames[2] = {48, 8200};

void* const kStream = slot("stream");

f5_convnext_weights convnext(const std::string& pre) {
  f5_convnext_weights c;
#define F(x) c.x = slot(pre + #x)
  F(dw_w); F(dw_b); F(ln_w); F(ln_b); F(pw1_w); F(pw1_b); F(grn_gamma); F(grn_beta); F(pw2_w); F(pw2_b);
#undef F
  return c;
}

// every pointer bound; fp8 / block-scaled fields are cleared per mode by weights_for()
f5_dit_block_weights block(const std::string& pre, int l) {
  f5_dit_block_weights k;
#define F(x) k.x = slot(pre + #x)
  F(qkv_w); F(qkv_b); F(out_w); F(out_b); F(ff1_w); F(ff1_b); F(ff2_w); F(ff2_b);
  F(qkv_w8); F(ff1_w8); F(out_w8); F(ff2_w8); F(qkv_ws); F(ff1_ws); F(out_ws); F(ff2_ws);
#undef F
  // distinct per-tensor scales, so that the trace shows which tensor's scale a GEMM got
  k.qkv_s8 = 0.5f + l; k.ff1_s8 = 0.25f + l; k.out_s8 = 0.125f + l; k.ff2_s8 = 0.0625f + l;
  return k;
}

struct Dit {
  f5_convnext_weights text_blocks[kConv];
  f5_dit_block_weights full[kDepth], blocks[kDepth];
  f5_dit_weights w;
  f5_dit_buffers all;   // every buffer bound
};

Dit* make_dit() {
  Dit* d = new Dit();
  for (int l = 0; l < kConv; ++l) d->text_blocks[l] = convnext("w.text_blocks[" + std::to_string(l) + "].");
  for (int l = 0; l < kDepth; ++l) d->full[l] = block("w.blocks[" + std::to_string(l) + "].", l);
  f5_dit_weights& w = d->w;
  memset(&w, 0, sizeof(w));
  w.dim = kDim; w.depth = kDepth; w.heads = kHeads; w.ff_inner = kFF; w.mel_dim = kMel;
  w.text_dim = kText; w.text_inner = kTextInner; w.conv_layers = kConv;
  w.text_rows = 41; w.text_max_pos = 4096; w.ct_ld = 256;
#define F(x) w.x = slot("w." #x)
  F(time_w0); F(time_b0); F(time_w2); F(time_b2); F(text_emb); F(text_pos); F(in_x_w); F(in_ct_w); F(in_b);
  F(conv_w[0]); F(conv_w[1]); F(conv_b[0]); F(conv_b[1]); F(mod_w); F(mod_b); F(proj_w); F(proj_b);
#undef F
  w.text_blocks = d->text_blocks;
  w.blocks = d->blocks;
  f5_dit_buffers& b = d->all;
  memset(&b, 0, sizeof(b));
#define F(x) b.x = slot("b." #x)
  F(text); F(text_len); F(seq_len); F(cond); F(tvals); F(rope); F(hoist); F(mod_table); F(text_x); F(text_a);
  F(text_h); F(text_g); F(grn_nx); F(ct_bf16); F(silu_t); F(y_bf16); F(x); F(h); F(a_bf16); F(c_bf16); F(qkv_bf16);
  F(ff_bf16); F(v); F(ln_stats); F(ln_tab); F(ln_prep); F(valid_len); F(a_fp8); F(a_fp8_scale); F(attn_scale);
  F(ff_scale); F(qk_fp8); F(vt_fp8); F(qkv_scale);
#undef F
  return d;
}

// the block weights a packer binds for `mode`: e4m3 copies from FP8 on, per-channel scales from block-scaled FP8 on
void weights_for(Dit* d, Mode mode) {
  for (int l = 0; l < kDepth; ++l) {
    f5_dit_block_weights& k = d->blocks[l];
    k = d->full[l];
    if (mode < FP8) k.qkv_w8 = k.ff1_w8 = k.out_w8 = k.ff2_w8 = nullptr;
    if (mode < BLK8) k.qkv_ws = k.ff1_ws = k.out_ws = k.ff2_ws = nullptr;
  }
}

// the buffers a session binds for `mode`
f5_dit_buffers buffers_for(const Dit* d, Mode mode, int cfg, int drop_flags, bool seq_len, bool valid_len, int frames,
                           int n_times) {
  f5_dit_buffers b = d->all;
  b.batch = kBatch; b.frames = frames; b.cfg = cfg; b.n_times = n_times; b.text_len_max = 24;
  b.drop_flags = drop_flags;
  if (!seq_len) b.seq_len = nullptr;
  if (!valid_len) b.valid_len = nullptr;
  if (mode < FUSED) b.ln_stats = nullptr, b.ln_tab = nullptr, b.ln_prep = nullptr;
  if (mode < FP8) b.a_fp8 = nullptr;
  if (mode < BLK8) b.a_fp8_scale = b.attn_scale = b.ff_scale = nullptr;
  if (mode < ATTN8) b.qk_fp8 = b.vt_fp8 = nullptr, b.qkv_scale = nullptr;
  return b;
}

const char* bound(const void* p) { return p ? "bound" : "NULL"; }

void dit_cases(Dit* d) {
  for (int mode = 0; mode < NMODES; ++mode) {
    weights_for(d, (Mode)mode);
    // CFG on, or off with each drop_flags value
    for (int cd = 0; cd < 5; ++cd) {
      const int cfg = cd == 0, drop = cd == 0 ? 0 : cd - 1;
      for (int seq = 1; seq >= 0; --seq)
        for (int valid = 1; valid >= 0; --valid)
          for (int frames : kFrames) {
            const f5_dit_buffers b = buffers_for(d, (Mode)mode, cfg, drop, seq, valid, frames, 3);
            printf("== dit mode=%s cfg=%d drop_flags=%d seq_len=%s valid_len=%s batch=%d frames=%d\n",
                   kModeName[mode], cfg, drop, bound(b.seq_len), bound(b.valid_len), b.batch, frames);
            printf("f5_dit_precompute -> %d\n", f5_dit_precompute(&d->w, &b, kStream));
            printf("f5_dit_forward(time_index=1) -> %d\n", f5_dit_forward(&d->w, &b, 1, kStream));
          }
    }
  }
}

void ode_cases(Dit* d) {
  const float grid[3] = {0.f, 0.375f, 1.f};
  weights_for(d, FUSED);
  for (int method = 0; method < 3; ++method) {
    const int per = method == 0 ? 1 : (method == 1 ? 2 : 4);
    for (int cfg = 1; cfg >= 0; --cfg) {
      const f5_dit_buffers b = buffers_for(d, FUSED, cfg, 0, true, false, kFrames[0], 2 * per);
      const bool traj = method != 1;   // the midpoint run updates y in place
      printf("== ode method=%d cfg=%d trajectory=%s mode=%s frames=%d\n", method, cfg, traj ? "bound" : "NULL",
             kModeName[FUSED], b.frames);
      const int rc = f5_ode_sample(&d->w, &b, grid, 3, method, cfg ? 2.f : 0.f, slot("y"),
                                   traj ? (float*)slot("trajectory") : nullptr, slot("scratch"), kStream);
      printf("f5_ode_sample -> %d\n", rc);
    }
  }
}

// partly bound modes: f5_dit_forward refuses each of them before launching anything
void rejected_cases(Dit* d) {
  struct Case {
    const char* what;
    Mode mode;
    void (*edit)(f5_dit_buffers&, f5_dit_block_weights*);
  };
  const Case cases[] = {
      {"fused AdaLN without ln_prep", FUSED, [](f5_dit_buffers& b, f5_dit_block_weights*) { b.ln_prep = nullptr; }},
      {"fused AdaLN with ln_stats only", FUSED,
       [](f5_dit_buffers& b, f5_dit_block_weights*) { b.ln_tab = nullptr; b.ln_prep = nullptr; }},
      {"FP8 without the fused AdaLN buffers", FP8,
       [](f5_dit_buffers& b, f5_dit_block_weights*) { b.ln_stats = b.ln_tab = nullptr; b.ln_prep = nullptr; }},
      {"block-scaled FP8 without a_fp8", BLK8, [](f5_dit_buffers& b, f5_dit_block_weights*) { b.a_fp8 = nullptr; }},
      {"block-scaled FP8 without attn_scale", BLK8,
       [](f5_dit_buffers& b, f5_dit_block_weights*) { b.attn_scale = nullptr; }},
      {"FP8 attention without vt_fp8", ATTN8, [](f5_dit_buffers& b, f5_dit_block_weights*) { b.vt_fp8 = nullptr; }},
      {"FP8 attention in the per-tensor FP8 mode", FP8, [](f5_dit_buffers& b, f5_dit_block_weights*) {
         b.qk_fp8 = slot("b.qk_fp8"); b.vt_fp8 = slot("b.vt_fp8"); b.qkv_scale = slot("b.qkv_scale");
       }},
      {"FP8 without blocks[1].ff2_w8", FP8, [](f5_dit_buffers&, f5_dit_block_weights* k) { k[1].ff2_w8 = nullptr; }},
      {"per-tensor FP8 on per-channel weights", FP8,
       [](f5_dit_buffers&, f5_dit_block_weights* k) { k[0].out_ws = slot("w.blocks[0].out_ws"); }},
      {"block-scaled FP8 without blocks[1].out_ws", BLK8,
       [](f5_dit_buffers&, f5_dit_block_weights* k) { k[1].out_ws = nullptr; }},
  };
  for (const Case& c : cases) {
    weights_for(d, c.mode);
    f5_dit_buffers b = buffers_for(d, c.mode, 1, 0, true, true, kFrames[0], 3);
    c.edit(b, d->blocks);
    printf("== rejected: %s\n", c.what);
    printf("f5_dit_forward(time_index=1) -> %d\n", f5_dit_forward(&d->w, &b, 1, kStream));
  }
}

void duration_case() {
  f5_convnext_weights tb[kConv];
  f5_dit_block_weights blocks[kDepth];
  for (int l = 0; l < kConv; ++l) tb[l] = convnext("dw.text_blocks[" + std::to_string(l) + "].");
  for (int l = 0; l < kDepth; ++l) {
    blocks[l] = block("dw.blocks[" + std::to_string(l) + "].", l);
    blocks[l].qkv_w8 = blocks[l].ff1_w8 = blocks[l].out_w8 = blocks[l].ff2_w8 = nullptr;
    blocks[l].qkv_ws = blocks[l].ff1_ws = blocks[l].out_ws = blocks[l].ff2_ws = nullptr;
  }
  f5_duration_weights w;
  memset(&w, 0, sizeof(w));
  w.dim = kDim; w.depth = kDepth; w.heads = kHeads; w.ff_inner = kFF; w.mel_dim = kMel;
  w.text_dim = kText; w.text_inner = kTextInner; w.conv_layers = kConv;
  w.text_rows = 41; w.text_max_pos = 4096; w.ct_ld = 256;
#define F(x) w.x = slot("dw." #x)
  F(text_emb); F(text_pos); F(in_w); F(in_b); F(conv_w[0]); F(conv_w[1]); F(conv_b[0]); F(conv_b[1]); F(zeros);
  F(norm_w); F(pred_w);
#undef F
  w.text_blocks = tb;
  w.blocks = blocks;
  f5_duration_buffers b;
  memset(&b, 0, sizeof(b));
  b.batch = kBatch; b.frames = 90; b.text_len_max = 30;
#define F(x) b.x = slot("db." #x)
  F(text); F(lens); F(inp); F(rope); F(text_x); F(text_a); F(text_h); F(text_g); F(grn_nx); F(ct_bf16); F(x); F(h);
  F(a_bf16); F(c_bf16); F(qkv_bf16); F(ff_bf16); F(out);
#undef F
  printf("== duration batch=%d frames=%d\n", b.batch, b.frames);
  printf("f5_duration_forward -> %d\n", f5_duration_forward(&w, &b, kStream));
}

}  // namespace

int main() {
  Dit* d = make_dit();
  dit_cases(d);
  ode_cases(d);
  rejected_cases(d);
  duration_case();
  return 0;
}
