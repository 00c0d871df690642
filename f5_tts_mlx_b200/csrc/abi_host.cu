// Host-side completion of the C ABI for hosts that are not Python (include/f5_b200.h, "host utilities"):
//   * the packed weight buffer: size, packing from MLX-named fp32 tensors (what weights.PackedDiT.load does in
//     Python — fused q/k/v, all AdaLN linears concatenated, grouped k=31 conv as tap-major block-diagonal-by-64,
//     the input projection split by source, bf16 conversion, the text position table of rope.py:63-73), binding of
//     f5_dit_weights to a device copy of it;
//   * the per-session workspace: size and carving of f5_dit_buffers out of ONE device allocation (+ the RoPE table
//     of rope.py:38-53 uploaded into it);
//   * the one collective of the multi-GPU path, ncclBroadcast of the packed buffer, resolved at run time from the
//     NCCL library already in the process (no link-time dependency).
// No kernels here; the layout below MUST stay in step with weights.PackedDiT._layout (tests/test_abi.py compares
// the two byte for byte).
#include <dlfcn.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "host_common.h"

namespace f5 {
namespace {

constexpr int64_t kAlign = 256;
inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

inline uint16_t f32_to_bf16(float f) {   // round to nearest even, NaN preserved (what torch's .to(bfloat16) does)
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}

struct Entry {
  std::string name;
  int64_t elems;
  bool bf16;
  int64_t offset;
};

struct Layout {
  std::vector<Entry> e;
  int64_t bytes = 0;
  int ct_ld = 0;
  const Entry* find(const std::string& n) const {
    for (const auto& x : e)
      if (x.name == n) return &x;
    return nullptr;
  }
};

Layout make_layout(const f5_dit_dims* d) {
  Layout L;
  const int64_t D = d->dim, F = d->ff_inner, Ct = d->text_dim, Ci = 2 * d->text_dim;
  L.ct_ld = (int)round_up(d->mel_dim + d->text_dim, 64);
  auto add = [&](const std::string& n, int64_t elems, bool bf) {
    L.e.push_back({n, elems, bf, L.bytes});
    L.bytes = round_up(L.bytes + elems * (bf ? 2 : 4), kAlign);
  };
  add("time_w0", D * 256, false); add("time_b0", D, false); add("time_w2", D * D, false); add("time_b2", D, false);
  add("text_emb", (int64_t)(d->text_num_embeds + 1) * Ct, false);
  add("text_pos", 4096 * Ct, false);
  for (int i = 0; i < d->conv_layers; ++i) {
    const std::string p = "tb" + std::to_string(i) + ".";
    add(p + "dw_w", 7 * Ct, false); add(p + "dw_b", Ct, false); add(p + "ln_w", Ct, false); add(p + "ln_b", Ct, false);
    add(p + "pw1_w", Ci * Ct, true); add(p + "pw1_b", Ci, false);
    add(p + "grn_gamma", Ci, false); add(p + "grn_beta", Ci, false);
    add(p + "pw2_w", Ct * Ci, true); add(p + "pw2_b", Ct, false);
  }
  add("in_x_w", D * 128, true); add("in_ct_w", D * L.ct_ld, true); add("in_b", D, false);
  for (int j = 0; j < 2; ++j) {
    add("conv_w" + std::to_string(j), D * 31 * 64, true);
    add("conv_b" + std::to_string(j), D, false);
  }
  const int64_t NM = (int64_t)d->depth * 6 * D + 2 * D;
  add("mod_w", NM * D, true); add("mod_b", NM, false);
  for (int i = 0; i < d->depth; ++i) {
    const std::string p = "blk" + std::to_string(i) + ".";
    add(p + "qkv_w", 3 * D * D, true); add(p + "qkv_b", 3 * D, false);
    add(p + "out_w", D * D, true); add(p + "out_b", D, false);
    add(p + "ff1_w", F * D, true); add(p + "ff1_b", F, false);
    add(p + "ff2_w", D * F, true); add(p + "ff2_b", D, false);
  }
  add("proj_w", (int64_t)d->mel_dim * D, true); add("proj_b", d->mel_dim, false);
  return L;
}

int check_dims(const f5_dit_dims* d) {
  F5_REQUIRE(d != nullptr, "null f5_dit_dims");
  F5_REQUIRE(d->dim % 128 == 0 && d->dim >= 256 && d->dim <= 1024 && 64 % (d->dim / 16) == 0 && d->dim == d->heads * 64,
             "f5_dit_dims: dim %d / heads %d", d->dim, d->heads);
  F5_REQUIRE(d->depth > 0 && d->ff_inner > 0 && d->mel_dim > 0 && d->mel_dim <= 128 && d->text_dim % 64 == 0 && d->conv_layers >= 0 &&
                 d->text_num_embeds > 0,
             "f5_dit_dims: bad field");
  F5_REQUIRE(d->text_unmasked == 0 || d->text_unmasked == 1, "f5_dit_dims: text_unmasked %d is not 0 or 1",
             d->text_unmasked);
  F5_REQUIRE(d->rope_heads >= 0 && d->rope_heads <= d->heads, "f5_dit_dims: rope_heads %d not in [0, heads %d]",
             d->rope_heads, d->heads);
  return 0;
}

struct Packer {
  const Layout& L;
  f5_tensor_lookup get;
  void* user;
  uint8_t* out;
  int err = 0;

  const float* src(const std::string& name, int64_t expect) {
    int64_t n = 0;
    const float* p = get(user, name.c_str(), &n);
    if (p == nullptr || n != expect) {
      err = set_error(F5_ERR_INVALID, "f5_pack_weights: tensor '%s' %s (have %lld elements, need %lld)", name.c_str(),
                      p ? "has the wrong size" : "is missing", (long long)n, (long long)expect);
      return nullptr;
    }
    return p;
  }
  void put(const std::string& dst, const float* v, int64_t n) {
    const Entry* e = L.find(dst);
    if (e->bf16) {
      uint16_t* o = reinterpret_cast<uint16_t*>(out + e->offset);
      for (int64_t i = 0; i < n; ++i) o[i] = f32_to_bf16(v[i]);
    } else {
      memcpy(out + e->offset, v, (size_t)n * 4);
    }
  }
  bool copy(const std::string& dst, const std::string& name) {
    const Entry* e = L.find(dst);
    const float* p = src(name, e->elems);
    if (!p) return false;
    put(dst, p, e->elems);
    return true;
  }
};

}  // namespace
}  // namespace f5

using namespace f5;

extern "C" int64_t f5_packed_weights_bytes(const f5_dit_dims* d) {
  if (check_dims(d)) return -1;
  return make_layout(d).bytes;
}

extern "C" int f5_pack_weights(const f5_dit_dims* d, f5_tensor_lookup get, void* user, void* host_out) {
  if (int e = check_dims(d)) return e;
  F5_REQUIRE(get && host_out, "f5_pack_weights: null argument");
  const Layout L = make_layout(d);
  memset(host_out, 0, (size_t)L.bytes);
  Packer P{L, get, user, reinterpret_cast<uint8_t*>(host_out)};
  const int64_t D = d->dim, F = d->ff_inner, Ct = d->text_dim, Ci = 2 * Ct, mel = d->mel_dim;
  const std::string T = "transformer.";
  bool ok = P.copy("time_w0", T + "time_embed.time_mlp.layers.0.weight") && P.copy("time_b0", T + "time_embed.time_mlp.layers.0.bias") &&
            P.copy("time_w2", T + "time_embed.time_mlp.layers.2.weight") && P.copy("time_b2", T + "time_embed.time_mlp.layers.2.bias") &&
            P.copy("text_emb", T + "text_embed.text_embed.weight");
  if (!ok) return P.err;
  {  // rope.py:63-73 precompute_freqs_cis(text_dim, 4096): [cos | sin] of t * theta^(-2i/dim)
    std::vector<float> tab((size_t)4096 * Ct);
    const int half = (int)Ct / 2;
    for (int i = 0; i < half; ++i) {
      const float fr = 1.0f / powf(10000.0f, (float)(2 * i) / (float)Ct);
      for (int t = 0; t < 4096; ++t) {
        const float a = (float)t * fr;
        tab[(size_t)t * Ct + i] = cosf(a);
        tab[(size_t)t * Ct + half + i] = sinf(a);
      }
    }
    P.put("text_pos", tab.data(), (int64_t)tab.size());
  }
  for (int i = 0; i < d->conv_layers; ++i) {
    const std::string p = T + "text_embed.text_blocks.layers." + std::to_string(i) + ".", q = "tb" + std::to_string(i) + ".";
    const float* dw = P.src(p + "dwconv.weight", Ct * 7);          // MLX (C, 7, 1) -> tap-major (7, C)
    if (!dw) return P.err;
    std::vector<float> t((size_t)7 * Ct);
    for (int64_t c = 0; c < Ct; ++c)
      for (int k = 0; k < 7; ++k) t[(size_t)k * Ct + c] = dw[c * 7 + k];
    P.put(q + "dw_w", t.data(), 7 * Ct);
    ok = P.copy(q + "dw_b", p + "dwconv.bias") && P.copy(q + "ln_w", p + "norm.weight") && P.copy(q + "ln_b", p + "norm.bias") &&
         P.copy(q + "pw1_w", p + "pwconv1.weight") && P.copy(q + "pw1_b", p + "pwconv1.bias") &&
         P.copy(q + "grn_gamma", p + "grn.gamma") && P.copy(q + "grn_beta", p + "grn.beta") &&
         P.copy(q + "pw2_w", p + "pwconv2.weight") && P.copy(q + "pw2_b", p + "pwconv2.bias");
    if (!ok) return P.err;
    (void)Ci;
  }
  {  // InputEmbedding.proj (dit.py:239): columns [x | cond | text] -> x part padded to 128, [cond|text] part padded to ct_ld
    const int64_t in = 2 * mel + Ct;
    const float* pw = P.src(T + "input_embed.proj.weight", D * in);
    if (!pw) return P.err;
    std::vector<float> wx((size_t)D * 128, 0.f), wct((size_t)D * L.ct_ld, 0.f);
    for (int64_t o = 0; o < D; ++o) {
      for (int64_t c = 0; c < mel; ++c) wx[(size_t)o * 128 + c] = pw[o * in + c];
      for (int64_t c = 0; c < mel + Ct; ++c) wct[(size_t)o * L.ct_ld + c] = pw[o * in + mel + c];
    }
    P.put("in_x_w", wx.data(), D * 128);
    P.put("in_ct_w", wct.data(), D * L.ct_ld);
    if (!P.copy("in_b", T + "input_embed.proj.bias")) return P.err;
  }
  for (int j = 0; j < 2; ++j) {  // grouped Conv1d(k=31, groups=16), MLX weight (O, 31, I/g) -> [O, 31*64] block-diagonal by 64
    const std::string p = T + "input_embed.conv_pos_embed.conv1d.layers." + std::to_string(2 * j) + ".";
    const int64_t cg = D / 16;
    const float* w = P.src(p + "weight", D * 31 * cg);
    if (!w) return P.err;
    std::vector<float> t((size_t)D * 31 * 64, 0.f);
    for (int64_t o = 0; o < D; ++o) {
      const int64_t base = (o / cg) * cg - (o / 64) * 64;   // first input channel of o's group inside its 64-block
      for (int k = 0; k < 31; ++k)
        for (int64_t i = 0; i < cg; ++i) t[((size_t)o * 31 + k) * 64 + base + i] = w[(o * 31 + k) * cg + i];
    }
    P.put("conv_w" + std::to_string(j), t.data(), D * 31 * 64);
    if (!P.copy("conv_b" + std::to_string(j), p + "bias")) return P.err;
  }
  {  // all AdaLN linears (dit.py:263,282) concatenated row-wise
    const int64_t NM = (int64_t)d->depth * 6 * D + 2 * D;
    std::vector<float> mw((size_t)NM * D), mb((size_t)NM);
    for (int i = 0; i <= d->depth; ++i) {
      const bool last = i == d->depth;
      const std::string p = last ? T + "norm_out.linear." : T + "transformer_blocks." + std::to_string(i) + ".attn_norm.linear.";
      const int64_t rows = last ? 2 * D : 6 * D;
      const float* w = P.src(p + "weight", rows * D);
      const float* b = P.src(p + "bias", rows);
      if (!w || !b) return P.err;
      memcpy(mw.data() + (size_t)i * 6 * D * D, w, (size_t)rows * D * 4);
      memcpy(mb.data() + (size_t)i * 6 * D, b, (size_t)rows * 4);
    }
    P.put("mod_w", mw.data(), NM * D);
    P.put("mod_b", mb.data(), NM);
  }
  for (int i = 0; i < d->depth; ++i) {
    const std::string p = T + "transformer_blocks." + std::to_string(i) + ".", q = "blk" + std::to_string(i) + ".";
    std::vector<float> w((size_t)3 * D * D), b((size_t)3 * D);
    const char* names[3] = {"q", "k", "v"};
    for (int j = 0; j < 3; ++j) {
      const float* wj = P.src(p + "attn.to_" + names[j] + ".weight", D * D);
      const float* bj = P.src(p + "attn.to_" + names[j] + ".bias", D);
      if (!wj || !bj) return P.err;
      memcpy(w.data() + (size_t)j * D * D, wj, (size_t)D * D * 4);
      memcpy(b.data() + (size_t)j * D, bj, (size_t)D * 4);
    }
    P.put(q + "qkv_w", w.data(), 3 * D * D);
    P.put(q + "qkv_b", b.data(), 3 * D);
    ok = P.copy(q + "out_w", p + "attn.to_out.layers.0.weight") && P.copy(q + "out_b", p + "attn.to_out.layers.0.bias") &&
         P.copy(q + "ff1_w", p + "ff.ff.layers.0.layers.0.weight") && P.copy(q + "ff1_b", p + "ff.ff.layers.0.layers.0.bias") &&
         P.copy(q + "ff2_w", p + "ff.ff.layers.2.weight") && P.copy(q + "ff2_b", p + "ff.ff.layers.2.bias");
    if (!ok) return P.err;
    (void)F;
  }
  if (!(P.copy("proj_w", T + "proj_out.weight") && P.copy("proj_b", T + "proj_out.bias"))) return P.err;
  return 0;
}

extern "C" int f5_bind_packed_weights(const f5_dit_dims* d, const void* device_base, f5_dit_weights* w,
                                      f5_convnext_weights* text_blocks, f5_dit_block_weights* blocks) {
  if (int e = check_dims(d)) return e;
  F5_REQUIRE(device_base && w && blocks && (text_blocks || d->conv_layers == 0), "f5_bind_packed_weights: null argument");
  const Layout L = make_layout(d);
  const char* base = reinterpret_cast<const char*>(device_base);
  auto at = [&](const std::string& n) -> const void* { return base + L.find(n)->offset; };
  auto f = [&](const std::string& n) { return reinterpret_cast<const float*>(at(n)); };
  memset(w, 0, sizeof(*w));
  w->dim = d->dim; w->depth = d->depth; w->heads = d->heads; w->ff_inner = d->ff_inner; w->mel_dim = d->mel_dim;
  w->text_dim = d->text_dim; w->text_inner = 2 * d->text_dim; w->conv_layers = d->conv_layers;
  w->text_rows = d->text_num_embeds + 1; w->text_max_pos = 4096; w->ct_ld = L.ct_ld;
  w->time_w0 = f("time_w0"); w->time_b0 = f("time_b0"); w->time_w2 = f("time_w2"); w->time_b2 = f("time_b2");
  w->text_emb = f("text_emb"); w->text_pos = f("text_pos");
  for (int i = 0; i < d->conv_layers; ++i) {
    const std::string q = "tb" + std::to_string(i) + ".";
    f5_convnext_weights& c = text_blocks[i];
    c.dw_w = f(q + "dw_w"); c.dw_b = f(q + "dw_b"); c.ln_w = f(q + "ln_w"); c.ln_b = f(q + "ln_b");
    c.pw1_w = at(q + "pw1_w"); c.pw1_b = f(q + "pw1_b"); c.grn_gamma = f(q + "grn_gamma"); c.grn_beta = f(q + "grn_beta");
    c.pw2_w = at(q + "pw2_w"); c.pw2_b = f(q + "pw2_b");
  }
  w->text_blocks = text_blocks;
  w->in_x_w = at("in_x_w"); w->in_ct_w = at("in_ct_w"); w->in_b = f("in_b");
  for (int j = 0; j < 2; ++j) {
    w->conv_w[j] = at("conv_w" + std::to_string(j));
    w->conv_b[j] = f("conv_b" + std::to_string(j));
  }
  w->mod_w = at("mod_w"); w->mod_b = f("mod_b");
  for (int i = 0; i < d->depth; ++i) {
    const std::string q = "blk" + std::to_string(i) + ".";
    f5_dit_block_weights& b = blocks[i];
    b.qkv_w = at(q + "qkv_w"); b.qkv_b = f(q + "qkv_b"); b.out_w = at(q + "out_w"); b.out_b = f(q + "out_b");
    b.ff1_w = at(q + "ff1_w"); b.ff1_b = f(q + "ff1_b"); b.ff2_w = at(q + "ff2_w"); b.ff2_b = f(q + "ff2_b");
  }
  w->blocks = blocks;
  w->proj_w = at("proj_w"); w->proj_b = f("proj_b");
  w->text_unmasked = d->text_unmasked; w->rope_heads = d->rope_heads;
  return 0;
}

// ---- workspace ----
namespace f5 {
namespace {
struct WsItem { size_t field_offset; int64_t bytes; };
std::vector<WsItem> ws_items(const f5_dit_dims* d, const f5_dit_shape* s) {
  const int64_t D = d->dim, F = d->ff_inner, Ct = d->text_dim, BU = (s->cfg ? 2 : 1) * (int64_t)s->batch, R = BU * s->frames;
  const int64_t NM = (int64_t)d->depth * 6 * D + 2 * D, T = s->n_times, ct_ld = round_up(d->mel_dim + d->text_dim, 64);
  const int64_t tab_ld = (int64_t)d->depth * (3 * D + F) + 128;
  std::vector<WsItem> v;
#define F5_WS(field, bytes) v.push_back({offsetof(f5_dit_buffers, field), (int64_t)(bytes)})
  F5_WS(text, (int64_t)s->batch * (s->text_len_max > 0 ? s->text_len_max : 1) * 4);
  F5_WS(text_len, BU * 4);
  F5_WS(seq_len, s->masked ? BU * 4 : 0);
  F5_WS(cond, (int64_t)s->batch * s->frames * d->mel_dim * 4);
  F5_WS(tvals, T * 4);
  F5_WS(rope, (int64_t)s->frames * 32 * 2 * 4);
  F5_WS(hoist, R * D * 4);
  F5_WS(mod_table, T * NM * 4);
  F5_WS(text_x, R * Ct * 4); F5_WS(text_a, R * Ct * 2); F5_WS(text_h, R * 2 * Ct * 2); F5_WS(text_g, R * 2 * Ct * 2);
  F5_WS(grn_nx, BU * (1 + (s->frames + 31) / 32) * 2 * Ct * 4);
  F5_WS(ct_bf16, R * ct_ld * 2);
  F5_WS(silu_t, T * D * 2);
  F5_WS(y_bf16, R * 128 * 2);
  F5_WS(x, R * D * 4); F5_WS(h, R * D * 4); F5_WS(a_bf16, R * D * 2); F5_WS(c_bf16, R * D * 2);
  F5_WS(qkv_bf16, R * 3 * D * 2); F5_WS(ff_bf16, R * F * 2);
  F5_WS(v, R * d->mel_dim * 4);
  F5_WS(ln_stats, s->fused_adaln ? R * (D / 64) * 2 * 4 : 0);
  F5_WS(ln_tab, s->fused_adaln ? 4 * T * tab_ld * 4 : 0);
  F5_WS(ln_prep, s->fused_adaln ? (2 * (int64_t)d->depth + 1) * 4 * T * D * 2 : 0);
  F5_WS(valid_len, s->bucketed ? BU * 4 : 0);
#undef F5_WS
  return v;
}
int check_shape(const f5_dit_shape* s) {
  F5_REQUIRE(s && s->batch > 0 && s->frames > 0 && s->n_times > 0, "f5_dit_shape: batch/frames/n_times must be positive");
  return 0;
}
}  // namespace
}  // namespace f5

extern "C" int64_t f5_workspace_bytes(const f5_dit_dims* d, const f5_dit_shape* s) {
  if (check_dims(d) || check_shape(s)) return -1;
  int64_t tot = 0;
  for (const auto& it : ws_items(d, s)) tot += round_up(it.bytes, kAlign);
  return tot;
}

extern "C" int f5_bind_workspace(const f5_dit_dims* d, const f5_dit_shape* s, void* device_base, f5_dit_buffers* b, void* stream_) {
  if (int e = check_dims(d)) return e;
  if (int e = check_shape(s)) return e;
  if (int e = device_check()) return e;
  F5_REQUIRE(device_base && b, "f5_bind_workspace: null argument");
  F5_REQUIRE((reinterpret_cast<uintptr_t>(device_base) & 255) == 0, "f5_bind_workspace: base must be 256-byte aligned");
  memset(b, 0, sizeof(*b));
  b->batch = s->batch; b->frames = s->frames; b->cfg = s->cfg ? 1 : 0; b->n_times = s->n_times;
  b->text_len_max = s->text_len_max > 0 ? s->text_len_max : 1;
  char* p = reinterpret_cast<char*>(device_base);
  for (const auto& it : ws_items(d, s)) {
    void* ptr = it.bytes > 0 ? p : nullptr;
    memcpy(reinterpret_cast<char*>(b) + it.field_offset, &ptr, sizeof(void*));
    p += round_up(it.bytes, kAlign);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  F5_CHECK_CUDA(cudaMemsetAsync(device_base, 0, (size_t)(p - reinterpret_cast<char*>(device_base)), st));
  // RoPE table (rope.py:38-53): (cos, sin) of n * 10000^(-2i/64), fp32 host math as in dit.rope_table
  std::vector<float> rope((size_t)s->frames * 64);
  for (int i = 0; i < 32; ++i) {
    const float inv = 1.0f / powf(10000.0f, (float)(2 * i) / 64.0f);
    for (int n = 0; n < s->frames; ++n) {
      const float a = (float)n * inv;
      rope[((size_t)n * 32 + i) * 2] = cosf(a);
      rope[((size_t)n * 32 + i) * 2 + 1] = sinf(a);
    }
  }
  F5_CHECK_CUDA(cudaMemcpyAsync(const_cast<float*>(b->rope), rope.data(), rope.size() * 4, cudaMemcpyHostToDevice, st));
  F5_CHECK_CUDA(cudaStreamSynchronize(st));   // `rope` is a stack-lifetime host buffer
  if (s->bucketed) {
    std::vector<int32_t> vl((size_t)(s->cfg ? 2 : 1) * s->batch, s->frames);
    F5_CHECK_CUDA(cudaMemcpy(const_cast<int32_t*>(b->valid_len), vl.data(), vl.size() * 4, cudaMemcpyHostToDevice));
  }
  return 0;
}

// ---- the one collective: broadcast of the packed weights (parallel.py / PackedDiT.broadcast in Python) ----
extern "C" int f5_nccl_broadcast_weights(void* device_buf, int64_t bytes, int32_t root, void* nccl_comm, void* stream_) {
  F5_REQUIRE(device_buf && bytes > 0 && nccl_comm, "f5_nccl_broadcast_weights: null argument");
  typedef int (*bcast_fn)(const void*, void*, size_t, int, int, void*, cudaStream_t);
  static bcast_fn fn = nullptr;
  if (!fn) {
    void* sym = dlsym(RTLD_DEFAULT, "ncclBroadcast");          // an NCCL already loaded by the host (e.g. torch's)
    if (!sym) {
      void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
      if (h) sym = dlsym(h, "ncclBroadcast");
    }
    if (!sym) return set_error(F5_ERR_CUDA, "f5_nccl_broadcast_weights: ncclBroadcast not found (load NCCL into the process first)");
    fn = reinterpret_cast<bcast_fn>(sym);
  }
  const int rc = fn(device_buf, device_buf, (size_t)bytes, /*ncclUint8*/ 1, root, nccl_comm, reinterpret_cast<cudaStream_t>(stream_));
  if (rc != 0) return set_error(F5_ERR_CUDA, "ncclBroadcast failed with ncclResult %d", rc);
  return 0;
}
