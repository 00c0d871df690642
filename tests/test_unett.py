"""E2TTS_Base (the UNetT backbone) on the CPU: the restatement's RMSNorm, skip pairing and time token, the loader and
its refusals, and the C layout of the new ABI structs."""
import ctypes as C
import math
import os
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

import unett_emul as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _small():
    from f5_tts_mlx_b200.unett import UNetTConfig
    return UNetTConfig(dim=256, depth=4, heads=4, ff_mult=4, text_num_embeds=10)


def _inputs(n=20, nt=12, seed=0):
    g = torch.Generator().manual_seed(seed)
    x, cond = torch.randn(1, n, 100, generator=g), torch.randn(1, n, 100, generator=g)
    text = torch.randint(0, 10, (1, nt), generator=g, dtype=torch.int32); text[0, 9:] = -1
    return x, cond, text


def test_rmsnorm_is_normalize_not_rsqrt_mean():
    g = torch.Generator().manual_seed(1)
    x, gain = torch.randn(3, 64, generator=g, dtype=torch.float64), 1 + 0.1 * torch.randn(64, generator=g, dtype=torch.float64)
    want = x / x.norm(dim=-1, keepdim=True).clamp_min(1e-12) * math.sqrt(64) * gain
    assert torch.allclose(U.rms_norm(x, gain), want, rtol=1e-12, atol=0)
    small = torch.full((1, 64), 1e-4, dtype=torch.float64)       # mean(x^2) = 1e-8, far below a 1e-6 epsilon
    eps_form = small * torch.rsqrt(small.pow(2).mean(-1, keepdim=True) + 1e-6) * gain
    assert (U.rms_norm(small, gain) - eps_form).abs().max() > 0.5
    assert torch.equal(U.rms_norm(torch.zeros(1, 64), torch.ones(64)), torch.zeros(1, 64))


def test_skip_pairing_is_lifo_with_x_first():
    from f5_tts_mlx_b200.unett import random_unett_weights
    cfg = _small()
    W = random_unett_weights(cfg, seed=5)
    x, cond, text = _inputs()
    t = torch.tensor(0.4)
    ref = U.unett_forward(x, cond, text, t, False, False, None, W, cfg)
    fifo = U.unett_forward(x, cond, text, t, False, False, None, W, cfg, skip_order="fifo")
    skip_first = U.unett_forward(x, cond, text, t, False, False, None, W, cfg, x_first=False)
    scale = ref.norm()
    assert (fifo - ref).norm() > 1e-3 * scale and (skip_first - ref).norm() > 1e-3 * scale
    # layer 2 pops layer 1's push and layer 3 layer 0's: swapping the two skip weights is not a no-op either
    W2 = dict(W)
    W2["transformer.layers.2.0.weight"], W2["transformer.layers.3.0.weight"] = W["transformer.layers.3.0.weight"], W["transformer.layers.2.0.weight"]
    assert (U.unett_forward(x, cond, text, t, False, False, None, W2, cfg) - ref).norm() > 1e-3 * scale


def test_time_token_is_row_zero_and_dropped():
    from f5_tts_mlx_b200.unett import random_unett_weights
    cfg = _small()
    W = random_unett_weights(cfg, seed=6)
    x, cond, text = _inputs(n=24)
    t = torch.tensor(0.7)
    full = U.unett_forward(x, cond, text, t, False, False, None, W, cfg, keep_time_row=True)
    out = U.unett_forward(x, cond, text, t, False, False, None, W, cfg)
    assert full.shape == (1, 25, 100) and out.shape == (1, 24, 100) and torch.equal(full[:, 1:], out)
    # the token is the time embedding itself: row 0's output moves with t, and so does every frame (through attention)
    other = U.unett_forward(x, cond, text, torch.tensor(0.2), False, False, None, W, cfg, keep_time_row=True)
    assert (other[:, 0] - full[:, 0]).norm() > 1e-3 * full[:, 0].norm()


def _save(d, W, name="model_1200000.safetensors", vocab=10):
    from safetensors.torch import save_file
    d.mkdir(parents=True, exist_ok=True)
    (d / "vocab.txt").write_text("\n".join(chr(ord("a") + i) for i in range(vocab)) + "\n")
    save_file({("ema_model." + k): v.contiguous() for k, v in W.items()}, str(d / name))


def test_from_pretrained_e2_round_trip_and_folds(tmp_path):
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.unett import UNetT, random_unett_weights
    import f5_tts_mlx_b200.pretrained as PT
    cfg = _small()
    W = random_unett_weights(cfg, seed=7)
    W["mel_spec.mel_stft.window"] = torch.ones(4)          # dropped, as upstream's loader drops them
    W["step"] = torch.tensor(3.0)
    _save(tmp_path / "e2", W)
    f5 = PT.from_pretrained(F5TTS, str(tmp_path / "e2"), device="cpu", vocoder=False, model_version="e2")
    net = f5.transformer
    assert isinstance(net, UNetT) and f5._duration_predictor is None
    c = net.config
    assert (c.dim, c.depth, c.heads, c.ff_mult, c.text_num_embeds, c.text_dim, c.pe_attn_head) == (256, 4, 4, 4, 10, 100, 1)
    P = net.packed
    T = "transformer."
    for i in range(cfg.depth):
        p = T + f"layers.{i}."
        wqkv = torch.cat([W[p + f"2.to_{n}.weight"] for n in "qkv"], 0)
        assert torch.equal(P.view(f"blk{i}.qkv_w"), (wqkv * W[p + "1.g"][None]).bfloat16())
        assert torch.equal(P.view(f"blk{i}.ff1_w"), (W[p + "4.ff.0.0.weight"] * W[p + "3.g"][None]).bfloat16())
        assert torch.equal(P.view(f"blk{i}.out_w"), W[p + "2.to_out.0.weight"].bfloat16())
        if i >= 2:
            assert torch.equal(P.view("skip_w")[i - 2], W[p + "0.weight"].bfloat16())
    assert torch.equal(P.view("proj_w"), (W[T + "proj_out.weight"] * W[T + "norm_out.g"][None]).bfloat16())
    w = P.c_struct()
    assert (w.dim, w.depth, w.rope_heads, w.text_rows, w.ct_ld) == (256, 4, 1, 11, 256)
    # a .safetensors file of another name, vocab.txt beside it, packs the same bytes
    (tmp_path / "e2" / "model_1200000.safetensors").rename(tmp_path / "e2" / "my_e2.safetensors")
    f5b = PT.from_pretrained(F5TTS, str(tmp_path / "e2" / "my_e2.safetensors"), device="cpu", vocoder=False,
                             model_version="e2")
    assert torch.equal(f5b.transformer.packed.buffer, P.buffer)
    # upstream's .pt training checkpoint
    torch.save({"ema_model_state_dict": {"ema_model." + k: v for k, v in W.items()}}, str(tmp_path / "e2" / "ck.pt"))
    f5c = PT.from_pretrained(F5TTS, str(tmp_path / "e2" / "ck.pt"), device="cpu", vocoder=False, model_version="e2")
    assert torch.equal(f5c.transformer.packed.buffer, P.buffer)


def test_loader_names_missing_and_unexpected_keys(tmp_path):
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.unett import checkpoint_state, random_unett_weights
    import f5_tts_mlx_b200.pretrained as PT
    cfg = _small()
    W = random_unett_weights(cfg, seed=8)
    missing = {k: v for k, v in W.items() if k != "transformer.layers.3.3.g"}
    with pytest.raises(ValueError, match=r"transformer\.layers\.3\.3\.g"):
        checkpoint_state(missing, cfg)
    extra = dict(W, **{"transformer.layers.1.0.weight": torch.zeros(256, 512)})   # a skip_proj in the first half
    with pytest.raises(ValueError, match=r"unexpected keys \['transformer\.layers\.1\.0\.weight'\]"):
        checkpoint_state(extra, cfg)
    with pytest.raises(ValueError, match="rotary"):
        checkpoint_state(dict(W, **{"transformer.rotary_embed.inv_freq": torch.ones(32)}), cfg)
    inv = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float32) / 64))
    assert checkpoint_state(dict(W, **{"transformer.rotary_embed.inv_freq": inv}), cfg).keys() == W.keys()
    _save(tmp_path / "bad", missing)
    with pytest.raises(ValueError, match=r"missing keys \['transformer\.layers\.3\.3\.g'\]"):
        PT.from_pretrained(F5TTS, str(tmp_path / "bad"), device="cpu", vocoder=False, model_version="e2")


def test_e2_refusals(tmp_path):
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.unett import UNetT
    import f5_tts_mlx_b200.pretrained as PT
    for kw in (dict(fp8="tensor"), dict(fp8="block"), dict(fp8="block", fp8_attention=True), dict(quantization_bits=4),
               dict(vocoder="bigvgan")):
        with pytest.raises(ValueError):
            PT.from_pretrained(F5TTS, "random", device="cpu", model_version="e2", **kw)
    base = dict(dim=256, depth=4, heads=4, device="cpu")
    for kw in (dict(skip_connect_type="add"), dict(skip_connect_type=None), dict(qk_norm="rms_norm"), dict(depth=3),
               dict(conv_layers=4), dict(text_mask_padding=True), dict(pe_attn_head=0)):
        with pytest.raises(ValueError):
            UNetT(**{**base, **kw})
    UNetT(**base)


def test_generate_cli_accepts_e2(monkeypatch):
    import f5_tts_mlx_b200.generate as G
    seen = {}
    monkeypatch.setattr(G, "generate", lambda **kw: seen.update(kw))
    G.main(["--text", "hi", "--model-version", "e2", "--duration", "2"])
    assert seen["model_version"] == "e2"


def test_new_structs_match_c(tmp_path):
    from f5_tts_mlx_b200 import _lib
    from f5_tts_mlx_b200.unett import UNetTBuffersC, UNetTWeightsC
    assert _lib.load().f5_abi_version() >= 2006
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    checks = {"sizeof(f5_unett_weights)": C.sizeof(UNetTWeightsC), "sizeof(f5_unett_buffers)": C.sizeof(UNetTBuffersC),
              "sizeof(f5_gemm_args)": C.sizeof(_lib.GemmArgs),
              "offsetof(f5_gemm_args, ln_rms)": _lib.GemmArgs.ln_rms.offset,
              "offsetof(f5_gemm_args, prefetch)": _lib.GemmArgs.prefetch.offset}
    for s, m in (("f5_unett_weights", UNetTWeightsC), ("f5_unett_buffers", UNetTBuffersC)):
        for name, _ in m._fields_:
            if name != "reserved":
                checks[f"offsetof({s}, {name})"] = getattr(m, name).offset
    exprs = list(checks)
    src = tmp_path / "l.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "f5_b200.h"\nint main(void) {\n' +
                   "".join(f'  printf("%d\\n", (int){e});\n' for e in exprs) + "  return 0;\n}\n")
    exe = str(tmp_path / "l")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = list(map(int, subprocess.run([exe], capture_output=True, text=True).stdout.split()))
    assert dict(zip(exprs, got)) == checks
