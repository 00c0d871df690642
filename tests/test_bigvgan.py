"""BigVGAN v2 on the CPU: the Slaney filterbank, the mel restatement against torch.stft, the Kaiser-sinc filter, the
weight-norm fold, the polyphase packing of the transposed convolutions, the activation kernel's index algebra, checkpoint
loading, config refusals, the C layout of the new ABI structs and the new kernels' compile reports."""
import ctypes as C
import json
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import bigvgan_emul as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_slaney_scale_and_filterbank():
    from f5_tts_mlx_b200 import bigvgan as BV
    assert E.hz_to_mel(1000.0) == pytest.approx(15.0, abs=1e-12)
    assert E.mel_to_hz(15.0) == pytest.approx(1000.0, abs=1e-9)
    assert float(BV.hz_to_mel_slaney(1000.0)) == pytest.approx(15.0, abs=1e-12)
    assert float(BV.mel_to_hz_slaney(BV.hz_to_mel_slaney(3210.0))) == pytest.approx(3210.0, rel=1e-12)
    f64 = BV.slaney_filterbank_f64()
    ref = E.slaney_filterbank()
    assert f64.shape == (100, 513) and np.abs(f64 - ref).max() <= 1e-12 * np.abs(ref).max()
    # the fp32 table is the float64 table rounded once
    assert torch.equal(BV.slaney_filterbank(), torch.from_numpy(f64).float())
    # Slaney area normalisation: each triangle has unit area in Hz, up to the sampling of the triangle on the bin grid
    df = 12000.0 / 512
    fmax = E.hz_to_mel(12000.0)
    mel_f = [E.mel_to_hz(fmax * i / 101) for i in range(102)]
    for i in range(100):
        width = mel_f[i + 2] - mel_f[i]
        area = f64[i].sum() * df
        assert abs(area - 1.0) <= 2.0 * df / width + 1e-9, (i, area)


def test_mel_restatement_equals_torch_stft():
    g = torch.Generator().manual_seed(0)
    wave = 0.3 * torch.randn(2, 5000, generator=g, dtype=torch.float64)
    fb = E.slaney_filterbank()
    got = E.mel(wave, fb)
    xp = F.pad(wave[:, None], (384, 384), mode="reflect")[:, 0]
    spec = torch.stft(xp, 1024, 256, 1024, torch.hann_window(1024, dtype=torch.float64), center=False,
                      return_complex=True)
    mag = torch.sqrt(spec.real ** 2 + spec.imag ** 2 + 1e-9)
    want = torch.log(torch.clamp(torch.from_numpy(fb) @ mag, min=1e-5)).transpose(1, 2)
    assert got.shape == want.shape == (2, (5000 + 768 - 1024) // 256 + 1, 100)
    assert (got - want).abs().max().item() < 1e-10


def test_bigvgan_frames_and_short_input():
    from f5_tts_mlx_b200.bigvgan import bigvgan_frames
    assert [bigvgan_frames(t) for t in (385, 511, 512, 24000)] == [(t + 768 - 1024) // 256 + 1 for t in (385, 511, 512, 24000)]
    for t in (1, 384):
        with pytest.raises(ValueError):
            bigvgan_frames(t)


def test_kaiser_filter():
    from f5_tts_mlx_b200.bigvgan import kaiser_sinc_filter1d
    h = kaiser_sinc_filter1d()
    assert h.shape == (12,) and h.dtype == torch.float32
    assert abs(h.double().sum().item() - 1.0) < 1e-6
    assert torch.equal(h, h.flip(0))


@pytest.mark.parametrize("transposed", [False, True])
def test_weight_norm_fold_matches_torch(transposed):
    from f5_tts_mlx_b200.bigvgan import conv_weight
    torch.manual_seed(0)
    m = torch.nn.ConvTranspose1d(16, 8, 4) if transposed else torch.nn.Conv1d(16, 8, 5)
    m = torch.nn.utils.weight_norm(m)
    with torch.no_grad():
        m.weight_g.mul_(torch.rand_like(m.weight_g) + 0.5)
    m(torch.zeros(1, 16, 10))                                   # the forward pre-hook recomputes .weight
    sd = {"c.weight_g": m.weight_g.detach(), "c.weight_v": m.weight_v.detach()}
    assert torch.allclose(conv_weight(sd, "c"), m.weight.detach(), rtol=1e-6, atol=1e-7)
    assert torch.equal(conv_weight({"c.weight": m.weight.detach()}, "c"), m.weight.detach())
    with pytest.raises(ValueError):
        conv_weight({}, "c")


@pytest.mark.parametrize("k,u", [(8, 4), (4, 2), (16, 8), (3, 1), (6, 2), (5, 3)])
def test_polyphase_packing_equals_conv_transpose(k, u):
    from f5_tts_mlx_b200.bigvgan import pack_polyphase
    g = torch.Generator().manual_seed(k * 10 + u)
    cin, cout, T = 6, 5, 13
    w = torch.randn(cin, cout, k, generator=g, dtype=torch.float64)
    x = torch.randn(2, cin, T, generator=g, dtype=torch.float64)
    want = F.conv_transpose1d(x, w, stride=u, padding=(k - u) // 2)
    pw, taps, pad = pack_polyphase(w, u)                       # [u * cout, taps, cin]
    got = F.conv1d(F.pad(x, (pad, taps - 1 - pad)), pw.permute(0, 2, 1))       # (2, u * cout, T)
    got = got.reshape(2, u, cout, T).permute(0, 2, 3, 1).reshape(2, cout, T * u)
    assert want.shape == got.shape and (got - want).abs().max().item() < 1e-12
    if k == 2 * u and u % 2 == 0:
        assert (taps, pad) == (3, 1)


def _act_direct(x, alpha, beta, hu, hd):
    """The activation kernel's index algebra (csrc/bigvgan.cu), element by element in float64: x (T, C)."""
    T = x.shape[0]
    out = np.zeros_like(x)
    xc = lambda i: x[min(max(i, 0), T - 1)]

    def a_at(m):
        m = min(max(m, 0), 2 * T - 1)
        j0 = (m + 1) & 1
        acc = sum(hu[j0 + 2 * jj] * xc((m + 5 - j0 - 2 * jj) // 2) for jj in range(6))
        u = 2 * acc
        return u + np.sin(alpha * u) ** 2 / (beta + 1e-9)
    for n in range(T):
        out[n] = sum(hd[j] * a_at(2 * n + j - 5) for j in range(12))
    return out


@pytest.mark.parametrize("T", [1, 2, 3, 5, 8, 33])
def test_activation_index_algebra_matches_definition(T):
    from f5_tts_mlx_b200.bigvgan import kaiser_sinc_filter1d
    g = torch.Generator().manual_seed(T)
    Cn = 3
    x = torch.randn(T, Cn, generator=g, dtype=torch.float64)
    alpha = torch.rand(Cn, generator=g, dtype=torch.float64) + 0.5
    beta = torch.rand(Cn, generator=g, dtype=torch.float64) + 0.5
    hu = kaiser_sinc_filter1d().double()
    hd = hu * (1 + 0.1 * torch.randn(12, generator=g, dtype=torch.float64))
    want = E.activation1d(x.t()[None], alpha, beta, hu, hd)[0].t()
    got = _act_direct(x.numpy(), alpha.numpy(), beta.numpy(), hu.numpy(), hd.numpy())
    assert want.shape == (T, Cn) and np.abs(got - want.numpy()).max() < 1e-12


def _small_cfg(**kw):
    from f5_tts_mlx_b200.bigvgan import BigVGANConfig
    d = dict(num_mels=100, upsample_rates=[4, 2], upsample_kernel_sizes=[8, 4], upsample_initial_channel=128,
             resblock="1", resblock_kernel_sizes=[3, 7], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5]],
             activation="snakebeta", snake_logscale=True, use_tanh_at_final=False, use_bias_at_final=False)
    d.update(kw)
    return d


def test_random_checkpoint_round_trip(tmp_path):
    from f5_tts_mlx_b200.bigvgan import BigVGANConfig, load_checkpoint, pack_bigvgan, random_bigvgan_weights
    d = _small_cfg()
    cfg = BigVGANConfig.from_dict(d)
    sd = random_bigvgan_weights(cfg, seed=3)
    assert "conv_post.bias" not in sd and "ups.1.0.weight_g" in sd and sd["ups.1.0.weight_g"].shape == (64, 1, 1)
    (tmp_path / "config.json").write_text(json.dumps(d))
    torch.save({"generator": sd}, str(tmp_path / "bigvgan_generator.pt"))
    cfg2, sd2 = load_checkpoint(tmp_path)
    assert cfg2 == cfg and sd2.keys() == sd.keys() and all(torch.equal(sd[k], sd2[k]) for k in sd)
    P = pack_bigvgan(cfg2, sd2)
    assert P["conv_pre_w"].shape == (128, 7 * 128) and P["up0_w"].shape == (4 * 64, 3 * 128)
    assert P["up1_w"].shape == (2 * 32, 3 * 64) and P["rb2.convs1.0_w"].shape == (32, 3 * 64)
    assert "conv_post_b" not in P and P["conv_post_w"].shape == (7, 32)
    # the emulation of the GPU's rounding points stays close to the float64 definition, and the output is not saturated
    mel = torch.randn(1, 5, 100, generator=torch.Generator().manual_seed(0)) - 3
    ref, emu = E.generator(mel, sd, cfg), E.generator(mel, sd, cfg, emulate=True)
    assert ref.shape == (1, 5 * 8) and 0 < ((emu - ref).norm() / ref.norm()).item() < 0.05
    assert ref.abs().max() < 1.0
    # missing defaults: use_tanh_at_final / use_bias_at_final default to true
    d3 = {k: v for k, v in d.items() if k not in ("use_tanh_at_final", "use_bias_at_final")}
    c3 = BigVGANConfig.from_dict(d3)
    assert c3.use_tanh_at_final and c3.use_bias_at_final


@pytest.mark.parametrize("change", [dict(resblock="2"), dict(activation="relu"), dict(upsample_kernel_sizes=[7, 4]),
                                    dict(upsample_kernel_sizes=[3, 4]), dict(resblock_kernel_sizes=[3, 4]),
                                    dict(upsample_initial_channel=120), dict(num_mels=200),
                                    dict(resblock_dilation_sizes=[[1, 3], [1, 3, 5]]),
                                    dict(upsample_rates=[4, 2, 2], upsample_kernel_sizes=[8, 4])])
def test_unsupported_configs_raise(change):
    from f5_tts_mlx_b200.bigvgan import BigVGANConfig
    with pytest.raises(ValueError):
        BigVGANConfig.from_dict(_small_cfg(**change))
    with pytest.raises(ValueError):
        BigVGANConfig.from_dict({k: v for k, v in _small_cfg().items() if k != "num_mels"})


def test_released_config_is_the_default():
    from f5_tts_mlx_b200.bigvgan import BigVGANConfig, stage_elems
    cfg = BigVGANConfig()
    assert cfg.hop_length == 256 and cfg.stage_channels() == [768, 384, 192, 96, 48, 24]
    assert stage_elems(cfg, 10) == 10 * 6144


def test_from_pretrained_pt_checkpoint_and_bigvgan_dir(tmp_path, monkeypatch):
    """A .pt DiT checkpoint (upstream keys under ema_model_state_dict) packs the same bytes as the same weights in
    .safetensors; vocoder="bigvgan" resolves bigvgan/ next to the model and sets the BigVGAN mel, with no duration
    predictor; a missing BigVGAN directory is an error."""
    from safetensors.torch import save_file
    from f5_tts_mlx_b200 import F5TTS
    import f5_tts_mlx_b200.pretrained as PT
    import f5_tts_mlx_b200.bigvgan as BV
    from f5_tts_mlx_b200.weights import BASE_CONFIG, random_dit_weights
    W = random_dit_weights(BASE_CONFIG._replace(text_num_embeds=10) if hasattr(BASE_CONFIG, "_replace") else
                           type(BASE_CONFIG)(**{**BASE_CONFIG.__dict__, "text_num_embeds": 10}), seed=2)
    up = {"ema_model." + k: v for k, v in _to_upstream(W).items()}
    d = tmp_path / "m"
    d.mkdir()
    (d / "vocab.txt").write_text("\n".join([chr(97 + i) for i in range(10)] + [""]))
    torch.save({"ema_model_state_dict": up, "step": 1}, str(d / "model_1200000.pt"))
    save_file({k: v.contiguous() for k, v in up.items()}, str(d / "model_1200000.safetensors"))
    a = PT.from_pretrained(F5TTS, str(d / "model_1200000.pt"), device="cpu", vocoder=False, model_version="v0")
    b = PT.from_pretrained(F5TTS, str(d / "model_1200000.safetensors"), device="cpu", vocoder=False, model_version="v0")
    assert torch.equal(a.transformer.packed.buffer, b.transformer.packed.buffer)
    with pytest.raises(FileNotFoundError):
        PT.from_pretrained(F5TTS, str(d / "model_1200000.pt"), device="cpu", vocoder="bigvgan", model_version="v0")
    with pytest.raises(ValueError):
        PT.from_pretrained(F5TTS, str(d / "model_1200000.pt"), device="cpu", vocoder="hifigan", model_version="v0")
    (d / "bigvgan").mkdir()
    cfg = _small_cfg()
    (d / "bigvgan" / "config.json").write_text(json.dumps(cfg))
    torch.save({"generator": BV.random_bigvgan_weights(BV.BigVGANConfig.from_dict(cfg), 1)},
               str(d / "bigvgan" / "bigvgan_generator.pt"))
    (d / "duration_v2.safetensors").write_bytes(b"not read")
    loaded = {}
    monkeypatch.setattr(BV.BigVGAN, "load_weights", lambda self, sd: loaded.setdefault("sd", sd) and self)
    f5 = PT.from_pretrained(F5TTS, str(d / "model_1200000.pt"), device="cpu", vocoder="bigvgan", model_version="v0")
    assert isinstance(f5._mel_spec, BV.BigVGANMelSpec) and f5._duration_predictor is None
    assert f5._vocoder.__self__.config == BV.BigVGANConfig.from_dict(cfg) and "conv_pre.weight_v" in loaded["sd"]
    monkeypatch.setenv("F5_BIGVGAN_PATH", str(d / "bigvgan"))
    assert PT._resolve_bigvgan(None) == d / "bigvgan"


def _to_upstream(W):
    """The inverse of weights.convert_upstream_keys on the keys it renames."""
    out = {}
    for k, v in W.items():
        if ".dwconv.weight" in k or ".conv1d.layers.0.weight" in k or ".conv1d.layers.2.weight" in k:
            v = v.transpose(1, 2)
        for a, b in ((".to_out.layers", ".to_out"), (".text_blocks.layers", ".text_blocks"),
                     (".ff.ff.layers.0.layers.0", ".ff.ff.0.0"), (".ff.ff.layers.2", ".ff.ff.2"),
                     (".time_mlp.layers", ".time_mlp"), (".conv1d.layers", ".conv1d")):
            k = k.replace(a, b)
        out[k] = v.contiguous()
    return out


def test_generate_cli_accepts_vocoder(monkeypatch):
    import f5_tts_mlx_b200.generate as G
    seen = {}
    monkeypatch.setattr(G, "generate", lambda **kw: seen.update(kw))
    G.main(["--text", "hi", "--vocoder", "bigvgan", "--model-version", "v0"])
    assert seen["vocoder"] == "bigvgan"
    seen.clear()
    G.main(["--text", "hi"])
    assert "vocoder" not in seen
    with pytest.raises(SystemExit):
        G.main(["--text", "hi", "--vocoder", "hifigan"])


def test_abi_version_and_c_layout_of_new_structs(tmp_path):
    from f5_tts_mlx_b200 import _lib
    import f5_tts_mlx_b200.bigvgan as BV
    assert _lib.load().f5_abi_version() >= 2007          # 2.007: the resblock-mean and conv_post test entries
    for name in ("f5_bigvgan_resblock_mean", "f5_bigvgan_conv_post"):
        assert hasattr(_lib.load(), name) and name in _lib.SYMBOLS
    assert C.sizeof(_lib.GemmArgsDilated) == C.sizeof(_lib.GemmArgs)
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    checks = {
        "sizeof(f5_gemm_args)": C.sizeof(_lib.GemmArgs),
        "offsetof(f5_gemm_args, conv_dilation)": _lib.GemmArgsDilated.conv_dilation.offset,
        "sizeof(f5_bigvgan_act)": C.sizeof(BV.BigVGANActC),
        "sizeof(f5_bigvgan_amp_weights)": C.sizeof(BV.BigVGANAmpWeightsC),
        "sizeof(f5_bigvgan_weights)": C.sizeof(BV.BigVGANWeightsC),
        "sizeof(f5_bigvgan_buffers)": C.sizeof(BV.BigVGANBuffersC),
    }
    for s, m in (("f5_bigvgan_amp_weights", BV.BigVGANAmpWeightsC), ("f5_bigvgan_weights", BV.BigVGANWeightsC),
                 ("f5_bigvgan_buffers", BV.BigVGANBuffersC), ("f5_bigvgan_act", BV.BigVGANActC)):
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


def _ptxas(src, tmp_path):
    from f5_tts_mlx_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-cubin", os.path.join(ROOT, "f5_tts_mlx_b200", "csrc", src),
           "-o", str(tmp_path / "k.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout + r.stderr


@pytest.mark.parametrize("src", ["bigvgan.cu", "audio_vocos.cu", "gemm.cu"])
def test_kernels_compile_without_spills(src, tmp_path):
    """Every kernel of the BigVGAN path compiles for sm_90a with no spills; every GEMM instantiation (the dilated
    convolution only changes its producer's row coordinate) keeps the launch's 168 registers, with no C7510."""
    log = _ptxas(src, tmp_path)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(s == ("0", "0") for s in spills), spills
    if src == "gemm.cu":
        regs = re.findall(r"Used (\d+) registers", log)
        assert len(regs) >= 30 and set(regs) == {"168"}, regs
        assert "C7510" not in log
    if src == "bigvgan.cu":
        assert log.count("bigvgan_act_kernel") >= 2 and "bigvgan_conv_post_kernel" in log
