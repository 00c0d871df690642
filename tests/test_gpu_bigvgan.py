"""BigVGAN v2 on the H100: the dilated and the polyphase-transposed implicit convolutions of the wgmma GEMM against
float64 convolutions of the same bf16 operands, the anti-aliased activation kernel and the BigVGAN mel against their
float64 definitions, the composed decode against the restatement's emulated drift (tests/bigvgan_emul.py), and the
end-to-end sample() / generate() path."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

import bigvgan_emul as E
from helpers import rel
from kernel_check import U32, U_BF16

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _lib():
    from f5_tts_mlx_b200 import _lib
    return _lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _conv_gemm(a, w_packed, B, T, Cin, n, taps, pad, dil, bias):
    """out[B*T, n] fp32 = implicit conv of a bf16 [B*T, Cin] with w_packed bf16 [n, taps * kp]."""
    L = _lib()
    out = torch.full((B * T, n), float("nan"), device=DEV)
    g = L.GemmArgsDilated()
    g.a, g.lda, g.w, g.ldw = a.data_ptr(), Cin, w_packed.data_ptr(), w_packed.shape[1]
    g.m, g.n, g.k = B * T, n, Cin
    g.rows_per_batch, g.num_batches, g.batched_tiles = T, B, 1
    g.conv_taps, g.conv_pad, g.conv_dilation = taps, pad, dil
    g.bias, g.out, g.ldo, g.q_scale = bias.data_ptr(), out.data_ptr(), n, 1.0
    L.check(L.load().f5_gemm_bf16(C.cast(C.pointer(g), C.POINTER(L.GemmArgs)), _stream()))
    torch.cuda.synchronize()
    return out


def _bound(a64, w64, ref, K, fn):
    """|err| <= (K + 2) u32 * (|a| * |w| conv) + u32 |ref|: fp32 accumulation of K products, one fp32 rounding."""
    return (K + 2) * U32 * fn(a64.abs(), w64.abs()) + U32 * ref.abs() + 1e-30


def _tap_major(w, kp):
    from f5_tts_mlx_b200.bigvgan import _tap_major
    return _tap_major(w, kp)


RELEASED_CONVS = sorted({(c, k, d) for c in (768, 384, 192, 96, 48, 24) for k in (3, 7, 11) for d in (1, 3, 5)})


@pytest.mark.parametrize("C_,k,d", RELEASED_CONVS)
def test_dilated_conv_gemm(C_, k, d):
    """Every (channels, kernel, dilation) the released config launches, two utterances of 200 frames (ragged tile
    edges: the zero padding must stay inside each utterance)."""
    g = torch.Generator().manual_seed(C_ * 100 + k * 10 + d)
    B, T = 2, 200
    x = torch.randn(B, C_, T, generator=g).bfloat16()
    w = (torch.randn(C_, C_, k, generator=g) / math.sqrt(C_ * k)).bfloat16()
    bias = torch.randn(C_, generator=g)
    pad = (k * d - d) // 2
    x64, w64 = x.double(), w.double()
    ref = F.conv1d(x64, w64, bias.double(), dilation=d, padding=pad)                    # (B, C, T)
    bnd = _bound(x64, w64, ref, C_ * k, lambda a, ww: F.conv1d(a, ww, dilation=d, padding=pad) + bias.double().abs()[None, :, None])
    a = x.transpose(1, 2).reshape(B * T, C_).contiguous().to(DEV)
    wp = _tap_major(w.float().permute(0, 2, 1), -(-C_ // 64) * 64).to(DEV)
    got = _conv_gemm(a, wp, B, T, C_, C_, k, pad, d, bias.to(DEV)).cpu().double().reshape(B, T, C_).transpose(1, 2)
    err = (got - ref).abs()
    assert torch.isfinite(got).all()
    assert (err <= bnd).all(), f"max err/bound {(err / bnd).max().item():.3g}"


@pytest.mark.parametrize("cin,k,u", [(1536, 8, 4), (768, 8, 4), (384, 4, 2), (192, 4, 2), (96, 4, 2), (48, 4, 2)])
def test_transposed_conv_polyphase_gemm(cin, k, u):
    from f5_tts_mlx_b200.bigvgan import pack_polyphase
    g = torch.Generator().manual_seed(cin + k + u)
    B, T, cout = 2, 150, cin // 2
    x = torch.randn(B, cin, T, generator=g).bfloat16()
    w = (torch.randn(cin, cout, k, generator=g) / math.sqrt(cin)).bfloat16()
    bias = torch.randn(cout, generator=g)
    p = (k - u) // 2
    x64, w64 = x.double(), w.double()
    ref = F.conv_transpose1d(x64, w64, bias.double(), stride=u, padding=p)            # (B, cout, u T)
    bnd = _bound(x64, w64, ref, cin * k, lambda a, ww: F.conv_transpose1d(a, ww, stride=u, padding=p) + bias.double().abs()[None, :, None])
    pw, taps, pad = pack_polyphase(w.float(), u)
    wp = _tap_major(pw, -(-cin // 64) * 64).to(DEV)
    a = x.transpose(1, 2).reshape(B * T, cin).contiguous().to(DEV)
    got = _conv_gemm(a, wp, B, T, cin, u * cout, taps, pad, 1, bias.repeat(u).to(DEV))
    got = got.cpu().double().reshape(B, u * T, cout).transpose(1, 2)
    err = (got - ref).abs()
    assert (err <= bnd).all(), f"max err/bound {(err / bnd).max().item():.3g}"


def _act_tables(Cn, beta: bool, logscale: bool, seed: int):
    from f5_tts_mlx_b200.bigvgan import kaiser_sinc_filter1d
    g = torch.Generator().manual_seed(seed)
    raw_a = 0.3 * torch.randn(Cn, generator=g) + (0.0 if logscale else 1.0)
    raw_b = 0.3 * torch.randn(Cn, generator=g) + (0.0 if logscale else 1.0)
    f = (lambda t: torch.exp(t.double()).float()) if logscale else (lambda t: t)
    h = kaiser_sinc_filter1d()
    hd = h * (1 + 0.05 * torch.randn(12, generator=g))                  # different up / down filters
    return {"alpha": f(raw_a), "h_up": h, "h_down": hd, **({"beta": f(raw_b)} if beta else {})}


@pytest.mark.parametrize("beta", [False, True])
@pytest.mark.parametrize("logscale", [False, True])
@pytest.mark.parametrize("Cn", [24, 48, 96, 768])
def test_activation_kernel(Cn, beta, logscale):
    """Every T in {1, 2, 3, 5, 6, 7, 8, 33, 1000} as the second utterance of a launch whose first one has 70 frames, in
    both output types, against Activation1d in float64."""
    from f5_tts_mlx_b200.bigvgan import act_struct
    L = _lib()
    tabs = _act_tables(Cn, beta, logscale, Cn + 2 * beta + logscale)
    dt = {k: v.to(DEV) for k, v in tabs.items()}
    st = act_struct(dt)
    al = tabs["alpha"].double()
    be = tabs["beta"].double() if beta else al
    for T in (1, 2, 3, 5, 6, 7, 8, 33, 1000):
        g = torch.Generator().manual_seed(T)
        lens = [70, T]
        rpb = max(lens)
        x = 2.0 * torch.randn(2, rpb, Cn, generator=g)
        xd, ld = x.to(DEV), torch.tensor(lens, dtype=torch.int32, device=DEV)     # held: the launch reads them
        for out_bf16 in (0, 1):
            out = torch.full((2, rpb, Cn), float("nan"), device=DEV, dtype=torch.bfloat16 if out_bf16 else torch.float32)
            L.check(L.load().f5_bigvgan_act_forward(
                C.c_void_p(xd.data_ptr()), 2, rpb, Cn, C.c_void_p(ld.data_ptr()),
                C.byref(st), out_bf16, C.c_void_p(out.data_ptr()), _stream()))
            torch.cuda.synchronize()
            got = out.cpu().double()
            for u, n in enumerate(lens):
                xs = x[u, :n].double().t()[None]
                ref = E.activation1d(xs, tabs["alpha"], tabs.get("beta"), tabs["h_up"], tabs["h_down"])[0].t()
                # fp32 arithmetic: ~36 roundings on values of size |x| + |a|; sin(alpha u) moves by alpha |du|
                scale = (xs.abs().max() + ref.abs().max() + 1.0)
                bnd = 64 * U32 * (1 + al * (1 + 1.0 / be)) * scale
                if out_bf16:
                    bnd = bnd + U_BF16 * ref.abs()
                err = (got[u, :n] - ref).abs()
                assert (err <= bnd).all(), f"T={T} utt {u} out_bf16={out_bf16}: max err/bound {(err / bnd).max().item():.3g}"
                if n < rpb:
                    assert torch.isnan(got[u, n:]).all(), "rows past the utterance were written"


def test_bigvgan_mel_matches_definition_and_torch_stft():
    from f5_tts_mlx_b200.bigvgan import bigvgan_mel_spectrogram, slaney_filterbank
    g = torch.Generator().manual_seed(3)
    for t in (385, 1000, 24000 * 2 + 17):
        wave = 0.3 * torch.randn(2, t, generator=g)
        got = bigvgan_mel_spectrogram(wave.to(DEV)).cpu().double()
        ref = E.mel(wave, E.slaney_filterbank())
        assert got.shape == ref.shape == (2, (t + 768 - 1024) // 256 + 1, 100)
        assert (got - ref).abs().max().item() < 2e-3
        # torch.stft on CUDA of the reflect-padded wave, the same filterbank
        xp = F.pad(wave.to(DEV)[:, None], (384, 384), mode="reflect")[:, 0]
        spec = torch.stft(xp, 1024, 256, 1024, torch.hann_window(1024, device=DEV), center=False, return_complex=True)
        mag = torch.sqrt(spec.real ** 2 + spec.imag ** 2 + 1e-9)
        st = torch.log(torch.clamp(slaney_filterbank().to(DEV) @ mag, min=1e-5)).transpose(1, 2)
        assert (got - st.cpu().double()).abs().max().item() < 2e-3
    with pytest.raises(ValueError):
        bigvgan_mel_spectrogram(torch.zeros(384, device=DEV))


SMALL = dict(num_mels=100, upsample_rates=(4, 2), upsample_kernel_sizes=(8, 4), upsample_initial_channel=128,
             resblock="1", resblock_kernel_sizes=(3, 7), resblock_dilation_sizes=((1, 3, 5), (1, 3, 5)),
             activation="snake", snake_logscale=False, use_tanh_at_final=True, use_bias_at_final=True)


@pytest.mark.parametrize("which", ["small", "released"])
def test_decode_against_emulated_drift_and_batch_isolation(which):
    from f5_tts_mlx_b200.bigvgan import BigVGAN, BigVGANConfig, random_bigvgan_weights
    cfg = BigVGANConfig.from_dict(SMALL) if which == "small" else BigVGANConfig()
    sd = random_bigvgan_weights(cfg, seed=11)
    voc = BigVGAN(cfg, DEV).load_weights(sd)
    g = torch.Generator().manual_seed(5)
    for b, n in ((1, 9), (2, 6)):
        mel = torch.randn(b, n, cfg.num_mels, generator=g) - 3.0
        got = voc.decode(mel.to(DEV))
        got = (got[None] if b == 1 else got).cpu().double()
        assert got.shape == (b, n * cfg.hop_length) and torch.isfinite(got).all()
        ref = E.generator(mel, sd, cfg)
        emu = E.generator(mel, sd, cfg, emulate=True)
        assert (ref.abs() >= 1).double().mean() < 0.01, "random weights saturate the output"
        r_emu, r_got = rel(emu, ref), rel(got, ref)
        assert r_got <= 3 * r_emu + 1e-6, f"{which} b={b}: drift {r_got:.3g} vs emulated {r_emu:.3g}"
        if b > 1:
            for i in range(b):
                alone = voc.decode(mel[i:i + 1].to(DEV)).cpu().double()
                assert torch.equal(alone, got[i]), f"row {i} differs from decoding it alone"


def test_sample_and_generate_with_bigvgan(tmp_path):
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.bigvgan import BigVGANMelSpec
    from f5_tts_mlx_b200.generate import generate, write_wav
    f5 = F5TTS.from_pretrained("random", model_version="v0", vocoder="bigvgan")
    assert isinstance(f5._mel_spec, BigVGANMelSpec) and f5._duration_predictor is None
    g = torch.Generator().manual_seed(1)
    ref = 0.1 * torch.randn(256 * 40 + 100, generator=g)
    wave, _ = f5.sample(ref[None].to(DEV), ["hello there"], duration=90, steps=2, method="euler", seed=0,
                        return_trajectory=False)
    assert wave.shape == (90 * 256,) and torch.isfinite(wave).all()
    path = tmp_path / "ref.wav"
    write_wav(str(path), ref)
    out = generate("Hello world.", duration=1.0, ref_audio_path=str(path), ref_audio_text="hi", steps=2, method="euler",
                   seed=0, f5tts=f5, model_version="v0", vocoder="bigvgan")
    frames = int(1.0 * 24000 / 256)
    assert out.shape == (frames * 256 - ref.shape[0],) and torch.isfinite(out).all()
