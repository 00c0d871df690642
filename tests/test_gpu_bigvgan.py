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
from composed_check import assert_rows
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


@pytest.mark.parametrize("out_bf16", [0, 1])
@pytest.mark.parametrize("nk", [1, 2, 3, 4])
def test_resblock_mean_kernel_bitwise(nk, out_bf16):
    """f5_bigvgan_resblock_mean: n in {1, 255, 257, 70001} (none a multiple of the 256-thread block), the nk streams
    stride = n + 37 apart with NaN in the gaps, out written into a NaN-filled buffer.  The kernel adds the streams in
    order in fp32 and divides once; the library is built without fast-math, so that is IEEE division, the same rounding
    as torch's fp32 `/` on the CPU.  The result must equal it bitwise (bf16: its round-to-nearest), and nothing past n
    may be written."""
    from kernel_check import assert_exact
    L = _lib()
    for n in (1, 255, 257, 70001):
        g = torch.Generator().manual_seed(n * 8 + nk)
        stride = n + 37
        xk = torch.full((nk, stride), float("nan"))
        xk[:, :n] = torch.randn(nk, n, generator=g) * torch.exp2(torch.randint(-8, 9, (nk, n), generator=g).float())
        s = xk[0, :n].clone()
        for j in range(1, nk):
            s = s + xk[j, :n]
        want = s / torch.tensor(float(nk))
        odt = torch.bfloat16 if out_bf16 else torch.float32
        want = want.to(odt)
        xd = xk.to(DEV)
        out = torch.full((n + 300,), float("nan"), device=DEV, dtype=odt)
        L.check(L.load().f5_bigvgan_resblock_mean(C.c_void_p(xd.data_ptr()), stride, nk, n, out_bf16,
                                                  C.c_void_p(out.data_ptr()), _stream()))
        torch.cuda.synchronize()
        got = out.cpu()
        assert_exact(got[:n][None], want[None], lambda r, c: f"element {c}", f"mean nk={nk} n={n} out_bf16={out_bf16}")
        assert torch.isnan(got[n:].float()).all(), f"n={n}: elements past n were written"


# the CUDA C Programming Guide (Mathematical Functions, single precision): tanhf has a maximum error of 2 ulp
TANHF_ULP = 2


def _conv_post_ref(x64, w64, bias):
    """float64 Conv1d(C, 1, 7, padding=3) of each utterance alone (zero padding at its edges) + bias: [B, T] and the
    same of |x| |w| (the accumulation bound's sum)."""
    xt, wt = x64.transpose(1, 2), w64.t()[None]                   # [B, C, T], [1, C, 7]
    acc = F.conv1d(xt, wt, padding=3)[:, 0]
    mag = F.conv1d(xt.abs(), wt.abs(), padding=3)[:, 0]
    if bias is not None:
        acc = acc + bias.double()[0]
        mag = mag + bias.double().abs()[0]
    return acc, mag


@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("Cn", [24, 32])
@pytest.mark.parametrize("use_tanh", [0, 1], ids=["clamp", "tanh"])
def test_conv_post_kernel(use_tanh, Cn, bias):
    """f5_bigvgan_conv_post at B = 3 utterances of T in {1, 2, 3, 4, 7, 255, 256, 257, 1000} frames, out written into a
    NaN-filled buffer that must stay NaN past B T.

    clamp (the released config): x integers in [-4, 4], w and the bias multiples of 2^-10 at most 2^-5 and 2^-2: every
    partial sum is a multiple of 2^-10 below 2^10 (7 C |x| |w| <= 28), so the fp32 result is exact in any order and the output
    must equal clamp(float64 conv, -1, 1) bitwise, the zero padding at every utterance edge included (a frame read
    from the neighbouring utterance would change it).
    tanh: x and w Gaussian.  The fp32 accumulation of the 7 C products (fma, one rounding each) and the bias add are
    within (7 C + 2) u sum |w||x| of the float64 sum; tanh' <= 1 carries that through, and tanhf adds TANHF_ULP ulp
    (<= 2^-23 |tanh| each) of its result."""
    from kernel_check import assert_exact, assert_within
    L = _lib()
    inside = saturated = 0
    for T in (1, 2, 3, 4, 7, 255, 256, 257, 1000):
        B = 3
        g = torch.Generator().manual_seed(T * 100 + Cn + 2 * bias + use_tanh)
        if use_tanh:
            x = torch.randn(B, T, Cn, generator=g)
            w = torch.randn(7, Cn, generator=g) / (7 * Cn) ** 0.5
            b = torch.randn(1, generator=g) * 0.1 if bias else None
        else:
            x = torch.randint(-4, 5, (B, T, Cn), generator=g).float()
            w = torch.randint(-32, 33, (7, Cn), generator=g).float() / 1024
            b = torch.randint(-256, 257, (1,), generator=g).float() / 1024 if bias else None
        acc, mag = _conv_post_ref(x.double(), w.double(), b)
        xd, wd = x.to(DEV), w.to(DEV)
        bd = b.to(DEV) if b is not None else None
        out = torch.full((B * T + 300,), float("nan"), device=DEV)
        L.check(L.load().f5_bigvgan_conv_post(C.c_void_p(xd.data_ptr()), B, T, Cn, C.c_void_p(wd.data_ptr()),
                                              C.c_void_p(bd.data_ptr()) if bd is not None else None, use_tanh,
                                              C.c_void_p(out.data_ptr()), _stream()))
        torch.cuda.synchronize()
        got = out.cpu()
        assert torch.isnan(got[B * T:]).all(), f"T={T}: samples past batch * frames were written"
        got = got[:B * T].view(B, T)
        loc = lambda r, c: f"utterance {r} frame {c}"
        what = f"conv_post {'tanh' if use_tanh else 'clamp'} C={Cn} bias={bias} T={T}"
        if use_tanh:
            ref = torch.tanh(acc)
            bnd = (7 * Cn + 2) * U32 * mag + TANHF_ULP * 2.0 ** -23 * ref.abs() + 2.0 ** -149
            assert_within(got, ref, bnd, loc, what)
        else:
            assert (mag < 2 ** 10).all() and torch.equal(acc.float().double(), acc)
            assert_exact(got, acc.clamp(-1, 1).float(), loc, what)
            inside += int(((acc.abs() < 1) & (acc != 0)).sum())
            saturated += int((acc.abs() > 1).sum())
    if not use_tanh:   # both sides of the clamp are reached
        assert inside > 4 * saturated > 0, (inside, saturated)


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


def _vocoder(which):
    from f5_tts_mlx_b200.bigvgan import BigVGAN, BigVGANConfig, random_bigvgan_weights
    cfg = BigVGANConfig.from_dict(SMALL) if which == "small" else BigVGANConfig()
    sd = random_bigvgan_weights(cfg, seed=11)
    return cfg, sd, BigVGAN(cfg, DEV).load_weights(sd)


def _decode_vs_emulated(cfg, sd, voc, mel, what):
    """decode(mel) [b, n hop] against the float64 restatement, hop segment by hop segment ([1, b, n, hop]: every
    segment within 3x the worst segment of the emulated drift, every utterance within the per-utterance rel rule), so
    damage in the first or last segments of an utterance is not diluted by the rest."""
    b, n = mel.shape[:2]
    got = voc.decode(mel.to(DEV))
    got = (got[None] if b == 1 else got).cpu().double()
    assert got.shape == (b, n * cfg.hop_length) and torch.isfinite(got).all()
    ref = E.generator(mel, sd, cfg)
    emu = E.generator(mel, sd, cfg, emulate=True)
    assert (ref.abs() >= 1).double().mean() < 0.01, "random weights saturate the output"
    seg = lambda t: t.reshape(1, b, n, cfg.hop_length)
    rep = assert_rows(seg(got), seg(ref), seg(emu), what=what)
    print(f"{what}: {rep}")
    return got


@pytest.mark.parametrize("which", ["small", "released"])
def test_decode_against_emulated_drift_and_batch_isolation(which):
    cfg, sd, voc = _vocoder(which)
    g = torch.Generator().manual_seed(5)
    for b, n in ((1, 9), (2, 6)):
        mel = torch.randn(b, n, cfg.num_mels, generator=g) - 3.0
        got = _decode_vs_emulated(cfg, sd, voc, mel, f"{which} b={b} n={n}")
        if b > 1:
            for i in range(b):
                alone = voc.decode(mel[i:i + 1].to(DEV)).cpu().double()
                assert torch.equal(alone, got[i]), f"row {i} differs from decoding it alone"


@pytest.mark.parametrize("which,n", [("small", 1), ("small", 2), ("small", 9), ("small", 64), ("released", 6),
                                     ("released", 16)])
def test_decode_edge_lengths(which, n):
    """B = 2 at n mel frames: below every conv's reach (n = 1, 2; the released stage 0 runs at T = 4 n), and across
    the GEMM's 128-row tiles at the later stages (the small config's n = 64 runs its last stage at T = 512)."""
    cfg, sd, voc = _vocoder(which)
    g = torch.Generator().manual_seed(100 + n)
    mel = torch.randn(2, n, cfg.num_mels, generator=g) - 3.0
    _decode_vs_emulated(cfg, sd, voc, mel, f"{which} b=2 n={n}")


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
