"""-m gpu: the windowed-sinc resampler (csrc/resample.cu, f5_resample) against the float64 restatement
(tests/resample_emul.py) within a bound derived per output sample, against torchaudio on CUDA, on known answers, and
composed into F5TTS.sample() and generate()."""
import math
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import resample_emul as E
from test_resample import PAIR_IDS, PAIRS, lengths, wav_bytes

pytestmark = pytest.mark.gpu
dev = "cuda"
ROOT = Path(__file__).resolve().parent.parent


def _resample(x, orig, new):
    from f5_tts_mlx_b200 import resample
    return resample(x, orig, new)


def _signal(batch, L, seed):
    g = torch.Generator().manual_seed(seed)
    n = torch.arange(L, dtype=torch.float64)
    x = 0.3 * torch.randn(batch, L, generator=g, dtype=torch.float64)
    x += 0.4 * torch.sin(2 * np.pi * 0.01 * (1 + torch.arange(batch, dtype=torch.float64))[:, None] * n) + 0.05
    return x.float()


def _check(got: torch.Tensor, x32: torch.Tensor, orig, new, what):
    xs = x32.double().numpy()
    ref = E.resample(xs, orig, new)
    bound = E.error_bound(xs, orig, new)
    g = got.double().cpu().numpy()
    assert g.shape == ref.shape, (what, g.shape, ref.shape)
    err = np.abs(g - ref)
    bad = err > bound
    assert not bad.any(), (what, int(bad.sum()), float(err[bad].max()), float(bound[bad].min()))
    return err, bound


# ---------------------------------------------------------------- element-wise accuracy
@pytest.mark.parametrize("orig,new", PAIRS, ids=PAIR_IDS)
def test_kernel_matches_float64_emulation(orig, new):
    for L in lengths(orig, new) + [10 * orig]:
        for batch in (1, 3):
            x = _signal(batch, L, seed=L + batch)
            got = _resample(x.to(dev), orig, new)
            assert got.shape == (batch, math.ceil(new * L / orig))
            _check(got, x, orig, new, (L, batch))
            if batch == 3:                                            # rows are independent: each equals batch 1
                one = _resample(x[1].to(dev), orig, new)
                assert torch.equal(one, got[1])


@pytest.mark.parametrize("orig,new", PAIRS, ids=PAIR_IDS)
def test_kernel_matches_torchaudio_on_cuda(orig, new):
    """torchaudio's fp32 result carries its own table's error and its own accumulation (bounded like the kernel's):
    |kernel - torchaudio| <= 2 * bound + sum_k |h_torchaudio[p][k] - h[p][k]| |x[...]|, with h_torchaudio the fp32
    table torchaudio builds on the device (its rounding there differs from its CPU table's).  Its conv1d runs without
    cuDNN, whose algorithm choice (TF32, FFT or Winograd convolutions) has no error bound per output sample; torch's
    own CUDA convolution is an fp32 GEMM over the same products."""
    torchaudio = pytest.importorskip("torchaudio")
    from torchaudio.functional.functional import _get_sinc_resample_kernel
    L = 2 * orig + 17
    x = _signal(2, L, seed=7)
    with torch.backends.cudnn.flags(enabled=False):
        ta = torchaudio.functional.resample(x.to(dev), orig, new).double().cpu().numpy()
    g = math.gcd(orig, new)
    h_ta32, width = _get_sinc_resample_kernel(orig, new, g, device=torch.device(dev), dtype=torch.float32)
    h_ta32 = h_ta32.cpu()                                             # the table it builds on the device, as it runs
    O, N, w, taps, _ = E.geometry(orig, new)
    assert width == w and h_ta32.shape == (N, 1, taps)
    dh = (h_ta32.double() - torch.from_numpy(E.table(orig, new))[:, None]).abs()[:, 0].numpy()
    xs = x.double().numpy()
    p, idx, valid = E.gather_index(orig, new, L)
    table_err = (dh[p] * np.where(valid, np.abs(xs[..., np.clip(idx, 0, L - 1)]), 0.0)).sum(-1)
    got = _resample(x.to(dev), orig, new).double().cpu().numpy()
    bound = 2 * E.error_bound(xs, orig, new) + table_err
    assert ta.shape == got.shape
    assert np.all(np.abs(got - ta) <= bound), float((np.abs(got - ta) / bound).max())


# ---------------------------------------------------------------- known answers
@pytest.mark.parametrize("orig,new", [(44100, 24000), (48000, 24000), (24000, 48000), (11025, 24000),
                                      (24000, 11025), (8000, 24000)])
def test_constant_input_gives_the_phase_sums(orig, new):
    c, L = 0.625, 20 * orig // 100
    got = _resample(torch.full((L,), c, device=dev), orig, new).double().cpu().numpy()
    O, N, w, taps, _ = E.geometry(orig, new)
    h = E.table(orig, new)
    j = np.arange(got.shape[0])
    interior = (j // N * O - w >= 0) & (j // N * O - w + taps <= L)
    assert interior.sum() > got.shape[0] // 2
    expect = c * h.sum(axis=1)[j % N]
    bound = taps * 2.0 ** -24 * c * np.abs(h).sum(axis=1)[j % N]
    assert np.all(np.abs(got - expect)[interior] <= bound[interior])


def _tone_amplitude(y, f, rate):
    t = np.arange(y.shape[0]) / rate
    A = np.stack([np.sin(2 * np.pi * f * t), np.cos(2 * np.pi * f * t)], 1)
    (a, b), *_ = np.linalg.lstsq(A, y, rcond=None)
    return math.hypot(a, b)


def test_tone_in_the_passband_keeps_its_amplitude():
    """1 kHz, 48 -> 24 kHz: the output tone's amplitude is the filter's gain |H(1 kHz)| (to fp32 rounding), which
    is within the windowed sinc's passband ripple (1e-3) of 1."""
    orig, new, f = 48000, 24000, 1000.0
    n = np.arange(orig)
    x = torch.from_numpy(np.sin(2 * np.pi * f / orig * n)).float()
    y = _resample(x.to(dev), orig, new).double().cpu().numpy()
    O, N, w, taps, _ = E.geometry(orig, new)
    k = np.arange(taps)
    gain = abs(np.sum(E.table(orig, new)[0] * np.exp(-2j * np.pi * f / orig * (k - w))))
    assert abs(gain - 1.0) < 1e-3
    amp = _tone_amplitude(y[100:-100], f, new)
    y0 = y[100:-100]
    assert abs(amp - gain) < 1e-5, (amp, gain)
    assert abs(np.sqrt(np.mean(y0 ** 2)) * math.sqrt(2) - gain) < 1e-3


def test_tone_above_the_new_nyquist_is_removed():
    orig, new, f = 48000, 24000, 15000.0
    n = np.arange(orig)
    x = torch.from_numpy(np.sin(2 * np.pi * f / orig * n)).float()
    y = _resample(x.to(dev), orig, new).double().cpu().numpy()
    rms_in = float(x.double().pow(2).mean().sqrt())
    rms_out = float(np.sqrt(np.mean(y[100:-100] ** 2)))
    assert rms_out < 1e-2 * rms_in, (rms_out, rms_in)


def test_launches_are_bitwise_reproducible_and_alignment_free():
    x = _signal(2, 441_000, seed=3).to(dev)
    a = _resample(x, 44100, 24000)
    b = _resample(x, 44100, 24000)
    assert torch.equal(a, b)
    # a row that does not start on a 16-byte boundary stages the same window
    buf = torch.zeros(441_001, device=dev)
    buf[1:] = x[0]
    assert buf[1:].data_ptr() % 16 == 4
    assert torch.equal(_resample(buf[1:], 44100, 24000), a[0])
    # equal rates: the input itself, no launch
    assert _resample(x, 24000, 24000) is x


def test_entry_point_checks_its_arguments():
    import ctypes as C
    from f5_tts_mlx_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(1000, device=dev)
    out = torch.zeros(1000, device=dev)
    tab = torch.zeros(1 << 16, device=dev)
    ptr = lambda t: C.c_void_p(t.data_ptr())
    for n_out in (544, 546):                                          # ceil(80 * 1000 / 147) = 545
        assert lib.f5_resample(ptr(x), 1, 1000, 44100, 24000, ptr(tab), ptr(out), n_out, None) == -1
        assert b"out_samples" in lib.f5_last_error()
    assert lib.f5_resample(ptr(x), 1, 1000, 0, 24000, ptr(tab), ptr(out), 545, None) == -1
    assert lib.f5_resample(ptr(x), 1, 1000, 44100, 24000, None, ptr(out), 545, None) == -1
    assert lib.f5_resample(ptr(x), 1, 1000, 44101, 24000, ptr(tab), ptr(out), 545, None) == -1
    assert lib.f5_resample(ptr(x), 1, 1000, 44100, 24000, ptr(tab), ptr(out), 545, None) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------- composition
@pytest.fixture(scope="module")
def gate_model():
    from f5_tts_mlx_b200 import DiT, GATE_CONFIG
    from f5_tts_mlx_b200.weights import random_dit_weights
    cfg = GATE_CONFIG
    return DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
               text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers,
               device=torch.device(dev)).load_weights(random_dit_weights(cfg, seed=1234))


def test_sample_with_cond_sample_rate_equals_resample_then_sample(gate_model):
    from f5_tts_mlx_b200 import F5TTS
    g = torch.Generator().manual_seed(11)
    wave48 = (0.1 * torch.randn(2 * 256 * 60, generator=g)).to(dev)
    text = torch.randint(0, 2545, (1, 30), generator=g, dtype=torch.int32)
    n = 150
    y0 = torch.randn(1, n, 100, generator=g)
    kw = dict(steps=3, method="euler", cfg_strength=2.0, y0=y0)
    f5 = F5TTS(gate_model)
    a, _ = f5.sample(wave48[None], text, n, cond_sample_rate=48000, **kw)
    b, _ = f5.sample(_resample(wave48, 48000, 24000)[None], text, n, **kw)
    assert a.shape == b.shape == (1, n, 100)
    assert torch.equal(a, b)
    c, _ = f5.sample(_resample(wave48, 48000, 24000)[None], text, n, cond_sample_rate=24000, **kw)
    assert torch.equal(c, b)


@pytest.fixture(scope="module")
def random_f5():
    from f5_tts_mlx_b200 import F5TTS
    return F5TTS.from_pretrained("random")


def test_generate_resamples_the_reference_and_the_output(random_f5, tmp_path):
    from f5_tts_mlx_b200 import generate as G
    f5 = random_f5
    L = 44100
    g = np.random.default_rng(5)
    codes = np.clip(np.round(g.standard_normal(L) * 0.05 * 2 ** 23), -2 ** 23, 2 ** 23 - 1).astype(np.int64)
    (tmp_path / "ref44k.wav").write_bytes(wav_bytes(codes[:, None], "s24", 44100))
    kw = dict(duration=2.0, ref_audio_path=str(tmp_path / "ref44k.wav"), ref_audio_text="A reference.", steps=2,
              method="euler", seed=3, f5tts=f5, resample_ref_audio=True)
    w24 = G.generate("Hello there.", **kw)
    frames = int(2.0 * G.FRAMES_PER_SEC)
    stripped = math.ceil(80 * L / 147)
    assert w24.shape[0] == f5._vocoder.__self__.out_len(frames) - stripped
    out = tmp_path / "out48k.wav"
    w48 = G.generate("Hello there.", output_path=str(out), output_sample_rate=48000, **kw)
    back, sr = G.read_wav(str(out))
    assert sr == 48000 and back.shape[0] == w48.shape[0] == 2 * w24.shape[0]
    assert torch.equal(w48, _resample(w24, 24000, 48000))
    with pytest.raises(ValueError, match="sample rate of 24kHz"):
        G.generate("Hello there.", **{**kw, "resample_ref_audio": False})


def test_generate_24k_reference_is_unchanged_by_the_option(random_f5, tmp_path):
    from f5_tts_mlx_b200 import generate as G
    ref = 0.05 * torch.randn(24000, generator=torch.Generator().manual_seed(2))
    G.write_wav(str(tmp_path / "ref24k.wav"), ref)
    kw = dict(duration=2.0, ref_audio_path=str(tmp_path / "ref24k.wav"), ref_audio_text="A reference.", steps=2,
              method="euler", seed=3, f5tts=random_f5)
    a = G.generate("Hello there.", **kw)
    b = G.generate("Hello there.", resample_ref_audio=True, **kw)
    assert torch.equal(a, b)


# ---------------------------------------------------------------- compiler output
def test_resample_kernel_compiles_without_spills(tmp_path):
    """Both instantiations (table in shared memory / through the read-only cache) compile for sm_90a with the build's
    own flags to 0 spill bytes."""
    from f5_tts_mlx_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-cubin", str(ROOT / "f5_tts_mlx_b200" / "csrc" / "resample.cu"), "-o",
           str(tmp_path / "k.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'(.*?)Used \d+ registers", log, re.S):
        found[m[1]] = sum(int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", m[2]))
    assert len(found) == 2 and all("resample_kernel" in n for n in found), sorted(found)
    assert all(v == 0 for v in found.values()), found
