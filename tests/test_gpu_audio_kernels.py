"""-m gpu: the warp-FFT audio kernels (csrc/audio_vocos.cu, csrc/fft.cuh) through f5_mel_forward and f5_istft, every
output sample against a float64 restatement within the per-frame bounds derived in hbm_check.py.

An identity filterbank (n_mels = 513) exposes every FFT bin, including 0 and 512, which the HTK filterbank weights by
0 and 2.7e-6; signals with a DC offset and a (-1)^n component make those two bins dominant."""
import numpy as np
import pytest
import torch

from hbm_check import istft_frames_ref_bound, istft_ola_ref_bound, mel_ref_bound
from kernel_check import Guarded, assert_within
from test_gpu_hbm_kernels import WORST, call, note

pytestmark = pytest.mark.gpu
dev = "cuda"
COVERED = {"mel_kernel", "istft_frames_kernel", "istft_ola_kernel"}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    mine = {k: v for k, v in WORST.items() if k.startswith(("mel", "istft"))}
    if mine:
        print("\nworst err/bound per kernel and mode:")
        for k, v in sorted(mine.items()):
            print(f"  {k:48s} {v:.3g}")


def _signals(T, seed):
    g = torch.Generator().manual_seed(seed)
    n = torch.arange(T, dtype=torch.float64)
    out = []
    for b in range(2):
        x = 0.3 * (1 + b) + (0.2 - 0.1 * b) * (-1.0) ** n + 0.1 * torch.randn(T, generator=g, dtype=torch.float64) \
            + 0.25 * torch.sin(2 * np.pi * (300 + 500 * b) / 24000 * n)
        out.append(x)
    return torch.stack(out).float().to(dev)


@pytest.mark.parametrize("T", [256, 700, 1024, 1025, 127985])
@pytest.mark.parametrize("window", ["hann", "rect"])
@pytest.mark.parametrize("bank", ["identity", "htk"])
def test_mel(T, window, bank):
    from f5_tts_mlx_b200.audio import hanning, mel_filters
    hop = 256
    frames = T // hop
    audio = _signals(T, T)
    w = (hanning(1024) if window == "hann" else torch.ones(1024)).to(dev)
    filt = torch.eye(513) if bank == "identity" else mel_filters(24000, 1024, 100).T.contiguous()
    filt = filt.to(dev)
    n_mels = filt.shape[1]
    out = Guarded(2 * frames, n_mels, torch.float32, dev, lr=False)
    call("f5_mel_forward", audio, 2, T, w, filt, n_mels, hop, out.view, frames)
    out.check(f"mel T={T}")
    ref, b = mel_ref_bound(audio, w, filt, hop, frames)
    if bank == "identity":      # bins 0 and 512 dominate: they are really being checked
        mags = ref.view(2, frames, 513).exp()
        assert (mags[..., 0] > 10 * mags[..., 1:512].median()).all()
        assert (mags[..., 512] > 10 * mags[..., 1:512].median()).all()
    note(f"mel {bank} {window}", assert_within(out.view, ref, b, lambda r, c: f"(batch {r // frames}, frame "
                                               f"{r % frames}) bin {c}", f"mel T={T} {window} {bank}"))


def _h(rows, ldh, seed):
    """[log-mag | phase | pad]: log-magnitudes in [-3, 6] (above ln 100 they clip), phases in [-4, 4], including the
    DC and Nyquist bins (their imaginary parts must be ignored)."""
    g = torch.Generator().manual_seed(seed)
    h = torch.full((rows, ldh), float("nan"))
    h[:, :513] = torch.rand(rows, 513, generator=g) * 9 - 3
    h[:, 513:1026] = torch.rand(rows, 513, generator=g) * 8 - 4
    return h.to(dev)


def _istft(h, ldh, B, F, w, hop, norm_sq, trim, out_len):
    scratch = torch.empty(B * F, 1024, device=dev)
    out = Guarded(B, out_len, torch.float32, dev, lr=False)
    call("f5_istft", h, ldh, B, F, w, hop, norm_sq, trim, scratch, out.view, out_len)
    out.check("istft")
    return out.view


@pytest.mark.parametrize("F", [1, 2, 3, 4, 5, 937])
def test_istft_is_per_frame_irfft(F):
    """hop 1024 and a window of ones: the output is each frame's irfft, sample for sample."""
    B, ldh = 2, 1030
    h = _h(B * F, ldh, F)
    w = torch.ones(1024, device=dev)
    got = _istft(h, ldh, B, F, w, 1024, 0, 0, F * 1024)
    fr, bf = istft_frames_ref_bound(h, w)
    ref, b = istft_ola_ref_bound(fr, bf, w, B, F, 1024, False, 0, F * 1024)
    note("istft irfft", assert_within(got, ref, b, lambda r, c: f"(batch {r}, frame {c // 1024}) sample {c % 1024}",
                                      f"istft irfft F={F}"))


@pytest.mark.parametrize("F", [1, 2, 3, 4, 5, 937])
@pytest.mark.parametrize("norm_sq", [0, 1])
@pytest.mark.parametrize("trim", [0, 512])
def test_istft_overlap_add(F, norm_sq, trim):
    """The Vocos configuration: periodic Hann, hop 256, both envelope norms, trim 0 / 512; batch 2 (frames must not
    leak across utterances, whose magnitudes differ by e^2)."""
    from f5_tts_mlx_b200.audio import hanning
    B, ldh, hop = 2, 1028, 256
    out_len = (F - 1) * hop + 1024 - 2 * trim
    if out_len <= 0:
        pytest.skip("no samples left after trimming")
    h = _h(B * F, ldh, 100 + F)
    h[F:, :513] -= 2.0
    w = hanning(1024).to(dev)
    got = _istft(h, ldh, B, F, w, hop, norm_sq, trim, out_len)
    fr, bf = istft_frames_ref_bound(h, w)
    ref, b = istft_ola_ref_bound(fr, bf, w, B, F, hop, bool(norm_sq), trim, out_len)
    note(f"istft ola norm_sq={norm_sq}", assert_within(got, ref, b, lambda r, c: f"(batch {r}) sample {c}",
                                                       f"istft F={F} norm_sq={norm_sq} trim={trim}"))


def test_vocos_batch_equals_single_decodes():
    """Every Vocos stage works per row or per utterance, so a batch-2 decode equals two batch-1 decodes up to the
    GEMM's tile choice for the different row counts (the accumulation order along K does not depend on it)."""
    from f5_tts_mlx_b200.vocos import Vocos
    from f5_tts_mlx_b200.weights import VocosConfig, random_vocos_weights
    vc = VocosConfig()
    voc = Vocos(vc).load_weights(random_vocos_weights(vc, seed=4321))
    g = torch.Generator().manual_seed(5)
    mel = (torch.randn(2, 187, 100, generator=g) * 2.24 - 1.27).to(dev)
    both = voc(mel)
    for b in range(2):
        one = voc(mel[b:b + 1])
        err = (both[b] - one).abs().max().item()
        assert err <= 1e-5 * one.abs().max().item(), (b, err)
