"""-m gpu: speech editing (F5TTS.sample(edit_mask=), f5_tts_mlx_b200.edit) on the H100.

  * edit_mask=None and an all-True mask are bitwise the same solve; a prefix-shaped mask is bitwise the matching lens=;
  * kept frames come back bitwise as cond, regenerated frames are finite and new, and stay within 3x the drift of the
    restatement's bf16 emulation (tests/edit_emul.py) on the gate and base DiTs, v0, the small E2 config, Euler and
    midpoint CFG and a ragged batch of two clips with different edits;
  * frame bucketing, block-scaled FP8, plan and CUDA-graph reuse;
  * speech_edit end to end through from_pretrained("random"), v1 (by the CLI) and E2, and the level restore.
"""
import functools

import pytest
import torch

from helpers import make_dit, ocfg_of, rel, synth_audio
from oracle import f5_oracle as O
import edit_emul as E
import unett_emul as U
import v0_emul as V

pytestmark = pytest.mark.gpu
DEV = "cuda"


def within_drift(got, ref, ref16, factor=3.0, floor=2e-3):
    drift, r = rel(ref16, ref), rel(got, ref)
    assert torch.isfinite(got).all() and r < max(factor * drift, floor), f"rel {r:.3e} vs bf16 drift {drift:.3e}"
    return r, drift


@pytest.fixture(scope="module")
def gate():
    from f5_tts_mlx_b200.weights import GATE_CONFIG, random_dit_weights
    W = random_dit_weights(GATE_CONFIG, seed=1234)
    return GATE_CONFIG, W, make_dit(GATE_CONFIG, W)


@pytest.fixture(scope="module")
def base():
    from f5_tts_mlx_b200.weights import BASE_CONFIG, random_dit_weights
    W = random_dit_weights(BASE_CONFIG, seed=1234)
    return BASE_CONFIG, W, make_dit(BASE_CONFIG, W)


def _v0_dit(cfg, W):
    from f5_tts_mlx_b200 import DiT
    return DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
               text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers, device=DEV,
               text_mask_padding=False, pe_attn_head=1).load_weights(W)


def _e2_small():
    from f5_tts_mlx_b200.unett import UNetT, UNetTConfig, random_unett_weights
    cfg = UNetTConfig(dim=256, depth=4, heads=4, ff_mult=4)
    W = random_unett_weights(cfg, seed=11)
    net = UNetT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, text_num_embeds=cfg.text_num_embeds,
                text_dim=cfg.text_dim, pe_attn_head=cfg.pe_attn_head, device=DEV).load_weights(W)
    return cfg, W, net


def _clip(B, nc, nt, seed, gaps):
    """cond [B, nc, 100], text [B, nt] and the edit mask [B, nc] with gaps[b] = [(first, last + 1), ...] False."""
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(B, nc, 100, generator=g) * 2.24 - 1.27
    text = torch.randint(0, 2545, (B, nt), generator=g, dtype=torch.int32)
    em = torch.ones(B, nc, dtype=torch.bool)
    for b, row in enumerate(gaps):
        for s, e in row:
            em[b, s:e] = False
    return cond, text, em, g


def _check_kept_and_gaps(out, cond, em):
    out = out.cpu()[:, : cond.shape[1]]
    assert torch.equal(out[em], cond[em]), "kept frames are not bitwise cond"
    gap = out[~em]
    assert torch.isfinite(gap).all() and ((gap - cond[~em]).abs().amax(-1) > 1e-3).all()


# ---------------------------------------------------------------- bitwise identities
@pytest.mark.parametrize("nc,nt", [(200, 60), (40, 70)])          # (40, 70): text longer than the clip
def test_all_true_mask_is_bitwise_no_mask(gate, nc, nt):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, model = gate
    cond, text, _, g = _clip(1, nc, nt, seed=nc, gaps=[[]])
    N = nc + 60
    kw = dict(steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0, y0=torch.randn(1, N, 100, generator=g))
    f5 = F5TTS(model)
    a, ta = f5.sample(cond.to(DEV), text, N, **kw)
    b, tb = f5.sample(cond.to(DEV), text, N, edit_mask=torch.ones(1, nc, dtype=torch.bool), **kw)
    assert torch.equal(a, b) and torch.equal(ta, tb)


def test_prefix_mask_is_bitwise_lens(gate):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, model = gate
    cond, text, _, g = _clip(1, 200, 60, seed=3, gaps=[[]])
    N, l = 260, 120
    kw = dict(steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0, y0=torch.randn(1, N, 100, generator=g))
    f5 = F5TTS(model)
    a, ta = f5.sample(cond.to(DEV), text, N, lens=torch.tensor([float(l)]), **kw)
    b, tb = f5.sample(cond.to(DEV), text, N, edit_mask=(torch.arange(200) < l)[None], **kw)
    assert torch.equal(a, b) and torch.equal(ta, tb)


# ---------------------------------------------------------------- against the restatement
CASES = {
    #  name: (backbone, method, steps, B, nc, nt, durations, gaps per utterance)
    "gate-euler": ("gate", "euler", 4, 1, 200, 60, [201], [[(40, 70), (120, 150)]]),
    "base-euler": ("base", "euler", 4, 1, 200, 60, [201], [[(40, 70), (120, 150)]]),
    "gate-midpoint": ("gate", "midpoint", 3, 1, 200, 60, [201], [[(0, 25), (170, 200)]]),
    "v0-gate": ("v0", "euler", 4, 1, 200, 60, [201], [[(40, 70), (120, 150)]]),
    "e2-small": ("e2", "euler", 4, 1, 200, 60, [201], [[(40, 70), (120, 150)]]),
    "gate-ragged": ("gate", "euler", 4, 2, 150, 50, [211, 151], [[(30, 60)], [(10, 20), (90, 140)]]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_edit_vs_restatement(case, request):
    from f5_tts_mlx_b200 import F5TTS
    which, method, steps, B, nc, nt, durs, gaps = CASES[case]
    forward = O.dit_forward
    if which == "e2":
        cfg, W, model = _e2_small()
        ocfg = cfg
        forward = U.unett_forward
    elif which == "v0":
        cfg, W, _ = request.getfixturevalue("gate")
        model, ocfg = _v0_dit(cfg, W), V.ocfg_v0(cfg)
        forward = functools.partial(V.dit_forward, pe_attn_head=1)
    else:
        cfg, W, model = request.getfixturevalue(which)
        ocfg = ocfg_of(cfg)
    cond, text, em, g = _clip(B, nc, nt, seed=17, gaps=gaps)
    if B > 1:
        text[1, nt - 13:] = -1
    dur = torch.tensor(durs)
    N = int(dur.max())
    y0 = torch.randn(B, N, 100, generator=g)
    for b in range(B):
        y0[b, int(dur[b]):] = 0
    kw = dict(steps=steps, method=method, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
    out, _ = F5TTS(model).sample(cond.to(DEV), text, dur, edit_mask=em, **kw)
    ref, _ = E.sample(cond, text, dur, W, ocfg, edit_mask=em, forward=forward, **kw)
    ref16, _ = E.sample(cond, text, dur, W, ocfg, edit_mask=em, forward=forward, prec=O.Precision(True), **kw)
    assert out.shape == ref.shape == (B, N, 100)
    _check_kept_and_gaps(out, cond, em)
    regen = torch.arange(N)[None] < dur[:, None]                        # each utterance's frames: its gaps and
    regen[:, :nc] &= ~em                                                 # every frame past the clip
    r, drift = within_drift(out.cpu()[regen], ref[regen], ref16[regen])
    print(f"{case}: regenerated frames rel {r:.3e}, bf16 drift {drift:.3e}")


def test_bucketed_plan_serves_two_edit_lengths(gate):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, model = gate
    kw = dict(steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0)
    exact, bucketed = F5TTS(model), F5TTS(model)
    bucketed.frame_bucket = 128
    plans = set()
    for nc, gaps in ((150, [(20, 45)]), (230, [(60, 100), (200, 230)])):
        cond, text, em, g = _clip(1, nc, 40, seed=nc, gaps=[gaps])
        y0 = torch.randn(1, nc + 1, 100, generator=g)
        a, _ = exact.sample(cond.to(DEV), text, nc + 1, edit_mask=em, y0=y0, **kw)
        b, _ = bucketed.sample(cond.to(DEV), text, nc + 1, edit_mask=em, y0=y0, **kw)
        plans.add(id(bucketed.last_plan))
        assert b.shape == a.shape == (1, nc + 1, 100)
        assert rel(b, a) < 1e-3, (nc, rel(b, a))
        _check_kept_and_gaps(b, cond, em)
    assert len(plans) == 1 and bucketed.last_plan.session.frames == 256


def test_block_fp8_edit_keeps_frames_exactly(gate):
    from f5_tts_mlx_b200 import DiT, F5TTS
    cfg, W, _ = gate
    model = DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
                text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers, device=DEV,
                fp8=True, fp8_scaling="block").load_weights(W)
    cond, text, em, _ = _clip(1, 200, 60, seed=5, gaps=[[(40, 70), (120, 150)]])
    out, _ = F5TTS(model).sample(cond.to(DEV), text, 201, edit_mask=em, steps=4, method="euler", seed=2)
    assert torch.isfinite(out).all()
    _check_kept_and_gaps(out, cond, em)


def test_edit_after_plain_call_adds_no_plan_and_no_capture(gate):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, model = gate
    cond, text, em, _ = _clip(1, 200, 60, seed=8, gaps=[[(40, 70)]])
    f5 = F5TTS(model)
    kw = dict(steps=4, method="euler", cfg_strength=2.0, seed=1, return_trajectory=False)
    plain, _ = f5.sample(cond.to(DEV), text, 201, **kw)
    plan, graph, n_plans = f5.last_plan, f5.last_plan.graph, len(f5._plans)
    assert graph is not None
    edited, _ = f5.sample(cond.to(DEV), text, 201, edit_mask=em, **kw)
    assert f5.last_plan is plan and plan.graph is graph and len(f5._plans) == n_plans
    _check_kept_and_gaps(edited, cond, em)
    assert not torch.equal(edited[:, 70:], plain[:, 70:])                # the solve saw the new conditioning


# ---------------------------------------------------------------- end to end
def test_speech_edit_cli_v1_random_writes_wav(tmp_path):
    """python -m f5_tts_mlx_b200.edit --model random on a 16 kHz clip: resampled to 24 kHz, two spans with new
    lengths; the WAV holds the edited wave's sample count."""
    from f5_tts_mlx_b200 import edit as ED
    from f5_tts_mlx_b200.generate import read_wav, write_wav
    src, out = tmp_path / "in.wav", tmp_path / "out.wav"
    write_wav(str(src), synth_audio(3 * 16000, seed=4), 16000)
    ED.main(["--audio", str(src), "--text", "Some call me nature, others call me mother nature.", "--edit", "0.5:1.0",
             "--edit", "2.0:2.5", "--fix-duration", "0.8", "--fix-duration", "0.3", "--output", str(out),
             "--model", "random", "--steps", "3", "--seed", "1"])
    expect = ED.edit_inputs(torch.zeros(3 * 24000), [(0.5, 1.0), (2.0, 2.5)], [0.8, 0.3])[0].shape[0]
    back, sr = read_wav(str(out))
    assert sr == 24000 and back.shape[0] == expect == 74400
    assert torch.isfinite(back).all() and float(back.abs().max()) > 0


@pytest.fixture(scope="module")
def e2_random():
    from f5_tts_mlx_b200 import F5TTS
    return F5TTS.from_pretrained("random", model_version="e2")


def test_speech_edit_e2_random_writes_wav(e2_random, tmp_path):
    from f5_tts_mlx_b200.edit import edit_inputs, speech_edit
    from f5_tts_mlx_b200.generate import read_wav, write_wav
    audio = synth_audio(2 * 24000, seed=6)
    parts = [(0.3, 0.7), (1.5, 2.0)]
    wave = speech_edit(e2_random, audio, 24000, "new words in the gaps.", parts, steps=3, seed=2)
    expect = edit_inputs(audio, parts)[0].shape[0]
    assert wave.shape == (expect,) and torch.isfinite(wave).all()
    write_wav(str(tmp_path / "e2.wav"), wave)
    back, sr = read_wav(str(tmp_path / "e2.wav"))
    assert sr == 24000 and back.shape[0] == expect


def test_quiet_clip_comes_back_at_its_level(e2_random):
    """A clip at RMS 0.01 is normalised to 0.1, edited, and scaled back by rms / 0.1: its output is the output of the
    same clip normalised beforehand (which speech_edit leaves as it is) times rms / 0.1, to fp32 rounding."""
    from f5_tts_mlx_b200.edit import speech_edit
    quiet = synth_audio(2 * 24000, seed=2) * 0.1
    rms = torch.sqrt(torch.mean(torch.square(quiet)))
    loud = quiet * 0.1 / rms                                             # exactly speech_edit's normalisation
    assert abs(rms.item() - 0.01) < 1e-6 and torch.sqrt(torch.mean(torch.square(loud))) >= 0.1
    kw = dict(steps=3, seed=5)
    parts = [(0.5, 1.1)]
    out_q = speech_edit(e2_random, quiet, 24000, "a few new words.", parts, **kw)
    out_n = speech_edit(e2_random, loud, 24000, "a few new words.", parts, **kw)
    assert torch.allclose(out_q, out_n * rms.to(out_n.device) / 0.1, rtol=1e-6, atol=1e-9)
    ratio = (out_q.norm() / out_n.norm()).item()
    assert abs(ratio - 0.1) < 1e-5, ratio
