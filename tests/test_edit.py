"""Speech editing on the CPU: edit_inputs known answers and refusals, the frame rule of edit_mask_frames and its length
against both mel front-ends, the test-side restatement (tests/edit_emul.py) pinned to the oracle's sample(), sample()'s
edit_mask refusals, the CLI's parsing, and the mask's sharding in parallel.sample_sharded (world size 2, gloo)."""
import functools
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import f5_oracle as O
import bigvgan_emul as B
import edit_emul as E
import unett_emul as U
import v0_emul as V
from f5_tts_mlx_b200.edit import edit_inputs, edit_mask_frames


def _ramp(n):
    return torch.arange(1, n + 1, dtype=torch.float32)        # every sample distinct and non-zero


# ---------------------------------------------------------------- edit_inputs
def test_one_part_known_answer():
    a = _ramp(50)                                              # 5 s at 10 Hz
    w, gaps = edit_inputs(a, [(1.0, 2.0)], sample_rate=10)
    assert torch.equal(w, torch.cat([a[:10], torch.zeros(10), a[20:]])) and gaps == [(10, 20)]


def test_two_parts_with_longer_and_shorter_new_durations():
    a = _ramp(50)
    w, gaps = edit_inputs(a, [(1.0, 2.0), (3.0, 3.5)], [1.5, 0.2], sample_rate=10)
    assert torch.equal(w, torch.cat([a[:10], torch.zeros(15), a[20:30], torch.zeros(2), a[35:]]))
    assert gaps == [(10, 25), (35, 37)]


def test_parts_at_the_start_and_at_the_end_of_the_clip():
    a = _ramp(50)
    w, gaps = edit_inputs(a, [(0.0, 0.5), (4.0, 5.0)], sample_rate=10)
    assert torch.equal(w, torch.cat([torch.zeros(5), a[5:40], torch.zeros(10)])) and gaps == [(0, 5), (40, 50)]


def test_known_answer_at_24khz_kept_samples_and_gaps_exact():
    """The issue's example spans on a 6 s clip: round(seconds · 24000) everywhere; without fix_duration each gap sits
    where its span was, kept samples are the input's bit for bit and the gaps are exactly zero."""
    a = torch.randn(6 * 24000, generator=torch.Generator().manual_seed(0))
    w, gaps = edit_inputs(a, [(1.42, 2.44), (4.04, 4.90)])
    assert gaps == [(34080, 58560), (96960, 117600)] and w.shape == a.shape
    keep = torch.ones(a.shape[0], dtype=torch.bool)
    for s, e in gaps:
        keep[s:e] = False
    assert torch.equal(w[keep], a[keep]) and torch.equal(w[~keep], torch.zeros(int((~keep).sum())))
    w2, gaps2 = edit_inputs(a, [(1.42, 2.44), (4.04, 4.90)], [0.5, 1.25])
    assert gaps2 == [(34080, 34080 + 12000), (34080 + 12000 + 38400, 34080 + 12000 + 38400 + 30000)]
    assert torch.equal(w2, torch.cat([a[:34080], torch.zeros(12000), a[58560:96960], torch.zeros(30000), a[117600:]]))


@pytest.mark.parametrize("parts,fix", [
    ([], None),                                   # nothing to edit
    ([(2.0, 3.0), (1.0, 1.5)], None),             # not sorted
    ([(1.0, 2.0), (1.5, 3.0)], None),             # overlapping
    ([(-0.1, 1.0)], None),                        # starts before the clip
    ([(1.0, 1.0)], None),                         # empty span
    ([(2.0, 1.0)], None),                         # end before start
    ([(4.0, 5.1)], None),                         # past the clip's end
    ([(float("nan"), 1.0)], None),
    ([(1.0, float("inf"))], None),
    ([(1.0, 2.0)], [1.0, 2.0]),                   # fix_duration: one entry per part
    ([(1.0, 2.0), (3.0, 4.0)], [1.0]),
    ([(1.0, 2.0)], [0.0]),                        # non-positive new durations
    ([(1.0, 2.0)], [-1.0]),
    ([(1.0, 2.0)], [float("nan")]),
    ([(1.0, 2.0)], [float("inf")]),
    ([(1.0, 2.0)], [1e-3]),                       # rounds to no sample at 10 Hz
])
def test_edit_inputs_refusals(parts, fix):
    with pytest.raises(ValueError):
        edit_inputs(_ramp(50), parts, fix, sample_rate=10)


def test_edit_inputs_refuses_a_multichannel_wave():
    with pytest.raises(ValueError, match="1-D"):
        edit_inputs(torch.zeros(2, 50), [(1.0, 2.0)], sample_rate=10)


# ---------------------------------------------------------------- edit_mask_frames
def test_frames_straddling_a_gap_boundary_are_regenerated():
    assert edit_mask_frames([(300, 600)], 4, 256).tolist() == [True, False, False, True]
    assert edit_mask_frames([(512, 768)], 4, 256).tolist() == [True, True, False, True]     # aligned: one frame
    assert edit_mask_frames([(511, 513)], 4, 256).tolist() == [True, False, False, True]
    assert edit_mask_frames([(0, 1), (1023, 1100)], 5, 256).tolist() == [False, True, True, False, False]
    assert edit_mask_frames([(700, 5000)], 4, 256).tolist() == [True, True, False, False]   # clipped at frames


def test_frame_rule_against_its_definition():
    g = np.random.default_rng(3)
    for _ in range(200):
        hop, frames = int(g.choice([4, 7, 256])), int(g.integers(0, 40))
        cuts = sorted(g.integers(0, frames * hop + 2 * hop, size=2 * int(g.integers(1, 4))).tolist())
        gaps = list(zip(cuts[0::2], cuts[1::2]))
        want = [not any(a < b and f * hop < b and a < (f + 1) * hop for a, b in gaps) for f in range(frames)]
        assert edit_mask_frames(gaps, frames, hop).tolist() == want


def test_edit_mask_frames_refusals():
    for gaps, frames, hop in (([(5, 3)], 4, 256), ([(-1, 3)], 4, 256), ([], -1, 256), ([], 4, 0)):
        with pytest.raises(ValueError):
            edit_mask_frames(gaps, frames, hop)


@pytest.mark.parametrize("clip,parts,fix", [(24000, [(0.2, 0.4)], None), (30011, [(0.0, 0.3), (1.0, 30011 / 24000)], [0.41, 0.2]),
                                            (12345, [(0.1, 0.11)], [0.0123])])
def test_mask_length_is_the_front_ends_frame_count(clip, parts, fix):
    """The mask has one entry per frame of the mel the model computes for the edited wave, for both front-ends: the
    oracle's Vocos-style log_mel_spectrogram (t // hop) and BigVGAN's (bigvgan_frames, restated in bigvgan_emul.mel);
    every gap's first frame lies inside it."""
    from f5_tts_mlx_b200.bigvgan import bigvgan_frames
    w, gaps = edit_inputs(torch.randn(clip, generator=torch.Generator().manual_seed(clip)), parts, fix)
    t = w.shape[0]
    vocos_frames, bigvgan_mel_frames = O.log_mel_spectrogram(w).shape[1], B.mel(w[None], B.slaney_filterbank()).shape[1]
    assert vocos_frames == t // 256 and bigvgan_mel_frames == bigvgan_frames(t)
    for frames in (vocos_frames, bigvgan_mel_frames):
        m = edit_mask_frames(gaps, frames, 256)
        assert m.shape == (frames,) and m.dtype == torch.bool
        assert all(not m[a // 256] for a, _ in gaps if a // 256 < frames)


# ---------------------------------------------------------------- the restatement, pinned to the oracle
@pytest.fixture(scope="module")
def tiny():
    from f5_tts_mlx_b200.weights import DiTConfig, random_dit_weights
    cfg = DiTConfig(dim=128, depth=2, heads=2, text_num_embeds=60, text_dim=64, conv_layers=1)
    W = random_dit_weights(cfg, seed=5)
    ocfg = O.DiTConfig(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult,
                       text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers)
    return W, ocfg


def _case(B_, nc, nt, seed):
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(B_, nc, 100, generator=g) * 2 - 1
    text = torch.randint(0, 60, (B_, nt), generator=g, dtype=torch.int32)
    return cond, text


KW = dict(steps=3, method="midpoint", cfg_strength=2.0, sway_sampling_coef=-1.0, seed=4)


def test_restatement_all_true_mask_is_the_oracle(tiny):
    W, ocfg = tiny
    cond, text = _case(2, 40, 50, seed=1)                      # text longer than the clip: lens = 50
    text[1, 30:] = -1
    dur = torch.tensor([70, 61])
    want, want_traj = O.sample(cond, text, dur, W, ocfg, **KW)
    got, traj = E.sample(cond, text, dur, W, ocfg, edit_mask=torch.ones(2, 40, dtype=torch.bool), **KW)
    assert torch.equal(got, want) and torch.equal(traj, want_traj)


def test_restatement_prefix_mask_is_the_oracle_with_lens(tiny):
    W, ocfg = tiny
    cond, text = _case(1, 40, 20, seed=2)
    want, want_traj = O.sample(cond, text, 60, W, ocfg, lens=torch.tensor([27.0]), **KW)
    got, traj = E.sample(cond, text, 60, W, ocfg, edit_mask=O.lens_to_mask(torch.tensor([27]), 40), **KW)
    assert torch.equal(got, want) and torch.equal(traj, want_traj)


def test_restatement_edit_keeps_cond_and_changes_the_gaps(tiny):
    W, ocfg = tiny
    cond, text = _case(1, 40, 20, seed=3)
    em = torch.ones(1, 40, dtype=torch.bool)
    em[0, 10:18] = False
    got, _ = E.sample(cond, text, 41, W, ocfg, edit_mask=em, **KW)
    assert torch.equal(got[0, :40][em[0]], cond[0][em[0]]) and torch.isfinite(got).all()
    assert ((got[0, 10:18] - cond[0, 10:18]).abs().amax(-1) > 1e-3).all()


def test_restatement_all_true_mask_is_the_v0_and_e2_restatements(tiny):
    W, ocfg = tiny
    cond, text = _case(1, 30, 20, seed=6)
    ones = torch.ones(1, 30, dtype=torch.bool)
    ocfg0 = V.ocfg_v0(ocfg)
    want, _ = V.sample(cond, text, 45, W, ocfg0, pe_attn_head=1, **KW)
    got, _ = E.sample(cond, text, 45, W, ocfg0, edit_mask=ones, forward=functools.partial(V.dit_forward, pe_attn_head=1),
                      **KW)
    assert torch.equal(got, want)
    from f5_tts_mlx_b200.unett import UNetTConfig, random_unett_weights
    ucfg = UNetTConfig(dim=128, depth=2, heads=2, ff_mult=2, text_num_embeds=60)
    Wu = random_unett_weights(ucfg, seed=7)
    want, _ = U.sample(cond, text, 45, Wu, ucfg, **KW)
    got, _ = E.sample(cond, text, 45, Wu, ucfg, edit_mask=ones, forward=U.unett_forward, **KW)
    assert torch.equal(got, want)


# ---------------------------------------------------------------- sample() refusals
class _StubBackbone:
    dim, device = 128, "cpu"


@pytest.mark.parametrize("mask,match", [(torch.ones(1, 40), "bool"), (np.ones((1, 40), dtype=bool), "bool"),
                                        (torch.ones(2, 40, dtype=torch.bool), "shape"),
                                        (torch.ones(1, 39, dtype=torch.bool), "shape"),
                                        (torch.ones(40, dtype=torch.bool), "shape")])
def test_sample_refuses_bad_edit_masks(mask, match):
    from f5_tts_mlx_b200 import F5TTS
    f5 = F5TTS(_StubBackbone())
    with pytest.raises(ValueError, match=match):
        f5.sample(torch.zeros(1, 40, 100), torch.zeros(1, 5, dtype=torch.int32), 60, edit_mask=mask)


def test_speech_edit_refuses_a_model_without_vocoder():
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.edit import speech_edit
    with pytest.raises(ValueError, match="vocoder"):
        speech_edit(F5TTS(_StubBackbone()), torch.zeros(24000), 24000, "hi", [(0.1, 0.2)])


# ---------------------------------------------------------------- CLI
def test_cli_parses_edits_and_fix_durations(monkeypatch, tmp_path):
    import f5_tts_mlx_b200.edit as ED
    from f5_tts_mlx_b200.generate import read_wav, write_wav
    src = tmp_path / "in.wav"
    write_wav(str(src), 0.1 * torch.ones(4410), 44100)
    seen = {}
    monkeypatch.setattr(ED.F5TTS, "from_pretrained", lambda name, **kw: seen.update(name=name, load=kw) or "MODEL")

    def fake_edit(model, audio, sr, text, parts, fix, **kw):
        seen.update(model=model, n=audio.shape[0], sr=sr, text=text, parts=parts, fix=fix, kw=kw)
        return torch.zeros(1234)

    monkeypatch.setattr(ED, "speech_edit", fake_edit)
    out = tmp_path / "out.wav"
    ED.main(["--audio", str(src), "--text", "new words here", "--edit", "1.42:2.44", "--edit", "4.04:4.90",
             "--fix-duration", "1.2", "--fix-duration", "1.0", "--output", str(out), "--model", "random",
             "--model-version", "e2", "--steps", "7", "--method", "midpoint", "--cfg", "1.5", "--sway-coef", "0",
             "--seed", "9"])
    assert seen["parts"] == [(1.42, 2.44), (4.04, 4.90)] and seen["fix"] == [1.2, 1.0]
    assert (seen["model"], seen["n"], seen["sr"], seen["text"]) == ("MODEL", 4410, 44100, "new words here")
    assert seen["kw"] == dict(steps=7, method="midpoint", cfg_strength=1.5, sway_sampling_coef=0.0, seed=9)
    assert seen["name"] == "random" and seen["load"] == dict(quantization_bits=None, fp8=None, fp8_attention=False,
                                                             model_version="e2", vocoder="vocos")
    back, sr = read_wav(str(out))
    assert sr == 24000 and back.shape[0] == 1234

    ED.main(["--audio", str(src), "--text", "x", "--edit", "0:0.05", "--output", str(out), "--fp8", "block",
             "--fp8-attention", "--vocoder", "bigvgan", "--q", "8"])
    assert seen["fix"] is None and seen["kw"]["steps"] == 32 and seen["kw"]["method"] == "euler"
    assert seen["load"] == dict(quantization_bits=8, fp8="block", fp8_attention=True, model_version="v1",
                                vocoder="bigvgan")
    for bad in (["--edit", "1.42-2.44"], ["--edit", "1:2", "--fix-duration", "1", "--fix-duration", "2"],
                ["--edit", "1:2", "--fp8-attention"], []):
        with pytest.raises(SystemExit):
            ED.main(["--audio", str(src), "--text", "x", "--output", str(out)] + bad)


# ---------------------------------------------------------------- sharding
class _StubF5:
    """Records what sample() receives; returns each utterance's edit mask as its 'mel'."""

    class transformer:
        device = "cpu"

    def sample(self, cond, text, duration, *, y0=None, edit_mask=None, pad_frames=None, return_trajectory=True, **kw):
        assert edit_mask.shape == cond.shape[:2] and y0.shape[0] == cond.shape[0]
        return torch.cat([edit_mask[..., None].float(), y0[:, : cond.shape[1], :1]], -1), None


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _shard_worker(rank: int, world: int, port: int, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from f5_tts_mlx_b200.parallel import sample_sharded
        g = torch.Generator().manual_seed(0)
        cond = torch.randn(5, 30, 100, generator=g)
        mask = torch.rand(5, 30, generator=g) < 0.5
        y0 = torch.arange(5 * 40, dtype=torch.float32).reshape(5, 40, 1).repeat(1, 1, 100)
        out = sample_sharded(_StubF5(), cond, torch.zeros(5, 4, dtype=torch.int32), torch.full((5,), 40), y0=y0,
                             edit_mask=mask, steps=2)
        # numpy, not tensors: a tensor crosses the queue as shared memory that dies with this process
        q.put((rank, None if out is None else torch.stack(out).numpy(), mask.numpy(), y0[:, :30, :1].numpy()))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_sample_sharded_slices_the_edit_mask_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=240) for _ in procs), key=lambda r: r[0])
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    (_, out0, mask, y0), (_, out1, _, _) = res
    assert out1 is None and out0.shape == (5, 30, 2)
    assert np.array_equal(out0[..., 0].astype(bool), mask)     # every utterance got its own row of the global mask
    assert np.array_equal(out0[..., 1:], y0)                   # in the same order as its noise
