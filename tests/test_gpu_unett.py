"""-m gpu: E2TTS_Base (the UNetT backbone) on the H100.

  * the GEMM epilogue's RMSNorm consumer mode (f5_gemm_args.ln_rms) against float64, all-zero rows included;
  * the time-token pack kernel, bitwise against torch;
  * UNetT.__call__ and sample() against the test-side restatement (tests/unett_emul.py), frame by frame
    (composed_check.assert_rows: every frame within 3x the worst frame of its bf16 emulation, every utterance within the
    per-utterance rel rule), on a small config and at E2TTS_Base size, at lengths whose N + 1 rows (the time row
    first) end just before, on and after a 128-row tile edge; frame bucketing; a ragged batch; generate().
"""
import ctypes as C

import pytest
import torch

from composed_check import assert_rows
from helpers import rel, synth_audio
from oracle import f5_oracle as O
import unett_emul as U

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ---------------------------------------------------------------- kernels
@pytest.mark.parametrize("act,out_bf16", [(0, True), (1, True), (0, False)])   # QKV-, FF1- and proj_out-like
@pytest.mark.parametrize("M,K,N", [(300, 1024, 1024), (129, 256, 512), (77, 1024, 100)])
def test_rms_consumer_epilogue_vs_float64(act, out_bf16, M, K, N):
    from f5_tts_mlx_b200 import ops
    if out_bf16 and N % 8:
        pytest.skip("a bf16 output needs n % 8 == 0 (the 100-column proj_out writes fp32)")
    g = torch.Generator(device=DEV).manual_seed(M + K + N)
    x = torch.randn(M, K, generator=g, device=DEV)
    x[1::3] += 40.0 * torch.randn(1, K, generator=g, device=DEV)     # rows with a large mean
    x[5] = 0.0                                                         # an all-zero row
    x[7] *= 1e-20                                                      # a tiny one
    gain = 1 + 0.1 * torch.randn(K, generator=g, device=DEV)
    w = torch.randn(N, K, generator=g, device=DEV) / K ** 0.5
    bias = torch.randn(N, generator=g, device=DEV)
    stats = torch.stack([x.view(M, K // 64, 64).sum(-1), x.view(M, K // 64, 64).pow(2).sum(-1)], -1).contiguous()
    xb, wg = x.bfloat16(), (w * gain).bfloat16()
    out = torch.full((M, N), float("nan"), device=DEV, dtype=torch.bfloat16 if out_bf16 else torch.float32)
    ops.gemm(xb, wg, out, bias=bias, act=act, ln_rms=True, ln_in_stats=stats)
    # float64 of the same operands: bf16(x) @ bf16(W g)^T * sqrt(K) / max(||x||, 1e-12) + b
    scale = K ** 0.5 / x.double().norm(dim=-1, keepdim=True).clamp_min(1e-12)
    ref = (xb.double() @ wg.double().t()) * scale + bias.double()
    if act == 1:
        ref = torch.nn.functional.gelu(ref, approximate="tanh")
    got = out.double()
    assert torch.isfinite(got).all()
    tol = 8e-3 if out_bf16 else 1e-3      # fp32: the accumulation order of the large-mean rows' big products
    err = (got - ref).abs() / (ref.abs() + 1e-2)
    assert err.max() < tol, err.max()
    zero_row = bias.double() if act == 0 else torch.nn.functional.gelu(bias.double(), approximate="tanh")
    assert torch.allclose(got[5], zero_row, rtol=tol, atol=1e-6)
    if act == 0 and not out_bf16:
        out0 = torch.empty(M, N, device=DEV)
        ops.gemm(xb, wg, out0, ln_rms=True, ln_in_stats=stats)
        assert torch.equal(out0[5], torch.zeros(N, device=DEV))        # zero row, no bias -> 0, not NaN


def test_rms_consumer_refusals():
    from f5_tts_mlx_b200 import _lib
    a = torch.zeros(128, 256, dtype=torch.bfloat16, device=DEV)
    w = torch.zeros(256, 256, dtype=torch.bfloat16, device=DEV)
    out = torch.zeros(128, 256, device=DEV)
    st = torch.zeros(128, 4, 2, device=DEV)
    g = _lib.GemmArgs()
    g.a, g.lda, g.w, g.ldw, g.m, g.n, g.k = a.data_ptr(), 256, w.data_ptr(), 256, 128, 256, 256
    g.num_batches, g.conv_taps, g.q_scale, g.out, g.ldo = 1, 1, 1.0, out.data_ptr(), 256
    g.ln_rms = 1
    assert _lib.load().f5_gemm_bf16(C.byref(g), None) == -1            # no statistics
    g.ln_in_stats, g.ln_tab, g.ln_tab_ld = st.data_ptr(), st.data_ptr(), 256
    assert _lib.load().f5_gemm_bf16(C.byref(g), None) == -1            # an AdaLN table as well


@pytest.mark.parametrize("BU,N,D", [(1, 937, 1024), (4, 130, 256), (2, 1, 512)])
def test_time_pack_bitwise(BU, N, D):
    from f5_tts_mlx_b200 import _lib
    g = torch.Generator(device=DEV).manual_seed(N)
    xe = torch.randn(BU, N, D, generator=g, device=DEV) * 3
    t = torch.randn(D, generator=g, device=DEV)
    x = torch.full((BU, N + 1, D), float("nan"), device=DEV)
    xb = torch.full((BU * (N + 1), 2 * D), float("nan"), dtype=torch.bfloat16, device=DEV)
    st = torch.full((BU * (N + 1), D // 64, 2), float("nan"), device=DEV)
    _lib.check(_lib.load().f5_unett_time_pack(xe.data_ptr(), t.data_ptr(), x.data_ptr(), xb[:, D:].data_ptr(), 2 * D,
                                              st.data_ptr(), BU, N, D, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    want = torch.cat([t.expand(BU, 1, D), xe], 1)
    assert torch.equal(x, want)
    assert torch.equal(xb[:, D:], want.reshape(-1, D).bfloat16())
    assert torch.isnan(xb[:, :D].float()).all()                        # the left half is not touched
    u = want.reshape(-1, D // 64, 64).double()
    assert torch.allclose(st.double(), torch.stack([u.sum(-1), u.pow(2).sum(-1)], -1), rtol=1e-5, atol=1e-4)


# ---------------------------------------------------------------- the backbone
def _net(cfg, W):
    from f5_tts_mlx_b200.unett import UNetT
    return UNetT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, text_num_embeds=cfg.text_num_embeds,
                 text_dim=cfg.text_dim, pe_attn_head=cfg.pe_attn_head, device=DEV).load_weights(W)


@pytest.fixture(scope="module")
def small():
    from f5_tts_mlx_b200.unett import UNetTConfig, random_unett_weights
    cfg = UNetTConfig(dim=256, depth=4, heads=4, ff_mult=4)
    W = random_unett_weights(cfg, seed=11)
    return cfg, W, _net(cfg, W)


@pytest.fixture(scope="module")
def base():
    from f5_tts_mlx_b200.unett import E2_BASE_CONFIG, random_unett_weights
    W = random_unett_weights(E2_BASE_CONFIG, seed=1234)
    return E2_BASE_CONFIG, W, _net(E2_BASE_CONFIG, W)


def _inputs(B, N, nt, seed, pad_from=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, 100, generator=g); cond = torch.randn(B, N, 100, generator=g) * 2 - 1
    text = torch.randint(0, 2545, (B, nt), generator=g, dtype=torch.int32)
    if pad_from is not None:
        text[:, pad_from:] = -1
    return x, cond, text


@pytest.mark.parametrize("which", ["small", "base"])
@pytest.mark.parametrize("drops", [(False, False), (True, False), (False, True), (True, True)])
def test_forward_vs_restatement(which, drops, request):
    cfg, W, net = request.getfixturevalue(which)
    x, cond, text = _inputs(1, 200, 48, seed=7, pad_from=37)
    t = torch.tensor(0.37)
    ref = U.unett_forward(x, cond, text, t, *drops, None, W, cfg)
    ref16 = U.unett_forward(x, cond, text, t, *drops, None, W, cfg, O.Precision(True))
    got = net(x.to(DEV), cond.to(DEV), text.to(DEV), t, *drops).cpu()
    rep = assert_rows(got[None], ref[None], ref16[None], what=f"{which} drops={drops}")
    print(f"{which} drops={drops}: {rep}")


def _forward_ragged(which, N, lens, request):
    """B = 2 with a row mask (seq_len), frame by frame over each utterance's valid frames."""
    cfg, W, net = request.getfixturevalue(which)
    x, cond, text = _inputs(2, N, 40, seed=9 + N, pad_from=31)
    mask = torch.arange(N)[None] < torch.tensor(lens)[:, None]
    t = torch.tensor(0.61)
    ref = U.unett_forward(x, cond, text, t, False, False, mask, W, cfg)
    ref16 = U.unett_forward(x, cond, text, t, False, False, mask, W, cfg, O.Precision(True))
    got = net(x.to(DEV), cond.to(DEV), text.to(DEV), t, mask=mask.to(DEV)).cpu()
    rep = assert_rows(got[None], ref[None], ref16[None], lens=lens, what=f"{which} ragged N={N} lens={lens}")
    print(f"{which} ragged N={N}: {rep}")


@pytest.mark.parametrize("which", ["small", "base"])
def test_forward_ragged_batch_vs_restatement(which, request):
    _forward_ragged(which, 150, (150, 97), request)


@pytest.mark.parametrize("which", ["small", "base"])
@pytest.mark.parametrize("N,lens", [(127, (127, 64)), (128, (128, 127)), (200, (200, 127))])
def test_forward_tile_edges_vs_restatement(which, N, lens, request):
    """The UNetT runs N + 1 rows per utterance (the time row first), so N = 127 / 128 / 200 put the last frame on, just
    past and well past a 128-row tile edge, and the second utterance's rows start mid-tile: a frame lost or shifted at
    the time row or at a tile edge is one bad row, which the per-frame check names."""
    _forward_ragged(which, N, lens, request)


@pytest.mark.parametrize("method", ["euler", "midpoint"])
def test_sample_cfg_vs_restatement(method, small):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, net = small
    g = torch.Generator().manual_seed(11)
    cond = torch.randn(1, 60, 100, generator=g) * 2.24 - 1.27
    text = torch.randint(0, 2545, (1, 40), generator=g, dtype=torch.int32); text[0, 33:] = -1
    N = 230
    y0 = torch.randn(1, N, 100, generator=g)
    kw = dict(steps=4, method=method, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
    out, _ = F5TTS(net).sample(cond.to(DEV), text, N, **kw)
    ref, _ = U.sample(cond, text, N, W, cfg, **kw)
    ref16, _ = U.sample(cond, text, N, W, cfg, prec=O.Precision(True), **kw)
    rep = assert_rows(out.cpu()[None], ref[None], ref16[None], what=f"{method} sample")
    print(f"{method} sample: {rep}")


def test_sample_ragged_batch_vs_restatement(small):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, net = small
    g = torch.Generator().manual_seed(31)
    cond = torch.randn(2, 70, 100, generator=g) * 2.24 - 1.27
    text = torch.randint(0, 2545, (2, 45), generator=g, dtype=torch.int32); text[1, 29:] = -1
    dur = torch.tensor([260, 201])
    kw = dict(steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0, seed=3)
    out, _ = F5TTS(net).sample(cond.to(DEV), text, dur, **kw)
    ref, _ = U.sample(cond, text, dur, W, cfg, **kw)
    ref16, _ = U.sample(cond, text, dur, W, cfg, prec=O.Precision(True), **kw)
    rep = assert_rows(out.cpu()[None], ref[None], ref16[None], lens=dur.tolist(), what="ragged sample")
    print(f"ragged sample: {rep}")


def test_frame_bucketing_equals_exact_shapes(small):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, net = small
    g = torch.Generator().manual_seed(21)
    cond = (torch.randn(1, 60, 100, generator=g) * 2.24 - 1.27).to(DEV)
    kw = dict(steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0)
    exact, bucketed = F5TTS(net), F5TTS(net)
    bucketed.frame_bucket = 128
    plans = set()
    for N, nt in ((150, 20), (201, 31), (255, 27)):
        text = torch.randint(0, 2545, (1, nt), generator=g, dtype=torch.int32)
        y0 = torch.randn(1, N, 100, generator=g)
        a, _ = exact.sample(cond, text, N, y0=y0, **kw)
        b, _ = bucketed.sample(cond, text, N, y0=y0, **kw)
        plans.add(id(bucketed.last_plan))
        assert b.shape == a.shape == (1, N, 100)
        assert rel(b, a) < 1e-3, (N, rel(b, a))
    assert len(plans) == 1 and bucketed.last_plan.session.frames == 256


def test_generate_e2_writes_wav(tmp_path):
    """generate(model_version="e2") with the random E2TTS_Base model: a given duration, and estimated durations in the
    serial loop and with batch_sentences=True; the wav holds the expected number of samples."""
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200 import generate as G
    ref = 0.05 * synth_audio(2 * 24000, seed=1)
    G.write_wav(str(tmp_path / "ref.wav"), ref)
    n_ref = ref.shape[0]
    f5 = F5TTS.from_pretrained("random", model_version="e2")
    out_len = f5._vocoder.__self__.out_len
    text, ref_text = "Hello there. This is a test!", "some reference text."
    kw = dict(ref_audio_path=str(tmp_path / "ref.wav"), ref_audio_text=ref_text, steps=3, method="euler", seed=7,
              f5tts=f5)
    w = G.generate(text, duration=4.0, output_path=str(tmp_path / "d.wav"), **kw)
    assert w.shape[0] == out_len(int(4.0 * G.FRAMES_PER_SEC)) - n_ref and torch.isfinite(w).all()
    expect = sum(out_len(max(int(G.estimated_duration(ref, ref_text, s) * G.FRAMES_PER_SEC), n_ref // 256 + 1)) - n_ref
                 for s in G.split_sentences(text))
    for batched in (False, True):
        out = tmp_path / f"out{int(batched)}.wav"
        w = G.generate(text, estimate_duration=True, output_path=str(out), batch_sentences=batched, **kw)
        assert torch.isfinite(w).all() and float(w.abs().max()) > 0
        assert abs(w.shape[0] - expect) <= 3 * 256, (w.shape, expect)
        back, sr = G.read_wav(str(out))
        assert sr == 24000 and back.shape[0] == w.shape[0]
