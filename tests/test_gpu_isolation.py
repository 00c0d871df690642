"""-m gpu: one utterance's result depends only on its own valid data.  Neither the keys the attention masks nor the other
utterances of the batch may change a single bit of it.

  a. masked keys, at kernel level: the four attention entry points with the rows at or beyond kv_len replaced;
  b. bucket rows, at session level: a frame-bucketed session with the rows beyond frames_valid replaced;
  c. batch neighbours, at session level: utterance 1 replaced, utterances 0 and 2 compared;
  d. batch neighbours through sample() on one plan and its captured graph;
  b-d again for the UNetT (E2TTS), whose rows are masked through seq_len1 / valid_len1 from the time row on;
  e. batch neighbours in the duration model, Vocos and BigVGAN.

Every comparison is bitwise.  Both runs of a comparison use the same plan, so shapes, tile choices and launches are
identical; no kernel reduces across utterances, and the one atomic (the FP8 quantise pass's atomicMax of a tile's
amax) is order-independent.  Padding frames of an utterance (at or beyond its seq_len) belong to it: they reach its
valid frames through the convolutions and GRN, as in the reference, so (c) and (d) keep them fixed."""
import pytest
import torch
import torch.nn.functional as F

from kernel_check import Guarded, assert_exact
from test_gpu_composed import _M, eval_times, inputs, model
from test_gpu_fp8_attention import expected_codes, run_attention
from test_gpu_kernel_exact import _attn_call, _qkv_buffer

pytestmark = pytest.mark.gpu
DEV = "cuda"

# the DiT modes: keyword arguments of test_gpu_composed.model
MODES = {"bf16-fused": {}, "bf16-unfused": dict(fused=False), "fp8-tensor": dict(fp8="tensor"),
         "fp8-block": dict(fp8="block"), "fp8-block-attn": dict(fp8="block", fp8_attention=True)}
STAGES = ("text_x", "hoist", "h", "x", "v")


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    _M.clear()
    torch.cuda.empty_cache()


def assert_rows_exact(got, want, frames, utts, what):
    """got, want [branches, B, frames, C]: bitwise on rows [0, frames[b]) of every utterance b in utts, naming the first
    differing (CFG branch, when there are two; utterance, frame, column)."""
    for br in range(got.shape[0]):
        tag = f"branch {br} " if got.shape[0] > 1 else ""
        for b in utts:
            n = int(frames[b])
            assert_exact(got[br, b, :n].contiguous(), want[br, b, :n].contiguous(),
                         lambda r, c, b=b, tag=tag: f"{tag}utterance {b} frame {r} column {c}", what)


def signs(shape, g):
    return (torch.randint(0, 2, shape, generator=g) * 2 - 1).float()


# ---------------------------------------------------------------- a. masked keys, kernel level
ENTRIES = ["bf16", "e4m3", "e4m3_scaled", "fp8"]
SHAPES = {300: (4, 4, [300, 263, 256, 1]), 937: (4, 4, [937, 900, 256, 1]), 5625: (2, 16, [5625, 4588])}


def run_entry(entry, qkv, B, N, H, kv):
    """One attention entry on bf16 qkv [B N, 3 H 64]: (output [B, N, H 64] as bf16 or e4m3 codes, scale_out [B, N, H]
    or None)."""
    D = H * 64
    if entry == "fp8":
        _, out, so = run_attention(qkv, B, N, H, kv)
        out.check(f"{entry} out guard"); so.check(f"{entry} scale guard")
        return out.view.cpu().reshape(B, N, D), so.view.cpu().T.reshape(B, N, H)
    buf = _qkv_buffer(B, N, H)
    buf.copy_(qkv)
    out = Guarded(B * N, D, torch.bfloat16 if entry == "bf16" else torch.uint8, DEV)
    so = Guarded(H, B * N, torch.float32, DEV, lr=False) if entry == "e4m3_scaled" else None
    _attn_call(buf, out.view, B, N, H, kv, fp8=entry != "bf16", scale_out=so.view if so is not None else None)
    out.check(f"{entry} out guard")
    if so is None:
        return out.view.cpu().reshape(B, N, D), None
    so.check(f"{entry} scale guard")
    return out.view.cpu().reshape(B, N, D), so.view.cpu().T.reshape(B, N, H)


@pytest.mark.parametrize("poison", ["3e4", "2^100", "neighbour"])
@pytest.mark.parametrize("N", sorted(SHAPES))
@pytest.mark.parametrize("entry", ENTRIES)
def test_attention_masked_keys_cannot_reach_valid_rows(entry, N, poison):
    """f5_attention_fwd, _e4m3, _e4m3_scaled and the quantise pass + f5_attention_fwd_fp8: the output rows below
    kv_len (bf16 bits, or e4m3 codes and their scales) are the same whether the rows at or beyond kv_len (q, k and v)
    hold random values, +-3e4, +-2^100 (in k and v; S stays finite in fp32) or another utterance's rows.  The FP8
    entry's quantise pass must keep those keys out of its tiles' k and v scales."""
    B, H, lens = SHAPES[N]
    D = H * 64
    kv = torch.tensor(lens, dtype=torch.int32)
    g = torch.Generator().manual_seed(N)
    x = torch.randn(B, N, 3 * D, generator=g)
    x[..., :D] *= 0.5
    masked = torch.arange(N)[None] >= kv[:, None]                       # [B, N]
    y = x.clone()
    if poison == "3e4":
        y[masked] = 3e4 * signs((int(masked.sum()), 3 * D), g)
    elif poison == "2^100":
        y[masked] = 2.0 ** 100 * signs((int(masked.sum()), 3 * D), g)
        y[..., :D][masked] = signs((int(masked.sum()), D), g)           # q of masked rows +-1: no overflow in S
    else:
        for b in range(B):
            y[b, masked[b]] = x[(b + 1) % B, masked[b]]
    assert torch.isfinite(y.bfloat16().float()).all()
    base = run_entry(entry, x.reshape(B * N, 3 * D).bfloat16().to(DEV), B, N, H, kv.to(DEV))
    got = run_entry(entry, y.reshape(B * N, 3 * D).bfloat16().to(DEV), B, N, H, kv.to(DEV))
    what = f"{entry} N={N} masked keys {poison}"
    assert_rows_exact(got[0][None], base[0][None], kv, range(B), what + ": output")
    if base[1] is not None:
        assert_rows_exact(got[1][None], base[1][None], kv, range(B), what + ": scale_out")


# ---------------------------------------------------------------- DiT sessions
def drive(m, x, cond, text, tvals, ti, seq_len, n_valid):
    """A CFG session of `m` (a DiT or a UNetT) with x and cond [B, frames, 100] as given on every row (frames > n_valid:
    a bucketed session with frames_valid = n_valid): inputs, precompute, one forward.  Returns the stages
    [2, B, rows, C]: rows = frames, or frames + 1 for the UNetT's x and v (each utterance's time row first)."""
    B, NB = x.shape[:2]
    bucketed = NB != n_valid
    s = m.session(B, NB, tvals.numel(), True, text.shape[1], seq_len is not None, bucketed=bucketed)
    s.set_inputs(text, cond.to(DEV), tvals.to(DEV), seq_len.to(DEV) if seq_len is not None else None,
                 frames_valid=n_valid if bucketed else None)
    s.c.drop_flags = 0
    s.y_bf16.zero_()
    xb = x.reshape(B * NB, -1).to(DEV)
    for half in range(2):
        s.y_bf16[half * B * NB:(half + 1) * B * NB, :x.shape[-1]].copy_(xb)
    m.precompute(s)
    m.forward_session(s, ti)
    torch.cuda.synchronize()
    return s, {k: (lambda t: t.view(2, B, t.shape[0] // (2 * B), -1))(getattr(s, k)).cpu() for k in STAGES}


def bucket_text(text):
    """sample()'s text bucketing: columns padded with -1 to a multiple of 32."""
    return F.pad(text, (0, -(-text.shape[1] // 32) * 32 - text.shape[1]), value=-1)


def fill(kind, shape, g):
    if kind == "zeros":
        return torch.zeros(shape)
    if kind == "1e4":
        return 1e4 * signs(shape, g)
    vals = torch.tensor([float("inf"), float("-inf"), float("nan")])
    return vals[torch.randint(0, 3, shape, generator=g)]


@pytest.mark.parametrize("mode", list(MODES))
def test_bucket_rows_cannot_reach_valid_rows(mode):
    """A bucketed session (256 frames, frames_valid 150, B = 2 with ragged seq_len, CFG): the bucket rows of y_bf16 and
    of the padded cond hold zeros, +-1e4, then inf and NaN; text_x, hoist, h, x and v on every row below 150 of both
    branches keep their bits.  The row masks assign +0 to the bucket rows, so nothing there is read."""
    B, N, NB = 2, 150, 256
    x, cond, text = inputs(B, N, 50, seed=21)
    text = bucket_text(text)
    seq_len = torch.tensor([150, 123], dtype=torch.int32)
    tvals = eval_times("rk4")
    m = model("gate", **MODES[mode])
    g = torch.Generator().manual_seed(22)
    runs = {}
    for kind in ("zeros", "1e4", "nonfinite"):
        xf = torch.cat([x, fill(kind, (B, NB - N, 100), g)], 1)
        cf = torch.cat([cond, fill(kind, (B, NB - N, 100), g)], 1)
        runs[kind] = drive(m, xf, cf, text, tvals, 2, seq_len, N)[1]
    for kind in ("1e4", "nonfinite"):
        for k in STAGES:
            assert_rows_exact(runs[kind][k], runs["zeros"][k], [N] * B, range(B), f"{mode} bucket rows {kind}: {k}")


NEIGHBOURS = ("text", "x64", "nonfinite")


def neighbour(kind, x, cond, text, seq_len, g):
    """Utterance 1 of (x, cond, text, seq_len) replaced: another text and a shorter seq_len; cond and x times 64 (the
    residual stream far beyond e4m3's 448); or x with inf and NaN in some frames."""
    x, cond, text, seq_len = x.clone(), cond.clone(), text.clone(), seq_len.clone()
    if kind == "text":
        nt = int((text[1] != -1).sum())
        text[1] = -1
        text[1, :nt - 9] = torch.randint(0, 2545, (nt - 9,), generator=g, dtype=torch.int32)
        seq_len[1] = 88
    elif kind == "x64":
        x[1] *= 64
        cond[1] *= 64
    else:
        x[1, 10:20] = float("inf")
        x[1, 40:43, ::3] = float("nan")
        x[1, 70:71] = float("-inf")
    return x, cond, text, seq_len


@pytest.mark.parametrize("bucket", [False, True], ids=["exact", "bucket256"])
@pytest.mark.parametrize("mode", list(MODES))
def test_batch_neighbour_cannot_reach_other_utterances(mode, bucket):
    """B = 3, N = 150 (exact, or a 256-frame bucket), CFG, ragged seq_len: with utterance 1 replaced (NEIGHBOURS),
    every frame of utterances 0 and 2 (their padding and bucket rows included) keeps its bits in text_x, hoist, h, x
    and v, in both branches."""
    B, N = 3, 150
    NB = 256 if bucket else N
    x, cond, text = inputs(B, N, 50, seed=31)
    if bucket:
        text = bucket_text(text)
    seq_len = torch.tensor([150, 131, 97], dtype=torch.int32)
    tvals = eval_times("rk4")
    m = model("gate", **MODES[mode])
    pad = lambda a: F.pad(a, (0, 0, 0, NB - N))
    g = torch.Generator().manual_seed(32)
    base = drive(m, pad(x), pad(cond), text, tvals, 2, seq_len, N)[1]
    for kind in NEIGHBOURS:
        x2, c2, t2, s2 = neighbour(kind, x, cond, text, seq_len, g)
        got = drive(m, pad(x2), pad(c2), t2, tvals, 2, s2, N)[1]
        assert not torch.equal(got["v"][:, 1], base["v"][:, 1]), f"{kind}: utterance 1 did not change"
        for k in STAGES:
            assert_rows_exact(got[k], base[k], [NB] * B, (0, 2), f"{mode} {'bucket' if bucket else 'exact'} "
                                                                  f"neighbour {kind}: {k}")


@pytest.mark.parametrize("bucket", [False, True], ids=["ragged", "bucket256"])
def test_dit_quantise_pass_takes_the_attention_kv_len(bucket):
    """The FP8 attention mode's quantise pass, as f5_dit_forward runs it: the last block's e4m3 Q | K codes and
    q / k / v scales equal the host rule on that block's bf16 qkv with the attention's kv_len, seq_len (ragged batch) or
    frames_valid (a bucket without seq_len), so the masked keys stay out of the tile scales."""
    B, N = (3, 150) if not bucket else (1, 150)
    NB = 256 if bucket else N
    x, cond, text = inputs(B, N, 50, seed=41)
    seq_len = None if bucket else torch.tensor([150, 131, 97], dtype=torch.int32)
    if bucket:
        text = bucket_text(text)
    m = model("gate", fp8="block", fp8_attention=True)
    pad = lambda a: F.pad(a, (0, 0, 0, NB - N))
    s, _ = drive(m, pad(x), pad(cond), text, eval_times("euler"), 1, seq_len, N)
    H, D, BU = m.config.heads, m.config.dim, 2 * B
    kv = (seq_len if seq_len is not None else torch.full((B,), N, dtype=torch.int32)).repeat(2)
    codes, scales = expected_codes(s.qkv_bf16.cpu(), BU, NB, H, kv)
    loc = lambda r, c: f"utterance {r // NB} frame {r % NB} column {c}"
    assert_exact(s.qk_fp8.cpu(), codes[:, :2 * D].contiguous(), loc, "session q|k codes")
    assert_exact(s.qkv_scale.cpu(), scales, lambda r, c: f"unit {r} utterance {c // NB} frame {c % NB}", "session scales")


# ---------------------------------------------------------------- d. sample() and its captured graph
def sample_call(B, N, seed, dur):
    g = torch.Generator().manual_seed(seed)
    cond = (torch.randn(B, N // 3, 100, generator=g) * 2.24 - 1.27).clamp(-11.51, 5)
    text = torch.randint(0, 2545, (B, 30), generator=g, dtype=torch.int32)
    y0 = torch.randn(B, N, 100, generator=g)
    for b in range(B):
        y0[b, int(dur[b]):] = 0
        text[b, 30 - 4 * b - seed % 3:] = -1
    return cond, text, y0


@pytest.mark.parametrize("bucket", [0, 128], ids=["exact", "bucket128"])
@pytest.mark.parametrize("method", ["euler", "rk4"])
@pytest.mark.parametrize("mode", list(MODES))
def test_sample_neighbours_cannot_reach_utterance_0(mode, method, bucket):
    """Two sample() calls (B = 3, CFG, 4 steps) on one plan, the second replaying the first's captured graph: the
    neighbours' text, duration, cond and y0 change, utterance 0 (the longest, so N, the text columns and the plan key
    stay) keeps the bits of its out and of its whole trajectory."""
    from f5_tts_mlx_b200 import F5TTS
    B, N = 3, 150
    f5 = F5TTS(model("gate", **MODES[mode]))
    kw = dict(steps=4, method=method, cfg_strength=2.0, sway_sampling_coef=-1.0, frame_bucket=bucket)
    dur1, dur2 = torch.tensor([N, 131, 97]), torch.tensor([N, 101, 140])
    cond1, text1, y01 = sample_call(B, N, 51, dur1)
    cond2, text2, y02 = sample_call(B, N, 52, dur2)
    cond2[0], text2[0], y02[0] = cond1[0], text1[0], y01[0]
    out1, traj1 = f5.sample(cond1.to(DEV), text1, dur1, y0=y01, **kw)
    plan, graph = f5.last_plan, f5.last_plan.graph
    assert graph is not None
    out2, traj2 = f5.sample(cond2.to(DEV), text2, dur2, y0=y02, **kw)
    assert f5.last_plan is plan and plan.graph is graph, "the second call did not replay the first call's graph"
    assert not torch.equal(out2[1], out1[1])
    what = f"sample {mode} {method} {'bucket' if bucket else 'exact'}"
    loc = lambda r, c: f"utterance 0 frame {r} column {c}"
    assert_exact(out2[0].cpu(), out1[0].cpu(), loc, what + ": out")
    for i in range(traj1.shape[0]):
        assert_exact(traj2[i, 0].cpu(), traj1[i, 0].cpu(), loc, what + f": trajectory[{i}]")


# ---------------------------------------------------------------- e. duration model and Vocos
def test_duration_neighbours_cannot_reach_utterance_0():
    """B = 3, same text columns: another text and mel for utterances 1 and 2 leave utterance 0's seconds bitwise."""
    from f5_tts_mlx_b200.duration import DurationPredictor, DurationTransformer
    from f5_tts_mlx_b200.weights import random_duration_weights
    pred = DurationPredictor(DurationTransformer(dim=512, depth=8, heads=8, text_dim=512, ff_mult=2, conv_layers=2,
                                                 text_num_embeds=2545), device=DEV).load_weights(random_duration_weights(seed=5))
    g = torch.Generator().manual_seed(61)
    B, N = 3, 130
    mel = torch.randn(B, N, 100, generator=g) * 2.24 - 1.27
    text = torch.randint(0, 2545, (B, 48), generator=g, dtype=torch.int32)
    text[1, 30:] = -1; text[2, 11:] = -1
    a = pred(mel.to(DEV), text).cpu()
    mel2, text2 = mel.clone(), text.clone()
    mel2[1:] = torch.randn(B - 1, N, 100, generator=g) * 8
    text2[1:] = torch.randint(0, 2545, (B - 1, 48), generator=g, dtype=torch.int32)
    text2[1, 20:] = -1
    b = pred(mel2.to(DEV), text2).cpu()
    assert not torch.equal(a[1:], b[1:])
    assert_exact(b[:1].reshape(1, 1), a[:1].reshape(1, 1), lambda r, c: "utterance 0", "duration seconds")


def test_vocos_neighbour_cannot_reach_utterance_0():
    """B = 2: the neighbour's mel times 64 leaves utterance 0's wave bitwise."""
    from f5_tts_mlx_b200.vocos import Vocos
    from f5_tts_mlx_b200.weights import VocosConfig, random_vocos_weights
    voc = Vocos(VocosConfig(), DEV).load_weights(random_vocos_weights(seed=4321))
    g = torch.Generator().manual_seed(62)
    mel = (torch.randn(2, 150, 100, generator=g) * 2.24 - 1.27).clamp(-11.5, 5)
    a = voc.decode(mel.to(DEV)).cpu()
    mel2 = mel.clone()
    mel2[1] *= 64
    b = voc.decode(mel2.to(DEV)).cpu()
    assert not torch.equal(a[1], b[1])
    assert_exact(b[:1], a[:1], lambda r, c: f"utterance 0 sample {c}", "vocos wave")


@pytest.mark.parametrize("which", ["small", "released"])
def test_bigvgan_neighbour_cannot_reach_other_utterances(which):
    """B = 3: utterance 1's mel times 64, then with inf and NaN frames, leaves the waves of utterances 0 and 2 bitwise.
    Every BigVGAN convolution runs batched tiles that never straddle utterances, with zero padding inside each one."""
    from test_gpu_bigvgan import _vocoder
    cfg, _, voc = _vocoder(which)
    g = torch.Generator().manual_seed(63)
    n = 20 if which == "small" else 8
    mel = torch.randn(3, n, cfg.num_mels, generator=g) - 3.0
    base = voc.decode(mel.to(DEV)).cpu()
    for kind in ("x64", "nonfinite"):
        mel2 = mel.clone()
        if kind == "x64":
            mel2[1] *= 64
        else:
            mel2[1, 2:4] = float("inf")
            mel2[1, 5, ::3] = float("nan")
            mel2[1, n - 1] = float("-inf")
        got = voc.decode(mel2.to(DEV)).cpu()
        assert not torch.equal(got[1], base[1]), f"{kind}: utterance 1 did not change"
        for u in (0, 2):
            assert_exact(got[u:u + 1], base[u:u + 1], lambda r, c, u=u: f"utterance {u} sample {c}",
                         f"bigvgan {which} neighbour {kind}")


# ---------------------------------------------------------------- b-d for the UNetT (E2TTS)
UNETT_ROWS1 = ("x", "v")          # the stages with N + 1 rows per utterance (the time row first)


def unett_model():
    """A 4-layer, 256-wide UNetT with random weights (the E2TTS_Base structure: skips, RoPE on one head)."""
    if "unett" not in _M:
        from f5_tts_mlx_b200.unett import UNetT, UNetTConfig, random_unett_weights
        cfg = UNetTConfig(dim=256, depth=4, heads=4, ff_mult=4)
        _M["unett"] = UNetT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult,
                            text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, pe_attn_head=cfg.pe_attn_head,
                            device=DEV).load_weights(random_unett_weights(cfg, seed=71))
    return _M["unett"]


def test_unett_bucket_rows_cannot_reach_valid_rows():
    """The UNetT in a bucketed session (256 frames, frames_valid 150, B = 2 with ragged seq_len, CFG): the bucket rows
    of y_bf16 and of the padded cond hold zeros, +-1e4, then inf and NaN; both branches keep every bit of the first 150
    rows of text_x, hoist and h and the first 151 rows (the time row and the 150 frames) of x and v."""
    B, N, NB = 2, 150, 256
    x, cond, text = inputs(B, N, 50, seed=81)
    text = bucket_text(text)
    seq_len = torch.tensor([150, 123], dtype=torch.int32)
    tvals = eval_times("rk4")
    m = unett_model()
    g = torch.Generator().manual_seed(82)
    runs = {}
    for kind in ("zeros", "1e4", "nonfinite"):
        xf = torch.cat([x, fill(kind, (B, NB - N, 100), g)], 1)
        cf = torch.cat([cond, fill(kind, (B, NB - N, 100), g)], 1)
        runs[kind] = drive(m, xf, cf, text, tvals, 2, seq_len, N)[1]
    for kind in ("1e4", "nonfinite"):
        for k in STAGES:
            n = N + 1 if k in UNETT_ROWS1 else N
            assert_rows_exact(runs[kind][k], runs["zeros"][k], [n] * B, range(B), f"unett bucket rows {kind}: {k}")


@pytest.mark.parametrize("bucket", [False, True], ids=["exact", "bucket256"])
def test_unett_batch_neighbour_cannot_reach_other_utterances(bucket):
    """The UNetT at B = 3, N = 150 (exact, or a 256-frame bucket), CFG, ragged seq_len: with utterance 1 replaced
    (NEIGHBOURS), every row of utterances 0 and 2 (their time row, padding and bucket rows included) keeps its bits in
    text_x, hoist, h, x and v, in both branches."""
    B, N = 3, 150
    NB = 256 if bucket else N
    x, cond, text = inputs(B, N, 50, seed=91)
    if bucket:
        text = bucket_text(text)
    seq_len = torch.tensor([150, 131, 97], dtype=torch.int32)
    tvals = eval_times("rk4")
    m = unett_model()
    pad = lambda a: F.pad(a, (0, 0, 0, NB - N))
    g = torch.Generator().manual_seed(92)
    base = drive(m, pad(x), pad(cond), text, tvals, 2, seq_len, N)[1]
    for kind in NEIGHBOURS:
        x2, c2, t2, s2 = neighbour(kind, x, cond, text, seq_len, g)
        got = drive(m, pad(x2), pad(c2), t2, tvals, 2, s2, N)[1]
        assert not torch.equal(got["v"][:, 1], base["v"][:, 1]), f"{kind}: utterance 1 did not change"
        for k in STAGES:
            n = NB + 1 if k in UNETT_ROWS1 else NB
            assert_rows_exact(got[k], base[k], [n] * B, (0, 2),
                              f"unett {'bucket' if bucket else 'exact'} neighbour {kind}: {k}")


@pytest.mark.parametrize("bucket", [0, 128], ids=["exact", "bucket128"])
@pytest.mark.parametrize("method", ["euler", "rk4"])
def test_unett_sample_neighbours_cannot_reach_utterance_0(method, bucket):
    """Two UNetT sample() calls (B = 3, CFG, 4 steps) on one plan, the second replaying the first's captured graph:
    the neighbours' text, duration, cond and y0 change, utterance 0 keeps the bits of its out and whole trajectory."""
    from f5_tts_mlx_b200 import F5TTS
    B, N = 3, 150
    f5 = F5TTS(unett_model())
    kw = dict(steps=4, method=method, cfg_strength=2.0, sway_sampling_coef=-1.0, frame_bucket=bucket)
    dur1, dur2 = torch.tensor([N, 131, 97]), torch.tensor([N, 101, 140])
    cond1, text1, y01 = sample_call(B, N, 51, dur1)
    cond2, text2, y02 = sample_call(B, N, 52, dur2)
    cond2[0], text2[0], y02[0] = cond1[0], text1[0], y01[0]
    out1, traj1 = f5.sample(cond1.to(DEV), text1, dur1, y0=y01, **kw)
    plan, graph = f5.last_plan, f5.last_plan.graph
    assert graph is not None
    out2, traj2 = f5.sample(cond2.to(DEV), text2, dur2, y0=y02, **kw)
    assert f5.last_plan is plan and plan.graph is graph, "the second call did not replay the first call's graph"
    assert not torch.equal(out2[1], out1[1])
    what = f"unett sample {method} {'bucket' if bucket else 'exact'}"
    loc = lambda r, c: f"utterance 0 frame {r} column {c}"
    assert_exact(out2[0].cpu(), out1[0].cpu(), loc, what + ": out")
    for i in range(traj1.shape[0]):
        assert_exact(traj2[i, 0].cpu(), traj1[i, 0].cpu(), loc, what + f": trajectory[{i}]")
