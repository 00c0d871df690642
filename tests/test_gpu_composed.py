"""-m gpu: the composed DiT, sample(), duration model and Vocos, row by row and stage by stage.

The kernels are tested one at a time elsewhere (test_gpu_kernel_exact.py, test_gpu_hbm_kernels.py).  Here the same
kernels run as the model composes them, and each stage is compared per row (tests/composed_check.py) with the oracle's
stages composed in the test: fp32 for the reference, and the rounding points of the CUDA path for the emulation.
  a. the DiT session buffers after precompute + forward: text_x, hoist, mod_table, h, the residual stream x after
     block L (depth-truncated models receive only blocks < L), v; bucket rows exactly zero;
  b. sample(): out and the last trajectory state per row, for every solver; one Euler step from two DiT calls;
  c. the duration model: seconds per utterance and its residual stream per row;
  d. Vocos: the wave per 256-sample hop segment and the head output per frame;
  e. state reuse: plans, sessions and buffer caches give the bits of a freshly built model (no kernel reduces through
     atomics, so a repeated call reproduces its bits).
Each check prints its worst row ratio (got's worst row error / the emulation's worst row error) on a COMPOSED line."""
import dataclasses

import pytest
import torch
import torch.nn.functional as F

from oracle import f5_oracle as O
from composed_check import assert_rows, exact_zero_rows, row_errors
from helpers import make_dit, ocfg_of

pytestmark = pytest.mark.gpu
dev = "cuda"


def report(what, rep):
    print(f"COMPOSED {what}: {rep}")


# ---------------------------------------------------------------- models
_W = {}


def weights(name):
    from f5_tts_mlx_b200.weights import BASE_CONFIG, GATE_CONFIG, DiTConfig, random_dit_weights
    if name not in _W:
        cfg = {"gate": GATE_CONFIG, "base": BASE_CONFIG,
               "d256": DiTConfig(dim=256, depth=3, heads=4, conv_layers=2)}[name]
        _W[name] = (cfg, random_dit_weights(cfg, seed=1234))
    return _W[name]


_M = {}


def model(name, depth=None, fused=True, fp8=None, fp8_attention=False):
    """DiT `name` truncated to its first `depth` blocks (the packer reads blocks < depth of the full weights)."""
    from f5_tts_mlx_b200 import DiT
    cfg, W = weights(name)
    depth = cfg.depth if depth is None else depth
    key = (name, depth, fused, fp8, fp8_attention)
    if key not in _M:
        c = dataclasses.replace(cfg, depth=depth)
        if fp8:
            kw = dict(fp8_attention=True) if fp8_attention else {}
            _M[key] = DiT(dim=c.dim, depth=c.depth, heads=c.heads, ff_mult=c.ff_mult, mel_dim=c.mel_dim,
                          text_num_embeds=c.text_num_embeds, text_dim=c.text_dim, conv_layers=c.conv_layers,
                          device=dev, fp8=True, fp8_scaling=fp8, **kw).load_weights(W)
        else:
            _M[key] = make_dit(c, W, fused_adaln=fused)
    return _M[key]


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    _M.clear()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- oracle stages, composed
def oracle_mod_table(W, cfg, tvals, prec):
    """Every AdaLN linear (blocks, then norm_out) at every evaluation time: [n_times, depth*6*D + 2*D]."""
    st = F.silu(O.timestep_embedding(tvals.float(), W))
    rows = [O.linear(st, W[f"transformer.transformer_blocks.{i}.attn_norm.linear.weight"],
                     W[f"transformer.transformer_blocks.{i}.attn_norm.linear.bias"], prec) for i in range(cfg.depth)]
    rows.append(O.linear(st, W["transformer.norm_out.linear.weight"], W["transformer.norm_out.linear.bias"], prec))
    return torch.cat(rows, -1)


def oracle_stages(W, cfg, x, cond, text, t, drops, mask, prec, block8=False, attn8=False):
    """One CFG branch of dit_forward, stage by stage: text_x, hoist, h, xs (after each block), v.  block8: the blocks
    of the block-scaled FP8 mode (fp8_block_emul); attn8: those of its FP8 attention mode (fp8_attn_emul)."""
    import fp8_attn_emul as A
    import fp8_block_emul as E
    B, N = x.shape[:2]
    temb = O.timestep_embedding(t.reshape(1).repeat(B).float(), W)
    te = O.text_embedding(text, N, drops[1], W, cfg, prec)
    c = torch.zeros_like(cond) if drops[0] else cond
    pw, pb = W["transformer.input_embed.proj.weight"], W["transformer.input_embed.proj.bias"]
    hoist = O.linear(torch.cat((c, te), -1), pw[:, x.shape[-1]:], pb, prec)
    h = O.linear(torch.cat((x, c, te), -1), pw, pb, prec)
    xx = O.conv_position_embedding(h, W, prec) + h
    rope = O.rotary_freqs(N, cfg.dim_head)
    xs = []
    for i in range(cfg.depth):
        if attn8:
            xx = A.dit_block8a(xx, temb, mask, rope, W, i, cfg)
        elif block8:
            xx = E.dit_block8(xx, temb, mask, rope, W, i, cfg)
        else:
            xx = O.dit_block(xx, temb, mask, rope, W, i, cfg, prec)
        xs.append(xx)
    emb = O.linear(F.silu(temb), W["transformer.norm_out.linear.weight"], W["transformer.norm_out.linear.bias"], prec)
    scale, shift = emb.chunk(2, dim=1)
    v = O.adaln_linear(xx, scale, shift, W["transformer.proj_out.weight"], W["transformer.proj_out.bias"], prec)
    return dict(text_x=te, hoist=hoist, h=h, xs=xs, v=v)


def branches(use_cfg, drop_flags):
    return [(False, False), (True, True)] if use_cfg else [(bool(drop_flags & 1), bool(drop_flags & 2))]


def run_session(m, x, cond, text, tvals, ti, seq_len, use_cfg, drop_flags, NB):
    """Drive a DitSession directly (as sample() does, without the ODE loop): inputs, precompute, one forward."""
    B, N = x.shape[:2]
    s = m.session(B, NB, tvals.numel(), use_cfg, text.shape[1], seq_len is not None, bucketed=NB != N)
    pad = lambda a: F.pad(a, (0, 0, 0, NB - N))
    s.set_inputs(text, pad(cond).to(dev), tvals.to(dev), seq_len.to(dev) if seq_len is not None else None,
                 frames_valid=N if NB != N else None)
    s.c.drop_flags = drop_flags
    s.y_bf16.zero_()
    xb = pad(x).reshape(B * NB, -1).to(dev)
    for half in range(2 if use_cfg else 1):
        s.y_bf16[half * B * NB:(half + 1) * B * NB, :x.shape[-1]].copy_(xb)
    m.precompute(s)
    m.forward_session(s, ti)
    torch.cuda.synchronize()
    return s


def inputs(B, N, nt, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, 100, generator=g)
    cond = torch.randn(B, N, 100, generator=g) * 2 - 1
    text = torch.randint(0, 2545, (B, nt), generator=g, dtype=torch.int32)
    for b in range(1, B):
        text[b, nt - 7 * b:] = -1
    return x, cond, text


def eval_times(method):
    from f5_tts_mlx_b200.cfm import ode_eval_times, time_grid
    return ode_eval_times(time_grid(3, -1.0), method)      # midpoint / rk4 repeat times and take half steps


# (model, B, N, lens (ragged seq_len), CFG, drop_flags, fused AdaLN, bucket frames, solver whose times fill mod_table)
STAGE_CASES = [
    ("gate", 1, 63, None, True, 0, True, None, "rk4"),
    ("gate", 1, 64, None, False, 1, False, None, "midpoint"),
    ("gate", 1, 65, None, False, 2, True, None, "rk4"),
    ("gate", 1, 127, None, False, 3, True, None, "euler"),
    ("gate", 3, 128, [128, 101, 64], True, 0, True, None, "rk4"),
    ("gate", 3, 129, [129, 100, 63], True, 0, False, None, "midpoint"),
    ("gate", 1, 300, None, True, 0, True, 384, "rk4"),
    ("gate", 3, 150, [150, 120, 97], True, 0, True, 256, "midpoint"),
    ("gate", 1, 200, None, False, 3, False, 256, "rk4"),
    ("gate", 1, 1, None, False, 0, True, None, "euler"),
    ("d256", 1, 129, None, True, 0, True, None, "rk4"),
    ("d256", 3, 65, [65, 40, 64], False, 0, False, 128, "midpoint"),
    ("base", 1, 300, None, False, 0, True, None, "rk4"),
]


def _case_id(c):
    name, B, N, lens, use_cfg, drop, fused, NB, meth = c
    return f"{name}-B{B}-N{N}{'-cfg' if use_cfg else f'-drop{drop}'}-{'fused' if fused else 'unfused'}" \
           f"{f'-bucket{NB}' if NB else ''}"


@pytest.mark.parametrize("case", STAGE_CASES, ids=_case_id)
def test_dit_session_stages_per_row(case):
    name, B, N, lens, use_cfg, drop, fused, NB, meth = case
    cfg, W = weights(name)
    ocfg = ocfg_of(cfg)
    NB = NB or N
    x, cond, text = inputs(B, N, max(N // 3, 5) + 3, seed=N * 10 + B)
    if NB != N:                                      # sample()'s text bucketing: columns padded to a multiple of 32
        text = F.pad(text, (0, -(-text.shape[1] // 32) * 32 - text.shape[1]), value=-1)
    tvals = eval_times(meth)
    ti = min(2, tvals.numel() - 1)
    seq_len = torch.tensor(lens, dtype=torch.int32) if lens is not None else None
    mask = (torch.arange(N)[None] < seq_len[:, None]) if lens is not None else None
    prec = O.Precision(True, fused)
    brs = branches(use_cfg, drop)
    ref = [oracle_stages(W, ocfg, x, cond, text, tvals[ti], d, mask, O.FP32) for d in brs]
    emu = [oracle_stages(W, ocfg, x, cond, text, tvals[ti], d, mask, prec) for d in brs]
    nb = len(brs)
    view = lambda buf: buf.view(nb, B, NB, -1)[:, :, :N].cpu()
    stack = lambda rs, k: torch.stack([r[k] for r in rs])
    tag = _case_id(case)

    marks = {"gate": [1, 2, 3, 4], "d256": [1, 2, 3], "base": [1, 2, 22]}[name]
    for L in marks:
        s = run_session(model(name, L, fused), x, cond, text, tvals, ti, seq_len, use_cfg, drop, NB)
        report(f"{tag} x after block {L}",
               assert_rows(view(s.x), torch.stack([r["xs"][L - 1] for r in ref]),
                           torch.stack([r["xs"][L - 1] for r in emu]), what=f"{tag}: x after block {L}"))
    # the full model's session still holds every stage of that forward
    for k in ("text_x", "hoist", "h", "v"):
        report(f"{tag} {k}", assert_rows(view(getattr(s, k)), stack(ref, k), stack(emu, k), what=f"{tag}: {k}"))
    mt = s.mod_table.cpu()[None, None]
    report(f"{tag} mod_table", assert_rows(mt, oracle_mod_table(W, ocfg, tvals, O.FP32)[None, None],
                                           oracle_mod_table(W, ocfg, tvals, prec)[None, None], what=f"{tag}: mod_table"))
    if NB != N:                                      # bucket rows: the reference's zero padding, exactly
        for k in ("text_x", "hoist", "h"):
            exact_zero_rows(getattr(s, k).view(nb * B, NB, -1), N, what=f"{tag}: {k}")


@pytest.mark.parametrize("mode", ["tensor", "block"])
def test_fp8_forward_v_per_row(mode):
    """The FP8 modes' final v against their emulations: per-tensor (Precision(True, True, True)) and block-scaled
    (tests/fp8_block_emul.py), ragged batch of 3 with CFG."""
    cfg, W = weights("gate")
    ocfg = ocfg_of(cfg)
    B, N = 3, 150
    x, cond, text = inputs(B, N, 40, seed=77)
    lens = [150, 131, 90]
    seq_len = torch.tensor(lens, dtype=torch.int32)
    mask = torch.arange(N)[None] < seq_len[:, None]
    tvals = eval_times("euler")
    brs = branches(True, 0)
    s = run_session(model("gate", fp8=mode), x, cond, text, tvals, 0, seq_len, True, 0, N)
    got = s.v.view(2, B, N, -1).cpu()
    ref = torch.stack([O.dit_forward(x, cond, text, tvals[0], *d, mask, W, ocfg) for d in brs])
    if mode == "tensor":
        emu = torch.stack([O.dit_forward(x, cond, text, tvals[0], *d, mask, W, ocfg, O.Precision(True, True, True))
                           for d in brs])
    else:
        emu = torch.stack([oracle_stages(W, ocfg, x, cond, text, tvals[0], d, mask, O.Precision(True, True), True)["v"]
                           for d in brs])
    report(f"fp8 {mode} v", assert_rows(got, ref, emu, what=f"fp8 {mode}: v"))


# (model, depth, B, N, lens (ragged seq_len), bucket frames, block marks where x is checked)
FP8A_CASES = [("gate", 4, 3, 150, [150, 131, 90], None, [1, 2, 3, 4]),
              ("gate", 4, 3, 150, [150, 120, 97], 256, [1, 4]),
              ("base", 2, 1, 5625, None, None, [1, 2])]


@pytest.mark.parametrize("case", FP8A_CASES, ids=lambda c: f"{c[0]}-d{c[1]}-B{c[2]}-N{c[3]}{f'-bucket{c[5]}' if c[5] else ''}")
def test_fp8_attention_stages_per_row(case):
    """DiT(fp8=True, fp8_scaling="block", fp8_attention=True) with CFG: the residual stream x after each marked block
    (depth-truncated models) and v, per row, against fp8_attn_emul's blocks.  The base model at N = 5625 (60 s) runs
    the FP8 attention over 44 key tiles."""
    name, depth, B, N, lens, NB, marks = case
    cfg, W = weights(name)
    ocfg = dataclasses.replace(ocfg_of(cfg), depth=depth)
    NB = NB or N
    x, cond, text = inputs(B, N, min(max(N // 3, 5) + 3, 512), seed=N * 10 + B)
    if NB != N:
        text = F.pad(text, (0, -(-text.shape[1] // 32) * 32 - text.shape[1]), value=-1)
    tvals = eval_times("euler")
    seq_len = torch.tensor(lens, dtype=torch.int32) if lens is not None else None
    mask = (torch.arange(N)[None] < seq_len[:, None]) if lens is not None else None
    brs = branches(True, 0)
    ref = [oracle_stages(W, ocfg, x, cond, text, tvals[1], d, mask, O.FP32) for d in brs]
    emu = [oracle_stages(W, ocfg, x, cond, text, tvals[1], d, mask, O.Precision(True, True), attn8=True) for d in brs]
    view = lambda buf: buf.view(2, B, NB, -1)[:, :, :N].cpu()
    tag = f"fp8 attention {name} B{B} N{N}{f' bucket{NB}' if NB != N else ''}"
    for L in marks:
        s = run_session(model(name, L, fp8="block", fp8_attention=True), x, cond, text, tvals, 1, seq_len, True, 0, NB)
        report(f"{tag} x after block {L}",
               assert_rows(view(s.x), torch.stack([r["xs"][L - 1] for r in ref]),
                           torch.stack([r["xs"][L - 1] for r in emu]), what=f"{tag}: x after block {L}"))
    assert marks[-1] == depth
    report(f"{tag} v", assert_rows(view(s.v), torch.stack([r["v"] for r in ref]), torch.stack([r["v"] for r in emu]),
                                   what=f"{tag}: v"))


# ---------------------------------------------------------------- b. sample()
def sample_inputs(B, N, seed):
    g = torch.Generator().manual_seed(seed)
    nref = N // 3
    cond = (torch.randn(B, nref, 100, generator=g) * 2.24 - 1.27).clamp(-11.51, 5)
    text = torch.randint(0, 2545, (B, 30), generator=g, dtype=torch.int32)
    dur = torch.tensor([N] + [N - 17 * b - 5 for b in range(1, B)])
    y0 = torch.randn(B, N, 100, generator=g)
    for b in range(B):
        y0[b, int(dur[b]):] = 0
        text[b, 30 - 4 * b:] = -1
    return cond, text, dur, y0


# (solver, steps, CFG strength, batch, bucket, graph)
SAMPLE_CASES = [("euler", 4, 2.0, 3, 0, True), ("euler", 4, 0.0, 1, 128, False), ("midpoint", 3, 0.0, 1, 128, False),
                ("midpoint", 3, 2.0, 3, 0, True), ("rk4", 3, 2.0, 3, 128, True), ("rk4", 3, 0.0, 1, 0, False)]


@pytest.mark.parametrize("method,steps,cfg_strength,B,bucket,graph", SAMPLE_CASES)
def test_sample_out_and_last_state_per_row(method, steps, cfg_strength, B, bucket, graph):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W = weights("gate")
    N = 150
    cond, text, dur, y0 = sample_inputs(B, N, seed=steps * 10 + B)
    kw = dict(steps=steps, method=method, cfg_strength=cfg_strength, sway_sampling_coef=-1.0, y0=y0)
    ref, rtraj = O.sample(cond, text, dur, W, ocfg_of(cfg), **kw)
    emu, etraj = O.sample(cond, text, dur, W, ocfg_of(cfg), prec=O.Precision(True, True), **kw)
    f5 = F5TTS(model("gate"))
    f5.use_cuda_graph = graph
    out, traj = f5.sample(cond.to(dev), text, dur, frame_bucket=bucket, **kw)
    tag = f"sample {method} cfg{cfg_strength:g} B{B} {'bucket' if bucket else 'exact'} {'graph' if graph else 'eager'}"
    report(f"{tag} out", assert_rows(out.cpu()[None], ref[None], emu[None], what=f"{tag}: out"))
    report(f"{tag} last state", assert_rows(traj[-1].cpu()[None], rtraj[-1][None], etraj[-1][None],
                                            what=f"{tag}: trajectory[-1]"))


@pytest.mark.parametrize("method,steps,bucket", [("euler", 4, 0), ("rk4", 3, 128)])
def test_fp8_attention_sample_out_and_last_state_per_row(method, steps, bucket, monkeypatch):
    """sample() in the FP8 attention mode, ragged batch of 3 with CFG, against the oracle's sample() whose DiT calls
    are fp8_attn_emul.dit_forward_block8a."""
    import fp8_attn_emul as A
    from f5_tts_mlx_b200 import F5TTS
    cfg, W = weights("gate")
    B, N = 3, 150
    cond, text, dur, y0 = sample_inputs(B, N, seed=steps * 10 + B + 1)
    kw = dict(steps=steps, method=method, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
    ref, rtraj = O.sample(cond, text, dur, W, ocfg_of(cfg), **kw)
    with monkeypatch.context() as mp:
        mp.setattr(O, "dit_forward", lambda x, c, t, time, da, dt, mask, W, cfg, prec=None:
                   A.dit_forward_block8a(x, c, t, time, da, dt, mask, W, cfg))
        emu, etraj = O.sample(cond, text, dur, W, ocfg_of(cfg), **kw)
    f5 = F5TTS(model("gate", fp8="block", fp8_attention=True))
    out, traj = f5.sample(cond.to(dev), text, dur, frame_bucket=bucket, **kw)
    tag = f"sample fp8 attention {method} B{B} {'bucket' if bucket else 'exact'}"
    report(f"{tag} out", assert_rows(out.cpu()[None], ref[None], emu[None], what=f"{tag}: out"))
    report(f"{tag} last state", assert_rows(traj[-1].cpu()[None], rtraj[-1][None], etraj[-1][None],
                                            what=f"{tag}: trajectory[-1]"))


def test_one_euler_step_per_row_equals_two_dit_calls():
    """The doubled-batch CFG step of sample() equals y0 + dt (pred + (pred - null) cfg) from two DiT calls, per row:
    the same kernels on the same rows, so only the update's fp32 arithmetic may differ."""
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.cfm import time_grid
    m = model("gate")
    B, N = 3, 150
    cond, text, dur, y0 = sample_inputs(B, N, seed=3)
    out, traj = F5TTS(m).sample(cond.to(dev), text, dur, steps=2, method="euler", cfg_strength=2.0,
                                sway_sampling_coef=-1.0, y0=y0)
    lens = torch.maximum((text != -1).sum(-1), torch.full((B,), cond.shape[1]))
    step_cond = torch.zeros(B, N, 100)
    for b in range(B):
        step_cond[b, :int(lens[b])] = F.pad(cond[b], (0, 0, 0, N - cond.shape[1]))[:int(lens[b])]
    mask = (torch.arange(N)[None] < dur[:, None]).to(dev)
    t = time_grid(2, -1.0)
    pred = m(y0.to(dev), step_cond.to(dev), text.to(dev), t[0], False, False, mask)
    null = m(y0.to(dev), step_cond.to(dev), text.to(dev), t[0], True, True, mask)
    y1 = y0.to(dev) + (t[1] - t[0]) * (pred + (pred - null) * 2.0)
    err = row_errors(traj[1][None], y1[None])
    worst = err.max().item()
    print(f"COMPOSED euler step vs two DiT calls: worst row error {worst:.2e}")
    assert worst < 1e-5, f"row {tuple(int(i) for i in (err == err.max()).nonzero()[0])}: {worst:.3e}"


# ---------------------------------------------------------------- c. duration model
def test_duration_predictor_per_utterance_and_per_row():
    from f5_tts_mlx_b200.duration import DurationPredictor, DurationTransformer
    from f5_tts_mlx_b200.weights import random_duration_weights
    dW = random_duration_weights(seed=5)
    dWo = {"duration." + k: v for k, v in dW.items()}
    dcfg = O.DurationConfig()
    pred = DurationPredictor(DurationTransformer(dim=512, depth=8, heads=8, text_dim=512, ff_mult=2, conv_layers=2,
                                                 text_num_embeds=2545), device=dev).load_weights(dW)
    g = torch.Generator().manual_seed(11)
    B, N = 3, 130
    mel = torch.randn(B, N, 100, generator=g) * 2.24 - 1.27
    text = torch.randint(0, 2545, (B, 48), generator=g, dtype=torch.int32)
    text[1, 30:] = -1; text[2, 11:] = -1
    lens = torch.tensor([130, 97, 64])
    got = pred(mel.to(dev), text, lens=lens).cpu()
    ref = O.duration_predictor(mel, text, dWo, dcfg, lens=lens)
    emu = O.duration_predictor(mel, text, dWo, dcfg, lens=lens, prec=O.Precision(True))
    for u in range(B):
        drift = abs(emu[u].item() - ref[u].item())
        err = abs(got[u].item() - ref[u].item())
        bound = max(3 * drift, 2e-3 * abs(ref[u].item()))
        print(f"COMPOSED duration seconds utterance {u}: {err:.2e} vs emulated drift {drift:.2e}")
        assert err <= bound, (u, got[u].item(), ref[u].item(), emu[u].item())
    # the residual stream before the head's RMSNorm, per row (apply the norm here)
    x = pred._bufs[(B, N, text.shape[1])][0]["x"].view(1, B, N, -1).cpu()
    nw = dW["transformer.norm_out.weight"].float()
    xn = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-5) * nw
    m = (torch.arange(N)[None] < lens[:, None])[..., None]
    inp = torch.where(m, mel, torch.zeros_like(mel))
    xr = O.duration_transformer(inp, text, dWo, dcfg)[None]
    xe = O.duration_transformer(inp, text, dWo, dcfg, O.Precision(True))[None]
    report("duration x (RMS-normed)", assert_rows(xn, xr, xe, what="duration: x"))


# ---------------------------------------------------------------- d. Vocos
@pytest.mark.parametrize("norm,trim", [("window", False), ("window_sq", True)])
def test_vocos_per_hop_segment_and_head_per_frame(norm, trim):
    from f5_tts_mlx_b200.vocos import Vocos
    from f5_tts_mlx_b200.weights import VocosConfig, random_vocos_weights
    vc, ovc = VocosConfig(istft_norm=norm, istft_trim=trim), O.VocosConfig(istft_norm=norm, istft_trim=trim)
    vw = random_vocos_weights(vc, seed=4321)
    voc = Vocos(vc, dev).load_weights(vw)
    g = torch.Generator().manual_seed(13)
    B, n = 2, 150
    mel = (torch.randn(B, n, 100, generator=g) * 2.24 - 1.27).clamp(-11.5, 5)
    got = voc.decode(mel.to(dev)).cpu()
    ref = torch.stack([O.vocos_decode(mel[b:b + 1], vw, ovc) for b in range(B)])
    emu = torch.stack([O.vocos_decode(mel[b:b + 1], vw, ovc, O.Precision(True)) for b in range(B)])
    hop = vc.hop_length
    assert got.shape == ref.shape and got.shape[1] % hop == 0
    seg = lambda w: w.reshape(1, B, -1, hop)            # every hop segment, the overlap-add and trim edges included
    report(f"vocos {norm} wave per hop", assert_rows(seg(got), seg(ref), seg(emu), what=f"vocos {norm}: wave"))
    head = voc._bufs[(B, n)][0]["head"].view(1, B, n, -1)[..., :vc.n_fft + 2].cpu()
    hw, hb = vw["vocos.head.out.weight"], vw["vocos.head.out.bias"]
    hr = torch.stack([O.linear(O.vocos_backbone(mel[b:b + 1], vw, ovc)[0], hw, hb) for b in range(B)])[None]
    he = torch.stack([O.linear(O.vocos_backbone(mel[b:b + 1], vw, ovc, O.Precision(True))[0], hw, hb, O.Precision(True))
                      for b in range(B)])[None]
    report(f"vocos {norm} head per frame", assert_rows(head, hr, he, what=f"vocos {norm}: head"))


# ---------------------------------------------------------------- e. state reuse, bitwise
def fresh_f5(**attrs):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W = weights("gate")
    f5 = F5TTS(make_dit(cfg, W))
    for k, v in attrs.items():
        setattr(f5, k, v)
    return f5


def assert_bitwise(a, b, what):
    assert a.shape == b.shape and torch.equal(a, b), \
        f"{what}: differs from a fresh model, max |diff| {(a.float() - b.float()).abs().max().item():.3e}"


def test_bucketed_plan_descending_lengths_bitwise():
    """One bucketed plan (256 frames) driven with N = 255, 150, 201, 150: a shorter utterance after a longer one must
    not see the longer one's rows."""
    f5 = fresh_f5(frame_bucket=128)
    g = torch.Generator().manual_seed(41)
    cond = (torch.randn(1, 60, 100, generator=g) * 2.24 - 1.27)
    kw = dict(steps=3, method="midpoint", cfg_strength=2.0, sway_sampling_coef=-1.0)
    plans = set()
    for N in (255, 150, 201, 150):
        text = torch.randint(0, 2545, (1, 20 + N % 13), generator=g, dtype=torch.int32)
        y0 = torch.randn(1, N, 100, generator=g)
        out, traj = f5.sample(cond.to(dev), text, N, y0=y0, **kw)
        plans.add(id(f5.last_plan))
        out_f, traj_f = fresh_f5(frame_bucket=128).sample(cond.to(dev), text, N, y0=y0, **kw)
        assert_bitwise(out, out_f, f"N={N} out")
        assert_bitwise(traj, traj_f, f"N={N} trajectory")
    assert len(plans) == 1


def test_dit_call_and_sample_share_a_session_bitwise():
    """DiT.__call__ and sample(steps=2, euler, no CFG) on one utterance have the same session key: interleaved, with
    drop flags set by the calls, each result equals that of a fresh model."""
    f5 = fresh_f5()
    m = f5.transformer
    g = torch.Generator().manual_seed(42)
    N = 130
    cond = (torch.randn(1, 40, 100, generator=g) * 2.24 - 1.27)
    text = torch.randint(0, 2545, (1, 25), generator=g, dtype=torch.int32)
    y0 = torch.randn(1, N, 100, generator=g)
    step_cond = F.pad(cond, (0, 0, 0, N - 40))
    skw = dict(steps=2, method="euler", cfg_strength=0.0, sway_sampling_coef=-1.0, y0=y0)
    t = torch.tensor(0.3)
    calls = [("call", (True, True)), ("sample", None), ("call", (False, True)), ("sample", None), ("call", (True, False))]
    for kind, drops in calls:
        if kind == "call":
            a = m(y0.to(dev), step_cond.to(dev), text.to(dev), t, *drops)
            b = make_dit(*weights("gate"))(y0.to(dev), step_cond.to(dev), text.to(dev), t, *drops)
        else:
            a = f5.sample(cond.to(dev), text, N, **skw)[0]
            b = fresh_f5().sample(cond.to(dev), text, N, **skw)[0]
        assert_bitwise(a, b, f"{kind} {drops}")
    assert len(m._sessions) == 1


def test_plan_cache_of_one_evicts_and_recaptures_bitwise():
    f5 = fresh_f5(plan_cache_size=1)
    g = torch.Generator().manual_seed(43)
    cond = (torch.randn(2, 50, 100, generator=g) * 2.24 - 1.27)
    text = torch.randint(0, 2545, (2, 30), generator=g, dtype=torch.int32)
    text[1, 21:] = -1
    shapes = {"A": torch.tensor([140, 120]), "B": torch.tensor([99, 99])}
    kw = dict(steps=3, method="rk4", cfg_strength=2.0, sway_sampling_coef=-1.0, seed=5)
    for name in "ABAB":
        a = f5.sample(cond.to(dev), text, shapes[name], **kw)[0]
        b = fresh_f5().sample(cond.to(dev), text, shapes[name], **kw)[0]
        assert len(f5._plans) == 1
        assert_bitwise(a, b, f"shape {name}")


def test_graph_replay_equals_eager_bitwise():
    g = torch.Generator().manual_seed(44)
    cond = (torch.randn(3, 50, 100, generator=g) * 2.24 - 1.27)
    text = torch.randint(0, 2545, (3, 30), generator=g, dtype=torch.int32)
    dur = torch.tensor([150, 131, 97])
    kw = dict(steps=3, method="midpoint", cfg_strength=2.0, sway_sampling_coef=-1.0, seed=9)
    f5 = fresh_f5()
    eager = fresh_f5(use_cuda_graph=False)
    for bucket in (0, 128):
        for _ in range(2):            # capture, then replay
            a, ta = f5.sample(cond.to(dev), text, dur, frame_bucket=bucket, **kw)
            b, tb = eager.sample(cond.to(dev), text, dur, frame_bucket=bucket, **kw)
            assert_bitwise(a, b, f"bucket {bucket} out")
            assert_bitwise(ta, tb, f"bucket {bucket} trajectory")


def test_vocos_and_duration_buffer_caches_bitwise():
    from f5_tts_mlx_b200.duration import DurationPredictor, DurationTransformer
    from f5_tts_mlx_b200.vocos import Vocos
    from f5_tts_mlx_b200.weights import VocosConfig, random_duration_weights, random_vocos_weights
    vw, dW = random_vocos_weights(), random_duration_weights(seed=5)
    mk_v = lambda: Vocos(VocosConfig(), dev).load_weights(vw)
    mk_d = lambda: DurationPredictor(DurationTransformer(dim=512, depth=8, heads=8, text_dim=512, ff_mult=2,
                                                         conv_layers=2, text_num_embeds=2545), device=dev).load_weights(dW)
    g = torch.Generator().manual_seed(45)
    mels = {"A": torch.randn(2, 120, 100, generator=g), "B": torch.randn(1, 77, 100, generator=g)}
    texts = {"A": torch.randint(0, 2545, (2, 40), generator=g, dtype=torch.int32),
             "B": torch.randint(0, 2545, (1, 20), generator=g, dtype=torch.int32)}
    texts["A"][1, 33:] = -1
    voc, dur = mk_v(), mk_d()
    for name in "ABA":
        assert_bitwise(voc.decode(mels[name].to(dev)), mk_v().decode(mels[name].to(dev)), f"vocos {name}")
        assert_bitwise(dur(mels[name].to(dev), texts[name]), mk_d()(mels[name].to(dev), texts[name]), f"duration {name}")
