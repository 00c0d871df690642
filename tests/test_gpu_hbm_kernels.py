"""-m gpu: the HBM-bound kernels of csrc/elementwise.cuh, each alone through its C entry, element-wise against a
float64 restatement within the bounds derived in hbm_check.py, or bitwise where the kernel's arithmetic is one fp32
operation per element.  Outputs land in NaN-filled guard buffers (kernel_check.Guarded).

COVERED names every kernel instantiation these tests launch; a CPU test (test_hbm_check.py) parses elementwise.cuh /
elementwise.cu and fails if a kernel or a dispatch case is missing from it."""
import math

import numpy as np
import pytest
import torch

from hbm_check import (U, dwconv7_ref_bound, duration_ref_bound, gam, grn_ref_bound, ln_ref_bound, ode_axpy_bound,
                       ode_k, rows, time_mlp_ref_bound)
from kernel_check import Guarded, assert_exact, assert_within, round_to

pytestmark = pytest.mark.gpu
dev = "cuda"

LN_DIMS = [256, 512, 768, 1024, 1536, 2048]
CONV_DIMS = [256, 512, 1024]
HEAD_DIMS = [256, 512, 1024]
COVERED = ({f"ln_mod_kernel<{d},bf16>" for d in LN_DIMS} | {f"ln_mod_kernel<{d},f32>" for d in LN_DIMS}
           | {f"dwconv7_ln_kernel<{c}>" for c in CONV_DIMS} | {f"duration_head_kernel<{d}>" for d in HEAD_DIMS}
           | {"ln_tab_prep_kernel", "grn_sumsq_kernel", "grn_finalize_kernel", "grn_apply_kernel",
              "text_embed_gather_kernel", "time_mlp_kernel", "cfg_ode_update_kernel", "cast_pad_bf16_kernel",
              "concat_cond_text_kernel"})


def lib():
    from f5_tts_mlx_b200 import _lib
    return _lib


def call(name, *args):
    _lib = lib()
    conv = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    _lib.check(getattr(_lib.load(), name)(*conv, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()


def randn(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dev)


WORST = {}


def note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst err/bound per kernel and mode:")
        for k, v in sorted(WORST.items()):
            print(f"  {k:48s} {v:.3g}")


# ---------------------------------------------------------------- LayerNorm + modulate / affine
def _ln_input(R, D, seed):
    """Random rows; from row 3 on every 5th row has offset 1e3 and spread 1, and rows 4 and 9 are constant."""
    x = randn(R, D, seed=seed) * 2 + 0.5
    if R > 3:
        x[3::5] = randn(len(range(3, R, 5)), D, seed=seed + 1) + 1e3
    for r in (4, 9):
        if r < R:
            x[r] = 3.0
    return x


@pytest.mark.parametrize("D", LN_DIMS)
@pytest.mark.parametrize("mode", ["modulate", "affine", "batched", "affine_f32"])
def test_ln_mod_kernel(D, mode):
    for R in (1, 7, 777):
        x = _ln_input(R, D, seed=D + R)
        out_dtype = torch.float32 if mode == "affine_f32" else torch.bfloat16
        y = Guarded(R, D, out_dtype, dev, lr=False)
        if mode == "batched":
            nb, per = 4, -(-R // 4)
            stride = 3 * D + 64
            mod = randn(nb, stride, seed=D, scale=0.5)
            g, h = mod[:, D:2 * D], mod[:, :D]
            call("f5_ln_modulate", x, y.view, R, D, per, g, h, stride, 1)
            bidx = torch.arange(R, device=dev) // per
            G, H = g[bidx], h[bidx]
        else:
            g = randn(D, seed=D + 1, scale=0.5) + (0.0 if mode == "modulate" else 1.0)
            h = randn(D, seed=D + 2, scale=0.5)
            if mode == "affine_f32":
                call("f5_ln_affine_f32", x, y.view, R, D, g, h)
            else:
                call("f5_ln_modulate", x, y.view, R, D, 0, g, h, 0, int(mode == "modulate"))
            G, H = g.expand(R, D), h.expand(R, D)
        y.check(f"ln {mode} D={D} R={R}")
        ref, b = ln_ref_bound(x, G, H, mode in ("modulate", "batched"), out_dtype)
        note(f"ln_mod {mode}", assert_within(y.view, ref, b, rows(), f"ln {mode} D={D} R={R}"))


# ---------------------------------------------------------------- fused-AdaLN operand rows (bitwise)
@pytest.mark.parametrize("depth,D", [(4, 512), (22, 1024)])
@pytest.mark.parametrize("T", [1, 7, 124])
def test_ln_tab_prep(depth, D, T):
    NM = depth * 6 * D + 2 * D
    mod = randn(T, NM, seed=T, scale=2.0)
    prep = Guarded((2 * depth + 1) * 4 * T, D, torch.bfloat16, dev, lr=False)
    call("f5_ln_tab_prep", mod, prep.view, T, depth, D, NM)
    prep.check("ln_tab_prep")
    m = mod.cpu()
    want = torch.empty((2 * depth + 1), 4 * T, D, dtype=torch.bfloat16)
    for site in range(2 * depth + 1):
        if site < 2 * depth:        # attention norm (even) and FF norm (odd) of block site // 2
            base = (site >> 1) * 6 * D + (3 * D if site & 1 else 0)
            sh, sc = base, base + D
        else:                       # final norm: scale, then shift
            sc = depth * 6 * D
            sh = sc + D
        a = 1.0 + m[:, sc:sc + D]              # one fp32 add
        bb = m[:, sh:sh + D]
        ah, bh = a.bfloat16(), bb.bfloat16()
        rows_ = torch.stack([ah, (a - ah.float()).bfloat16(), bh, (bb - bh.float()).bfloat16()], 1)
        want[site] = rows_.reshape(4 * T, D)
    assert_exact(prep.view.cpu(), want.reshape(-1, D), rows("prep row"), f"ln_tab_prep depth={depth} T={T}")


# ---------------------------------------------------------------- depthwise conv 7 + LayerNorm
@pytest.mark.parametrize("C", CONV_DIMS)
@pytest.mark.parametrize("N", [1, 2, 3, 6, 7, 8, 333])
def test_dwconv7_ln(C, N):
    """B = 3 utterances with different scales and offsets: an edge row that read the neighbouring utterance instead of
    zero padding is off by far more than the bound."""
    B = 3
    x = torch.stack([randn(N, C, seed=N + b) * (1 + b) + 3 * b for b in range(B)])
    wt = randn(7, C, seed=C, scale=0.4)
    wb, lw, lb = randn(C, seed=1), 1 + 0.1 * randn(C, seed=2), 0.1 * randn(C, seed=3)
    y = Guarded(B * N, C, torch.bfloat16, dev, lr=False)
    call("f5_dwconv7_ln", x, y.view, B, N, C, wt, wb, lw, lb)
    y.check(f"dwconv7 C={C} N={N}")
    ref, b = dwconv7_ref_bound(x, wt, wb, lw, lb)
    note("dwconv7_ln", assert_within(y.view, ref, b, lambda r, c: f"(utt {r // N}, frame {r % N}) col {c}",
                                     f"dwconv7 C={C} N={N}"))


# ---------------------------------------------------------------- GRN
@pytest.mark.parametrize("N", [1, 31, 32, 33, 333])
@pytest.mark.parametrize("valid", [False, True])
def test_grn(N, valid):
    B, C = 3, 1024
    h = (randn(B, N, C, seed=N) * 2).bfloat16()
    gamma, beta = randn(C, seed=5, scale=0.5), randn(C, seed=6, scale=0.5)
    nblk = -(-N // 32)
    vl = torch.tensor([N, max(1, N - 5), max(1, N // 2)], dtype=torch.int32, device=dev) if valid else None
    if valid:
        for b in range(B):      # excluded rows carry large values: they must not enter the norm
            h[b, int(vl[b]):] = 200.0
    outs = []
    for _ in range(2):
        y = Guarded(B * N, C, torch.bfloat16, dev, lr=False)
        nx = torch.full((B, 1 + nblk, C), float("nan"), device=dev)
        if valid:
            call("f5_grn_valid", h, y.view, nx, gamma, beta, B, N, C, vl)
        else:
            call("f5_grn", h, y.view, nx, gamma, beta, B, N, C)
        y.check(f"grn N={N}")
        outs.append(y.view.clone())
    assert_exact(outs[1], outs[0], rows(), "grn run-to-run")
    ref, b = grn_ref_bound(h, gamma, beta, vl)
    note(f"grn valid={valid}", assert_within(outs[0], ref, b, lambda r, c: f"(utt {r // N}, frame {r % N}) col {c}",
                                             f"grn N={N} valid={valid}"))


# ---------------------------------------------------------------- text embedding gather (bitwise)
VOCAB = 2546


def _text_ref(text, B, nt, N, emb, pos, max_pos, Bout, drop_from, mask_padding, valid_len):
    t, e, p = text.cpu(), emb.cpu(), pos.cpu()
    C = e.shape[1]
    out = torch.zeros(Bout, N, C)
    for bo in range(Bout):
        ids = torch.zeros(N, dtype=torch.long)
        k = min(nt, N)
        ids[:k] = t[bo % B, :k].long() + 1
        masked = (ids == 0) if mask_padding else torch.zeros(N, dtype=torch.bool)
        if valid_len is not None:
            masked |= torch.arange(N) >= int(valid_len[bo])
        if bo >= drop_from:
            ids[:] = 0
        pidx = torch.arange(N).clamp(max=max_pos - 1)
        v = e[ids] + p[pidx]                   # one fp32 add
        out[bo] = torch.where(masked[:, None], torch.zeros(()), v)
    return out.reshape(Bout * N, C)


@pytest.mark.parametrize("case", ["cfg", "drop_all", "no_mask", "nt_gt_N", "long_N", "bucketed"])
def test_text_embed(case):
    C, max_pos = 512, 4096
    B, N, nt, Bout, drop_from, mask_padding, vl = 2, 150, 60, 4, 2, 1, None
    if case == "drop_all":
        Bout, drop_from = 2, 0
    elif case == "no_mask":
        Bout, drop_from, mask_padding = 2, 2, 0
    elif case == "nt_gt_N":
        N, nt = 150, 200
    elif case == "long_N":
        B, N, nt, Bout, drop_from = 1, 5625, 300, 2, 1
    elif case == "bucketed":     # a 256-row bucket holding N = 150 real frames, text longer than N
        N, nt = 256, 288
        vl = torch.tensor([150] * Bout, dtype=torch.int32, device=dev)
    g = torch.Generator().manual_seed(7)
    text = torch.randint(0, VOCAB - 1, (B, nt), generator=g, dtype=torch.int32)
    text[0, :3] = torch.tensor([VOCAB - 2, 0, VOCAB - 2], dtype=torch.int32)     # vocabulary edges
    text[1 % B, nt - 7:] = -1                                                     # right padding
    text = text.to(dev)
    emb, pos = randn(VOCAB, C, seed=8), randn(max_pos, C, seed=9)
    x = Guarded(Bout * N, C, torch.float32, dev, lr=False)
    call("f5_text_embed", text, B, nt, N, C, emb, pos, max_pos, x.view, Bout, drop_from, mask_padding, vl)
    x.check(f"text_embed {case}")
    want = _text_ref(text, B, nt, N, emb, pos, max_pos, Bout, drop_from, mask_padding, vl)
    assert_exact(x.view.cpu(), want, lambda r, c: f"(utt {r // N}, frame {r % N}) col {c}", f"text_embed {case}")
    if vl is not None:
        assert (x.view.view(Bout, N, C)[:, 150:] == 0).all()


# ---------------------------------------------------------------- timestep MLP
def _sway_rk4_times(steps=32, sway=-1.0):
    t = np.linspace(0, 1, steps, dtype=np.float32)
    t = (t + sway * (np.cos(np.pi / 2 * t) - 1 + t)).astype(np.float32)
    out = []
    for i in range(steps - 1):
        dt = np.float32(t[i + 1] - t[i])
        out += [t[i], t[i] + np.float32(0.5) * dt, t[i] + np.float32(0.5) * dt, t[i] + dt]
    return torch.tensor(np.array(out, dtype=np.float32))


@pytest.mark.parametrize("D", [512, 1024])
@pytest.mark.parametrize("grid", ["points", "sway_rk4"])
def test_time_mlp(D, grid):
    tv = torch.tensor([0.0, 1e-3, 0.37, 1.0]) if grid == "points" else _sway_rk4_times()
    T = tv.shape[0]
    tv = tv.to(dev)
    w0, b0 = randn(D, 256, seed=D, scale=1 / 16), randn(D, seed=D + 1, scale=0.1)
    w2, b2 = randn(D, D, seed=D + 2, scale=D ** -0.5), randn(D, seed=D + 3, scale=0.1)
    te = Guarded(T, D, torch.float32, dev, lr=False)
    sb = Guarded(T, D, torch.bfloat16, dev, lr=False)
    call("f5_time_mlp", tv, T, D, w0, b0, w2, b2, te.view, sb.view)
    te.check("t_emb"); sb.check("silu bf16")
    v, bv, s, bs = time_mlp_ref_bound(tv, w0, b0, w2, b2)
    note("time_mlp t_emb", assert_within(te.view, v, bv, rows("time"), f"time_mlp t_emb D={D} {grid}"))
    note("time_mlp silu bf16", assert_within(sb.view, s, bs, rows("time"), f"time_mlp silu D={D} {grid}"))
    sb2 = torch.empty(T, D, dtype=torch.bfloat16, device=dev)    # t_emb = NULL: the bf16 output alone, unchanged
    call("f5_time_mlp", tv, T, D, w0, b0, w2, b2, None, sb2)
    assert_exact(sb2, sb.view, rows("time"), "time_mlp without t_emb")


# ---------------------------------------------------------------- CFG combine + solver stage update
def _ode_stage(v, ldv, null_off, cfg, y_base, a, k_acc, acc_w, acc_init, use_acc, rows_, d, dup):
    y_out = Guarded(rows_, d, torch.float32, dev, lr=False)
    yb = Guarded(rows_ + dup, d, torch.bfloat16, dev)
    ld_bf16 = yb.buf.stride(0)
    call("f5_ode_update", v, ldv, null_off, cfg, y_base, y_out.view, a, k_acc, acc_w, acc_init, use_acc, yb.view,
         ld_bf16, dup, rows_, d)
    y_out.check("ode y_out")
    if dup:
        yb.check("ode y_bf16")
        assert_exact(yb.view[dup:], yb.view[:dup], rows(), "ode duplicated bf16 rows")
    else:
        yb.check("ode y_bf16")
    assert_exact(yb.view[:rows_], y_out.view.bfloat16(), rows(), "ode bf16 copy")
    return y_out.view


@pytest.mark.parametrize("use_cfg", [False, True])
@pytest.mark.parametrize("ldv", [100, 128])
def test_ode_update_stages(use_cfg, ldv):
    """Every stage configuration f5_ode_sample launches (Euler; both midpoint stages; rk4's four), then the four rk4
    stages chained on synthetic flows against a float64 RK4 step."""
    rows_, d, cfg = 300, 100, 2.0
    null_off = rows_ if use_cfg else 0
    dup = rows_ if use_cfg else 0
    y0 = randn(rows_, d, seed=1)
    dt = 0.0421
    vs = [randn(2 * rows_ if use_cfg else rows_, ldv, seed=10 + s) for s in range(4)]
    ks = [ode_k(v, rows_, d, null_off, cfg) for v in vs]
    # Euler and the midpoint stages: y = y0 + a k
    for a in (dt, np.float32(0.5) * np.float32(dt)):
        got = _ode_stage(vs[0], ldv, null_off, cfg, y0, float(a), None, 0.0, 0, 0, rows_, d, dup)
        k, bk = ks[0]
        note("ode stage", assert_within(got, y0.double() + float(a) * k, ode_axpy_bound(y0, float(a), k, bk),
                                        rows(), f"ode stage a={a}"))
    # rk4: acc = k1 + 2 k2 + 2 k3 + k4, y_tmp = y0 + a_s k_s, y_next = y0 + (dt / 6) acc
    f32 = np.float32
    as_ = [f32(0.5) * f32(dt), f32(0.5) * f32(dt), f32(dt), f32(dt) / f32(6)]
    ws = [1.0, 2.0, 2.0, 1.0]
    k_acc = torch.full((rows_, d), float("nan"), device=dev)
    acc = torch.zeros(rows_, d, dtype=torch.float64, device=dev)
    bacc = torch.zeros_like(acc)
    for s in range(4):
        got = _ode_stage(vs[s], ldv, null_off, cfg, y0, float(as_[s]), k_acc, ws[s], int(s == 0), int(s == 3),
                         rows_, d, dup)
        k, bk = ks[s]
        acc = acc + ws[s] * k
        bacc = bacc + ws[s] * bk + U * ws[s] * k.abs() + U * acc.abs()
        note("ode rk4 k_acc", assert_within(k_acc, acc, bacc + 1e-300, rows(), f"rk4 k_acc stage {s}"))
        if s < 3:
            note("ode stage", assert_within(got, y0.double() + float(as_[s]) * k,
                                            ode_axpy_bound(y0, float(as_[s]), k, bk), rows(), f"rk4 stage {s}"))
    ref = y0.double() + dt / 6 * acc
    b = ode_axpy_bound(y0, dt / 6, acc, bacc) + 2 * U * abs(dt / 6) * acc.abs()   # fp32 dt and dt/6 vs float64
    note("ode rk4 chain", assert_within(got, ref, b, rows(), "rk4 step vs float64"))


# ---------------------------------------------------------------- cast / concat (bitwise)
@pytest.mark.parametrize("copy", [0, 1])
def test_cast_pad_bf16(copy):
    R, d, ld = 300, 100, 128
    src = randn(R, d, seed=3) * 5
    dst = Guarded(R * (1 + copy), ld, torch.bfloat16, dev, lr=False)
    call("f5_cast_pad_bf16", src, d, dst.view, ld, R, R if copy else 0)
    dst.check("cast_pad_bf16")
    want = torch.zeros(R, ld, dtype=torch.bfloat16)
    want[:, :d] = src.cpu().bfloat16()
    assert_exact(dst.view.cpu(), want.repeat(1 + copy, 1), rows(), "cast_pad_bf16")


@pytest.mark.parametrize("case", ["cfg", "cond_len", "drop_all"])
def test_concat_cond_text(case):
    Bc, N, dc, dt, ld = 2, 150, 100, 512, 640
    rows_ = 2 * Bc * N if case == "cfg" else Bc * N
    drop_from = {"cfg": Bc * N, "cond_len": rows_, "drop_all": 0}[case]
    cond, text = randn(Bc, N, dc, seed=4), randn(rows_, dt, seed=5)
    cl = torch.tensor([N - 40, 0], dtype=torch.int32, device=dev) if case == "cond_len" else None
    dst = Guarded(rows_, ld, torch.bfloat16, dev, lr=False)
    call("f5_concat_cond_text", cond, dc, Bc, N, text, dt, dst.view, ld, rows_, drop_from, cl)
    dst.check(f"concat {case}")
    want = torch.zeros(rows_, ld)
    c = cond.cpu()
    for r in range(min(drop_from, rows_)):
        b, n = (r // N) % Bc, r % N
        if cl is None or n < int(cl[b]):
            want[r, :dc] = c[b, n]
    want[:, dc:dc + dt] = text.cpu()
    assert_exact(dst.view.cpu(), want.bfloat16(), rows(), f"concat {case}")


# ---------------------------------------------------------------- duration head
@pytest.mark.parametrize("D", HEAD_DIMS)
def test_duration_head(D):
    N = 2000
    lens = torch.tensor([0, 1, 7, N, N + 500, 1, 1], dtype=torch.int32)
    B = lens.shape[0]
    x = randn(B, N, D, seed=D) * 1.5 + 0.2
    nw, pw = 1 + 0.2 * randn(D, seed=D + 1), randn(D, seed=D + 2) * 0.5
    v = (nw * pw).sign()
    x[5] = x[5].abs() * v            # a large positive head value: softplus's t > 20 branch
    x[6] = -x[6].abs() * v           # and a large negative one (t < -20)
    out = Guarded(B, 1, torch.float32, dev, lr=False)
    call("f5_duration_head", x, B, N, D, lens.to(dev), nw, pw, out.view)
    out.check("duration head")
    ref, b, t = duration_ref_bound(x, lens, nw, pw)
    assert t[5] > 20 and t[6] < -20, t
    note("duration_head", assert_within(out.view, ref[:, None], b[:, None], rows("utt"), f"duration head D={D}"))
