"""CPU: the checkers of hbm_check.py accept an fp32 torch restatement of each kernel and reject, naming the location,
the mistakes these kernels could make; fft16's hand-written constants and swaps compute the DFT; and every kernel and
dispatch case of elementwise.cuh / elementwise.cu / audio_vocos.cu has a GPU test."""
import math
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from hbm_check import (U, duration_ref_bound, dwconv7_ref_bound, grn_ref_bound, istft_frames_ref_bound,
                       istft_ola_ref_bound, ln_ref_bound, mel_ref_bound, ode_axpy_bound, ode_k, rows)
from kernel_check import assert_exact, assert_within

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "f5_tts_mlx_b200" / "csrc"


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


# ---------------------------------------------------------------- LayerNorm
def ln_fp32(x, G, h, one_pass=False):
    x = x.float()
    mu = x.mean(-1, keepdim=True)
    if one_pass:
        var = (x * x).mean(-1, keepdim=True) - mu * mu
    else:
        var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return ((x - mu) * torch.rsqrt(var + 1e-6) * G + h).bfloat16()


def _ln_rows(R=40, D=512):
    x = rnd(R, D) * 2 + 0.5
    x[3::5] = rnd(len(range(3, R, 5)), D, seed=1) + 1e3
    x[4] = 3.0
    return x, 1 + 0.5 * rnd(D, seed=2), 0.5 * rnd(D, seed=3)


def test_ln_accepts_two_pass_and_rejects_one_pass_variance_on_offset_rows():
    x, g, h = _ln_rows()
    ref, b = ln_ref_bound(x, g.expand_as(x), h.expand_as(x), False, torch.bfloat16)
    assert assert_within(ln_fp32(x, g, h), ref, b, rows(), "two-pass") <= 1
    with pytest.raises(AssertionError, match=r"row (3|8|13|18|23|28|33|38) "):
        assert_within(ln_fp32(x, g, h, one_pass=True), ref, b, rows(), "one-pass")


# ---------------------------------------------------------------- dwconv7 + LayerNorm
def dwconv7_fp32(x, wt, wb, lw, lb, shift_tap=None):
    B, N, C = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 3, 4))
    acc = wb.expand(B, N, C).clone()
    for t in range(7):
        s = t + 1 if t == shift_tap else t
        acc = acc + xp[:, s:s + N] * wt[t]
    return torch.nn.functional.layer_norm(acc, (C,), lw, lb, eps=1e-6).bfloat16().reshape(B * N, C)


def test_dwconv7_accepts_fp32_and_rejects_a_shifted_tap():
    B, N, C = 3, 9, 256
    x = torch.stack([rnd(N, C, seed=b) * (1 + b) + 3 * b for b in range(B)])
    wt, wb, lw, lb = rnd(7, C, seed=4) * 0.4, rnd(C, seed=5), 1 + 0.1 * rnd(C, seed=6), 0.1 * rnd(C, seed=7)
    ref, b = dwconv7_ref_bound(x, wt, wb, lw, lb)
    loc = lambda r, c: f"(utt {r // N}, frame {r % N}) col {c}"
    assert assert_within(dwconv7_fp32(x, wt, wb, lw, lb), ref, b, loc, "dwconv7") <= 1
    with pytest.raises(AssertionError, match=r"\(utt \d, frame \d\)"):
        assert_within(dwconv7_fp32(x, wt, wb, lw, lb, shift_tap=6), ref, b, loc, "shifted tap")


# ---------------------------------------------------------------- GRN
def grn_fp32(h, gamma, beta, nv):
    hf = h.float()
    keep = (torch.arange(h.shape[1])[None, :] < nv[:, None]).float()[..., None]
    gx = (hf * hf * keep).sum(1, keepdim=True).sqrt()
    nx = gx / (gx.mean(-1, keepdim=True) + 1e-6)
    return (gamma * (hf * nx) + beta + hf).bfloat16().reshape(-1, h.shape[2])


def test_grn_accepts_fp32_and_rejects_rows_beyond_valid_len():
    B, N, C = 3, 33, 256
    h = (rnd(B, N, C) * 2).bfloat16()
    vl = torch.tensor([33, 28, 16], dtype=torch.int32)
    for b in range(B):
        h[b, int(vl[b]):] = 200.0
    gamma, beta = 0.5 * rnd(C, seed=1), 0.5 * rnd(C, seed=2)
    ref, bd = grn_ref_bound(h, gamma, beta, vl)
    loc = lambda r, c: f"(utt {r // N}, frame {r % N}) col {c}"
    assert assert_within(grn_fp32(h, gamma, beta, vl), ref, bd, loc, "grn") <= 1
    with pytest.raises(AssertionError, match=r"\(utt [12], frame"):
        assert_within(grn_fp32(h, gamma, beta, torch.full((B,), N)), ref, bd, loc, "grn all rows")


# ---------------------------------------------------------------- duration head
def test_duration_head_accepts_fp32():
    B, N, D = 4, 50, 256
    x = rnd(B, N, D) * 1.5 + 0.2
    lens = torch.tensor([0, 1, 50, 70])
    nw, pw = 1 + 0.2 * rnd(D, seed=1), 0.5 * rnd(D, seed=2)
    xr = x * torch.rsqrt((x * x).mean(-1, keepdim=True) + 1e-5)
    keep = (torch.arange(N)[None] < lens.clamp(max=N)[:, None]).float()[..., None]
    t = ((xr * keep).sum(1) / lens.clamp(1, N)[:, None] * nw * pw).sum(-1)
    ref, b, _ = duration_ref_bound(x, lens, nw, pw)
    assert assert_within(torch.nn.functional.softplus(t)[:, None], ref[:, None], b[:, None], rows("utt"), "dur") <= 1


# ---------------------------------------------------------------- ODE update
def test_rk4_accepts_fp32_and_rejects_a_wrong_stage_weight():
    R, d, cfg, dt = 64, 100, 2.0, 0.0421
    y0 = rnd(R, d)
    vs = [rnd(2 * R, d, seed=10 + s) for s in range(4)]
    ks = [ode_k(v, R, d, R, cfg) for v in vs]

    def chain(ws):
        acc = torch.zeros(R, d)
        for s in range(4):
            k = vs[s][:R] + (vs[s][:R] - vs[s][R:]) * cfg
            acc = acc + ws[s] * k
        return y0 + torch.tensor(dt, dtype=torch.float32) / 6 * acc

    acc = torch.zeros(R, d, dtype=torch.float64)
    bacc = torch.zeros_like(acc)
    for s, w in enumerate([1.0, 2.0, 2.0, 1.0]):
        acc = acc + w * ks[s][0]
        bacc = bacc + w * ks[s][1] + U * w * ks[s][0].abs() + U * acc.abs()
    ref = y0.double() + dt / 6 * acc
    b = ode_axpy_bound(y0, dt / 6, acc, bacc) + 2 * U * abs(dt / 6) * acc.abs()
    assert assert_within(chain([1.0, 2.0, 2.0, 1.0]), ref, b, rows(), "rk4") <= 1
    with pytest.raises(AssertionError, match="rk4 w=1"):
        assert_within(chain([1.0, 1.0, 2.0, 1.0]), ref, b, rows(), "rk4 w=1")


# ---------------------------------------------------------------- text embedding
def test_text_embed_exact_check_names_an_unmasked_row():
    from test_gpu_hbm_kernels import _text_ref
    B, N, nt, C = 1, 20, 30, 8
    text = torch.randint(0, 50, (B, nt), generator=torch.Generator().manual_seed(0), dtype=torch.int32)
    emb, pos = rnd(51, C), rnd(64, C, seed=1)
    vl = torch.tensor([12])
    want = _text_ref(text, B, nt, N, emb, pos, 64, 1, 1, 1, vl)
    assert (want[12:] == 0).all() and (want[:12] != 0).any()
    got = _text_ref(text, B, nt, N, emb, pos, 64, 1, 1, 1, None)     # forgets the rows beyond valid_len
    with pytest.raises(AssertionError, match=r"frame 12\) col 0"):
        assert_exact(got, want, lambda r, c: f"(utt {r // N}, frame {r % N}) col {c}", "text")


# ---------------------------------------------------------------- mel / iSTFT
def mel_fp32(audio, window, filt_t, hop, frames, nyquist_sign=1.0):
    """The mel kernel's steps in fp32: frames, z = x_even + i x_odd, 512-point FFT, split step, |.|, filterbank, log."""
    B, T = audio.shape
    idx = torch.arange(frames)[:, None] * hop - 512 + torch.arange(1024)
    ok = (idx >= 0) & (idx < T)
    fr = (torch.where(ok, audio[:, idx.clamp(0, T - 1)], torch.zeros(())) * window).reshape(B * frames, 1024)
    Z = torch.fft.fft(torch.complex(fr[:, 0::2], fr[:, 1::2]), dim=-1)
    k = torch.arange(513)
    zk, zc = Z[:, k % 512], Z[:, (512 - k) % 512].conj()
    W = torch.polar(torch.ones(513), -2 * math.pi * k.float() / 1024)
    sgn = torch.ones(513)
    sgn[512] = nyquist_sign
    X = (zk + zc) / 2 - sgn * 1j * W * (zk - zc) / 2
    return torch.log((X.abs() @ filt_t).clamp(min=1e-5))


def test_mel_accepts_fp32_and_rejects_a_sign_flip_on_bin_512():
    T, hop = 2048, 256
    n = torch.arange(T, dtype=torch.float64)
    audio = torch.stack([0.3 + 0.2 * (-1.0) ** n + 0.1 * rnd(T).double(), 0.5 - 0.1 * (-1.0) ** n]).float()
    w = torch.from_numpy(np.hanning(1025)[:-1].astype(np.float32))
    eye = torch.eye(513)
    ref, b = mel_ref_bound(audio, w, eye, hop, T // hop)
    loc = lambda r, c: f"frame {r} bin {c}"
    assert assert_within(mel_fp32(audio, w, eye, hop, T // hop), ref, b, loc, "mel") <= 1
    with pytest.raises(AssertionError, match="bin 512"):
        assert_within(mel_fp32(audio, w, eye, hop, T // hop, nyquist_sign=-1.0), ref, b, loc, "mel")


def test_istft_accepts_fp32_and_rejects_a_dropped_frame():
    B, F, hop = 2, 5, 256
    g = torch.Generator().manual_seed(3)
    h = torch.cat([torch.rand(B * F, 513, generator=g) * 9 - 3, torch.rand(B * F, 513, generator=g) * 8 - 4], 1)
    w = torch.from_numpy(np.hanning(1025)[:-1].astype(np.float32))
    S = torch.polar(torch.exp(h[:, :513]).clamp(max=100), h[:, 513:])
    frames = (torch.fft.irfft(S, 1024, dim=-1) * w).reshape(B, F, 1024)
    out_len = (F - 1) * hop + 1024

    def ola(skip=None):
        acc, env = torch.zeros(B, out_len), torch.zeros(out_len)
        for f in range(F):
            if f != skip:
                acc[:, f * hop:f * hop + 1024] += frames[:, f]
            env[f * hop:f * hop + 1024] += w
        return torch.where(env > 1e-11, acc / torch.where(env > 1e-11, env, torch.ones(())), acc)

    fr, bf = istft_frames_ref_bound(h, w)
    ref, b = istft_ola_ref_bound(fr, bf, w, B, F, hop, False, 0, out_len)
    loc = lambda r, c: f"(batch {r}) sample {c}"
    assert assert_within(ola(), ref, b, loc, "istft") <= 1
    with pytest.raises(AssertionError, match=r"sample (7[6-9]\d|8\d\d|9\d\d|1[0-7]\d\d)\b"):
        assert_within(ola(skip=3), ref, b, loc, "istft dropped frame 3")


# ---------------------------------------------------------------- fft16 from its source
def _fft16_from_source():
    src = (CSRC / "fft.cuh").read_text()
    body = src[src.index("void fft16("):src.index("void fft512_warp(")]
    table = lambda name: [float(v.rstrip("f")) for v in
                          re.search(rf"constexpr float {name}\[8\] = \{{([^}}]*)\}}", body).group(1).replace("\n", " ")
                          .replace(" ", "").split(",")]
    Ct, St = table("C"), table("S")
    swaps = [(int(a), int(b)) for a, b in re.findall(r"t = a\[(\d+)\]; a\[\1\] = a\[(\d+)\];", body)]
    return np.array(Ct, np.float32), np.array(St, np.float32), swaps


def fft16_np(a, Ct, St, swaps):
    """fft16 exactly as written: radix-2 DIF with the C / S tables, then the listed swaps."""
    a = a.astype(np.complex128).copy()
    half = 8
    while half >= 1:
        for blk in range(0, 16, 2 * half):
            for j in range(half):
                p, q = blk + j, blk + j + half
                u, v = a[p], a[q]
                a[p] = u + v
                d = u - v
                tw = j * (8 // half)
                a[q] = complex(d.real * Ct[tw] - d.imag * St[tw], d.real * St[tw] + d.imag * Ct[tw])
        half //= 2
    for p, q in swaps:
        a[p], a[q] = a[q], a[p]
    return a


def test_fft16_constants_and_swaps_compute_the_dft():
    Ct, St, swaps = _fft16_from_source()
    assert len(swaps) == 6
    assert np.allclose(Ct + 1j * St, np.exp(-2j * np.pi * np.arange(8) / 16), atol=1e-7)
    rng = np.random.default_rng(0)
    for _ in range(20):
        a = rng.standard_normal(16) + 1j * rng.standard_normal(16)
        assert np.abs(fft16_np(a, Ct, St, swaps) - np.fft.fft(a)).max() < 1e-5 * np.abs(a).sum()
    for k in range(16):     # every basis vector: no bin is silently swapped with another
        e = np.zeros(16, complex)
        e[k] = 1
        assert np.abs(fft16_np(e, Ct, St, swaps) - np.fft.fft(e)).max() < 1e-6


# ---------------------------------------------------------------- coverage
def _cases(src, func):
    body = src[src.index(func):]
    body = body[:body.index("\n}\n")]
    return [int(v) for v in re.findall(r"case (\d+):", body)] + [int(v) for v in re.findall(r"F5_LN_CASE\((\d+)\)", body)]


def test_every_hbm_and_audio_kernel_has_a_gpu_test():
    import test_gpu_audio_kernels as ta
    import test_gpu_hbm_kernels as th
    covered = th.COVERED | ta.COVERED
    names = {c.split("<")[0] for c in covered}
    for f in ("elementwise.cuh", "audio_vocos.cu"):
        for k in re.findall(r"__global__ void(?: __launch_bounds__\([^)]*\))?\s+(\w+)\(", (CSRC / f).read_text()):
            assert k in names, f"{f}: kernel {k} has no GPU test"
    cu = (CSRC / "elementwise.cu").read_text()
    ln = _cases(cu, "static int launch_ln_any(")
    assert len(ln) == 6
    for d in ln:
        for out in ("bf16", "f32"):
            assert f"ln_mod_kernel<{d},{out}>" in covered, (d, out)
    for func, kern in (("int launch_dwconv7_ln(", "dwconv7_ln_kernel"), ("int launch_duration_head(",
                                                                      "duration_head_kernel")):
        cases = _cases(cu, func)
        assert cases
        for c in cases:
            assert f"{kern}<{c}>" in covered, (kern, c)
