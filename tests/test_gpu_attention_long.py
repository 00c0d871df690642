"""-m gpu: both attention kernels at 60 s lengths and beyond (N up to max_duration = 8192, B = 2, H = 16, ragged kv_len).

  * position codes: exact answers in every key tile through the four attention entry points;
  * the online softmax tile by tile: every output code against tests/attn_online_emul.py."""
import pytest
import torch

import attn_online_emul as M
from kernel_check import Guarded, assert_exact, attn_tiles, round_to
from test_gpu_fp8_attention import run_attention
from test_gpu_kernel_exact import _attn_call, _qkv_buffer

pytestmark = pytest.mark.gpu
DEV = "cuda"
F8 = torch.float8_e4m3fn
B, H = 2, 16
D = H * 64


def run_bf16_kernel(qkv, N, kv, out):
    """The bf16-operand attention with a "bf16", "e4m3" or "e4m3_scaled" output, on a [B N, 3 D] view of a wider
    buffer: (output guard, scale guard or None)."""
    buf = _qkv_buffer(B, N, H)
    buf.copy_(qkv)
    g = Guarded(B * N, D, torch.bfloat16 if out == "bf16" else torch.uint8, DEV)
    so = Guarded(H, B * N, torch.float32, DEV, lr=False) if out == "e4m3_scaled" else None
    _attn_call(buf, g.view, B, N, H, kv, fp8=out != "bf16", scale_out=so.view if so is not None else None)
    return g, so


# ---------------------------------------------------------------- position codes, exact
def hadamard64() -> torch.Tensor:
    h = torch.ones(1, 1)
    while h.shape[0] < 64:
        h = torch.cat([torch.cat([h, h], 1), torch.cat([h, -h], 1)], 0)
    return h


def hot_positions(L: int, g: torch.Generator) -> torch.Tensor:
    """128 distinct keys in [0, L): positions 0, 127, 128 and L - 1, one in every 128-key tile, every residue mod 32."""
    pos = {0, 127, 128, L - 1}
    for t in range((L + 127) // 128):
        lo, hi = 128 * t, min(L, 128 * t + 128)
        pos.add(lo + int(torch.randint(0, hi - lo, (1,), generator=g)))
    for r in range(32):
        if all(p % 32 != r for p in pos):
            pos.add(r + 32 * int(torch.randint(0, (L - 1 - r) // 32 + 1, (1,), generator=g)))
    while len(pos) < 128:
        pos.add(int(torch.randint(0, L, (1,), generator=g)))
    assert len(pos) == 128
    return torch.tensor(sorted(pos))


def position_coded_qkv(N: int, kv: torch.Tensor, seed: int):
    """Key codes: +-the rows of a 64 x 64 Hadamard matrix (code c < 64: row c, else -row c - 64); two distinct codes
    have dot product 0 or -64, a code with itself 64.  Per (utterance, head) 128 hot keys carry the 128 codes (placed
    by hot_positions, in a random order), every other valid key is zero, and key n >= kv_len carries twice code
    n % 128 (logit 128 for the queries of that code: a leak would dominate).  Query row i carries code
    (i + offset) % 128, so its output is V at the hot key of that code: every query tile reads every key tile.  V from
    {+-1, +-1.5, +-2, +-3}, exact in bf16 and e4m3 at any power-of-two scale."""
    g = torch.Generator().manual_seed(seed)
    hd = hadamard64()
    codes = torch.cat([hd, -hd], 0)                                 # [128, 64]
    vals = torch.tensor([1.0, -1.0, 1.5, -1.5, 2.0, -2.0, 3.0, -3.0])
    q = torch.zeros(B, N, H, 64)
    k = torch.zeros(B, N, H, 64)
    v = vals[torch.randint(0, 8, (B, N, H, 64), generator=g)]
    want = torch.empty(B, N, H, 64)
    for b in range(B):
        L = int(kv[b])
        k[b, L:] = 2 * codes[torch.arange(L, N) % 128][:, None]
        for h in range(H):
            pos = hot_positions(L, g)
            code_of = torch.randperm(128, generator=g)              # hot key pos[i] carries code code_of[i]
            k[b, pos, h] = codes[code_of]
            key_of = torch.empty(128, dtype=torch.long)
            key_of[code_of] = pos
            a = (torch.arange(N) + int(torch.randint(0, 128, (1,), generator=g))) % 128
            q[b, :, h] = codes[a]
            want[b, :, h] = v[b, key_of[a], h]
    qkv = torch.cat([t.reshape(B * N, D) for t in (q, k, v)], 1).bfloat16()
    return qkv, want.reshape(B * N, D)


@pytest.mark.parametrize("entry", ["bf16", "e4m3", "e4m3_scaled", "fp8"])
@pytest.mark.parametrize("N", [937, 5625, 6000, 8192])
def test_attention_position_codes_exact(N, entry):
    """Every output row is V at its query's hot key, exactly, through f5_attention_fwd, f5_attention_fwd_e4m3,
    f5_attention_fwd_e4m3_scaled and the quantise pass + f5_attention_fwd_fp8 (the other keys weigh below
    8192 e^-64); the second utterance's kv_len ends inside a key tile; guard bands untouched."""
    kv = torch.tensor([N, N - 1037 if N > 2000 else N - 237], dtype=torch.int32)
    qkv, want = position_coded_qkv(N, kv, seed=N)
    what = f"position codes N={N} {entry}"
    loc = attn_tiles(N)
    if entry == "fp8":
        deq, out, so = run_attention(qkv.to(DEV), B, N, H, kv.to(DEV))
        assert_exact(deq, want, loc, what)
        out.check(what + " out guard"); so.check(what + " scale guard")
        return
    g, so = run_bf16_kernel(qkv.to(DEV), N, kv.to(DEV), entry)
    if entry == "e4m3_scaled":
        deq = (g.view.cpu().view(F8).float().reshape(B * N, H, 64) * so.view.cpu().T[..., None]).reshape(B * N, D)
        assert_exact(deq, want, loc, what)
        so.check(what + " scale guard")
    else:
        assert_exact(g.view.cpu(), round_to(want.double(), torch.bfloat16 if entry == "bf16" else torch.uint8), loc, what)
    g.check(what + " out guard")


# ---------------------------------------------------------------- the online softmax, tile by tile
CASES = [(c, n) for n in (300, 937, 5625) for c in ("random", "rising", "falling")] + [("random", 8192), ("tail", 5625)]


def _heads(t: torch.Tensor, N: int) -> torch.Tensor:
    """[B N, H, ...] -> [B, H, N, ...]"""
    return t.reshape(B, N, H, *t.shape[2:]).transpose(1, 2)


@pytest.mark.parametrize("kind", ["bf16", "fp8"])
@pytest.mark.parametrize("case,N", CASES, ids=[f"{c}-{n}" for c, n in CASES])
def test_attention_online_softmax_emulated(case, N, kind):
    """Integer-valued q and k (exact logits), ragged kv_len: every output code of the bf16 kernel (bf16 output) and of
    the FP8 kernel (block-scaled e4m3 output, with its scales) is one that the tile-by-tile emulation's O within beta
    rounds to.  The long tail also prints its drift from the float64 softmax and stays within fp8_attention_bound."""
    qkv = M.make_qkv(case, B, N, H, seed=N + len(case))
    kv = torch.tensor([N, M.KV_LEN[N]], dtype=torch.int32)
    ops = M.operands(qkv, B, N, H, kind, kv)
    M.assert_exact_logits(ops[0], ops[2], kind)
    O, beta = M.online_softmax(*[t.to(DEV) for t in ops], kv.to(DEV), kind)
    what = f"online softmax {kind} {case} N={N}"
    if kind == "bf16":
        g, _ = run_bf16_kernel(qkv.to(DEV), N, kv.to(DEV), "bf16")
        g.check(what + " guard")
        M.check_output(_heads(g.view.cpu().reshape(B * N, H, 64), N), O, beta, "bf16", what=what)
        return
    deq, out, so = run_attention(qkv.to(DEV), B, N, H, kv.to(DEV))
    out.check(what + " out guard"); so.check(what + " scale guard")
    codes = _heads(out.view.cpu().view(F8).double().reshape(B * N, H, 64), N)
    scale = _heads(so.view.cpu().T, N)
    M.check_output(codes, O, beta, "e4m3_scaled", scale, what=what)
    if case == "tail":
        from kernel_check import E4M3_SUB, U_E4M3, assert_within
        from test_gpu_fp8_attention import fp8_attention_bound
        qc, sq, kc, sk, vc, sv = ops
        rep = lambda s: s.repeat_interleave(M.TILE, -1)[..., :N, None]
        q, k, v = qc * sq[..., None], kc * rep(sk), vc * rep(sv)
        flat = lambda t: t.permute(0, 2, 1, 3).reshape(B * N, D)
        ref, bd = [], []
        for h in range(0, H, 2):
            o, b = fp8_attention_bound(q[:, h:h + 2], k[:, h:h + 2], v[:, h:h + 2], kv)
            ref.append(o.cpu()); bd.append(b.cpu())
        ref, bd = flat(torch.cat(ref, 1)), flat(torch.cat(bd, 1))
        bound = bd + U_E4M3 * (ref.abs() + bd) + E4M3_SUB * so.view.cpu().T.repeat_interleave(64, 1).double()
        rel = ((deq.double() - ref).norm() / ref.norm()).item()
        tail_lost = ((flat(O.cpu()) - ref).norm() / ref.norm()).item()
        print(f"{what}: drift from float64 {rel:.3e} (emulated O before output rounding: {tail_lost:.3e})")
        assert_within(deq, ref, bound, attn_tiles(N), what + " vs float64")
