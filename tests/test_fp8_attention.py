"""CPU: the FP8 attention mode (DiT(fp8=True, fp8_scaling="block", fp8_attention=True), DESIGN.md sections 5 and 8) —
its kernels compile cleanly, the host's V^T key order, the emulated drift of the mode, and the refusals of the Python
surface and the CLI outside the block-scaled mode."""
import re
import subprocess
from pathlib import Path

import pytest
import torch

from f5_tts_mlx_b200.weights import GATE_CONFIG, fp8_vt_key_order, random_dit_weights

ROOT = Path(__file__).resolve().parent.parent


def test_fp8_attention_kernels_compile_without_spills(tmp_path):
    """Both new kernels compile for sm_90a with the build's own flags to 0 spill bytes and without wgmma
    serialisation (warning C7510)."""
    from f5_tts_mlx_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-cubin", str(ROOT / "f5_tts_mlx_b200" / "csrc" / "attention_fp8.cu"), "-o",
           str(tmp_path / "k.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    assert "C7510" not in log and "serialized" not in log
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'(.*?)Used \d+ registers", log, re.S):
        found[m[1]] = sum(int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", m[2]))
    assert {n for n in found if "attn_fp8_kernel" in n or "qkv_quant_e4m3_kernel" in n} == set(found), sorted(found)
    assert len(found) == 2 and all(v == 0 for v in found.values()), found


def test_vt_key_order_is_the_fragment_mapping(tmp_path):
    """Position 4l + i of each 32-key group holds key (2l, 2l+1, 2l+8, 2l+9)[i] and position 16 + 4l + i holds 16 plus
    that key: the keys the S accumulator fragment of lane l holds, in the k order of the e4m3 register A fragment.  The
    kernels' own fp8_vt_key / fp8_vt_pos (attention_fp8_sm90.cuh, compiled into a host program here) give the host's
    order and its inverse."""
    order = fp8_vt_key_order()
    assert sorted(order.tolist()) == list(range(32))
    for l in range(4):
        for i in range(4):
            key = (2 * l, 2 * l + 1, 2 * l + 8, 2 * l + 9)[i]
            assert order[4 * l + i] == key and order[16 + 4 * l + i] == 16 + key
    from f5_tts_mlx_b200 import build
    src = tmp_path / "order.cu"
    src.write_text('#include <cstdio>\n#include "attention_fp8_sm90.cuh"\n'
                   'int main() { for (int p = 0; p < 32; ++p) printf("%d %d\\n", f5::fp8_vt_key(p), '
                   'f5::fp8_vt_pos(p)); return 0; }\n')
    exe = tmp_path / "order"
    r = subprocess.run([build._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-I", str(ROOT / "f5_tts_mlx_b200" / "csrc"), str(src), "-o",
                        str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    key, pos = zip(*[map(int, line.split()) for line in out if line])
    assert list(key) == order.tolist()
    assert [key[p] for p in pos] == list(range(32))           # fp8_vt_pos is the inverse of fp8_vt_key


def test_emulated_drift_fp8_attention():
    """The emulation of the FP8 attention mode, rel-L2 from fp32 on the gate model (N = 300), printed beside the block
    mode's, on the seeded random weights and the outlier construction: finite and below 5e-2."""
    from oracle import f5_oracle as O
    from helpers import ocfg_of, rel
    import fp8_attn_emul as A
    import fp8_block_emul as E
    cfg = GATE_CONFIG
    W = random_dit_weights(cfg, seed=1234)
    oc = ocfg_of(cfg)
    N = 300
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, N, 100, generator=g); cond = torch.randn(1, N, 100, generator=g) * 2 - 1
    text = torch.randint(0, 2545, (1, 60), generator=g, dtype=torch.int32)
    t = torch.tensor(0.25)
    d = {}
    for name, (xx, cc) in (("random", (x, cond)), ("outlier", E.outlier_inputs(1, N))):
        ref = O.dit_forward(xx, cc, text, t, False, False, None, W, oc)
        d[name, "block"] = rel(E.dit_forward_block8(xx, cc, text, t, False, False, None, W, oc), ref)
        d[name, "block_attn"] = rel(A.dit_forward_block8a(xx, cc, text, t, False, False, None, W, oc), ref)
    print({k: f"{v:.3e}" for k, v in d.items()})
    for name in ("random", "outlier"):
        assert 0 < d[name, "block_attn"] < 5e-2, d


def test_emulated_attention_matches_float64_on_exact_operands():
    """The emulation's attention on operands that e4m3 represents exactly: it equals the float64 softmax up to the
    rounding of P~ = e4m3(2^8 p)."""
    import fp8_attn_emul as A
    g = torch.Generator().manual_seed(0)
    q = torch.zeros(1, 2, 300, 64); q[..., 0] = 1.0
    k = torch.zeros(1, 2, 300, 64); k[..., 0] = torch.randint(0, 4, (1, 2, 300), generator=g).float()
    v = torch.randint(-3, 4, (1, 2, 300, 64), generator=g).float()
    mask = torch.arange(300)[None] < 211
    got = A.attention_fp8(q, k, v, mask).double()
    s = (q.double() @ k.double().transpose(-1, -2)).masked_fill(~mask[:, None, None, :], float("-inf"))
    want = torch.softmax(s, -1) @ v.double()
    # P~ rounds p relative 2^-4 (plus the subnormal floor): the only rounding left
    assert ((got - want).abs() <= 2.0 ** -4 * (torch.softmax(s, -1) @ v.double().abs()) + 1e-3).all()


def test_emulated_tile_scales_ignore_masked_keys():
    """q_tiles with a mask: keys beyond kv_len (here +-3e4, 2^15 times the valid ones) neither set their tile's scale
    nor carry a code, so the valid keys quantise as if those keys were zero, and attention_fp8 keeps its bits."""
    import fp8_attn_emul as A
    g = torch.Generator().manual_seed(1)
    B, H, N = 2, 2, 300
    lens = torch.tensor([300, 201])
    mask = torch.arange(N)[None] < lens[:, None]
    q, k, v = [torch.randn(B, H, N, 64, generator=g).bfloat16().float() for _ in range(3)]
    poison = 3e4 * (torch.randint(0, 2, (B, H, N, 64), generator=g) * 2 - 1).float()
    k2 = torch.where(mask[:, None, :, None], k, poison)
    v2 = torch.where(mask[:, None, :, None], v, -poison)
    zero = lambda t: torch.where(mask[:, None, :, None], t, torch.zeros(()))
    for a, b in ((k, k2), (v, v2)):
        c1, s1 = A.q_tiles(zero(a))
        c2, s2 = A.q_tiles(b, mask)
        assert torch.equal(c1, c2) and torch.equal(s1, s2)
        assert not torch.equal(A.q_tiles(b)[1], s2)                 # without the mask the poison sets the scales
    assert torch.equal(A.attention_fp8(q, k, v, mask), A.attention_fp8(q, k2, v2, mask))


def test_fp8_attention_needs_the_block_mode():
    from f5_tts_mlx_b200 import DiT
    kw = dict(dim=256, depth=1, heads=4, text_dim=64, device="cpu")
    for bad in (dict(), dict(fp8=True), dict(fp8=True, fp8_scaling="tensor")):
        with pytest.raises(ValueError, match="fp8_attention"):
            DiT(fp8_attention=True, **kw, **bad)
    assert DiT(fp8=True, fp8_scaling="block", fp8_attention=True, **kw).fp8_attention
    assert not DiT(fp8=True, fp8_scaling="block", **kw).fp8_attention


def test_cli_refuses_fp8_attention_without_block():
    from f5_tts_mlx_b200.generate import generate, main
    for argv in (["--text", "hi", "--fp8-attention"], ["--text", "hi", "--fp8", "tensor", "--fp8-attention"]):
        with pytest.raises(SystemExit) as e:
            main(argv)
        assert e.value.code == 2
    with pytest.raises(ValueError, match="fp8_attention"):
        generate("hi", fp8="tensor", fp8_attention=True)
