"""CPU: the block-scaled FP8 mode (DESIGN.md section 8) — the power-of-two scale rule, the block-scaled pack, the
coverage of dispatch_scaled (gemm.cu) by the GPU cases, and the emulated drift of the mode against per-tensor FP8."""
import hashlib
import re
from pathlib import Path

import pytest
import torch

from f5_tts_mlx_b200.weights import DiTConfig, PackedDiT, e4m3_block_scale, quantize_e4m3_blocks, random_dit_weights

ROOT = Path(__file__).resolve().parent.parent
SMALL = DiTConfig(dim=256, depth=2, heads=4, text_dim=64, conv_layers=1, text_num_embeds=50)


# ---------------------------------------------------------------- the scale rule
@pytest.mark.parametrize("amax,want", [(448.0, 1.0), (448.00003, 2.0), (224.0, 0.5), (256.0, 1.0), (1.0, 2.0 ** -8),
                                       (1.75, 2.0 ** -8), (1.7500001, 2.0 ** -7), (896.0, 2.0), (0.0, 1.0),
                                       (3e38, 2.0 ** 120), (1e-40, 2.0 ** -126), (2.0 ** -120, 2.0 ** -126)])
def test_scale_rule_known_answers(amax, want):
    assert e4m3_block_scale(torch.tensor([amax])).item() == want


def test_scale_rule_is_the_smallest_power_of_two_that_fits():
    g = torch.Generator().manual_seed(0)
    amax = torch.exp2(torch.rand(20000, generator=g) * 200 - 100)
    amax = torch.cat([amax, 448.0 * torch.exp2(torch.arange(-100, 100).float())])     # exactly on the boundaries
    s = e4m3_block_scale(amax)
    m, e = torch.frexp(s)
    assert (m == 0.5).all()                                          # powers of two
    assert (amax <= 448.0 * s).all() and ((amax > 224.0 * s) | (s == 2.0 ** -126)).all()
    on = amax[-200:]
    assert torch.equal(e4m3_block_scale(on), on / 448.0)             # amax = 448 * 2^j -> 2^j


def test_scale_rule_non_finite_stays_non_finite():
    s = e4m3_block_scale(torch.tensor([float("inf"), float("nan")]))
    assert torch.isinf(s[0]) and torch.isnan(s[1])
    x = torch.tensor([[1.0, float("inf")] + [0.0] * 62])
    q, sc = quantize_e4m3_blocks(x)
    assert not torch.isfinite(q.view(torch.float8_e4m3fn).float() * sc).all()


# ---------------------------------------------------------------- the pack
def test_block_pack_round_trips_within_half_an_e4m3_ulp():
    W = random_dit_weights(SMALL, seed=5)
    p = PackedDiT(SMALL, "cpu", fp8=True, fp8_scaling="block").load(W)
    pre = "transformer.transformer_blocks.1."
    w = {"qkv": torch.cat([W[pre + f"attn.to_{n}.weight"] for n in "qkv"], 0), "out": W[pre + "attn.to_out.layers.0.weight"],
         "ff1": W[pre + "ff.ff.layers.0.layers.0.weight"], "ff2": W[pre + "ff.ff.layers.2.weight"]}
    for n, wf in w.items():
        q = p.view(f"blk1.{n}_w8c").view(torch.float8_e4m3fn).float()
        s = p.view(f"blk1.{n}_s8c")
        assert torch.equal(torch.frexp(s)[0], torch.full_like(s, 0.5))
        deq = q * s[:, None]
        # half an ulp: 2^-4 relative for normal codes, 2^-10 s absolute (half the subnormal spacing) below 2^-6 s
        bound = torch.maximum(2.0 ** -4 * wf.abs(), 2.0 ** -10 * s[:, None])
        assert ((deq - wf).abs() <= bound).all(), n
        assert ((q.abs().amax(1) >= 224) & (q.abs().amax(1) <= 448)).all()
    c = p.c_struct()
    assert c.blocks[1].qkv_ws == p.buffer.data_ptr() + p.specs["blk1.qkv_s8c"].offset and c.blocks[0].ff2_s8 == 1.0


def test_tensor_mode_pack_is_unchanged():
    """The per-tensor FP8 pack of a small seeded model: the SHA-256 of its bytes as the previous release packed them."""
    W = random_dit_weights(SMALL, seed=5)
    p = PackedDiT(SMALL, "cpu", fp8=True).load(W)
    assert p.nbytes == 8884992
    assert hashlib.sha256(p.buffer.numpy().tobytes()).hexdigest() == \
        "3c3671cd401d2c3143b3cabaacfbaa4f312c393a1bfa1392d6c632792c88c5a2"
    assert PackedDiT(SMALL, "cpu", fp8=True, fp8_scaling="tensor").specs.keys() == p.specs.keys()
    with pytest.raises(ValueError):
        PackedDiT(SMALL, "cpu", fp8=True, fp8_scaling="channel")


# ---------------------------------------------------------------- coverage of dispatch_scaled
_ACT = {"ACT_NONE": 0, "ACT_GELU_TANH": 1, "ACT_GELU_ERF": 2, "ACT_MISH": 3}
_B = {"true": True, "false": False}


def built_scaled_instantiations():
    """(ACT, OUT_BF16, ROPE, FP8, RESID) of every launch_gemm instantiation dispatch_scaled (gemm.cu) can reach."""
    src = (ROOT / "f5_tts_mlx_b200" / "csrc" / "gemm.cu").read_text()
    body = src[src.index("static int dispatch_scaled"):]
    body = body[:body.index("\n}\n")]
    out = set()
    pat = r"launch_gemm<BN, kStages, (ACT_\w+), (true|false), (true|false), (true|false), (true|false), (true|false)>"
    for m in re.finditer(pat, body):
        assert m[6] == "true"                     # every instantiation of the block-scaled dispatcher is SCALED
        out.add((_ACT[m[1]], _B[m[2]], _B[m[3]], _B[m[4]], _B[m[5]]))
    return out


def test_scaled_dispatch_parse_and_gpu_coverage():
    import test_gpu_fp8_block as t
    built = built_scaled_instantiations()
    assert built == {(0, True, True, True, False), (0, False, False, True, True), (1, True, False, True, False),
                     (3, False, False, True, True)}, sorted(built)
    declared = set(t.INSTANTIATIONS)
    assert {d[:5] for d in declared} <= built, sorted({d[:5] for d in declared} - built)
    missing = sorted((i, bn) for i in built for bn in (64, 128) if i + (bn,) not in declared)
    assert not missing, f"block-scaled instantiations without a GPU case: {missing}"


# ---------------------------------------------------------------- compilation
@pytest.mark.parametrize("src", ["gemm.cu", "attention.cu"])
def test_block_scaled_instantiations_compile_without_spills(src, tmp_path):
    """Every block-scaled instantiation (the GEMM's SCALED, the attention's kScaled) compiles for sm_90a with the build's
    own flags to 0 spill bytes and without wgmma serialisation (warning C7510)."""
    import subprocess
    from f5_tts_mlx_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-cubin", str(ROOT / "f5_tts_mlx_b200" / "csrc" / src), "-o",
           str(tmp_path / "k.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    assert "C7510" not in log and "serialized" not in log
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'(.*?)Used \d+ registers", log, re.S):
        name = m[1]
        # the last template argument of gemm_bf16_tn_kernel (SCALED) / attn_fwd_kernel (kScaled) is true
        if re.search(r"(gemm_bf16_tn_kernel|attn_fwd_kernel)I.*Lb1EEEv", name) and \
                re.search(r"Lb[01]EEEv", name).group(0) == "Lb1EEEv":
            spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", m[2])]
            found[name] = sum(spills)
    want = 8 if src == "gemm.cu" else 1
    assert len(found) == want, sorted(found)
    assert all(v == 0 for v in found.values()), {k: v for k, v in found.items() if v}


# ---------------------------------------------------------------- emulated drift
def test_emulated_drift_block_vs_tensor():
    """The oracle's emulation of each FP8 mode, rel-L2 from fp32 (gate model, N = 300): on the seeded random weights the
    two modes drift alike (DESIGN.md section 8); with residual rows far beyond 448 the per-tensor mode saturates and
    drifts more than twice as far, while the block mode stays at its random-weight figure."""
    from oracle import f5_oracle as O
    from helpers import ocfg_of, rel
    import fp8_block_emul as E
    from f5_tts_mlx_b200.weights import GATE_CONFIG
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
        d[name, "tensor"] = rel(O.dit_forward(xx, cc, text, t, False, False, None, W, oc, O.Precision(True, True, True)), ref)
        d[name, "block"] = rel(E.dit_forward_block8(xx, cc, text, t, False, False, None, W, oc), ref)
    # recorded, not asserted: a few 40x outlier weight channels (DESIGN.md section 8) do not separate the modes
    Wo = E.outlier_weights(W, cfg)
    ref = O.dit_forward(x, cond, text, t, False, False, None, Wo, oc)
    d["channels", "tensor"] = rel(O.dit_forward(x, cond, text, t, False, False, None, Wo, oc, O.Precision(True, True, True)), ref)
    d["channels", "block"] = rel(E.dit_forward_block8(x, cond, text, t, False, False, None, Wo, oc), ref)
    print({k: f"{v:.3e}" for k, v in d.items()})
    assert 2e-3 < d["random", "block"] < 2e-2 and d["random", "block"] < 1.5 * d["random", "tensor"]
    assert d["outlier", "tensor"] > 2 * d["outlier", "block"]
    assert d["outlier", "block"] < 1.5 * d["random", "block"]
