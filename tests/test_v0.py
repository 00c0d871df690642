"""F5TTS_Base (v0) checkpoints on the CPU: the unmasked-text oracle path against the reference's own code, the test-side
v0 restatement (tests/v0_emul.py) against an independent statement of upstream's first-head rotation, the C ABI's
version fields, and from_pretrained(model_version=...)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import f5_oracle as O
from helpers import rel
import v0_emul as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 2e-6


def T(a):
    return torch.from_numpy(np.asarray(a))


@pytest.fixture(scope="module")
def gate_w():
    from f5_tts_mlx_b200.weights import GATE_CONFIG, random_dit_weights
    return GATE_CONFIG, random_dit_weights(GATE_CONFIG, seed=1234)


# ---------------------------------------------------------------- unmasked text: pinned to the reference
def test_oracle_unmasked_text_forward_matches_reference_code(gate_w, golden_dir):
    """DiT(text_mask_padding=False) of the unmodified reference (tests/golden/make_ref_golden_v0.py): the oracle's
    mask_padding=False text embedding, composed into a forward, for drop_text False and True."""
    cfg, W = gate_w
    z = np.load(os.path.join(golden_dir, "ref_dit_v0.npz"))
    x, cond, text, t = T(z["x"]), T(z["cond"]), T(z["text"]), T(z["t"])
    ocfg = V.ocfg_v0(cfg)
    for name, (dac, dt) in {"out": (False, False), "out_drop_text": (False, True), "out_drop": (True, True)}.items():
        assert rel(V.dit_forward(x, cond, text, t, dac, dt, None, W, ocfg), T(z[name])) < TOL, name
    # the filler rows matter: the masked (v1) text embedding gives a different answer on the same inputs
    assert rel(O.dit_forward(x, cond, text, t, False, False, None, W, ocfg), T(z["out"])) > 1e-3


def test_oracle_unmasked_text_sample_matches_reference_code(gate_w, golden_dir):
    cfg, W = gate_w
    z = np.load(os.path.join(golden_dir, "ref_dit_v0.npz"))
    out, traj = V.sample(T(z["scond"]), T(z["stext"]), int(z["duration"]), W, V.ocfg_v0(cfg), steps=4, method="euler",
                         cfg_strength=2.0, sway_sampling_coef=-1.0, seed=7)
    assert out.shape == z["sample_out"].shape and traj.shape == z["sample_traj"].shape
    assert rel(out, T(z["sample_out"])) < TOL and rel(traj, T(z["sample_traj"])) < TOL


# ---------------------------------------------------------------- first-head rotation: the restatement
@pytest.mark.parametrize("masked", [False, True])
def test_per_head_table_is_upstream_v0_rotation(gate_w, masked):
    """The oracle's attention with the per-head angle table (zero past pe_attn_head = 1) equals upstream v0's attention,
    which rotates columns [0, 64) of the un-split q and k projections."""
    cfg, W = gate_w
    g = torch.Generator().manual_seed(5)
    B, N = 2, 70
    x = torch.randn(B, N, cfg.dim, generator=g)
    mask = (torch.arange(N)[None] < torch.tensor([N, 41])[:, None]) if masked else None
    pfx = "transformer.transformer_blocks.1.attn."
    got = O.attention(x, mask, V.head_rope(N, cfg.heads, 1), W, pfx, cfg.heads)
    want = V.upstream_v0_attention(x, mask, W, pfx, cfg.heads)
    assert rel(got, want) < 1e-5
    # and it is not the all-heads rotation
    assert rel(O.attention(x, mask, O.rotary_freqs(N, 64), W, pfx, cfg.heads), want) > 1e-3


def test_per_head_table_all_heads_is_the_oracle_bitwise(gate_w):
    """pe_attn_head=None composes the oracle's own forward exactly (the table is the oracle's, repeated per head)."""
    cfg, W = gate_w
    g = torch.Generator().manual_seed(6)
    N = 60
    x = torch.randn(1, N, 100, generator=g); cond = torch.randn(1, N, 100, generator=g)
    text = torch.randint(0, 2545, (1, 20), generator=g, dtype=torch.int32)
    t = torch.tensor(0.3)
    got = V.dit_forward(x, cond, text, t, False, False, None, W, V.ocfg_v0(cfg, text_mask_padding=True))
    assert torch.equal(got, O.dit_forward(x, cond, text, t, False, False, None, W, V.ocfg_v0(cfg, True)))


# ---------------------------------------------------------------- C ABI 2.004
def _dims(cfg, *extra):
    from f5_tts_mlx_b200 import _lib
    return _lib.DitDims(cfg.dim, cfg.depth, cfg.heads, cfg.ff_inner, cfg.mel_dim, cfg.text_dim, cfg.conv_layers,
                        cfg.text_num_embeds, *extra)


def _bind(cfg, d):
    from f5_tts_mlx_b200 import _lib
    from f5_tts_mlx_b200.weights import ConvNextWeightsC, DitBlockWeightsC, DitWeightsC
    w = DitWeightsC(); tbs = (ConvNextWeightsC * cfg.conv_layers)(); blks = (DitBlockWeightsC * cfg.depth)()
    rc = _lib.load().f5_bind_packed_weights(C.byref(d), C.c_void_p(1 << 20), C.byref(w), tbs, blks)
    return rc, w


def test_abi_version_and_mirrors():
    from f5_tts_mlx_b200 import _lib
    from f5_tts_mlx_b200.weights import DitWeightsC
    lib = _lib.load()
    assert lib.f5_abi_version() >= 2004
    out = (C.c_int32 * 10)()
    lib.f5_struct_sizes(out, 10)
    assert out[0] == C.sizeof(_lib.GemmArgs) and out[3] == C.sizeof(DitWeightsC)
    assert [n for n, _ in _lib.GemmArgs._fields_][-1] == "rope_col2"
    assert [n for n, _ in DitWeightsC._fields_][-2:] == ["text_unmasked", "rope_heads"]
    assert C.sizeof(_lib.DitDims) == 10 * 4


def test_c_sizeof_dit_dims_matches_mirror(tmp_path):
    """f5_dit_dims is not in f5_struct_sizes: compare its sizeof and the new fields' offsets with a C compiler."""
    from f5_tts_mlx_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "dims.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "f5_b200.h"\nint main(void) {\n'
                   '  printf("%d %d %d\\n", (int)sizeof(f5_dit_dims), (int)offsetof(f5_dit_dims, text_unmasked),\n'
                   '         (int)offsetof(f5_dit_dims, rope_heads));\n  return 0;\n}\n')
    exe = str(tmp_path / "dims")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    size, off_u, off_r = map(int, subprocess.run([exe], capture_output=True, text=True).stdout.split())
    assert (size, off_u, off_r) == (C.sizeof(_lib.DitDims), _lib.DitDims.text_unmasked.offset,
                                    _lib.DitDims.rope_heads.offset)


def test_bind_packed_weights_carries_the_version_fields():
    from f5_tts_mlx_b200.weights import DiTConfig
    cfg = DiTConfig(dim=256, depth=2, heads=4, text_num_embeds=40, text_dim=128, conv_layers=2)
    rc, w = _bind(cfg, _dims(cfg))                       # positional initialiser of the 8 v1 fields: the rest is zero
    assert rc == 0 and (w.text_unmasked, w.rope_heads) == (0, 0)
    for extra in ((1, 1), (1, 0), (0, 4)):
        rc, w = _bind(cfg, _dims(cfg, *extra))
        assert rc == 0 and (w.text_unmasked, w.rope_heads) == extra


@pytest.mark.parametrize("extra,msg", [((0, -1), b"rope_heads"), ((0, 5), b"rope_heads"), ((2, 0), b"text_unmasked")])
def test_bind_packed_weights_refuses_bad_version_fields(extra, msg):
    from f5_tts_mlx_b200 import _lib
    from f5_tts_mlx_b200.weights import DiTConfig
    cfg = DiTConfig(dim=256, depth=2, heads=4, text_num_embeds=40, text_dim=128, conv_layers=2)
    rc, _ = _bind(cfg, _dims(cfg, *extra))
    assert rc == -1 and msg in _lib.load().f5_last_error()
    assert _lib.load().f5_packed_weights_bytes(C.byref(_dims(cfg, *extra))) == -1


def test_python_weights_struct_carries_the_version_fields():
    from f5_tts_mlx_b200.weights import DiTConfig, PackedDiT
    base = dict(dim=256, depth=1, heads=4, text_num_embeds=10, text_dim=64, conv_layers=1)
    for kw, want in ((dict(), (0, 0)), (dict(text_mask_padding=False, pe_attn_head=1), (1, 1)),
                     (dict(pe_attn_head=4), (0, 4))):
        w = PackedDiT(DiTConfig(**base, **kw), "cpu").c_struct()
        assert (w.text_unmasked, w.rope_heads) == want


# ---------------------------------------------------------------- Python surface
def test_dit_constructor_validates_pe_attn_head():
    from f5_tts_mlx_b200 import DiT
    kw = dict(dim=512, depth=1, heads=8, ff_mult=2, text_dim=512, conv_layers=1, device="cpu")
    m = DiT(text_mask_padding=False, pe_attn_head=1, **kw)
    assert m.config.text_mask_padding is False and m.config.pe_attn_head == 1
    assert DiT(pe_attn_head=8, **kw).config.pe_attn_head == 8
    for bad in (0, 9, -1, 1.0, True):
        with pytest.raises(ValueError):
            DiT(pe_attn_head=bad, **kw)


def _save_v0_checkpoint(d, name):
    """Random base-architecture weights with a 10-entry vocabulary, upstream-free MLX names."""
    from safetensors.torch import save_file
    from f5_tts_mlx_b200.weights import BASE_CONFIG, random_dit_weights
    d.mkdir(parents=True, exist_ok=True)
    (d / "vocab.txt").write_text("\n".join(chr(ord("a") + i) for i in range(10)) + "\n")
    W = random_dit_weights(type(BASE_CONFIG)(text_num_embeds=10), seed=3)
    save_file({k: v.contiguous() for k, v in W.items() if "inv_freq" not in k}, str(d / name))
    return W


def test_from_pretrained_model_version(tmp_path):
    """model_version="v0" builds text_mask_padding=False, pe_attn_head=1: from a directory (upstream's
    model_1200000.safetensors) and from a checkpoint file of any name with vocab.txt beside it; the same file loaded
    as v1 packs the same bytes (the version is never read from the keys)."""
    from f5_tts_mlx_b200 import F5TTS
    import f5_tts_mlx_b200.pretrained as PT
    W = _save_v0_checkpoint(tmp_path / "base", "model_1200000.safetensors")
    f5 = PT.from_pretrained(F5TTS, str(tmp_path / "base"), convert_weights=False, device="cpu", vocoder=False,
                            model_version="v0")
    c = f5.transformer.config
    assert (c.text_mask_padding, c.pe_attn_head, c.text_num_embeds) == (False, 1, 10)
    w = f5.transformer.packed.c_struct()
    assert (w.text_unmasked, w.rope_heads) == (1, 1)
    got = f5.transformer.packed.view("blk3.qkv_w").float()
    want = torch.cat([W[f"transformer.transformer_blocks.3.attn.to_{n}.weight"] for n in "qkv"], 0).bfloat16().float()
    assert torch.equal(got, want)
    # a fine-tune under its own name, addressed as a file
    (tmp_path / "base" / "model_1200000.safetensors").rename(tmp_path / "base" / "my_finetune.safetensors")
    f5f = PT.from_pretrained(F5TTS, str(tmp_path / "base" / "my_finetune.safetensors"), convert_weights=False,
                             device="cpu", vocoder=False, model_version="v0")
    assert (f5f.transformer.config.text_mask_padding, f5f.transformer.config.pe_attn_head) == (False, 1)
    assert torch.equal(f5f.transformer.packed.buffer, f5.transformer.packed.buffer)
    f51 = PT.from_pretrained(F5TTS, str(tmp_path / "base" / "my_finetune.safetensors"), convert_weights=False,
                             device="cpu", vocoder=False)
    assert (f51.transformer.config.text_mask_padding, f51.transformer.config.pe_attn_head) == (True, None)
    assert torch.equal(f51.transformer.packed.buffer, f5.transformer.packed.buffer)


def test_from_pretrained_refusals(tmp_path):
    from f5_tts_mlx_b200 import F5TTS
    import f5_tts_mlx_b200.pretrained as PT
    for kw in (dict(model_version="v2"), dict(model_version="V0"), dict(model_version="v0", quantization_bits=4),
               dict(model_version="v0", quantization_bits=8)):
        with pytest.raises(ValueError):
            PT.from_pretrained(F5TTS, str(tmp_path), device="cpu", vocoder=False, **kw)
    (tmp_path / "weights.bin").write_bytes(b"\0" * 8)
    with pytest.raises(ValueError):
        PT.from_pretrained(F5TTS, str(tmp_path / "weights.bin"), device="cpu", vocoder=False, model_version="v0")
    assert PT.model_file_name("v0") == "model_1200000.safetensors"
    assert PT.model_file_name("v1", 4) == "model_v1_4b.safetensors"


def test_generate_cli_accepts_model_version(monkeypatch):
    import f5_tts_mlx_b200.generate as G
    seen = {}
    monkeypatch.setattr(G, "generate", lambda **kw: seen.update(kw))
    G.main(["--text", "hi", "--model-version", "v0"])
    assert seen["model_version"] == "v0"
    G.main(["--text", "hi"])
    assert seen["model_version"] == "v1"
    with pytest.raises(SystemExit):
        G.main(["--text", "hi", "--model-version", "v2"])
