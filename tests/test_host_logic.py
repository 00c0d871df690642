"""Host-side logic of the package (no GPU): helpers mirror the reference's utils, the solver
evaluation-time schedule, weight packing, key conversion, sharding."""

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import f5_oracle as O
from f5_tts_mlx_b200 import cfm, utils
from f5_tts_mlx_b200.dit import DiT, rope_table, _check_prefix_padding
from f5_tts_mlx_b200.parallel import shard_range
from f5_tts_mlx_b200.weights import (GATE_CONFIG, PackedDiT, convert_upstream_keys, pack_grouped_conv,
                                     random_dit_weights, text_pos_table)


def test_utils_match_oracle():
    lens = torch.tensor([3, 0, 5])
    assert torch.equal(utils.lens_to_mask(lens), O.lens_to_mask(lens))
    assert torch.equal(utils.lens_to_mask(lens, 7), O.lens_to_mask(lens, 7))
    ts = [torch.arange(3), torch.arange(5), torch.arange(1)]
    assert torch.equal(utils.pad_sequence(ts, -1), O.pad_sequence(ts, -1))
    vocab = {c: i for i, c in enumerate(" abcdefgh")}
    txt = [list("abc hx"), list("a")]
    assert torch.equal(utils.list_str_to_idx(txt, vocab), O.list_str_to_idx(txt, vocab))
    assert utils.list_str_to_idx(txt, vocab)[0].tolist() == [1, 2, 3, 0, 8, 0]          # unknown -> 0
    assert utils.list_str_to_idx(txt, vocab)[1].tolist() == [1, -1, -1, -1, -1, -1]     # pad -1
    assert torch.equal(utils.list_str_to_tensor(["hé", "a"]), O.list_str_to_tensor(["hé", "a"]))
    with pytest.raises(ValueError):
        utils.pad_to_length(torch.zeros(2, 2, 2), 4)


def test_convert_char_to_pinyin_ascii():
    out = utils.convert_char_to_pinyin(["Some call me nature; others call me “mother nature”."])
    assert "".join(out[0]) == 'Some call me nature, others call me "mother nature".'
    assert utils.convert_char_to_pinyin(["a,b"])[0] == list("a,b")
    assert utils.convert_char_to_pinyin(["ab,cd"])[0] == list("ab, cd")          # space before a word after ','


def test_time_grid_and_eval_times_match_oracle():
    for steps in (2, 8, 32):
        for sway in (None, -1.0):
            t = cfm.time_grid(steps, sway)
            assert torch.equal(t, O.time_grid(steps, sway))
            for method in ("euler", "midpoint", "rk4"):
                seen = []
                solver = {"euler": O.odeint_euler, "midpoint": O.odeint_midpoint, "rk4": O.odeint_rk4}[method]
                solver(lambda tt, y: (seen.append(float(tt)), y * 0)[1], torch.zeros(1), t)
                got = cfm.ode_eval_times(t, method)            # computed by libf5b200 (host code, no GPU)
                assert got.numel() == len(seen) == O.dit_forwards_per_sample(steps, method, 0.0)
                np.testing.assert_array_equal(got.numpy(), np.array(seen, dtype=np.float32))


def test_public_solvers_match_oracle():
    f = lambda t, y: torch.sin(3 * t) - 0.5 * y
    t = cfm.time_grid(9, -1.0)
    y0 = torch.randn(4)
    for name in ("euler", "midpoint", "rk4"):
        a = getattr(cfm, f"odeint_{name}")(f, y0, t)
        b = getattr(O, f"odeint_{name}")(f, y0, t)
        assert torch.allclose(a, b, atol=1e-6) and a.shape == (9, 4)


def test_rope_table_matches_oracle_freqs():
    fr = O.rotary_freqs(40, 64)
    tab = rope_table(40, 64)
    assert torch.allclose(tab[..., 0], fr[:, 0::2].cos()) and torch.allclose(tab[..., 1], fr[:, 1::2].sin())
    assert torch.equal(text_pos_table(512), O.precompute_freqs_cis(512, 4096))


@pytest.mark.parametrize("dim", [384, 640, 768, 896])
def test_dim_whose_conv_groups_straddle_64_channel_blocks_is_rejected_at_construction(dim):
    """The implicit grouped conv reads 64-channel blocks, so its dim/16-channel groups must tile them.  Widths where
    they straddle a block (dim/16 = 24, 40, 48, 56) are refused when the model is built, not at load time."""
    from f5_tts_mlx_b200.duration import DurationTransformer
    with pytest.raises(ValueError, match="64-channel blocks"):
        DiT(dim=dim, heads=dim // 64, device="cpu")
    with pytest.raises(ValueError, match="64-channel blocks"):
        DurationTransformer(dim=dim, heads=dim // 64, conv_layers=2)


@pytest.mark.parametrize("dim", [1024, 512, 256])
def test_pack_grouped_conv_is_the_grouped_conv(dim):
    """The implicit-GEMM weight layout ([O, 31*64] tap-major, block-diagonal by 64 channels) computes
    exactly Conv1d(groups=16): emulate the kernel's access pattern on the CPU."""
    cg = dim // 16
    w = torch.randn(dim, 31, cg)
    x = torch.randn(1, 50, dim)
    ref = O.conv1d_nlc(x, w, None, padding=15, groups=16)
    wp = pack_grouped_conv(w).view(dim, 31, 64)
    xp = F.pad(x, (0, 0, 15, 15))
    out = torch.zeros(1, 50, dim)
    for blk in range(dim // 64):
        cols = slice(blk * 64, blk * 64 + 64)
        for tap in range(31):
            out[:, :, cols] += xp[:, tap:tap + 50, cols] @ wp[cols, tap, :].T
    assert torch.allclose(out, ref, atol=1e-3)


def test_packed_layout_is_config_determined_and_roundtrips():
    cfg = GATE_CONFIG
    W = random_dit_weights(cfg, seed=7)
    a = PackedDiT(cfg, "cpu").load(W)
    b = PackedDiT(cfg, "cpu")
    assert a.nbytes == b.nbytes and {k: v.offset for k, v in a.specs.items()} == {k: v.offset for k, v in b.specs.items()}
    q = W["transformer.transformer_blocks.2.attn.to_k.weight"]
    assert torch.equal(a.view("blk2.qkv_w")[cfg.dim:2 * cfg.dim].float(), q.bfloat16().float())
    mod = a.view("mod_w")
    assert mod.shape == (cfg.depth * 6 * cfg.dim + 2 * cfg.dim, cfg.dim)
    assert torch.equal(mod[-2 * cfg.dim:].float(), W["transformer.norm_out.linear.weight"].bfloat16().float())
    pw = W["transformer.input_embed.proj.weight"]
    assert torch.equal(a.view("in_x_w")[:, :100].float(), pw[:, :100].bfloat16().float())
    assert (a.view("in_x_w")[:, 100:] == 0).all()
    assert torch.equal(a.view("in_ct_w")[:, :612].float(), pw[:, 100:].bfloat16().float())
    c = a.c_struct()
    assert c.dim == 512 and c.depth == 4 and c.ct_ld == 640 and c.text_rows == 2546
    assert c.blocks[3].ff2_w == a.buffer.data_ptr() + a.specs["blk3.ff2_w"].offset


def test_convert_upstream_keys():
    up = {"ema_model.transformer.transformer_blocks.0.attn.to_out.0.weight": torch.zeros(4, 4),
          "ema_model.transformer.transformer_blocks.0.ff.ff.0.0.weight": torch.zeros(8, 4),
          "ema_model.transformer.transformer_blocks.0.ff.ff.2.bias": torch.zeros(4),
          "ema_model.transformer.time_embed.time_mlp.0.weight": torch.zeros(4, 2),
          "ema_model.transformer.text_embed.text_blocks.1.dwconv.weight": torch.zeros(6, 1, 7),
          "ema_model.transformer.input_embed.conv_pos_embed.conv1d.0.weight": torch.zeros(6, 3, 31),
          "ema_model.mel_spec.mel_stft.window": torch.zeros(3), "initted": torch.zeros(1), "step": torch.zeros(1)}
    out = convert_upstream_keys(up)
    assert set(out) == {"transformer.transformer_blocks.0.attn.to_out.layers.0.weight",
                        "transformer.transformer_blocks.0.ff.ff.layers.0.layers.0.weight",
                        "transformer.transformer_blocks.0.ff.ff.layers.2.bias",
                        "transformer.time_embed.time_mlp.layers.0.weight",
                        "transformer.text_embed.text_blocks.layers.1.dwconv.weight",
                        "transformer.input_embed.conv_pos_embed.conv1d.layers.0.weight"}
    assert out["transformer.text_embed.text_blocks.layers.1.dwconv.weight"].shape == (6, 7, 1)
    assert out["transformer.input_embed.conv_pos_embed.conv1d.layers.0.weight"].shape == (6, 31, 3)


def test_prefix_padding_check_and_constructor_errors():
    _check_prefix_padding(torch.tensor([[1, 2, -1, -1], [3, -1, -1, -1]]))
    with pytest.raises(ValueError):
        _check_prefix_padding(torch.tensor([[1, -1, 2, -1]]))
    with pytest.raises(ValueError):
        DiT(dim=512, heads=4, device="cpu")                 # dim != heads * 64
    with pytest.raises(RuntimeError):
        DiT(dim=512, heads=8, device="cpu")._require_weights()


def test_sample_raises_like_the_reference_without_touching_the_gpu():
    from f5_tts_mlx_b200 import F5TTS
    m = DiT(dim=512, depth=1, heads=8, text_num_embeds=10, text_dim=512, conv_layers=0, device="cpu")
    f5 = F5TTS(m)
    with pytest.raises(ValueError, match="Unknown method"):
        f5.sample(torch.zeros(1, 4, 100), torch.zeros(1, 2, dtype=torch.int32), 8, method="heun")
    with pytest.raises(ValueError, match="Duration must be provided"):
        f5.sample(torch.zeros(1, 4, 100), torch.zeros(1, 2, dtype=torch.int32), None)
    with pytest.raises(ValueError):
        f5.sample(torch.zeros(2, 1000), ["a", "b"], 8)     # raw wave must be batch 1 (cfm.py:284)
    with pytest.raises(NotImplementedError):
        f5(torch.zeros(1))


@pytest.mark.parametrize("n,w", [(512, 8), (10, 4), (3, 8), (0, 2), (65, 8)])
def test_shard_range_partitions(n, w):
    parts = [shard_range(n, w, r) for r in range(w)]
    assert [i for p in parts for i in p] == list(range(n))
    assert max(len(p) for p in parts) - min(len(p) for p in parts) <= 1


def test_from_pretrained_local_directory_roundtrip(tmp_path):
    """cfm.py:404-520 against a local directory: MLX-named and upstream-named safetensors both load into
    the same packed weights (key rename + conv transposes of cfm.py:477-508), vocab gives text_num_embeds =
    len(vocab) - 1, Vocos weights are picked up, the duration checkpoint builds a predictor.  CPU only."""
    from safetensors.torch import save_file
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.weights import BASE_CONFIG, random_duration_weights, random_vocos_weights
    import f5_tts_mlx_b200.pretrained as PT
    vocab_chars = [chr(ord("a") + i) for i in range(10)]
    (tmp_path / "vocab.txt").write_text("\n".join(vocab_chars) + "\n")          # trailing '' entry like the real file
    # a SMALL stand-in for the base architecture is not possible (from_pretrained hard-codes it, cfm.py:459-469),
    # so build the real shapes once with tiny text table (len(vocab) - 1 = 10)
    cfg = type(BASE_CONFIG)(text_num_embeds=10)
    W = random_dit_weights(cfg, seed=3)
    save_file({k: v.contiguous() for k, v in W.items() if "inv_freq" not in k}, str(tmp_path / "model_v1.safetensors"))
    vw = {k[len("vocos."):]: v for k, v in random_vocos_weights().items()}
    up = {}
    for k, v in vw.items():                                                    # upstream torch layouts (O, I, K)
        up[k] = v.transpose(1, 2).contiguous() if (k.endswith("dwconv.weight") or k == "backbone.embed.weight") else v.contiguous()
    save_file(up, str(tmp_path / "vocos.safetensors"))
    save_file({k: v.contiguous() for k, v in random_duration_weights(text_num_embeds=10, seed=4).items()},
              str(tmp_path / "duration_v2.safetensors"))
    f5 = PT.from_pretrained(F5TTS, str(tmp_path), convert_weights=False, device="cpu")
    assert f5.transformer.config.text_num_embeds == 10 and f5._vocoder is not None and f5._duration_predictor is not None
    got = f5.transformer.packed.view("blk5.ff1_w").float()
    assert torch.equal(got, W["transformer.transformer_blocks.5.ff.ff.layers.0.layers.0.weight"].bfloat16().float())
    # the same checkpoint in upstream naming / layouts goes through convert_upstream_keys
    inv = {}
    for k, v in W.items():
        if "inv_freq" in k:
            continue
        k2 = (k.replace(".to_out.layers", ".to_out").replace(".text_blocks.layers", ".text_blocks")
               .replace(".ff.ff.layers.0.layers.0", ".ff.ff.0.0").replace(".ff.ff.layers.2", ".ff.ff.2")
               .replace(".time_mlp.layers", ".time_mlp").replace(".conv1d.layers", ".conv1d"))
        if ".dwconv.weight" in k or ".conv1d.layers.0.weight" in k or ".conv1d.layers.2.weight" in k:
            v = v.transpose(1, 2)
        inv["ema_model." + k2] = v.contiguous()
    inv["ema_model.mel_spec.mel_stft.window"] = torch.zeros(4)
    save_file(inv, str(tmp_path / "model_v1.safetensors"))
    f5b = PT.from_pretrained(F5TTS, str(tmp_path), device="cpu")
    assert torch.equal(f5b.transformer.packed.buffer, f5.transformer.packed.buffer)
    with pytest.raises(ValueError):
        PT.from_pretrained(F5TTS, str(tmp_path / "missing"))
    # MLX affine 4/8-bit checkpoints (cfm.py:450-453, 510-517; generate.py --q): model_v1_{bits}b.safetensors with
    # (weight uint32, scales, biases) per Linear whose input dim is a multiple of 64 -> dequantised at pack time
    from f5_tts_mlx_b200.weights import dequantize_mlx_affine, dequantize_mlx_checkpoint, quantize_mlx_affine
    for bits in (8, 4):
        q = {}
        for k, v in W.items():
            if "inv_freq" in k:
                continue
            if k.endswith(".weight") and v.ndim == 2 and v.shape[1] % 64 == 0 and not k.endswith("text_embed.text_embed.weight"):
                wq, sc, bi = quantize_mlx_affine(v, bits)
                q[k], q[k[:-7] + ".scales"], q[k[:-7] + ".biases"] = wq, sc, bi
            else:
                q[k] = v.contiguous()
        save_file(q, str(tmp_path / f"model_v1_{bits}b.safetensors"))
        f5q = PT.from_pretrained(F5TTS, str(tmp_path), quantization_bits=bits, device="cpu")
        name = "transformer.transformer_blocks.5.ff.ff.layers.0.layers.0.weight"
        dense = dequantize_mlx_checkpoint(q, bits)[name]
        assert torch.equal(f5q.transformer.packed.view("blk5.ff1_w").float(), dense.bfloat16().float())
        step = (W[name].view(W[name].shape[0], -1, 64).amax(-1) - W[name].view(W[name].shape[0], -1, 64).amin(-1)) / (2 ** bits - 1)
        assert ((dense - W[name]).abs().view(W[name].shape[0], -1, 64).amax(-1) <= 0.5001 * step + 1e-7).all()
    with pytest.raises(ValueError):
        PT.from_pretrained(F5TTS, str(tmp_path), quantization_bits=3)
    # the vocoder is mandatory like in the reference (cfm.py:446): no checkpoint anywhere -> loud failure, unless
    # the caller opts out explicitly
    (tmp_path / "vocos.safetensors").unlink()
    with pytest.raises(FileNotFoundError):
        PT.from_pretrained(F5TTS, str(tmp_path), device="cpu")
    assert PT.from_pretrained(F5TTS, str(tmp_path), device="cpu", vocoder=False)._vocoder is None


def test_mlx_affine_dequantisation_known_answer():
    """mx.dequantize layout: code j of a uint32 word sits in bits [j*bits, (j+1)*bits); one (scale, bias) per 64 inputs."""
    from f5_tts_mlx_b200.weights import dequantize_mlx_affine
    codes = (torch.arange(128) % 16).view(1, 128)
    words4 = (codes.view(1, 16, 8).long() << (torch.arange(8) * 4)).sum(-1)
    words4 = torch.where(words4 >= 2 ** 31, words4 - 2 ** 32, words4).to(torch.int32)
    sc, bi = torch.tensor([[0.5, 2.0]]), torch.tensor([[-1.0, 3.0]])
    w = dequantize_mlx_affine(words4, sc, bi, 4)
    exp = torch.cat([codes[0, :64] * 0.5 - 1.0, codes[0, 64:] * 2.0 + 3.0])[None]
    assert torch.equal(w, exp)
    codes8 = (torch.arange(64) * 3 + 7).view(1, 64)
    words8 = (codes8.view(1, 16, 4).long() << (torch.arange(4) * 8)).sum(-1)
    words8 = torch.where(words8 >= 2 ** 31, words8 - 2 ** 32, words8).to(torch.int32)
    assert torch.equal(dequantize_mlx_affine(words8, torch.tensor([[0.25]]), torch.tensor([[1.0]]), 8), codes8 * 0.25 + 1.0)
