"""F5TTS.from_pretrained — host-side mirror of cfm.py:404-520 (load-time only).

There is no network in the build/bench environment, so `hf_model_name_or_path` is a local directory
(or, when `huggingface_hub` is importable and online, a hub repo id exactly like the reference's
`fetch_from_hub`, utils.py:179-192) holding `model_v1.safetensors` (or `model_v1_{4,8}b.safetensors`, MLX affine
quantised, dequantised at load), `vocab.txt` and optionally `duration_v2.safetensors`.  The vocoder is resolved
separately, like the reference's `Vocos.from_pretrained("lucasnewman/vocos-mel-24khz")` (cfm.py:446): a
`vocos.safetensors` / `vocos-mel-24khz/` next to the model, `$F5_VOCOS_PATH`, or that hub repo; if none can be
found the load FAILS (the reference always has a vocoder) unless `vocoder=False` is passed explicitly.
The special name "random" builds the base model with seeded random weights (what the tests and bench.py use); its
vocabulary is `vocab_path` / `$F5_VOCAB_PATH` when given, else a printable-ASCII table, stated in `vocab_source`.

Multi-GPU: only rank 0 reads / converts / packs; every other rank allocates the same packed layout
and receives it in ONE broadcast (parallel.load_weights_distributed).
"""
from __future__ import annotations

from pathlib import Path
from typing import Optional

import torch

from .dit import DiT
from .parallel import load_weights_distributed
from .vocos import Vocos
from .weights import (BASE_CONFIG, FP8_SCALINGS, VocosConfig, Weights, convert_upstream_keys, dequantize_mlx_checkpoint,
                      random_dit_weights, random_vocos_weights)

VOCOS_REPO = "lucasnewman/vocos-mel-24khz"
VOCOS_FILES = ("vocos.safetensors", "vocos-mel-24khz/model.safetensors", "vocos-mel-24khz/vocos.safetensors")


# model_version -> (checkpoint file of a model directory, DiT arguments).  Both versions have the same parameter names
# and shapes, so the version is never guessed from a checkpoint's keys.  v0 is upstream's F5TTS_Base (and the fine-tunes
# built on it): TextEmbedding(mask_padding=False) and rotary embedding on the first attention head only.
MODEL_VERSIONS = {
    "v1": ("model_v1.safetensors", dict(text_mask_padding=True, pe_attn_head=None)),    # cfm.py:459-469
    "v0": ("model_1200000.safetensors", dict(text_mask_padding=False, pe_attn_head=1)),
    # E2TTS_Base: the UNetT backbone (unett.py), upstream's E2TTS_Base/model_1200000.safetensors
    "e2": ("model_1200000.safetensors", dict(text_mask_padding=False, pe_attn_head=1)),
}


def model_file_name(model_version: str = "v1", quantization_bits: Optional[int] = None) -> str:
    """The checkpoint a model directory of this version holds; ValueError for an unknown version, or for quantised v0
    weights (there are no MLX-quantised v0 files)."""
    if model_version not in MODEL_VERSIONS:
        raise ValueError(f"model_version must be one of {tuple(MODEL_VERSIONS)}, not {model_version!r}")
    if quantization_bits is None:
        return MODEL_VERSIONS[model_version][0]
    if model_version != "v1":
        raise ValueError(f"quantization_bits is only available for model_version='v1' (there are no quantised "
                         f"{model_version} checkpoints)")
    return f"model_v1_{quantization_bits}b.safetensors"


def _resolve(path_or_repo: str, quantization_bits: Optional[int], model_version: str = "v1") -> Optional[Path]:
    p = Path(path_or_repo)
    if p.is_dir():
        return p
    try:                                               # same behaviour as utils.py:179-192 when online
        from huggingface_hub import snapshot_download  # type: ignore
        fn = model_file_name(model_version, quantization_bits)
        return Path(snapshot_download(repo_id=path_or_repo, allow_patterns=[fn, "duration_v2.safetensors", "*.txt"]))
    except Exception:
        return None


def checkpoint_weights(path: Path, quantization_bits: Optional[int] = None, convert_weights=None,
                       model_file: Optional[str] = None):
    """(vocab, weights_fn) of a local model directory as from_pretrained reads it: weights_fn() returns the DiT's
    weights with the reference's parameter names (converted from the upstream keys, or dequantised).  `model_file`:
    the checkpoint inside `path` (default: the v1 one, model_v1[_{4,8}b].safetensors)."""
    from safetensors.torch import load_file
    vocab = read_vocab(path / "vocab.txt")
    convert = True if convert_weights is None else convert_weights               # cfm.py:455
    if model_file is None:
        model_file = model_file_name("v1", quantization_bits)
    if quantization_bits is not None:                                            # cfm.py:450-453
        convert = False

    def weights_fn() -> Weights:
        w = load_file(str(path / model_file))
        if quantization_bits is not None:     # nn.quantize + load_weights (cfm.py:510-517): dense again at pack time
            return dequantize_mlx_checkpoint(w, quantization_bits)
        return convert_upstream_keys(w) if convert else w

    return vocab, weights_fn


def _resolve_vocos(model_dir: Optional[Path]) -> Optional[Path]:
    """The vocoder checkpoint: next to the model, $F5_VOCOS_PATH (file or directory), or the hub repo the reference
    uses (cfm.py:446)."""
    import os
    cands = []
    env = os.environ.get("F5_VOCOS_PATH")
    if env:
        e = Path(env)
        cands += [e] if e.is_file() else [e / "model.safetensors", e / "vocos.safetensors"]
    if model_dir is not None:
        cands += [model_dir / f for f in VOCOS_FILES]
    for c in cands:
        if c.is_file():
            return c
    try:
        from huggingface_hub import snapshot_download  # type: ignore
        d = Path(snapshot_download(repo_id=VOCOS_REPO, allow_patterns=["*.safetensors", "*.yaml", "*.json"]))
        for c in sorted(d.glob("*.safetensors")):
            return c
    except Exception:
        pass
    return None


def _resolve_bigvgan(model_dir: Optional[Path]) -> Path:
    """The BigVGAN directory (bigvgan_generator.pt and config.json): $F5_BIGVGAN_PATH, or bigvgan/ next to the model.
    Local only: there is no hub download."""
    import os
    cands = []
    env = os.environ.get("F5_BIGVGAN_PATH")
    if env:
        cands.append(Path(env))
    if model_dir is not None:
        cands.append(model_dir / "bigvgan")
    for c in cands:
        if (c / "bigvgan_generator.pt").is_file() and (c / "config.json").is_file():
            return c
    raise FileNotFoundError(f"no BigVGAN checkpoint found (looked for bigvgan_generator.pt and config.json in "
                            f"{', '.join(map(str, cands)) or '$F5_BIGVGAN_PATH (unset)'})")


def ascii_vocab() -> dict:
    """Printable ASCII, in the file layout read_vocab() expects (trailing '' entry)."""
    chars = [chr(i) for i in range(32, 127)] + [""]
    return {v: i for i, v in enumerate(chars)}


def read_vocab(vocab_path: Path) -> dict:
    """cfm.py:418-421 — note the trailing '' entry: text_num_embeds = len(vocab) - 1."""
    vocab = {v: i for i, v in enumerate(Path(vocab_path).read_text().split("\n"))}
    if len(vocab) == 0:
        raise ValueError(f"Could not load vocab from {vocab_path}")
    return vocab


def convert_vocos_upstream(w: Weights) -> Weights:
    """Upstream (PyTorch) Vocos checkpoint names/layouts -> the names used here; conv weights
    (O, I/g, K) -> (O, K, I/g)."""
    out: Weights = {}
    for k, v in w.items():
        if k.startswith("feature_extractor") or "istft.window" in k:
            continue
        if k.endswith("dwconv.weight") or k == "backbone.embed.weight":
            v = v.transpose(1, 2)
        out["vocos." + k] = v
    return out


def from_pretrained(cls, hf_model_name_or_path: str, convert_weights=None, quantization_bits: Optional[int] = None,
                    device: str | torch.device = "cuda", vocab_path: Optional[str] = None, vocoder=None,
                    fp8: Optional[str] = None, fp8_attention: bool = False, model_version: str = "v1"):
    """`vocoder`: None = resolve and REQUIRE one (reference behaviour), False = none (sample() returns mels),
    or a callable mel -> waveform.  `fp8`: None = bf16, "tensor" or "block" = the DiT's FP8 mode with that weight /
    activation scaling (DESIGN.md section 8); the weights (dequantised first for quantization_bits) are quantised to
    e4m3 at pack time.  `fp8_attention` (needs fp8="block"): the attention on e4m3 Q, K and V as well.
    `vocoder="bigvgan"`: an F5TTS_Base_bigvgan model (upstream's `--vocoder_name bigvgan`): BigVGAN v2 decodes, and the
    reference clip goes through BigVGAN's mel (bigvgan.BigVGANMelSpec).  bigvgan_generator.pt and config.json are read
    from $F5_BIGVGAN_PATH or bigvgan/ next to the model (no download); "random" builds the released config with random
    weights.  No duration predictor is attached, since duration_v2 was trained on the other mel: pass a duration.
    State model_version="v0" for these checkpoints (nothing is guessed).  `vocoder="vocos"` is the default behaviour.
    `model_version`: "v1" (default, the reference's model), "v0" (upstream's F5TTS_Base and its fine-tunes: unmasked
    text padding, rotary embedding on the first attention head only; a directory holds model_1200000.safetensors) or
    "e2" (upstream's E2TTS_Base on the UNetT backbone: see _from_pretrained_e2).
    The version is the caller's to state: v0 and v1 checkpoints have identical keys.  `hf_model_name_or_path` may
    also name a .safetensors file, with vocab.txt (and optionally duration_v2.safetensors) beside it, or an upstream
    training checkpoint .pt (its ema_model_state_dict, read with torch.load(weights_only=True))."""
    import os
    if model_version == "e2":
        return _from_pretrained_e2(cls, hf_model_name_or_path, quantization_bits, device, vocab_path, vocoder, fp8,
                                   fp8_attention)
    if vocoder == "vocos":
        vocoder = None
    use_bigvgan = isinstance(vocoder, str) and vocoder == "bigvgan"
    if isinstance(vocoder, str) and not use_bigvgan:
        raise ValueError(f"vocoder must be \"vocos\", \"bigvgan\", False, None or a callable, not {vocoder!r}")
    mel_kw = {}
    if use_bigvgan:
        from .bigvgan import BigVGANMelSpec
        mel_kw = dict(mel_spec_module=BigVGANMelSpec())
    if quantization_bits is not None and quantization_bits not in (4, 8):
        raise ValueError(f"quantization_bits must be 4 or 8 (generate.py --q), got {quantization_bits}")
    model_file = model_file_name(model_version, quantization_bits)     # ValueError: unknown version, quantised v0
    version_kw = MODEL_VERSIONS[model_version][1]
    if fp8 is not None and fp8 not in FP8_SCALINGS:
        raise ValueError(f"fp8 must be None or one of {FP8_SCALINGS}, got {fp8!r}")
    fp8_kw = dict(fp8=fp8 is not None, fp8_scaling=fp8 or "tensor", fp8_attention=fp8_attention)
    if hf_model_name_or_path == "random":
        vp = vocab_path or os.environ.get("F5_VOCAB_PATH")
        if vp is not None:
            vocab, vocab_source = read_vocab(Path(vp)), str(vp)     # missing file -> FileNotFoundError, not a silent switch
        else:
            vocab, vocab_source = ascii_vocab(), "ascii"
        cfg = BASE_CONFIG
        dit = DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, text_dim=cfg.text_dim,
                  conv_layers=cfg.conv_layers, text_num_embeds=cfg.text_num_embeds, device=device, **version_kw,
                  **fp8_kw)
        load_weights_distributed(dit, lambda: random_dit_weights(cfg, seed=1234))
        if use_bigvgan:
            from .bigvgan import BigVGAN, BigVGANConfig, random_bigvgan_weights
            vocoder = BigVGAN(BigVGANConfig(), device).load_weights(random_bigvgan_weights(BigVGANConfig(), seed=1234)).decode
        elif vocoder is None:
            vocoder = Vocos(VocosConfig(), device).load_weights(random_vocos_weights()).decode
        m = cls(transformer=dit, vocab_char_map=vocab, vocoder=vocoder or None, **mel_kw)
        m.vocab_source = vocab_source
        return m

    given = Path(hf_model_name_or_path)
    if given.is_file():                  # a checkpoint file (fine-tunes have their own names), vocab.txt beside it
        if given.suffix not in (".safetensors", ".pt"):
            raise ValueError(f"{given} is not a .safetensors or .pt checkpoint")
        if given.suffix == ".pt" and quantization_bits is not None:
            raise ValueError("quantization_bits applies to MLX .safetensors checkpoints, not to a .pt file")
        path, model_file = given.parent, given.name
    else:
        path = _resolve(hf_model_name_or_path, quantization_bits, model_version)
    if path is None:
        raise ValueError(f"Could not find model {hf_model_name_or_path}")        # cfm.py:413-414
    from safetensors.torch import load_file
    if given.is_file() and given.suffix == ".pt":      # upstream training checkpoint: the EMA weights, upstream keys
        vocab = read_vocab(path / "vocab.txt")

        def weights_fn() -> Weights:
            ck = torch.load(str(given), map_location="cpu", weights_only=True)
            if "ema_model_state_dict" not in ck:
                raise ValueError(f"{given} has no ema_model_state_dict")
            return convert_upstream_keys({k: v.float() for k, v in ck["ema_model_state_dict"].items()})
    else:
        vocab, weights_fn = checkpoint_weights(path, quantization_bits, convert_weights, model_file)
    dit = DiT(dim=1024, depth=22, heads=16, ff_mult=2, text_dim=512, conv_layers=4,
              text_num_embeds=len(vocab) - 1, device=device, **version_kw, **fp8_kw)     # cfm.py:459-469
    load_weights_distributed(dit, weights_fn)
    if use_bigvgan:
        from .bigvgan import BigVGAN, load_checkpoint
        bcfg, bsd = load_checkpoint(_resolve_bigvgan(path))
        vocoder = BigVGAN(bcfg, device).load_weights(bsd).decode
        return cls(transformer=dit, vocab_char_map=vocab, vocoder=vocoder, **mel_kw)
    if vocoder is None:                                                          # cfm.py:446: always present
        vpath = _resolve_vocos(path)
        if vpath is None:
            raise FileNotFoundError(
                f"no Vocos checkpoint found (looked for {', '.join(VOCOS_FILES)} in {path}, $F5_VOCOS_PATH and the hub "
                f"repo {VOCOS_REPO}); pass vocoder=False to get mel spectrograms from sample() instead")
        vocoder = Vocos(VocosConfig(), device).load_weights(convert_vocos_upstream(load_file(str(vpath)))).decode
    elif vocoder is False:
        vocoder = None
    duration_predictor = None
    dpath = path / "duration_v2.safetensors"
    if dpath.exists():                                                           # cfm.py:425-442
        from .duration import DurationPredictor, DurationTransformer
        duration_predictor = DurationPredictor(
            transformer=DurationTransformer(dim=512, depth=8, heads=8, text_dim=512, ff_mult=2, conv_layers=2,
                                            text_num_embeds=len(vocab) - 1),
            vocab_char_map=vocab, device=device).load_weights(load_file(str(dpath)))
    return cls(transformer=dit, vocab_char_map=vocab, vocoder=vocoder, duration_predictor=duration_predictor)


def _from_pretrained_e2(cls, hf_model_name_or_path: str, quantization_bits, device, vocab_path, vocoder, fp8,
                        fp8_attention):
    """E2TTS_Base (upstream F5-TTS `--model E2TTS_Base`): a UNetT backbone (unett.UNetT) with the Vocos vocoder and no
    duration predictor (pass `duration` to sample(), or estimate it).  Reads a directory holding
    model_1200000.safetensors and vocab.txt, or a .safetensors / upstream training .pt file (its ema_model_state_dict)
    with vocab.txt beside it; every key must be one of the model's (unett.checkpoint_state).  "random" builds seeded
    random E2TTS_Base weights.  There is no FP8 mode, no quantised checkpoint and no BigVGAN for this backbone yet."""
    import os
    from .unett import E2_BASE_CONFIG, UNetT, random_unett_weights
    if fp8 is not None or fp8_attention:
        raise ValueError("model_version='e2' has no FP8 mode (fp8 / fp8_attention): it runs in bf16")
    if quantization_bits is not None:
        raise ValueError("model_version='e2' has no quantised checkpoints (quantization_bits)")
    if isinstance(vocoder, str) and vocoder != "vocos":
        raise ValueError(f"model_version='e2' decodes with Vocos only, not vocoder={vocoder!r}")
    if vocoder == "vocos":
        vocoder = None
    cfg = E2_BASE_CONFIG

    def backbone(text_num_embeds: int, dim: int = cfg.dim, depth: int = cfg.depth, ff_mult: int = cfg.ff_mult) -> UNetT:
        return UNetT(dim=dim, depth=depth, heads=dim // 64, ff_mult=ff_mult, mel_dim=cfg.mel_dim,
                     text_num_embeds=text_num_embeds, text_dim=cfg.text_dim, text_mask_padding=False, conv_layers=0,
                     pe_attn_head=cfg.pe_attn_head, skip_connect_type="concat", device=device)

    if hf_model_name_or_path == "random":
        vp = vocab_path or os.environ.get("F5_VOCAB_PATH")
        vocab, vocab_source = (read_vocab(Path(vp)), str(vp)) if vp is not None else (ascii_vocab(), "ascii")
        net = backbone(cfg.text_num_embeds)
        load_weights_distributed(net, lambda: random_unett_weights(cfg, seed=1234))
        if vocoder is None:
            vocoder = Vocos(VocosConfig(), device).load_weights(random_vocos_weights()).decode
        m = cls(transformer=net, vocab_char_map=vocab, vocoder=vocoder or None)
        m.vocab_source = vocab_source
        return m

    given = Path(hf_model_name_or_path)
    if given.is_file():
        if given.suffix not in (".safetensors", ".pt"):
            raise ValueError(f"{given} is not a .safetensors or .pt checkpoint")
        path, model_file = given.parent, given
    else:
        path = _resolve(hf_model_name_or_path, None, "e2")
        if path is None:
            raise ValueError(f"Could not find model {hf_model_name_or_path}")
        model_file = path / MODEL_VERSIONS["e2"][0]
    vocab = read_vocab(path / "vocab.txt")

    if model_file.suffix == ".pt":
        ck = torch.load(str(model_file), map_location="cpu", weights_only=True)
        if "ema_model_state_dict" not in ck:
            raise ValueError(f"{model_file} has no ema_model_state_dict")
        sd = {k: v.float() for k, v in ck["ema_model_state_dict"].items()}
    else:
        from safetensors.torch import load_file
        sd = load_file(str(model_file))
    # width, depth and FF width from the tensors (E2TTS_Base: 1024, 24, 4); the key check then covers every layer
    sd = {k[len("ema_model."):] if k.startswith("ema_model.") else k: v for k, v in sd.items()}
    try:
        dim = sd["transformer.proj_out.weight"].shape[1]
        depth = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transformer.layers."))
        ff_mult = sd["transformer.layers.0.4.ff.0.0.weight"].shape[0] // dim
    except (KeyError, ValueError) as e:
        raise ValueError(f"{model_file} is not an E2TTS_Base-form UNetT checkpoint ({e!r})") from None
    net = backbone(len(vocab) - 1, dim, depth, ff_mult)
    load_weights_distributed(net, lambda: sd)
    if vocoder is None:
        vpath = _resolve_vocos(path)
        if vpath is None:
            raise FileNotFoundError(
                f"no Vocos checkpoint found (looked for {', '.join(VOCOS_FILES)} in {path}, $F5_VOCOS_PATH and the hub "
                f"repo {VOCOS_REPO}); pass vocoder=False to get mel spectrograms from sample() instead")
        from safetensors.torch import load_file
        vocoder = Vocos(VocosConfig(), device).load_weights(convert_vocos_upstream(load_file(str(vpath)))).decode
    elif vocoder is False:
        vocoder = None
    return cls(transformer=net, vocab_char_map=vocab, vocoder=vocoder)
