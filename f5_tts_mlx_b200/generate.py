"""generate() — host-side mirror of f5_tts_mlx/generate.py:113-244 (+ a real `main()`, which the
reference's console script points at but never defines).

Same keyword arguments and flow: load the 24 kHz reference clip (any rate with `resample_ref_audio`),
RMS-normalise it to 0.1 if quieter, split the text into sentences, one `F5TTS.sample()` per sentence with
the SAME reference audio, strip the reference samples from each waveform, concatenate, write a wav.
Deviations: wav files are read by a small RIFF chunk reader and written by the stdlib `wave` module
(soundfile is not in the image); live playback (AudioPlayer, sounddevice) is out of scope, so
`output_path=None` just returns the waveform; `duration=None` without `estimate_duration` needs a duration predictor exactly like the reference (ValueError otherwise).

Pinned against the reference's own generate() executed through tests/mlx_shim
(tests/golden/ref_generate_calls.json, tests/test_ref_pins.py): sentence split, text assembly,
RMS normalisation, the single-generation path and every keyword that reaches `sample()` are identical.
One deliberate difference, in the multi-sentence loop with `estimate_duration=True`: the reference
estimates from the WHOLE text for every sentence and then re-scales its own previous result
(`duration = int(duration * FRAMES_PER_SEC)` on the already-converted frame count, generate.py:206-209),
so from the second sentence on the request grows by x93.75 per sentence and is clipped to
max_duration = 4096 frames inside sample().  Here each sentence gets its own estimate.
"""
from __future__ import annotations

import argparse
import datetime
import re
import struct
import wave as wavmod
from typing import Literal, Optional

import numpy as np
import torch

from .audio import resample
from .cfm import F5TTS
from .utils import convert_char_to_pinyin

SAMPLE_RATE = 24_000
HOP_LENGTH = 256
FRAMES_PER_SEC = SAMPLE_RATE / HOP_LENGTH
TARGET_RMS = 0.1
DEFAULT_REF_TEXT = "Some call me nature, others call me mother nature."


def split_sentences(text: str):
    """generate.py:30-36."""
    sentence_endings = re.compile(r"([.!?;:])")
    sentences = sentence_endings.split(text)
    sentences = ["".join(i) for i in zip(sentences[0::2], sentences[1::2])]
    return [s.strip() for s in sentences if s.strip()]


def estimated_duration(ref_audio: torch.Tensor, ref_text: str, gen_text: str, speed: float = 1.0) -> float:
    """generate.py:104-111 (byte-length heuristic, zh pause punctuation weighs 3 extra)."""
    ref_audio_len = ref_audio.shape[0] // HOP_LENGTH
    zh_pause_punc = r"。，、；：？！"
    ref_text_len = len(ref_text.encode("utf-8")) + 3 * len(re.findall(zh_pause_punc, ref_text))
    gen_text_len = len(gen_text.encode("utf-8")) + 3 * len(re.findall(zh_pause_punc, gen_text))
    duration_in_frames = ref_audio_len + int(ref_audio_len / ref_text_len * gen_text_len / speed)
    print(f"Got estimated duration: {duration_in_frames / FRAMES_PER_SEC}")
    return duration_in_frames / FRAMES_PER_SEC


WAVE_FORMAT_PCM, WAVE_FORMAT_IEEE_FLOAT, WAVE_FORMAT_EXTENSIBLE = 0x0001, 0x0003, 0xFFFE


def _wav_chunks(raw: bytes, path: str):
    """RIFF/WAVE chunk reader: {chunk id: payload} of the top-level chunks (first occurrence of each)."""
    if len(raw) < 12 or raw[:4] != b"RIFF" or raw[8:12] != b"WAVE":
        raise ValueError(f"{path}: not a RIFF/WAVE file")
    chunks, pos = {}, 12
    while pos + 8 <= len(raw):
        cid, size = raw[pos:pos + 4], struct.unpack_from("<I", raw, pos + 4)[0]
        chunks.setdefault(cid, raw[pos + 8:pos + 8 + size])       # a truncated last chunk keeps what is there
        pos += 8 + size + (size & 1)                               # chunks are padded to an even size
    return chunks


def read_wav(path: str):
    """Mono fp32 waveform and sample rate of a WAV file: 8-bit unsigned, 16-, 24- and 32-bit PCM, or 32-bit IEEE
    float, with a plain or WAVE_FORMAT_EXTENSIBLE header; channels are averaged.  Integer PCM is scaled by 2^-(bits-1)
    (16-bit: x / 32768), float samples are taken as they are.  Other formats raise ValueError."""
    with open(path, "rb") as f:
        chunks = _wav_chunks(f.read(), path)
    fmt, data = chunks.get(b"fmt "), chunks.get(b"data")
    if fmt is None or len(fmt) < 16 or data is None:
        raise ValueError(f"{path}: WAVE file without a complete 'fmt ' and 'data' chunk")
    tag, ch, sr, _, block, bits = struct.unpack_from("<HHIIHH", fmt)
    if tag == WAVE_FORMAT_EXTENSIBLE:
        if len(fmt) < 40:
            raise ValueError(f"{path}: WAVE_FORMAT_EXTENSIBLE header of {len(fmt)} bytes (< 40)")
        tag = struct.unpack_from("<H", fmt, 24)[0]                 # first two bytes of the SubFormat GUID
    kind = {(WAVE_FORMAT_PCM, 8): "u8", (WAVE_FORMAT_PCM, 16): "s16", (WAVE_FORMAT_PCM, 24): "s24",
            (WAVE_FORMAT_PCM, 32): "s32", (WAVE_FORMAT_IEEE_FLOAT, 32): "f32"}.get((tag, bits))
    if kind is None or ch < 1 or block != ch * bits // 8:
        name = {WAVE_FORMAT_PCM: "PCM", WAVE_FORMAT_IEEE_FLOAT: "IEEE float"}.get(tag, f"format tag 0x{tag:04x}")
        raise ValueError(f"{path}: unsupported WAV format: {name}, {bits} bits, {ch} channel(s); supported are "
                         "8-bit unsigned, 16-, 24- and 32-bit PCM and 32-bit IEEE float")
    raw = data[: len(data) // block * block]
    if kind == "s16":
        x = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    elif kind == "u8":
        x = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    elif kind == "s24":
        b3 = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
        v = b3[:, 0] | (b3[:, 1] << 8) | (b3[:, 2] << 16)
        x = (v - ((v & 0x800000) << 1)).astype(np.float32) / 8388608.0
    elif kind == "s32":
        x = (np.frombuffer(raw, dtype="<i4").astype(np.float64) / 2147483648.0).astype(np.float32)
    else:
        x = np.frombuffer(raw, dtype="<f4").astype(np.float32)
    if ch > 1:
        x = x.reshape(-1, ch).mean(axis=1)
    return torch.from_numpy(x), sr


def write_wav(path: str, wave: torch.Tensor, sr: int = SAMPLE_RATE) -> None:
    pcm = (wave.detach().float().cpu().clamp(-1, 1) * 32767.0).round().to(torch.int16).numpy()
    with wavmod.open(path, "wb") as f:
        f.setnchannels(1); f.setsampwidth(2); f.setframerate(sr)
        f.writeframes(pcm.tobytes())


def generate(
    generation_text: str,
    duration: Optional[float] = None,
    estimate_duration: bool = False,
    model_name: str = "lucasnewman/f5-tts-mlx",
    ref_audio_path: Optional[str] = None,
    ref_audio_text: Optional[str] = None,
    steps: int = 8,
    method: Literal["euler", "midpoint", "rk4"] = "rk4",
    cfg_strength: float = 2.0,
    sway_sampling_coef: float = -1.0,
    speed: float = 1.0,
    seed: Optional[int] = None,
    quantization_bits: Optional[int] = None,
    output_path: Optional[str] = None,
    f5tts: Optional[F5TTS] = None,
    batch_sentences: bool = False,
    frame_bucket: int = 128,
    fp8: Optional[str] = None,
    fp8_attention: bool = False,
    resample_ref_audio: bool = False,
    output_sample_rate: int = SAMPLE_RATE,
    model_version: str = "v1",
    vocoder: Literal["vocos", "bigvgan"] = "vocos",
):
    """generate.py:113-244.  Extensions: `f5tts` reuses a loaded model; `batch_sentences=True` runs all
    sentences as ONE ragged `sample()` batch instead of the reference's serial loop
    (numerically it differs from the serial loop only through the reference's own padding caveat — GRN
    statistics and the ODE on padded frames see the batch-maximum length); `frame_bucket` (default 128 frames) lets
    the sentences of the serial loop share one set of buffers and ONE captured CUDA graph per length bucket instead of
    re-capturing for every distinct length (0 = the exact shapes); results are unchanged (F5TTS.sample).  `fp8`: None
    (bf16), "tensor" or "block" — the lossy FP8 mode of the DiT and its scaling (DESIGN.md section 8);
    `fp8_attention` (with fp8="block"): the attention on e4m3 Q, K and V as well.  `resample_ref_audio`: a reference
    clip at any sample rate is RMS-normalised, then resampled to 24 kHz on the GPU (audio.resample, torchaudio's
    default windowed sinc, as upstream F5-TTS does); without it a clip that is not 24 kHz is refused, as in the
    reference.  `output_sample_rate`: the returned / written waveform is resampled from 24 kHz to this rate.
    `model_version`: "v1" (default), "v0" — F5TTS_Base checkpoints — or "e2" — E2TTS_Base, which has no duration
    predictor: pass `duration` or `estimate_duration` (F5TTS.from_pretrained); `model_name` may also name a .safetensors
    file with vocab.txt beside it.  `vocoder`: "vocos" (default) or "bigvgan" — an F5TTS_Base_bigvgan
    model: BigVGAN v2 and its mel front-end, from bigvgan/ next to the model or $F5_BIGVGAN_PATH; it has no duration
    predictor, so pass `duration` or `estimate_duration`."""
    if vocoder not in ("vocos", "bigvgan"):
        raise ValueError(f'vocoder must be "vocos" or "bigvgan", not {vocoder!r}')
    if fp8_attention and fp8 != "block":
        raise ValueError('fp8_attention needs fp8="block"')
    output_sample_rate = int(output_sample_rate)
    if output_sample_rate <= 0:
        raise ValueError(f"output_sample_rate must be positive, got {output_sample_rate}")
    if f5tts is None:
        f5tts = F5TTS.from_pretrained(model_name, quantization_bits=quantization_bits, fp8=fp8,
                                      fp8_attention=fp8_attention, model_version=model_version,
                                      **({"vocoder": "bigvgan"} if vocoder == "bigvgan" else {}))
    dev = f5tts.transformer.device
    if f5tts._vocoder is None:
        raise ValueError("generate() needs a model with a vocoder (F5TTS(..., vocoder=Vocos(...).decode)); "
                         "without one sample() returns mel spectrograms, not a waveform")
    if ref_audio_path is None:
        raise ValueError("ref_audio_path is required (the reference's packaged default clip is not redistributed here)")
    audio, sr = read_wav(ref_audio_path)
    if sr != SAMPLE_RATE and not resample_ref_audio:                              # generate.py:147-148
        raise ValueError(f"Reference audio must have a sample rate of 24kHz (got {sr} Hz; "
                         "resample_ref_audio=True / --resample converts it)")
    if ref_audio_text is None:
        ref_audio_text = DEFAULT_REF_TEXT
    print(f"Got reference audio with duration: {audio.shape[0] / sr:.2f} seconds")
    rms = torch.sqrt(torch.mean(torch.square(audio)))
    if rms < TARGET_RMS:
        audio = audio * TARGET_RMS / rms                                          # generate.py:154-156
    audio_d = audio.to(dev)
    if sr != SAMPLE_RATE:
        audio_d = resample(audio_d, sr, SAMPLE_RATE)                              # normalised first, as upstream
    ref_len = audio_d.shape[0]                                                    # reference samples at 24 kHz

    sentences = split_sentences(generation_text)
    single = len(sentences) <= 1 or duration is not None                          # generate.py:158-159
    todo = [generation_text] if single else sentences
    start = datetime.datetime.now()
    waves = []
    frames = None
    if duration is not None:
        frames = int(duration * FRAMES_PER_SEC)
    if batch_sentences and len(todo) > 1:
        if duration is None and not estimate_duration and f5tts._duration_predictor is None:
            raise ValueError("Duration must be provided or a duration predictor must be set.")
        mel = f5tts._mel_spec(audio_d)                                    # (1, n_ref, 100), computed once
        texts = convert_char_to_pinyin([ref_audio_text + " " + s_ for s_ in todo])
        if duration is None and estimate_duration:
            durs = torch.tensor([int(estimated_duration(audio_d, ref_audio_text, s_, speed) * FRAMES_PER_SEC) for s_ in todo])
        elif duration is None:
            durs = None
        else:
            durs = torch.full((len(todo),), frames)
        cond = mel.repeat(len(todo), 1, 1)
        vocoder, f5tts._vocoder = f5tts._vocoder, None                    # decode per utterance at its own length
        try:
            out, _ = f5tts.sample(cond, text=texts, duration=durs, steps=steps, method=method, speed=speed,
                                  cfg_strength=cfg_strength, sway_sampling_coef=sway_sampling_coef, seed=seed,
                                  return_trajectory=False)
        finally:
            f5tts._vocoder = vocoder
        plan = f5tts.last_plan
        lens_i = plan.session.seq_len[: len(todo)].tolist() if plan.session.seq_len is not None else [out.shape[1]] * len(todo)
        for i in range(len(todo)):
            wave_i = vocoder(out[i:i + 1, : lens_i[i]]) if vocoder is not None else out[i, : lens_i[i]]
            waves.append(wave_i[ref_len:] if vocoder is not None else wave_i)
        todo = []
    for sentence in todo:
        if duration is None and estimate_duration:
            frames = int(estimated_duration(audio_d, ref_audio_text, sentence if not single else generation_text, speed)
                         * FRAMES_PER_SEC)
        text = convert_char_to_pinyin([ref_audio_text + " " + sentence])
        wave, _ = f5tts.sample(audio_d[None], text=text, duration=frames, steps=steps, method=method, speed=speed,
                               cfg_strength=cfg_strength, sway_sampling_coef=sway_sampling_coef, seed=seed,
                               return_trajectory=False, frame_bucket=frame_bucket)
        waves.append(wave[ref_len:])                                              # strip the reference (generate.py:183)
    wave = torch.cat(waves, dim=0)
    if wave.is_cuda:
        torch.cuda.synchronize()
    print(f"Generated {wave.shape[0] / SAMPLE_RATE:.2f}s of audio in {datetime.datetime.now() - start}.")
    if output_sample_rate != SAMPLE_RATE:
        wave = resample(wave, SAMPLE_RATE, output_sample_rate)
    if output_path is not None:
        write_wav(output_path, wave, output_sample_rate)
    return wave


def main(argv=None) -> None:
    p = argparse.ArgumentParser(description="Generate speech from text using F5-TTS on H100")
    p.add_argument("--model", type=str, default="lucasnewman/f5-tts-mlx")
    p.add_argument("--text", type=str, default=None)
    p.add_argument("--duration", type=float, default=None)
    p.add_argument("--estimate-duration", type=bool, default=False)
    p.add_argument("--ref-audio", type=str, default=None)
    p.add_argument("--ref-text", type=str, default=None)
    p.add_argument("--output", type=str, default=None)
    p.add_argument("--steps", type=int, default=8)
    p.add_argument("--method", type=str, default="rk4", choices=["euler", "midpoint", "rk4"])
    p.add_argument("--cfg", type=float, default=2.0)
    p.add_argument("--sway-coef", type=float, default=-1.0)
    p.add_argument("--speed", type=float, default=1.0)
    p.add_argument("--seed", type=int, default=None)
    p.add_argument("--q", type=int, default=None, choices=[4, 8])
    p.add_argument("--fp8", type=str, default=None, choices=["tensor", "block"],
                   help="run the DiT's GEMMs on e4m3 operands (lossy) with per-tensor or block (per-channel / per-64) scales")
    p.add_argument("--fp8-attention", action="store_true",
                   help="with --fp8 block: run the attention's Q·K^T and P·V on e4m3 too (lossy)")
    p.add_argument("--resample", action="store_true",
                   help="accept a reference clip at any sample rate: resample it to 24 kHz on the GPU")
    p.add_argument("--output-sample-rate", type=int, default=SAMPLE_RATE,
                   help="sample rate of the written waveform (resampled on the GPU from 24 kHz)")
    p.add_argument("--model-version", type=str, default="v1", choices=["v1", "v0", "e2"],
                   help="v0: an F5TTS_Base checkpoint (unmasked text padding, rotary embedding on the first head only); "
                        "e2: an E2TTS_Base checkpoint (UNetT backbone; pass --duration or --estimate-duration)")
    p.add_argument("--vocoder", type=str, default="vocos", choices=["vocos", "bigvgan"],
                   help="bigvgan: an F5TTS_Base_bigvgan model (BigVGAN v2 and its mel; bigvgan/ next to the model)")
    a = p.parse_args(argv)
    if a.fp8_attention and a.fp8 != "block":
        p.error("--fp8-attention needs --fp8 block")
    if a.text is None:
        import sys
        if not sys.stdin.isatty():
            a.text = sys.stdin.read().strip()
        else:
            a.text = input("Enter text to generate: ")
    generate(generation_text=a.text, duration=a.duration, estimate_duration=a.estimate_duration, model_name=a.model,
             ref_audio_path=a.ref_audio, ref_audio_text=a.ref_text, steps=a.steps, method=a.method, cfg_strength=a.cfg,
             sway_sampling_coef=a.sway_coef, speed=a.speed, seed=a.seed, quantization_bits=a.q, output_path=a.output,
             fp8=a.fp8, fp8_attention=a.fp8_attention, resample_ref_audio=a.resample,
             output_sample_rate=a.output_sample_rate, model_version=a.model_version,
             **({"vocoder": "bigvgan"} if a.vocoder == "bigvgan" else {}))


if __name__ == "__main__":
    main()
