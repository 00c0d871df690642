"""generate() — host-side mirror of f5_tts_mlx/generate.py:113-244 (+ a real `main()`, which the
reference's console script points at but never defines).

Same keyword arguments and flow: load the 24 kHz reference clip, RMS-normalise it to 0.1 if quieter,
split the text into sentences, one `F5TTS.sample()` per sentence with the SAME reference audio,
strip the reference samples from each waveform, concatenate, write a wav.  Deviations: wav I/O uses
the stdlib `wave` module (soundfile is not in the image); live playback (AudioPlayer, sounddevice)
is out of scope, so `output_path=None` just returns the waveform; `duration=None` without
`estimate_duration` needs a duration predictor exactly like the reference (ValueError otherwise).

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
import wave as wavmod
from typing import Literal, Optional

import numpy as np
import torch

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


def read_wav(path: str):
    with wavmod.open(path, "rb") as f:
        sr, ch, sw, n = f.getframerate(), f.getnchannels(), f.getsampwidth(), f.getnframes()
        raw = f.readframes(n)
    if sw != 2:
        raise ValueError("only 16-bit PCM wav files are supported")
    x = np.frombuffer(raw, dtype=np.int16).astype(np.float32) / 32768.0
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
):
    """generate.py:113-244.  Extensions: `f5tts` reuses a loaded model; `batch_sentences=True` runs all
    sentences as ONE ragged `sample()` batch instead of the reference's serial loop
    (numerically it differs from the serial loop only through the reference's own padding caveat — GRN
    statistics and the ODE on padded frames see the batch-maximum length); `frame_bucket` (default 128 frames) lets
    the sentences of the serial loop share one set of buffers and ONE captured CUDA graph per length bucket instead of
    re-capturing for every distinct length (0 = the exact shapes); results are unchanged (F5TTS.sample)."""
    if f5tts is None:
        f5tts = F5TTS.from_pretrained(model_name, quantization_bits=quantization_bits)
    dev = f5tts.transformer.device
    if f5tts._vocoder is None:
        raise ValueError("generate() needs a model with a vocoder (F5TTS(..., vocoder=Vocos(...).decode)); "
                         "without one sample() returns mel spectrograms, not a waveform")
    if ref_audio_path is None:
        raise ValueError("ref_audio_path is required (the reference's packaged default clip is not redistributed here)")
    audio, sr = read_wav(ref_audio_path)
    if sr != SAMPLE_RATE:
        raise ValueError("Reference audio must have a sample rate of 24kHz")      # generate.py:147-148
    if ref_audio_text is None:
        ref_audio_text = DEFAULT_REF_TEXT
    print(f"Got reference audio with duration: {audio.shape[0] / SAMPLE_RATE:.2f} seconds")
    rms = torch.sqrt(torch.mean(torch.square(audio)))
    if rms < TARGET_RMS:
        audio = audio * TARGET_RMS / rms                                          # generate.py:154-156
    audio_d = audio.to(dev)

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
            durs = torch.tensor([int(estimated_duration(audio, ref_audio_text, s_, speed) * FRAMES_PER_SEC) for s_ in todo])
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
            waves.append(wave_i[audio.shape[0]:] if vocoder is not None else wave_i)
        todo = []
    for sentence in todo:
        if duration is None and estimate_duration:
            frames = int(estimated_duration(audio, ref_audio_text, sentence if not single else generation_text, speed)
                         * FRAMES_PER_SEC)
        text = convert_char_to_pinyin([ref_audio_text + " " + sentence])
        wave, _ = f5tts.sample(audio_d[None], text=text, duration=frames, steps=steps, method=method, speed=speed,
                               cfg_strength=cfg_strength, sway_sampling_coef=sway_sampling_coef, seed=seed,
                               return_trajectory=False, frame_bucket=frame_bucket)
        waves.append(wave[audio.shape[0]:])                                       # strip the reference (generate.py:183)
    wave = torch.cat(waves, dim=0)
    if wave.is_cuda:
        torch.cuda.synchronize()
    print(f"Generated {wave.shape[0] / SAMPLE_RATE:.2f}s of audio in {datetime.datetime.now() - start}.")
    if output_path is not None:
        write_wav(output_path, wave)
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
    a = p.parse_args(argv)
    if a.text is None:
        import sys
        if not sys.stdin.isatty():
            a.text = sys.stdin.read().strip()
        else:
            a.text = input("Enter text to generate: ")
    generate(generation_text=a.text, duration=a.duration, estimate_duration=a.estimate_duration, model_name=a.model,
             ref_audio_path=a.ref_audio, ref_audio_text=a.ref_text, steps=a.steps, method=a.method, cfg_strength=a.cfg,
             sway_sampling_coef=a.sway_coef, speed=a.speed, seed=a.seed, quantization_bits=a.q, output_path=a.output)


if __name__ == "__main__":
    main()
