"""Sample-rate conversion without a GPU: the float64 restatement (tests/resample_emul.py) against
torchaudio.functional.resample, the library's host table (f5_resample_table) against the restatement, the C entry
point's refusal to run without a device, and the WAV reader on hand-built files."""
import ctypes as C
import math
import struct

import numpy as np
import pytest
import torch

import resample_emul as E
from f5_tts_mlx_b200 import _lib

torchaudio = pytest.importorskip("torchaudio")

RATES = [8000, 11025, 16000, 22050, 32000, 44100, 48000, 88200, 96000]
PAIRS = [(r, 24000) for r in RATES] + [(24000, r) for r in RATES]
PAIR_IDS = [f"{o}-{n}" for o, n in PAIRS]


def lengths(orig, new):
    O, _, _, taps, _ = E.geometry(orig, new)
    odd = 7 * O + 3 if O > 1 else 1001                 # not a multiple of O (every length is one when O = 1)
    return [1, 5, taps - 1, odd]


@pytest.mark.parametrize("orig,new", PAIRS, ids=PAIR_IDS)
def test_emulation_matches_torchaudio_float64(orig, new):
    g = torch.Generator().manual_seed(orig + new)
    for L in lengths(orig, new):
        x = torch.randn(2, L, generator=g, dtype=torch.float64)
        ref = torchaudio.functional.resample(x, orig, new).numpy()
        got = E.resample(x.numpy(), orig, new)
        assert got.shape == ref.shape == (2, math.ceil(new * L / orig)), (L, got.shape, ref.shape)
        assert np.abs(got - ref).max() <= 1e-12, (L, np.abs(got - ref).max())


def test_emulation_identity_and_table_sizes():
    x = np.random.default_rng(0).standard_normal(100)
    assert np.array_equal(E.resample(x, 24000, 24000), x)
    # N x taps of the pairs the header's limit is stated for
    assert E.table(48000, 24000).shape == (1, 28)
    assert E.table(44100, 24000).shape == (80, 171)
    assert E.table(22050, 24000).shape == (160, 161)
    assert max(E.table(o, n).size for o, n in PAIRS) <= 1 << 16


def _c_table(orig, new):
    lib = _lib.load()
    n = lib.f5_resample_table(orig, new, None, 0)
    assert n > 0, lib.f5_last_error()
    buf = (C.c_float * n)()
    assert lib.f5_resample_table(orig, new, None, n) == n            # size query leaves nothing written
    assert lib.f5_resample_table(orig, new, buf, n - 1) == n         # too small a buffer: size only
    assert not any(buf)
    assert lib.f5_resample_table(orig, new, buf, n) == n
    return np.frombuffer(buf, dtype=np.float32).copy()


@pytest.mark.parametrize("orig,new", PAIRS, ids=PAIR_IDS)
def test_c_table_equals_emulation_to_one_ulp(orig, new):
    ref = E.table(orig, new)
    got = _c_table(orig, new)
    assert got.size == ref.size
    ref32 = ref.reshape(-1).astype(np.float32)
    ulp = np.spacing(np.abs(ref32)).astype(np.float64)
    # fp32 rounding of the same double computation: within one ulp of the float64 value's fp32 rounding
    assert np.all(np.abs(got.astype(np.float64) - ref32.astype(np.float64)) <= ulp), \
        np.abs(got.astype(np.float64) - ref32).max()


def test_c_table_rejects_bad_rates():
    lib = _lib.load()
    for orig, new in [(0, 24000), (24000, 0), (-8000, 24000), (24000, -1)]:
        assert lib.f5_resample_table(orig, new, None, 0) == -1        # F5_ERR_INVALID
        assert b"positive" in lib.f5_last_error()
    # coprime rates: N x taps far beyond the stated limit
    assert lib.f5_resample_table(44101, 24000, None, 0) == -1
    assert b"table" in lib.f5_last_error()
    assert lib.f5_resample_table(24000, 24000, None, 0) == 0          # the identity has no filter


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_resample_has_no_cpu_path():
    lib = _lib.load()
    assert lib.f5_resample(None, 1, 100, 44100, 24000, None, None, 55, None) == -3     # F5_ERR_NO_DEVICE
    from f5_tts_mlx_b200 import resample
    with pytest.raises(_lib.F5Error):
        resample(torch.zeros(100), 44100, 24000)


def test_generate_refuses_other_rates_without_the_option(tmp_path):
    from f5_tts_mlx_b200 import generate as G

    class Model:                                      # never reached: the rate check comes first
        _duration_predictor = None
        _vocoder = staticmethod(lambda mel: mel)

        class transformer:
            device = torch.device("cpu")

        def sample(self, *a, **k):
            raise AssertionError("sample() must not run")

    path = tmp_path / "clip44k.wav"
    path.write_bytes(wav_bytes(np.zeros((441, 1)), "s16", 44100))
    with pytest.raises(ValueError, match="sample rate of 24kHz"):
        G.generate("Hello.", duration=2.0, ref_audio_path=str(path), f5tts=Model())


# ---------------------------------------------------------------- read_wav
def wav_bytes(codes: np.ndarray, kind: str, sr: int, extensible: bool = False) -> bytes:
    """A WAV file written field by field with struct: codes [frames, channels] are integer sample codes (float
    values for f32)."""
    bits = {"u8": 8, "s16": 16, "s24": 24, "s32": 32, "f32": 32, "f64": 64}[kind]
    tag = 3 if kind in ("f32", "f64") else 1
    ch = codes.shape[1]
    block = ch * bits // 8
    if kind == "u8":
        data = struct.pack(f"<{codes.size}B", *codes.reshape(-1).astype(int))
    elif kind == "s16":
        data = struct.pack(f"<{codes.size}h", *codes.reshape(-1).astype(int))
    elif kind == "s24":
        data = b"".join(struct.pack("<i", int(v))[:3] for v in codes.reshape(-1))
    elif kind == "s32":
        data = struct.pack(f"<{codes.size}i", *codes.reshape(-1).astype(int))
    elif kind == "f32":
        data = struct.pack(f"<{codes.size}f", *codes.reshape(-1))
    else:
        data = struct.pack(f"<{codes.size}d", *codes.reshape(-1))
    if extensible:
        guid_tail = b"\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"
        fmt = struct.pack("<HHIIHHHHI", 0xFFFE, ch, sr, sr * block, block, bits, 22, bits, 0) \
            + struct.pack("<H", tag) + guid_tail
    else:
        fmt = struct.pack("<HHIIHH", tag, ch, sr, sr * block, block, bits)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt
    body += b"LIST" + struct.pack("<I", 5) + b"INFOx" + b"\x00"      # an odd-sized chunk before the data, padded
    body += b"data" + struct.pack("<I", len(data)) + data + (b"\x00" if len(data) & 1 else b"")
    return b"RIFF" + struct.pack("<I", len(body)) + body


CODES = {
    "u8": (np.array([0, 1, 127, 128, 129, 200, 255]), lambda c: (c - 128) / 128),
    "s16": (np.array([-32768, -1, 0, 1, 12345, 32767, -20000]), lambda c: c / 32768),
    "s24": (np.array([-8388608, -1, 0, 1, 4660803, 8388607, -123457]), lambda c: c / 8388608),
    "s32": (np.array([-2147483648, -1, 0, 1, 305419896, 2147483647, -98765432]), lambda c: c / 2147483648),
    "f32": (np.array([-1.0, -0.25, 0.0, 1e-3, 0.5, 1.0, 0.7071067690849304]), lambda c: c),
}


@pytest.mark.parametrize("extensible", [False, True], ids=["plain", "extensible"])
@pytest.mark.parametrize("kind", sorted(CODES))
def test_read_wav_decodes_hand_built_files_exactly(kind, extensible, tmp_path):
    from f5_tts_mlx_b200.generate import read_wav
    codes, scale = CODES[kind]
    expect_mono = np.array([scale(float(c)) for c in codes], dtype=np.float64).astype(np.float32)
    p = tmp_path / "mono.wav"
    p.write_bytes(wav_bytes(codes[:, None], kind, 44100, extensible))
    x, sr = read_wav(str(p))
    assert sr == 44100 and x.dtype == torch.float32
    assert np.array_equal(x.numpy(), expect_mono), (x.numpy(), expect_mono)
    # stereo: channels averaged in fp32
    right = codes[::-1].copy()
    p.write_bytes(wav_bytes(np.stack([codes, right], 1), kind, 22050, extensible))
    x, sr = read_wav(str(p))
    r32 = np.array([scale(float(c)) for c in right], dtype=np.float64).astype(np.float32)
    assert sr == 22050 and np.array_equal(x.numpy(), np.stack([expect_mono, r32], 1).mean(axis=1))


def test_read_wav_16_bit_decodes_as_before(tmp_path):
    """16-bit PCM written by the stdlib wave module decodes as x / 32768, exactly as the wave-module reader did."""
    import wave as wavmod
    from f5_tts_mlx_b200.generate import read_wav
    pcm = np.random.default_rng(1).integers(-32768, 32768, size=(999, 2)).astype(np.int16)
    with wavmod.open(str(tmp_path / "a.wav"), "wb") as f:
        f.setnchannels(2); f.setsampwidth(2); f.setframerate(24000); f.writeframes(pcm.tobytes())
    x, sr = read_wav(str(tmp_path / "a.wav"))
    expect = (pcm.reshape(-1).astype(np.float32) / 32768.0).reshape(-1, 2).mean(axis=1)
    assert sr == 24000 and np.array_equal(x.numpy(), expect)


@pytest.mark.parametrize("kind,extensible", [("f64", False), ("f64", True)])
def test_read_wav_refuses_64_bit_float(kind, extensible, tmp_path):
    from f5_tts_mlx_b200.generate import read_wav
    p = tmp_path / "f64.wav"
    p.write_bytes(wav_bytes(np.zeros((4, 1)), kind, 48000, extensible))
    with pytest.raises(ValueError, match="IEEE float, 64 bits"):
        read_wav(str(p))


def test_read_wav_refuses_compressed_formats(tmp_path):
    from f5_tts_mlx_b200.generate import read_wav
    # IMA ADPCM (tag 0x0011), 4 bits per sample
    fmt = struct.pack("<HHIIHHHH", 0x0011, 1, 8000, 4055, 256, 4, 2, 505)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", 256) + bytes(256)
    p = tmp_path / "adpcm.wav"
    p.write_bytes(b"RIFF" + struct.pack("<I", len(body)) + body)
    with pytest.raises(ValueError, match="format tag 0x0011"):
        read_wav(str(p))
    p.write_bytes(b"not a wav file at all")
    with pytest.raises(ValueError, match="RIFF"):
        read_wav(str(p))
