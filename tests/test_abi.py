"""The C-ABI library loads, exports every symbol include/f5_b200.h declares, its struct layouts
match the ctypes mirrors, and — on a box without a GPU — every compute entry point fails loudly
instead of falling back to a CPU path.  No compute calls are made here."""
import ctypes as C
import os
import re

import pytest
import torch

from f5_tts_mlx_b200 import _lib
from f5_tts_mlx_b200.dit import DitBuffersC
from f5_tts_mlx_b200.duration import DurationBuffersC, DurationWeightsC
from f5_tts_mlx_b200.vocos import VocosBlockWeightsC, VocosBuffersC, VocosWeightsC
from f5_tts_mlx_b200.weights import ConvNextWeightsC, DitBlockWeightsC, DitWeightsC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "f5_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(f5_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_are_exported_and_bound():
    lib = _lib.load()
    names = declared_symbols()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/f5_b200.h but not exported by libf5b200.so"
        assert n in _lib.SYMBOLS, f"{n} has no ctypes prototype in _lib.SYMBOLS"
    for n in _lib.SYMBOLS:
        assert n in names, f"{n} bound in _lib.py but not declared in the header"


def test_struct_layouts_match_ctypes():
    lib = _lib.load()
    out = (C.c_int32 * 10)()
    assert lib.f5_struct_sizes(out, 10) == 10
    mirrors = [_lib.GemmArgs, ConvNextWeightsC, DitBlockWeightsC, DitWeightsC, DitBuffersC, VocosBlockWeightsC,
               VocosWeightsC, VocosBuffersC, DurationWeightsC, DurationBuffersC]
    for got, m in zip(list(out), mirrors):
        assert got == C.sizeof(m), f"{m.__name__}: C sizeof {got} != ctypes {C.sizeof(m)}"


def test_abi_version():
    assert _lib.load().f5_abi_version() >= 1000


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_no_cpu_fallback_entry_points_fail_loudly():
    lib = _lib.load()
    assert lib.f5_device_check() == -3                     # F5_ERR_NO_DEVICE
    g = _lib.GemmArgs()
    assert lib.f5_gemm_bf16(C.byref(g), None) == -3
    assert b"no CPU fallback" in lib.f5_last_error() or b"sm_90a" in lib.f5_last_error()
    assert lib.f5_attention_fwd(None, 0, None, 0, 1, 1, 1, 64, None, None) == -3
    assert lib.f5_dit_forward(None, None, 0, None) == -3
    assert lib.f5_mel_forward(None, 1, 1, None, None, 100, 256, None, 1, None) == -3
    assert lib.f5_vocos_decode(None, None, None, None, None) == -3
    with pytest.raises(_lib.F5Error):
        _lib.check(lib.f5_device_check())


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_python_surface_refuses_cpu_tensors():
    from f5_tts_mlx_b200 import MelSpec
    with pytest.raises(_lib.F5Error):
        MelSpec()(torch.zeros(2048))


def test_product_package_never_imports_the_oracle():
    """oracle/ is test infrastructure: the product path must not route through it."""
    pkg = os.path.join(ROOT, "f5_tts_mlx_b200")
    pat = re.compile(r"^\s*(from\s+oracle|import\s+oracle)", re.M)
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, fn)).read()
                assert not pat.search(src), f"{fn} imports the oracle"


def test_library_reads_no_environment_variables():
    """What the library computes depends on its arguments alone: no environment variable selects another code path
    that the tests and the benchmark never run."""
    csrc = os.path.join(ROOT, "f5_tts_mlx_b200", "csrc")
    srcs = sorted(os.listdir(csrc))
    assert any(fn.endswith(".cu") for fn in srcs)
    for fn in srcs:
        src = open(os.path.join(csrc, fn)).read()
        assert not re.search(r"\bgetenv\b", src), f"csrc/{fn} calls getenv"


def test_header_is_plain_c99_and_links_from_c(tmp_path):
    """include/f5_b200.h compiles as strict C99 and a C program links against libf5b200.so: the boundary has no
    C++ or torch types.  The consumer also checks that the C compiler's struct layout equals the library's."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    _lib.load()                                            # builds the library if needed
    pkg = os.path.join(ROOT, "f5_tts_mlx_b200")
    exe = str(tmp_path / "consumer")
    cmd = [gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi", "consumer.c"), "-o", exe, "-L", pkg, "-l:libf5b200.so",
           f"-Wl,-rpath,{pkg}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "abi=" in r.stdout and "structs=10" in r.stdout
    if not torch.cuda.is_available():
        assert "device_check=-3" in r.stdout and "gemm_rc=-3" in r.stdout     # F5_ERR_NO_DEVICE, no CPU fallback


# ---------------- host utilities for non-Python hosts (f5_pack_weights / f5_workspace_bytes) ----------------
def _dims(cfg):
    d = _lib.DitDims()
    d.dim, d.depth, d.heads, d.ff_inner, d.mel_dim = cfg.dim, cfg.depth, cfg.heads, cfg.ff_inner, cfg.mel_dim
    d.text_dim, d.conv_layers, d.text_num_embeds = cfg.text_dim, cfg.conv_layers, cfg.text_num_embeds
    return d


def test_c_weight_packer_matches_the_python_pack_byte_for_byte():
    """f5_pack_weights (C, callback over MLX-named fp32 host tensors) produces the same packed buffer as
    weights.PackedDiT.load: same layout, same fused / re-laid-out matrices, same bf16 rounding — except the text
    position table, whose cos/sin come from libm instead of torch (compared to 1e-6)."""
    import numpy as np
    from f5_tts_mlx_b200.weights import DiTConfig, PackedDiT, random_dit_weights
    lib = _lib.load()
    cfg = DiTConfig(dim=256, depth=2, heads=4, text_num_embeds=40, text_dim=128, conv_layers=2)
    W = random_dit_weights(cfg, seed=5)
    ref = PackedDiT(cfg, "cpu").load(W)
    d = _dims(cfg)
    assert lib.f5_packed_weights_bytes(C.byref(d)) == ref.nbytes
    keep = {k: v.detach().float().contiguous() for k, v in W.items()}
    asked = []

    @_lib.TENSOR_LOOKUP
    def get(user, name, numel):
        t = keep.get(name.decode())
        asked.append(name.decode())
        if t is None:
            return None
        numel[0] = t.numel()
        return t.data_ptr()

    out = torch.zeros(ref.nbytes, dtype=torch.uint8)
    assert lib.f5_pack_weights(C.byref(d), get, None, C.c_void_p(out.data_ptr())) == 0, lib.f5_last_error()
    pos = ref.specs["text_pos"]
    n_pos = 4096 * cfg.text_dim * 4
    mask = torch.ones(ref.nbytes, dtype=torch.bool); mask[pos.offset:pos.offset + n_pos] = False
    assert torch.equal(out[mask], ref.buffer[mask])
    a = out[pos.offset:pos.offset + n_pos].view(torch.float32); b = ref.buffer[pos.offset:pos.offset + n_pos].view(torch.float32)
    assert (a - b).abs().max().item() < 1e-6
    assert len(set(asked)) > 40
    # a missing tensor is an error with the tensor's name in it, not a silent zero
    del keep["transformer.proj_out.weight"]
    assert lib.f5_pack_weights(C.byref(d), get, None, C.c_void_p(out.data_ptr())) == -1
    assert b"transformer.proj_out.weight" in lib.f5_last_error()
    # binding: every pointer of f5_dit_weights lands at the offset the Python side uses
    from f5_tts_mlx_b200.weights import ConvNextWeightsC, DitBlockWeightsC, DitWeightsC
    w = DitWeightsC(); tbs = (ConvNextWeightsC * cfg.conv_layers)(); blks = (DitBlockWeightsC * cfg.depth)()
    base = 1 << 20
    assert lib.f5_bind_packed_weights(C.byref(d), C.c_void_p(base), C.byref(w), tbs, blks) == 0
    assert w.mod_w - base == ref.specs["mod_w"].offset and blks[1].ff2_w - base == ref.specs["blk1.ff2_w"].offset
    assert tbs[1].grn_beta - base == ref.specs["tb1.grn_beta"].offset and w.proj_b - base == ref.specs["proj_b"].offset
    assert w.ct_ld == ref.ct_ld and w.text_rows == cfg.text_num_embeds + 1


def test_workspace_bytes_covers_the_python_session():
    """f5_workspace_bytes >= the bytes dit.DitSession allocates for the same shape (each buffer 256-byte aligned)."""
    from f5_tts_mlx_b200.weights import BASE_CONFIG
    lib = _lib.load()
    d = _dims(BASE_CONFIG)
    s = _lib.DitShape()
    s.batch, s.frames, s.cfg, s.n_times, s.text_len_max, s.masked, s.fused_adaln, s.bucketed = 1, 937, 1, 31, 152, 0, 1, 0
    got = lib.f5_workspace_bytes(C.byref(d), C.byref(s))
    D, F, Ct, R, T = 1024, 2048, 512, 2 * 937, 31
    NM, ld = 22 * 6 * D + 2 * D, 22 * (3 * D + F) + 128
    expect = (R * D * 4 * 3 + R * D * 2 * 2 + R * 3 * D * 2 + R * F * 2 + R * 100 * 4 + R * 128 * 2 + R * 640 * 2      # x,h,hoist / a,c / qkv / ff / v / y / ct
              + R * Ct * 4 + R * Ct * 2 + 2 * R * 2 * Ct * 2 + 2 * 31 * 2 * Ct * 4                                       # text path
              + T * NM * 4 + T * D * 2 + R * 16 * 2 * 4 + 4 * T * ld * 4 + 45 * 4 * T * D * 2                              # mod table, LN tables
              + 152 * 4 + 2 * 4 + 937 * 100 * 4 + T * 4 + 937 * 64 * 4)
    assert expect <= got <= expect + 40 * 256
    s.fused_adaln = 0
    assert lib.f5_workspace_bytes(C.byref(d), C.byref(s)) < got - 4 * T * ld * 4
    s.batch = 0
    assert lib.f5_workspace_bytes(C.byref(d), C.byref(s)) == -1


@pytest.mark.parametrize("src", ["gemm.cu", "attention.cu"])
def test_wgmma_kernels_compile_without_serialization(src, tmp_path):
    """ptxas serialises every wgmma of a kernel when the wgmma pipeline crosses a function call (warning C7510) — e.g.
    a printf on a wait path between MMA issue and wait.  The tensor-core kernels must compile without it."""
    import subprocess
    from f5_tts_mlx_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-cubin", os.path.join(ROOT, "f5_tts_mlx_b200", "csrc", src),
           "-o", str(tmp_path / "k.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    assert "C7510" not in log and "serialized" not in log, [l for l in log.splitlines() if "C7510" in l][:3]
