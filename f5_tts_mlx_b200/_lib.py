"""ctypes binding of libf5b200.so (the C ABI declared in include/f5_b200.h).

There is no fallback: if the shared object is missing the import of any compute module raises, and
if no sm_90 GPU is present every entry point returns F5_ERR_NO_DEVICE which `check()` turns into a
RuntimeError.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import os as _os

# F5_LIB: an alternative build of the SAME library (A/B measurements of kernel variants); default: the in-tree build
_LIB_PATH = Path(_os.environ["F5_LIB"]) if _os.environ.get("F5_LIB") else Path(__file__).resolve().parent / "libf5b200.so"
_lib = None


class F5Error(RuntimeError):
    pass


def lib_path() -> Path:
    return _LIB_PATH


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise F5Error(
                f"{_LIB_PATH} is missing: build it with `python -m f5_tts_mlx_b200.build` "
                "(nvcc, sm_90a). This package has no CPU / PyTorch fallback."
            )
        _lib = C.CDLL(str(_LIB_PATH))
        _lib.f5_last_error.restype = C.c_char_p
        _declare(_lib)
    return _lib


def check(code: int) -> None:
    if code != 0:
        msg = load().f5_last_error().decode("utf-8", "replace")
        raise F5Error(f"libf5b200 error {code}: {msg}")


class GemmArgs(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("lda", C.c_int64),
        ("w", C.c_void_p), ("ldw", C.c_int64),
        ("m", C.c_int32), ("n", C.c_int32), ("k", C.c_int32),
        ("rows_per_batch", C.c_int32), ("num_batches", C.c_int32), ("batched_tiles", C.c_int32),
        ("conv_taps", C.c_int32), ("conv_pad", C.c_int32), ("conv_grouped", C.c_int32),
        ("act", C.c_int32), ("out_bf16", C.c_int32),
        ("bias", C.c_void_p),
        ("out", C.c_void_p), ("ldo", C.c_int64),
        ("resid", C.c_void_p), ("ldr", C.c_int64),
        ("gate", C.c_void_p), ("gate_ld", C.c_int64),
        ("row_len", C.c_void_p),
        ("rope", C.c_void_p), ("rope_cols", C.c_int32),
        ("q_scale", C.c_float), ("q_cols", C.c_int32),
        ("tile_n", C.c_int32),
        ("out2_bf16", C.c_void_p), ("ldo2", C.c_int64),
        ("variant", C.c_int32), ("w_static", C.c_int32),
        ("debug_ts", C.c_void_p),
        ("prefetch", C.c_void_p), ("prefetch_bytes", C.c_int64),
        ("ln_scale", C.c_void_p), ("ln_stats", C.c_void_p), ("ln_in_stats", C.c_void_p),
        ("ln_tab", C.c_void_p), ("ln_tab_ld", C.c_int64),
        ("ab_fp8", C.c_int32), ("out2_fp8", C.c_int32), ("acc_scale", C.c_float), ("out_fp8", C.c_int32),
    ]


class DitDims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("dim", "depth", "heads", "ff_inner", "mel_dim", "text_dim", "conv_layers",
                                         "text_num_embeds")]


class DitShape(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("batch", "frames", "cfg", "n_times", "text_len_max", "masked", "fused_adaln",
                                         "bucketed")]


TENSOR_LOOKUP = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_char_p, C.POINTER(C.c_int64))


# exported symbols -> (restype, argtypes); tests check that every one of these resolves
SYMBOLS: dict[str, tuple] = {
    "f5_last_error": (C.c_char_p, []),
    "f5_abi_version": (C.c_int, []),
    "f5_device_check": (C.c_int, []),
    "f5_struct_sizes": (C.c_int, [C.POINTER(C.c_int32), C.c_int32]),
    "f5_launch_count": (C.c_longlong, []),
    "f5_prof_enable": (C.c_int, [C.c_int]),
    "f5_prof_summary": (C.c_int, [C.POINTER(C.c_double), C.c_int]),
    "f5_prof_graph_begin": (C.c_int, [C.c_void_p, C.c_int32]),
    "f5_prof_graph_meta": (C.c_int, [C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int32]),
    "f5_gemm_bf16": (C.c_int, [C.POINTER(GemmArgs), C.c_void_p]),
    "f5_debug_gemm_ts": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32]),
    "f5_debug_attention_ts": (C.c_int, [C.c_void_p]),
    "f5_attention_fwd": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                   C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "f5_attention_fwd_e4m3": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "f5_ln_modulate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                 C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "f5_dwconv7_ln": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "f5_grn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                         C.c_int32, C.c_void_p]),
    "f5_dit_precompute": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "f5_dit_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "f5_dit_ln_tab_ld": (C.c_int64, [C.c_void_p]),
    "f5_ode_eval_times": (C.c_int, [C.POINTER(C.c_float), C.c_int32, C.c_int32, C.POINTER(C.c_float), C.c_int32]),
    "f5_duration_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "f5_mel_forward": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_int32, C.c_void_p]),
    "f5_istft": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                           C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "f5_vocos_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "f5_ode_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_int32, C.c_int32, C.c_float,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "f5_packed_weights_bytes": (C.c_int64, [C.POINTER(DitDims)]),
    "f5_pack_weights": (C.c_int, [C.POINTER(DitDims), TENSOR_LOOKUP, C.c_void_p, C.c_void_p]),
    "f5_bind_packed_weights": (C.c_int, [C.POINTER(DitDims), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "f5_workspace_bytes": (C.c_int64, [C.POINTER(DitDims), C.POINTER(DitShape)]),
    "f5_bind_workspace": (C.c_int, [C.POINTER(DitDims), C.POINTER(DitShape), C.c_void_p, C.c_void_p, C.c_void_p]),
    "f5_nccl_broadcast_weights": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
}


def _declare(lib: C.CDLL) -> None:
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
