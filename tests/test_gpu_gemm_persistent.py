"""-m gpu: known-answer tests of the wgmma GEMM at launches with more output tiles than the GPU has SMs.

The production launches at batch 1 fit in about one wave of 128 x BN tiles; batched requests and the convolutions do
not.  These cases size the problem from the SM count so that every CTA of a one-CTA-per-SM launch would own 2, 3 or 8+
tiles, exactly one, or one tile more than the SMs, with ragged M / N tails, and so that an in-place residual, a fused-LN
producer and a 31-tap grouped convolution run over many waves.  Operands are small integers (run_exact of
test_gpu_kernel_exact): every output must equal the float64 reference bitwise, whatever the order in which tiles run.
"""
import pytest
import torch
import torch.nn.functional as F

from kernel_check import Guarded, assert_exact, gemm_tiles
from test_gpu_kernel_exact import DEV, ints, round_to, run_exact

pytestmark = pytest.mark.gpu


def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("per_sm", [2, 3, 9])
def test_many_tiles_per_sm_ragged(per_sm, tile):
    """per_sm x SMs tiles (or a few more) with a 40-column N tail and a 37-row M tail."""
    nt = 8
    N = nt * tile - 40
    mt = cdiv(per_sm * sms(), nt)
    run_exact(M=mt * 128 - 37, N=N, K=192, tile=tile, w_static=per_sm % 2, seed=per_sm)


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("extra", [0, 1])
def test_sm_count_tiles(extra, tile):
    """Exactly SMs tiles (one column tile, SMs row tiles), then one more row tile holding a single row."""
    run_exact(M=sms() * 128 + extra, N=56, K=128, tile=tile, w_static=1, out="f32", seed=10 + extra)


@pytest.mark.parametrize("tile", [64, 128])
def test_in_place_residual_over_many_waves(tile):
    """Out-projection / FF2 form over >= 3 tiles per SM: fp32 stream updated in place (each tile reads its residual
    before any store to it), shared gate, row mask, bf16 operand and LN statistics of the next block."""
    N = 1024
    rpb = cdiv(3 * sms(), N // tile) * 64 + 5          # two utterances, each ending mid-tile
    run_exact(M=2 * rpb, N=N, K=256, tile=tile, w_static=1, rpb=rpb, nb=2, row_len=True, gate="shared",
              resid="alias", out="f32", out2="bf16", ln_scale=True, amax=1, density=0.125, seed=20)


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("form", ["qkv_rope", "fp8_qkv_rope", "fp8_out_proj", "fp8_e4m3_out"])
def test_block_forms_over_many_waves(form, tile):
    """The block GEMMs' epilogue forms at >= 3 tiles per SM, batched rows (tiles never straddle utterances)."""
    N = {"qkv_rope": 768, "fp8_qkv_rope": 768, "fp8_out_proj": 512, "fp8_e4m3_out": 512}[form]
    rt = cdiv(3 * sms(), N // tile)
    rpb = cdiv(rt, 3) * 128 - 17
    kw = dict(M=3 * rpb, N=N, K=256, tile=tile, w_static=1, rpb=rpb, nb=3, batched=True, seed=30)
    if form == "qkv_rope":
        kw.update(rope=True, amax=2)
    elif form == "fp8_qkv_rope":
        kw.update(rope=True, ab8=True, density=0.5)
    elif form == "fp8_out_proj":
        kw.update(row_len=True, gate="shared", resid="alias", out="f32", out2="e4m3", ln_scale=True, ab8=True,
                  density=0.125)
    else:
        kw.update(ab8=True, out="e4m3", density=0.25)
    run_exact(**kw)


@pytest.mark.parametrize("ws", [0, 1])
def test_grouped_conv31_many_waves(ws):
    """The conv position embedding's grouped Conv1d(k=31, pad 15) over three utterances whose row tiles spread over
    >= 3 tiles per SM, the last row tile of each utterance ragged."""
    from f5_tts_mlx_b200 import ops
    Cc, B = 256, 3
    NF = cdiv(3 * sms(), B * (Cc // 64)) * 128 - 50
    x = ints((B * NF, Cc), 4, 41)
    wt = ints((Cc, 64, 31), 2, 42)
    wp = wt.permute(0, 2, 1).reshape(Cc, 31 * 64).contiguous()
    bias = ints((Cc,), 8, 43, dtype=torch.float32)
    g = Guarded(B * NF, Cc, torch.bfloat16, DEV)
    ops.gemm(x, wp, g.view, n=Cc, k=64, bias=bias, rows_per_batch=NF, num_batches=B, batched_tiles=True,
             conv_taps=31, conv_pad=15, conv_grouped=True, w_static=bool(ws))
    torch.cuda.synchronize()
    ref = F.conv1d(x.double().view(B, NF, Cc).transpose(1, 2), wt.double(), bias.double(), padding=15, groups=Cc // 64)
    assert_exact(g.view, round_to(ref.transpose(1, 2).reshape(B * NF, Cc), torch.bfloat16), gemm_tiles(64, NF, True),
                 "conv31")
    g.check("conv31 guard")
