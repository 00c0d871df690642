"""-m gpu: the split drain of each CTA's last GEMM tile (gemm_sm90.cuh) changes no output bit.

At BN = 128 the persistent GEMM drains the CTA's last tile on both consumer warpgroups, one 64-column unit each (the
RoPE instantiation excepted: there both runs take the single-warpgroup drain).  Every
instantiation of the many-waves table (test_gpu_gemm_persistent.WAVES: both dispatchers, BN 64 and 128, bf16, per-tensor
and block-scaled FP8, RoPE, GELU, Mish, fused-LN producer and consumer), plus the RMSNorm consumer and the plain-copy
producer of the UNetT, runs at grids whose CTAs own at most 1, 2 or 3 tiles.  Each launch runs twice, with the split
turned off (f5_gemm_test_tail_split(0): the owner alone drains the tile) and on; every output, second output, ln_stats
and e4m3 scale buffer must be bitwise equal, and the split run must also pass run_exact's known answers.
"""
import pytest
import torch

from kernel_check import bits, cdiv
from test_gpu_gemm_persistent import WAVES, wave_geometry
from test_gpu_kernel_exact import run_exact

pytestmark = pytest.mark.gpu

CASES = {
    **WAVES,
    "rms_qkv_64": dict(N=960, K=256, tile=64, rope=True, ln_rms=True, rows=("utt", 3)),
    "rms_qkv_128": dict(N=960, K=256, tile=128, rope=True, ln_rms=True, rows=("utt", 3)),
    "rms_ff1_128": dict(N=704, K=256, tile=128, act=1, ln_rms=True, rows="flat"),
    "unett_producer_128": dict(N=512, K=320, tile=128, resid="alias", out="f32", out2="bf16", ln_stats=True, amax=1,
                               density=0.25, rows="flat"),
}
OUTPUTS = ("out2", "ln_stats", "out_scale", "out2_scale")


def sized(name: str, per_cta: int, sms: int) -> dict:
    """CASES[name] as run_exact arguments with tiles in ((per_cta - 1) sms, per_cta sms]: every CTA owns per_cta tiles
    or one fewer (per_cta = 1: a third of the SMs idle, as in the out-projection at batch 1), ragged M tails."""
    c = dict(CASES[name])
    rows = c.pop("rows")
    tiles_n = cdiv(c["N"], 64 if c.get("conv_grouped") else c["tile"])
    mt = cdiv(per_cta * sms - sms // 3, tiles_n)
    while True:
        if rows == "flat":
            c.update(M=mt * 128 - 37)
        elif rows[0] == "utt":
            rpb = (mt * 128 - 37) // rows[1]
            c.update(M=rows[1] * rpb, rpb=rpb, nb=rows[1])
        else:
            rpb = cdiv(mt, rows[1]) * 128 - 50
            c.update(M=rows[1] * rpb, rpb=rpb, nb=rows[1], batched=True)
        if CASES[name].get("a_scale_ld") == -1:     # A's scales in a [K/64][M] buffer
            c["a_scale_ld"] = c["M"]
        if wave_geometry(c, sms)["tiles"] <= per_cta * sms:
            break
        mt -= 1
    c["w_static"] = per_cta % 2
    c["seed"] = 300 + 7 * list(CASES).index(name) + per_cta
    return c


@pytest.mark.parametrize("per_cta", [1, 2, 3])
@pytest.mark.parametrize("name", list(CASES))
def test_split_drain_is_bitwise_the_single_warpgroup_drain(name, per_cta, monkeypatch):
    from f5_tts_mlx_b200 import _lib, ops
    lib = _lib.load()
    S = torch.cuda.get_device_properties(0).multi_processor_count
    c = sized(name, per_cta, S)
    geo = wave_geometry(c, S)
    assert geo["per_cta"][1] == per_cta and geo["tiles"] > (per_cta - 1) * S, geo
    gemm = ops.gemm
    launches = []

    def gemm_both(a, w, out, **kw):
        outs = [out] + [kw[k] for k in OUTPUTS if kw.get(k) is not None]
        before = [t.clone() for t in outs]          # the out-proj form updates its residual in place
        prev = lib.f5_gemm_test_tail_split(0)
        try:
            gemm(a, w, out, **kw)
            torch.cuda.synchronize()
        finally:
            lib.f5_gemm_test_tail_split(prev)
        alone = [t.clone() for t in outs]
        for t, b in zip(outs, before):
            t.copy_(b)
        gemm(a, w, out, **kw)
        torch.cuda.synchronize()
        for i, (t, want) in enumerate(zip(outs, alone)):
            what = "out" if i == 0 else [k for k in OUTPUTS if kw.get(k) is not None][i - 1]
            assert torch.equal(bits(t.contiguous()), bits(want.contiguous())), \
                f"{name} at {per_cta} tile(s) per CTA ({geo}): {what} differs with the split drain"
        launches.append(geo)

    monkeypatch.setattr(ops, "gemm", gemm_both)
    assert lib.f5_gemm_test_tail_split(1) == 1      # on by default
    run_exact(**c)
    assert launches
