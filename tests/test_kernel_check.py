"""CPU: the element-wise checkers of kernel_check.py accept a correct result and reject, naming the right tile, the
mistakes kernels make; and every GEMM instantiation gemm.cu builds has a GPU test at each tile width that reaches it."""
import re
from pathlib import Path

import pytest
import torch

from kernel_check import (U32, Guarded, assert_exact, assert_within, attention_bound, attention_ref, attn_tiles,
                          gemm_acc_bound, gemm_tiles, out_bound, rope_bound, rope_ref)

ROOT = Path(__file__).resolve().parent.parent


def _operands(M=300, N=136, K=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).bfloat16()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).bfloat16()
    return a, w


def _fp32_matmul(a, w):
    return a.float() @ w.float().T


def _check(got, a, w, bn=64):
    ref = a.double() @ w.double().T
    b = out_bound(ref, gemm_acc_bound(a, w), torch.float32)
    return assert_within(got, ref, b, gemm_tiles(bn), "self-test")


def test_accepts_fp32_matmul():
    a, w = _operands()
    assert _check(_fp32_matmul(a, w), a, w) <= 1.0


def test_exact_accepts_integer_matmul_and_names_first_bad_element():
    g = torch.Generator().manual_seed(1)
    a = torch.randint(-8, 9, (300, 200), generator=g).bfloat16()
    w = torch.randint(-8, 9, (136, 200), generator=g).bfloat16()
    got = _fp32_matmul(a, w)
    want = (a.double() @ w.double().T).float()
    assert_exact(got, want, gemm_tiles(64), "exact")
    want[want == 0] = -0.0                   # signed zeros compare equal
    assert_exact(got, want, gemm_tiles(64), "exact")
    got[200, 70] += 1
    with pytest.raises(AssertionError, match=r"tile \(m 1, n 1\) row 200 col 70"):
        assert_exact(got, want, gemm_tiles(64), "exact")
    got[200, 70] -= 1
    got[5, 3] = 2.0 ** -140                  # a denormal is not zero
    want[5, 3] = 0.0
    with pytest.raises(AssertionError, match=r"row 5 col 3"):
        assert_exact(got, want, gemm_tiles(64), "exact")


def test_rejects_dropped_k_block():
    a, w = _operands()
    got = _fp32_matmul(a, w)
    r, c = slice(128, 256), slice(64, 128)
    got[r, c] -= a[r, 64:128].float() @ w[c, 64:128].float().T
    with pytest.raises(AssertionError, match=r"tile \(m 1, n 1\)"):
        _check(got, a, w)


def test_rejects_row_shift_in_tile_tail():
    a, w = _operands()
    got = _fp32_matmul(a, w)
    got[299] = got[298]               # last tile holds rows 256..299
    with pytest.raises(AssertionError, match=r"tile \(m 2, n \d\) row 299"):
        _check(got, a, w)


def test_rejects_swapped_columns():
    a, w = _operands()
    got = _fp32_matmul(a, w)
    got[:, [70, 71]] = got[:, [71, 70]]
    with pytest.raises(AssertionError, match=r"tile \(m \d, n 1\) row \d+ col 7[01]"):
        _check(got, a, w)


def test_rejects_rope_position_off_by_one():
    from f5_tts_mlx_b200.dit import rope_table
    a, w = _operands(M=300, N=192, K=128)
    tab = rope_table(301)
    pos = torch.arange(300)
    x = a.double() @ w.double().T
    bx = gemm_acc_bound(a, w) + U32 * x.abs()
    ref, b = rope_ref(x, tab, pos, 128), rope_bound(x, bx, tab, pos, 128)
    b = out_bound(ref, b, torch.float32)
    good = rope_ref(_fp32_matmul(a, w).double(), tab, pos, 128).float()
    assert_within(good, ref, b, gemm_tiles(64), "rope")
    bad_pos = pos.clone()
    bad_pos[128:256] += 1
    bad = rope_ref(_fp32_matmul(a, w).double(), tab, bad_pos, 128).float()
    with pytest.raises(AssertionError, match=r"tile \(m 1, n [01]\)"):
        assert_within(bad, ref, b, gemm_tiles(64), "rope")


def test_rejects_leaked_masked_key():
    B, N, H = 2, 300, 2
    g = torch.Generator().manual_seed(3)
    q, k, v = [(torch.randn(B, H, N, 64, generator=g) * s).bfloat16().float() for s in (0.4, 0.4, 1.0)]
    kv = torch.tensor([300, 200])
    o, pv, qk = attention_ref(q, k, v, kv)
    b = attention_bound(o, pv, qk, qk.max().item(), 3)
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(B * N, H * 64)
    got = flat(o).bfloat16()
    assert_within(got, flat(o), flat(b), attn_tiles(N), "attention")
    leak, _, _ = attention_ref(q, k, v, torch.tensor([300, 201]))
    bad = o.clone()
    bad[1, 1, 128:256] = leak[1, 1, 128:256]
    with pytest.raises(AssertionError, match=r"\(batch 1, head 1, q-tile 1\)"):
        assert_within(flat(bad).bfloat16(), flat(o), flat(b), attn_tiles(N), "attention")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.uint8])
def test_guard_detects_overwrite_and_unwritten(dtype):
    g = Guarded(10, 20, dtype, "cpu")
    assert g.view.stride(0) > 20
    g.view.zero_()
    g.check("clean")
    g.buf.view(torch.uint8)[0, 0] ^= 1       # one byte of the first guard row
    with pytest.raises(AssertionError, match="guard element overwritten at buffer row -3"):
        g.check("overwrite")
    g2 = Guarded(10, 20, dtype, "cpu")
    g2.view[:, :19].zero_()
    with pytest.raises(AssertionError, match="never written; first at row 0 col 19"):
        g2.check("unwritten")


# ---------------------------------------------------------------- instantiation coverage
_ACT = {"ACT_NONE": 0, "ACT_GELU_TANH": 1, "ACT_GELU_ERF": 2, "ACT_MISH": 3}
_B = {"true": True, "false": False}


def built_instantiations():
    """(ACT, OUT_BF16, ROPE, FP8, RESID) of every launch_gemm instantiation dispatch_epi (gemm.cu) can reach."""
    src = (ROOT / "f5_tts_mlx_b200" / "csrc" / "gemm.cu").read_text()
    body = src[src.index("static int dispatch_epi"):]
    body = body[:body.index("\n}\n")]
    out = set()
    for m in re.finditer(r"launch_gemm<BN, kStages, (ACT_\w+), (true|false), (true|false), (true|false), (true|false)>", body):
        out.add((_ACT[m[1]], _B[m[2]], _B[m[3]], _B[m[4]], _B[m[5]]))
    for m in re.finditer(r"^\s*F5_CASE(8?)\((ACT_\w+), (true|false), (true|false)\)", body, re.M):
        out.add((_ACT[m[2]], _B[m[3]], _B[m[4]], m[1] == "8", True))
    return out


def test_dispatch_parse_sees_every_instantiation():
    built = built_instantiations()
    assert len(built) == 14, sorted(built)
    assert (1, True, False, True, False) in built and (1, True, False, False, False) in built


def test_every_instantiation_has_gpu_cases_at_each_tile_width():
    import test_gpu_kernel_exact as ex
    import test_gpu_kernels as kn
    declared = set(ex.INSTANTIATIONS) | set(kn.INSTANTIATIONS)
    built = built_instantiations()
    # every declared case launches an instantiation that exists (the Python restatement of dispatch_epi is right)
    assert {d[:5] for d in declared} <= built, sorted({d[:5] for d in declared} - built)
    # every instantiation at both tile widths (only the grouped convolution is limited to 64, and none is grouped-only)
    missing = sorted((i, bn) for i in built for bn in (64, 128) if i + (bn,) not in declared)
    assert not missing, f"instantiations without a GPU case: {missing}"


def gemm_form(f: dict) -> tuple:
    """The form of one f5_gemm_bf16 launch, from its nonzero fields (names of f5_gemm_args): which optional inputs and
    outputs are set, the activation and output type, and how lda compares with k and ldo2 with n ('=' or '2x': half of
    a slot twice as wide)."""
    rel = lambda ld, x: "=" if ld == x else ("2x" if ld == 2 * x else ">")
    return (("bias", "bias" in f),
            ("resid", ("alias" if f["resid"] == f["out"] else "sep") if "resid" in f else None),
            ("act", int(f.get("act", 0))), ("out_bf16", "out_bf16" in f),
            ("rope", (int(f["rope_cols"]), int(f.get("rope_col2", 0)), int(f["q_cols"])) if "rope" in f else None),
            ("ln_rms", "ln_rms" in f), ("ln_stats", "ln_stats" in f), ("row_len", "row_len" in f),
            ("rows_per_batch", "rows_per_batch" in f), ("gate", "gate" in f), ("conv_taps", int(f.get("conv_taps", 1))),
            ("lda", rel(int(f["lda"]), int(f["k"]))),
            ("out2", rel(int(f["ldo2"]), int(f["n"])) if "out2_bf16" in f else None))


def case_form(c: dict) -> tuple:
    """gemm_form of a run_exact case (test_gpu_kernel_exact.UNETT): the fields unett.cu would set for it."""
    f = {"k": c["K"], "n": c["N"], "lda": 2 * c["K"] if c.get("a_slot") else c["K"], "out": "x"}
    if c.get("bias", True):
        f["bias"] = 1
    if c.get("resid"):
        f["resid"] = "x" if c["resid"] == "alias" else "r"
    if c.get("act"):
        f["act"] = c["act"]
    if c.get("out", "bf16") == "bf16":
        f["out_bf16"] = 1
    if c.get("rope"):
        f.update(rope=1, rope_cols=c["rope_cols"], rope_col2=c.get("rope_col2", 0), q_cols=c["q_cols"])
    for k in ("ln_rms", "ln_stats", "row_len", "gate"):
        if c.get(k):
            f[k] = 1
    if c.get("rpb"):
        f["rows_per_batch"] = c["rpb"]
    if c.get("out2"):
        f.update(out2_bf16=1, ldo2=2 * c["N"] if c.get("out2_slot") else c["N"])
    return gemm_form(f)


def _scale_dims(form: tuple, D: int) -> tuple:
    """A form with the rope column counts in units of the model width (the trace runs a narrower model than E2TTS_Base)."""
    d = dict(form)
    if d["rope"] is not None:
        rc, c2, qc = d["rope"]
        d["rope"] = (rc, c2 / D, qc / D)
    return tuple(d.items())


def test_every_unett_gemm_form_has_a_known_answer_case():
    """Every f5_gemm_bf16 launch of f5_unett_forward from the time token to proj_out (the UNetT's own launches; the input
    embedding is the DiT's, tested as test_gpu_kernel_exact.PROD) in every traced mode is the form of one of the
    declared UNETT cases.  A new UNetT launch form without a known-answer GPU case fails here."""
    import sys
    sys.path.insert(0, str(ROOT / "tests" / "golden"))
    import make_launch_trace as T
    import test_gpu_kernel_exact as ex
    declared = {_scale_dims(case_form(c), 1024): name for name, c in ex.UNETT.items()}
    seen = {}
    for header, lines in T.cases(T.launch_trace()):
        if not header.startswith("unett"):
            continue
        pack = re.search(r"launch_unett_time_pack\(.*\bD=(\d+)", "\n".join(lines))
        if pack is None:         # a case that stops before the forward (precompute alone, a refusal)
            continue
        D = int(pack[1])
        after = False
        for line in lines:
            if "launch_unett_time_pack(" in line:
                after = True
            elif after and line.startswith("  f5_gemm_bf16("):
                f = dict(re.findall(r"(\w+)=([^,()]+)", line[line.index("(") + 1:]))
                form = _scale_dims(gemm_form(f), D)
                assert form in declared, f"{header}: a UNetT GEMM form without a known-answer case:\n{line}\n{form}"
                seen[declared[form]] = True
                after = f["out"] != "ub.v"          # proj_out into v ends the forward
    assert set(seen) == set(ex.UNETT), f"declared UNETT cases the trace never launches: {set(ex.UNETT) - set(seen)}"


# BigVGAN's host code (bigvgan.cu f5_bigvgan_decode) is not traced: its GEMM forms, listed from the source, and the
# BIGVGAN cases of test_gpu_kernel_exact that launch each one.  (taps, dilation > 1, bf16 out, residual)
BIGVGAN_FORMS = {
    "conv_pre": (7, False, True, None),          # 7 taps over the mel padded to 128 columns, bf16 operand out
    "ups": ("polyphase", False, False, None),    # polyphase transposed conv, fp32 out
    "conv1": ("k", True, False, None),           # dilated conv, fp32 out
    "conv2_m0": ("k", False, False, "sep"),      # conv2 of m = 0: the stage input as residual
    "conv2_m12": ("k", False, False, "alias"),   # conv2 of m = 1, 2: resid == out, the stream updated in place
}


def test_bigvgan_gemm_forms_have_known_answer_cases():
    import test_gpu_kernel_exact as ex
    src = (ROOT / "f5_tts_mlx_b200" / "csrc" / "bigvgan.cu").read_text()
    # the launches BIGVGAN_FORMS restates are still the ones decode makes.  The lines are matched verbatim, so a mere
    # reformatting of f5_bigvgan_decode trips this too: then update the lines here after checking that the forms (taps,
    # dilation, output type, residual) are unchanged, or add a case to BIGVGAN and BIGVGAN_FORMS if one is new.
    for line in ("g.a = b->mel_bf16; g.lda = 128; g.w = w->conv_pre_w; g.ldw = 7 * 128;",
                 "g.conv_taps = 7; g.conv_pad = 3;",
                 "g.out_bf16 = 1; g.q_scale = 1.f;",
                 "conv(b->a_bf16, T, C, w->up_w[i], w->up_taps[i], w->up_pad[i], 1, w->up_b[i], u * Co, b->x_up, false,",
                 "conv(b->a_bf16, T, C, blk.conv1_w[m], k, (k * d - d) / 2, d, blk.conv1_b[m], C, b->t, false,",
                 "conv(b->a_bf16, T, C, blk.conv2_w[m], k, (k - 1) / 2, 1, blk.conv2_b[m], C, xj, false, xin)",
                 "xin = xj;"):
        assert line in src, line
    assert src.count("f5_gemm_bf16(&g, st)") == 2 and src.count("conv(b->a_bf16") == 3
    forms = {"conv_pre": [], "ups": [], "conv1": [], "conv2_m0": [], "conv2_m12": []}
    for name, c in ex.BIGVGAN.items():
        if name == "conv_pre":
            forms["conv_pre"].append(name)
            assert c["conv_taps"] == 7 and c["conv_pad"] == 3 and c.get("out", "bf16") == "bf16" and c["K"] == 128
        elif name.startswith("ups"):
            forms["ups"].append(name)
        elif name.startswith("conv1"):
            forms["conv1"].append(name)
        else:
            forms["conv2_m0" if c["resid"] == "sep" else "conv2_m12"].append(name)
    assert all(forms.values()), forms
    released = {(c, k, d) for c in ex.BIGVGAN_C for k in (3, 7, 11) for d in (1, 3, 5)}
    assert {(c["N"], c["conv_taps"], c.get("conv_dilation", 1)) for n, c in ex.BIGVGAN.items()
            if n.startswith("conv1")} == released
    assert set(BIGVGAN_FORMS) == set(forms)


def test_launch_geometry_restates_the_launcher():
    """kernel_check's tile width and tile count follow f5_gemm_bf16 (gemm.cu) on known answers."""
    from kernel_check import gemm_bn, gemm_num_kb, gemm_tile_count
    assert gemm_bn(1024, 1874, sms=132) == 128                    # 15 x 8 = 120 tiles >= 107: 128 wide
    assert gemm_bn(1024, 937, sms=132) == 64                      # 8 x 8 = 64 < 107
    assert gemm_bn(64, 100000, sms=132) == 64 and gemm_bn(100, 128, tile_n=128, sms=132) == 128
    assert gemm_bn(512, 300, tile_n=128, conv_grouped=True, sms=132) == 64
    assert gemm_bn(1024, 3 * 300, rows_per_batch=300, num_batches=3, batched=True, sms=132) == 64   # 3 x 3 x 8 = 72
    assert gemm_tile_count(1000, 300, 128) == 8 * 3
    assert gemm_tile_count(1000, 300, 64, rows_per_batch=150, num_batches=2, batched=True) == 16 * 4
    assert gemm_num_kb(320) == 5 and gemm_num_kb(640, ab8=True) == 5 and gemm_num_kb(64, conv_taps=31) == 31
    # the restated lines of gemm.cu are still there
    src = (ROOT / "f5_tts_mlx_b200" / "csrc" / "gemm.cu").read_text()
    for line in ("if (a->conv_grouped) bn = 64;",
                 "const int mt = batched ? nb * cdiv(rpb, 128) : cdiv(a->m, 128);",
                 "bn = (mt * cdiv(a->n, 128) >= (sm_count() * 13) / 16 || a->n <= 64) ? 128 : 64;",
                 "const int tiles = cdiv(a->n, bn) * (batched ? nb * cdiv(rpb, 128) : cdiv(a->m, 128));",
                 "dim3 grid(std::min(tiles, sm_count()), 1, 1);",
                 "return dispatch_scaled<64, 6>", "return dispatch_scaled<128, 4>", "return dispatch_epi<64, 6>",
                 "return dispatch_epi<128, 4>"):
        assert line in src, line


def test_every_instantiation_has_a_many_waves_case():
    """Every (instantiation, BN) of dispatch_epi and dispatch_scaled has exactly one WAVES case (test_gpu_gemm_persistent)
    that, on a 132-SM H100, launches more than 3 x 132 tiles (every CTA runs at least 3, on both consumer warpgroups)
    with num_kb not a multiple of the ring depth.  A new instantiation without such a case fails here, named."""
    from test_fp8_block import built_scaled_instantiations
    import test_gpu_gemm_persistent as P
    from test_gpu_kernel_exact import inst_of
    sms = 132
    pairs = {(False,) + i + (bn,) for i in built_instantiations() for bn in (64, 128)}
    pairs |= {(True,) + i + (bn,) for i in built_scaled_instantiations() for bn in (64, 128)}
    assert len(pairs) == 36
    covered = {}
    for name in P.WAVES:
        c = P.wave_case(name, sms)
        geo = P.wave_geometry(c, sms)
        key = (c.get("scaled", False) or c.get("out_blocks", False),) + inst_of(c)
        assert key in pairs, f"{name}: launches {key}, which gemm.cu does not build"
        assert key[-1] == geo["bn"], (name, geo)
        assert key not in covered, f"{name} and {covered.get(key)} both cover {key}"
        assert 3 * sms < geo["tiles"] < 4 * sms and geo["per_cta"][0] >= 3, (name, geo)
        assert geo["num_kb"] % geo["stages"] != 0, (name, geo)
        covered[key] = name
    missing = sorted(pairs - set(covered))
    assert not missing, f"(SCALED, ACT, OUT_BF16, ROPE, FP8, RESID, BN) without a many-waves case: {missing}"
