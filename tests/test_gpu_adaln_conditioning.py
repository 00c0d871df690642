"""-m gpu: every LayerNorm path of the DiT against a float64 LayerNorm, on rows whose mean is large against their spread.

The fused AdaLN (DiT(fused_adaln=True), the default) finishes the QKV, FF1 and proj_out LayerNorms in the consuming
GEMM's epilogue: rstd (x~ W^T - mean c1) + c2 with x~ = bf16 / e4m3(x (1 + s)) rounded before it is centred and
(mean, rstd) from the producer's fp32 (sum, sum of squares) per 64 columns.  Both rounding points depend on the row's
conditioning r = |mean| / std (tests/adaln_emul.py emulates them on the CPU).  Here the real chain runs: the out-proj /
FF2 form of the producer GEMM (shared gate, in-place residual, ln_scale, ln_stats) writes x, the operand and the
statistics; the QKV (RoPE, q_scale), FF1 (GELU-tanh) and proj_out (fp32, N = 100) consumers read them, in the bf16,
per-tensor FP8 and block-scaled FP8 modes and at 64- and 128-wide tiles.  One launch holds rows of every r (alternating
sign, so a neighbour's statistics differ), rows with one outlier channel, and rows that are constant but for one element.

Each consumer output is checked twice against float64 Linear(LayerNorm(x)(1 + s) + b) on the producer's float64 x:
* within kernel_check.fused_ln_ref_bound, which charges the operand's rounding relative to |x| (it grows like 1 + r);
* on the operand the producer wrote, within the same bound without its operand term: at the fp32 level, so a wrong
  table row, a wrong unit or a wrong eps exceeds it.
The separate f5_ln_modulate, f5_ln_affine_f32 and f5_dwconv7_ln run on the same rows within hbm_check's bounds, which do
not grow with r (two-pass statistics)."""
import pytest
import torch

import adaln_emul as A
from hbm_check import dwconv7_ref_bound, ln_depth, ln_ref_bound
from kernel_check import (E4M3_SUB, U32, U_BF16, U_E4M3, Guarded, act_bound, act_ref, e4m3, fused_ln_ref_bound,
                          gemm_acc_bound, gemm_acc_bound_fp8, gemm_tiles, instantiation, out_bound, rope_bound,
                          rope_ref)

pytestmark = pytest.mark.gpu
DEV = "cuda"
F8 = torch.float8_e4m3fn
D = 1024
ROWS = 32                                      # rows per group
R_FUSED = [0, 0.25, 1, 4, 16, 64, 256]
R_SEPARATE = R_FUSED + [1024, 4096]
FORMS = {"qkv": 3 * D, "ff1": 2 * D, "proj_out": 100}
MODES = ["bf16", "fp8_tensor", "fp8_block"]
WORST = {}

# instantiations the consumer launches select: (ACT, OUT_BF16, ROPE, FP8, RESID, BN)
INSTANTIATIONS = sorted({instantiation(rope=True, fp8=m != "bf16", scaled=m == "fp8_block", tile=t) for m in MODES
                         for t in (64, 128)}
                        | {instantiation(act=1, fp8=m != "bf16", scaled=m == "fp8_block", tile=t) for m in MODES
                           for t in (64, 128)}
                        | {instantiation(out_dtype=torch.float32, tile=t) for t in (64, 128)})


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst err/bound per path and row group:")
        for k, v in sorted(WORST.items()):
            print(f"  {k:56s} {v:.3g}")


def ops():
    from f5_tts_mlx_b200 import ops as _ops
    return _ops


def groups(r_values):
    return [("r", r) for r in r_values] + [("outlier", 100), ("outlier", 1000), ("const1", None)]


def gname(kind, p):
    return f"r={p:g}" if kind == "r" else (f"outlier {p}" if kind == "outlier" else "constant but one")


def make_rows(r_values, sigma, seed=0):
    """fp32 rows, ROWS per group: x = sigma_row (z + r sign) (conditioned_rows), the same at r = 0 with one channel
    raised by 100 or 1000 sigma, and 0.01 sigma everywhere but one element (0.15 sigma higher): r ~ 2 and a variance
    of about 2e-5 sigma^2, where the LayerNorm's eps = 1e-6 is a visible part of rstd."""
    out = []
    for i, (kind, p) in enumerate(groups(r_values)):
        if kind == "r":
            x = A.conditioned_rows(ROWS, D, p, seed=seed + i, sigma=sigma)
        elif kind == "outlier":
            x = A.conditioned_rows(ROWS, D, 0, seed=seed + i, sigma=sigma)
            x[:, 7 + i] += p * sigma
        else:
            x = torch.full((ROWS, D), 0.01 * sigma)
            x[torch.arange(ROWS), (torch.arange(ROWS) * 37) % D] += 0.15 * sigma
        out.append(x)
    return torch.cat(out)


def modulation(seed=5):
    """s with a coherent lo part: 1 + s = hi (1 + 2^-9) for bf16 hi, so c1's lo table row is 2^-9 of its hi row (a
    consumer that drops the lo row is off by rstd |mean| 2^-9 |c1|, which the one-signed weight rows of
    consumer_weights make several times the operand-free bound); b ~ 0.5 N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    hi = (1 + torch.randn(D, generator=g) * 0.3).bfloat16().float()
    s = hi * (1 + 2.0 ** -9) - 1
    return s, torch.randn(D, generator=g) * 0.5


def ln_tab(s, b, w):
    a = 1 + s
    ah = a.bfloat16().float(); al = (a - ah).bfloat16().float()
    bh = b.bfloat16().float(); bl = (b - bh).bfloat16().float()
    wf = w.float()
    return torch.stack([ah @ wf.T, al @ wf.T, bh @ wf.T, bl @ wf.T]).contiguous()


def producer(x0, s, mode, tile, seed=1):
    """The out-proj / FF2 form on exact operands (e4m3 codes in {0, +-1, +-2}, power-of-two scales): x = x0 + gate v
    with v exact, so the kernel's x is within u |x| of the float64 x.  Rows of the constant group get a zero A row.
    Returns (float64 x, its bound, the kernel's fp32 x, its operand out2 as written, the operand's block scales or
    None, that operand as float64, the unit statistics)."""
    M = x0.shape[0]
    K = 512
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(-2, 3, (M, K), generator=g).float()
    a[-ROWS:] = 0
    w = torch.randint(-2, 3, (D, K), generator=g).float()
    gate = torch.randn(D, generator=g) * float(x0.abs().median()) / 200
    xg = Guarded(M, D, torch.float32, DEV); xg.view.copy_(x0)
    st = Guarded(M, D // 64 * 2, torch.float32, DEV, lr=False)
    kw = dict(resid=xg.view, gate=gate.to(DEV), ln_scale=s.to(DEV), ln_stats=st.view.view(M, D // 64, 2), tile_n=tile,
              w_static=True)
    if mode == "bf16":
        o2 = Guarded(M, D, torch.bfloat16, DEV)
        ops().gemm(a.bfloat16().to(DEV), w.bfloat16().to(DEV), xg.view, out2=o2.view, **kw)
    else:
        o2 = Guarded(M, D, torch.uint8, DEV)
        kw.update(out2=o2.view, out2_fp8=True, ab_fp8=True)
        if mode == "fp8_block":
            s2 = Guarded(D // 64, M, torch.float32, DEV, lr=False)
            ops().gemm(a.to(F8).to(DEV), w.to(F8).to(DEV), xg.view, a_scale=torch.ones(K // 64, M, device=DEV),
                       w_scale=torch.ones(D, device=DEV), out2_scale=s2.view, **kw)
        else:
            ops().gemm(a.to(F8).to(DEV), w.to(F8).to(DEV), xg.view, **kw)
    torch.cuda.synchronize()
    x = x0.double() + gate.double() * (a.double() @ w.double().T)
    bx = U32 * x.abs()
    for gd, what in ((xg, "x"), (o2, "out2"), (st, "ln_stats")):
        gd.check(f"producer {mode} {what} guard")
    xs = x * (1 + s.double())
    if mode == "bf16":
        xt, sc = o2.view.cpu().double(), None
        err = U_BF16 * (xs.abs() + bx) + bx * (1 + s.double()).abs()
    else:
        xt = o2.view.cpu().view(F8).double()
        sc = s2.view.cpu().T.double().repeat_interleave(64, 1) if mode == "fp8_block" else torch.ones_like(xt)
        xt = xt * sc
        err = U_E4M3 * (xs.abs() + bx) + E4M3_SUB * sc + bx * (1 + s.double()).abs()
    assert ((xt - xs).abs() <= err).all(), f"producer {mode}: operand not within its rounding of x (1 + s)"
    return x, bx, xg.view, o2.view, (s2.view if mode == "fp8_block" else None), xt, st.view.view(M, D // 64, 2)


ONE_SIGNED = 16     # every 16th consumer weight row (rows 5, 21, ...: in every 64- and 128-wide tile) is one-signed


def consumer_weights(N, mode, seed=2):
    """Random N(0, 1/D) bf16 weight rows, and one-signed ones: for those |c1| = |sum (1 + s) w| is sum |1 + s| |w|
    rather than that over sqrt(D), so a table error relative to c1 is not hidden below the accumulation term.
    Returns (bf16 w, bias, the weight the GEMM reads, its tensor scale, per-channel scales, dequantised e4m3 or None)."""
    g = torch.Generator().manual_seed(seed + N)
    w16 = (torch.randn(N, D, generator=g) * D ** -0.5).bfloat16()
    w16[5::ONE_SIGNED] = w16[5::ONE_SIGNED].abs()
    bias = torch.randn(N, generator=g) * 0.5
    if mode == "bf16":
        return w16, bias, w16, 1.0, None, None
    if mode == "fp8_tensor":
        sc = float(w16.float().abs().max()) / 448.0
        w8 = e4m3(w16.float() / sc)
        return w16, bias, w8, sc, None, w8.float().double() * sc
    from fp8_block_emul import q_channels
    codes, ws = q_channels(w16.float())
    return w16, bias, codes.to(F8), 1.0, ws.float(), codes.double() * ws.double()[:, None]


def run_consumer(form, mode, tile, chain, w, bias, tab, wk, sc, ws, ln_in=True, a=None):
    """One consumer launch; returns the output as float64 (e4m3 outputs dequantised) and the output scales."""
    x, bx, xf, o2, s2, xt, st = chain
    M, N = x.shape[0], w.shape[0]
    kw = dict(bias=bias.to(DEV), tile_n=tile, w_static=True)
    if ln_in:
        kw.update(ln_in_stats=st, ln_tab=tab.to(DEV))
    if form == "qkv":
        from f5_tts_mlx_b200.dit import rope_table
        kw.update(rope=rope_table(M).to(DEV), rope_cols=2 * N // 3, q_scale=0.125, q_cols=N // 3, rows_per_batch=M,
                  num_batches=1)
    if form == "ff1":
        kw.update(act=1)
    odt = torch.float32 if form == "proj_out" else torch.bfloat16
    fp8_out = form == "ff1" and mode != "bf16"
    if fp8_out:
        odt = torch.uint8
        kw.update(out_fp8=True)
    out = Guarded(M, N, odt, DEV)
    osc = None
    if mode != "bf16" and form != "proj_out":
        kw.update(ab_fp8=True, acc_scale=sc)
        if mode == "fp8_block":
            kw.update(a_scale=s2, w_scale=ws.to(DEV))
            if fp8_out:
                osc = Guarded(N // 64, M, torch.float32, DEV, lr=False)
                kw.update(out_scale=osc.view)
        ops().gemm(o2.view(F8) if a is None else a, wk.to(DEV), out.view, **kw)
    else:
        ops().gemm(o2 if a is None else a, w.to(DEV), out.view, **kw)
    torch.cuda.synchronize()
    out.check(f"{form} {mode} tile {tile} out guard")
    got = out.view.cpu()
    got = got.view(F8).double() if fp8_out else got.double()
    if osc is not None:
        osc.check("out scale guard")
        osc = osc.view.cpu().T.double().repeat_interleave(64, 1)
        got = got * osc
    return got, osc, fp8_out


def finish(form, v, bd, osc, fp8_out, M):
    """The consumer's activation / RoPE / q_scale and the output rounding on a pre-activation reference and bound."""
    if form == "ff1":
        ref, bd = act_ref(v, 1), act_bound(v, bd, 1)
    elif form == "qkv":
        N = v.shape[1]
        from f5_tts_mlx_b200.dit import rope_table
        tab, pos = rope_table(M).double(), torch.arange(M)
        ref, bd = rope_ref(v, tab, pos, 2 * N // 3), rope_bound(v, bd, tab, pos, 2 * N // 3)
        ref[:, :N // 3] *= 0.125; bd[:, :N // 3] *= 0.125
    else:
        ref = v
    if osc is not None:
        return ref, bd + U_E4M3 * (ref.abs() + bd) + E4M3_SUB * osc
    return ref, out_bound(ref, bd, torch.uint8 if fp8_out else (torch.float32 if form == "proj_out" else torch.bfloat16))


def per_group(got, ref, bd, r_values, key):
    """Assert |got - ref| <= bd everywhere, record the worst ratio of each row group, name the worst element."""
    ratio = (got - ref).abs() / bd
    ratio = torch.where(torch.isfinite(got), ratio, torch.full_like(ratio, float("inf")))
    for i, (kind, p) in enumerate(groups(r_values)):
        rr = ratio[i * ROWS:(i + 1) * ROWS]
        WORST[f"{key} {gname(kind, p)}"] = max(WORST.get(f"{key} {gname(kind, p)}", 0.0), rr.max().item())
    worst = ratio.max().item()
    r, c = divmod(int(ratio.argmax()), ratio.shape[1])
    kind, p = groups(r_values)[r // ROWS]
    msg = (f"{key}: worst err/bound {worst:.3g} in group {gname(kind, p)} at row {r} col {c} "
           f"({gemm_tiles(128)(r, c)}): got {got[r, c].item()!r} ref {ref[r, c].item()!r} bound {bd[r, c].item():.3g}")
    assert worst <= 1.0, msg
    print(msg)


def _chain_case(form, mode, tile):
    sigma = 2.0 ** -3 if mode == "fp8_tensor" else 1.0          # per-tensor e4m3 operands hold |x (1 + s)| <= 448
    x0 = make_rows(R_FUSED, sigma)
    s, b = modulation()
    chain = producer(x0, s, mode, tile)
    x, bx, xf, o2, s2, xt, st = chain
    N = FORMS[form]
    w, bias, wk, sc, ws, w_eff = consumer_weights(N, mode if form != "proj_out" else "bf16")
    tab = ln_tab(s, b, w)
    got, osc, fp8_out = run_consumer(form, mode, tile, chain, w, bias, tab, wk, sc, ws)
    xsa = x.abs() * (1 + s.double()).abs()
    if mode == "bf16" or form == "proj_out":
        op_err = U_BF16 * (xsa + bx)
        acc = gemm_acc_bound(xt, w)
    else:
        op_err = U_E4M3 * (xsa + bx) + E4M3_SUB * (s2.cpu().T.double().repeat_interleave(64, 1)
                                                   if mode == "fp8_block" else 1.0)
        acc = gemm_acc_bound_fp8(xt, w_eff.float()) if mode == "fp8_block" else gemm_acc_bound_fp8(xt, wk, sc)
    M = x.shape[0]
    key = f"{form} {mode} tile {tile}"
    v, bd = fused_ln_ref_bound(x, bx, s, b, w, bias, acc, op_err=op_err, w_eff=w_eff)
    ref, bd = finish(form, v, bd, osc, fp8_out, M)
    per_group(got, ref, bd, R_FUSED, key + " vs float64")
    v2, bd2 = fused_ln_ref_bound(x, bx, s, b, w, bias, acc, operand=xt, w_eff=w_eff)
    ref2, bd2 = finish(form, v2, bd2, osc, fp8_out, M)
    per_group(got, ref2, bd2, R_FUSED, key + " on its operand")
    return chain, got, ref, (w, bias, s, b)


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", ["qkv", "ff1"])
def test_fused_chain_against_float64_layernorm(form, mode, tile):
    """Producer then consumer, each consumer output within fused_ln_ref_bound of the float64 LayerNorm -> Linear, in
    every row group (r from 0 to 256, outlier channels, constant-but-one rows), and within the operand-free bound on
    the operand the producer wrote."""
    _chain_case(form, mode, tile)


@pytest.mark.parametrize("tile", [64, 128])
def test_fused_chain_proj_out(tile):
    """proj_out: N = 100 mel columns, fp32 output; its operand is bf16 in every mode (the last FF2 writes it so)."""
    _chain_case("proj_out", "bf16", tile)


@pytest.mark.parametrize("form", ["qkv", "ff1"])
def test_fused_against_unfused_error_ratio(form):
    """The fused and the separate path on the same producer output, both against float64.  At r <= 1 the fused error
    norm is at most 2x the unfused one (the CPU emulation gives 1.3x); beyond, the ratio follows the operand law
    sqrt(1 + r^2) (adaln_emul.predicted_ratio) within a factor 2.5 either way; every output is finite up to r = 256."""
    from f5_tts_mlx_b200 import _lib
    chain, got, ref, (w, bias, s, b) = _chain_case(form, "bf16", 128)
    x, bx, xf, *_ = chain
    M = x.shape[0]
    y = torch.empty(M, D, device=DEV, dtype=torch.bfloat16)
    xc, sd, bd = xf.contiguous(), s.to(DEV), b.to(DEV)
    _lib.check(_lib.load().f5_ln_modulate(xc.data_ptr(), y.data_ptr(), M, D, 0, sd.data_ptr(), bd.data_ptr(), 0, 1,
                                          torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    unf, _, _ = run_consumer(form, "bf16", 128, chain, w, bias, None, None, 1.0, None, ln_in=False, a=y)
    lines = []
    for i, (kind, p) in enumerate(groups(R_FUSED)):
        sl = slice(i * ROWS, (i + 1) * ROWS)
        ef = ((got[sl] - ref[sl]).norm() / ref[sl].norm()).item()
        eu = ((unf[sl] - ref[sl]).norm() / ref[sl].norm()).item()
        assert torch.isfinite(got[sl]).all()
        ratio = ef / eu
        lines.append(f"  {gname(kind, p):18s} fused {ef:.3e} unfused {eu:.3e} ratio {ratio:.3g}")
        if kind == "r" and p <= 1:
            assert ratio <= 2.0, lines[-1]
        if kind == "r" and p >= 4:
            pred = A.predicted_ratio(p)
            assert pred / 2.5 <= ratio <= 2.5 * pred, lines[-1] + f" predicted {pred:.3g}"
        if kind == "outlier":
            assert ratio <= 3.0, lines[-1]
    print(f"\n{form}: fused / unfused error against float64 per row group\n" + "\n".join(lines))


def test_separate_layernorm_paths_do_not_grow_with_r():
    """f5_ln_modulate, f5_ln_affine_f32 and f5_dwconv7_ln on the same rows, r up to 4096: within hbm_check's bounds,
    and each bf16 path's error norm at every r stays within 2x of its error at r = 0 (two-pass statistics); the fp32
    output may add the mean's rounding, gam(ln_depth) r."""
    from f5_tts_mlx_b200 import _lib
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    x = make_rows(R_SEPARATE, 1.0, seed=40).to(DEV)
    M = x.shape[0]
    s, b = modulation(9)
    s, b = s.to(DEV), b.to(DEV)
    lw, lb = 1 + s, b
    g = torch.Generator().manual_seed(3)
    wt = torch.zeros(7, D); wt[3] = 1
    wt = (wt + torch.randn(7, D, generator=g) * 0.01).to(DEV)
    wb = (torch.randn(D, generator=g) * 0.1).to(DEV)
    runs = {}
    y = Guarded(M, D, torch.bfloat16, DEV, lr=False)
    _lib.check(lib.f5_ln_modulate(x.data_ptr(), y.view.data_ptr(), M, D, 0, s.data_ptr(), b.data_ptr(), 0, 1, stream))
    runs["ln_modulate"] = (y, *ln_ref_bound(x, s.expand(M, D), b.expand(M, D), True, torch.bfloat16))
    y32 = Guarded(M, D, torch.float32, DEV, lr=False)
    _lib.check(lib.f5_ln_affine_f32(x.data_ptr(), y32.view.data_ptr(), M, D, lw.data_ptr(), lb.data_ptr(), stream))
    runs["ln_affine_f32"] = (y32, *ln_ref_bound(x, lw.expand(M, D), lb.expand(M, D), False, torch.float32))
    yc = Guarded(M, D, torch.bfloat16, DEV, lr=False)
    _lib.check(lib.f5_dwconv7_ln(x.data_ptr(), yc.view.data_ptr(), 1, M, D, wt.data_ptr(), wb.data_ptr(), lw.data_ptr(),
                                 lb.data_ptr(), stream))
    runs["dwconv7_ln"] = (yc, *dwconv7_ref_bound(x.view(1, M, D), wt, wb, lw, lb))
    torch.cuda.synchronize()
    for name, (out, ref, bd) in runs.items():
        out.check(name + " guard")
        got = out.view.double()
        per_group(got.cpu(), ref.cpu(), bd.cpu(), R_SEPARATE, name)
        errs = []
        for i in range(len(R_SEPARATE)):
            sl = slice(i * ROWS, (i + 1) * ROWS)
            errs.append(((got[sl] - ref[sl]).norm() / ref[sl].norm()).item())
        print(f"{name}: error norm per r {dict(zip(R_SEPARATE, ['%.2e' % e for e in errs]))}")
        # the bf16 outputs' error is their output rounding at every r; the fp32 output resolves the one r-dependent
        # term of the two-pass bound, the mean's fp32 rounding (at most gam(ln_depth) r of the row's spread)
        slack = [ln_depth(D) * U32 * r if name == "ln_affine_f32" else 0.0 for r in R_SEPARATE]
        assert all(e <= 2 * errs[0] + sl for e, sl in zip(errs, slack)), (name, errs)


R_PAST = [1024, 4096]


def test_fused_chain_past_cancellation():
    """r = 1024 and 4096, where E[x^2] - mean^2 may cancel to zero and fused_ln_stats_bound is infinite, so no
    element-wise bound applies (R_FUSED stops at 256 for that reason).  What the kernel does there is pinned instead:
    every output is finite, and on each r group the proj_out error norm against float64 is within 2x of the CPU
    emulation's (adaln_emul.fused_linear: the producer's unit sums, the consumer's formula) on the same fp32 rows."""
    from kernel_check import fused_ln_stats_bound
    x0 = make_rows(R_PAST, 1.0, seed=60)
    s, b = modulation()
    chain = producer(x0, s, "bf16", 128)
    x, bx, xf = chain[:3]
    w, bias, *_ = consumer_weights(100, "bf16")
    got, _, _ = run_consumer("proj_out", "bf16", 128, chain, w, bias, ln_tab(s, b, w), None, 1.0, None)
    assert torch.isfinite(got).all()
    ref = A.reference_linear(x, s, b, w, bias)
    emu = A.fused_linear(xf.cpu(), s, b, w) + bias.double()
    dr = fused_ln_stats_bound(x)[3][:, 0]
    lines = []
    for i, r in enumerate(R_PAST):
        sl = slice(i * ROWS, (i + 1) * ROWS)
        assert torch.isinf(dr[sl]).any(), r
        ek, ee = A.rel(got[sl], ref[sl]), A.rel(emu[sl], ref[sl])
        lines.append(f"  r={r}: kernel {ek:.3g} emulation {ee:.3g}")
        assert ee / 2 <= ek <= 2 * ee, lines[-1]
    print("\nproj_out error against float64 past the cancellation:\n" + "\n".join(lines))


# ---------------------------------------------------------------- the DiT with an offset residual stream
R_DIT = [1.0, 4.0, 16.0]


def _script():
    import importlib.util
    from pathlib import Path
    path = Path(__file__).resolve().parent.parent / "scripts" / "adaln_conditioning.py"
    spec = importlib.util.spec_from_file_location("adaln_conditioning", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _offset_for(target, key, base, measure):
    """The constant c added to base[key] that brings the median r of the stream (over all LayerNorm sites) to within
    10 % of target: bisection on c, r being monotone in it."""
    lo, hi = 0.0, 64.0
    for _ in range(40):
        c = 0.5 * (lo + hi)
        W = dict(base)
        W[key] = base[key] + c
        rs = measure(W)
        med = float(torch.tensor([r.median().item() for _, r in rs]).median())
        if abs(med / target - 1) < 0.1:
            return c, W, rs
        lo, hi = (c, hi) if med < target else (lo, c)
    raise AssertionError(f"no offset reaches r = {target} through {key}")


def test_dit_drift_against_stream_conditioning():
    """The gate-config DiT with a constant c added to every residual row: the median r the stream carries into the
    blocks' LayerNorms (measured with scripts/adaln_conditioning.py's stream_conditioning on the fp32 oracle) is
    brought to 1, 4 and 16.  The offset goes into input_embed.proj.bias for r = 1 and 4.  Through that bias r levels
    off near 7.5, because the conv position embedding's response grows with c, so r = 16 takes the offset in that
    embedding's last convolution bias instead (after which the stream carries it unchanged).  The separate-LayerNorm
    model's drift from the fp32 oracle stays at the bf16 level.  The fused model's drift follows the per-block
    prediction: with P the largest predicted fused / unfused ratio sqrt(1 + mean r^2) over the sites, it is at most
    (2 + P) times the unfused drift, and at least P / 4 times it once r >= 4 (the LayerNorm operand is one of several
    rounding points, so the whole forward's ratio stays below P)."""
    from f5_tts_mlx_b200.weights import GATE_CONFIG, random_dit_weights
    from helpers import make_dit, ocfg_of, rel
    from oracle import f5_oracle as O
    S = _script()
    cfg = GATE_CONFIG
    ocfg = ocfg_of(cfg)
    g = torch.Generator().manual_seed(2)
    N = 300
    x = torch.randn(1, N, 100, generator=g); cond = torch.randn(1, N, 100, generator=g) * 2 - 1
    text = torch.randint(0, 2545, (1, 60), generator=g, dtype=torch.int32)
    t = torch.tensor(0.5)
    base = random_dit_weights(cfg, seed=1234)
    measure = lambda W: S.stream_conditioning(x, cond, text, t, W, ocfg)
    lines = []
    for target in [0.0] + R_DIT:
        key = ("transformer.input_embed.proj.bias" if target <= 4 else
               "transformer.input_embed.conv_pos_embed.conv1d.layers.2.bias")
        if target == 0:
            c, W, rs = 0.0, base, measure(base)
        else:
            c, W, rs = _offset_for(target, key, base, measure)
        pred = max(S.predicted_ratio(r) for _, r in rs)
        med = [r.median().item() for _, r in rs]
        ref = O.dit_forward(x, cond, text, t, False, False, None, W, ocfg)
        fused = make_dit(cfg, W)(x.to(DEV), cond.to(DEV), text.to(DEV), t).cpu()
        sep = make_dit(cfg, W, fused_adaln=False)(x.to(DEV), cond.to(DEV), text.to(DEV), t).cpu()
        df, du = rel(fused, ref), rel(sep, ref)
        lines.append(f"  target r {target:4.1f} (c {c:.3g} in {key.split('.', 1)[1]}): median r per site "
                     f"{min(med):.2f}..{max(med):.2f}, predicted ratio <= {pred:.3g}; fused drift {df:.3e}, "
                     f"unfused {du:.3e}, ratio {df / du:.3g}")
        assert torch.isfinite(fused).all() and du < 2e-2, lines[-1]
        assert df <= du * (2 + pred), lines[-1]
        if target >= 4:
            assert df >= du * pred / 4, lines[-1]
        torch.cuda.empty_cache()
    print("\nDiT drift against the residual stream's conditioning:\n" + "\n".join(lines))
