"""CPU: the fused AdaLN's emulated arithmetic (adaln_emul) against float64 LayerNorm -> modulate -> Linear on rows of
conditioning r = |mean| / std, as a regression test of the bound in kernel_check.fused_ln_ref_bound itself."""
import math

import pytest
import torch

import adaln_emul as A
from kernel_check import U_BF16, fused_ln_ref_bound, gemm_acc_bound

R_VALUES = [0, 0.25, 1, 4, 16, 64, 256, 1024, 4096]

# relative error against float64 (D = N = 1024, M = 256 rows z + r): unfused, fused, fused with exact statistics,
# and the largest relative error of the emulated rstd
TABLE = {0: (1.65e-3, 1.50e-3, 1.50e-3, 1.5e-7), 1: (1.66e-3, 2.12e-3, 2.11e-3, 3.9e-7),
         4: (1.66e-3, 6.2e-3, 6.2e-3, 4.6e-6), 16: (1.65e-3, 2.4e-2, 2.4e-2, 5.1e-5),
         64: (1.66e-3, 9.8e-2, 9.8e-2, 1.2e-3), 1024: (1.66e-3, 1.6, 1.56, 0.25)}


@pytest.fixture(scope="module")
def table():
    return A.error_table(list(TABLE) + [4096])


@pytest.mark.parametrize("r", list(TABLE))
def test_error_table_reproduces(table, r):
    """The operand term dominates the fused error at every r below about 1000: fused and fused-with-exact-statistics
    agree, grow like sqrt(1 + r^2), and the unfused error does not move.  The rstd error grows like r^2."""
    unf, fus, fex, drs = table[r]
    want = TABLE[r]
    assert want[0] / 1.25 < unf < want[0] * 1.25, (r, unf)
    assert want[1] / 1.25 < fus < want[1] * 1.25, (r, fus)
    assert want[2] / 1.25 < fex < want[2] * 1.25, (r, fex)
    assert want[3] / 8 < drs < want[3] * 8, (r, drs)
    if r <= 64:
        assert abs(fus / fex - 1) < 0.02, (r, fus, fex)
        ratio = fus / unf
        assert 0.5 * A.predicted_ratio(r) < ratio < 1.5 * A.predicted_ratio(r), (r, ratio)


def test_error_table_clamped_variance(table):
    """At r = 4096 the variance cancels to zero or below, is clamped, and rstd becomes 1 / sqrt(1e-6) = 1000: the
    fused output is wrong by orders of magnitude while the unfused path is untouched."""
    unf, fus, fex, drs = table[4096]
    assert unf < 2e-3 and fus > 100 and drs > 100


@pytest.mark.parametrize("r", R_VALUES)
def test_rstd_within_statistics_bound(r):
    """The emulated rstd (unit sums in the producer's order, E[x^2] - mean^2 in the consumer's) is within the bound
    of fused_ln_stats_bound on every row, and that bound is within 64x of the worst error it allows for (it is a
    worst case over summation orders, not an estimate)."""
    x = A.conditioned_rows(64, 1024, r, seed=int(r * 4) + 1)
    _, rstd = A.row_stats(A.unit_sums(x))
    rt = A.exact_stats(x)[2]
    err = (rstd.double() / rt - 1).abs()
    bd = A.rstd_rel_bound(x)
    finite = torch.isfinite(bd)
    assert (err[finite] <= bd[finite]).all(), (r, (err / bd).max().item())
    if r <= 256:
        assert finite.all(), r
    if 16 <= r <= 256:
        assert bd.max().item() < 64 * err.max().item(), (r, bd.max().item(), err.max().item())


def test_rstd_bound_infinite_once_variance_may_cancel():
    """Past r ~ 1000 (D = 1024) the bound admits a zero variance: it is infinite rather than wrong."""
    x = A.conditioned_rows(16, 1024, 4096, seed=5)
    assert torch.isinf(A.rstd_rel_bound(x)).all()


@pytest.mark.parametrize("r", [0, 1, 16, 256])
def test_emulated_fused_linear_within_derived_bound(r):
    """The emulated fused path (bf16 operand of x (1 + s), emulated statistics, fp32 tables) is within
    fused_ln_ref_bound of float64 Linear(LN(x)(1 + s) + b), and the bound's operand term is what grows with r."""
    M, D, N = 64, 1024, 256
    g = torch.Generator().manual_seed(3)
    w = (torch.randn(N, D, generator=g) * D ** -0.5).bfloat16()
    s = torch.randn(D, generator=g) * 0.3
    b = torch.randn(D, generator=g) * 0.5
    bias = torch.zeros(N)
    x = A.conditioned_rows(M, D, r, seed=9)
    got = A.fused_linear(x, s, b, w)
    xt = (x * (1 + s)).bfloat16()
    xs = x.double() * (1 + s.double())
    v, bd = fused_ln_ref_bound(x.double(), torch.zeros(M, D, dtype=torch.float64), s, b, w, bias,
                               gemm_acc_bound(xt, w), op_err=U_BF16 * xs.abs())
    ratio = ((got - v).abs() / bd).max().item()
    assert ratio <= 1, ratio
    assert torch.allclose(v, A.reference_linear(x, s, b, w), rtol=1e-12, atol=1e-12)
    # the operand term alone, normalised by the output's rms, grows like sqrt(1 + r^2)
    rstd = A.exact_stats(x)[2][:, None]
    op = (rstd * (U_BF16 * xs.abs()) @ w.double().abs().T).mean().item() / v.pow(2).mean().sqrt().item()
    assert 0.03 < op / A.predicted_ratio(r) < 0.15, (r, op)
    print(f"r {r}: worst err/bound {ratio:.3g}, operand term / rms {op:.3g}")


def test_oracle_fused_adaln_documents_its_statistics():
    """The oracle's ln_by_linearity emulation uses exact two-pass statistics; the kernel stores (sum, sum of squares)
    per 64 columns.  The docstring says which, so the derived DiT tolerances are read for what they emulate."""
    from oracle import f5_oracle as O
    doc = O.adaln_linear.__doc__
    assert "sum of squares" in doc and "two-pass" in doc and "(mean, M2)" not in doc
    assert math.isfinite(A.EPS) and A.EPS == float(torch.tensor(1e-6, dtype=torch.float32))
