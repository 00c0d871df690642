"""CPU emulation of the fused AdaLN's arithmetic (gemm_epilogue.cuh), for rows of any conditioning r = |mean| / std.

The fused AdaLN finishes LayerNorm -> modulate -> Linear inside the consuming GEMM's epilogue by linearity:
    Linear(LN(x)(1 + s) + b) = rstd (x~ W^T - mean c1) + c2,   x~ = bf16(x (1 + s)),  c1 = (1 + s) W^T,  c2 = b W^T + bias.
Its two r-dependent rounding points are emulated here in fp32, in the kernels' order:
* producer (the out-projection / FF2 epilogue): per 64-column unit of the fp32 row, the sum and the sum of squares, each
  over 32 columns in four chains of 8 (chain i takes columns i, i + 4, ...; the squares by fma), the chains combined as
  (c0 + c1) + (c2 + c3); the second 32 columns start chain 0 from the first half's result (unit_sums);
* consumer (epi_load_ln_row): the units' sums added in unit order, mean = s1 / K, var = max(s2 / K - mean^2, 0),
  rstd = rsqrt(var + 1e-6) (row_stats).  The operand x~ is rounded before it is centred, so its error is relative to
  |x|, not to the row's spread (fused_linear).
The unfused path rounds bf16(LN(x)(1 + s) + b) after normalising (unfused_linear).  Both are compared with the float64
reference (reference_linear)."""
from __future__ import annotations

import math

import torch

EPS = float(torch.tensor(1e-6, dtype=torch.float32))


def conditioned_rows(M: int, D: int, r: float, seed: int = 0, sigma: float = 1.0) -> torch.Tensor:
    """fp32 rows x = sigma_row (z + r sign_row): row mean r sigma_row (alternating sign), row std ~ sigma_row, with
    sigma_row = sigma 2^u, u uniform in [-1, 1] (row-level variation)."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(M, D, generator=g, dtype=torch.float64)
    z = (z - z.mean(1, keepdim=True)) / z.std(1, unbiased=False, keepdim=True)     # exact r per row
    sig = sigma * torch.pow(2.0, torch.rand(M, 1, generator=g, dtype=torch.float64) * 2 - 1)
    sign = torch.where(torch.arange(M)[:, None] % 2 == 0, 1.0, -1.0).double()
    return (sig * (z + r * sign)).float()


def _fma32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """fp32 fma (a b + c rounded once): the product of two fp32 values is exact in float64."""
    return (a.double() * b.double() + c.double()).float()


def unit_sums(x: torch.Tensor) -> torch.Tensor:
    """[M, D] fp32 -> [M, D / 64, 2] fp32 (sum, sum of squares) per 64-column unit, in the producer epilogue's order."""
    M, D = x.shape
    u = x.float().reshape(M, D // 64, 2, 8, 4)        # unit, half, step j, chain i  (column 32 h + 4 j + i)
    out = torch.zeros(M, D // 64, 2)
    carry1 = torch.zeros(M, D // 64)
    carry2 = torch.zeros(M, D // 64)
    for h in range(2):
        s1 = torch.zeros(M, D // 64, 4)
        s2 = torch.zeros(M, D // 64, 4)
        s1[..., 0], s2[..., 0] = carry1, carry2
        for j in range(8):
            v = u[:, :, h, j, :]
            s1 = s1 + v
            s2 = _fma32(v, v, s2)
        carry1 = (s1[..., 0] + s1[..., 1]) + (s1[..., 2] + s1[..., 3])
        carry2 = (s2[..., 0] + s2[..., 1]) + (s2[..., 2] + s2[..., 3])
    out[..., 0], out[..., 1] = carry1, carry2
    return out


def row_stats(stats: torch.Tensor):
    """(mean, rstd) fp32 [M] from the unit statistics, as epi_load_ln_row forms them (rsqrtf rounded to nearest)."""
    s1 = torch.zeros(stats.shape[0])
    s2 = torch.zeros(stats.shape[0])
    for u in range(stats.shape[1]):
        s1 = s1 + stats[:, u, 0]
        s2 = s2 + stats[:, u, 1]
    inv_k = torch.tensor(1.0 / (64 * stats.shape[1]), dtype=torch.float32)
    mean = s1 * inv_k
    var = torch.clamp(s2 * inv_k - mean * mean, min=0)
    rstd = (1 / torch.sqrt((var + EPS).double())).float()
    return mean, rstd


def exact_stats(x: torch.Tensor):
    """float64 (mean, var, rstd) of each row."""
    xd = x.double()
    mean = xd.mean(1)
    var = xd.var(1, unbiased=False)
    return mean, var, 1 / torch.sqrt(var + EPS)


def rstd_rel_bound(x: torch.Tensor) -> torch.Tensor:
    """kernel_check.fused_ln_stats_bound's relative rstd bound, per row (float64 [M])."""
    from kernel_check import fused_ln_stats_bound
    return fused_ln_stats_bound(x.double())[3][:, 0]


def reference_linear(x, s, b, w, bias=None):
    """float64 Linear(LayerNorm(x)(1 + s) + b)."""
    xd = x.double()
    mean, _, rstd = exact_stats(x)
    y = (xd - mean[:, None]) * rstd[:, None] * (1 + s.double()) + b.double()
    v = y @ w.double().T
    return v if bias is None else v + bias.double()


def unfused_linear(x, s, b, w):
    """The separate path: bf16(LN(x)(1 + s) + b) (a two-pass LayerNorm, rounded after normalising) times W."""
    xd = x.double()
    mean, _, rstd = exact_stats(x)
    y = ((xd - mean[:, None]) * rstd[:, None] * (1 + s.double()) + b.double()).float().bfloat16()
    return y.double() @ w.double().T


def fused_linear(x, s, b, w, exact_statistics: bool = False):
    """The fused path: rstd (bf16(x (1 + s)) W^T - mean c1) + c2 with the emulated unit statistics (or the exact ones)."""
    if exact_statistics:
        mean, _, rstd = exact_stats(x)
    else:
        mean, rstd = row_stats(unit_sums(x))
        mean, rstd = mean.double(), rstd.double()
    xt = (x.float() * (1 + s.float())).bfloat16().double()
    wd = w.double()
    acc = (xt @ wd.T).float().double()
    c1 = ((1 + s.double()) @ wd.T).float().double()
    c2 = (b.double() @ wd.T).float().double()
    return rstd[:, None] * acc - (mean * rstd)[:, None] * c1[None] + c2[None]


def rel(a: torch.Tensor, ref: torch.Tensor) -> float:
    return ((a - ref).norm() / ref.norm()).item()


def error_table(r_values, D: int = 1024, N: int = 1024, M: int = 256, seed: int = 0):
    """{r: (unfused, fused, fused with exact statistics, max rstd relative error)}: relative errors against
    reference_linear on M rows x = z + r (std 1, mean r), random bf16 W [N, D], s ~ 0.3 N(0, 1), b ~ 0.5 N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(N, D, generator=g) * D ** -0.5).bfloat16()
    s = torch.randn(D, generator=g) * 0.3
    b = torch.randn(D, generator=g) * 0.5
    out = {}
    for r in r_values:
        z = torch.randn(M, D, generator=g, dtype=torch.float64)
        x = (z + r).float()
        ref = reference_linear(x, s, b, w)
        _, rstd = row_stats(unit_sums(x))
        rt = exact_stats(x)[2]
        out[r] = (rel(unfused_linear(x, s, b, w), ref), rel(fused_linear(x, s, b, w), ref),
                  rel(fused_linear(x, s, b, w, exact_statistics=True), ref),
                  (rstd.double() / rt - 1).abs().max().item())
    return out


def predicted_ratio(r: float) -> float:
    """Fused / unfused error ratio the operand rounding predicts for rows of conditioning r: the operand's error is
    relative to |x|, whose rms is std sqrt(1 + r^2), while the unfused operand's is relative to the normalised value
    (rms 1).  The constant in front (about 0.9 with s ~ 0.3 N(0, 1)) is the rest of the two paths' error budgets."""
    return math.sqrt(1 + r * r)
