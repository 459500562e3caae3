"""Float64 reference and per-element error bound of the synchronized BatchNorm entry points (`csnet_train_bn_sync_*`,
include/csnet_b200.h), in the style of tests/trainref.py: {output: (ref, bound)}, a kernel output `got` being correct when
|got - ref| <= bound on every element.

Each stage is checked on the values the kernel actually read, so a stage's bound covers that stage alone:
    partial      one rank's shard z [N, C, H, W] -> (count, mean, M2) per channel.  The kernel's sums are those of
                 csnet_train_bn_stats (same grid, shift and part-order merge in float64), kept in float64: mean has
                 trainref.bn_stats' mean bound, M2 = M var has M times its variance bound.  count is exact.
    merge        the gathered rows [G, C, 3] -> fp32 mean / biased var and the float64 count.  Exact:
                     n = sum n_r,  mean = sum n_r mean_r / n,  var = (sum M2_r + sum n_r (mean_r - mean)^2) / n.
                 The kernel runs Chan's pairwise update in float64 (2^-53 per operation, G steps) and rounds to fp32 once:
                     |d mean| <= u |mean| + 4 G e max|mean_r|
                     |d var|  <= u var + 8 G e (var + D^2) + 4 G^2 e D max|mean_r|,   D = max_r |mean_r - mean|, e = 2^-53
    bwd_reduce   one rank's (z, dy) with the merged mean / var -> dbeta / dgamma / dslope and the float64 row (S1, S2):
                 trainref.bn_prelu_bwd's sums and bounds (its fp32 part merge bounds the kernel's float64 one).
    bwd_apply    dz = gamma r (du - S1 / M - xhat S2 / M), S1 / S2 the gathered rows summed exactly, M the merged count:
                 trainref.bn_prelu_bwd's dz bound without its reduction terms (S1 / M and S2 / M are float64 values rounded
                 once to fp32); a bf16 dz adds its rounding, 2^-8 of its magnitude.

`defect=` applies one realistic mistake (the GPU test checks each is flagged):
    no_chan       merge: the shards' M2 are added without Chan's between-shard term n_r (mean_r - mean)^2
    local_count   bwd_apply: S1 / S2 divided by this rank's element count instead of the global one
"""
from __future__ import annotations

import torch

from tests import trainref as R

E64 = 2.0 ** -53                    # float64 unit roundoff
U_BF16 = 2.0 ** -8                  # bf16 unit roundoff (round to nearest even)
DEFECTS = ("no_chan", "local_count")


def partial(z):
    """{"count", "mean", "M2"}: [C] each, of one rank's shard."""
    z = R._d(z)
    N, C, H, W = z.shape
    M = N * H * W
    st = R.bn_stats(z)
    mean, bmean = st["mean"]
    var, bvar = st["var"]
    count = torch.full((C,), float(M), dtype=torch.float64, device=z.device)
    return {"count": (count, torch.full_like(count, 0.5)), "mean": (mean, bmean), "M2": (var * M, bvar * M)}


def merge(rows, defect=None):
    """{"mean", "var", "count"} of the gathered rows [G, C, 3] (count: a [1] tensor)."""
    rows = R._d(rows)
    G = rows.shape[0]
    n_r, mu_r, m2_r = rows[..., 0], rows[..., 1], rows[..., 2]
    n = n_r.sum(0)
    mean = (n_r * mu_r).sum(0) / n
    between = (n_r * (mu_r - mean) ** 2).sum(0)
    m2 = m2_r.sum(0) + (0.0 if defect == "no_chan" else between)
    var = m2 / n
    D = (mu_r - mean).abs().amax(0)
    mx = mu_r.abs().amax(0)
    bmean = R.U * mean.abs() + 4 * G * E64 * mx + R.TINY
    bvar = R.U * var + 8 * G * E64 * (var + D ** 2) + 4 * G * G * E64 * D * mx + R.TINY
    cnt = n[:1]
    return {"mean": (mean, bmean), "var": (var, bvar), "count": (cnt, torch.full_like(cnt, 0.5))}


def bwd_reduce(z, dy, mean, var, gamma, beta, slope, eps):
    """{"dgamma", "dbeta", "dslope", "S1", "S2"}: [C] each, of one rank's shard with the merged statistics."""
    b = R.bn_prelu_bwd(z, dy, mean, var, gamma, beta, slope, eps, frozen=0)
    out = {k: b[k] for k in ("dgamma", "dbeta", "dslope")}
    out["S1"], out["S2"] = b["dbeta"], b["dgamma"]
    return out


def bwd_apply(z, dy, mean, var, gamma, beta, slope, eps, rows, count, bf16=False, defect=None):
    """{"dz"} of one rank's shard; rows: the gathered [G, C, 2] (S1, S2), count: the merged [1] count."""
    z, dy = R._d(z), R._d(dy)
    N, C, H, W = z.shape
    rows = R._d(rows)
    M = float(N * H * W) if defect == "local_count" else float(R._d(count).reshape(-1)[0])
    e = lambda t: t.reshape(1, C, 1, 1)
    m1, m2 = e(rows[..., 0].sum(0) / M), e(rows[..., 1].sum(0) / M)
    xh, u, bu, r, g = R._bn_pre(z, mean, var, gamma, beta, eps)
    a = R._d(slope).reshape(1, C, 1, 1)
    pos = u > 0
    amb = (u.abs() <= bu).to(torch.float64)
    du = torch.where(pos, dy, a * dy)
    bdu = R.U * (a * dy).abs() + amb * (1 - a).abs() * dy.abs() + R.TINY
    bxh = xh.abs() * (R.RSQRT + 2 * R.U) + R.TINY
    gr = g * r
    dz = gr * (du - m1 - xh * m2)
    core = bdu + 5 * R.U * du.abs() + bxh * m2.abs() + 6 * R.U * (m1.abs() + xh.abs() * m2.abs())
    bdz = gr.abs() * core + (dz.abs() + gr.abs() * amb * (1 - a).abs() * dy.abs()) * (R.RSQRT + 2 * R.U) + R.TINY
    if bf16:
        bdz = bdz * (1 + U_BF16) + U_BF16 * dz.abs()
    return {"dz": (dz, bdz)}
