"""Float64 reference and per-element error bound of every `csnet_train_*` entry point (include/csnet_b200.h).

Each function takes the values an entry point read (torch tensors on any device; they are evaluated in float64 on that
device) and returns {output name: (ref, bound)}: a kernel output `got` is correct when |got - ref| <= bound on every
element.  The semantics are those of the C ABI's comments (the F.* calls each entry point replaces); nothing here is
shared with sod100k_b200/train_ops.py or the kernels.

Bounds are per element and come from that element's own magnitude, never from the tensor's maximum.  For the bilinear
ops (convolution, resampling, their data and weight gradients) the magnitude m is the same linear map evaluated on |x|,
|w| and |dy| (the data / weight gradients: the VJP at those absolute values), and

    bound = depth * 2^-24 * m + depth * 2^-126

where `depth` is the longest chain of fp32 roundings any one term of the sum can pass through: the accumulation chain of
one thread plus the tree / partial merges that follow.  An fp32 evaluation whose every term passes through at most
`depth` roundings is within depth * 2^-24 * sum |terms| (first order; the second-order term is far below the slack the
constants below carry).  2^-126 per rounding covers underflow, where relative bounds do not hold.  The depths are
functions of the shape only and are given in each function's docstring; they are upper bounds over every launch form the
entry point may choose (the generic kernel and the register-tiled one), taking the GPU's SM count (`sms`, 132 on an
H100 SXM) as the one device constant.

`defect=` applies one realistic kernel mistake to the reference (tests/test_trainref_cpu.py checks that each is flagged on
the inputs the GPU test uses):
    drop_last_channel   the last input channel of a sum (the last output channel, for a data gradient) is left out
    drop_image          the last image is left out of a batch reduction (weight gradients, BatchNorm statistics / sums)
    drop_border         the operand's last row is read as zero (a row band or halo that misses the border)
    drop_partial        the last partial of a reduction is lost (the last row of the last image; BCE: the last 2048 logits)
    resample_shift      the bilinear taps are shifted by one source pixel
    slice_shift         a channel slice starts one channel late (c0 + 1)
    pool_last_max       a max-pool tie takes the last maximum instead of the first
    frozen_terms        frozen BatchNorm backward keeps the batch-statistic terms
    no_bias_correction  Adam without its bias corrections
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F

U = 2.0 ** -24                      # fp32 unit roundoff
TINY = 2.0 ** -126                  # absolute error of one fp32 operation near underflow
RSQRT = 2.0 ** -21                  # relative error of rsqrtf(var + eps) (rsqrtf: 2 ulp, plus the rounding of the sum)
SMS = 132                           # streaming multiprocessors of an H100 SXM
DEFECTS = ("drop_last_channel", "drop_image", "drop_border", "drop_partial", "resample_shift", "slice_shift",
           "pool_last_max", "frozen_terms", "no_bias_correction")


def _d(t):
    return t.detach().to(torch.float64)


def _cdiv(a, b):
    return -(-a // b)


def _bound(m, depth):
    return depth * U * m + depth * TINY


def check(got, ref, bound):
    """q = max |got - ref| / bound and a description of the worst element (NaN / inf in `got` give q = inf)."""
    got = _d(got).to(ref.device)
    ratio = (got - ref).abs() / bound
    ratio = torch.where(torch.isfinite(got), ratio, torch.full_like(ratio, float("inf")))
    flat = ratio.reshape(-1)
    i = int(torch.argmax(flat))
    q = float(flat[i])
    idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), tuple(ratio.shape))) if ratio.dim() else ()
    return q, (f"q={q:.3g} at {idx} of {tuple(ratio.shape)}: got {float(got[idx]):.7g} ref {float(ref[idx]):.7g} "
               f"bound {float(bound[idx]):.3g}")


# ---- shape-only chain lengths ------------------------------------------------------------------------------------------
def wgrad_depth(N, H, W, cin, cout, k, sms=SMS):
    """Longest rounding chain of one weight-gradient element (csnet_train_mix_wgrad), the larger of:
      * the generic kernel: z = min(N, 32) image splits; a thread sums ceil(N / z) * ceil(H W / 256) products, the
        256-thread block tree adds 10 levels, the z block sums are added atomically in any order (z);
      * the register-tiled kernel + its partial merge: a block owns a share ceil(units / gx) of the (image, row band)
        units, units = N ceil(H / R), gx = min(units, 2 sms / groups) blocks, groups = ceil(tiles / 256) (tiles =
        ceil(cin / 4) ceil(cout / 4), x 3 for 3x3); a thread adds one 4-product group per quad of its pixel split
        (<= R ceil(W / 4) quads per unit), the pixel splits (<= 256) are added in order, and the gx partials are merged
        by 4 interleaved sums (ceil(gx / 4) + 2).  R is the row band (1..16); the bound takes the worst R."""
    z = min(N, 32)
    generic = _cdiv(N, z) * _cdiv(H * W, 256) + 10 + z
    kt = 3 if k == 3 else 1
    tiles = _cdiv(cin, 4) * kt * _cdiv(cout, 4)
    groups = _cdiv(tiles, 256) if tiles > 256 else 1
    quads = _cdiv(W, 4)
    fast = 0
    for R in range(1, min(16, H) + 1):
        units = N * _cdiv(H, R)
        gx = max(1, min(units, 2 * sms // groups))
        fast = max(fast, 3 + _cdiv(units, gx) * R * quads + 256 + _cdiv(gx, 4) + 2)
    return max(generic, fast) + 1


def dw_wgrad_depth(N, C, H, W, sms=SMS):
    """Longest rounding chain of one depthwise weight-gradient element (csnet_train_dw_wgrad / dw_bwd): tasks = N bands
    ceil(W / 4) 4-pixel strips of rows = min(H, 8) rows; bx = min(ceil(tasks / 256), max(1, 4 sms / C)) blocks per channel
    (dw_bwd allows 8 sms / C: more blocks, shorter chains); a thread's chain is ceil(tasks / (256 bx)) strips of 4 rows
    FMAs, then a 5-level warp tree, 8 warp sums in order, the bx partials by 4 interleaved sums and the scale product."""
    quads, rows = _cdiv(W, 4), min(H, 8)
    tasks = N * _cdiv(H, rows) * quads
    bx_max = _cdiv(tasks, 256)
    bx_min = min(bx_max, max(1, 4 * sms // C))
    return _cdiv(tasks, 256 * bx_min) * 4 * rows + 5 + 8 + _cdiv(bx_max, 4) + 2 + 1


def bn_parts_max(N, C):
    """Partials per channel of the BatchNorm reductions: N images x S segments, S = 1 or S < 64 with N C S < 2 x 1184."""
    return min(64 * N, max(N, _cdiv(2 * 1184, C)))


def bn_thread_depth(HW):
    """One thread of a BatchNorm reduction: ceil(HW / 256) elements (float4 groups add 3 levels), then the 256-thread tree
    (5 shuffle levels in each of two warp sums)."""
    return _cdiv(HW, 256) + 3 + 10


def bce_depth(n):
    """BCE loss: blocks = min(ceil(n / 2048), 1184); a thread sums ceil(n / (256 blocks)) terms, the block tree adds 10
    levels, the scaling by 1 / n one, and the block sums are added atomically in any order (blocks)."""
    blocks = max(1, min(_cdiv(n, 2048), 1184))
    return _cdiv(n, 256 * blocks) + 10 + 1 + blocks + 1


# ---- convolution helpers (unfold / fold, chunked over images) ------------------------------------------------------------
_CHUNK = 1 << 27                    # float64 elements of one unfolded chunk


def _img_chunks(N, per_image):
    step = max(1, _CHUNK // max(1, per_image))
    return [(a, min(N, a + step)) for a in range(0, N, step)]


def _conv_fwd(x, wf, k, dil, pad, stride, Ho, Wo):
    """Cross-correlation: x [N, cin, H, W], wf [cin * k * k, cout] -> [N, cout, Ho, Wo]."""
    N = x.shape[0]
    out = []
    for a, b in _img_chunks(N, wf.shape[0] * Ho * Wo):
        cols = F.unfold(x[a:b], k, dilation=dil, padding=pad, stride=stride)
        out.append(torch.einsum("nkl,ko->nol", cols, wf).reshape(b - a, wf.shape[1], Ho, Wo))
    return torch.cat(out)


def _conv_dgrad(dy, wf, k, dil, pad, stride, Hs, Ws):
    """Adjoint of _conv_fwd with respect to x: dy [N, cout, Ho, Wo] -> [N, cin, Hs, Ws]."""
    N, cout, Ho, Wo = dy.shape
    Hf = (Ho - 1) * stride + dil * (k - 1) + 1 - 2 * pad          # rows the sliding window covers; the rest gets nothing
    Wf = (Wo - 1) * stride + dil * (k - 1) + 1 - 2 * pad
    Hf, Wf = max(Hf, Hs), max(Wf, Ws)
    out = []
    for a, b in _img_chunks(N, wf.shape[0] * Ho * Wo):
        cols = torch.einsum("ko,nol->nkl", wf, dy[a:b].reshape(b - a, cout, Ho * Wo))
        out.append(F.fold(cols, (Hf, Wf), k, dilation=dil, padding=pad, stride=stride)[:, :, :Hs, :Ws])
    return torch.cat(out)


def _conv_wgrad(x, dy, k, dil, pad, stride):
    """Weight gradient in kernel layout [cin, k * k, cout]."""
    N, cin = x.shape[:2]
    cout, Ho, Wo = dy.shape[1:]
    acc = torch.zeros(cin * k * k, cout, dtype=torch.float64, device=x.device)
    for a, b in _img_chunks(N, cin * k * k * Ho * Wo):
        cols = F.unfold(x[a:b], k, dilation=dil, padding=pad, stride=stride)
        acc += torch.einsum("nkl,nol->ko", cols, dy[a:b].reshape(b - a, cout, Ho * Wo))
    return acc.reshape(cin, k * k, cout)


def bilinear_matrix(n_in, up, shift=False, device="cpu"):
    """[n_in * up, n_in]: F.interpolate(scale_factor=up, mode='bilinear', align_corners=False) along one axis; source index
    (d + 0.5) / up - 0.5 clamped at 0, upper tap clamped at the border.  shift: taps one source pixel to the right."""
    n_out = n_in * up
    M = torch.zeros(n_out, n_in, dtype=torch.float64)
    for d in range(n_out):
        s = max((d + 0.5) / up - 0.5, 0.0)
        i0 = min(int(s), n_in - 1)
        i1 = min(i0 + 1, n_in - 1)
        l = s - i0
        if shift:
            i0, i1 = min(i0 + 1, n_in - 1), min(i1 + 1, n_in - 1)
        M[d, i0] += 1.0 - l
        M[d, i1] += l
    return M.to(device)


def _zero_last_row(x):
    x = x.clone()
    x[..., -1, :] = 0.0
    return x


# ---- MIX paths ---------------------------------------------------------------------------------------------------------
@dataclass
class Path:
    """One csnet_train_path: src [N, Cs, Hs, Ws]; w [cin, k*k, cout] (None for a resample-add path, ksize 0)."""
    src: torch.Tensor
    w: Optional[torch.Tensor]
    cin: int
    cout: int
    c0: int = 0
    cout0: int = 0
    ksize: int = 1
    dil: int = 1
    stride: int = 1
    pad: int = 0
    up: int = 1


def _slice(p: Path, defect):
    c0 = p.c0
    if defect == "slice_shift":                   # one channel late where the source has room, else one early
        c0 = c0 + 1 if c0 + p.cin < p.src.shape[1] else max(c0 - 1, 0)
    return _d(p.src[:, c0:c0 + p.cin])


def mix_fwd(paths, C, H, W, defect=None):
    """csnet_train_mix_fwd: dst[N, C, H, W] = sum of paths; channels no path writes are 0.
    A conv path adds conv(src[c0:c0+cin], w) (zero padding `pad`, dilation, stride) to dst[cout0:cout0+cout]; a resample
    path (ksize 0) adds the bilinear x up of src[c0 + c] to dst[cout0 + c], c < cout.
    depth = sum over conv paths of cin k^2 (one accumulation chain) + 5 per resample path (four products and three adds
    of the blend, one add into the chain) + 2."""
    N, dev = paths[0].src.shape[0], paths[0].src.device
    v = torch.zeros(N, C, H, W, dtype=torch.float64, device=dev)
    m = torch.zeros_like(v)
    depth, first_conv = 2, True
    for p in paths:
        x = _slice(p, defect)
        sl = slice(p.cout0, p.cout0 + p.cout)
        if p.ksize == 0:
            Mh = bilinear_matrix(x.shape[2], p.up, defect == "resample_shift", dev)
            Mw = bilinear_matrix(x.shape[3], p.up, defect == "resample_shift", dev)
            up = lambda t: torch.einsum("yi,nciw,xw->ncyx", Mh, t, Mw)
            v[:, sl] += up(x[:, :p.cout])
            m[:, sl] += up(x[:, :p.cout].abs())
            depth += 5
            continue
        if first_conv and defect == "drop_last_channel":
            x = x.clone()
            x[:, -1] = 0.0
        if defect == "drop_border":
            x = _zero_last_row(x)
        first_conv = False
        k = p.ksize
        wf = _d(p.w).reshape(p.cin * k * k, p.cout)
        v[:, sl] += _conv_fwd(x, wf, k, p.dil, p.pad, p.stride, H, W)
        m[:, sl] += _conv_fwd(x.abs(), wf.abs(), k, p.dil, p.pad, p.stride, H, W)
        depth += p.cin * k * k
    return {"dst": (v, _bound(m, depth))}


def mix_dgrad(ddst, p: Path, defect=None):
    """csnet_train_mix_dgrad: dsrc [N, cin, Hs, Ws], the gradient of mix_fwd with respect to src[c0:c0+cin] for one path.
    conv path: depth = cout k^2 + 2 (one chain over output channels and taps);
    resample path: the transposed bilinear map, depth = (2 up)^2 + 3 (the destination pixels that can reach one source
    pixel, each through a two-factor weight)."""
    Hs, Ws = p.src.shape[2], p.src.shape[3]
    dy = _d(ddst[:, p.cout0:p.cout0 + p.cout])
    if defect == "drop_border":
        dy = _zero_last_row(dy)
    if p.ksize == 0:
        Mh = bilinear_matrix(Hs, p.up, defect == "resample_shift", dy.device)
        Mw = bilinear_matrix(Ws, p.up, defect == "resample_shift", dy.device)
        adj = lambda t: torch.einsum("yi,ncyx,xw->nciw", Mh, t, Mw)
        return {"dsrc": (adj(dy), _bound(adj(dy.abs()), (2 * p.up) ** 2 + 3))}
    if defect == "drop_last_channel":
        dy = dy.clone()
        dy[:, -1] = 0.0
    k = p.ksize
    wf = _d(p.w).reshape(p.cin * k * k, p.cout)
    v = _conv_dgrad(dy, wf, k, p.dil, p.pad, p.stride, Hs, Ws)
    m = _conv_dgrad(dy.abs(), wf.abs(), k, p.dil, p.pad, p.stride, Hs, Ws)
    return {"dsrc": (v, _bound(m, p.cout * k * k + 2))}


def mix_wgrad(ddst, p: Path, sms=SMS, defect=None):
    """csnet_train_mix_wgrad: dw [cin, k*k, cout] = sum over (n, y, x) of src * ddst (kernel layout).
    depth = wgrad_depth(N, H, W, cin, cout, k) (H, W: the destination's)."""
    x = _slice(p, None)
    dy = _d(ddst[:, p.cout0:p.cout0 + p.cout])
    if defect == "drop_image":
        x = x.clone()
        x[-1] = 0.0
    if defect == "drop_partial":
        dy = dy.clone()
        dy[-1, :, -1, :] = 0.0
    k = p.ksize
    v = _conv_wgrad(x, dy, k, p.dil, p.pad, p.stride)
    m = _conv_wgrad(x.abs(), dy.abs(), k, p.dil, p.pad, p.stride)
    N, _, H, W = ddst.shape
    return {"dw": (v, _bound(m, wgrad_depth(N, H, W, p.cin, p.cout, k, sms)))}


# ---- depthwise 3x3 ---------------------------------------------------------------------------------------------------
def _dw3(x, w9):
    """y[n, c] = sum over taps of w9[c, t] * x[n, c, y + ky - 1, x + kx - 1] (zero padding)."""
    H, W = x.shape[2:]
    xp = F.pad(x, (1, 1, 1, 1))
    y = torch.zeros_like(x)
    for t in range(9):
        ky, kx = divmod(t, 3)
        y += w9[None, :, t, None, None] * xp[:, :, ky:ky + H, kx:kx + W]
    return y


def dw_conv(x, w, scale, transposed=0, defect=None):
    """csnet_train_dw_conv: y = depthwise 3x3 (pad 1) with weights scale * w[C][9]; transposed: the data gradient, i.e. the
    same with the taps flipped.  depth = 9 FMAs + the scale product + 1 = 11."""
    x = _d(x)
    if defect == "drop_border":
        x = _zero_last_row(x)
    w9 = _d(w).reshape(-1, 9) * float(scale)
    if transposed:
        w9 = w9.flip(1)
    return {"y": (_dw3(x, w9), _bound(_dw3(x.abs(), w9.abs()), 11))}


def _dw_wgrad(x, dy):
    H, W = x.shape[2:]
    xp = F.pad(x, (1, 1, 1, 1))
    return torch.stack([(dy * xp[:, :, ky:ky + H, kx:kx + W]).sum((0, 2, 3)) for ky in range(3) for kx in range(3)], 1)


def dw_wgrad(x, dy, scale, sms=SMS, defect=None):
    """csnet_train_dw_wgrad: dw[c][ky*3+kx] = scale * sum over (n, y, x) of dy[n,c,y,x] x[n,c,y+ky-1,x+kx-1].
    depth = dw_wgrad_depth(N, C, H, W)."""
    x, dy = _d(x), _d(dy)
    if defect == "drop_image":
        x = x.clone()
        x[-1] = 0.0
    if defect == "drop_partial":
        dy = dy.clone()
        dy[-1, :, -1, :] = 0.0
    s = abs(float(scale))
    N, C, H, W = x.shape
    return {"dw": (float(scale) * _dw_wgrad(x, dy), _bound(s * _dw_wgrad(x.abs(), dy.abs()), dw_wgrad_depth(N, C, H, W, sms)))}


def dw_bwd(x, dy, w, scale, sms=SMS, defect=None):
    """csnet_train_dw_bwd: dx = dw_conv(dy, w, scale, transposed=1) and dw = dw_wgrad(x, dy, scale)."""
    return {"dx": dw_conv(dy, w, scale, 1, defect if defect == "drop_border" else None)["y"],
            "dw": dw_wgrad(x, dy, scale, sms, defect if defect != "drop_border" else None)["dw"]}


# ---- BatchNorm (train) + PReLU ---------------------------------------------------------------------------------------
def _bn_defect_z(z, defect):
    if defect == "drop_image":
        return z[:-1]
    return z


def bn_stats(z, defect=None):
    """csnet_train_bn_stats: per-channel mean and biased variance over (N, HW).  The kernel sums z - K and (z - K)^2 in
    fp32 with a shift K (an fp32 mean of 32 of the samples, so |K - mean| <= max|z - mean| + 31 u max|z|) and merges its
    partials in float64.  With D = bn_thread_depth(HW) + 1, d = z - K:
        |d mean| <= (D + 1) u E|d| + u |mean|
        |d var|  <= (D + 3) u E[d^2] + 2 |K - mean| dm + dm^2 + u var,   dm = (D + 1) u E|d|
    where E|d| <= E|z - mean| + |K - mean| and E[d^2] = var + (K - mean)^2."""
    z = _d(z)
    N, C = z.shape[:2]
    zc = z.transpose(0, 1).reshape(C, -1)
    if defect == "drop_image":
        zd = z[:-1].transpose(0, 1).reshape(C, -1)
    elif defect == "drop_partial":
        zd = torch.cat([z[:-1].transpose(0, 1).reshape(C, -1), z[-1, :, :-1].reshape(C, -1)], 1)
    else:
        zd = zc
    mean = zd.mean(1)
    var = ((zd - mean[:, None]) ** 2).mean(1)
    mu = zc.mean(1)
    dev = (zc - mu[:, None]).abs()
    dK = dev.amax(1) + 31 * U * zc.abs().amax(1)
    D = bn_thread_depth(z[0, 0].numel()) + 1
    Ed, Ed2 = dev.mean(1) + dK, ((zc - mu[:, None]) ** 2).mean(1) + dK ** 2
    dm = (D + 1) * U * Ed
    bmean = dm + U * mu.abs() + TINY
    bvar = (D + 3) * U * Ed2 + 2 * dK * dm + dm ** 2 + U * ((zc - mu[:, None]) ** 2).mean(1) + TINY
    return {"mean": (mean, bmean), "var": (var, bvar)}


def _bn_pre(z, mean, var, gamma, beta, eps):
    """xhat, u = gamma xhat + beta and the bound of u (the kernel: r = rsqrtf(var + eps), g = gamma r, b = beta - mean g,
    u = z g + b)."""
    C = z.shape[1]
    e = lambda t: _d(t).reshape(1, C, 1, 1)
    mu, r, g, b = e(mean), 1.0 / torch.sqrt(e(var) + float(eps)), e(gamma), e(beta)
    xh = (z - mu) * r
    u = g * xh + b
    bu = (RSQRT + 4 * U) * g.abs() * r * (z.abs() + mu.abs()) + 4 * U * (b.abs() + u.abs()) + 4 * TINY
    return xh, u, bu, r, g


def bn_prelu_fwd(z, mean, var, gamma, beta, slope, eps, defect=None):
    """csnet_train_bn_prelu_fwd: y = PReLU(gamma (z - mean) / sqrt(var + eps) + beta) with the given mean / var, and
    gap[n, c] = mean over HW of y.  bound(y) = max(1, |slope|) bound(u) + u |y|; gap: the mean of bound(y) plus
    (bn_thread_depth(HW) + 1) u mean|y| + u |gap|."""
    z = _d(z)
    N, C, H, W = z.shape
    xh, u, bu, _, _ = _bn_pre(z, mean, var, gamma, beta, eps)
    a = _d(slope).reshape(1, C, 1, 1)
    y = torch.where(u > 0, u, a * u)
    by = torch.clamp(a.abs(), min=1.0) * bu + U * y.abs() + TINY
    ys = y[:, :, :-1] if defect == "drop_partial" else y
    gap = ys.sum((2, 3)) / (H * W)
    HW = H * W
    bgap = by.mean((2, 3)) + (bn_thread_depth(HW) + 1) * U * y.abs().mean((2, 3)) + U * gap.abs() + TINY
    return {"y": (y, by), "gap": (gap, bgap)}


def bn_prelu_bwd(z, dy, mean, var, gamma, beta, slope, eps, frozen, parts=None, defect=None):
    """csnet_train_bn_prelu_bwd: autograd of bn_prelu_fwd with batch statistics (frozen = 0) or constant mean / var
    (frozen = 1).  With u, xhat as in the forward, du = dy (u > 0) or slope dy:
        dbeta = sum du,  dgamma = sum du xhat,  dslope = sum over u <= 0 of dy u,
        dz = gamma r (du - dbeta / M - xhat dgamma / M)   (frozen: gamma r du),  M = N HW.
    An element whose u lies within its own bound of 0 may take either PReLU branch in fp32: its |1 - slope| |dy| (and for
    dslope |dy u|) is added to the bounds.  The sums have depth D = bn_thread_depth(HW) + bn_parts_max(N, C) (the
    partials are merged in fp32; `parts` overrides the partial count, for a reference run on a slice of the channels);
    dz adds gamma r (bound(dbeta) + |xhat| bound(dgamma)) / M, the propagated errors of the kernel's own reductions."""
    z, dy = _d(z), _d(dy)
    N, C, H, W = z.shape
    xh, u, bu, r, g = _bn_pre(z, mean, var, gamma, beta, eps)
    a = _d(slope).reshape(1, C, 1, 1)
    pos = u > 0
    amb = (u.abs() <= bu).to(torch.float64)
    du = torch.where(pos, dy, a * dy)
    bdu = U * (a * dy).abs() + amb * (1 - a).abs() * dy.abs() + TINY
    bxh = xh.abs() * (RSQRT + 2 * U) + TINY
    mask = lambda t: t[:-1] if defect == "drop_image" else t
    S = lambda t: mask(t).sum((0, 2, 3))
    Sa = lambda t: t.sum((0, 2, 3))
    D = bn_thread_depth(H * W) + (bn_parts_max(N, C) if parts is None else parts)
    neg = (~pos).to(torch.float64)
    dbeta, dgamma, dslope = S(du), S(du * xh), S(dy * u * neg)
    b_dbeta = Sa(bdu) + D * U * Sa(du.abs())
    b_dgamma = Sa(bdu * xh.abs() + du.abs() * bxh) + (D + 1) * U * Sa((du * xh).abs())
    nb = torch.clamp(neg + amb, max=1.0)
    b_dslope = Sa(dy.abs() * bu * nb) + (D + 1) * U * Sa((dy * u).abs() * nb) + Sa(amb * (dy * u).abs())
    M = N * H * W
    e = lambda t: t.reshape(1, C, 1, 1)
    frozen_eff = (not frozen) if defect == "frozen_terms" else bool(frozen)
    gr = g * r
    if frozen_eff:
        dz = gr * du
    else:
        dz = gr * (du - e(dbeta) / M - xh * e(dgamma) / M)
    m1, m2 = e(dbeta).abs() / M, e(dgamma).abs() / M
    core = bdu + 5 * U * du.abs()
    if not frozen:
        core = core + e(b_dbeta) / M + xh.abs() * e(b_dgamma) / M + bxh * m2 + 5 * U * (m1 + xh.abs() * m2)
    # On an ambiguous element (|u| within its bound of 0) the kernel may take the other PReLU branch: |1 - slope| |dy| is
    # then almost all of that element's bound, so a kernel that flipped the branch sits at q just below 1 by construction.
    # The relative rounding applies to the kernel's value, which on such an element is the other branch's.
    bdz = gr.abs() * core + (dz.abs() + gr.abs() * amb * (1 - a).abs() * dy.abs()) * (RSQRT + 2 * U) + TINY
    return {"dz": (dz, bdz), "dgamma": (dgamma, b_dgamma + TINY), "dbeta": (dbeta, b_dbeta + TINY),
            "dslope": (dslope, b_dslope + TINY)}


# ---- pooling ---------------------------------------------------------------------------------------------------------
def pool_fwd(src, c0, cin, pre_avg, pool, defect=None):
    """csnet_train_pool_fwd: dst [N, cin, Hs / f, Ws / f], f = (pre_avg ? 2 : 1) pool, the max over pool x pool windows of
    (pre_avg ? the 2x2 mean : the value) of src[c0:c0+cin]; rows / columns past f * (Hs / f) are not read.
    The 2x2 mean is three fp32 adds and an exact quarter: bound 3 u (its mean of |values|); a plain max copies a value
    (bound 0, plus the tiny absolute term).  Also returns "idx": (first, admissible), the row-major position of the first
    exact maximum of each window and the positions whose value lies within twice the bound of the maximum; the kernel's
    idx must be admissible and not later than `first` (pool_last_max: first is the LAST exact maximum).  With pre_avg the
    compared values are fp32 averages: where every partial sum of every 2x2 cell of a window is exact in fp32 (in any
    order: all 16 subset sums are fp32 values), they equal the float64 averages and the first-maximum rule holds; in any
    other window rounding may order a float64 tie either way, so `first` is the window's last position there."""
    x = _d(src[:, c0:c0 + cin])
    N = x.shape[0]
    f = (2 if pre_avg else 1) * pool
    Hc, Wc = x.shape[2] // f, x.shape[3] // f
    x = x[:, :, :Hc * f, :Wc * f]
    if pre_avg:
        t = x.reshape(N, cin, Hc * pool, 2, Wc * pool, 2)
        a, am = t.mean((3, 5)), t.abs().mean((3, 5))
        ba = 3 * U * am + TINY
    else:
        a, ba = x, torch.full_like(x, TINY)
    win = lambda t: t.reshape(N, cin, Hc, pool, Wc, pool).permute(0, 1, 2, 4, 3, 5).reshape(N, cin, Hc, Wc, pool * pool)
    aw, bw = win(a), win(ba)
    v = aw.amax(-1)
    b = bw.amax(-1)
    exact = aw == v[..., None]
    pos = torch.arange(pool * pool, device=x.device)
    if defect == "pool_last_max":
        first = torch.where(exact, pos, -1).amax(-1)
    else:
        first = torch.where(exact, pos, pool * pool).amin(-1)
    if pre_avg:
        cells = t.permute(0, 1, 2, 4, 3, 5).reshape(N, cin, Hc * pool, Wc * pool, 4)
        subsets = torch.tensor([[(m >> i) & 1 for i in range(4)] for m in range(16)], dtype=torch.float64, device=x.device)
        sums = cells @ subsets.T
        exact_cell = (sums.float().double() == sums).all(-1)
        first = torch.where(win(exact_cell).all(-1), first, torch.full_like(first, pool * pool - 1))
    admissible = aw >= v[..., None] - 2 * b[..., None]
    return {"dst": (v, b), "idx": (first, admissible)}


def check_idx(got_idx, first, admissible):
    """Number of windows whose recorded arg-max is not admissible or comes after the first exact maximum."""
    return sum(idx_violations(got_idx, first, admissible))


def idx_violations(got_idx, first, admissible):
    """(windows whose recorded position is not admissible, windows whose position comes after the first exact maximum)."""
    k = got_idx.to(torch.int64).to(first.device)
    adm = admissible.gather(-1, k.clamp(0, admissible.shape[-1] - 1)[..., None])[..., 0] & (k < admissible.shape[-1])
    return int((~adm).sum()), int((adm & (k > first)).sum())


def pool_bwd(dpool, idx, Hs, Ws, pre_avg, pool, defect=None):
    """csnet_train_pool_bwd: dsrc [N, cin, Hs, Ws] routes dpool to the window position idx records (pool > 1) and, with
    pre_avg, a quarter of it to each pixel of that 2x2 cell; pixels no window reads get 0.  Exact (bound: tiny)."""
    g = _d(dpool)
    if defect == "drop_border":
        g = _zero_last_row(g)
    N, cin, Hc, Wc = g.shape
    if pool > 1:
        k = idx.to(torch.int64).to(g.device)
        oh = F.one_hot(k, pool * pool).to(torch.float64).reshape(N, cin, Hc, Wc, pool, pool)
        g = (g[..., None, None] * oh).permute(0, 1, 2, 4, 3, 5).reshape(N, cin, Hc * pool, Wc * pool)
    if pre_avg:
        g = 0.25 * g.repeat_interleave(2, 2).repeat_interleave(2, 3)
    out = torch.zeros(N, cin, Hs, Ws, dtype=torch.float64, device=g.device)
    out[:, :, :g.shape[2], :g.shape[3]] = g
    return {"dsrc": (out, torch.full_like(out, TINY))}


# ---- loss, optimiser ---------------------------------------------------------------------------------------------------
def bce(logits, target, grad_scale=1.0, defect=None):
    """csnet_train_bce: loss = mean(max(z, 0) - z t + log1p(exp(-|z|))), dlogits = (sigmoid(z) - t) / n * grad_scale.
    One term is within 6 u (|max(z, 0)| + |z t| + log1p(exp(-|z|))) (expf / log1pf to 2 ulp); the loss adds
    bce_depth(n) u of the summed magnitudes over n.  dlogits: sigmoid to 4 u relative, the difference, 1 / n and the
    scale products: (4 u sigmoid + 6 u |sigmoid - t|) |grad_scale| / n."""
    z, t = _d(logits).reshape(-1), _d(target).reshape(-1)
    n = z.numel()
    l = torch.log1p(torch.exp(-z.abs()))
    term = torch.clamp(z, min=0) - z * t + l
    mag = torch.clamp(z, min=0) + (z * t).abs() + l
    ts = term[:-2048] if defect == "drop_partial" else term
    loss = ts.sum() / n
    bloss = (6 * U * mag.sum() + bce_depth(n) * U * mag.sum()) / n + U * loss.abs() + TINY
    sig = torch.sigmoid(z)
    gs = float(grad_scale)
    dl = (sig - t) / n * gs
    bdl = (4 * U * sig + 6 * U * (sig - t).abs()) * abs(gs) / n + 4 * TINY
    shape = logits.shape
    return {"loss": (loss, bloss), "dlogits": (dl.reshape(shape), bdl.reshape(shape))}


def adam(params, grads, weight_decays, lr, betas, eps, grad_scales, defect=None):
    """csnet_train_adam over several steps: params = initial tensors, grads[s][i] = the fp32 gradient of tensor i at step
    s (scaled by grad_scales[s]), weight_decays[i] = its group's L2 decay; torch.optim.Adam semantics:
        g = grad * scale + wd p,  m = b1 m + (1 - b1) g,  v = b2 v + (1 - b2) g^2,
        p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps).
    Pass the hyper-parameters as the fp32 values the kernel receives.  The bound is propagated step by step next to the
    values: magnitudes G = |grad scale| + |wd p|, bounds of g (3 u G + wd bound(p)), m, v (their recursions plus 3-4 u of
    their magnitudes), the bias corrections from powf (2 ulp of b^t, relative to 1 - b^t), sqrt and the division to first
    order, and u |p| per stored parameter."""
    b1, b2 = betas
    P = [_d(p).clone() for p in params]
    BP = [torch.zeros_like(p) for p in P]
    Mv = [torch.zeros_like(p) for p in P]
    Vv = [torch.zeros_like(p) for p in P]
    Mm = [torch.zeros_like(p) for p in P]
    Vm = [torch.zeros_like(p) for p in P]
    Bm = [torch.zeros_like(p) for p in P]
    Bv = [torch.zeros_like(p) for p in P]
    for s, (gl, gs) in enumerate(zip(grads, grad_scales)):
        t = s + 1
        bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
        c2 = math.sqrt(bc2)
        dc1 = (2 * U * b1 ** t + U) / bc1
        dc2 = (2 * U * b2 ** t + U) / bc2 / 2 + U
        if defect == "no_bias_correction":
            bc1, c2 = 1.0, 1.0
        for i, wd in enumerate(weight_decays):
            p, g0 = P[i], _d(gl[i]).to(P[i].device)
            g = g0 * float(gs) + wd * p
            G = (g0 * float(gs)).abs() + abs(wd) * p.abs()
            Bg = 3 * U * G + abs(wd) * BP[i]
            Mv[i] = b1 * Mv[i] + (1 - b1) * g
            Vv[i] = b2 * Vv[i] + (1 - b2) * g * g
            Mm[i] = b1 * Mm[i] + (1 - b1) * G
            Vm[i] = b2 * Vm[i] + (1 - b2) * G * G
            Bm[i] = b1 * Bm[i] + (1 - b1) * Bg + 3 * U * Mm[i]
            Bv[i] = b2 * Bv[i] + (1 - b2) * (2 * G * Bg + Bg * Bg) + 4 * U * Vm[i]
            sv = torch.sqrt(Vv[i])
            bsq = torch.minimum(torch.sqrt(Bv[i]), Bv[i] / torch.clamp(sv, min=1e-300)) + U * sv
            den = sv / c2 + eps
            bden = bsq / c2 + sv / c2 * (dc2 + 2 * U) + U * den
            upd = lr / bc1 * Mv[i] / den
            rel = torch.clamp(bden / den, max=0.5)
            bupd = lr / bc1 * (Bm[i] / den + Mv[i].abs() * bden / den ** 2) / (1 - rel) + upd.abs() * (dc1 + 4 * U)
            P[i] = p - upd
            BP[i] = BP[i] + bupd + U * P[i].abs() + TINY
    return [(p, b) for p, b in zip(P, BP)]
