"""Float64 reference and per-element error bound of the CSF+Res2Net head's training entry points (csnet_train_conv_*, _bias_grad,
_gn_*, _resize_*; include/csnet_b200.h), in the style of tests/trainref.py: {output: (ref, bound)}, a kernel output `got` being
correct when |got - ref| <= bound element by element.

    bound = depth * 2^-24 * m + depth * 2^-126

m is the same linear map applied to |operands|; depth is the longest chain of fp32 roundings an output passes through, from the
shape and the launch (`chain` and `splits` as csnet_train_conv_plan reports them).  `defect=` applies one realistic kernel mistake to
the reference; the GPU test checks that each is flagged on its own inputs:
    drop_segment      a K segment of a conv sum is left out (fwd / dgrad)
    drop_partial      the last split-K partial of a weight gradient is lost (its last image's last pixel row)
    wrong_group       GroupNorm statistics taken over a group boundary shifted by one channel
    shifted_tap       the resize adjoint reads its taps one source pixel over
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24
TINY = 2.0 ** -126
RSQRT = 2.0 ** -21


def _d(t):
    return torch.as_tensor(t).detach().to(torch.float64)


def _bound(m, depth):
    return depth * U * m + depth * TINY


def _conv(x, w, dil):
    k = w.shape[2]
    return F.conv2d(x, w, padding=dil if k == 3 else 0, dilation=dil)


def _convT(dy, w, dil):
    k = w.shape[2]
    return F.conv_transpose2d(dy, w, padding=dil if k == 3 else 0, dilation=dil)


def conv_fwd(segs, bias=None, old=None, chain=1, splits=1, defect=None):
    """segs = [(x [N, cin, H, W], w [cout, cin, k, k], dil)]: bias + sum_s conv(x_s, w_s) (+ old)."""
    if defect == "drop_segment":
        segs = segs[:-1]
    ref = sum(_conv(_d(x), _d(w), dl) for x, w, dl in segs)
    m = sum(_conv(_d(x).abs(), _d(w).abs(), dl) for x, w, dl in segs)
    if bias is not None:
        ref = ref + _d(bias).view(1, -1, 1, 1)
        m = m + _d(bias).abs().view(1, -1, 1, 1)
    depth = chain + splits + 2
    if old is not None:
        ref = ref + _d(old)
        m = m + _d(old).abs()
    return ref, _bound(m, depth)


def conv_dgrad(segs, old=None, chain=1, splits=1, defect=None):
    """segs = [(dy [N, cout, H, W], w [cout, cin, k, k], dil)]: the gradient of sum_s conv(x, w_s) with respect to x."""
    if defect == "drop_segment":
        segs = segs[:-1]
    ref = sum(_convT(_d(dy), _d(w), dl) for dy, w, dl in segs)
    m = sum(_convT(_d(dy).abs(), _d(w).abs(), dl) for dy, w, dl in segs)
    if old is not None:
        ref, m = ref + _d(old), m + _d(old).abs()
    return ref, _bound(m, chain + splits + 2)


def conv_wgrad(x, dy, wshape, dil, old=None, chain=1, splits=1, defect=None):
    """Weight gradient of conv(x, w) [cout, cin, k, k] at output gradient dy."""
    x, dy = _d(x), _d(dy)
    if defect == "drop_partial":
        dy = dy.clone()
        dy[-1, :, -1] = 0
    k = wshape[2]
    pad = dil if k == 3 else 0
    ref = torch.nn.grad.conv2d_weight(x, wshape, dy, padding=pad, dilation=dil)
    m = torch.nn.grad.conv2d_weight(x.abs(), wshape, dy.abs(), padding=pad, dilation=dil)
    if old is not None:
        ref, m = ref + _d(old), m + _d(old).abs()
    return ref, _bound(m, chain + splits + 2)


def bias_grad(dy):
    """sum over images and pixels; a 256-thread tree per image plane, then the images in order."""
    dy = _d(dy)
    n, c, h, w = dy.shape
    depth = math.ceil(h * w / 256) + 8 + 5 + n + 1
    return dy.sum(dim=(0, 2, 3)), _bound(dy.abs().sum(dim=(0, 2, 3)), depth)


# ---- GroupNorm + PReLU ---------------------------------------------------------------------------------------------------
def _groups(z, G, defect):
    n, c, h, w = z.shape
    if defect == "wrong_group":                       # boundaries one channel late: the group of channel c starts at g Cg + 1
        return torch.roll(z, -1, 1), 1
    return z, 0


def _gn64(z, G, gamma, beta, a, eps, defect=None):
    z = _d(z)
    zz, sh = _groups(z, G, defect)
    n, c, h, w = z.shape
    g = zz.reshape(n, G, -1)
    mean, var = g.mean(-1, keepdim=True), g.var(-1, unbiased=False, keepdim=True)
    xh = ((g - mean) / torch.sqrt(var + eps)).reshape(n, c, h, w)
    if sh:
        xh = torch.roll(xh, 1, 1)
    u = xh * _d(gamma).view(1, -1, 1, 1) + _d(beta).view(1, -1, 1, 1)
    return u, xh


def gn_prelu_fwd(z, G, gamma, beta, a, eps=1e-5, defect=None):
    """y = PReLU(GroupNorm(z)).  Error of u: the statistics' (gn_stats' bound, rsqrtf's 2^-21) and 4 roundings of the affine;
    PReLU multiplies it by at most max(1, |a|) (a branch flip at the kink is within the error of u)."""
    u, xh = _gn64(z, G, gamma, beta, a, eps, defect)
    aa = _d(a).view(1, -1, 1, 1)
    y = torch.where(u > 0, u, aa * u)
    z64 = _d(z)
    n, c, h, w = z64.shape
    L = (c // G) * h * w
    g = z64.reshape(n, G, -1)
    dev = (g - g.mean(-1, keepdim=True)).abs().amax(-1)
    var = g.var(-1, unbiased=False)
    r = 1 / torch.sqrt(var + eps)
    depth = math.ceil(L / 512) + 4
    rel_r = RSQRT + (_bound(8 * dev * dev, depth) + 4 * U * var) / (2 * (var + eps))      # relative error of r
    err_mean = _bound(2 * dev, depth) + 2 * U * g.mean(-1).abs()
    rg = lambda t: t.repeat_interleave(c // G, 1).view(n, c, 1, 1)
    gm = _d(gamma).abs().view(1, -1, 1, 1)
    eu = gm * (xh.abs() * (rg(rel_r) + 3 * U) + rg(r * err_mean)) + 2 * U * u.abs() + TINY
    return y, torch.maximum(aa.abs(), torch.ones_like(aa)) * eu * 1.5


def gn_prelu_bwd(z, dy, G, gamma, beta, a, eps=1e-5, defect=None):
    """float64 autograd of F.prelu(F.group_norm(...)): (dz, dgamma, dbeta, dslope), each with its bound.  The fp32 evaluation
    carries the forward's error of xhat and u into every term and adds the per-plane trees (ceil(HW / 256) + 13), the group sums
    over C / G channels in double and the image sums in order."""
    z64 = _d(z).requires_grad_(True)
    g64, b64, a64 = (_d(v).requires_grad_(True) for v in (gamma, beta, a))
    n, c, h, w = z64.shape
    zz = torch.roll(z64, -1, 1) if defect == "wrong_group" else z64
    y = F.group_norm(zz, G, None, None, eps)
    if defect == "wrong_group":
        y = torch.roll(y, 1, 1)
    y = F.prelu(y * g64.view(1, -1, 1, 1) + b64.view(1, -1, 1, 1), a64)
    dz, dg, db, da = torch.autograd.grad(y, (z64, g64, b64, a64), _d(dy))
    with torch.no_grad():
        u, xh = _gn64(z, G, gamma, beta, a, eps)
        _, eu = gn_prelu_fwd(z, G, gamma, beta, a, eps)
        aa = _d(a).view(1, -1, 1, 1)
        dyv = _d(dy)
        du = torch.where(u > 0, dyv, aa * dyv).abs() + (1 - aa).abs() * dyv.abs() * (u.abs() <= eu)
        gm = _d(gamma).abs().view(1, -1, 1, 1)
        g = z64.detach().reshape(n, G, -1)
        r = (1 / torch.sqrt(g.var(-1, unbiased=False) + eps)).repeat_interleave(c // G, 1).view(n, c, 1, 1)
        L = (c // G) * h * w
        t1 = (gm * du).reshape(n, G, -1).sum(-1) / L
        t2 = (gm * du * xh.abs()).reshape(n, G, -1).sum(-1) / L
        rg = lambda t: t.repeat_interleave(c // G, 1).view(n, c, 1, 1)
        depth = math.ceil(h * w / 256) + 13 + c // G + 8 + math.ceil(L / 512)
        xe = xh.abs() + 1
        m_dz = r * (gm * du + rg(t1) + xe * rg(t2)) * xe
        m_dg = (du * xe).sum(dim=(0, 2, 3))
        m_db = du.sum(dim=(0, 2, 3))
        m_da = (dyv.abs() * (u.abs() + eu)).sum(dim=(0, 2, 3))
        dd = depth + n + 8
        return (dz, _bound(m_dz, dd)), (dg, _bound(m_dg, dd)), (db, _bound(m_db, dd)), (da, _bound(m_da, dd))


# ---- bilinear resize (fp32 taps) -----------------------------------------------------------------------------------------
def tap_matrix(n_in: int, n_out: int, fma: bool = False) -> np.ndarray:
    """[n_out, n_in] float64 matrix of mae_tap's fp32 taps (image_io.cuh): row o holds l0 at i0 and l1 at i1.  fma=True rounds
    scale * (o + 0.5) - 0.5 once, as a contracted multiply-add does."""
    scale = np.float32(n_in) / np.float32(n_out)
    A = np.zeros((n_out, n_in))
    for o in range(n_out):
        if fma:
            src = np.float32(float(scale) * (o + 0.5) - 0.5)
        else:
            src = np.float32(np.float32(scale * np.float32(o + 0.5)) - np.float32(0.5))
        src = max(src, np.float32(0))
        i0 = int(src)
        i1 = i0 + 1 if i0 < n_in - 1 else i0
        l1 = np.float32(src - np.float32(i0))
        l0 = np.float32(np.float32(1) - l1)
        A[o, i0] += l0
        A[o, i1] += l1
    return A


def resize_bwd(dout, Hs, Ws, defect=None):
    """dsrc = Ay^T dout Ax with the kernel's fp32 taps.  Depth: the longest row (rx) and column (ry) ranges plus 3; 6 (Hs + Ws + 2)
    more rounding units cover a tap whose source coordinate the kernel rounds differently (a contracted multiply-add), as
    tests/resize_ref.py bounds the forward."""
    dout = _d(dout)
    Hd, Wd = dout.shape[2:]
    Ay, Ax = (torch.from_numpy(tap_matrix(Hs, Hd)), torch.from_numpy(tap_matrix(Ws, Wd)))
    Ay, Ax = Ay.to(dout.device), Ax.to(dout.device)
    if defect == "shifted_tap":
        Ax = torch.roll(Ax, 1, 1)
    ref = torch.einsum("yo,ncyx,xp->ncop", Ay, dout, Ax)
    m = torch.einsum("yo,ncyx,xp->ncop", Ay.abs(), dout.abs(), Ax.abs())
    ry, rx = int((Ay != 0).sum(0).max()), int((Ax != 0).sum(0).max())
    return ref, _bound(m, ry + rx + 3 + 6 * (Hs + Ws + 2))


def resize_fwd(src, Hd, Wd, old=None):
    """The RESIZE kernel's forward with the fp32 taps; the blend's 8 roundings and tests/resize_ref.py's tap term."""
    src = _d(src)
    Hs, Ws = src.shape[2:]
    Ay, Ax = (torch.from_numpy(tap_matrix(Hs, Hd)).to(src.device), torch.from_numpy(tap_matrix(Ws, Wd)).to(src.device))
    ref = torch.einsum("oy,ncyx,px->ncop", Ay, src, Ax)
    m = torch.einsum("oy,ncyx,px->ncop", Ay.abs(), src.abs(), Ax.abs())
    if old is not None:
        ref, m = ref + _d(old), m + _d(old).abs()
    return ref, _bound(m, 8 + 6 * (Hs + Ws + 2))
