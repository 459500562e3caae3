"""Float64 references and per-element bounds of the CSF+Res2Net head's bf16-storage calls (csnet_train_conv_*_bf16 on tensor cores,
csnet_train_gn_*_bf16, csnet_train_resize_*_bf16), on top of tests/trainref_r.py and tests/trainref_bf16.py.

Every reference is float64 evaluated on the kernel's own bf16 operands: bf16 activations, and the weights as the kernel reads them, the
fp32 parameters rounded to nearest-even bf16 (`round_bf16`).

Tensor-core GEMM.  An output element is c = sum_k a_k b_k over K products (K the k extent of the call: fwd sum of cin k^2 over the
segments, dgrad of cout k^2, wgrad N H W), then + bias, then + old.  Let m = sum_k |a_k b_k| (+ |bias| + |old|).
  * a_k b_k of two bf16 values (8-bit significands) is exact in fp32 (16 bits), and in the mma's wide product.
  * mma.sync.m16n8k16 adds 16 products to the fp32 accumulator per k16 step.  Whatever internal order and alignment the tensor core
    uses, its sum of 17 terms is within 2^-22 of their magnitude per term added (a relative 2^-23 per addition, with one guard bit
    lost to alignment); over the chain of one split every product is added once: at most K steps of 2^-22 m.
  * A split's partial is rounded once when stored (fp32, 2^-24), and the merge adds the S partials in split order (S - 1 additions),
    then bias and old: S + 2 more fp32 roundings of at most 2^-24 m each.  16 (S + 1) 2^-22 >= (S + 2) 2^-24 covers them with room
    for a tile boundary's alignment.
So |c_fp32 - r| <= b = (K + 16 (S + 1)) (2^-22 m + 2^-126), the last term for underflow.  Stored in bf16 (round to nearest even): |got - r| <= b + 2^-8 (|r| + b) + 2^-134.

GroupNorm and resize read bf16 values and compute exactly what their fp32 twins compute, so trainref_r's fp32 bound on the bf16
inputs holds for the fp32 value, and a bf16 store widens it as trainref_bf16.widen does.

Defects (`defect=`) the GPU test injects into the reference, each of which must exceed the bound:
    drop_k16        one k16 step (the first 16 k of the first segment; wgrad: image 0's first 16 pixels) left out of the sum
    truncated_w     the weights truncated to bf16 (low 16 bits cleared) instead of rounded to nearest even
    shifted_tap     (resize adjoint) the taps read one source pixel over
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from tests import trainref_r as R
from tests.trainref_bf16 import TINY_BF16, U_BF16, round_bf16, truncate_bf16, widen

U_TC = 2.0 ** -22


def _d(t):
    return torch.as_tensor(t).detach().to(torch.float64)


def gemm_bound(m: torch.Tensor, K: int, splits: int) -> torch.Tensor:
    """(K + 16 (splits + 1)) (2^-22 m + 2^-126): the fp32 result of a tensor-core GEMM element of magnitude m (module docstring); the
    2^-126 per step covers fp32 underflow, and keeps the bound positive where every product is zero (taps outside the plane)."""
    return (K + 16 * (splits + 1)) * (U_TC * m + R.TINY)


def store(ref: torch.Tensor, bound: torch.Tensor, bf16_out: bool):
    """(ref, bound) of an output stored in bf16 (widened by the store's rounding) or fp32 (unchanged)."""
    return (ref, widen(ref, bound)) if bf16_out else (ref, bound)


def weights(w: torch.Tensor, defect=None) -> torch.Tensor:
    """The weights the GEMM reads: fp32 parameters rounded to nearest-even bf16 (truncated under the `truncated_w` defect)."""
    return truncate_bf16(w) if defect == "truncated_w" else round_bf16(w)


def _conv(x, w, dil):
    k = w.shape[2]
    return F.conv2d(x, w, padding=dil if k == 3 else 0, dilation=dil)


def _convT(dy, w, dil):
    k = w.shape[2]
    return F.conv_transpose2d(dy, w, padding=dil if k == 3 else 0, dilation=dil)


def _drop_first_k16(w: torch.Tensor, dgrad: bool) -> torch.Tensor:
    """w [cout, cin, k, k] with the products of k indices 0..15 removed: fwd k = (ci, t), dgrad k = (co, t)."""
    w = w.clone()
    if dgrad:
        f = w.permute(0, 2, 3, 1).reshape(-1, w.shape[1])          # rows (co, t)
        f[:16] = 0
        return f.reshape(w.shape[0], w.shape[2], w.shape[3], w.shape[1]).permute(0, 3, 1, 2).contiguous()
    f = w.reshape(w.shape[0], -1)                                  # columns (ci, t)
    f[:, :16] = 0
    return f.reshape(w.shape)


def conv_fwd(segs, bias=None, old=None, splits=1, bf16_out=True, defect=None):
    """segs = [(x [N, cin, H, W] bf16 values, w [cout, cin, k, k] fp32 parameter, dil)]: bias + sum_s conv(x_s, rn_bf16(w_s)) (+ old)."""
    ws = [_d(weights(w, defect)) for _, w, _ in segs]
    if defect == "drop_k16":
        ws[0] = _drop_first_k16(ws[0], dgrad=False)
    xs = [_d(x) for x, _, _ in segs]
    dils = [dl for _, _, dl in segs]
    ref = sum(_conv(x, w, dl) for x, w, dl in zip(xs, ws, dils))
    m = sum(_conv(x.abs(), w.abs(), dl) for x, w, dl in zip(xs, ws, dils))
    K = sum(w.shape[1] * w.shape[2] * w.shape[3] for w in ws)
    if bias is not None:
        ref = ref + _d(bias).view(1, -1, 1, 1)
        m = m + _d(bias).abs().view(1, -1, 1, 1)
    if old is not None:
        ref, m = ref + _d(old), m + _d(old).abs()
    return store(ref, gemm_bound(m, K, splits), bf16_out)


def conv_dgrad(segs, old=None, splits=1, bf16_out=True, defect=None):
    """segs = [(dy [N, cout, H, W] bf16 values, w [cout, cin, k, k] fp32 parameter, dil)]: the gradient of sum_s conv(x, rn_bf16(w_s))."""
    ws = [_d(weights(w, defect)) for _, w, _ in segs]
    if defect == "drop_k16":
        ws[0] = _drop_first_k16(ws[0], dgrad=True)
    dys = [_d(dy) for dy, _, _ in segs]
    dils = [dl for _, _, dl in segs]
    ref = sum(_convT(dy, w, dl) for dy, w, dl in zip(dys, ws, dils))
    m = sum(_convT(dy.abs(), w.abs(), dl) for dy, w, dl in zip(dys, ws, dils))
    K = sum(w.shape[0] * w.shape[2] * w.shape[3] for w in ws)
    if old is not None:
        ref, m = ref + _d(old), m + _d(old).abs()
    return store(ref, gemm_bound(m, K, splits), bf16_out)


def conv_wgrad(x, dy, wshape, dil, old=None, splits=1, defect=None):
    """Weight gradient (fp32) of conv(x, w) [cout, cin, k, k] at output gradient dy, both bf16 values."""
    x, dy = _d(x), _d(dy)
    if defect == "drop_k16":
        dy = dy.clone()
        dy[0].reshape(dy.shape[1], -1)[:, :16] = 0
    k = wshape[2]
    pad = dil if k == 3 else 0
    ref = torch.nn.grad.conv2d_weight(x, wshape, dy, padding=pad, dilation=dil)
    m = torch.nn.grad.conv2d_weight(x.abs(), wshape, dy.abs(), padding=pad, dilation=dil)
    if old is not None:
        ref, m = ref + _d(old), m + _d(old).abs()
    K = x.shape[0] * x.shape[2] * x.shape[3]
    return ref, gemm_bound(m, K, splits)


def gn_prelu_fwd(z, G, gamma, beta, a, eps=1e-5, defect=None):
    """y (bf16) of GroupNorm + PReLU on bf16 z: trainref_r's bound, widened by the store."""
    return store(*R.gn_prelu_fwd(z, G, gamma, beta, a, eps, defect), True)


def gn_prelu_bwd(z, dy, G, gamma, beta, a, eps=1e-5, defect=None):
    """(dz bf16, dgamma, dbeta, dslope fp32) on bf16 z and dy."""
    dz, dg, db, da = R.gn_prelu_bwd(z, dy, G, gamma, beta, a, eps, defect)
    return store(*dz, True), dg, db, da


def resize_fwd(src, Hd, Wd, old=None):
    """bf16 -> bf16 resize (an accumulate adds the bf16 old value once in fp32)."""
    return store(*R.resize_fwd(src, Hd, Wd, old), True)


def resize_bwd(dout, Hs, Ws, defect=None):
    return store(*R.resize_bwd(dout, Hs, Ws, defect), True)


__all__ = ["U_TC", "U_BF16", "TINY_BF16", "gemm_bound", "store", "weights", "round_bf16", "truncate_bf16", "conv_fwd", "conv_dgrad",
           "conv_wgrad", "gn_prelu_fwd", "gn_prelu_bwd", "resize_fwd", "resize_bwd"]
