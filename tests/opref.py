"""Float64 reference and per-element error bound of one program op (include/csnet_b200.h).

`opref(prog, k, inputs)` evaluates op k of `prog` on its stored inputs (`inputs[tensor id]` = [N, C, H, W] arrays, the values
the kernel read) in torch float64 on the CPU and returns {destination tensor id: (ref, bound)}.  It is written from the IR
semantics only: the header's path / op descriptions, the comments of generic_ops.cuh and the ILBLOCK `ext_off` layout.  It
shares no code with the compiler, the host emulation or the kernels, so a kernel is checked against an independent
statement of what it must compute:  |got - ref| <= bound  on every element.

The bound is propagated element by element next to the reference.  Every intermediate carries three arrays: its value v, a
magnitude m >= |v| (the same linear maps applied to |w| and |a|), and an error bound b.
  * Linear stage z = sum w a + bias (n accumulated terms):
        b_z = sum |w| b_a + (u_w + n 2^-24) (sum |w| m_a + |bias|) + e_w sum m_a
    u_w is the unit roundoff of the op's 16-bit operand type (2^-11 fp16, 2^-8 bf16, 2^-24 for all-fp32 ops), for a kernel
    that rounds fp32 blob weights to 16 bits; it is 0 for the ILBLOCK GEMM weights, which the blob already holds as 16-bit
    values.  e_w is half the smallest subnormal of that type (a tiny weight may round to a subnormal or to zero, where
    the relative rule does not hold).  n counts the products, the resample-adds, the bias and the PReLU product.  The
    fp32 arithmetic adds n 2^-126 absolute: relative error bounds do not hold below the smallest normal fp32 value.
  * A resampled operand p (bilinear, 2x2 average, max-pool, and the resample-add of a MIX op) takes the input bounds
    through the same convex weights (max-pool: the maximum of the input bounds), then adds (u_s + 2^-22) m_p + e_s:
    u_s covers a kernel that stages p in the op's 16-bit type, 2^-22 the fp32 blend arithmetic, and m_p (the convex
    map of |a|) >= |p|.  It is applied to every such operand, and to an fp32 source that a 16-bit op reads, and to
    ILBLOCK's T1 and T2, whether or not a given kernel rounds there: the bound then holds for every kernel.
  * PReLU:  b_y = max(1, |slope|) b_z.
  * Store to the destination: + u_dst |ref| + half the destination type's smallest subnormal.
  * GN: see `_gn`.

`defect` applies one deliberate mistake to the reference (tests/test_opref_cpu.py checks that each one is flagged).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from sod100k_b200 import ir

U = {ir.F32: 2.0 ** -24, ir.F16: 2.0 ** -11, ir.BF16: 2.0 ** -8}
HALF_SUBNORMAL = {ir.F32: 2.0 ** -150, ir.F16: 2.0 ** -25, ir.BF16: 2.0 ** -134}
ARITH = 2.0 ** -22                    # fp32 blend of a bilinear / average (a few roundings relative to the convex map of |a|)
FP32_TINY = 2.0 ** -126               # absolute error of one fp32 operation near underflow (gradual or flushed to zero)
DEFECTS = ("replicate_pad", "drop_bias", "slice_shift", "align_corners", "row_above", "dil_minus_1", "max_first",
           "t1_pre_prelu")


class V:
    """An intermediate: value v, magnitude m >= |v|, error bound b (float64 tensors of one shape)."""

    def __init__(self, v, m=None, b=None):
        self.v = v
        self.m = v.abs() if m is None else m
        self.b = torch.zeros_like(v) if b is None else b

    def map(self, f, g=None):
        """The same linear (or max) map applied to the value, the magnitude and the bound (g for m and b if given)."""
        g = g or f
        return V(f(self.v), g(self.m), g(self.b))

    def staged(self, u, e):
        """Rounded to a storage type of unit roundoff u (half subnormal e): one more rounding error."""
        return V(self.v, self.m, self.b + u * self.m + e)


def _t(a):
    return a.detach().to(torch.float64) if torch.is_tensor(a) else torch.from_numpy(np.asarray(a, np.float64))


def _blob(prog, off, n):
    return torch.from_numpy(np.asarray(prog.blob[off:off + n], np.float64))


def _bits16(prog, off, n, dtype):
    """n 16-bit values (raw fp16 / bf16 bits packed two per blob word) -> float64."""
    u = np.asarray(prog.blob, np.float32).view(np.uint16)[2 * off:2 * off + n]
    if dtype == ir.F16:
        return torch.from_numpy(u.view(np.float16).astype(np.float64))
    return torch.from_numpy((u.astype(np.uint32) << 16).view(np.float32).astype(np.float64))


# ---- resampling: separable convex maps ---------------------------------------------------------------------------------
def _bilinear_matrix(n_in, up, align_corners=False):
    """[n_in * up, n_in]: bilinear up-sampling, align_corners=False, source index (d + 0.5) / up - 0.5 clamped at 0."""
    n_out = n_in * up
    M = torch.zeros(n_out, n_in, dtype=torch.float64)
    for d in range(n_out):
        if align_corners:
            s = d * (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
        else:
            s = max((d + 0.5) / up - 0.5, 0.0)
        i0 = min(int(s), n_in - 1)
        i1 = min(i0 + 1, n_in - 1)
        l = s - i0
        M[d, i0] += 1.0 - l
        M[d, i1] += l
    return M


def _avg_matrix(n_in, f):
    """[n_in / f, n_in]: the mean of the 2 samples at offset f/2 - 1 of every f-cell (2x2 mean when applied on both axes)."""
    M = torch.zeros(n_in // f, n_in, dtype=torch.float64)
    for d in range(n_in // f):
        M[d, f * d + f // 2 - 1] = 0.5
        M[d, f * d + f // 2] = 0.5
    return M


def _sep(x, Mh, Mw):
    return torch.einsum("yi,nciw,xw->ncyx", Mh, x, Mw)


def _maxpool(x, k, first=False):
    N, C, H, W = x.shape
    t = x.reshape(N, C, H // k, k, W // k, k)
    return t[:, :, :, 0, :, 0] if first else t.amax(dim=(3, 5))


def _upsample(a: V, up, u_s, e_s, defect):
    if up == 1:
        return a
    Mh = _bilinear_matrix(a.v.shape[2], up, defect == "align_corners")
    Mw = _bilinear_matrix(a.v.shape[3], up, defect == "align_corners")
    p = a.map(lambda x: _sep(x, Mh, Mw))
    return p.staged(u_s + ARITH, e_s)


def _downsample(a: V, pre_avg, pool, u_s, e_s, defect):
    """pre_avg = f: 2x2 mean at offset f/2 - 1 of every f x f cell; then max_pool2d(pool)."""
    if not pre_avg and pool == 1:
        return a
    if pre_avg:
        f = 2 if pre_avg == 1 else pre_avg
        Mh, Mw = _avg_matrix(a.v.shape[2], f), _avg_matrix(a.v.shape[3], f)
        a = a.map(lambda x: _sep(x, Mh, Mw))
        a = V(a.v, a.m, a.b + ARITH * a.m)
    if pool > 1:
        a = a.map(lambda x: _maxpool(x, pool, defect == "max_first"), lambda x: _maxpool(x, pool))
    return a.staged(u_s, e_s)


# ---- linear stages -----------------------------------------------------------------------------------------------------
class Acc:
    """Running sum of a linear stage: value, A = sum |w| m_a + |bias|, propagated bound, weight-underflow term, term count."""

    def __init__(self, shape):
        z = torch.zeros(shape, dtype=torch.float64)
        self.v, self.A, self.B, self.S, self.n = z, z.clone(), z.clone(), z.clone(), 0

    def add(self, v, A, B, S=None, n=1):
        self.v = self.v + v
        self.A = self.A + A
        self.B = self.B + B
        if S is not None:
            self.S = self.S + S
        self.n += n

    def finish(self, bias, u_w, e_w):
        """z = acc + bias as a V (bias: [C] or None)."""
        if bias is not None:
            bb = bias[None, :, None, None]
            self.v, self.A = self.v + bb, self.A + bb.abs()
            self.n += 1
        self.n += 1                                          # the PReLU product
        b = self.B + (u_w + self.n * 2.0 ** -24) * self.A + e_w * self.S + self.n * FP32_TINY
        return V(self.v, self.A, b)


def _pad(x, pad, defect):
    if pad == 0:
        return x
    return F.pad(x, (pad,) * 4, mode="replicate" if defect == "replicate_pad" else "constant")


def _conv(a: V, w, pad, dil, stride, defect, groups=1):
    """Cross-correlation (zero padding) of value, magnitude and bound; returns (value, sum |w| m, sum |w| b, sum m)."""
    cv = lambda x, ww: F.conv2d(_pad(x, pad, defect), ww, stride=stride, dilation=dil, groups=groups)
    wa = w.abs()
    return cv(a.v, w), cv(a.m, wa), cv(a.b, wa), cv(a.m, torch.ones_like(w))


def _prelu(z: V, slope):
    if slope is None:
        return z
    s = slope[None, :, None, None]
    v = torch.where(z.v > 0, z.v, s * z.v)
    return V(v, v.abs() + z.b, torch.clamp(s.abs(), min=1.0) * z.b)


def _prelu_v(x, slope):
    return torch.where(x > 0, x, slope[None, :, None, None] * x)


def _store(y: V, dtype):
    return y.v, y.b + U[dtype] * y.v.abs() + HALF_SUBNORMAL[dtype]


def _row_above(x):
    """Defect: the right-most 8-pixel group of every row (but the first) holds the row above's values."""
    x = x.clone()
    x[:, :, 1:, -8:] = x[:, :, :-1, -8:].clone()
    return x


# ---- ops ---------------------------------------------------------------------------------------------------------------
def _op_dtype(prog, op):
    """The 16-bit operand type of an op (the destination's, else the first 16-bit conv source's); F32 if there is none."""
    d = prog.tensors[op.dst].dtype
    if d != ir.F32:
        return d
    for q in op.paths:
        if q.ksize > 0 and prog.tensors[q.src].dtype != ir.F32:
            return prog.tensors[q.src].dtype
    return ir.F32


def _source(prog, op, q, inputs, ut, defect):
    """The path's channel slice as a V (an fp32 source in a 16-bit op is staged once more)."""
    x = _t(inputs[q.src])
    if defect == "row_above":
        x = _row_above(x)
    c0 = q.c0
    if defect == "slice_shift":
        c0 = c0 + 1 if c0 + q.cin < x.shape[1] else c0 - 1
    a = V(x[:, c0:c0 + q.cin])
    if prog.tensors[q.src].dtype == ir.F32 and ut != ir.F32:
        a = a.staged(U[ut], HALF_SUBNORMAL[ut])
    return a


def _mix(prog, op, inputs, defect):
    D = prog.tensors[op.dst]
    ut = _op_dtype(prog, op)
    u, e = U[ut], max(HALF_SUBNORMAL[ut], FP32_TINY)
    C = op.ext_off[2] if op.kind == ir.OP_MIXPROJ else D.C
    N = _t(inputs[op.paths[0].src]).shape[0]
    acc = Acc((N, C, D.H, D.W))
    dil_cut = max((q.dil for q in op.paths if q.ksize == 3), default=0) if defect == "dil_minus_1" else 0
    for q in op.paths:
        a = _source(prog, op, q, inputs, ut, defect)
        sl = slice(q.cout0, q.cout0 + q.cout)
        if q.ksize == 0:                                      # resample-add: out[cout0 + c] += resample(src[c0 + c])
            p = _upsample(a, q.up, u, e, defect) if q.up > 1 else _downsample(a, q.pre_avg, q.pool, u, e, defect)
            if q.up == 1 and not q.pre_avg and q.pool == 1:
                p = a
            z = torch.zeros_like(acc.v)
            zv, zm, zb = z.clone(), z.clone(), z.clone()
            zv[:, sl], zm[:, sl], zb[:, sl] = p.v, p.m, p.b
            acc.add(zv, zm, zb, n=1)
            continue
        k = q.ksize
        w = _blob(prog, q.w_off, q.cin * k * k * q.cout).reshape(q.cin, k, k, q.cout).permute(3, 0, 1, 2).contiguous()
        p = _upsample(a, q.up, u, e, defect) if q.up > 1 else _downsample(a, q.pre_avg, q.pool, u, e, defect)
        dil, pad = q.dil, q.pad
        if dil_cut and q.ksize == 3 and q.dil == dil_cut and dil > 1:
            dil, pad = dil - 1, pad - 1
        v, A, B, S = _conv(p, w, pad, dil, q.stride, defect)
        assert v.shape[2:] == (D.H, D.W), (op.name, v.shape, D)
        z = torch.zeros_like(acc.v)
        zv, zA, zB, zS = z.clone(), z.clone(), z.clone(), z.clone()
        zv[:, sl], zA[:, sl], zB[:, sl], zS[:, sl] = v, A, B, S
        acc.add(zv, zA, zB, zS, n=q.cin * k * k)
    bias = _blob(prog, op.bias_off, C) if op.bias_off >= 0 else None
    if bias is not None and defect == "drop_bias":
        bias = bias.clone()
        bias[-1] = 0.0
    slope = _blob(prog, op.slope_off, C) if op.slope_off >= 0 else None
    y = _prelu(acc.finish(bias, u, e), slope)
    if op.kind == ir.OP_MIXPROJ:                              # dst = proj_b + sum_c proj_w[c] y[c]
        y = y.staged(u, e)
        pw = _blob(prog, op.ext_off[0], C)[None, :, None, None]
        pj = Acc((N, 1, D.H, D.W))
        pj.add((pw * y.v).sum(1, keepdim=True), (pw.abs() * y.m).sum(1, keepdim=True),
               (pw.abs() * y.b).sum(1, keepdim=True), y.m.sum(1, keepdim=True), n=C)
        pb = _blob(prog, op.ext_off[1], 1) if op.ext_off[1] >= 0 else None
        y = pj.finish(pb, u, e)
    return {op.dst: _store(y, D.dtype)}


def _dw_stage(a: V, w, bias, slope, u, e, defect):
    """prelu(dw3x3(a) + bias): w [C][9] fp32."""
    C = w.shape[0]
    v, A, B, S = _conv(a, w.reshape(C, 1, 3, 3), 1, 1, 1, defect, groups=C)
    acc = Acc(v.shape)
    acc.add(v, A, B, S, n=9)
    return _prelu(acc.finish(bias, u, e), slope)


def _dw(prog, op, inputs, defect):
    D = prog.tensors[op.dst]
    q = op.paths[0]
    ut = D.dtype if D.dtype != ir.F32 else prog.tensors[q.src].dtype
    u, e = U[ut], max(HALF_SUBNORMAL[ut], FP32_TINY)
    a = _source(prog, op, q, inputs, ut, defect if defect != "slice_shift" else None)
    bias = _blob(prog, op.bias_off, D.C) if op.bias_off >= 0 else None
    if bias is not None and defect == "drop_bias":
        bias = bias.clone()
        bias[-1] = 0.0
    slope = _blob(prog, op.slope_off, D.C) if op.slope_off >= 0 else None
    y = _dw_stage(a, _blob(prog, q.w_off, D.C * 9).reshape(D.C, 9), bias, slope, u, e, defect)
    return {op.dst: _store(y, D.dtype)}


def _ilblock(prog, op, inputs, defect):
    """ILBlock (1x1 or stem form): GEMMs with the blob's 16-bit weights, bias + PReLU (T1), then dw1 (T2) and dw2."""
    dt = prog.tensors[op.dst].dtype
    u, e = U[dt], max(HALF_SUBNORMAL[dt], FP32_TINY)
    ext = op.ext_off
    stem = op.paths[0].ksize == 3
    Yh = prog.tensors[op.dst]
    Cho, Clo = Yh.C, (prog.tensors[op.dst2].C if op.dst2 >= 0 else 0)
    xh = _t(inputs[op.paths[0].src])
    if defect == "row_above":
        xh = _row_above(xh)
    if stem:
        Ci = xh.shape[1]
        K, K8 = Ci * 9, 32
        img = V(xh).staged(u, e)                                # the fp32 image becomes a 16-bit GEMM operand
        ops_ = {"h": img, "l": _downsample(V(xh), 0, 2, u, e, defect)}
    else:
        xl = _t(inputs[op.paths[1].src])
        if defect == "row_above":
            xl = _row_above(xl)
        Chi, Cli = xh.shape[1], xl.shape[1]
        K = Chi + Cli
        K8 = (K + 7) // 8 * 8
        up = _upsample(V(xl), 2, u, e, defect)
        pool = _downsample(V(xh), 0, 2, u, e, defect)
        cat = lambda a, b: V(torch.cat([a.v, b.v], 1), torch.cat([a.m, b.m], 1), torch.cat([a.b, b.b], 1))
        ops_ = {"h": cat(V(xh), up), "l": cat(V(xl), pool)}
    out = {}
    for br, dst, C, wo, bo, so, d1, d2 in (("h", op.dst, Cho, ext[0], ext[2], ext[3], 6, 12),
                                           ("l", op.dst2, Clo, ext[1], ext[4], ext[5], 9, 15)):
        if C <= 0:
            continue
        rows = (C + 15) // 16 * 16 if br == "h" else max((C + 15) // 16 * 16, 16)
        Wt = _bits16(prog, wo, rows * K8, dt).reshape(rows, K8)[:C, :K]
        a = ops_[br]
        if stem:
            w4 = Wt.reshape(C, Ci, 3, 3)
            v, A, B, S = _conv(a, w4, 1, 1, 1, defect)
        else:
            w4 = Wt.reshape(C, K, 1, 1)
            v, A, B, S = _conv(a, w4, 0, 1, 1, defect)
        acc = Acc(v.shape)
        acc.add(v, A, B, S, n=K)
        bias, slope = _blob(prog, bo, C), _blob(prog, so, C)
        if defect == "drop_bias":
            bias = bias.clone()
            bias[-1] = 0.0
        z = acc.finish(bias, 0.0, 0.0)                         # 16-bit weights in the blob: no weight rounding
        t1 = _prelu(z, slope).staged(u, e)
        if defect == "t1_pre_prelu":
            t1 = V(z.v, z.m, t1.b)
        dw = lambda base, x: _dw_stage(x, _blob(prog, ext[base], C * 9).reshape(C, 9), _blob(prog, ext[base + 1], C),
                                       _blob(prog, ext[base + 2], C), u, e, defect)
        t2 = dw(d1, t1).staged(u, e)
        out[dst] = _store(dw(d2, t2), dt)
    return out


def _gn(prog, op, inputs, defect):
    """GroupNorm(groups) + PReLU: y = prelu(gamma (x - mu) r + beta), r = 1 / sqrt(var + 1e-5), biased variance per
    (image, group) over n = (C / groups) H W elements.  The input values are exact (they are what the kernel read); the
    bound covers an fp32 evaluation with any summation order:
        |d mu|  <= n 2^-24 mean|x|                                     (fp32 sum of n terms, then / n)
        |d var| <= d mu^2 + (n + 3) 2^-24 var^ + 2 |d mu| mean|x - mu| (squares of x - mu^ summed in fp32)
        |d r|   <= r (|d var| / (2 (var + eps - |d var|)) + 2^-22)     (rsqrt to ~2 ulp)
        |d y|   <= |gamma| (r |d mu| + |x - mu| |d r|) + 4 2^-24 (|gamma r x| + |gamma r mu| + |beta|)
    then PReLU and the store as for the other ops."""
    D = prog.tensors[op.dst]
    q = op.paths[0]
    G = q.up
    x = _t(inputs[q.src])
    N, C, H, W = x.shape
    gamma, beta = _blob(prog, op.ext_off[0], C), _blob(prog, op.ext_off[1], C)
    if defect == "drop_bias":
        beta = beta.clone()
        beta[-1] = 0.0
    slope = _blob(prog, op.slope_off, C) if op.slope_off >= 0 else None
    xg = x.reshape(N, G, -1)
    n = xg.shape[2]
    mu = xg.mean(2, keepdim=True)
    var = ((xg - mu) ** 2).mean(2, keepdim=True)
    r = 1.0 / torch.sqrt(var + 1e-5)
    uf = 2.0 ** -24
    dmu = n * uf * xg.abs().mean(2, keepdim=True)
    dvar = dmu ** 2 + (n + 3) * uf * var + 2 * dmu * (xg - mu).abs().mean(2, keepdim=True)
    dr = r * (dvar / (2 * torch.clamp(var + 1e-5 - dvar, min=1e-30)) + 4 * uf)
    ex = lambda t: t.expand(N, G, n).reshape(N, C, H, W)
    mu_, r_, dmu_, dr_ = ex(mu), ex(r), ex(dmu), ex(dr)
    g, bt = gamma[None, :, None, None], beta[None, :, None, None]
    v = g * (x - mu_) * r_ + bt
    b = g.abs() * (r_ * dmu_ + (x - mu_).abs() * dr_) + 4 * uf * ((g * r_ * x).abs() + (g * r_ * mu_).abs() + bt.abs())
    y = _prelu(V(v, v.abs(), b), slope)
    return {op.dst: _store(y, D.dtype)}


def opref(prog: ir.Program, k: int, inputs, defect=None):
    """{destination tensor id: (ref, bound)} of op k (float64 torch tensors of the destination's [N, C, H, W] shape)."""
    assert defect is None or defect in DEFECTS, defect
    op = prog.ops[k]
    with torch.no_grad():
        if op.kind in (ir.OP_MIX, ir.OP_MIXPROJ):
            return _mix(prog, op, inputs, defect)
        if op.kind == ir.OP_DW:
            return _dw(prog, op, inputs, defect)
        if op.kind == ir.OP_ILBLOCK:
            return _ilblock(prog, op, inputs, defect)
        if op.kind == ir.OP_GN:
            return _gn(prog, op, inputs, defect)
    raise ValueError(f"op kind {op.kind}")


def check(got, ref, bound):
    """q = max |got - ref| / bound, and a description of the worst element (NaN / inf in `got` give q = inf)."""
    got = _t(got)
    err = (got - ref).abs()
    ratio = err / bound
    ratio = torch.where(torch.isfinite(got), ratio, torch.full_like(ratio, float("inf")))
    i = int(torch.argmax(ratio.reshape(-1)))
    idx = np.unravel_index(i, tuple(ratio.shape))
    q = float(ratio.reshape(-1)[i])
    return q, (f"q={q:.3g} at (n,c,y,x)={tuple(int(t) for t in idx)} of {tuple(ratio.shape)}: got {float(got[idx]):.6g} "
               f"ref {float(ref[idx]):.6g} bound {float(bound[idx]):.3g}")
