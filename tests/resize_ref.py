"""Float64 reference and per-element error bound of a CSNET_OP_RESIZE op (include/csnet_b200.h), for the tests.

The reference is F.interpolate(size=(H, W), mode='bilinear', align_corners=False) in float64, which computes the scale as
in / out and the taps in float64.  The kernel computes them in fp32 (scale = (float)in / out, source index
max(scale * (d + 0.5) - 0.5, 0)), so its source index is off by at most 3 2^-24 n_in per axis; bilinear interpolation is
continuous in the source index with slope at most 2 M (M = max |x| of the source plane), which bounds that error by
6 2^-24 n_in M per axis.  The fp32 blend of the four taps adds at most 8 2^-24 M.  An accumulate adds one fp32 rounding of
|old + v|, the store the destination type's rounding and half its smallest subnormal:
    bound = 2^-24 M (6 (Hs + Ws + 2) + 8) + [accumulate] 2^-24 |ref| + u_dst |ref| + subnormal_dst / 2 + 4 2^-126
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from sod100k_b200 import ir

U = {ir.F32: 2.0 ** -24, ir.F16: 2.0 ** -11, ir.BF16: 2.0 ** -8}
HALF_SUBNORMAL = {ir.F32: 2.0 ** -150, ir.F16: 2.0 ** -25, ir.BF16: 2.0 ** -134}


def resize64(src, H: int, W: int, old=None, dst_dtype: int = ir.F32):
    """(ref, bound) of resizing float64 src [N, C, Hs, Ws] to (H, W), added to `old` (same shape as the result) when given."""
    src = torch.as_tensor(src, dtype=torch.float64)
    Hs, Ws = src.shape[2], src.shape[3]
    v = F.interpolate(src, size=(H, W), mode="bilinear", align_corners=False)
    M = src.abs().amax(dim=(2, 3), keepdim=True)
    bound = 2.0 ** -24 * M * (6 * (Hs + Ws + 2) + 8) + 4 * 2.0 ** -126
    if old is not None:
        v = torch.as_tensor(old, dtype=torch.float64) + v
        bound = bound + 2.0 ** -24 * v.abs()
    bound = bound + U[dst_dtype] * v.abs() + HALF_SUBNORMAL[dst_dtype]
    return v, bound.expand_as(v).clone()


def resize_op_ref(prog: ir.Program, k: int, inputs, old):
    """{dst tensor id: (ref, bound)} of RESIZE op k: `inputs[src id]` = the source the kernel read, `old` = the destination before
    the op (read only when the op accumulates).  Channels outside the op's slice are not part of the result."""
    op = prog.ops[k]
    assert op.kind == ir.OP_RESIZE
    q, D = op.paths[0], prog.tensors[op.dst]
    src = torch.as_tensor(inputs[q.src], dtype=torch.float64)[:, q.c0:q.c0 + q.cin]
    prev = torch.as_tensor(old, dtype=torch.float64)[:, q.cout0:q.cout0 + q.cout] if op.ext_off[0] == 1 else None
    return {op.dst: resize64(src, D.H, D.W, prev, D.dtype)}
