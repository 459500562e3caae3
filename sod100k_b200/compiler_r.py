"""Lower the CSF head of CSF+Res2Net (config 5) to the engine's program IR.

Mirrors `CSFNet.forward` after the backbone (/root/reference/CSF+Res2Net/networks/csf_res2net.py:253-258):
    fuse     gOctaveCBR 4 -> 4, 1x1, GroupNorm(32)   (networks/gOctConv.py:60-152)
    ms       PallMSBlock: per branch five dilated 3x3 convs, concat, GroupNorm(32), PReLU   (csf_res2net.py:190-225)
    fuse1x1  gOctaveCBR 4 -> 1 (1408 channels at 1/4 resolution)
    cls_layer + bilinear to the input size
GroupNorm statistics are per image, so nothing folds: every conv mix writes its raw sum and a CSNET_OP_GN op
normalises it.  Differences to the CSNet lowering: the down paths resize the conv INPUT bilinearly (pre_avg = 2/4/8:
for exact integer ratios `F.interpolate` to a smaller size is the mean of the centre 2x2 of every cell), the weight
parameter is called `weights`, and widths are 128...2048, so the tensor-core MIX kernel runs 80-channel output slices.
Inputs of any size: when H and W are multiples of 32 every resize is an exact integer ratio and is folded into the MIX ops'
reads (pre_avg / up paths).  At any other size the stage ratios are not integers (Res2Net-50 gives each stage ceil(h / 2)) and
the resizes run as CSNET_OP_RESIZE ops at the reference's ratios (`F.interpolate(size=...)`).
The Res2Net-50 backbone is NOT lowered: it runs on torch (cuDNN) — a library call, see DESIGN.md.
"""
from __future__ import annotations

from typing import Mapping, Sequence, Tuple

import numpy as np

from . import ir, splits
from .compiler import _np, upsample_input_side

FUSE_IN_SPLIT = [1 / 15, 2 / 15, 4 / 15, 8 / 15]       # csf_res2net.py:240
FUSE_OUT_SPLIT = [1 / 11, 2 / 11, 4 / 11, 4 / 11]      # :242
GN_GROUPS = 32


def res2net_feat_dims(H: int, W: int):
    """(h, w) of the four Res2Net-50 stage outputs for an H x W input: the stem conv and the max-pool each give ceil(n / 2), every
    later stage halves with ceil again (stride-2 3x3 convs, pad 1, and ceil_mode average pools)."""
    h, w = -(-(-(-H // 2)) // 2), -(-(-(-W // 2)) // 2)
    out = []
    for _ in range(4):
        out.append((h, w))
        h, w = -(-h // 2), -(-w // 2)
    return out


def compile_csf_head(params: Mapping[str, object], feat_dims: Sequence[Tuple[int, int, int]], H: int, W: int, dtype="fp32",
                     reuse_arena: bool = True, tensor_core=True) -> ir.Program:
    """feat_dims: (C, h, w) of the four backbone stages (externals 0..3, in the plan dtype); external 4 = fp32 logits.

    H, W both multiples of 32 (`exact`): the resizes are folded into the MIX ops.  Otherwise (gOctConv.py:97-103 resizes to
    `xset[j].shape[2:]`, csf_res2net.py:258 to the input):
      fuse.j:   each down path (i < j) is a RESIZE of feat_i to stage j in the plan dtype, read by a 1x1 conv path; the MIX
                writes fuse/raw{j} in fp32; each up path (i > j) convolves at stage i (fuse.low{i}to{j}) and is RESIZE-added to
                the raw sum in ascending i, the order of the reference's `sum(ysets[j])`
      fuse1x1:  the i = 0 conv writes fp32 fuse1x1/raw; fuse1x1.low{i} (i = 1, 2, 3) are RESIZE-added to it
      cls:      the 1x1 conv at stage 0 in fp32, then a RESIZE to (H, W) writes external 4
    GroupNorm reads the fp32 raw sums; ms is the same at every size."""
    if [tuple(d[1:]) for d in feat_dims] != res2net_feat_dims(H, W):
        raise ValueError(f"feature sizes {[tuple(d[1:]) for d in feat_dims]} are not the Res2Net-50 stage sizes "
                         f"{res2net_feat_dims(H, W)} of a {H}x{W} input")
    exact = H % 32 == 0 and W % 32 == 0
    dt = ir.DTYPE_NAMES[dtype] if isinstance(dtype, str) else int(dtype)
    raw_dt = dt if exact else ir.F32
    b = ir.Builder()
    p = lambda k: _np(params[k]).astype(np.float64)

    def conv_w(w):
        co, ci, kh, kw = w.shape
        return b.param(np.transpose(w.reshape(co, ci, kh * kw), (1, 2, 0)))

    def gn(src, prefix_gn, prefix_prelu, name):
        C_, h, w = (b.prog.tensors[src].C, b.prog.tensors[src].H, b.prog.tensors[src].W)
        dst = b.tensor(C_, h, w, dt, name=name)
        op = b.op(ir.OP_GN, dst, [ir.Path(src, C_, C_, ksize=0, up=GN_GROUPS)], slope=p(prefix_prelu + ".weight"), name=name)
        op.ext_off = [b.param(p(prefix_gn + ".weight")), b.param(p(prefix_gn + ".bias"))]
        return dst

    def resize(dst, src, C_, accumulate, name):
        """dst[:, :C_] (+)= bilinear resize of src[:, :C_] to dst's size; ext_off[0] = the accumulate flag."""
        b.op(ir.OP_RESIZE, dst, [ir.Path(src, C_, C_, ksize=0)], name=name).ext_off = [int(accumulate)]

    feats = [b.tensor(c, h, w, dt, external=i, name=f"feat{i}") for i, (c, h, w) in enumerate(feat_dims)]
    # ---- fuse -----------------------------------------------------------------------------------------------------
    Wf = p("fuse.conv.weights")
    ci, co = splits.cuts(Wf.shape[1], FUSE_IN_SPLIT), splits.cuts(Wf.shape[0], FUSE_OUT_SPLIT)
    y = []
    for j in range(4):
        cj, (_, hj, wj) = co[j + 1] - co[j], feat_dims[j]
        paths, ups = [], []
        for i in range(4):
            cin = ci[i + 1] - ci[i]
            w = Wf[co[j]:co[j + 1], ci[i]:ci[i + 1]]
            if i == j:
                paths.append(ir.Path(feats[i], cin, cj, ksize=1, w_off=conv_w(w)))
            elif i < j:                                   # resize the input down, then conv (gOctConv.py:101-103)
                if exact:
                    paths.append(ir.Path(feats[i], cin, cj, ksize=1, pre_avg=2 ** (j - i), w_off=conv_w(w)))
                else:
                    down = b.tensor(cin, hj, wj, dt, name=f"fuse/down{i}to{j}")
                    resize(down, feats[i], cin, False, f"fuse.down{i}to{j}")
                    paths.append(ir.Path(down, cin, cj, ksize=1, w_off=conv_w(w)))
            else:                                         # conv at low resolution, resize the output up (:98-100)
                low = b.tensor(cj, feat_dims[i][1], feat_dims[i][2], ir.F32, name=f"fuse/low{i}to{j}")
                b.op(ir.OP_MIX, low, [ir.Path(feats[i], cin, cj, ksize=1, w_off=conv_w(w))], name=f"fuse.low{i}to{j}")
                if exact:
                    paths.append(ir.Path(low, cj, cj, ksize=0, up=2 ** (i - j)))
                else:
                    ups.append((i, low))
        z = b.tensor(cj, hj, wj, raw_dt, name=f"fuse/raw{j}")
        b.op(ir.OP_MIX, z, paths, name=f"fuse.{j}")
        for i, low in ups:
            resize(z, low, cj, True, f"fuse.up{i}to{j}")
        y.append(gn(z, f"fuse.bns.{j}", f"fuse.prelus.{j}", f"fuse/{j}"))
        b.prog.taps[f"fuse/{j}"] = y[-1]
    # ---- ms -------------------------------------------------------------------------------------------------------
    zs = []
    for br in range(4):
        C_, h, w = b.prog.tensors[y[br]].C, b.prog.tensors[y[br]].H, b.prog.tensors[y[br]].W
        paths, c = [], 0
        for d, dil in enumerate(splits.DILATIONS):
            wd = p(f"ms.convs.{br}.msconv.{d}.weight")
            paths.append(ir.Path(y[br], C_, wd.shape[0], cout0=c, ksize=3, dil=dil, pad=dil, w_off=conv_w(wd)))
            c += wd.shape[0]
        raw = b.tensor(c, h, w, dt, name=f"ms/raw{br}")
        b.op(ir.OP_MIX, raw, paths, name=f"ms.convs.{br}")
        zs.append(gn(raw, f"ms.convs.{br}.bn", f"ms.convs.{br}.prelu", f"ms/{br}"))
        b.prog.taps[f"ms/{br}"] = zs[-1]
    # ---- fuse1x1: 4 -> 1.  Exact sizes: up paths input- or output-side by the cost model in compiler.upsample_input_side;
    # otherwise every i > 0 is convolved at its own stage and RESIZE-added --------------------------------------------
    W1 = p("fuse1x1.conv.weights")
    c1 = splits.cuts(W1.shape[1], FUSE_OUT_SPLIT)
    cout = W1.shape[0]
    paths, ups = [], []
    for i in range(4):
        cin_i, w_i = c1[i + 1] - c1[i], W1[:, c1[i]:c1[i + 1]]
        if i == 0 or (exact and dt != ir.F32 and upsample_input_side(cin_i, cout, 2 ** i)):
            paths.append(ir.Path(zs[i], cin_i, cout, ksize=1, up=2 ** i, w_off=conv_w(w_i)))
        else:                                             # wide layers: conv at the low resolution, resample the output
            low = b.tensor(cout, feat_dims[i][1], feat_dims[i][2], ir.F32, name=f"fuse1x1/low{i}")
            b.op(ir.OP_MIX, low, [ir.Path(zs[i], cin_i, cout, ksize=1, w_off=conv_w(w_i))], name=f"fuse1x1.low{i}")
            if exact:
                paths.append(ir.Path(low, cout, cout, ksize=0, up=2 ** i))
            else:
                ups.append((i, low))
    raw = b.tensor(cout, feat_dims[0][1], feat_dims[0][2], raw_dt, name="fuse1x1/raw")
    b.op(ir.OP_MIX, raw, paths, name="fuse1x1.0")
    for i, low in ups:
        resize(raw, low, cout, True, f"fuse1x1.up{i}")
    f0 = gn(raw, "fuse1x1.bns.0", "fuse1x1.prelus.0", "fuse1x1/0")
    b.prog.taps["fuse1x1/0"] = f0
    # ---- cls + final bilinear -------------------------------------------------------------------------------------
    wc = p("cls_layer.weight")
    low = b.tensor(wc.shape[0], feat_dims[0][1], feat_dims[0][2], ir.F32, name="cls/low")
    b.op(ir.OP_MIX, low, [ir.Path(f0, cout, wc.shape[0], ksize=1, w_off=conv_w(wc))], bias=p("cls_layer.bias"), name="cls_layer")
    out = b.tensor(wc.shape[0], H, W, ir.F32, external=4, name="logits")
    if exact:
        b.op(ir.OP_MIX, out, [ir.Path(low, wc.shape[0], wc.shape[0], ksize=0, up=H // feat_dims[0][1])], name="upsample")
    else:
        resize(out, low, wc.shape[0], False, "upsample")
    prog = b.finish(reuse=reuse_arena)
    for o in prog.ops:                                    # same veto convention as compiler.finalize_flags
        if o.kind == ir.OP_MIX and not (tensor_core is True or (tensor_core and any(o.name.startswith(x) for x in tensor_core))):
            o.ext_off = [-1] * 23 + [1]
    prog.input, prog.output = feats[0], out
    return prog
