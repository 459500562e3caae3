"""`model.utils.simplesum_octconv.simplesum` — parameter / FLOP summary with the reference's accounting rules
(/root/reference/CSNet/model/utils/parm_octconv_v2.py:13-234), computed ANALYTICALLY from the module tree instead of
with forward hooks: the engine's fused forward never calls the leaf modules, and the reference's hooks are never
removed (they would stay on the model for the whole `test.py` run).

Rules reproduced (batch 1, `multiply_adds=False`), quirks included so the printed numbers match the reference's own:
  * nn.Conv2d / Conv2dX100 leaf: out_elems * (k*k*cin/groups + [bias])                                   (:19-32)
  * gOctaveConv as a unit (:72-126): per (in-branch i, out-branch j) conv MACs with slices TRUNCATED
    (`int(C*alpha)`, not the forward's `round`), avg-pool 2x2 at stride 2 = in_elems*5, the max-pool of a down path
    counted with the CONV kernel size, 9 ops per interpolated element
  * BatchNorm2d: 4 per element, PReLU: 3 per element; the final F.interpolate is functional and not counted.
"""
from __future__ import annotations

import torch.nn as nn


def print_model_parm_nums(model):
    total = sum(p.numel() for p in model.parameters())
    print("  + Number of params: %.4fM" % (total / 1e6))
    return total


def _conv_leaf(m, out_shape):
    k = m.kernel_size[0] * m.kernel_size[1] * (m.in_channels / m.groups)
    return out_shape[0] * (k + (1 if m.bias is not None else 0)) * out_shape[1] * out_shape[2]


def _goct_conv(m, in_shapes):
    """in_shapes: [(C, H, W) | None]; returns (flops, out spatial sizes per out-branch) following octconv_hook."""
    flops, k = 0.0, m.weight.shape[-1]
    base = None
    for i, s in enumerate(in_shapes):
        if s is None:
            continue
        c, h, w = s
        if m.stride == 2:
            flops += c * h * w * 5
            h, w = h / 2, w / 2
        if base is None:
            base = (h * 2 ** i, w * 2 ** i)
        for j in range(m.outbranch):
            bx, ex = int(m.in_channels * m.alpha_in[i] / m.groups), int(m.in_channels * m.alpha_in[i + 1] / m.groups)
            by, ey = int(m.out_channels * m.alpha_out[j]), int(m.out_channels * m.alpha_out[j + 1])
            sf = 2 ** (i - j)
            kops = k * k * ((ex - bx) / m.groups)
            if sf > 1:
                flops += kops * (ey - by) * h * w + 9 * (ey - by) * h * sf * w * sf
            elif sf < 1:
                flops += (ex - bx) * h * sf * w * sf * k * k + kops * (ey - by) * h * sf * w * sf
            else:
                flops += kops * (ey - by) * h * w
    return flops, base


def _norm_act(bn, prelu, shape):
    n = shape[0] * shape[1] * shape[2]
    return (4 * n if isinstance(bn, (nn.BatchNorm2d, nn.SyncBatchNorm)) else 0) + (3 * n if isinstance(prelu, nn.PReLU) else 0)


def print_model_parm_flops(model, inputsize, device=-1):
    c, h, w = inputsize
    total = 0.0

    def cbr(m, shapes):
        nonlocal total
        if m.std_conv:
            ci, hi, wi = shapes[0]
            k, s, p = m.conv.kernel_size[0], m.conv.stride[0], m.conv.padding[0]
            out = [(m.conv.out_channels, (hi + 2 * p - k) // s + 1, (wi + 2 * p - k) // s + 1)]
            total += _conv_leaf(m.conv, out[0])
        else:
            f, base = _goct_conv(m.conv, shapes)
            total += f
            out = []
            for j, bn in enumerate(m.bns):
                out.append(None if bn is None else (bn.num_features, int(base[0]) >> j, int(base[1]) >> j))
        for j, o in enumerate(out):
            if o is not None:
                total += _norm_act(m.bns[j], m.prelus[j], o)
        return out

    def dwbr(m, shapes):
        nonlocal total
        for b, s in enumerate(shapes):
            if s is not None:
                total += _conv_leaf(m.convs[b], s) + _norm_act(m.bns[b], m.prelus[b], s)
        return shapes

    cur, feats = [(c, h, w)], {}
    for s in range(5):
        for blk in getattr(model, f"stage{s}"):
            cur = dwbr(blk.conv3x3_2, dwbr(blk.conv3x3_1, cbr(blk.conv1x1, cur)))
        feats[s] = cur
    head = model.oct_fuse
    y = cbr(head.fuse, [feats[2][0], feats[3][0], feats[4][0]])
    z = []
    for b, ms in enumerate(head.ms.convs):
        if ms is None:
            z.append(None)
            continue
        _, hh, ww = y[b]
        for conv in ms.msconv:
            if conv is not None:
                total += _conv_leaf(conv, (conv.out_channels, hh, ww))
        z.append((ms.bn.num_features, hh, ww))
        total += _norm_act(ms.bn, ms.prelu, z[-1])
    f = cbr(head.fuse1x1, z)
    total += _conv_leaf(model.cls_layer, (model.cls_layer.out_channels, f[0][1], f[0][2]))
    print("  + Number of FLOPs: %.4fG" % (total / 1e9))
    return total


def simplesum(model, inputsize=(3, 224, 224), device=-1):
    parms = print_model_parm_nums(model)
    flops = print_model_parm_flops(model, inputsize=inputsize, device=device)
    return parms, flops
