"""Module-granular execution: the reference's module tree run module by module on the training primitives
(sod100k_b200/train_ops.py) — train-mode BatchNorm statistics, autograd through every piece, the dynamic-weight-decay
term of Oct_bn_hook.  Used by `CSNet.forward` whenever gradients or batch statistics are needed; eval-mode inference
goes through the fused program (engine.py) instead.

Each function mirrors one reference forward:
    goct_cbr_forward  gOctaveCBR.forward  (csnet.py:778-792, gOctaveConv.forward :664-726)
    dw_cbr_forward    SimplifiedGOctConvBR.forward (:838-851)
    ms_block_forward  MSBlock.forward (:141-149)
    csnet_forward     CSNet.forward (:365-387)
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn

from . import splits
from . import train_ops as T


def _as_list(xset):
    return [xset] if isinstance(xset, torch.Tensor) else list(xset)


def _bn_act(m_bn, m_prelu, z):
    """train mode: batch statistics (+ running-stat update); eval mode inside a graph: frozen running statistics."""
    return T.bn_prelu_train(z, m_bn, m_prelu)


def _flops_term(module, gaps, bns):
    """Oct_bn_hook (csnet.py:391-410): all_flops += 0.5 * sum_b w_b * sum(|GAP(out_b)| * gamma_b^2); gradient only via gamma."""
    if getattr(module, "baseflop", None) is None:
        return
    branches = len(gaps)
    wts, f = [], module.baseflop * (module.expandflop ** (branches - 1))
    for _ in range(branches):
        wts.append(f)
        f /= module.expandflop
    terms = [(wts[b] * gaps[b].abs() * torch.pow(bns[b].weight, 2)).sum() for b in range(branches) if gaps[b] is not None]
    val = 0.5 * sum(terms)
    if not T.RECOMPUTING:            # (a checkpointed re-run repeats the same autograd ops — it must save the same tensors — but not the side effect)
        module.all_flops = module.all_flops + val


def goct_conv_raw(conv, xs: List[Optional[torch.Tensor]], alpha_in, alpha_out, ksize: int, stride: int):
    """Pre-BN outputs of a gOctaveConv, one MixFn per output branch (+ one per up path at low resolution)."""
    W = conv.weight
    pad = 1 if ksize == 3 else 0
    ci, co = splits.cuts(W.shape[1], alpha_in), splits.cuts(W.shape[0], alpha_out)
    base = None
    for i, x in enumerate(xs):
        if x is not None:
            base = (x.shape[2] * 2 ** i // stride, x.shape[3] * 2 ** i // stride)
            break
    outs = []
    for j in range(len(alpha_out)):
        cj = co[j + 1] - co[j]
        if cj == 0:
            outs.append(None)
            continue
        tensors, paths = [], []
        for i, x in enumerate(xs):
            if x is None or ci[i] == ci[i + 1]:
                continue
            cin = ci[i + 1] - ci[i]
            w = T.pack_conv_weight(W[co[j]:co[j + 1], ci[i]:ci[i + 1]])
            if i > j:                                    # conv at low resolution, then bilinear (csnet.py:702-707)
                low = T.MixFn.apply((cj, x.shape[2] // stride, x.shape[3] // stride,
                                     [T.PathSpec(0, 1, cin, cj, pre_avg=int(stride == 2), ksize=ksize, pad=pad)]), x, w)
                tensors.append(low)
                paths.append(T.PathSpec(len(tensors) - 1, None, cj, cj, ksize=0, up=2 ** (i - j)))
            else:
                tensors += [x, w]
                paths.append(T.PathSpec(len(tensors) - 2, len(tensors) - 1, cin, cj, pre_avg=int(stride == 2),
                                        pool=2 ** (j - i), ksize=ksize, pad=pad))
        if not paths:
            outs.append(None)
            continue
        outs.append(T.MixFn.apply((cj, base[0] // 2 ** j, base[1] // 2 ** j, paths), *tensors))
    return outs


def goct_conv_forward(m, xset):
    ks = m.kernel_size[0]
    return goct_conv_raw(m, _as_list(xset), _decum(m.alpha_in), _decum(m.alpha_out), ks, m.stride)


def _decum(cum):
    return [cum[i + 1] - cum[i] for i in range(len(cum) - 1)]


def conv2d_x100_forward(m, x):
    if m.groups == m.in_channels and m.groups == m.out_channels and m.kernel_size == (3, 3) and m.dilation == (1, 1):
        return T.DwFn.apply(x, m.weight, 100.0)
    if m.groups != 1:
        raise NotImplementedError("Conv2dX100 with 1 < groups < channels is not used by CSNet")
    k, d = m.kernel_size[0], m.dilation[0]
    w = T.pack_conv_weight(m.weight, 100.0)
    ho = (x.shape[2] + 2 * m.padding[0] - d * (k - 1) - 1) // m.stride[0] + 1
    wo = (x.shape[3] + 2 * m.padding[1] - d * (k - 1) - 1) // m.stride[1] + 1
    return T.MixFn.apply((m.out_channels, ho, wo, [T.PathSpec(0, 1, m.in_channels, m.out_channels, ksize=k, dil=d,
                                                             stride=m.stride[0], pad=m.padding[0])]), x, w)


def goct_cbr_forward(m, xset):
    xs = _as_list(xset)
    if m.std_conv:
        z = [conv2d_x100_forward(m.conv, xs[0])]
    else:
        z = goct_conv_raw(m.conv, xs, m.alpha_in, m.alpha_out, m.kernel_size[0], m.stride)
    outs, gaps = [], []
    for j, zj in enumerate(z):
        if zj is None:
            outs.append(None), gaps.append(None)
            continue
        y, gap = _bn_act(m.bns[j], m.prelus[j], zj)
        outs.append(y), gaps.append(gap)
    _flops_term(m, gaps, m.bns)
    return outs


def dw_cbr_forward(m, xset):
    xs = _as_list(xset)
    outs, gaps = [], []
    for b, x in enumerate(xs):
        if x is None:
            outs.append(None), gaps.append(None)
            continue
        y, gap = _bn_act(m.bns[b], m.prelus[b], T.DwFn.apply(x, m.convs[b].weight, 100.0))
        outs.append(y), gaps.append(gap)
    _flops_term(m, gaps, m.bns)
    return outs


def ms_block_forward(m, x):
    tensors, paths, c = [x], [], 0
    for d, conv in zip(m.dilations, m.msconv):
        if conv is None:
            continue
        n = conv.out_channels
        tensors.append(T.pack_conv_weight(conv.weight, 100.0))
        paths.append(T.PathSpec(0, len(tensors) - 1, conv.in_channels, n, cout0=c, ksize=3, dil=d, pad=d))
        c += n
    z = T.MixFn.apply((c, x.shape[2], x.shape[3], paths), *tensors)
    return _bn_act(m.bn, m.prelu, z)[0]


def csnet_forward(model, x):
    """CSNet.forward (csnet.py:365-387) on the module-granular kernels.

    Activation storage (`model.train_storage`, set by Trainer(storage=...)): "fp32" (default) or "bf16".  In bf16 every
    activation a module passes on or saves for backward, and its gradient, is bf16: conv outputs, BN + PReLU outputs,
    depthwise outputs and pooled copies of bf16 sources.  The network input, the stem's max-pooled input, the 1-channel maps
    after cls_layer, the logits and the loss stay fp32, and so do parameters, their gradients and the BatchNorm statistics."""
    if not x.is_cuda:
        raise T.runtime.EngineError("CSNet (CUDA engine) needs CUDA tensors; there is no CPU path")
    if x.shape[2] % 16 or x.shape[3] % 16:
        raise ValueError(f"input size {tuple(x.shape[2:])} must be a multiple of 16")
    storage = getattr(model, "train_storage", "fp32")
    if storage not in T.STORAGES:
        raise ValueError(f"train_storage must be one of {sorted(T.STORAGES)}, got {storage!r}")
    dt = T.STORAGES[storage]
    feats, cur = {}, [x.float()]
    # recompute mode (Trainer(recompute=True) / model.recompute = True): an ILBlock keeps only its inputs; its six modules' saved tensors
    # (conv outputs, BN inputs, pooled copies) are rebuilt block by block in the backward pass — ~3.4x less activation memory for one
    # extra forward, which is what lets batch 1024 at 224 x 224 train on one 180 GB GPU in fp32 (SURVEY config c3's batch)
    ckpt = bool(getattr(model, "recompute", False)) and torch.is_grad_enabled()
    if ckpt:
        import contextlib
        from torch.utils.checkpoint import checkpoint
        ctx = lambda: (contextlib.nullcontext(), T.recomputing(dt))       # the re-run stores what the first run stored
    with T.storage(dt):
        for s in range(5):
            for blk in getattr(model, f"stage{s}"):
                cur = checkpoint(blk, cur, use_reentrant=False, context_fn=ctx) if ckpt else blk(cur)
            feats[s] = cur
        fuse = model.oct_fuse([feats[2][0], feats[3][0], feats[4][0]])
    cls = model.cls_layer
    w = T.pack_conv_weight(cls.weight)
    f0 = fuse[0]
    with T.storage(torch.float32):                      # cls_layer writes fp32: the 1-channel maps and the logits stay fp32
        low = T.MixFn.apply((cls.out_channels, f0.shape[2], f0.shape[3], [T.PathSpec(0, 1, f0.shape[1], cls.out_channels, ksize=1)]), f0, w)
        low = low + cls.bias.view(1, -1, 1, 1)
        up = x.shape[2] // f0.shape[2]
        return T.MixFn.apply((cls.out_channels, x.shape[2], x.shape[3], [T.PathSpec(0, None, cls.out_channels, cls.out_channels, ksize=0, up=up)]), low)
