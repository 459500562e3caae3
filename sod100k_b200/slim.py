"""Channel slimming on the device (SURVEY §8 f4): restates `finetune_model` (CSNet_training/model/csnet.py:821-879) and
`build_model_with_weight` (:763-818, with its loaders :571-760) without the reference's O(Cout x Cin) Python loops.

    new_config, masks = finetune_config(model, base_layer_config, thres)      # |gamma| >= thres per BatchNorm channel
    slim = build_model_with_weight(new_config, model, masks)                  # gather-copy the surviving channels

The BatchNorm gammas never leave the device: the masks are device tensors, the gathers run as one `csnet_slim_gather` kernel per
tensor (include/csnet_b200.h); only the per-branch channel COUNTS come to the host (one copy), because the new module tree — and
the next `csnet_plan_create` — are sized by them.  Like the reference, running statistics are NOT carried over (the slimmed model
is fine-tuned next, CSNet_training/finetune.py).  CPU tensors take the same code with torch indexing (tests on machines without a GPU).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import runtime

# a model converted by nn.SyncBatchNorm.convert_sync_batchnorm keeps its BatchNorm names and state_dict keys: it slims the same
_BN = (nn.BatchNorm2d, nn.SyncBatchNorm)

def _gather(v: torch.Tensor, out_idx: torch.Tensor, in_idx, shape) -> torch.Tensor:
    """zeros(shape) with [len(out_idx), len(in_idx)] leading block = v[out_idx][:, in_idx] (in_idx None: all of dim 1 / a vector)."""
    v = v.detach()
    dst = torch.zeros(shape, dtype=v.dtype, device=v.device)
    no = int(out_idx.numel())
    ni = None if in_idx is None else int(in_idx.numel())
    if no > shape[0] or (ni is not None and ni > shape[1]):
        raise IndexError(f"mask keeps {no} x {ni} channels but the new tensor is {tuple(shape)}")     # the reference's loops fail here too
    if v.is_cuda and v.dtype == torch.float32:
        lib = runtime.load_library()
        src = v.contiguous()
        co = src.shape[0]
        ci = src.shape[1] if src.dim() > 1 else 1
        kk = int(np.prod(src.shape[2:])) if src.dim() > 2 else 1
        ii = in_idx if in_idx is not None else torch.arange(ci, device=v.device)
        dci = shape[1] if len(shape) > 1 else 1
        rc = lib.csnet_slim_gather(C.c_void_p(src.data_ptr()), co, ci, kk, C.c_void_p(out_idx.data_ptr()), no, C.c_void_p(ii.data_ptr()),
                                   int(ii.numel()), C.c_void_p(dst.data_ptr()), int(shape[0]), int(dci),
                                   C.c_void_p(torch.cuda.current_stream(v.device).cuda_stream))
        if rc != 0:
            raise runtime.EngineError(f"csnet_slim_gather failed ({rc}): {lib.csnet_train_last_error().decode()}")
        return dst
    g = v.index_select(0, out_idx)
    if in_idx is not None:
        g = g.index_select(1, in_idx)
        dst[:no, :ni] = g
    else:
        dst[:no] = g
    return dst


def _idx(mask_list: Sequence[torch.Tensor]) -> torch.Tensor:
    return torch.nonzero(torch.cat([m.reshape(-1) for m in mask_list])).reshape(-1)


def finetune_config(model, base_layer_config, thres):
    """(new_layer_config, masks): masks[layer] = list of bool tensors, one per output branch (csnet.py:821-879)."""
    from .model import csnet as M

    thres = float(thres)
    n = len(base_layer_config)
    stages = base_layer_config[-1]
    masks: List[List[torch.Tensor]] = []
    counts = []
    for m in model.modules():
        if not isinstance(m, (M.gOctaveCBR, M.PallMSBlock)):
            continue
        layer = len(masks)
        this_out = [int(c) for c in np.asarray(base_layer_config[layer][1]).reshape(-1)]
        gam = torch.cat([b.weight.detach().reshape(-1) for b in m.modules() if isinstance(b, _BN)])
        keep = gam.abs() >= thres                                   # reference: mask[abs(gamma) < thres] = 0
        parts = list(torch.split(keep, this_out)) if sum(this_out) == keep.numel() else None
        if parts is None:
            raise ValueError(f"layer {layer}: {keep.numel()} BatchNorm channels but the base config says {this_out}")
        masks.append(parts)
        counts.append(torch.stack([p.sum() for p in parts]))
    # the ONE device -> host copy: per-branch channel counts (+ the head's per-dilation counts below)
    head = n - 3                                                     # the PallMSBlock layer (csnet.py:866)
    dil_old = np.asarray(base_layer_config[head][2]).astype(np.int32)
    dil_counts = []
    for i, pm in enumerate(masks[head]):
        off = 0
        for j in range(dil_old.shape[1]):
            dil_counts.append(pm[off:off + int(dil_old[i][j])].sum())
            off += int(dil_old[i][j])
    flat = torch.cat([torch.cat(counts), torch.stack(dil_counts)]).cpu().numpy().astype(np.float64)
    new_cfg = [None] * n
    pos = 0
    for layer, parts in enumerate(masks):
        newsplit = flat[pos:pos + len(parts)].copy()
        pos += len(parts)
        if layer == 0:
            new_cfg[layer] = [3, newsplit]
        elif layer == n - 4:
            side4 = sum(new_cfg[layer - 1][1])
            side3 = sum(new_cfg[layer - stages[3] - 1][1])
            side2 = sum(new_cfg[layer - stages[3] - stages[2] - 1][1])
            new_cfg[layer] = [np.array([side2, side3, side4]), newsplit]
        elif layer == n - 3:
            new_cfg[layer] = [new_cfg[layer - 1][1], newsplit, None]          # the dilation split is filled in below
        else:
            new_cfg[layer] = [new_cfg[layer - 1][1], newsplit]
    new_cfg[head][2] = flat[sum(len(p) for p in masks):].reshape(dil_old.shape)
    new_cfg[-1] = stages
    return new_cfg, masks


def _load_bn(mod, name, mask, new_sd):
    if name + ".weight" not in new_sd:
        return
    idx = torch.nonzero(mask).reshape(-1)
    shape = new_sd[name + ".weight"].shape
    new_sd[name + ".weight"] = _gather(mod.weight, idx, None, shape)
    new_sd[name + ".bias"] = _gather(mod.bias, idx, None, shape)


def _load_prelu(mod, name, mask, new_sd):
    if name + ".weight" not in new_sd:
        return
    new_sd[name + ".weight"] = _gather(mod.weight, torch.nonzero(mask).reshape(-1), None, new_sd[name + ".weight"].shape)


def _load_goct_cbr(M, mod, full, this_mask, last_mask, new_sd):
    """csnet.py:571-608: the gOctaveConv weight by (out, in) masks, per-branch BN / PReLU by the branch's mask."""
    for name, m in mod.named_modules():
        if not name:
            continue
        if isinstance(m, M.gOctaveConv):
            key = f"{full}.{name}.weight"
            new_sd[key] = _gather(m.weight, _idx(this_mask), _idx(last_mask), new_sd[key].shape)
        elif isinstance(m, _BN):
            _load_bn(m, f"{full}.{name}", this_mask[int(name.split(".")[-1])], new_sd)
        elif isinstance(m, nn.PReLU):
            _load_prelu(m, f"{full}.{name}", this_mask[int(name.split(".")[-1])], new_sd)


def _load_dw_cbr(M, mod, full, this_mask, new_sd):
    """csnet.py:677-706: depthwise weights / BN / PReLU of branch k by this_mask[k]."""
    for name, m in mod.named_modules():
        if isinstance(m, M.Conv2dX100):
            key = f"{full}.{name}.weight"
            if key in new_sd:
                new_sd[key] = _gather(m.weight, torch.nonzero(this_mask[int(name.split(".")[-1])]).reshape(-1), None, new_sd[key].shape)
        elif isinstance(m, _BN):
            _load_bn(m, f"{full}.{name}", this_mask[int(name.split(".")[-1])], new_sd)
        elif isinstance(m, nn.PReLU):
            _load_prelu(m, f"{full}.{name}", this_mask[int(name.split(".")[-1])], new_sd)


def _load_pall_ms(M, mod, full, this_mask, last_mask, new_sd):
    """csnet.py:709-760: per branch k an MSBlock whose dilated convs take consecutive slices of this_mask[k]."""
    for name, m in mod.named_modules():
        if isinstance(m, M.MSBlock):
            k = int(name.split(".")[-1])
            off = 0
            in_idx = torch.nonzero(last_mask[k]).reshape(-1)
            for cname, c in m.named_modules():
                if not cname or not isinstance(c, M.Conv2dX100):
                    continue
                oc = c.weight.shape[0]
                sub = this_mask[k][off:off + oc]
                off += oc
                key = f"{full}.{name}.{cname}.weight"
                if key in new_sd:
                    new_sd[key] = _gather(c.weight, torch.nonzero(sub).reshape(-1), in_idx, new_sd[key].shape)
        elif isinstance(m, _BN):
            _load_bn(m, f"{full}.{name}", this_mask[int(name.split(".")[-2])], new_sd)
        elif isinstance(m, nn.PReLU):
            _load_prelu(m, f"{full}.{name}", this_mask[int(name.split(".")[-2])], new_sd)


def build_model_with_weight(layer_config, old_model, masks):
    """A CSNet of `layer_config` holding the surviving channels of `old_model` (csnet.py:763-818)."""
    from .model import csnet as M

    dev = next(old_model.parameters()).device
    model = M.CSNet(layer_config=layer_config).to(dev)
    new_sd = dict(model.state_dict())
    stages = layer_config[-1]
    mask_id, first_oct = 0, True
    for name, m in old_model.named_modules():
        if isinstance(m, M.ILBlock):
            for sub_name, sub in m.named_modules():
                full = f"{name}.{sub_name}"
                if isinstance(sub, M.gOctaveCBR):
                    last = [torch.ones(3, dtype=torch.bool, device=dev)] if mask_id == 0 else masks[mask_id - 1]
                    _load_goct_cbr(M, sub, full, masks[mask_id], last, new_sd)
                elif isinstance(sub, M.SimplifiedGOctConvBR):
                    _load_dw_cbr(M, sub, full, masks[mask_id], new_sd)
            mask_id += 1
        elif isinstance(m, M.CSFHead):
            for sub_name, sub in m.named_modules():
                full = f"{name}.{sub_name}"
                if isinstance(sub, M.gOctaveCBR):
                    if first_oct:                         # the head's inputs: the high branch of the last block of stages 2, 3, 4
                        last = [masks[mask_id - stages[3] - stages[2] - 1][0], masks[mask_id - stages[3] - 1][0], masks[mask_id - 1][0]]
                        first_oct = False
                    else:
                        last = masks[mask_id - 1]
                    _load_goct_cbr(M, sub, full, masks[mask_id], last, new_sd)
                    mask_id += 1
                elif isinstance(sub, M.PallMSBlock):
                    _load_pall_ms(M, sub, full, masks[mask_id], masks[mask_id - 1], new_sd)
                    mask_id += 1
        elif isinstance(m, nn.Conv2d) and name == "cls_layer":
            key = name + ".weight"
            last = masks[mask_id - 1]
            if new_sd[key].shape[0] != m.weight.shape[0]:
                raise ValueError("channels for cls must be the same.")
            new_sd[key] = _gather(m.weight, torch.arange(m.weight.shape[0], device=dev), _idx(last), new_sd[key].shape)
            if m.bias is not None:
                new_sd[name + ".bias"] = m.bias.detach().clone()
    model.load_state_dict(new_sd)
    return model
