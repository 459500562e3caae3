"""`model.csnet` — the reference's module surface on the CUDA engine.

Same class names, constructor arguments, parameter names, buffers and `state_dict()` keys as
/root/reference/CSNet/model/csnet.py (SURVEY.md §8b), so `test.py` / `train.py` / checkpoints work
unchanged — but the modules here are PARAMETER CONTAINERS: `CSNet.forward` lowers the whole network to one
program of fused sm_90a kernels (sod100k_b200/compiler.py -> libcsnet_b200.so) instead of calling
torch.nn.functional per layer.  There is no torch/cuDNN fallback: without the library or a GPU it raises.

Construction order and initialisers follow the reference (conv weights `kaiming_uniform_(a=sqrt(5))`,
default BatchNorm2d / PReLU), so the same `torch.manual_seed` yields the same initial parameters.
"""
from __future__ import annotations

import math
import os
import pickle
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn
from torch.nn import init

try:
    from .. import modular, splits
    from ..engine import ModelEngine
except ImportError:      # imported as the top-level package `model` (dropped under the reference's scripts, INTEGRATION.md)
    from sod100k_b200 import modular, splits
    from sod100k_b200.engine import ModelEngine
from .conv2d import Conv2dX100

__all__ = ["CSNet", "ILBlock", "gOctaveConv", "gOctaveCBR", "SimplifiedGOctConvBR", "CSFHead", "PallMSBlock",
           "MSBlock", "Conv2dX100", "build_model", "init_layers", "load_layer_config", "save_layer_config"]


def _module_list(mods):
    ml = nn.ModuleList()
    for m in mods:
        ml.append(m)          # None entries keep the reference's indices (pruned branches / dilations)
    return ml


class gOctaveConv(nn.Module):
    """One weight [out_total, in_total, k, k] shared by all (in-branch, out-branch) paths; branch slices are
    `int(round(C * cumulative_alpha))` (reference csnet.py:604-726)."""

    def __init__(self, in_channels, out_channels, kernel_size, alpha_in=(0.5, 0.5), alpha_out=(0.5, 0.5), stride=1,
                 padding=1, dilation=1, groups=1, bias=False, up_kwargs=None):
        super().__init__()
        if bias or groups != 1 or dilation != 1:
            raise NotImplementedError("CSNet uses gOctaveConv with bias=False, groups=1, dilation=1")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.stride, self.padding, self.dilation, self.groups = stride, padding, dilation, groups
        self.kernel_size = tuple(kernel_size)
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels, *self.kernel_size))
        self.register_parameter("bias", None)
        self.h2g_pool = nn.AvgPool2d(kernel_size=(2, 2), stride=2)   # kept: part of the reference's module tree
        self.alpha_in = splits.cumulative(alpha_in)
        self.alpha_out = splits.cumulative(alpha_out)
        self.inbranch, self.outbranch = len(alpha_in), len(alpha_out)
        init.kaiming_uniform_(self.weight, a=math.sqrt(5))

    def forward(self, xset):
        return modular.goct_conv_forward(self, xset)


class gOctaveCBR(nn.Module):
    """gOctConv + per-branch BatchNorm2d + PReLU (reference csnet.py:729-792)."""

    def __init__(self, in_channels, out_channels, kernel_size=(3, 3), alpha_in=(0.5, 0.5), alpha_out=(0.5, 0.5),
                 stride=1, padding=1, dilation=1, groups=1, bias=False, up_kwargs=None, norm_layer=nn.BatchNorm2d):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding = tuple(kernel_size), stride, padding
        self.std_conv = len(alpha_in) == 1 and len(alpha_out) == 1
        if self.std_conv:
            self.conv = Conv2dX100(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)
        else:
            self.conv = gOctaveConv(in_channels, out_channels, kernel_size, alpha_in, alpha_out, stride, padding,
                                    dilation, groups, bias)
        w = splits.widths(out_channels, alpha_out)
        self.bns = _module_list([norm_layer(c) if c != 0 else None for c in w])
        self.prelus = _module_list([nn.PReLU(c) if c != 0 else None for c in w])
        self.outbranch = len(alpha_out)
        self.alpha_in, self.alpha_out = list(alpha_in), list(alpha_out)
        self.all_flops, self.baseflop, self.expandflop = 0, None, None

    def forward(self, xset):
        return modular.goct_cbr_forward(self, xset)


class SimplifiedGOctConvBR(nn.Module):
    """Per-branch depthwise 3x3 (Conv2dX100, groups=C) + BatchNorm2d + PReLU (reference csnet.py:795-851)."""

    def __init__(self, in_channels, out_channels, kernel_size=(3, 3), alpha=(0.5, 0.5), stride=1, padding=1,
                 dilation=1, groups=1, bias=False, norm_layer=nn.BatchNorm2d):
        super().__init__()
        self.std_conv = False
        convs, bns, prelus = [], [], []
        for a in alpha:
            cin, cout = int(round(in_channels * a)), int(round(out_channels * a))
            if cin >= 1:
                convs.append(Conv2dX100(cin, cout, kernel_size=(3, 3), groups=cout, padding=padding,
                                        dilation=dilation, bias=bias))
                bns.append(norm_layer(cout))
                prelus.append(nn.PReLU(cout))
            else:
                convs.append(None), bns.append(None), prelus.append(None)
        self.convs, self.bns, self.prelus = _module_list(convs), _module_list(bns), _module_list(prelus)
        self.outbranch = len(alpha)
        self.all_flops, self.baseflop, self.expandflop = 0, None, None

    def forward(self, xset):
        return modular.dw_cbr_forward(self, xset)


class ILBlock(nn.Module):
    """gOctaveCBR (3x3 when `first` or stride 2, else 1x1) then two depthwise 3x3 layers
    (reference csnet.py:17-76)."""

    def __init__(self, inlist, outlist, stride=1, nextstride=1, nextoutlist=None, first=False):
        super().__init__()
        ninput, noutput = splits.total(inlist), splits.total(outlist)
        a_in, a_out = splits.alphas(inlist), splits.alphas(outlist)
        self.first, self.stride, self.nextstride, self.nextoutlist = first, stride, nextstride, nextoutlist
        k, pad = ((3, 3), 1) if (first or stride == 2) else ((1, 1), 0)
        self.conv1x1 = gOctaveCBR(ninput, noutput, kernel_size=k, padding=pad, alpha_in=a_in, alpha_out=a_out,
                                  stride=stride if k == (3, 3) else 1)
        self.conv3x3_1 = SimplifiedGOctConvBR(noutput, noutput, alpha=a_out, groups=noutput)
        self.conv3x3_2 = SimplifiedGOctConvBR(noutput, noutput, alpha=a_out, groups=noutput)
        self.all_flops, self.baseflop, self.expandflop = 0, None, None

    def forward(self, x):
        return self.conv3x3_2(self.conv3x3_1(self.conv1x1(x)))


class MSBlock(nn.Module):
    """Parallel dilated 3x3 convs (d = 1,2,4,8,16; entries pruned to 0 channels are None), concat, BN, PReLU
    (reference csnet.py:116-149)."""

    def __init__(self, in_channels, out_channels, dil_channels, dilations=splits.DILATIONS):
        super().__init__()
        self.dilations = list(dilations)
        self.real_dil_branch = len(self.dilations)
        self.msconv = _module_list([
            Conv2dX100(in_channels, int(dil_channels[i]), 3, padding=d, dilation=d, bias=False)
            if dil_channels[i] != 0 else None for i, d in enumerate(self.dilations)])
        self.bn = nn.BatchNorm2d(out_channels)
        self.prelu = nn.PReLU(out_channels)

    def forward(self, x):
        return modular.ms_block_forward(self, x)


class PallMSBlock(nn.Module):
    """One MSBlock per branch (reference csnet.py:79-113)."""

    def __init__(self, in_channels, out_channels, dil_channels, alpha_in=(0.5, 0.5), alpha_out=(0.5, 0.5),
                 bias=False, norm_layer=nn.BatchNorm2d):
        super().__init__()
        self.std_conv = False
        self.convs = _module_list([
            MSBlock(int(round(in_channels * alpha_in[i])), int(round(out_channels * alpha_out[i])), dil_channels[i])
            if max(dil_channels[i]) != 0 else None for i in range(len(alpha_in))])
        self.outbranch = len(alpha_in)

    def forward(self, xset):
        if isinstance(xset, torch.Tensor):
            xset = [xset]
        return [self.convs[i](xset[i]) if self.convs[i] is not None else None for i in range(self.outbranch)]


class CSFHead(nn.Module):
    """Cross-Stage-Fusion head: fuse (3->3 gOctaveCBR 1x1) -> PallMSBlock -> fuse1x1 (3->1)
    (reference csnet.py:152-206)."""

    def __init__(self, fuse_layer_config):
        super().__init__()
        self.layer_config = fuse_layer_config
        c_in, c_mid, c_out = fuse_layer_config
        n_in, n_mid_in, n_mid_out = splits.total(c_in[0]), splits.total(c_mid[0]), splits.total(c_mid[1])
        a_in, a_mid_in, a_mid_out = splits.alphas(c_in[0]), splits.alphas(c_mid[0]), splits.alphas(c_mid[1])
        self.fuse = gOctaveCBR(n_in, n_mid_in, kernel_size=(1, 1), padding=0, alpha_in=a_in, alpha_out=a_mid_in)
        self.ms = PallMSBlock(n_mid_in, n_mid_out, alpha_in=a_mid_in, alpha_out=a_mid_out, dil_channels=c_mid[2])
        self.fuse1x1 = gOctaveCBR(n_mid_out, splits.total(c_out[1]), kernel_size=(1, 1), padding=0,
                                  alpha_in=a_mid_out, alpha_out=[1])

    def forward(self, xset):
        return self.fuse1x1(self.ms(self.fuse(xset)))


class CSNet(nn.Module):
    """Reference csnet.py:209-387.  `forward` runs the fused engine program."""

    def __init__(self, layer_config, num_classes=1):
        super().__init__()
        self.stages = layer_config[-1]
        self.layer_config = layer_config
        walk, idx = splits.block_walk(layer_config)
        n_stage = [1] + [int(s) for s in self.stages]
        for s in range(5):
            setattr(self, f"stage{s}", nn.ModuleList())
        for prefix, ci, stride, first in walk:
            s, k = (int(v) for v in prefix[5:].split("."))
            last = k == n_stage[s] - 1
            nxt = layer_config[ci + 1][1] if (s < 4 or k == 0) and ci + 1 < idx else None
            blk = ILBlock(np.array([3]) if first else layer_config[ci][0], layer_config[ci][1], stride=stride,
                          nextstride=2 if (last and 0 < s < 4) else 1, nextoutlist=nxt, first=first)
            getattr(self, f"stage{s}").append(blk)
        self.oct_fuse = CSFHead(layer_config[idx:idx + 3])
        self.cls_layer = nn.Conv2d(splits.total(layer_config[-2][1]), num_classes, kernel_size=1)
        self.all_flops = 0
        self.batchsize = 0
        self._engine = None

    # ---- engine -------------------------------------------------------------------------------------
    def engine(self):
        if self._engine is None:
            object.__setattr__(self, "_engine", ModelEngine(self))
        return self._engine

    def invalidate(self):
        """Tell the engine that parameters / buffers were modified in a way it cannot observe (it already notices in-place
        torch ops, `.data` writes — by a device-side value checksum — and load_state_dict); needed only after `freeze()`."""
        if self._engine is not None:
            self._engine.invalidate()

    # The engine holds ctypes handles (device plans): a copy / pickle of the module must not carry them.  The reference module
    # supports copy.deepcopy (EMA / AveragedModel) and torch.save(model); so does this one — the copy builds its own plans.
    def __getstate__(self):
        d = dict(self.__dict__)
        d["_engine"] = None
        return d

    def __deepcopy__(self, memo):
        import copy

        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k == "_engine" else copy.deepcopy(v, memo)
        return new

    def set_precision(self, dtype: str):
        """Activation storage type of the fused inference program: 'fp32' (default, 1e-3 parity gate),
        'fp16' or 'bf16' (fp32 accumulation)."""
        self.engine().set_precision(dtype)
        return self

    def forward(self, x):
        return self.engine().forward(x)

    # ---- reference bookkeeping surface (csnet.py:313-363) --------------------------------------------
    def set_batchsize(self, batchsize):
        self.batchsize = batchsize

    def clear_flops(self):
        self.all_flops = 0
        for m in self.modules():
            if isinstance(m, ILBlock):
                m.conv1x1.all_flops = m.conv3x3_1.all_flops = m.conv3x3_2.all_flops = 0

    def get_flops(self):
        for m in self.modules():
            if isinstance(m, ILBlock):
                self.all_flops = m.conv1x1.all_flops + m.conv3x3_1.all_flops + m.conv3x3_2.all_flops + self.all_flops
        return self.all_flops / self.batchsize

    def flops_hook(self, expandflop=2):
        """Record the dynamic-weight-decay coefficients (reference :332-355); the engine's training path
        accumulates the regulariser itself, so no torch forward hooks are registered."""
        base = expandflop ** (len(self.stages) - 1)
        real = [int(s) for s in self.stages]
        real[0] += 1
        stage = in_stage = 0
        for m in self.modules():
            if isinstance(m, ILBlock):
                for sub in (m.conv1x1, m.conv3x3_1, m.conv3x3_2):
                    sub.baseflop, sub.expandflop = base, expandflop
                in_stage += 1
                if in_stage == real[stage]:
                    base /= expandflop
                    stage += 1
                    in_stage = 0
        self.flops_enabled = True

    def updateWeight(self, s=0.001):
        for m in self.modules():
            if isinstance(m, gOctaveCBR):
                for n in m.modules():
                    if isinstance(n, (nn.BatchNorm2d, nn.SyncBatchNorm)) and n.weight.grad is not None:
                        n.weight.grad.data.add_(s * torch.sign(n.weight.data))


# ---- layer_config helpers (reference csnet.py:414-597) ------------------------------------------------
def init_layers(basewidth, basic_split=(1,)):
    """Un-pruned layer_config: stage widths basewidth x (1,2,4,4) split by `basic_split`, last block of
    stages 2-4 single-branch, CSF head widths side//3 with an even 5-way dilation split."""
    bs = np.array([float(v) for v in basic_split])
    one = np.array([1.0])
    stages = [3, 4, 6, 4]
    w = {1: basewidth, 2: basewidth * 2, 3: basewidth * 4, 4: basewidth * 4}
    cfg = [[np.array([3]), w[1] * bs]] + [[w[1] * bs, w[1] * bs] for _ in range(stages[0])]
    for s in (2, 3, 4):
        cfg.append([w[s - 1] * (bs if s == 2 else one), w[s] * bs])
        cfg += [[w[s] * bs, w[s] * bs] for _ in range(stages[s - 1] - 2)]
        cfg.append([w[s] * bs, w[s] * one])
    mid = np.array([w[2] // 3, w[3] // 3, w[4] // 3])
    dil = [[b // 5] * 4 + [b - (b // 5) * 4] for b in mid]
    cfg += [[np.array([w[2], w[3], w[4]]), mid.copy()], [mid.copy(), mid.copy(), np.array(dil)],
            [mid.copy(), np.array([int(mid.sum())])]]
    for c in cfg:
        c[0], c[1] = np.round(c[0]).astype(np.int32), np.round(c[1]).astype(np.int32)
    cfg.append(stages)
    return cfg


def load_layer_config(predefine):
    with open(predefine, "rb") as f:
        return pickle.load(f)


def save_layer_config(layer_config, save_path, epoch, latest=False, finetune=False):
    os.makedirs(save_path, exist_ok=True)
    name = f"layer_config_finetune_{epoch}.bin" if finetune else f"layer_config_{epoch}.bin"
    targets = [name] + (["layer_config_latest.bin"] if latest and not finetune else [])
    for t in targets:
        with open(os.path.join(save_path, t), "wb") as f:
            pickle.dump(layer_config, f)
    print("Saved in:", os.path.join(save_path, name))


def build_model(epoch=0, predefine="", basic_split=(1,), save_path="tmp", model=None, expand=1.0, load_weight="NO",
                finetune_thres="1e-20", finetune=False):
    """Reference build_model (CSNet/model/csnet.py:571-597; the training variant CSNet_training/model/csnet.py:885-948 adds the
    slimming arguments): load the pruned layer_config pickle if `predefine` exists, else the un-pruned config of base width 20
    (x expand when > 1).  finetune=True slims `model` against the config in `predefine`: BatchNorm channels with
    |gamma| < finetune_thres are dropped (`slim.finetune_config`, on the model's device), the new config is saved like the reference
    saves it, and with load_weight='FINETUNE' (epoch != 0) the surviving weights are gather-copied into the new model
    (`slim.build_model_with_weight`); otherwise the new model is freshly initialised."""
    width = int(round(20 * expand)) if expand > 1 else 20
    masks = None
    if finetune:
        from .. import slim

        layer_config, masks = slim.finetune_config(model, load_layer_config(predefine), finetune_thres)
        save_layer_config(layer_config, save_path, epoch, finetune=True)
    elif os.path.isfile(predefine):
        layer_config = load_layer_config(predefine)
    elif epoch == 0:
        layer_config = init_layers(width, basic_split)
    else:
        raise NotImplementedError("epoch != 0 without predefine / finetune: the reference calls redefine_model here (CSNet_training/model/csnet.py:918), "
                                  "a function it defines nowhere; pass predefine= or finetune=True")
    if masks is None or load_weight == "NO":
        return CSNet(layer_config=layer_config)
    if load_weight == "FINETUNE" and epoch != 0:
        from .. import slim

        return slim.build_model_with_weight(layer_config, model, masks)
    raise ValueError(f"load_weight={load_weight!r} with epoch={epoch}: the reference leaves the new model undefined here")
